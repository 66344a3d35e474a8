// stockham_generic.cu -- the general path: one kernel per Stockham autosort stage over HBM, plus the
// pointwise kernels of the unfused Bluestein path.
//
// This is the GPU counterpart of the reference's stage functions radix_{2,3,4,8}_{wide,narrow}
// (fourier-algorithms/src/autosort/mod.rs:174-310): same index map -- read (k*m+i)*stride+j,
// DFT_R, post-twiddle by w_S^{i*k}, write (i*R+k)*stride+j -- with the batch as an outer grid
// dimension.  It handles every {2,3}-smooth N of any size and is the fallback for sizes the
// fused kernels (onchip.cu, twopass.cu) do not cover; it streams the array once per stage, so
// it is NOT the path the headline numbers are measured on.
#include "plan.h"

namespace fb200 {

namespace {

// One thread = one radix-R butterfly.  q = i*stride + j enumerates butterflies of one transform with
// j (contiguous in memory) fastest, so loads are coalesced for every stride.
template <typename T, int R, bool FWD>
__global__ void __launch_bounds__(kThreads)
stockham_stage_kernel(const cpx<T>* __restrict__ in, cpx<T>* __restrict__ out,
                      const cpx<T>* __restrict__ wtab, size_t n, size_t sub_size, size_t stride,
                      size_t batch, bool last, T scale) {
  const size_t per = n / R;  // butterflies per transform
  const size_t total = per * batch;
  const size_t m = sub_size / R;
  for (size_t g = blockIdx.x * (size_t)blockDim.x + threadIdx.x; g < total;
       g += (size_t)gridDim.x * blockDim.x) {
    const size_t b = g / per;
    const size_t q = g - b * per;
    const size_t i = q / stride;
    const size_t j = q - i * stride;
    const cpx<T>* src = in + b * n + i * stride + j;
    cpx<T> x[R];
#pragma unroll
    for (int k = 0; k < R; ++k) x[k] = src[(size_t)k * m * stride];

    cpx<T> y[R];
    if constexpr (R == 3) {
      dft3<FWD, T>(x);
#pragma unroll
      for (int k = 0; k < R; ++k) y[k] = x[k];
    } else {
      dft_pow2<R, FWD, T>(x);
      static_for<0, R>([&](auto K) FB_LAMBDA {
        constexpr int k = decltype(K)::value;
        y[k] = x[rev<R>(k)];
      });
    }
    if (sub_size != (size_t)R) {
      // w_S^{i*k} = w_N^{i*k*stride}; i*k < S so the index stays below N
#pragma unroll
      for (int k = 1; k < R; ++k) y[k] = ctw<FWD>(y[k], wtab[i * k * stride]);
    }
    if (last) {
#pragma unroll
      for (int k = 0; k < R; ++k) y[k] = cscale(y[k], scale);
    }
    cpx<T>* dst = out + b * n + i * R * stride + j;
#pragma unroll
    for (int k = 0; k < R; ++k) dst[(size_t)k * stride] = y[k];
  }
}

template <typename T>
__global__ void __launch_bounds__(kThreads)
scale_copy_kernel(const cpx<T>* __restrict__ in, cpx<T>* __restrict__ out, size_t count, T scale) {
  for (size_t g = blockIdx.x * (size_t)blockDim.x + threadIdx.x; g < count;
       g += (size_t)gridDim.x * blockDim.x)
    out[g] = cscale(in[g], scale);
}

// Bluestein step 1+2 (bluesteins.rs:229-234): work[i] = chirp[i] * in[i] for i < n, 0 up to m.
template <typename T, bool FWD>
__global__ void __launch_bounds__(kThreads)
chirp_in_kernel(const cpx<T>* __restrict__ in, cpx<T>* __restrict__ work,
                const cpx<T>* __restrict__ chirp, size_t n, size_t m, size_t batch) {
  const size_t total = m * batch;
  for (size_t g = blockIdx.x * (size_t)blockDim.x + threadIdx.x; g < total;
       g += (size_t)gridDim.x * blockDim.x) {
    const size_t b = g / m, i = g - b * m;
    cpx<T> v = mk<T>((T)0, (T)0);
    if (i < n) v = ctw<FWD>(in[b * n + i], chirp[i]);
    work[g] = v;
  }
}

// Bluestein step 4 (bluesteins.rs:236-238): work[i] *= W[i].
template <typename T, bool FWD>
__global__ void __launch_bounds__(kThreads)
pointwise_kernel(cpx<T>* __restrict__ work, const cpx<T>* __restrict__ w, size_t m, size_t batch) {
  const size_t total = m * batch;
  for (size_t g = blockIdx.x * (size_t)blockDim.x + threadIdx.x; g < total;
       g += (size_t)gridDim.x * blockDim.x) {
    const size_t i = g % m;
    work[g] = ctw<FWD>(work[g], w[i]);  // inverse direction: W_inv = conj(W_fwd)
  }
}

// Bluestein step 6 (bluesteins.rs:240-258): out[i] = work[i] * chirp[i] * scale, i < n.
template <typename T, bool FWD>
__global__ void __launch_bounds__(kThreads)
chirp_out_kernel(const cpx<T>* __restrict__ work, cpx<T>* __restrict__ out,
                 const cpx<T>* __restrict__ chirp, size_t n, size_t m, size_t batch, T scale) {
  const size_t total = n * batch;
  for (size_t g = blockIdx.x * (size_t)blockDim.x + threadIdx.x; g < total;
       g += (size_t)gridDim.x * blockDim.x) {
    const size_t b = g / n, i = g - b * n;
    out[g] = cscale(ctw<FWD>(work[b * m + i], chirp[i]), scale);
  }
}

}  // namespace

template <typename T>
cudaError_t launch_stockham_stage(int radix, const cpx<T>* in, cpx<T>* out, const cpx<T>* wtab, size_t n,
                                  size_t sub_size, size_t stride, size_t batch, bool forward, bool last,
                                  T scale, cudaStream_t s) {
  const unsigned grid = grid_for(n / radix * batch);
#define FB_LAUNCH(R)                                                                                   \
  if (forward)                                                                                         \
    stockham_stage_kernel<T, R, true><<<grid, kThreads, 0, s>>>(in, out, wtab, n, sub_size, stride,    \
                                                                batch, last, scale);                   \
  else                                                                                                 \
    stockham_stage_kernel<T, R, false><<<grid, kThreads, 0, s>>>(in, out, wtab, n, sub_size, stride,   \
                                                                 batch, last, scale);
  switch (radix) {
    case 2: FB_LAUNCH(2) break;
    case 3: FB_LAUNCH(3) break;
    case 4: FB_LAUNCH(4) break;
    case 8: FB_LAUNCH(8) break;
    case 16: FB_LAUNCH(16) break;
    default: return cudaErrorInvalidValue;
  }
#undef FB_LAUNCH
  return cudaGetLastError();
}

template <typename T>
cudaError_t launch_scale_copy(const cpx<T>* in, cpx<T>* out, size_t count, T scale, cudaStream_t s) {
  scale_copy_kernel<T><<<grid_for(count), kThreads, 0, s>>>(in, out, count, scale);
  return cudaGetLastError();
}

template <typename T>
cudaError_t launch_chirp_in(const cpx<T>* in, cpx<T>* work, const cpx<T>* chirp, size_t n, size_t m,
                            size_t batch, bool forward, cudaStream_t s) {
  if (forward) chirp_in_kernel<T, true><<<grid_for(m * batch), kThreads, 0, s>>>(in, work, chirp, n, m, batch);
  else chirp_in_kernel<T, false><<<grid_for(m * batch), kThreads, 0, s>>>(in, work, chirp, n, m, batch);
  return cudaGetLastError();
}

template <typename T>
cudaError_t launch_pointwise(cpx<T>* work, const cpx<T>* w, size_t m, size_t batch, bool forward,
                             cudaStream_t s) {
  if (forward) pointwise_kernel<T, true><<<grid_for(m * batch), kThreads, 0, s>>>(work, w, m, batch);
  else pointwise_kernel<T, false><<<grid_for(m * batch), kThreads, 0, s>>>(work, w, m, batch);
  return cudaGetLastError();
}

template <typename T>
cudaError_t launch_chirp_out(const cpx<T>* work, cpx<T>* out, const cpx<T>* chirp, size_t n, size_t m,
                             size_t batch, bool forward, T scale, cudaStream_t s) {
  if (forward)
    chirp_out_kernel<T, true><<<grid_for(n * batch), kThreads, 0, s>>>(work, out, chirp, n, m, batch, scale);
  else
    chirp_out_kernel<T, false><<<grid_for(n * batch), kThreads, 0, s>>>(work, out, chirp, n, m, batch, scale);
  return cudaGetLastError();
}

#define FB_INST(T)                                                                                      \
  template cudaError_t launch_stockham_stage<T>(int, const cpx<T>*, cpx<T>*, const cpx<T>*, size_t,     \
                                                size_t, size_t, size_t, bool, bool, T, cudaStream_t);   \
  template cudaError_t launch_scale_copy<T>(const cpx<T>*, cpx<T>*, size_t, T, cudaStream_t);           \
  template cudaError_t launch_chirp_in<T>(const cpx<T>*, cpx<T>*, const cpx<T>*, size_t, size_t,        \
                                          size_t, bool, cudaStream_t);                                  \
  template cudaError_t launch_pointwise<T>(cpx<T>*, const cpx<T>*, size_t, size_t, bool, cudaStream_t); \
  template cudaError_t launch_chirp_out<T>(const cpx<T>*, cpx<T>*, const cpx<T>*, size_t, size_t,       \
                                           size_t, bool, T, cudaStream_t);
FB_INST(float)
FB_INST(double)
#undef FB_INST

}  // namespace fb200
