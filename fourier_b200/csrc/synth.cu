// synth.cu -- synthetic input generator for the benchmarks and the large-size parity tests.
// Same counter hash as oracle/fourier_oracle.c (fo_hash64 / fo_fill_input_*): scalar number g of the
// whole batch (re of sample s is g = 2s, im is g = 2s+1) -> splitmix64 finaliser -> U[-1, 1).
// The mapping uses only exact operations, so CPU and GPU produce identical bits (SURVEY.md 8d).
#include "plan.h"

namespace fb200 {
namespace {

__host__ __device__ inline unsigned long long hash64(unsigned long long seed, unsigned long long counter) {
  unsigned long long z = seed + (counter + 1ull) * 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
__device__ inline float unit(unsigned long long h, float) {
  return (float)(h >> 40) * (1.0f / 8388608.0f) - 1.0f;
}
__device__ inline double unit(unsigned long long h, double) {
  return (double)(h >> 11) * (1.0 / 4503599627370496.0) - 1.0;
}

template <typename T>
__global__ void __launch_bounds__(256)
fill_kernel(T* __restrict__ out, unsigned long long first, size_t count, unsigned long long seed) {
  for (size_t g = blockIdx.x * (size_t)blockDim.x + threadIdx.x; g < count;
       g += (size_t)gridDim.x * blockDim.x)
    out[g] = unit(hash64(seed, first + g), T());
}


// ---- helpers of the distributed six-step transform (BASELINE config 5) ------------------------------------------
// Batched 2-D transpose out[b][c][r] = in[b][r][c] through a padded 32x32 shared-memory tile: both the read
// and the write are contiguous along the fastest index.
template <typename V>
__global__ void __launch_bounds__(256)
transpose_kernel(const V* __restrict__ in, V* __restrict__ out, size_t rows, size_t cols) {
  __shared__ V tile[32][33];
  const size_t b = blockIdx.z;
  const V* src = in + b * rows * cols;
  V* dst = out + b * rows * cols;
  const size_t c0 = (size_t)blockIdx.x * 32, r0 = (size_t)blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int i = ty; i < 32; i += 8)
    if (r0 + i < rows && c0 + tx < cols) tile[i][tx] = src[(r0 + i) * cols + c0 + tx];
  __syncthreads();
  for (int i = ty; i < 32; i += 8)
    if (c0 + i < cols && r0 + tx < rows) dst[(c0 + i) * rows + r0 + tx] = tile[tx][i];
}

// Pack step of a pipelined exchange: a batched transpose of column blocks of one row-major matrix with
// leading dimension ld, optionally fused with the inter-step twiddle of the six-step algorithm:
//   out[b*obs + c*rows + r] = in[b*ibs + r*ld + c] * w_N^{(row0 + r) * (col0 + b*ibs + c)}     (TW != 0)
// (b < batch, r < rows, c < cols; TW = 1 forward, 2 inverse/conjugated, 0 no twiddle).  The angle index is
// reduced exactly mod N in 64-bit integers; each thread evaluates one twiddle and one step with sincospi
// in double and walks its 4 rows (8 apart) by recurrence, so the kernel stays memory-bound.
template <typename T, int TW>
__global__ void __launch_bounds__(256)
pack_kernel(const cpx<T>* __restrict__ in, cpx<T>* __restrict__ out, size_t rows, size_t cols, size_t ld,
            size_t ibs, size_t obs, unsigned long long row0, unsigned long long col0, unsigned long long n_total) {
  using V = cpx<T>;
  __shared__ V tile[32][33];
  const size_t b = blockIdx.z;
  const V* src = in + b * ibs;
  V* dst = out + b * obs;
  const size_t c0 = (size_t)blockIdx.x * 32, r0 = (size_t)blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  double wr = 1.0, wi = 0.0, sr = 1.0, si = 0.0;
  if constexpr (TW != 0) {
    const unsigned long long cg = (col0 + b * ibs + c0 + tx) % n_total;
    // 128-bit products are not needed: row index and column index are both < 2^32 for any N <= 2^62 that is
    // split as N1*N2 with N1, N2 < 2^32 (checked by the launcher)
    const unsigned long long m0 = ((row0 + r0 + ty) % n_total) * cg % n_total, ms = 8ull * cg % n_total;
    sincospi(2.0 * (double)m0 / (double)n_total, &wi, &wr);
    sincospi(2.0 * (double)ms / (double)n_total, &si, &sr);
    if (TW == 1) { wi = -wi; si = -si; }
  }
  for (int i = ty; i < 32; i += 8) {
    if (r0 + i < rows && c0 + tx < cols) {
      V v = src[(r0 + i) * ld + c0 + tx];
      if constexpr (TW != 0) {
        const double xr = (double)v.x, xi = (double)v.y;
        v = mk<T>((T)(xr * wr - xi * wi), (T)(xr * wi + xi * wr));
      }
      tile[i][tx] = v;
    }
    if constexpr (TW != 0) {
      const double nr = wr * sr - wi * si;
      wi = wr * si + wi * sr;
      wr = nr;
    }
  }
  __syncthreads();
  for (int i = ty; i < 32; i += 8)
    if (c0 + i < cols && r0 + tx < rows) dst[(c0 + i) * rows + r0 + tx] = tile[tx][i];
}

// out[b][a][i] = in[a][b][i]: swaps the two leading axes of a 3-D array whose innermost runs (i < inner)
// stay contiguous -- the unpack step after an all-to-all (received [src rank][my row][their rows]).
template <typename V>
__global__ void __launch_bounds__(256)
swap_leading_kernel(const V* __restrict__ in, V* __restrict__ out, size_t a, size_t b, size_t inner) {
  const size_t total = a * b * inner;
  for (size_t g = blockIdx.x * (size_t)blockDim.x + threadIdx.x; g < total; g += (size_t)gridDim.x * blockDim.x) {
    const size_t i = g % inner, ab = g / inner, aa = ab % a, bb = ab / a;   // g enumerates out[bb][aa][i]
    out[g] = in[(aa * b + bb) * inner + i];
  }
}

// data[r][c] *= w_N^{(row0 + r) * c} (conjugated for the inverse direction).  The angle index is reduced
// mod N in 64-bit integers and the twiddle evaluated in double (sincospi), so it is exact to T's precision
// even for N = 2^30, where a float cannot hold the index.
template <typename T, bool FWD>
__global__ void __launch_bounds__(256)
twiddle_rows_kernel(cpx<T>* __restrict__ data, size_t rows, size_t cols, unsigned long long row0,
                    unsigned long long n_total) {
  const size_t total = rows * cols;
  for (size_t g = blockIdx.x * (size_t)blockDim.x + threadIdx.x; g < total; g += (size_t)gridDim.x * blockDim.x) {
    const size_t r = g / cols, c = g - r * cols;
    const unsigned long long m = ((row0 + r) * (unsigned long long)c) % n_total;
    double sn, cs;
    sincospi(2.0 * (double)m / (double)n_total, &sn, &cs);
    const cpx<T> w = mk<T>((T)cs, (T)(-sn));
    data[g] = ctw<FWD>(data[g], w);
  }
}

}  // namespace

template <typename T>
cudaError_t launch_transpose(const cpx<T>* in, cpx<T>* out, size_t batch, size_t rows, size_t cols, cudaStream_t s) {
  if (batch == 0 || rows == 0 || cols == 0) return cudaSuccess;
  if (batch > 65535 || (rows + 31) / 32 > 65535) return cudaErrorInvalidValue;
  dim3 grid((unsigned)((cols + 31) / 32), (unsigned)((rows + 31) / 32), (unsigned)batch);
  transpose_kernel<cpx<T>><<<grid, 256, 0, s>>>(in, out, rows, cols);
  return cudaGetLastError();
}
template <typename T>
cudaError_t launch_pack(const cpx<T>* in, cpx<T>* out, size_t batch, size_t rows, size_t cols, size_t ld, size_t ibs,
                        size_t obs, int twiddle, unsigned long long row0, unsigned long long col0,
                        unsigned long long n_total, cudaStream_t s) {
  if (batch == 0 || rows == 0 || cols == 0) return cudaSuccess;
  if (batch > 65535 || (rows + 31) / 32 > 65535 || twiddle < 0 || twiddle > 2) return cudaErrorInvalidValue;
  if (twiddle != 0 && (n_total == 0 || row0 + rows > (1ull << 32) || col0 + (batch - 1) * ibs + cols > (1ull << 32)))
    return cudaErrorInvalidValue;
  dim3 grid((unsigned)((cols + 31) / 32), (unsigned)((rows + 31) / 32), (unsigned)batch);
  if (twiddle == 0) pack_kernel<T, 0><<<grid, 256, 0, s>>>(in, out, rows, cols, ld, ibs, obs, row0, col0, n_total);
  else if (twiddle == 1) pack_kernel<T, 1><<<grid, 256, 0, s>>>(in, out, rows, cols, ld, ibs, obs, row0, col0, n_total);
  else pack_kernel<T, 2><<<grid, 256, 0, s>>>(in, out, rows, cols, ld, ibs, obs, row0, col0, n_total);
  return cudaGetLastError();
}
template cudaError_t launch_pack<float>(const cpx<float>*, cpx<float>*, size_t, size_t, size_t, size_t, size_t, size_t,
                                        int, unsigned long long, unsigned long long, unsigned long long, cudaStream_t);
template cudaError_t launch_pack<double>(const cpx<double>*, cpx<double>*, size_t, size_t, size_t, size_t, size_t, size_t,
                                         int, unsigned long long, unsigned long long, unsigned long long, cudaStream_t);
template <typename T>
cudaError_t launch_swap_leading(const cpx<T>* in, cpx<T>* out, size_t a, size_t b, size_t inner, cudaStream_t s) {
  size_t blocks = (a * b * inner + 255) / 256;
  if (blocks > 132u * 32u) blocks = 132u * 32u;
  if (blocks == 0) return cudaSuccess;
  swap_leading_kernel<cpx<T>><<<(unsigned)blocks, 256, 0, s>>>(in, out, a, b, inner);
  return cudaGetLastError();
}
template cudaError_t launch_swap_leading<float>(const cpx<float>*, cpx<float>*, size_t, size_t, size_t, cudaStream_t);
template cudaError_t launch_swap_leading<double>(const cpx<double>*, cpx<double>*, size_t, size_t, size_t, cudaStream_t);
template <typename T>
cudaError_t launch_twiddle_rows(cpx<T>* data, size_t rows, size_t cols, unsigned long long row0,
                                unsigned long long n_total, bool forward, cudaStream_t s) {
  size_t blocks = (rows * cols + 255) / 256;
  if (blocks > 132u * 32u) blocks = 132u * 32u;
  if (blocks == 0) return cudaSuccess;
  if (forward) twiddle_rows_kernel<T, true><<<(unsigned)blocks, 256, 0, s>>>(data, rows, cols, row0, n_total);
  else twiddle_rows_kernel<T, false><<<(unsigned)blocks, 256, 0, s>>>(data, rows, cols, row0, n_total);
  return cudaGetLastError();
}
template cudaError_t launch_transpose<float>(const cpx<float>*, cpx<float>*, size_t, size_t, size_t, cudaStream_t);
template cudaError_t launch_transpose<double>(const cpx<double>*, cpx<double>*, size_t, size_t, size_t, cudaStream_t);
template cudaError_t launch_twiddle_rows<float>(cpx<float>*, size_t, size_t, unsigned long long, unsigned long long, bool, cudaStream_t);
template cudaError_t launch_twiddle_rows<double>(cpx<double>*, size_t, size_t, unsigned long long, unsigned long long, bool, cudaStream_t);

template <typename T>
cudaError_t launch_fill_input(T* out, unsigned long long first_scalar, size_t count,
                              unsigned long long seed, cudaStream_t s) {
  size_t blocks = (count + 255) / 256;
  if (blocks > 132u * 16u) blocks = 132u * 16u;
  if (blocks == 0) blocks = 1;
  fill_kernel<T><<<(unsigned)blocks, 256, 0, s>>>(out, first_scalar, count, seed);
  return cudaGetLastError();
}
template cudaError_t launch_fill_input<float>(float*, unsigned long long, size_t, unsigned long long, cudaStream_t);
template cudaError_t launch_fill_input<double>(double*, unsigned long long, size_t, unsigned long long, cudaStream_t);

}  // namespace fb200
