// real.cu -- real-input transforms (DESIGN.md §4.10): plan construction, path selection, and the O(N) kernels
// around the inner complex plan.
//
//   kRealFused  N = 2M, M an on-chip size class: onchip_real_kernel (onchip_kernels.cuh), one launch.
//   kRealHalf   other even N: the reals as M = N/2 complex values through a complex plan of length M, and one
//               untangle (forward) / tangle (inverse) kernel over a plan-owned scratch chunk.
//   kRealFull   odd N: widen to complex, complex plan of length N, first (N+1)/2 bins; the inverse extends the bins
//               to a Hermitian spectrum, runs the complex inverse and keeps the real parts.  Correctness path only.
// Convolution of real rows (DESIGN.md §4.11) runs on the same three paths: onchip_conv_kernel; the inner FFT,
// conv_pair_kernel and the inner inverse, in place in `out`; widen, FFT, hermitian_mul_kernel, inverse, real part.
// Linear convolution by overlap-save (DESIGN.md §4.12): onchip_lconv_kernel on the fused path; otherwise chunks of
// segments gathered into seg_, convolved there in place as above and scattered.
// Short-time Fourier transform (DESIGN.md §4.13): onchip_stft_kernel on the fused path; otherwise chunks of windowed
// frames gathered into seg_ and transformed from there by the plan's own rfft.  The inverse inverts runs of frames into
// seg_ with the plan's own irfft and overlap-adds them on every path.
// Mel spectrogram (DESIGN.md §4.14): mel_bands_kernel, then onchip_mel_kernel on the fused path; otherwise chunks of
// windowed frames gathered into seg_, their spectra by the plan's own rfft into seg_ behind them, and
// mel_spectra_kernel from there into the output rows.
// Welch power spectral density (DESIGN.md §4.15): welch_scale_kernel, then per chunk of rows onchip_welch_kernel on the
// fused path, or chunks of detrended windowed frames gathered into seg_, their spectra by the plan's own rfft behind
// them and welch_accumulate_kernel into the partials; then welch_finish_kernel unless the fused kernel wrote the rows.
// Cross-spectral density and coherence (DESIGN.md §4.17): Welch's steps on frame pairs, in the same row driver
// (welch_cross_rows): welch_scale_kernel (csd only), then per chunk of rows onchip_csd_kernel, or chunks of x frames and
// their y frames gathered into seg_ (csd_gather_kernel), their spectra by the plan's own rfft behind them and
// cross_accumulate_kernel into the partials; then cross_finish_kernel unless the fused kernel wrote the rows.
// Off the fused path, every chunk of frames above goes through one loop, frame_chunks: the gather, the plan's own rfft
// (rfft_rows) and the transform's consumer kernels.
// Discrete cosine transforms (DESIGN.md §4.16): onchip_dct_kernel on the fused path; otherwise per chunk of rows an O(N)
// kernel into seg_, the inner plan in place there and an O(N) kernel into the output: dct_permute_kernel, Fft and
// dct_untangle_kernel (type 2) or dct_tangle_kernel, UnscaledIfft and dct_unpermute_kernel (type 3) at half length;
// dct_widen_kernel, Fft and dct_post_kernel or dct_pre_kernel, UnscaledIfft and dct_unpermute_kernel at full length.
// Analytic signal and envelope (DESIGN.md §4.19): onchip_hilbert_kernel on the fused path; otherwise per chunk of rows
// through seg_: Fft of the rows read as M complex values, hilbert_pair_kernel, UnscaledIfft and hilbert_out_kernel at
// half length; widen_kernel, Fft, hilbert_mul_kernel, UnscaledIfft and hilbert_out_kernel at full length.
// Type-IV DCT and MDCT (DESIGN.md §4.20), even N only: onchip_dct4_kernel / onchip_mdct_kernel on the fused path;
// otherwise per chunk of rows or frames through seg_: dct4_pre_kernel or mdct_gather_kernel, the inner Fft in place and
// dct4_post_kernel.  The IMDCT runs the plan's own DCT-IV over runs of frames into seg_ (real::istft_runs), then
// imdct_overlap_add_kernel, on every path.
#include <algorithm>
#include <string>
#include <vector>

#include "plan.h"
#include "real_kernels.cuh"
#include "tables.cuh"  // make_twa

namespace fb200 {

namespace {

// One thread per pair (k, M-k), k <= M/2, of one row: consecutive threads read Z[k] ascending and Z[M-k] descending.
template <typename T, bool FWD>
__global__ void __launch_bounds__(kThreads)
untangle_kernel(const cpx<T>* __restrict__ in, cpx<T>* __restrict__ out, const cpx<T>* __restrict__ tab, long m,
                long batch, T h) {
  const long pairs = m / 2 + 1, total = pairs * batch;
  for (long g = blockIdx.x * (long)blockDim.x + threadIdx.x; g < total; g += (long)gridDim.x * blockDim.x) {
    const long b = g / pairs, k = g - b * pairs;
    if (FWD) real::untangle(in + b * m, out + b * (m + 1), m, k, tab, h);
    else real::tangle(in + b * (m + 1), out + b * m, m, k, tab, h);
  }
}

// One thread per pair (k, M-k), k <= M/2, of one row, in place on z (M complex values per row); row b uses spectrum
// row ((row0 + b) / per) mod rows.
template <typename T>
__global__ void __launch_bounds__(kThreads)
conv_pair_kernel(cpx<T>* __restrict__ z, const cpx<T>* __restrict__ spec, const cpx<T>* __restrict__ tab, long m,
                 long batch, long rows, long row0, long per, T h) {
  const long pairs = m / 2 + 1, total = pairs * batch;
  for (long g = blockIdx.x * (long)blockDim.x + threadIdx.x; g < total; g += (long)gridDim.x * blockDim.x) {
    const long b = g / pairs, k = g - b * pairs;
    real::conv_pair(z + b * m, spec + (((row0 + b) / per) % rows) * (m + 1), m, k, tab, h);
  }
}

template <typename T>
__global__ void __launch_bounds__(kThreads)
widen_kernel(const T* __restrict__ in, cpx<T>* __restrict__ out, size_t count) {
  for (size_t g = blockIdx.x * (size_t)blockDim.x + threadIdx.x; g < count; g += (size_t)gridDim.x * blockDim.x)
    out[g] = mk<T>(in[g], (T)0);
}

template <typename T>
__global__ void __launch_bounds__(kThreads)
copy_bins_kernel(const cpx<T>* __restrict__ y, cpx<T>* __restrict__ x, long n, long batch) {
  const long bins = n / 2 + 1, total = bins * batch;
  for (long g = blockIdx.x * (long)blockDim.x + threadIdx.x; g < total; g += (long)gridDim.x * blockDim.x) {
    const long b = g / bins, k = g - b * bins;
    real::copy_bin(y + b * n, x + b * bins, k);
  }
}

// grid.y runs over rows, grid.x along a row
template <typename T>
__global__ void __launch_bounds__(kThreads)
hermitian_kernel(const cpx<T>* __restrict__ x, cpx<T>* __restrict__ y, long n, long batch) {
  const long bins = n / 2 + 1;
  for (long b = blockIdx.y; b < batch; b += gridDim.y)
    for (long k = blockIdx.x * (long)blockDim.x + threadIdx.x; k < n; k += (long)gridDim.x * blockDim.x)
      y[b * n + k] = real::hermitian(x + b * bins, n, k);
}

// y[k] *= s * (Hermitian extension of the spectrum row ((row0 + b) / per) mod rows)[k]; grid as hermitian_kernel
template <typename T>
__global__ void __launch_bounds__(kThreads)
hermitian_mul_kernel(cpx<T>* __restrict__ y, const cpx<T>* __restrict__ spec, long n, long batch, long rows, long row0,
                     long per, T s) {
  const long bins = n / 2 + 1;
  for (long b = blockIdx.y; b < batch; b += gridDim.y) {
    const cpx<T>* hs = spec + (((row0 + b) / per) % rows) * bins;
    for (long k = blockIdx.x * (long)blockDim.x + threadIdx.x; k < n; k += (long)gridDim.x * blockDim.x)
      y[b * n + k] = cscale(cmul(y[b * n + k], real::hermitian(hs, n, k)), s);
  }
}

// Linear convolution (real::SegMap): one thread per sample p < N of segment q of the launch.  gather: the N input
// samples of each segment into seg, zero outside the row's [lo, hi); scatter: the kept outputs of each segment.
template <typename T>
__global__ void __launch_bounds__(kThreads)
gather_segments_kernel(const T* __restrict__ in, T* __restrict__ seg, const real::SegMap m, long nseg) {
  const long total = nseg * m.n;
  for (long g = blockIdx.x * (long)blockDim.x + threadIdx.x; g < total; g += (long)gridDim.x * blockDim.x) {
    const long q = g / m.n;
    real::gather_one(m, in, seg, q, g - q * m.n);
  }
}
template <typename T>
__global__ void __launch_bounds__(kThreads)
scatter_segments_kernel(const T* __restrict__ seg, T* __restrict__ out, const real::SegMap m, long nseg) {
  const long total = nseg * m.n;
  for (long g = blockIdx.x * (long)blockDim.x + threadIdx.x; g < total; g += (long)gridDim.x * blockDim.x) {
    const long q = g / m.n;
    real::scatter_one(m, seg, out, q, g - q * m.n);
  }
}

// Short-time Fourier transform (real::FrameMap).  gather: one thread per sample p < N of frame q of the launch, the
// windowed frame into seg.  overlap-add: one thread per output i0 <= i < i1 of rows b0 .. b0 + nb - 1, from the
// inverted frames in seg (global frames gs on); out is output 0 of row b0, rows out_ld apart.
template <typename T>
__global__ void __launch_bounds__(kThreads)
gather_frames_kernel(const T* __restrict__ in, const T* __restrict__ win, T* __restrict__ seg, const real::FrameMap m,
                     long nframes) {
  const long total = nframes * m.n;
  for (long g = blockIdx.x * (long)blockDim.x + threadIdx.x; g < total; g += (long)gridDim.x * blockDim.x) {
    const long q = g / m.n;
    real::gather_frame_one(m, in, win, seg, q, g - q * m.n);
  }
}
template <typename T>
__global__ void __launch_bounds__(kThreads)
overlap_add_kernel(const T* __restrict__ seg, const T* __restrict__ win, T* __restrict__ out, const real::FrameMap m,
                   long gs, long b0, long nb, long i0, long i1, long out_ld) {
  const long cnt = i1 - i0, total = nb * cnt;
  for (long g = blockIdx.x * (long)blockDim.x + threadIdx.x; g < total; g += (long)gridDim.x * blockDim.x) {
    const long r = g / cnt;
    real::overlap_add_one(m, seg, win, gs, out + r * out_ld, b0 + r, i0 + (g - r * cnt));
  }
}

// Mel spectrogram (real::band_scan / mel_dot).  bands: one CTA per filter row, each thread scanning every kThreads-th
// weight, merged in shared memory.  spectra: one thread per mel m of frame q of the chunk, consecutive threads on
// consecutive mels of a frame, from the chunk's spectra into the output rows (frame g0 + q).
template <typename T>
__global__ void __launch_bounds__(kThreads)
mel_bands_kernel(const T* __restrict__ filters, long bins, long n_mels, real::Band* __restrict__ bands) {
  __shared__ real::Band part[kThreads];
  for (long m = blockIdx.x; m < n_mels; m += gridDim.x) {
    part[threadIdx.x] = real::band_scan(filters + m * bins, bins, (long)threadIdx.x, (long)kThreads);
    __syncthreads();
    for (int w = kThreads / 2; w > 0; w /= 2) {
      if ((int)threadIdx.x < w) part[threadIdx.x] = real::band_merge(part[threadIdx.x], part[threadIdx.x + w]);
      __syncthreads();
    }
    if (threadIdx.x == 0) bands[m] = part[0];
    __syncthreads();
  }
}
template <typename T>
__global__ void __launch_bounds__(kThreads)
mel_spectra_kernel(const cpx<T>* __restrict__ spec, const T* __restrict__ filters, const real::Band* __restrict__ bands,
                   long bins, long n_mels, int power, T* __restrict__ out, long nframes, long g0) {
  const long total = nframes * n_mels;
  for (long g = blockIdx.x * (long)blockDim.x + threadIdx.x; g < total; g += (long)gridDim.x * blockDim.x) {
    const long q = g / n_mels;
    real::mel_spectrum_one(spec, filters, bands, bins, n_mels, power, out, q, g - q * n_mels, g0 + q);
  }
}

// MFCC (real::log_mel / mfcc_dot) of a chunk's mels: the frame's n_mels mels at mel + q * n_mels, frame g0 + q of
// rows of `frames` frames.  MAX: CTA c takes a contiguous run of frames, and each thread folds the key of its largest
// log-mel (m = t, t + kThreads, ...) into a group's slot once per group the run meets.  Otherwise one CTA per frame: the
// threads write the frame's clamped log-mels over its mels, and after a barrier thread t computes outputs j = t,
// t + kThreads, ... into out (n_out reals per frame).
template <typename T, bool MAX>
__global__ void __launch_bounds__(kThreads)
mfcc_frames_kernel(T* mel, long n_mels, const real::MfccArgs<T> p, T* __restrict__ out, long nframes, long g0,
                   long frames) {
  if constexpr (MAX) {
    const long per = (nframes + gridDim.x - 1) / gridDim.x, q1 = std::min(nframes, (blockIdx.x + 1) * per);
    real::MaxKey<T> hi = 0;
    long grp = -1;
    for (long q = blockIdx.x * per; q < q1; ++q) {
      const long g = real::clamp_group(p, (g0 + q) / frames);
      if (g != grp) {
        if (grp >= 0) real::max_fold(p.slots + grp, hi);
        grp = g;
        hi = 0;
      }
      for (long m = threadIdx.x; m < n_mels; m += kThreads) {
        const real::MaxKey<T> k = real::max_key(real::log_mel(mel[q * n_mels + m], p));
        hi = k > hi ? k : hi;
      }
    }
    if (grp >= 0) real::max_fold(p.slots + grp, hi);
    return;
  }
  for (long q = blockIdx.x; q < nframes; q += gridDim.x) {
    T* x = mel + q * n_mels;
    const long b = (g0 + q) / frames;
    {
      const T theta = real::clamp_threshold(p, b);
      for (long m = threadIdx.x; m < n_mels; m += kThreads) x[m] = real::clamp_db(real::log_mel(x[m], p), theta);
      __syncthreads();
      for (long j = threadIdx.x; j < p.n_out; j += kThreads)
        real::lin_st(out + q * p.n_out + j, real::mfcc_dot(p, n_mels, j, [&](long m) { return x[m]; }), g0 + q);
      __syncthreads();
    }
  }
}

// Welch (real::WelchItems).  scale: one CTA, the window sums in double, each thread over every kThreads-th sample in
// ascending order, then a tree in shared memory.  gather: one CTA per frame q of the chunk (frame g0 + q of the rows'
// FrameMap), the frame mean by the same two steps in T, then (x - mu) w into seg.  accumulate: one thread per (item, bin)
// of the items that have frames in the chunk.  finish: one thread per (row, bin).
template <typename T>
__global__ void __launch_bounds__(kThreads)
welch_scale_kernel(const T* __restrict__ win, long n, int scaling, double fs, long frames, T* __restrict__ base) {
  __shared__ double s1[kThreads], s2[kThreads];
  double a = 0, b = 0;
  for (long p = threadIdx.x; p < n; p += kThreads) {
    const double w = win[p];
    a += w;
    b += w * w;
  }
  s1[threadIdx.x] = a;
  s2[threadIdx.x] = b;
  __syncthreads();
  for (int w = kThreads / 2; w > 0; w /= 2) {
    if ((int)threadIdx.x < w) {
      s1[threadIdx.x] += s1[threadIdx.x + w];
      s2[threadIdx.x] += s2[threadIdx.x + w];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) *base = (T)real::welch_base(s1[0], s2[0], scaling, fs, frames);
}
// one frame of a gather: its mean by a fixed tree in shared memory (detrend constant), then (x - mu) w into dst
template <typename T>
__device__ __forceinline__ void gather_detrended(const T* __restrict__ src, const T* __restrict__ win, T* __restrict__ dst,
                                                 long n, int detrend, T* part) {
  T mu = 0;
  if (detrend == real::kDetrendConstant) {
    T s = 0;
    for (long p = threadIdx.x; p < n; p += kThreads) s += src[p];
    part[threadIdx.x] = s;
    __syncthreads();
    for (int w = kThreads / 2; w > 0; w /= 2) {
      if ((int)threadIdx.x < w) part[threadIdx.x] += part[threadIdx.x + w];
      __syncthreads();
    }
    mu = part[0] / (T)n;
    __syncthreads();
  }
  for (long p = threadIdx.x; p < n; p += kThreads) dst[p] = (src[p] - mu) * win[p];
}
template <typename T>
__global__ void __launch_bounds__(kThreads)
welch_gather_kernel(const T* __restrict__ in, const T* __restrict__ win, T* __restrict__ seg, const real::FrameMap m,
                    long nframes, int detrend) {
  __shared__ T part[kThreads];
  for (long q = blockIdx.x; q < nframes; q += gridDim.x) {
    const long g = m.g0 + q, b = m.row_of(g);
    gather_detrended(in + (b - m.r0) * m.in_ld + m.start(g, b), win, seg + q * m.n, m.n, detrend, part);
  }
}
template <typename T>
__global__ void __launch_bounds__(kThreads)
welch_accumulate_kernel(const cpx<T>* __restrict__ spec, const real::WelchItems w, long bins, long q0, long nq, long i0,
                        long ni, T* __restrict__ part) {
  const long total = ni * bins;
  for (long g = blockIdx.x * (long)blockDim.x + threadIdx.x; g < total; g += (long)gridDim.x * blockDim.x) {
    const long i = i0 + g / bins, k = g - (g / bins) * bins, b = i / w.items;
    real::welch_accumulate_one(spec, bins, q0, nq, b * w.frames + (i - b * w.items) * w.block, w.count(i), part, i, k);
  }
}
template <typename T>
__global__ void __launch_bounds__(kThreads)
welch_finish_kernel(const T* __restrict__ part, long items, long n, const T* __restrict__ base, T* __restrict__ out,
                    long rows) {
  const long bins = n / 2 + 1, total = rows * bins;
  const T s = *base;
  for (long g = blockIdx.x * (long)blockDim.x + threadIdx.x; g < total; g += (long)gridDim.x * blockDim.x) {
    const long b = g / bins;
    real::welch_finish_one(part, items, n, s, out, b, g - b * bins);
  }
}
// Cross-spectral density and coherence (DESIGN.md §4.17) on frame pairs.  gather: welch_gather_kernel's frames of x
// into seg and those of their y rows (row b of the rows' FrameMap with y row (y_off + b) mod y_rows) nframes frames
// behind.  accumulate: welch_accumulate_kernel's threads over the item's x and y spectra.  finish: one thread per
// (row, bin).
template <typename T>
__global__ void __launch_bounds__(kThreads)
csd_gather_kernel(const T* __restrict__ x, const T* __restrict__ y, long y_rows, long y_off,
                  const T* __restrict__ win, T* __restrict__ seg, const real::FrameMap m, long nframes, int detrend) {
  __shared__ T part[kThreads];
  for (long q = blockIdx.x; q < nframes; q += gridDim.x) {
    const long g = m.g0 + q, b = m.row_of(g), t0 = m.start(g, b);
    gather_detrended(x + (b - m.r0) * m.in_ld + t0, win, seg + q * m.n, m.n, detrend, part);
    gather_detrended(y + ((y_off + b) % y_rows) * m.in_ld + t0, win, seg + (nframes + q) * m.n, m.n, detrend, part);
  }
}
template <typename T>
__global__ void __launch_bounds__(kThreads)
cross_accumulate_kernel(const cpx<T>* __restrict__ specx, const cpx<T>* __restrict__ specy, const real::WelchItems w,
                        long bins, long q0, long nq, long i0, long ni, int planes, T* __restrict__ part) {
  const long total = ni * bins;
  for (long g = blockIdx.x * (long)blockDim.x + threadIdx.x; g < total; g += (long)gridDim.x * blockDim.x) {
    const long i = i0 + g / bins, k = g - (g / bins) * bins, b = i / w.items;
    real::cross_accumulate_one(specx, specy, bins, q0, nq, b * w.frames + (i - b * w.items) * w.block, w.count(i),
                               planes, part, i, k);
  }
}
template <typename T>
__global__ void __launch_bounds__(kThreads)
cross_finish_kernel(const T* __restrict__ part, long items, long n, const T* __restrict__ base, bool coh,
                    void* __restrict__ out, long rows) {
  const long bins = n / 2 + 1, total = rows * bins;
  for (long g = blockIdx.x * (long)blockDim.x + threadIdx.x; g < total; g += (long)gridDim.x * blockDim.x) {
    const long b = g / bins;
    if (coh) real::coherence_finish_one(part, items, n, (T*)out, b, g - b * bins);
    else real::csd_finish_one(part, items, n, *base, (cpx<T>*)out, b, g - b * bins);
  }
}

// Discrete cosine transforms (real::dct2_pair, dct3_pair, dct2_post, dct3_pre).  Rows of N reals in `in` / `out`, rows of the inner
// plan's length in seg; one thread per element or pair of a row, consecutive threads along a row.
//   permute: v into seg, N reals per row (half length) or N complex values with zero imaginary parts (full length);
//   untangle: the pair k <= M/2 of Z in seg -> four outputs;  tangle: the pair k <= M/2 of Z' from the row into seg;
//   post: the bin k <= N/2 of V in seg -> y[k], y[N-k];  pre: V'[k], k < N, from the row into seg;
//   unpermute: output i from u in seg, N reals per row (half length) or the real parts of N complex values.
template <typename T, bool WIDE>
__global__ void __launch_bounds__(kThreads)
dct_permute_kernel(const T* __restrict__ in, void* __restrict__ seg, long n, long batch) {
  const long total = n * batch;
  for (long g = blockIdx.x * (long)blockDim.x + threadIdx.x; g < total; g += (long)gridDim.x * blockDim.x) {
    const long b = g / n, j = g - b * n;
    const T x = real::lin_ld(in + b * n + real::dct_src(n, j), b);
    if (WIDE) ((cpx<T>*)seg)[g] = mk<T>(x, (T)0);
    else ((T*)seg)[g] = x;
  }
}
template <typename T>
__global__ void __launch_bounds__(kThreads)
dct_untangle_kernel(const cpx<T>* __restrict__ z, T* __restrict__ out, const cpx<T>* __restrict__ tab,
                    const cpx<T>* __restrict__ wq, long m, long batch, T h, T h0) {
  const long pairs = m / 2 + 1, total = pairs * batch;
  for (long g = blockIdx.x * (long)blockDim.x + threadIdx.x; g < total; g += (long)gridDim.x * blockDim.x) {
    const long b = g / pairs, k = g - b * pairs, n = 2 * m;
    const cpx<T>* zb = z + b * m;
    T* y = out + b * n;
    cpx<T> lo, hi;
    real::dct2_pair(zb[k], zb[k ? m - k : 0], m, k, tab, wq, h, h0, lo, hi);
    real::lin_st(y + k, lo.x, b);
    if (k == 0) { real::lin_st(y + m, lo.y, b); continue; }
    real::lin_st(y + (n - k), lo.y, b);
    if (m - k == k) continue;
    real::lin_st(y + (m - k), hi.x, b);
    real::lin_st(y + (m + k), hi.y, b);
  }
}
template <typename T>
__global__ void __launch_bounds__(kThreads)
dct_tangle_kernel(const T* __restrict__ in, cpx<T>* __restrict__ z, const cpx<T>* __restrict__ tab,
                  const cpx<T>* __restrict__ wq, long m, long batch, T h, T h0) {
  const long pairs = m / 2 + 1, total = pairs * batch;
  for (long g = blockIdx.x * (long)blockDim.x + threadIdx.x; g < total; g += (long)gridDim.x * blockDim.x) {
    const long b = g / pairs, k = g - b * pairs;
    cpx<T> p, q;
    real::dct3_pair(in + b * 2 * m, m, k, tab, wq, h, h0, p, q);
    z[b * m + k] = p;
    if (k > 0 && m - k != k) z[b * m + m - k] = q;
  }
}
template <typename T>
__global__ void __launch_bounds__(kThreads)
dct_post_kernel(const cpx<T>* __restrict__ v, T* __restrict__ out, const cpx<T>* __restrict__ wq, long n, long batch,
                T h, T h0) {
  const long bins = n / 2 + 1, total = bins * batch;
  for (long g = blockIdx.x * (long)blockDim.x + threadIdx.x; g < total; g += (long)gridDim.x * blockDim.x) {
    const long b = g / bins, k = g - b * bins;
    real::dct2_post(v + b * n, out + b * n, n, k, wq, h, h0, b);
  }
}
template <typename T>
__global__ void __launch_bounds__(kThreads)
dct_pre_kernel(const T* __restrict__ in, cpx<T>* __restrict__ v, const cpx<T>* __restrict__ wq, long n, long batch, T h,
               T h0) {
  const long total = n * batch;
  for (long g = blockIdx.x * (long)blockDim.x + threadIdx.x; g < total; g += (long)gridDim.x * blockDim.x) {
    const long b = g / n;
    v[g] = real::dct3_pre(in + b * n, n, g - b * n, wq, h, h0);
  }
}
template <typename T, bool WIDE>
__global__ void __launch_bounds__(kThreads)
dct_unpermute_kernel(const void* __restrict__ seg, T* __restrict__ out, long n, long batch) {
  const long total = n * batch;
  for (long g = blockIdx.x * (long)blockDim.x + threadIdx.x; g < total; g += (long)gridDim.x * blockDim.x) {
    const long b = g / n, s = b * n + real::dct_pos(n, g - b * n);
    real::lin_st(out + g, WIDE ? ((const cpx<T>*)seg)[s].x : ((const T*)seg)[s], b);
  }
}

// Type-IV DCT and MDCT (real::dct4_pre, dct4_post, mdct_fold_one, imdct_add_one), even N = 2M.  One thread per position
// k < M of a row or frame, consecutive threads along it.  pre: z[k] of the rows into z (M complex values per row);
// mdct gather: z[k] of the windowed, folded frames q of the launch (global frame m.g0 + q) into z; post: (y[2k],
// y[N-1-2k]) from Z[k] in z into the output rows (row b of the launch is row g0 + b, for the emulator's log).
// overlap-add: one thread per output i0 <= i < i1 of rows b0 .. b0 + nb - 1, as overlap_add_kernel.
template <typename T>
__global__ void __launch_bounds__(kThreads)
dct4_pre_kernel(const T* __restrict__ in, cpx<T>* __restrict__ z, const cpx<T>* __restrict__ wq, long n, long batch) {
  const long m = n / 2, total = m * batch;
  for (long g = blockIdx.x * (long)blockDim.x + threadIdx.x; g < total; g += (long)gridDim.x * blockDim.x) {
    const long b = g / m, k = g - b * m;
    const T* x = in + b * n;
    z[g] = real::dct4_pre(real::lin_ld(x + 2 * k, b), real::lin_ld(x + (n - 1 - 2 * k), b), wq, n, k);
  }
}
template <typename T>
__global__ void __launch_bounds__(kThreads)
mdct_gather_kernel(const T* __restrict__ in, const T* __restrict__ win, cpx<T>* __restrict__ z, const real::FrameMap m,
                   const cpx<T>* __restrict__ wq, long nframes) {
  const long n = m.hop, half = n / 2, total = half * nframes;
  for (long g = blockIdx.x * (long)blockDim.x + threadIdx.x; g < total; g += (long)gridDim.x * blockDim.x) {
    const long q = g / half, k = g - q * half;
    z[g] = real::dct4_pre(real::mdct_fold_one(m, in, win, q, 2 * k), real::mdct_fold_one(m, in, win, q, n - 1 - 2 * k),
                          wq, n, k);
  }
}
template <typename T>
__global__ void __launch_bounds__(kThreads)
dct4_post_kernel(const cpx<T>* __restrict__ z, T* __restrict__ out, const cpx<T>* __restrict__ wq, cpx<T> c, long n,
                 long batch, long g0) {
  const long m = n / 2, total = m * batch;
  for (long g = blockIdx.x * (long)blockDim.x + threadIdx.x; g < total; g += (long)gridDim.x * blockDim.x) {
    const long b = g / m, k = g - b * m;
    const cpx<T> p = real::dct4_post(z[g], c, wq, n, k);
    real::lin_st(out + b * n + 2 * k, p.x, g0 + b);
    real::lin_st(out + b * n + (n - 1 - 2 * k), p.y, g0 + b);
  }
}
template <typename T>
__global__ void __launch_bounds__(kThreads)
imdct_overlap_add_kernel(const T* __restrict__ seg, const T* __restrict__ win, T* __restrict__ out,
                         const real::FrameMap m, long gs, long b0, long nb, long i0, long i1, long out_ld) {
  const long cnt = i1 - i0, total = nb * cnt;
  for (long g = blockIdx.x * (long)blockDim.x + threadIdx.x; g < total; g += (long)gridDim.x * blockDim.x) {
    const long r = g / cnt;
    real::imdct_add_one(m, seg, win, gs, out + r * out_ld, b0 + r, i0 + (g - r * cnt));
  }
}

// Analytic signal (real::hilbert_pair, hilbert_bin, hilbert_out_one).  pair: one thread per pair k <= M/2 of a row, in
// place on z (M complex values per row).  mul: one thread per bin k < N of a row of length-N spectra, in place.  out: one
// thread per output n of a row, from x[n] and y[n] (seg holds N reals per row at half length, N complex values whose
// real parts are y at full length); it is the only kernel that writes `out`, so in == out is safe.
template <typename T>
__global__ void __launch_bounds__(kThreads)
hilbert_pair_kernel(cpx<T>* __restrict__ z, const cpx<T>* __restrict__ tab, long m, long batch, T h) {
  const long pairs = m / 2 + 1, total = pairs * batch;
  for (long g = blockIdx.x * (long)blockDim.x + threadIdx.x; g < total; g += (long)gridDim.x * blockDim.x) {
    const long b = g / pairs;
    real::hilbert_pair(z + b * m, m, g - b * pairs, tab, h);
  }
}
template <typename T>
__global__ void __launch_bounds__(kThreads)
hilbert_mul_kernel(cpx<T>* __restrict__ y, long n, long batch, T s) {
  const long total = n * batch;
  for (long g = blockIdx.x * (long)blockDim.x + threadIdx.x; g < total; g += (long)gridDim.x * blockDim.x)
    y[g] = real::hilbert_bin(y[g], n, g - (g / n) * n, s);
}
template <typename T, bool WIDE>
__global__ void __launch_bounds__(kThreads)
hilbert_out_kernel(const T* in, const void* __restrict__ seg, void* out, long n, long batch, int output) {
  const long total = n * batch;
  for (long g = blockIdx.x * (long)blockDim.x + threadIdx.x; g < total; g += (long)gridDim.x * blockDim.x) {
    const long b = g / n;
    const T y = WIDE ? ((const cpx<T>*)seg)[g].x : ((const T*)seg)[g];
    real::hilbert_out_one(real::lin_ld(in + g, b), y, out, g, output, b);
  }
}

template <typename T>
__global__ void __launch_bounds__(kThreads)
real_part_kernel(const cpx<T>* __restrict__ y, T* __restrict__ out, size_t count) {
  for (size_t g = blockIdx.x * (size_t)blockDim.x + threadIdx.x; g < count; g += (size_t)gridDim.x * blockDim.x)
    out[g] = y[g].x;
}

// the DCT-IV's post-step constant c of a norm (real::dct4_const), rounded once
template <typename T> cpx<T> dct4_c(int norm, size_t n) {
  double re, im;
  real::dct4_const(norm, (long)n, re, im);
  return mk<T>((T)re, (T)im);
}

// Items of item_bytes that one chunk of plan scratch holds: as many as fit kScratchTargetBytes, at least 1, at most total.
size_t scratch_chunk(size_t total, size_t item_bytes) {
  return std::min(total, std::max<size_t>(1, kScratchTargetBytes / item_bytes));
}

}  // namespace

template <typename T>
RealPlan<T>::~RealPlan() {
  DeviceGuard g(device_);
  if (host_stream_) cudaStreamDestroy(host_stream_);
}

template <typename T>
cudaError_t RealPlan<T>::init(size_t n, int device, bool allow_fast_paths) {
  n_ = n;
  device_ = device;
  DeviceGuard g(device_);
  if (!g.ok) { set_last_error("cudaSetDevice failed"); return cudaErrorInvalidDevice; }
  std::vector<C> wq(n / 2 + 1);
  for (size_t k = 0; k < wq.size(); ++k) {
    double re, im;
    host_twiddle(k, 4 * n, &re, &im);
    wq[k] = mk<T>((T)re, (T)im);
  }
  FB_CHECK(upload(dct_tab_, wq));
  if (n % 2 != 0) {
    inner_.reset(Plan<T>::create(n, device, allow_fast_paths));
    if (!inner_) return cudaErrorUnknown;
    path_ = Path::kRealFull;
    kernel_desc_ = std::string("real::widen_kernel / real::hermitian_kernel + ") + inner_->kernel_name();
    return cudaSuccess;
  }
  m_ = n / 2;
  std::vector<C> tab(m_ / 2 + 1);
  for (size_t k = 0; k < tab.size(); ++k) {
    double re, im;
    host_twiddle(k, n, &re, &im);
    tab[k] = mk<T>((T)re, (T)im);
  }
  FB_CHECK(upload(tab_, tab));
  if (allow_fast_paths && (fused_ = real_onchip_lookup<T>(m_)) != nullptr) {
    FB_CHECK(fused_->prepare());
    FB_CHECK(upload(twa_, twopass::make_twa<T>(fused_->ra, fused_->rb)));
    sm_count_ = sm_count(device_);
    path_ = Path::kRealFused;
    kernel_desc_ = "onchip::onchip_real_kernel";
    return cudaSuccess;
  }
  inner_.reset(Plan<T>::create(m_, device, allow_fast_paths));
  if (!inner_) return cudaErrorUnknown;
  path_ = Path::kRealHalf;
  kernel_desc_ = std::string("real::untangle_kernel / real::tangle_kernel + ") + inner_->kernel_name();
  return cudaSuccess;
}

template <typename T>
PlanInfo RealPlan<T>::info() const {
  PlanInfo i;
  if (inner_) i = inner_->info();
  i.inner_size = inner_ ? inner_->size() : 0;
  i.inner_path = inner_ ? (int)inner_->path() : 0;
  i.size = n_;
  i.path = (int)path_;
  i.precision_bytes = (int)sizeof(T);
  i.device = device_;
  i.table_bytes = tab_.bytes() + twa_.bytes() + dct_tab_.bytes() + (inner_ ? inner_->info().table_bytes : 0);
  return i;
}

template <typename T>
cudaError_t RealPlan<T>::check_code(bool forward, int code) const {
  if (code < 0 || code > 4) { set_last_error("unknown transform code"); return cudaErrorInvalidValue; }
  if (transform_is_forward(code) != forward) {
    set_last_error(forward ? "the forward real transform takes Fft or SqrtScaledFft"
                           : "the inverse real transform takes Ifft, UnscaledIfft or SqrtScaledIfft");
    return cudaErrorInvalidValue;
  }
  return cudaSuccess;
}

template <typename T>
cudaError_t RealPlan<T>::exec_device(bool forward, const void* in, void* out, size_t batch, int code,
                                     cudaStream_t s) {
  launches_ = 0;
  if (cudaError_t e = check_code(forward, code)) return e;
  if (batch == 0) return cudaSuccess;
  DeviceGuard g(device_);
  return rfft_rows(forward, in, out, batch, code, s);
}

template <typename T>
cudaError_t RealPlan<T>::rfft_rows(bool forward, const void* in, void* out, size_t batch, int code, cudaStream_t s) {
  const T scale = scale_for<T>(code, n_);
  if (path_ == Path::kRealFused) {
    FB_CHECK(fused_->run(in, out, twa_.data(), (const C*)tab_.data(), batch, forward, forward ? scale / 2 : scale,
                         sm_count_, s));
    launches_ += 1;
    return cudaSuccess;
  }
  const size_t len = inner_->size(), bins = n_ / 2 + 1;
  const size_t chunk = scratch_chunk(batch, len * sizeof(C));
  FB_CHECK(work_.reserve(chunk * len * sizeof(C)));
  C* work = (C*)work_.data();
  for (size_t b0 = 0; b0 < batch; b0 += chunk) {
    const size_t nb = std::min(chunk, batch - b0);
    if (path_ == Path::kRealHalf) {
      if (forward) {
        FB_CHECK(inner_->exec_device((const C*)in + b0 * m_, work, nb, kFft, s));
        launches_ += inner_->launches();
        untangle_kernel<T, true><<<grid_for((m_ / 2 + 1) * nb), kThreads, 0, s>>>(
            work, (C*)out + b0 * bins, (const C*)tab_.data(), (long)m_, (long)nb, scale / 2);
        FB_CHECK(cudaGetLastError());
      } else {
        untangle_kernel<T, false><<<grid_for((m_ / 2 + 1) * nb), kThreads, 0, s>>>(
            (const C*)in + b0 * bins, work, (const C*)tab_.data(), (long)m_, (long)nb, scale);
        FB_CHECK(cudaGetLastError());
        FB_CHECK(inner_->exec_device(work, (C*)out + b0 * m_, nb, kUnscaledIfft, s));
        launches_ += inner_->launches();
      }
      launches_ += 1;
    } else {
      if (forward) {
        widen_kernel<T><<<grid_for(nb * n_), kThreads, 0, s>>>((const T*)in + b0 * n_, work, nb * n_);
        FB_CHECK(cudaGetLastError());
        FB_CHECK(inner_->exec_device(work, work, nb, code, s));
        launches_ += inner_->launches();
        copy_bins_kernel<T><<<grid_for(nb * bins), kThreads, 0, s>>>(work, (C*)out + b0 * bins, (long)n_, (long)nb);
        FB_CHECK(cudaGetLastError());
      } else {
        const dim3 grid(grid_for(n_), (unsigned)std::min<size_t>(nb, 65535));
        hermitian_kernel<T><<<grid, kThreads, 0, s>>>((const C*)in + b0 * bins, work, (long)n_, (long)nb);
        FB_CHECK(cudaGetLastError());
        FB_CHECK(inner_->exec_device(work, work, nb, code, s));
        launches_ += inner_->launches();
        real_part_kernel<T><<<grid_for(nb * n_), kThreads, 0, s>>>(work, (T*)out + b0 * n_, nb * n_);
        FB_CHECK(cudaGetLastError());
      }
      launches_ += 2;
    }
  }
  return cudaSuccess;
}

template <typename T>
cudaError_t RealPlan<T>::open_host_stream() {
  if (!host_stream_) FB_CHECK(cudaStreamCreateWithFlags(&host_stream_, cudaStreamNonBlocking));
  return cudaSuccess;
}

// Host pointers: chunks of rows go H2D into stage_in_, through `step` into stage_out_, and D2H, one chunk at a time on
// the plan's own stream (no pipelining: the results are those of the device path, bit for bit).  The caller holds the
// DeviceGuard.
template <typename T>
template <class Step>
cudaError_t RealPlan<T>::stage_rows(const void* in, void* out, size_t batch, size_t in_row, size_t out_row, Step step) {
  FB_CHECK(open_host_stream());
  const size_t rows = std::min(batch, std::max<size_t>(1, kHostChunkBytes / std::max(in_row, out_row)));
  FB_CHECK(stage_in_.reserve(rows * in_row));
  FB_CHECK(stage_out_.reserve(rows * out_row));
  for (size_t b0 = 0; b0 < batch; b0 += rows) {
    const size_t nb = std::min(rows, batch - b0);
    FB_CHECK(cudaMemcpyAsync(stage_in_.data(), (const char*)in + b0 * in_row, nb * in_row, cudaMemcpyHostToDevice,
                             host_stream_));
    FB_CHECK(step(stage_in_.data(), stage_out_.data(), b0, nb));
    if (out_row)
      FB_CHECK(cudaMemcpyAsync((char*)out + b0 * out_row, stage_out_.data(), nb * out_row, cudaMemcpyDeviceToHost,
                               host_stream_));
    FB_CHECK(cudaStreamSynchronize(host_stream_));
  }
  return cudaSuccess;
}

template <typename T>
template <class A, class B>
cudaError_t RealPlan<T>::stage_consts(const A* a, size_t a_bytes, const A** da, const B* b, size_t b_bytes,
                                      const B** db) {
  FB_CHECK(open_host_stream());
  const size_t b_off = (a_bytes + 255) / 256 * 256;
  FB_CHECK(stage_spec_.reserve(b ? b_off + b_bytes : a_bytes));
  char* base = (char*)stage_spec_.data();
  FB_CHECK(cudaMemcpyAsync(base, a, a_bytes, cudaMemcpyHostToDevice, host_stream_));
  *da = (const A*)base;
  if (b) {
    FB_CHECK(cudaMemcpyAsync(base + b_off, b, b_bytes, cudaMemcpyHostToDevice, host_stream_));
    *db = (const B*)(base + b_off);
  }
  return cudaSuccess;
}

template <typename T>
cudaError_t RealPlan<T>::exec_host(bool forward, const void* in, void* out, size_t batch, int code) {
  launches_ = 0;
  if (cudaError_t e = check_code(forward, code)) return e;
  if (batch == 0) return cudaSuccess;
  DeviceGuard g(device_);
  return stage_rows(in, out, batch, row_bytes(forward, true), row_bytes(forward, false),
                    [&](const void* din, void* dout, size_t, size_t nb) {
                      return rfft_rows(forward, din, dout, nb, code, host_stream_);
                    });
}

template <typename T>
cudaError_t RealPlan<T>::convolve_rows(const T* in, const C* spec, size_t rows, size_t row0, size_t per, T* out,
                                       size_t batch, cudaStream_t s) {
  if (batch == 0) return cudaSuccess;
  DeviceGuard g(device_);
  row0 %= rows * per;
  if (path_ == Path::kRealFused) {
    FB_CHECK(fused_->conv(in, out, twa_.data(), (const C*)tab_.data(), spec, rows, row0, per, batch, (T)1 / (T)(2 * n_),
                          sm_count_, s));
    launches_ += 1;
    return cudaSuccess;
  }
  if (path_ == Path::kRealHalf) {
    // z = x as M complex values per row: the forward, the pair step and the inverse all run in `out`
    FB_CHECK(inner_->exec_device((const C*)in, (C*)out, batch, kFft, s));
    launches_ += inner_->launches();
    conv_pair_kernel<T><<<grid_for((m_ / 2 + 1) * batch), kThreads, 0, s>>>(
        (C*)out, spec, (const C*)tab_.data(), (long)m_, (long)batch, (long)rows, (long)row0, (long)per,
        (T)1 / (T)(2 * n_));
    FB_CHECK(cudaGetLastError());
    launches_ += 1;
    FB_CHECK(inner_->exec_device((C*)out, (C*)out, batch, kUnscaledIfft, s));
    launches_ += inner_->launches();
    return cudaSuccess;
  }
  const size_t chunk = scratch_chunk(batch, n_ * sizeof(C));
  FB_CHECK(work_.reserve(chunk * n_ * sizeof(C)));
  C* work = (C*)work_.data();
  for (size_t b0 = 0; b0 < batch; b0 += chunk) {
    const size_t nb = std::min(chunk, batch - b0);
    widen_kernel<T><<<grid_for(nb * n_), kThreads, 0, s>>>(in + b0 * n_, work, nb * n_);
    FB_CHECK(cudaGetLastError());
    FB_CHECK(inner_->exec_device(work, work, nb, kFft, s));
    launches_ += inner_->launches();
    const dim3 grid(grid_for(n_), (unsigned)std::min<size_t>(nb, 65535));
    hermitian_mul_kernel<T><<<grid, kThreads, 0, s>>>(work, spec, (long)n_, (long)nb, (long)rows,
                                                      (long)((row0 + b0) % (rows * per)), (long)per, (T)1 / (T)n_);
    FB_CHECK(cudaGetLastError());
    FB_CHECK(inner_->exec_device(work, work, nb, kUnscaledIfft, s));
    launches_ += inner_->launches();
    real_part_kernel<T><<<grid_for(nb * n_), kThreads, 0, s>>>(work, out + b0 * n_, nb * n_);
    FB_CHECK(cudaGetLastError());
    launches_ += 3;
  }
  return cudaSuccess;
}

// Host pointers: the spectra go H2D once into stage_spec_; chunks of rows then go through convolve_rows as in
// exec_host, each chunk starting at its own spectrum row, so the bits are those of one device call.
template <typename T>
cudaError_t RealPlan<T>::convolve_host(const T* in, const C* spec, size_t rows, T* out, size_t batch) {
  launches_ = 0;
  if (batch == 0) return cudaSuccess;
  DeviceGuard g(device_);
  const C* dspec;
  FB_CHECK(stage_consts(spec, spec_bytes(rows), &dspec));
  return stage_rows(in, out, batch, n_ * sizeof(T), n_ * sizeof(T),
                    [&](const void* din, void* dout, size_t b0, size_t nb) {
                      return convolve_rows((const T*)din, dspec, rows, b0, 1, (T*)dout, nb, host_stream_);
                    });
}

template <typename T>
cudaError_t RealPlan<T>::linear_segments(const T* in, T* out, const real::SegMap& m, size_t nseg, const C* spec,
                                         size_t rows, cudaStream_t s) {
  if (nseg == 0) return cudaSuccess;
  if (path_ == Path::kRealFused) {
    FB_CHECK(fused_->lconv(in, out, m, nseg, twa_.data(), (const C*)tab_.data(), spec, rows, (T)1 / (T)(2 * n_),
                           sm_count_, s));
    launches_ += 1;
    return cudaSuccess;
  }
  // chunks of segments through seg_: gather, the circular convolution in place (segment q of the chunk uses spectrum
  // row ((g0 + q) / per) mod rows), scatter
  const size_t chunk = scratch_chunk(nseg, n_ * sizeof(T));
  FB_CHECK(seg_.reserve(chunk * n_ * sizeof(T)));
  T* seg = (T*)seg_.data();
  for (size_t q0 = 0; q0 < nseg; q0 += chunk) {
    const size_t nq = std::min(chunk, nseg - q0);
    real::SegMap mc = m;
    mc.g0 = m.g0 + (long)q0;
    gather_segments_kernel<T><<<grid_for(nq * n_), kThreads, 0, s>>>(in, seg, mc, (long)nq);
    FB_CHECK(cudaGetLastError());
    FB_CHECK(convolve_rows(seg, spec, rows, (size_t)mc.g0, (size_t)m.per, seg, nq, s));
    scatter_segments_kernel<T><<<grid_for(nq * n_), kThreads, 0, s>>>(seg, out, mc, (long)nq);
    FB_CHECK(cudaGetLastError());
    launches_ += 2;
  }
  return cudaSuccess;
}

template <typename T>
cudaError_t RealPlan<T>::linear_convolve_device(const T* in, size_t in_len, const C* spec, size_t rows, size_t taps,
                                                int mode, T* out, size_t batch, cudaStream_t s) {
  launches_ = 0;
  if (batch == 0) return cudaSuccess;
  DeviceGuard g(device_);
  const real::SegMap m = real::linear_map((long)n_, (long)taps, mode, (long)in_len);
  return linear_segments(in, out, m, batch * (size_t)m.per, spec, rows, s);
}

// Host pointers, on the plan's own stream and synchronised after every piece, as stage_rows does.
template <typename T>
cudaError_t RealPlan<T>::linear_convolve_host(const T* in, size_t in_len, const C* spec, size_t rows, size_t taps,
                                              int mode, T* out, size_t batch) {
  launches_ = 0;
  if (batch == 0) return cudaSuccess;
  DeviceGuard g(device_);
  const C* dspec;
  FB_CHECK(stage_consts(spec, spec_bytes(rows), &dspec));
  const real::SegMap m = real::linear_map((long)n_, (long)taps, mode, (long)in_len);
  const size_t out_len = (size_t)m.out_len;
  if (std::max(in_len, out_len) * sizeof(T) <= kHostChunkBytes) {
    // whole rows: row b0 of the piece is global row b0 at the start of the staged buffers
    return stage_rows(in, out, batch, in_len * sizeof(T), out_len * sizeof(T),
                      [&](const void* din, void* dout, size_t b0, size_t nb) {
                        real::SegMap mp = m;
                        mp.g0 = (long)b0 * m.per;
                        mp.r0 = (long)b0;
                        return linear_segments((const T*)din, (T*)dout, mp, nb * (size_t)m.per, dspec, rows,
                                               host_stream_);
                      });
  }
  // runs of R segments of one row: input window [off + j0*S - (K-1), off + j1*S) within [0, L), outputs [j0*S, j1*S)
  const size_t cap = kHostChunkBytes / sizeof(T);
  const size_t run = cap > n_ ? std::max<size_t>(1, (cap - n_) / (size_t)m.s) : 1;
  FB_CHECK(stage_in_.reserve((run * (size_t)m.s + n_) * sizeof(T)));
  FB_CHECK(stage_out_.reserve(run * (size_t)m.s * sizeof(T)));
  for (size_t b = 0; b < batch; ++b)
    for (long j0 = 0; j0 < m.per; j0 += (long)run) {
      const long j1 = std::min(m.per, j0 + (long)run);
      real::SegMap mp = m;
      mp.g0 = (long)b * m.per + j0;
      mp.r0 = (long)b;
      mp.lo = std::max(0L, m.off + j0 * m.s - (m.k - 1));
      mp.hi = std::min((long)in_len, m.off + j1 * m.s);
      mp.out_lo = j0 * m.s;
      const long out_hi = std::min(m.out_len, j1 * m.s);
      if (mp.hi > mp.lo)
        FB_CHECK(cudaMemcpyAsync(stage_in_.data(), in + b * in_len + mp.lo, (mp.hi - mp.lo) * sizeof(T),
                                 cudaMemcpyHostToDevice, host_stream_));
      FB_CHECK(linear_segments((const T*)stage_in_.data(), (T*)stage_out_.data(), mp, (size_t)(j1 - j0), dspec, rows,
                               host_stream_));
      FB_CHECK(cudaMemcpyAsync(out + b * out_len + mp.out_lo, stage_out_.data(), (out_hi - mp.out_lo) * sizeof(T),
                               cudaMemcpyDeviceToHost, host_stream_));
      FB_CHECK(cudaStreamSynchronize(host_stream_));
    }
  return cudaSuccess;
}

// Chunks of frames 0 .. total-1 of m through seg_, k frames per index (a frame, or an x frame and its y frame): per
// chunk, gather(seg, mc, nq) launches one kernel that writes the chunk's k * nq frames into seg (mc is m with g0 at the
// chunk's first index), the plan's own rfft turns them into spectra (at spec_out + k * q0 spectra, or in seg_ behind
// the frames without spec_out), and use(spec, q0, nq, extra) runs the chunk's consumers, `extra` pointing at `extra`
// bytes per index in seg_ behind the spectra, and adds their launches.
template <typename T>
template <class Gather, class Use>
cudaError_t RealPlan<T>::frame_chunks(const real::FrameMap& m, size_t total, size_t k, C* spec_out, size_t extra,
                                      cudaStream_t s, Gather gather, Use use) {
  const size_t bins = n_ / 2 + 1, frame = n_ * sizeof(T), spectrum = bins * sizeof(C);
  const size_t chunk = scratch_chunk(total, k * (frame + (spec_out ? 0 : spectrum)) + extra);
  auto align = [](size_t bytes) { return (bytes + 255) / 256 * 256; };
  const size_t spec_off = align(k * chunk * frame);
  size_t end = spec_out ? k * chunk * frame : spec_off + k * chunk * spectrum;
  const size_t extra_off = align(end);
  if (extra) end = extra_off + chunk * extra;
  FB_CHECK(seg_.reserve(end));
  char* seg = (char*)seg_.data();
  for (size_t q0 = 0; q0 < total; q0 += chunk) {
    const size_t nq = std::min(chunk, total - q0);
    real::FrameMap mc = m;
    mc.g0 = (long)q0;
    gather((T*)seg, mc, nq);
    FB_CHECK(cudaGetLastError());
    launches_ += 1;
    C* spec = spec_out ? spec_out + k * q0 * bins : (C*)(seg + spec_off);
    FB_CHECK(rfft_rows(true, seg, spec, k * nq, kFft, s));
    FB_CHECK(use(spec, q0, nq, (T*)(seg + extra_off)));
  }
  return cudaSuccess;
}

template <typename T>
cudaError_t RealPlan<T>::stft_device(const T* in, size_t in_len, const T* win, size_t hop, int boundary, C* out,
                                     size_t batch, cudaStream_t s) {
  launches_ = 0;
  if (batch == 0) return cudaSuccess;
  DeviceGuard g(device_);
  return stft_rows(in, in_len, win, hop, boundary, out, batch, s);
}

template <typename T>
cudaError_t RealPlan<T>::stft_rows(const T* in, size_t in_len, const T* win, size_t hop, int boundary, C* out,
                                   size_t batch, cudaStream_t s) {
  const real::FrameMap m = real::frame_map((long)n_, (long)in_len, (long)hop, boundary);
  const size_t total = batch * (size_t)m.frames;
  if (path_ == Path::kRealFused) {
    FB_CHECK(fused_->stft(in, win, out, m, total, twa_.data(), (const C*)tab_.data(), sm_count_, s));
    launches_ += 1;
    return cudaSuccess;
  }
  // the windowed frames, then the plan's own rfft straight into the output rows
  return frame_chunks(
      m, total, 1, out, 0, s,
      [&](T* seg, const real::FrameMap& mc, size_t nq) {
        gather_frames_kernel<T><<<grid_for(nq * n_), kThreads, 0, s>>>(in, win, seg, mc, (long)nq);
      },
      [](C*, size_t, size_t, T*) { return cudaSuccess; });
}

// Runs of frames through seg_ (real::istft_runs): each run's spectra are inverted there by the plan's own irfft, then
// overlap_add_kernel writes the outputs the run owns.  Every output is written once, by the same sum in the same order
// wherever the runs are cut.
template <typename T>
cudaError_t RealPlan<T>::istft_device(const C* in, size_t frames, const T* win, size_t hop, bool center, T* out,
                                      size_t out_len, size_t batch, cudaStream_t s) {
  launches_ = 0;
  if (batch == 0) return cudaSuccess;
  DeviceGuard g(device_);
  return istft_rows(in, frames, win, hop, center, out, out_len, batch, s);
}

template <typename T>
cudaError_t RealPlan<T>::istft_rows(const C* in, size_t frames, const T* win, size_t hop, bool center, T* out,
                                    size_t out_len, size_t batch, cudaStream_t s) {
  real::FrameMap m = real::frame_map((long)n_, (long)n_, (long)hop, real::kStftNone);
  m.pad = center ? (long)n_ / 2 : 0;
  m.frames = (long)frames;
  m.rcp = 1.0 / (double)frames;
  const size_t bins = n_ / 2 + 1;
  // cap <= batch * frames: istft_scratch_frames raises the chunk to at most `frames`
  const size_t cap = real::istft_scratch_frames(scratch_chunk(batch * frames, n_ * sizeof(T)), n_, hop, frames);
  FB_CHECK(seg_.reserve(cap * n_ * sizeof(T)));
  T* seg = (T*)seg_.data();
  return (cudaError_t)real::istft_runs(n_, hop, (size_t)m.pad, frames, out_len, batch, cap,
                                       [&](size_t gs, size_t ge, size_t b0, size_t nb, size_t i0, size_t i1) -> int {
    FB_CHECK(rfft_rows(false, in + gs * bins, seg, ge - gs, kIfft, s));
    overlap_add_kernel<T><<<grid_for(nb * (i1 - i0)), kThreads, 0, s>>>(
        seg, win, out + b0 * out_len, m, (long)gs, (long)b0, (long)nb, (long)i0, (long)i1, (long)out_len);
    FB_CHECK(cudaGetLastError());
    launches_ += 1;
    return 0;
  });
}

template <typename T>
cudaError_t RealPlan<T>::stft_host(const T* in, size_t in_len, const T* win, size_t hop, int boundary, C* out,
                                   size_t batch) {
  launches_ = 0;
  if (batch == 0) return cudaSuccess;
  DeviceGuard g(device_);
  const T* dwin;
  FB_CHECK(stage_consts(win, n_ * sizeof(T), &dwin));
  return stage_rows(in, out, batch, in_len * sizeof(T), stft_row_bytes(in_len, hop, boundary),
                    [&](const void* din, void* dout, size_t, size_t nb) {
                      return stft_rows((const T*)din, in_len, dwin, hop, boundary, (C*)dout, nb, host_stream_);
                    });
}

template <typename T>
cudaError_t RealPlan<T>::istft_host(const C* in, size_t frames, const T* win, size_t hop, bool center, T* out,
                                    size_t out_len, size_t batch) {
  launches_ = 0;
  if (batch == 0) return cudaSuccess;
  DeviceGuard g(device_);
  const T* dwin;
  FB_CHECK(stage_consts(win, n_ * sizeof(T), &dwin));
  return stage_rows(in, out, batch, spec_bytes(frames), out_len * sizeof(T),
                    [&](const void* din, void* dout, size_t, size_t nb) {
                      return istft_rows((const C*)din, frames, dwin, hop, center, (T*)dout, out_len, nb, host_stream_);
                    });
}

// The bands are recomputed on every call: the caller may change the filter matrix between calls.
template <typename T>
cudaError_t RealPlan<T>::mel_bands(const T* filters, size_t n_mels, cudaStream_t s) {
  FB_CHECK(bands_.reserve(n_mels * sizeof(real::Band)));
  mel_bands_kernel<T><<<(unsigned)std::min<size_t>(n_mels, 4096), kThreads, 0, s>>>(
      filters, (long)(n_ / 2 + 1), (long)n_mels, (real::Band*)bands_.data());
  FB_CHECK(cudaGetLastError());
  launches_ += 1;
  return cudaSuccess;
}

template <typename T>
cudaError_t RealPlan<T>::mel_rows(const T* in, size_t in_len, const T* win, size_t hop, int boundary, const T* filters,
                                  size_t n_mels, int power, T* out, size_t batch, cudaStream_t s) {
  const real::FrameMap m = real::frame_map((long)n_, (long)in_len, (long)hop, boundary);
  const size_t total = batch * (size_t)m.frames, bins = n_ / 2 + 1;
  const real::Band* bands = (const real::Band*)bands_.data();
  if (path_ == Path::kRealFused) {
    FB_CHECK(fused_->mel(in, win, filters, bands, n_mels, power, out, m, total, twa_.data(), (const C*)tab_.data(),
                         sm_count_, s));
    launches_ += 1;
    return cudaSuccess;
  }
  // the windowed frames, their spectra behind them, then the mels of those spectra straight into the output rows
  return frame_chunks(
      m, total, 1, nullptr, 0, s,
      [&](T* seg, const real::FrameMap& mc, size_t nq) {
        gather_frames_kernel<T><<<grid_for(nq * n_), kThreads, 0, s>>>(in, win, seg, mc, (long)nq);
      },
      [&](C* spec, size_t q0, size_t nq, T*) {
        mel_spectra_kernel<T><<<grid_for(nq * n_mels), kThreads, 0, s>>>(
            spec, filters, bands, (long)bins, (long)n_mels, power, out + q0 * n_mels, (long)nq, (long)q0);
        FB_CHECK(cudaGetLastError());
        launches_ += 1;
        return cudaSuccess;
      });
}

template <typename T>
cudaError_t RealPlan<T>::mel_device(const T* in, size_t in_len, const T* win, size_t hop, int boundary,
                                    const T* filters, size_t n_mels, int power, T* out, size_t batch, cudaStream_t s) {
  launches_ = 0;
  if (batch == 0) return cudaSuccess;
  DeviceGuard g(device_);
  FB_CHECK(mel_bands(filters, n_mels, s));
  return mel_rows(in, in_len, win, hop, boundary, filters, n_mels, power, out, batch, s);
}

template <typename T>
cudaError_t RealPlan<T>::mel_host(const T* in, size_t in_len, const T* win, size_t hop, int boundary, const T* filters,
                                  size_t n_mels, int power, T* out, size_t batch) {
  launches_ = 0;
  if (batch == 0) return cudaSuccess;
  DeviceGuard g(device_);
  const T *dwin, *dfilt;
  FB_CHECK(stage_consts(win, n_ * sizeof(T), &dwin, filters, n_mels * (n_ / 2 + 1) * sizeof(T), &dfilt));
  FB_CHECK(mel_bands(dfilt, n_mels, host_stream_));
  return stage_rows(in, out, batch, in_len * sizeof(T), mel_row_bytes(in_len, hop, boundary, n_mels),
                    [&](const void* din, void* dout, size_t, size_t nb) {
                      return mel_rows((const T*)din, in_len, dwin, hop, boundary, dfilt, n_mels, power, (T*)dout, nb,
                                      host_stream_);
                    });
}

template <typename T>
cudaError_t RealPlan<T>::mfcc_args(double log_offset, double log_floor, double log_scale, double top_db,
                                   size_t top_db_rows, const T* dct, size_t n_out, double bias, size_t batch,
                                   cudaStream_t s, real::MfccArgs<T>* p) {
  const bool clamp = std::isfinite(top_db);
  p->offset = (T)log_offset;
  p->floor = (T)log_floor;
  p->scale = (T)log_scale;
  p->top_db = clamp ? (T)top_db : (T)0;
  p->bias = (T)bias;
  p->dct = dct;
  p->n_out = (long)n_out;
  p->rows = clamp ? (long)top_db_rows : 0;
  p->row0 = 0;
  p->rows_rcp = clamp ? 1.0 / (double)top_db_rows : 0.0;
  p->slots = nullptr;
  if (clamp) {
    const size_t bytes = batch / top_db_rows * sizeof(real::MaxKey<T>);
    FB_CHECK(slots_.reserve(bytes));
    FB_CHECK(cudaMemsetAsync(slots_.data(), 0, bytes, s));
    p->slots = (real::MaxKey<T>*)slots_.data();
  }
  return cudaSuccess;
}

template <typename T>
cudaError_t RealPlan<T>::mfcc_rows(const T* in, size_t in_len, const T* win, size_t hop, int boundary, int power,
                                   const T* filters, size_t n_mels, const real::MfccArgs<T>& p, bool max_sweep, T* out,
                                   size_t batch, cudaStream_t s) {
  const real::FrameMap m = real::frame_map((long)n_, (long)in_len, (long)hop, boundary);
  const size_t total = batch * (size_t)m.frames, bins = n_ / 2 + 1;
  const real::Band* bands = (const real::Band*)bands_.data();
  if (mfcc_fused(n_mels)) {
    FB_CHECK(fused_->mfcc(in, win, filters, bands, n_mels, power, p, max_sweep, out, m, total, twa_.data(),
                          (const C*)tab_.data(), sm_count_, s));
    launches_ += 1;
    return cudaSuccess;
  }
  // as in mel_rows, the mels into a third region behind the spectra, then mfcc_frames_kernel from there
  return frame_chunks(
      m, total, 1, nullptr, n_mels * sizeof(T), s,
      [&](T* seg, const real::FrameMap& mc, size_t nq) {
        gather_frames_kernel<T><<<grid_for(nq * n_), kThreads, 0, s>>>(in, win, seg, mc, (long)nq);
      },
      [&](C* spec, size_t q0, size_t nq, T* mel) {
        mel_spectra_kernel<T><<<grid_for(nq * n_mels), kThreads, 0, s>>>(spec, filters, bands, (long)bins,
                                                                          (long)n_mels, power, mel, (long)nq, (long)q0);
        FB_CHECK(cudaGetLastError());
        const unsigned grid = (unsigned)std::min<size_t>(nq, (size_t)sm_count_ * 16);
        if (max_sweep)
          mfcc_frames_kernel<T, true><<<grid, kThreads, 0, s>>>(mel, (long)n_mels, p, nullptr, (long)nq, (long)q0,
                                                                m.frames);
        else
          mfcc_frames_kernel<T, false><<<grid, kThreads, 0, s>>>(mel, (long)n_mels, p, out + q0 * p.n_out, (long)nq,
                                                                 (long)q0, m.frames);
        FB_CHECK(cudaGetLastError());
        launches_ += 2;
        return cudaSuccess;
      });
}

template <typename T>
cudaError_t RealPlan<T>::mfcc_device(const T* in, size_t in_len, const T* win, size_t hop, int boundary, int power,
                                     const T* filters, size_t n_mels, double log_offset, double log_floor,
                                     double log_scale, double top_db, size_t top_db_rows, const T* dct, size_t n_out,
                                     double bias, T* out, size_t batch, cudaStream_t s) {
  launches_ = 0;
  if (batch == 0) return cudaSuccess;
  DeviceGuard g(device_);
  real::MfccArgs<T> p;
  FB_CHECK(mfcc_args(log_offset, log_floor, log_scale, top_db, top_db_rows, dct, n_out, bias, batch, s, &p));
  FB_CHECK(mel_bands(filters, n_mels, s));
  if (p.rows) FB_CHECK(mfcc_rows(in, in_len, win, hop, boundary, power, filters, n_mels, p, true, out, batch, s));
  return mfcc_rows(in, in_len, win, hop, boundary, power, filters, n_mels, p, false, out, batch, s);
}

// The max sweep stages every row once more (through stage_rows with no output), in chunks of its own size: the group
// slots are indexed by the call's rows, so where the chunks cut a group does not matter.
template <typename T>
cudaError_t RealPlan<T>::mfcc_host(const T* in, size_t in_len, const T* win, size_t hop, int boundary, int power,
                                   const T* filters, size_t n_mels, double log_offset, double log_floor,
                                   double log_scale, double top_db, size_t top_db_rows, const T* dct, size_t n_out,
                                   double bias, T* out, size_t batch) {
  launches_ = 0;
  if (batch == 0) return cudaSuccess;
  DeviceGuard g(device_);
  const T *dwin, *dfilt, *ddct = nullptr;
  FB_CHECK(stage_consts(win, n_ * sizeof(T), &dwin, filters, n_mels * (n_ / 2 + 1) * sizeof(T), &dfilt));
  if (dct) {
    FB_CHECK(stage_dct_.reserve(n_mels * n_out * sizeof(T)));
    FB_CHECK(cudaMemcpyAsync(stage_dct_.data(), dct, n_mels * n_out * sizeof(T), cudaMemcpyHostToDevice, host_stream_));
    ddct = (const T*)stage_dct_.data();
  }
  real::MfccArgs<T> p;
  FB_CHECK(mfcc_args(log_offset, log_floor, log_scale, top_db, top_db_rows, ddct, n_out, bias, batch, host_stream_, &p));
  FB_CHECK(mel_bands(dfilt, n_mels, host_stream_));
  auto sweep = [&](bool max_sweep, void* dst, size_t out_row) {
    return stage_rows(in, dst, batch, in_len * sizeof(T), out_row, [&](const void* din, void* dout, size_t b0, size_t nb) {
      real::MfccArgs<T> pc = p;
      pc.row0 = (long)b0;
      return mfcc_rows((const T*)din, in_len, dwin, hop, boundary, power, dfilt, n_mels, pc, max_sweep, (T*)dout, nb,
                       host_stream_);
    });
  };
  if (p.rows) FB_CHECK(sweep(true, out, 0));
  return sweep(false, out, mel_row_bytes(in_len, hop, boundary, n_out));
}

template <typename T>
cudaError_t RealPlan<T>::welch_scale(const T* win, int scaling, double fs, size_t frames, cudaStream_t s) {
  FB_CHECK(welch_base_.reserve(sizeof(T)));
  welch_scale_kernel<T><<<1, kThreads, 0, s>>>(win, (long)n_, scaling, fs, (long)frames, (T*)welch_base_.data());
  FB_CHECK(cudaGetLastError());
  launches_ += 1;
  return cudaSuccess;
}

template <typename T>
cudaError_t RealPlan<T>::welch_cross_rows(const T* x, const T* y, size_t y_rows, size_t y_off, size_t in_len,
                                          const T* win, size_t hop, int detrend, bool coh, void* out, size_t batch,
                                          cudaStream_t s) {
  const real::FrameMap m = real::frame_map((long)n_, (long)in_len, (long)hop, real::kStftNone);
  const size_t bins = n_ / 2 + 1, frames = (size_t)m.frames, k = y ? 2 : 1;
  const size_t planes = !y ? 1 : coh ? real::kCoherencePlanes : real::kCsdPlanes;
  const size_t out_row = bins * (y && !coh ? sizeof(C) : sizeof(T));
  const bool fused = path_ == Path::kRealFused;
  const long cols = fused ? fused_->cols / (long)k : 1;
  const size_t items = (size_t)real::welch_items(m.frames, cols, 1).items;
  // the fused kernel writes a row of one item itself; every other row goes through partials and the finish
  const bool direct = fused && items == 1;
  const size_t rows = direct ? batch : scratch_chunk(batch, items * planes * bins * sizeof(T));
  if (!direct) FB_CHECK(part_.reserve(rows * items * planes * bins * sizeof(T)));
  T* part = (T*)part_.data();
  const T* base = (const T*)welch_base_.data();
  for (size_t r0 = 0; r0 < batch; r0 += rows) {
    const size_t nr = std::min(rows, batch - r0), yo = (y_off + r0) % y_rows;
    const real::WelchItems w = real::welch_items(m.frames, cols, (long)nr);
    const T* xr = x + r0 * in_len;
    void* o = (char*)out + r0 * out_row;
    if (fused) {
      if (y)
        FB_CHECK(fused_->csd(xr, y, y_rows, yo, win, base, detrend, coh, part, o, m, w, twa_.data(),
                             (const C*)tab_.data(), sm_count_, s));
      else
        FB_CHECK(fused_->welch(xr, win, base, detrend, part, (T*)o, m, w, twa_.data(), (const C*)tab_.data(),
                               sm_count_, s));
      launches_ += 1;
    } else {
      // the detrended windowed frames (x frames, then their y frames), their spectra behind them, and the items with
      // frames in the chunk accumulated from there
      auto item_of = [&](size_t q) { return (q / frames) * items + (q % frames) / (size_t)w.block; };
      FB_CHECK(frame_chunks(
          m, nr * frames, k, nullptr, 0, s,
          [&](T* seg, const real::FrameMap& mc, size_t nq) {
            const unsigned grid = (unsigned)std::min<size_t>(nq, 132u * 32u);
            if (y)
              csd_gather_kernel<T><<<grid, kThreads, 0, s>>>(xr, y, (long)y_rows, (long)yo, win, seg, mc, (long)nq,
                                                             detrend);
            else
              welch_gather_kernel<T><<<grid, kThreads, 0, s>>>(xr, win, seg, mc, (long)nq, detrend);
          },
          [&](C* spec, size_t q0, size_t nq, T*) {
            const size_t i0 = item_of(q0), ni = item_of(q0 + nq - 1) + 1 - i0;
            if (y)
              cross_accumulate_kernel<T><<<grid_for(ni * bins), kThreads, 0, s>>>(
                  spec, spec + nq * bins, w, (long)bins, (long)q0, (long)nq, (long)i0, (long)ni, (int)planes, part);
            else
              welch_accumulate_kernel<T><<<grid_for(ni * bins), kThreads, 0, s>>>(spec, w, (long)bins, (long)q0,
                                                                                  (long)nq, (long)i0, (long)ni, part);
            FB_CHECK(cudaGetLastError());
            launches_ += 1;
            return cudaSuccess;
          }));
    }
    if (!direct) {
      if (y)
        cross_finish_kernel<T><<<grid_for(nr * bins), kThreads, 0, s>>>(part, (long)items, (long)n_, base, coh, o,
                                                                         (long)nr);
      else
        welch_finish_kernel<T><<<grid_for(nr * bins), kThreads, 0, s>>>(part, (long)items, (long)n_, base, (T*)o,
                                                                         (long)nr);
      FB_CHECK(cudaGetLastError());
      launches_ += 1;
    }
  }
  return cudaSuccess;
}

template <typename T>
cudaError_t RealPlan<T>::welch_device(const T* in, size_t in_len, const T* win, size_t hop, int detrend, int scaling,
                                      double fs, T* out, size_t batch, cudaStream_t s) {
  return cross_device(in, nullptr, 1, in_len, win, hop, detrend, false, scaling, fs, out, batch, s);
}

template <typename T>
cudaError_t RealPlan<T>::welch_host(const T* in, size_t in_len, const T* win, size_t hop, int detrend, int scaling,
                                    double fs, T* out, size_t batch) {
  return cross_host(in, nullptr, 1, in_len, win, hop, detrend, false, scaling, fs, out, batch);
}

template <typename T>
cudaError_t RealPlan<T>::cross_device(const T* x, const T* y, size_t y_rows, size_t in_len, const T* win, size_t hop,
                                      int detrend, bool coh, int scaling, double fs, void* out, size_t batch,
                                      cudaStream_t s) {
  launches_ = 0;
  if (batch == 0) return cudaSuccess;
  DeviceGuard g(device_);
  if (!coh) FB_CHECK(welch_scale(win, scaling, fs, frame_count(in_len, hop, real::kStftNone), s));
  return welch_cross_rows(x, y, y_rows, 0, in_len, win, hop, detrend, coh, out, batch, s);
}

template <typename T>
cudaError_t RealPlan<T>::cross_host(const T* x, const T* y, size_t y_rows, size_t in_len, const T* win, size_t hop,
                                    int detrend, bool coh, int scaling, double fs, void* out, size_t batch) {
  launches_ = 0;
  if (batch == 0) return cudaSuccess;
  DeviceGuard g(device_);
  const T* dwin;
  FB_CHECK(stage_consts(win, n_ * sizeof(T), &dwin));
  if (!coh) FB_CHECK(welch_scale(dwin, scaling, fs, frame_count(in_len, hop, real::kStftNone), host_stream_));
  const size_t row = in_len * sizeof(T), bins = n_ / 2 + 1;
  return stage_rows(x, out, batch, row, bins * (y && !coh ? sizeof(C) : sizeof(T)),
                    [&](const void* din, void* dout, size_t b0, size_t nb) {
                      // y rows (b0 + j) mod y_rows, j < cnt, in one or two runs: row b of the chunk pairs with j =
                      // b mod cnt
                      const T* dy = nullptr;
                      const size_t cnt = std::min(nb, y_rows), first = b0 % y_rows;
                      if (y) {
                        const size_t run = std::min(cnt, y_rows - first);
                        FB_CHECK(stage_y_.reserve(cnt * row));
                        FB_CHECK(cudaMemcpyAsync(stage_y_.data(), y + first * in_len, run * row,
                                                 cudaMemcpyHostToDevice, host_stream_));
                        if (run < cnt)
                          FB_CHECK(cudaMemcpyAsync((char*)stage_y_.data() + run * row, y, (cnt - run) * row,
                                                   cudaMemcpyHostToDevice, host_stream_));
                        dy = (const T*)stage_y_.data();
                      }
                      return welch_cross_rows((const T*)din, dy, cnt, 0, in_len, dwin, hop, detrend, coh, dout, nb,
                                              host_stream_);
                    });
}

template <typename T>
cudaError_t RealPlan<T>::dct_device(const T* in, T* out, size_t batch, int type, int norm, cudaStream_t s) {
  launches_ = 0;
  if (batch == 0) return cudaSuccess;
  DeviceGuard g(device_);
  return dct_rows(in, out, batch, type, norm, s);
}

template <typename T>
cudaError_t RealPlan<T>::dct_rows(const T* in, T* out, size_t batch, int type, int norm, cudaStream_t s) {
  double hd, h0d;
  real::dct_scales(type, norm, (long)n_, hd, h0d);
  const T h = (T)hd, h0 = (T)h0d;
  const C* wq = (const C*)dct_tab_.data();
  const C* tab = (const C*)tab_.data();
  if (path_ == Path::kRealFused) {
    FB_CHECK(fused_->dct(in, out, type, twa_.data(), tab, wq, batch, h, h0, sm_count_, s));
    launches_ += 1;
    return cudaSuccess;
  }
  // chunks of rows through seg_: N reals per row (half length) or N complex values (full length); the first kernel reads
  // the chunk's input rows whole and only the last one writes its output rows, so in == out is safe
  const bool half = path_ == Path::kRealHalf;
  const size_t row = half ? n_ * sizeof(T) : n_ * sizeof(C);
  const size_t chunk = scratch_chunk(batch, row);
  FB_CHECK(seg_.reserve(chunk * row));
  void* seg = seg_.data();
  for (size_t b0 = 0; b0 < batch; b0 += chunk) {
    const size_t nb = std::min(chunk, batch - b0);
    const T* x = in + b0 * n_;
    T* y = out + b0 * n_;
    if (half) {
      const unsigned pairs = grid_for((m_ / 2 + 1) * nb);
      if (type == 2) {
        dct_permute_kernel<T, false><<<grid_for(nb * n_), kThreads, 0, s>>>(x, seg, (long)n_, (long)nb);
        FB_CHECK(cudaGetLastError());
        FB_CHECK(inner_->exec_device((C*)seg, (C*)seg, nb, kFft, s));
        dct_untangle_kernel<T><<<pairs, kThreads, 0, s>>>((const C*)seg, y, tab, wq, (long)m_, (long)nb, h, h0);
      } else {
        dct_tangle_kernel<T><<<pairs, kThreads, 0, s>>>(x, (C*)seg, tab, wq, (long)m_, (long)nb, h, h0);
        FB_CHECK(cudaGetLastError());
        FB_CHECK(inner_->exec_device((C*)seg, (C*)seg, nb, kUnscaledIfft, s));
        dct_unpermute_kernel<T, false><<<grid_for(nb * n_), kThreads, 0, s>>>(seg, y, (long)n_, (long)nb);
      }
    } else {
      if (type == 2) {
        dct_permute_kernel<T, true><<<grid_for(nb * n_), kThreads, 0, s>>>(x, seg, (long)n_, (long)nb);
        FB_CHECK(cudaGetLastError());
        FB_CHECK(inner_->exec_device((C*)seg, (C*)seg, nb, kFft, s));
        dct_post_kernel<T><<<grid_for((n_ / 2 + 1) * nb), kThreads, 0, s>>>((const C*)seg, y, wq, (long)n_, (long)nb, h,
                                                                           h0);
      } else {
        dct_pre_kernel<T><<<grid_for(nb * n_), kThreads, 0, s>>>(x, (C*)seg, wq, (long)n_, (long)nb, h, h0);
        FB_CHECK(cudaGetLastError());
        FB_CHECK(inner_->exec_device((C*)seg, (C*)seg, nb, kUnscaledIfft, s));
        dct_unpermute_kernel<T, true><<<grid_for(nb * n_), kThreads, 0, s>>>(seg, y, (long)n_, (long)nb);
      }
    }
    FB_CHECK(cudaGetLastError());
    launches_ += 2 + inner_->launches();
  }
  return cudaSuccess;
}

template <typename T>
cudaError_t RealPlan<T>::dct_host(const T* in, T* out, size_t batch, int type, int norm) {
  launches_ = 0;
  if (batch == 0) return cudaSuccess;
  DeviceGuard g(device_);
  return stage_rows(in, out, batch, n_ * sizeof(T), n_ * sizeof(T), [&](const void* din, void* dout, size_t, size_t nb) {
    return dct_rows((const T*)din, (T*)dout, nb, type, norm, host_stream_);
  });
}

template <typename T>
cudaError_t RealPlan<T>::hilbert_device(const T* in, void* out, size_t batch, int output, cudaStream_t s) {
  launches_ = 0;
  if (batch == 0) return cudaSuccess;
  DeviceGuard g(device_);
  return hilbert_rows(in, out, batch, output, s);
}

template <typename T>
cudaError_t RealPlan<T>::hilbert_rows(const T* in, void* out, size_t batch, int output, cudaStream_t s) {
  const C* tab = (const C*)tab_.data();
  if (path_ == Path::kRealFused) {
    FB_CHECK(fused_->hilbert(in, out, output, twa_.data(), tab, batch, (T)1 / (T)(2 * n_), sm_count_, s));
    launches_ += 1;
    return cudaSuccess;
  }
  // chunks of rows through seg_: y of N reals per row (half length) or N complex values (full length); only the last
  // kernel of a chunk writes its output rows, after reading their input, so in == out is safe
  const bool half = path_ == Path::kRealHalf;
  const size_t row = half ? n_ * sizeof(T) : n_ * sizeof(C);
  const size_t out_row = output == real::kHilbertAnalytic ? n_ * sizeof(C) : n_ * sizeof(T);
  const size_t chunk = scratch_chunk(batch, row);
  FB_CHECK(seg_.reserve(chunk * row));
  C* w = (C*)seg_.data();
  for (size_t b0 = 0; b0 < batch; b0 += chunk) {
    const size_t nb = std::min(chunk, batch - b0);
    const T* x = in + b0 * n_;
    void* y = (char*)out + b0 * out_row;
    if (half) {
      FB_CHECK(inner_->exec_device((const C*)x, w, nb, kFft, s));
      launches_ += inner_->launches();
      hilbert_pair_kernel<T><<<grid_for((m_ / 2 + 1) * nb), kThreads, 0, s>>>(w, tab, (long)m_, (long)nb,
                                                                              (T)1 / (T)(2 * n_));
      FB_CHECK(cudaGetLastError());
      FB_CHECK(inner_->exec_device(w, w, nb, kUnscaledIfft, s));
      launches_ += inner_->launches();
      hilbert_out_kernel<T, false><<<grid_for(nb * n_), kThreads, 0, s>>>(x, w, y, (long)n_, (long)nb, output);
    } else {
      widen_kernel<T><<<grid_for(nb * n_), kThreads, 0, s>>>(x, w, nb * n_);
      FB_CHECK(cudaGetLastError());
      FB_CHECK(inner_->exec_device(w, w, nb, kFft, s));
      launches_ += inner_->launches();
      hilbert_mul_kernel<T><<<grid_for(nb * n_), kThreads, 0, s>>>(w, (long)n_, (long)nb, (T)1 / (T)n_);
      FB_CHECK(cudaGetLastError());
      FB_CHECK(inner_->exec_device(w, w, nb, kUnscaledIfft, s));
      launches_ += inner_->launches();
      hilbert_out_kernel<T, true><<<grid_for(nb * n_), kThreads, 0, s>>>(x, w, y, (long)n_, (long)nb, output);
      launches_ += 1;
    }
    FB_CHECK(cudaGetLastError());
    launches_ += 2;
  }
  return cudaSuccess;
}

template <typename T>
cudaError_t RealPlan<T>::hilbert_host(const T* in, void* out, size_t batch, int output) {
  launches_ = 0;
  if (batch == 0) return cudaSuccess;
  DeviceGuard g(device_);
  const size_t out_row = output == real::kHilbertAnalytic ? n_ * sizeof(C) : n_ * sizeof(T);
  return stage_rows(in, out, batch, n_ * sizeof(T), out_row, [&](const void* din, void* dout, size_t, size_t nb) {
    return hilbert_rows((const T*)din, dout, nb, output, host_stream_);
  });
}

template <typename T>
cudaError_t RealPlan<T>::dct4_device(const T* in, T* out, size_t batch, int norm, cudaStream_t s) {
  launches_ = 0;
  if (batch == 0) return cudaSuccess;
  DeviceGuard g(device_);
  return dct4_rows(in, out, batch, norm, seg_, s);
}

template <typename T>
cudaError_t RealPlan<T>::dct4_rows(const T* in, T* out, size_t batch, int norm, DeviceBuffer& scratch, cudaStream_t s) {
  const C c = dct4_c<T>(norm, n_);
  const C* wq = (const C*)dct_tab_.data();
  if (path_ == Path::kRealFused) {
    FB_CHECK(fused_->dct4(in, out, twa_.data(), wq, c, batch, sm_count_, s));
    launches_ += 1;
    return cudaSuccess;
  }
  // chunks of rows through scratch, M complex values per row; the pre kernel reads the chunk's rows whole and only the
  // post kernel writes them, so in == out is safe
  const size_t chunk = scratch_chunk(batch, n_ * sizeof(T));
  FB_CHECK(scratch.reserve(chunk * n_ * sizeof(T)));
  C* z = (C*)scratch.data();
  for (size_t b0 = 0; b0 < batch; b0 += chunk) {
    const size_t nb = std::min(chunk, batch - b0);
    dct4_pre_kernel<T><<<grid_for(nb * m_), kThreads, 0, s>>>(in + b0 * n_, z, wq, (long)n_, (long)nb);
    FB_CHECK(cudaGetLastError());
    FB_CHECK(inner_->exec_device(z, z, nb, kFft, s));
    dct4_post_kernel<T><<<grid_for(nb * m_), kThreads, 0, s>>>(z, out + b0 * n_, wq, c, (long)n_, (long)nb, (long)b0);
    FB_CHECK(cudaGetLastError());
    launches_ += 2 + inner_->launches();
  }
  return cudaSuccess;
}

template <typename T>
cudaError_t RealPlan<T>::dct4_host(const T* in, T* out, size_t batch, int norm) {
  launches_ = 0;
  if (batch == 0) return cudaSuccess;
  DeviceGuard g(device_);
  return stage_rows(in, out, batch, n_ * sizeof(T), n_ * sizeof(T), [&](const void* din, void* dout, size_t, size_t nb) {
    return dct4_rows((const T*)din, (T*)dout, nb, norm, seg_, host_stream_);
  });
}

template <typename T>
cudaError_t RealPlan<T>::mdct_device(const T* in, size_t in_len, const T* win, bool center, int norm, T* out,
                                     size_t batch, cudaStream_t s) {
  launches_ = 0;
  if (batch == 0) return cudaSuccess;
  DeviceGuard g(device_);
  return mdct_rows(in, in_len, win, center, norm, out, batch, s);
}

template <typename T>
cudaError_t RealPlan<T>::mdct_rows(const T* in, size_t in_len, const T* win, bool center, int norm, T* out,
                                   size_t batch, cudaStream_t s) {
  const real::FrameMap m = real::mdct_map((long)n_, (long)in_len, center);
  const size_t total = batch * (size_t)m.frames;
  const C c = dct4_c<T>(norm, n_);
  const C* wq = (const C*)dct_tab_.data();
  if (path_ == Path::kRealFused) {
    FB_CHECK(fused_->mdct(in, win, out, m, total, twa_.data(), wq, c, sm_count_, s));
    launches_ += 1;
    return cudaSuccess;
  }
  // chunks of frames through seg_: the gather frames, windows, folds and pre-twiddles them, the inner plan transforms
  // them in place, and the post kernel writes their coefficients
  const size_t chunk = scratch_chunk(total, n_ * sizeof(T));
  FB_CHECK(seg_.reserve(chunk * n_ * sizeof(T)));
  C* z = (C*)seg_.data();
  for (size_t q0 = 0; q0 < total; q0 += chunk) {
    const size_t nq = std::min(chunk, total - q0);
    real::FrameMap mc = m;
    mc.g0 = (long)q0;
    mdct_gather_kernel<T><<<grid_for(nq * m_), kThreads, 0, s>>>(in, win, z, mc, wq, (long)nq);
    FB_CHECK(cudaGetLastError());
    FB_CHECK(inner_->exec_device(z, z, nq, kFft, s));
    dct4_post_kernel<T><<<grid_for(nq * m_), kThreads, 0, s>>>(z, out + q0 * n_, wq, c, (long)n_, (long)nq, (long)q0);
    FB_CHECK(cudaGetLastError());
    launches_ += 2 + inner_->launches();
  }
  return cudaSuccess;
}

// Runs of frames through seg_ (real::istft_runs with frames of 2N samples every N): each run's DCT-IV goes into seg_
// (dct4_rows, its own scratch in work_), then imdct_overlap_add_kernel writes the outputs the run owns.  Every output
// is written once, by the same sum in the same order wherever the runs are cut.
template <typename T>
cudaError_t RealPlan<T>::imdct_device(const T* in, size_t frames, const T* win, bool center, int norm, T* out,
                                      size_t out_len, size_t batch, cudaStream_t s) {
  launches_ = 0;
  if (batch == 0) return cudaSuccess;
  DeviceGuard g(device_);
  return imdct_rows(in, frames, win, center, norm, out, out_len, batch, s);
}

template <typename T>
cudaError_t RealPlan<T>::imdct_rows(const T* in, size_t frames, const T* win, bool center, int norm, T* out,
                                    size_t out_len, size_t batch, cudaStream_t s) {
  real::FrameMap m = real::mdct_map((long)n_, 2 * (long)n_, center);
  m.frames = (long)frames;
  m.rcp = 1.0 / (double)frames;
  const int inv = real::dct_swapped_norm(norm);
  // cap <= batch * frames: istft_scratch_frames raises the chunk to at most `frames`
  const size_t cap = real::istft_scratch_frames(scratch_chunk(batch * frames, n_ * sizeof(T)), 2 * n_, n_, frames);
  FB_CHECK(seg_.reserve(cap * n_ * sizeof(T)));
  T* seg = (T*)seg_.data();
  return (cudaError_t)real::istft_runs(2 * n_, n_, (size_t)m.pad, frames, out_len, batch, cap,
                                       [&](size_t gs, size_t ge, size_t b0, size_t nb, size_t i0, size_t i1) -> int {
    FB_CHECK(dct4_rows(in + gs * n_, seg, ge - gs, inv, work_, s));
    imdct_overlap_add_kernel<T><<<grid_for(nb * (i1 - i0)), kThreads, 0, s>>>(
        seg, win, out + b0 * out_len, m, (long)gs, (long)b0, (long)nb, (long)i0, (long)i1, (long)out_len);
    FB_CHECK(cudaGetLastError());
    launches_ += 1;
    return 0;
  });
}

template <typename T>
cudaError_t RealPlan<T>::mdct_host(const T* in, size_t in_len, const T* win, bool center, int norm, T* out,
                                   size_t batch) {
  launches_ = 0;
  if (batch == 0) return cudaSuccess;
  DeviceGuard g(device_);
  const T* dwin;
  FB_CHECK(stage_consts(win, 2 * n_ * sizeof(T), &dwin));
  return stage_rows(in, out, batch, in_len * sizeof(T), mdct_frames(in_len, center) * n_ * sizeof(T),
                    [&](const void* din, void* dout, size_t, size_t nb) {
                      return mdct_rows((const T*)din, in_len, dwin, center, norm, (T*)dout, nb, host_stream_);
                    });
}

template <typename T>
cudaError_t RealPlan<T>::imdct_host(const T* in, size_t frames, const T* win, bool center, int norm, T* out,
                                    size_t out_len, size_t batch) {
  launches_ = 0;
  if (batch == 0) return cudaSuccess;
  DeviceGuard g(device_);
  const T* dwin;
  FB_CHECK(stage_consts(win, 2 * n_ * sizeof(T), &dwin));
  return stage_rows(in, out, batch, frames * n_ * sizeof(T), out_len * sizeof(T),
                    [&](const void* din, void* dout, size_t, size_t nb) {
                      return imdct_rows((const T*)din, frames, dwin, center, norm, (T*)dout, out_len, nb, host_stream_);
                    });
}

template class RealPlan<float>;
template class RealPlan<double>;

}  // namespace fb200
