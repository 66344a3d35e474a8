/*
 * fourier_b200.h -- additive entry points of libfourier.so that the reference ABI has no
 * counterpart for: batched transforms, device-resident buffers, caller-supplied CUDA streams,
 * device selection and plan introspection.  Nothing here changes the eight reference symbols
 * declared in fourier.h.
 *
 * Why they exist: the reference's hot path is Fft::transform_in_place on ONE transform
 * (fourier-algorithms/src/fft.rs:48); a GPU needs many independent transforms per call to fill
 * 132 SMs and HBM, and callers that already hold data on the device must not pay PCIe.  A batch
 * is `batch` contiguous transforms of size() samples each: transform b occupies samples
 * [b*size, (b+1)*size).  Every transform of a batch is independent, exactly as if the reference's
 * transform() were called in a loop (fourier-bench/benches/fft_bench.rs:36).
 *
 * All functions return 0 on success and a non-zero cudaError_t value otherwise;
 * fourier_b200_last_error() returns a description for the calling thread.
 */
#ifndef FOURIER_B200_H_
#define FOURIER_B200_H_

#include "fourier.h"

#ifdef __cplusplus
extern "C" {
#define FB200_F ::fourier::c::fourier_fft_float
#define FB200_D ::fourier::c::fourier_fft_double
#else
#define FB200_F struct fourier_fft_float
#define FB200_D struct fourier_fft_double
#endif
#define FB200_PLAN_F const FB200_F
#define FB200_PLAN_D const FB200_D

/* Device used by plans created afterwards on this thread (default: the current CUDA device). */
int fourier_b200_set_device(int device);
int fourier_b200_get_device(void);
int fourier_b200_device_count(void);

/* Batched Fft::transform (in != out) / Fft::transform_in_place (in == out).  Pointers may be host
 * memory (pipelined H2D -> transform -> D2H, returns when `out` is complete) or device memory on
 * the plan's GPU (enqueued on the plan's stream and synchronised before returning). */
int fourier_b200_transform_batch_float(FB200_PLAN_F *plan, const void *in, void *out, size_t batch,
                                       int transform);
int fourier_b200_transform_batch_double(FB200_PLAN_D *plan, const void *in, void *out, size_t batch,
                                        int transform);

/* Device pointers only; enqueued on `cuda_stream` (a cudaStream_t, NULL = default stream) and NOT
 * synchronised: the call returns as soon as the kernels are queued.
 * Device buffers (here and above) must be 16-byte aligned (cudaMalloc / torch allocations are; a slice that
 * starts at an odd f32 sample is not): a misaligned pointer is refused with cudaErrorMisalignedAddress.
 * A plan owns ONE set of scratch buffers and work-queue counters: besides "not two threads at once" (a plan is
 * Send, not Sync, as in the reference) this means ONE STREAM AT A TIME -- do not enqueue a plan on a second
 * stream while a call on another stream is still running; use one plan per stream. */
int fourier_b200_transform_batch_async_float(FB200_PLAN_F *plan, const void *in_dev, void *out_dev,
                                             size_t batch, int transform, void *cuda_stream);
int fourier_b200_transform_batch_async_double(FB200_PLAN_D *plan, const void *in_dev, void *out_dev,
                                              size_t batch, int transform, void *cuda_stream);

/* Plan introspection (Fft::size, fourier-algorithms/src/fft.rs:45, and the chosen strategy). */
struct fourier_b200_plan_info {
  size_t size;        /* transform length N */
  int path;           /* 0 trivial, 1 onchip, 2 twopass, 3 global_stages, 4 bluestein, 5 bluestein_fused, 6 onchip_cta, 7 threepass;
                         real plans: 8 real_fused, 9 real_half, 10 real_full */
  size_t inner_size;  /* Bluestein inner length next_pow2(2N-1) (bluesteins.rs:110); real plans: length of the inner
                         complex plan (N/2 for real_half, N for real_full, 0 for real_fused); else 0 */
  int inner_path;
  size_t n1, n2;      /* two-pass split N = n1*n2 (real plans: that of the inner plan), else 0 */
  int precision_bytes;
  int device;
  size_t table_bytes; /* twiddle / chirp tables resident in HBM */
  unsigned long long last_launches; /* kernels launched by the most recent transform call */
};
int fourier_b200_plan_info_float(FB200_PLAN_F *plan, struct fourier_b200_plan_info *out);
int fourier_b200_plan_info_double(FB200_PLAN_D *plan, struct fourier_b200_plan_info *out);
const char *fourier_b200_path_name(int path);
/* Name of the kernel that moves (nearly) all of the plan's bytes, as a profiler lists it. */
const char *fourier_b200_plan_kernel_float(FB200_PLAN_F *plan);
const char *fourier_b200_plan_kernel_double(FB200_PLAN_D *plan);

/* Plans restricted to the general one-kernel-per-stage path (testing / comparison). */
FB200_F *fourier_b200_create_general_float(size_t size);
FB200_D *fourier_b200_create_general_double(size_t size);

/* Synthetic benchmark input on the device: scalars [first_scalar, first_scalar+count) of the
 * counter-hash stream with `seed`, uniform in [-1, 1) (re of sample s is scalar 2s, im 2s+1). */
int fourier_b200_fill_input_float(void *dev_out, unsigned long long first_scalar, size_t count,
                                  unsigned long long seed, void *cuda_stream);
int fourier_b200_fill_input_double(void *dev_out, unsigned long long first_scalar, size_t count,
                                   unsigned long long seed, void *cuda_stream);

/* Building blocks of the distributed six-step transform (one huge N = N1*N2 over several GPUs with
 * all-to-all transposes between local batched FFTs; fourier_b200/distributed.py drives them):
 * batched 2-D transpose out[b][c][r] = in[b][r][c], and data[r][c] *= w_N^{(row0+r)*c} (conj if !forward)
 * with the index reduced exactly mod N.  Device pointers, enqueued on cuda_stream. */
int fourier_b200_transpose_float(const void *in_dev, void *out_dev, size_t batch, size_t rows, size_t cols,
                                 void *cuda_stream);
int fourier_b200_transpose_double(const void *in_dev, void *out_dev, size_t batch, size_t rows, size_t cols,
                                  void *cuda_stream);
/* Pack step of a pipelined exchange: batched transpose of column blocks of a row-major matrix with leading
 * dimension ld, optionally fused with the inter-step twiddle (twiddle = 0 none, 1 forward, 2 inverse):
 *   out[b*out_batch_stride + c*rows + r] = in[b*in_batch_stride + r*ld + c] * w_N^{(row0+r)*(col0+b*in_batch_stride+c)} */
int fourier_b200_pack_float(const void *in_dev, void *out_dev, size_t batch, size_t rows, size_t cols, size_t ld,
                            size_t in_batch_stride, size_t out_batch_stride, int twiddle, unsigned long long row0,
                            unsigned long long col0, unsigned long long n_total, void *cuda_stream);
int fourier_b200_pack_double(const void *in_dev, void *out_dev, size_t batch, size_t rows, size_t cols, size_t ld,
                             size_t in_batch_stride, size_t out_batch_stride, int twiddle, unsigned long long row0,
                             unsigned long long col0, unsigned long long n_total, void *cuda_stream);
/* The whole exchange as ONE kernel over NVLink peer memory: rank `me` of `nranks` holds `rows` rows of
 * ld = nranks*cb columns and stores columns [q*cb, (q+1)*cb) transposed into rank q's buffer outs[q]
 * (device pointers valid on this GPU: own memory for q == me, fourier_b200_peer_open()ed memory otherwise):
 *   outs[q][out_off + c*out_ld + r] = in[r*ld + q*cb + c] * w_N^{(row0+r)*(q*cb+c)}      (twiddle as above)
 * `outs` is a HOST array of nranks pointers.  The caller orders ranks with a stream-ordered barrier. */
int fourier_b200_exchange_float(const void *in_dev, void *const *outs, int nranks, int me, size_t rows, size_t cb,
                                size_t ld, size_t out_ld, size_t out_off, int twiddle, unsigned long long row0,
                                unsigned long long n_total, void *cuda_stream);
int fourier_b200_exchange_double(const void *in_dev, void *const *outs, int nranks, int me, size_t rows, size_t cb,
                                 size_t ld, size_t out_ld, size_t out_off, int twiddle, unsigned long long row0,
                                 unsigned long long n_total, void *cuda_stream);
/* The row FFTs of a step AND the exchange that follows them as one pass over the data: `rows` contiguous rows of the
 * plan's size N are transformed (unscaled; forward != 0: Fft, else UnscaledIfft) and the last register stage of the
 * transform stores its results straight into the destination ranks' buffers, transposed and twiddled:
 *   outs[q][c*out_ld + out_off + r] = FFT_N(in[r*N ..])[q*cb + c] * w_Ntot^{(row0+r)*(q*cb+c)},   cb = N / nranks
 * i.e. what fourier_b200_transform_batch_async_* followed by fourier_b200_exchange_* delivers, with one kernel and
 * one sweep over HBM less and the NVLink stores overlapping the butterflies.  Two-pass plans only (power-of-two N,
 * 2^11 .. 2^20 f32 / 2^9 .. 2^16 f64); nranks a power of two; rows a multiple of the tile height (32 up to N = 2^12 (f32), 8 from 2^17, else 16); twiddle 0,
 * 1 (with forward) or 2 (with inverse); `in` is left intact.  Returns cudaErrorNotSupported (801) for other plans. */
int fourier_b200_fft_rows_exchange_float(const FB200_F *plan, const void *in_dev, size_t rows,
                                         int forward, void *const *outs, int nranks, size_t out_ld, size_t out_off,
                                         int twiddle, unsigned long long row0, unsigned long long n_total,
                                         void *cuda_stream);
int fourier_b200_fft_rows_exchange_double(const FB200_D *plan, const void *in_dev, size_t rows,
                                          int forward, void *const *outs, int nranks, size_t out_ld, size_t out_off,
                                          int twiddle, unsigned long long row0, unsigned long long n_total,
                                          void *cuda_stream);
/* Buffers other ranks of the box (one process per GPU) can store into: cudaMalloc + CUDA IPC.  `handle64` is
 * the 64-byte cudaIpcMemHandle_t to send to the peers (any transport), who open it with _peer_open. */
int fourier_b200_peer_alloc(size_t bytes, void **dev_ptr, void *handle64);
int fourier_b200_peer_open(const void *handle64, void **dev_ptr);
int fourier_b200_peer_close(void *dev_ptr);
int fourier_b200_peer_free(void *dev_ptr);
/* out[b][a][i] = in[a][b][i] (i < inner contiguous): unpack step after an all-to-all */
int fourier_b200_swap_leading_float(const void *in_dev, void *out_dev, size_t a, size_t b, size_t inner,
                                    void *cuda_stream);
int fourier_b200_swap_leading_double(const void *in_dev, void *out_dev, size_t a, size_t b, size_t inner,
                                     void *cuda_stream);
int fourier_b200_twiddle_rows_float(void *data_dev, size_t rows, size_t cols, unsigned long long row0,
                                    unsigned long long n_total, int forward, void *cuda_stream);
int fourier_b200_twiddle_rows_double(void *data_dev, size_t rows, size_t cols, unsigned long long row0,
                                     unsigned long long n_total, int forward, void *cuda_stream);

/* ---- Real-input transforms (numpy's rfft / irfft) ----
 * A plan for real length N >= 1.  Forward: `batch` rows of N reals -> `batch` rows of N/2+1 complex bins, row b
 * starting at complex element b*(N/2+1); transform Fft (0) or SqrtScaledFft (3, times 1/sqrt(N)).  Inverse: the
 * other way round; Ifft (1) is numpy.fft.irfft(X, n=N), UnscaledIfft (2) N times that, SqrtScaledIfft (4) sqrt(N)
 * times that.  Scales are relative to N.  The inverse ignores the imaginary part of bin 0 and, for even N, of bin
 * N/2; the forward writes them as exactly +0.  A code of the other direction, or an unknown one, is refused with
 * cudaErrorInvalidValue.  Out of place only: overlapping `in` and `out` are refused with cudaErrorInvalidValue.
 * batch == 0 succeeds and launches nothing.  create returns NULL for N = 0 and without a usable device.
 * Alignment: device base pointers must be 16-byte aligned (cudaErrorMisalignedAddress otherwise).  Spectrum rows
 * need not be: for f32 with N a multiple of 4 (every power of two), N/2+1 is odd and every odd row starts 8 bytes
 * off a 16-byte boundary; the kernels move the spectrum one complex value (8 bytes) at a time.
 * The synchronous calls take host or device memory (both alike) and return when `out` is complete; host memory
 * is staged through the plan's device buffers in chunks and gives the same bits.  The _async calls take device
 * memory, are enqueued on `cuda_stream` and not synchronised.  Threading as for complex plans: Send, not Sync,
 * one stream at a time. */
struct fourier_b200_rfft_float;
struct fourier_b200_rfft_double;
struct fourier_b200_rfft_float *fourier_b200_rfft_create_float(size_t n);
struct fourier_b200_rfft_double *fourier_b200_rfft_create_double(size_t n);
void fourier_b200_rfft_destroy_float(struct fourier_b200_rfft_float *plan);
void fourier_b200_rfft_destroy_double(struct fourier_b200_rfft_double *plan);
int fourier_b200_rfft_forward_float(struct fourier_b200_rfft_float *plan, const float *in, void *out, size_t batch,
                                    int transform);
int fourier_b200_rfft_forward_double(struct fourier_b200_rfft_double *plan, const double *in, void *out,
                                     size_t batch, int transform);
int fourier_b200_rfft_forward_async_float(struct fourier_b200_rfft_float *plan, const float *in_dev, void *out_dev,
                                          size_t batch, int transform, void *cuda_stream);
int fourier_b200_rfft_forward_async_double(struct fourier_b200_rfft_double *plan, const double *in_dev,
                                           void *out_dev, size_t batch, int transform, void *cuda_stream);
int fourier_b200_rfft_inverse_float(struct fourier_b200_rfft_float *plan, const void *in, float *out, size_t batch,
                                    int transform);
int fourier_b200_rfft_inverse_double(struct fourier_b200_rfft_double *plan, const void *in, double *out,
                                     size_t batch, int transform);
int fourier_b200_rfft_inverse_async_float(struct fourier_b200_rfft_float *plan, const void *in_dev, float *out_dev,
                                          size_t batch, int transform, void *cuda_stream);
int fourier_b200_rfft_inverse_async_double(struct fourier_b200_rfft_double *plan, const void *in_dev,
                                           double *out_dev, size_t batch, int transform, void *cuda_stream);
/* path 8 / 9 / 10; inner_size, inner_path, n1, n2 describe the inner complex plan; last_launches counts every
 * kernel of the last call */
int fourier_b200_rfft_info_float(const struct fourier_b200_rfft_float *plan, struct fourier_b200_plan_info *out);
int fourier_b200_rfft_info_double(const struct fourier_b200_rfft_double *plan, struct fourier_b200_plan_info *out);
const char *fourier_b200_rfft_kernel_float(const struct fourier_b200_rfft_float *plan);
const char *fourier_b200_rfft_kernel_double(const struct fourier_b200_rfft_double *plan);

/* ---- Convolution of real rows, y = irfft(rfft(x) . H) ----
 * On a real plan of length N: out[b] = numpy.fft.irfft(numpy.fft.rfft(in[b]) * H[b mod F], n=N) for `batch` rows of
 * N reals, where `spectrum` holds F = spectrum_rows >= 1 rows of N/2+1 complex bins in exactly the layout the plan's
 * rfft writes (row f starting at complex element f*(N/2+1)).  With H = rfft(h) this is the circular convolution
 * out[b][n] = sum_m in[b][m] h[(n-m) mod N]; F = 1 applies one filter to every row, F = C one filter per channel of
 * rows ordered (batch, channel), F = batch one per row.  Correlation is the same call with conj(H).  The imaginary
 * parts of the products at bin 0 and, for even N, bin N/2 are ignored, as irfft ignores them.  Linear convolution:
 * zero-pad x and h to N >= len(x) + len(h) - 1.  One launch on the real_fused path, 2 x (inner plan) + 1 on
 * real_half, 3 + 2 x (inner plan) per scratch chunk on real_full; last_launches of the info call reports it.
 * `in` and `out` must be the same buffer (in place) or disjoint, and `spectrum` must not overlap `out`
 * (cudaErrorInvalidValue otherwise); a NULL argument or spectrum_rows == 0 is refused with cudaErrorInvalidValue.
 * batch == 0 succeeds and launches nothing.  Device pointers must be 16-byte aligned (cudaErrorMisalignedAddress).
 * The synchronous calls take all three buffers as host memory or all three as device memory (a mix is refused with
 * cudaErrorInvalidValue) and return when `out` is complete; host memory gives the same bits.  The _async calls take
 * device memory, are enqueued on `cuda_stream` and not synchronised.  Threading as for the plan: Send, not Sync. */
int fourier_b200_convolve_real_float(struct fourier_b200_rfft_float *plan, const float *in, const void *spectrum,
                                     size_t spectrum_rows, float *out, size_t batch);
int fourier_b200_convolve_real_double(struct fourier_b200_rfft_double *plan, const double *in, const void *spectrum,
                                      size_t spectrum_rows, double *out, size_t batch);
int fourier_b200_convolve_real_async_float(struct fourier_b200_rfft_float *plan, const float *in_dev,
                                           const void *spectrum_dev, size_t spectrum_rows, float *out_dev,
                                           size_t batch, void *cuda_stream);
int fourier_b200_convolve_real_async_double(struct fourier_b200_rfft_double *plan, const double *in_dev,
                                            const void *spectrum_dev, size_t spectrum_rows, double *out_dev,
                                            size_t batch, void *cuda_stream);

/* ---- Linear convolution of real rows of any length, by overlap-save ----
 * On a real plan of length N: `batch` rows of in_len = L >= 1 reals (row b starting at element b*L) are convolved with
 * the filter c = irfft(H[b mod F], n=N), H as for the circular convolution above (F = spectrum_rows >= 1 rows of N/2+1
 * bins in the plan's rfft layout), of which only the first `taps` = K samples may be non-zero, 1 <= K <= N:
 *   y_full[t] = sum_{m<K} in[b][t-m] c[m],   out[b][i] = y_full[o + i],   output row b starting at element b*out_len,
 *   mode FOURIER_B200_LINEAR_FULL  (0): out_len = L + K - 1, o = 0
 *   mode FOURIER_B200_LINEAR_SAME  (1): out_len = L,         o = (K - 1) / 2
 *   mode FOURIER_B200_LINEAR_VALID (2): out_len = L - K + 1, o = K - 1 (needs L >= K)
 * With H[f] = rfft(h) of a K-tap h zero-padded to N this is scipy.signal.convolve(in[b], h, mode).  Keeping c[K..N) zero
 * is the caller's contract: any other H gives the overlap-save output, which is unspecified.  Correlation is the same
 * call with conj(H).  Rows are cut into segments of S = N - K + 1 outputs (N reads each, the K - 1 before them
 * overlapping the previous segment's), so S / N is the useful fraction of every transform: choose N a few times K.
 * Launches: 1 on the real_fused path; on the others, per scratch chunk of segments, 2 + those of the circular
 * convolution of that many rows; last_launches of the info call reports the total.
 * Refused with cudaErrorInvalidValue and a message: a NULL argument, spectrum_rows == 0, taps == 0, taps > N,
 * in_len == 0, an unknown mode, mode valid with in_len < taps (these also when batch == 0, which otherwise succeeds and
 * launches nothing), `in` and `out` overlapping at all (out of place only), `spectrum` overlapping `out`, and a mix of
 * host and device buffers in the synchronous calls.  Device base pointers must be 16-byte aligned
 * (cudaErrorMisalignedAddress); rows inside them may start at any element.  Host memory is staged through the plan's
 * buffers, whole rows while a row fits 64 MB and otherwise only the input each run of segments reads, and gives the
 * same bits as device memory.  The _async calls take device memory, are enqueued on `cuda_stream` and not
 * synchronised. */
#define FOURIER_B200_LINEAR_FULL 0
#define FOURIER_B200_LINEAR_SAME 1
#define FOURIER_B200_LINEAR_VALID 2
int fourier_b200_linear_convolve_real_float(struct fourier_b200_rfft_float *plan, const float *in, size_t in_len,
                                            const void *spectrum, size_t spectrum_rows, size_t taps, int mode,
                                            float *out, size_t batch);
int fourier_b200_linear_convolve_real_double(struct fourier_b200_rfft_double *plan, const double *in, size_t in_len,
                                             const void *spectrum, size_t spectrum_rows, size_t taps, int mode,
                                             double *out, size_t batch);
int fourier_b200_linear_convolve_real_async_float(struct fourier_b200_rfft_float *plan, const float *in_dev,
                                                  size_t in_len, const void *spectrum_dev, size_t spectrum_rows,
                                                  size_t taps, int mode, float *out_dev, size_t batch,
                                                  void *cuda_stream);
int fourier_b200_linear_convolve_real_async_double(struct fourier_b200_rfft_double *plan, const double *in_dev,
                                                   size_t in_len, const void *spectrum_dev, size_t spectrum_rows,
                                                   size_t taps, int mode, double *out_dev, size_t batch,
                                                   void *cuda_stream);

/* ---- Short-time Fourier transform of real rows ----
 * On a real plan of length N (the frame length): `batch` rows of in_len = L reals (row b starting at element b*L),
 * `window` N reals applied to every frame (zero-pad a shorter window to N), hop H >= 1 (H > N leaves gaps).  With
 * pad = N/2 for FOURIER_B200_STFT_ZEROS / _REFLECT and 0 for _NONE, a row has F = 1 + (L + 2*pad - N) / H frames and
 *   u_f[p] = x_b[f*H - pad + p] * window[p],  p < N,   out[b][f][k] = rfft(u_f)[k],  k <= N/2 (numpy's scale),
 * where samples outside [0, L) are 0 (_ZEROS) or mirrored without repeating the edge, -t -> t and L-1+t -> L-1-t
 * (_REFLECT).  This is torch.stft(x, N, H, window=window, center=boundary != _NONE, pad_mode="constant" / "reflect",
 * return_complex=True) with the last two dimensions swapped: the output is frame-major, row b starting at complex
 * element b*F*(N/2+1), each frame one row in the plan's rfft layout (tf.signal.stft's layout).  _NONE needs L >= N,
 * _REFLECT L > N/2.  Launches: 1 on the real_fused path; otherwise, per scratch chunk of frames, 1 + those of the
 * plan's rfft of that many rows.
 * Inverse: `frames` = F >= 1 spectra per row in that layout -> out_len >= 1 reals per row (row b at element b*out_len).
 * Output i has padded position t = i + pad, pad = N/2 if `center` is non-zero and 0 otherwise, and is
 *   y[i] = sum_f window[t - f*H] * v_f[t - f*H]  /  sum_f window[t - f*H]^2,   v_f = irfft(out[b][f], n=N),
 * over the frames f < F with 0 <= t - f*H < N in ascending f (deterministic).  Where the denominator is below 1e-11,
 * including positions no frame covers, the output is 0 (torch.istft raises there instead).  With out_len =
 * H*(F-1) + N - 2*pad this is torch.istft(..., center=center, length=out_len).  Launches: per run of frames that fits
 * the plan's scratch, those of the plan's irfft of the run plus 1.
 * Refused with cudaErrorInvalidValue and a message: a NULL argument, hop == 0, an unknown boundary, in_len == 0,
 * frames == 0, out_len == 0 (these also when batch == 0, which otherwise succeeds and launches nothing), in_len < N with
 * _NONE, in_len <= N/2 with _REFLECT, the input or window overlapping the output (out of place only), and a mix of
 * host and device buffers in the synchronous calls.  Device base pointers of input and output must be 16-byte
 * aligned (cudaErrorMisalignedAddress).  Host memory is staged through the plan's buffers (the window once, whole
 * rows in chunks) and gives the same bits as device memory.  The _async calls take device memory, are enqueued on
 * `cuda_stream` and not synchronised. */
#define FOURIER_B200_STFT_NONE 0
#define FOURIER_B200_STFT_ZEROS 1
#define FOURIER_B200_STFT_REFLECT 2
int fourier_b200_stft_float(struct fourier_b200_rfft_float *plan, const float *in, size_t in_len, const float *window,
                            size_t hop, int boundary, void *out, size_t batch);
int fourier_b200_stft_double(struct fourier_b200_rfft_double *plan, const double *in, size_t in_len,
                             const double *window, size_t hop, int boundary, void *out, size_t batch);
int fourier_b200_stft_async_float(struct fourier_b200_rfft_float *plan, const float *in_dev, size_t in_len,
                                  const float *window_dev, size_t hop, int boundary, void *out_dev, size_t batch,
                                  void *cuda_stream);
int fourier_b200_stft_async_double(struct fourier_b200_rfft_double *plan, const double *in_dev, size_t in_len,
                                   const double *window_dev, size_t hop, int boundary, void *out_dev, size_t batch,
                                   void *cuda_stream);
int fourier_b200_istft_float(struct fourier_b200_rfft_float *plan, const void *in, size_t frames, const float *window,
                             size_t hop, int center, float *out, size_t out_len, size_t batch);
int fourier_b200_istft_double(struct fourier_b200_rfft_double *plan, const void *in, size_t frames,
                              const double *window, size_t hop, int center, double *out, size_t out_len, size_t batch);
int fourier_b200_istft_async_float(struct fourier_b200_rfft_float *plan, const void *in_dev, size_t frames,
                                   const float *window_dev, size_t hop, int center, float *out_dev, size_t out_len,
                                   size_t batch, void *cuda_stream);
int fourier_b200_istft_async_double(struct fourier_b200_rfft_double *plan, const void *in_dev, size_t frames,
                                    const double *window_dev, size_t hop, int center, double *out_dev, size_t out_len,
                                    size_t batch, void *cuda_stream);

/* ---- Mel spectrogram of real rows ----
 * On a real plan of length N, with the stft's framing above (in_len, window, hop, boundary and the frame count F
 * unchanged): out[b][f][m] = sum_{k <= N/2} filters[m][k] * |X_{b,f}[k]|^power, where X_{b,f} is the stft of frame f
 * of row b, power is 1 or 2 and `filters` is a dense row-major (n_mels, N/2+1) matrix of any real weights, n_mels >= 1
 * (librosa's and Whisper's layout; torchaudio's melscale_fbanks returns the transpose).  The output is frame-major,
 * row b starting at element b*F*n_mels, frame f at b*F*n_mels + f*n_mels: with power 2 and torchaudio's own window
 * and bank this is torchaudio.transforms.MelSpectrogram(...)(x).transpose(-1, -2).  No log is taken.
 * Row m of the matrix is read only from its first to its last non-zero weight (its band, recomputed on every call), so
 * a triangular bank touches about 2(N/2+1) weights per frame; zeros inside a band are multiplied like any weight, and
 * an all-zero row gives exactly 0.  Launches: 2 on the real_fused path; on the others 1, plus per scratch chunk of
 * frames 2 + those of the plan's rfft of that many rows.
 * Refused with cudaErrorInvalidValue and a message: a NULL argument, hop == 0, an unknown boundary, in_len == 0, power
 * other than 1 and 2, n_mels == 0 (these also when batch == 0, which otherwise succeeds and launches nothing), in_len < N
 * with _NONE, in_len <= N/2 with _REFLECT, the input, window or filters overlapping the output (out of place only), and
 * a mix of host and device buffers in the synchronous calls.  Device base pointers of input and output must be
 * 16-byte aligned (cudaErrorMisalignedAddress).  Host memory is staged through the plan's buffers (the window and
 * filters once, whole rows in chunks) and gives the same bits as device memory.  The _async calls take device memory,
 * are enqueued on `cuda_stream` and not synchronised. */
int fourier_b200_mel_spectrogram_float(struct fourier_b200_rfft_float *plan, const float *in, size_t in_len,
                                       const float *window, size_t hop, int boundary, int power,
                                       const float *filters, size_t n_mels, float *out, size_t batch);
int fourier_b200_mel_spectrogram_double(struct fourier_b200_rfft_double *plan, const double *in, size_t in_len,
                                        const double *window, size_t hop, int boundary, int power,
                                        const double *filters, size_t n_mels, double *out, size_t batch);
int fourier_b200_mel_spectrogram_async_float(struct fourier_b200_rfft_float *plan, const float *in_dev, size_t in_len,
                                             const float *window_dev, size_t hop, int boundary, int power,
                                             const float *filters_dev, size_t n_mels, float *out_dev, size_t batch,
                                             void *cuda_stream);
int fourier_b200_mel_spectrogram_async_double(struct fourier_b200_rfft_double *plan, const double *in_dev,
                                              size_t in_len, const double *window_dev, size_t hop, int boundary,
                                              int power, const double *filters_dev, size_t n_mels, double *out_dev,
                                              size_t batch, void *cuda_stream);

/* ---- MFCC and log-mel spectrogram of real rows ----
 * On a real plan of length N, with the mel spectrogram's framing, window, power and filters above (mel[b][f][m], F
 * frames per row), in the plan's precision T (each double scalar rounded to T once):
 *   lm[b][f][m]  = log_scale * ln(max(mel[b][f][m] + log_offset, log_floor)),
 *   lc           = max(lm, theta_g) with theta_g = (max of lm over the rows, frames and mels of clamp group g) - top_db,
 *                  the rows [g*top_db_rows, (g+1)*top_db_rows) forming group g; lc = lm when top_db is +inf,
 *   out[b][f][j] = bias + sum_{m = 0 .. n_mels-1, ascending} lc[b][f][m] * dct[m*n_out + j],   j < n_out,
 * where dct is a dense row-major (n_mels, n_out) matrix of any real values (torchaudio's create_dct layout; fold a
 * lifter into its columns), or NULL for the identity with n_out == n_mels, which gives the log-mel spectrogram lc + bias.
 * The output is frame-major, row b from element b*F*n_out on.  Recipes: torchaudio's MFCC(log_mels=False) with
 * log_scale 10/ln 10, log_floor 1e-10, log_offset 0, top_db 80, top_db_rows = the channel count (1 for 1-D input);
 * MFCC(log_mels=True) with log_scale 1, log_floor the smallest normal of T, log_offset 1e-6, top_db +inf; librosa's
 * mfcc with top_db_rows = batch; Whisper's log-mel with log_scale 1/(4 ln 10), log_floor 1e-10, top_db 2, dct NULL,
 * bias 1 (Whisper drops the last frame before its max; this takes the max over all F frames).
 * The group maximum is exact and order-independent, and each output a fixed ascending sum, so a row's bits depend only on
 * its clamp group's rows, the arguments and the plan: not on the rest of the batch, host or device memory or the stream.
 * With the clamp (top_db finite) the frames are swept twice: once for the group maxima (kept in a plan-owned buffer),
 * once for the outputs.  Launches: on the real_fused path with n_mels <= N/2 - 1, 2 (3 with the clamp); otherwise 1,
 * plus per sweep and scratch chunk of frames 3 + those of the plan's rfft of that many rows.
 * Refused with cudaErrorInvalidValue and a message (these also when batch == 0, which otherwise succeeds and launches
 * nothing): a NULL in, window, filters or out, hop == 0, an unknown boundary, in_len == 0, power other than 1 and 2,
 * n_mels == 0, n_out == 0, dct NULL with n_out != n_mels, log_offset or bias not finite, log_floor or log_scale not
 * finite and > 0, top_db NaN or < 0, top_db_rows == 0, and with top_db finite a batch that is not a multiple of
 * top_db_rows.  Also refused: in_len < N with _NONE, in_len <= N/2 with _REFLECT, the output overlapping the input,
 * window, filters or dct (out of place only), and a mix of host and device buffers in the synchronous calls.  Device base
 * pointers of input and output must be 16-byte aligned (cudaErrorMisalignedAddress).  Host memory is staged through the
 * plan's buffers (the window, filters and dct once, whole rows in chunks) and gives the same bits as device memory.
 * The _async calls take device memory, are enqueued on `cuda_stream` and never synchronise the host. */
int fourier_b200_mfcc_float(struct fourier_b200_rfft_float *plan, const float *in, size_t in_len, const float *window,
                            size_t hop, int boundary, int power, const float *filters, size_t n_mels, double log_offset,
                            double log_floor, double log_scale, double top_db, size_t top_db_rows, const float *dct,
                            size_t n_out, double bias, float *out, size_t batch);
int fourier_b200_mfcc_double(struct fourier_b200_rfft_double *plan, const double *in, size_t in_len,
                             const double *window, size_t hop, int boundary, int power, const double *filters,
                             size_t n_mels, double log_offset, double log_floor, double log_scale, double top_db,
                             size_t top_db_rows, const double *dct, size_t n_out, double bias, double *out,
                             size_t batch);
int fourier_b200_mfcc_async_float(struct fourier_b200_rfft_float *plan, const float *in_dev, size_t in_len,
                                  const float *window_dev, size_t hop, int boundary, int power,
                                  const float *filters_dev, size_t n_mels, double log_offset, double log_floor,
                                  double log_scale, double top_db, size_t top_db_rows, const float *dct_dev,
                                  size_t n_out, double bias, float *out_dev, size_t batch, void *cuda_stream);
int fourier_b200_mfcc_async_double(struct fourier_b200_rfft_double *plan, const double *in_dev, size_t in_len,
                                   const double *window_dev, size_t hop, int boundary, int power,
                                   const double *filters_dev, size_t n_mels, double log_offset, double log_floor,
                                   double log_scale, double top_db, size_t top_db_rows, const double *dct_dev,
                                   size_t n_out, double bias, double *out_dev, size_t batch, void *cuda_stream);

/* ---- Welch power spectral density of real rows ----
 * On a real plan of length N, for `batch` rows of in_len >= N reals (row b at element b*in_len), a window of N reals
 * and hop >= 1: the F = 1 + (in_len - N) / hop frames x_bf[p] = in[b*in_len + f*hop + p], p < N (no padding, F =
 * the stft's frame count with FOURIER_B200_STFT_NONE), and
 *   out[b][k] = c_k * s / F * sum_{f < F} |X_bf[k]|^2,   X_bf = rfft(w * (x_bf - mu_bf)),   k <= N/2,
 * where mu_bf is the frame's mean (FOURIER_B200_DETREND_CONSTANT, taken off before the window) or 0 (_NONE),
 * s = 1 / (fs * sum w^2) (FOURIER_B200_WELCH_DENSITY) or 1 / (sum w)^2 (_SPECTRUM), and c_k = 2 for 0 < k < N/2 (N even)
 * or 0 < k <= (N-1)/2 (N odd), else 1.  With nperseg = N and noverlap = N - hop this is
 * scipy.signal.welch(x, fs, window=w, nperseg=N, noverlap=N-hop, detrend="constant" | False,
 * scaling="density" | "spectrum")[1].  out holds N/2+1 reals per row.  A window with sum w^2 = 0 gives the IEEE
 * result (inf / NaN), as scipy does.
 * Frames are summed in items of consecutive frames whose size depends only on F and the plan, so a row's bits depend
 * only on the row, the window, hop, detrend, scaling, fs and the plan: not on the batch, the other rows, host or device
 * memory or the stream.  The window sums are formed on the device on every call.  Launches: at most 3 on the real_fused
 * path while the rows' partials fit one scratch chunk (512 MB); on the others 2, plus per scratch chunk of frames 2 and
 * those of the plan's rfft of that many rows.
 * Refused with cudaErrorInvalidValue and a message: a NULL argument, hop == 0, in_len == 0, detrend other than 0 and 1,
 * scaling other than 0 and 1, fs not finite and > 0 (these also when batch == 0, which otherwise succeeds and launches
 * nothing), in_len < N, the input or window overlapping the output (out of place only), and a mix of host and device
 * buffers in the synchronous calls.  Device base pointers of input and output must be 16-byte aligned
 * (cudaErrorMisalignedAddress).  Host memory is staged through the plan's buffers (the window once, whole rows in
 * chunks) and gives the same bits as device memory.  The _async calls take device memory, are enqueued on
 * `cuda_stream` and never synchronise the host. */
#define FOURIER_B200_DETREND_NONE 0
#define FOURIER_B200_DETREND_CONSTANT 1
#define FOURIER_B200_WELCH_DENSITY 0
#define FOURIER_B200_WELCH_SPECTRUM 1
int fourier_b200_welch_float(struct fourier_b200_rfft_float *plan, const float *in, size_t in_len,
                             const float *window, size_t hop, int detrend, int scaling, double fs, float *out,
                             size_t batch);
int fourier_b200_welch_double(struct fourier_b200_rfft_double *plan, const double *in, size_t in_len,
                              const double *window, size_t hop, int detrend, int scaling, double fs, double *out,
                              size_t batch);
int fourier_b200_welch_async_float(struct fourier_b200_rfft_float *plan, const float *in_dev, size_t in_len,
                                   const float *window_dev, size_t hop, int detrend, int scaling, double fs,
                                   float *out_dev, size_t batch, void *cuda_stream);
int fourier_b200_welch_async_double(struct fourier_b200_rfft_double *plan, const double *in_dev, size_t in_len,
                                    const double *window_dev, size_t hop, int detrend, int scaling, double fs,
                                    double *out_dev, size_t batch, void *cuda_stream);

/* ---- discrete cosine transforms of real rows (types II and III) ----
 * On a real plan of length N >= 1, for `batch` rows of N reals (row b at element b*N), with W = exp(-i pi / (2N)) and
 * Makhoul's reordering v[j] = x[2j] (j < ceil(N/2)), v[N-1-j] = x[2j+1] (j < floor(N/2)):
 *   type 2:  V = FFT_N(v),  y[k] = 2 h Re(W^k V[k]) (0 <= k <= N/2),  y[N-k] = -2 h Im(W^k V[k]) (0 < k <= N/2),
 *            i.e. y[k] = 2 h sum_n x[n] cos(pi k (2n+1) / (2N));
 *   type 3:  V'[k] = h conj(W^k) (x[k] - i x[N-k]) (0 < k <= N/2),  V'[0] = h x[0],  u = N irfft(V', n = N),
 *            y[2j] = u[j], y[2j+1] = u[N-1-j], i.e. y[k] = h x[0] + 2 h sum_{n>0} x[n] cos(pi (2k+1) n / (2N)).
 * The norm sets h: 1 (FOURIER_B200_DCT_NORM_BACKWARD), 1 / (2N) (_FORWARD) or 1 / sqrt(2N) (_ORTHO, which also scales
 * y[0] of type 2 by 1 / sqrt(2) and x[0] of type 3 by sqrt(2)).  This is scipy.fft.dct(x, type, norm) with
 * orthogonalize=True, and FFTW's REDFT10 (type 2) and REDFT01 (type 3) with the backward norm.  scipy.fft.idct(x, type,
 * norm) is the call with type 5 - type and norm backward and forward swapped.  torch has no DCT.
 * Launches: 1 on the real_fused path (N = 128 .. 2048 in f32, 128 .. 512 in f64); on the others, per scratch chunk of
 * rows (512 MB), 2 plus those of the inner plan: a reordering or twiddle kernel, the inner complex plan of length N/2
 * (even N) or N (odd N) in place in the scratch, and a kernel that writes the output rows.
 * Refused with cudaErrorInvalidValue and a message: a NULL argument, a type other than 2 and 3, a norm other than the
 * three macros (these also when batch == 0, which otherwise succeeds and launches nothing), input and output
 * overlapping without being the same buffer, and a mix of host and device buffers in the synchronous calls.  in == out
 * transforms in place.  Device base pointers must be 16-byte aligned (cudaErrorMisalignedAddress).  Host memory is
 * staged through the plan's buffers in whole rows and gives the same bits as device memory.  The _async calls take
 * device memory, are enqueued on `cuda_stream` and never synchronise the host. */
#define FOURIER_B200_DCT_NORM_BACKWARD 0
#define FOURIER_B200_DCT_NORM_ORTHO 1
#define FOURIER_B200_DCT_NORM_FORWARD 2
int fourier_b200_dct_float(struct fourier_b200_rfft_float *plan, const float *in, float *out, size_t batch, int type,
                           int norm);
int fourier_b200_dct_double(struct fourier_b200_rfft_double *plan, const double *in, double *out, size_t batch,
                            int type, int norm);
int fourier_b200_dct_async_float(struct fourier_b200_rfft_float *plan, const float *in_dev, float *out_dev,
                                 size_t batch, int type, int norm, void *cuda_stream);
int fourier_b200_dct_async_double(struct fourier_b200_rfft_double *plan, const double *in_dev, double *out_dev,
                                  size_t batch, int type, int norm, void *cuda_stream);

/* ---- cross-spectral density and coherence of real rows ----
 * On a real plan of length N, for `batch` rows x_b of in_len >= N reals (row b at element b*in_len) and y_rows >= 1
 * rows of in_len reals y: row b of x pairs with y row b mod y_rows (1: one y for every row; batch: one y per row).  Both
 * are framed as by fourier_b200_welch_*: X_bf = rfft(w * (x_bf - mu_bf)), Y_bf = rfft(w * (y_bf - nu_bf)), the frame
 * means taken off with FOURIER_B200_DETREND_CONSTANT, F = 1 + (in_len - N) / hop frames.  Then, for k <= N/2,
 *   csd:        out[b][k] = c_k * s / F * sum_{f < F} conj(X_bf[k]) * Y_bf[k]             (complex),
 *   coherence:  out[b][k] = |sum_f conj(X_bf[k]) Y_bf[k]|^2 / (sum_f |X_bf[k]|^2 * sum_f |Y_bf[k]|^2)   (real),
 * with c_k and s as in fourier_b200_welch_*.  That is scipy.signal.csd(x, y, fs, window=w, nperseg=N,
 * noverlap=N-hop, detrend=..., scaling=...)[1] and scipy.signal.coherence(x, y, fs, window=w, nperseg=N,
 * noverlap=N-hop, detrend=...)[1].  The csd writes N/2+1 complex values per row in the rfft layout (row b from complex
 * element b*(N/2+1) on), with Im exactly +0 at bins 0 and N/2; the coherence N/2+1 reals per row, NaN where the
 * denominator is 0 (0/0, as scipy gives, e.g. for a row of zeros).
 * A row's bits depend only on its x row, its y row, the window, hop, detrend, scaling, fs and the plan: not on the batch,
 * the other rows, y_rows repetition, host or device memory or the stream.  Launches: the csd makes at most 3 on the
 * real_fused path while the rows' partials fit one scratch chunk, the coherence at most 2 (no window sums).
 * Refused with cudaErrorInvalidValue and a message: a NULL argument, y_rows == 0, hop == 0, in_len == 0, detrend other
 * than 0 and 1, for the csd scaling other than 0 and 1 and fs not finite and > 0 (these also when batch == 0, which
 * otherwise succeeds and launches nothing), in_len < N, the output overlapping the x rows, the y rows or the window
 * (out of place only; x and y may overlap, y == x is allowed), and a mix of host and device buffers in the synchronous
 * calls.  Device base pointers of x, y and the output must be 16-byte aligned (cudaErrorMisalignedAddress).  Host memory
 * is staged through the plan's buffers (the window once, whole x rows in chunks with the y rows they pair with) and gives
 * the same bits as device memory.  The _async calls take device memory, are enqueued on `cuda_stream` and never
 * synchronise the host. */
int fourier_b200_csd_float(struct fourier_b200_rfft_float *plan, const float *x, const float *y, size_t y_rows,
                           size_t in_len, const float *window, size_t hop, int detrend, int scaling, double fs,
                           void *out, size_t batch);
int fourier_b200_csd_double(struct fourier_b200_rfft_double *plan, const double *x, const double *y, size_t y_rows,
                            size_t in_len, const double *window, size_t hop, int detrend, int scaling, double fs,
                            void *out, size_t batch);
int fourier_b200_csd_async_float(struct fourier_b200_rfft_float *plan, const float *x_dev, const float *y_dev,
                                 size_t y_rows, size_t in_len, const float *window_dev, size_t hop, int detrend,
                                 int scaling, double fs, void *out_dev, size_t batch, void *cuda_stream);
int fourier_b200_csd_async_double(struct fourier_b200_rfft_double *plan, const double *x_dev, const double *y_dev,
                                  size_t y_rows, size_t in_len, const double *window_dev, size_t hop, int detrend,
                                  int scaling, double fs, void *out_dev, size_t batch, void *cuda_stream);
int fourier_b200_coherence_float(struct fourier_b200_rfft_float *plan, const float *x, const float *y, size_t y_rows,
                                 size_t in_len, const float *window, size_t hop, int detrend, float *out,
                                 size_t batch);
int fourier_b200_coherence_double(struct fourier_b200_rfft_double *plan, const double *x, const double *y,
                                  size_t y_rows, size_t in_len, const double *window, size_t hop, int detrend,
                                  double *out, size_t batch);
int fourier_b200_coherence_async_float(struct fourier_b200_rfft_float *plan, const float *x_dev, const float *y_dev,
                                       size_t y_rows, size_t in_len, const float *window_dev, size_t hop, int detrend,
                                       float *out_dev, size_t batch, void *cuda_stream);
int fourier_b200_coherence_async_double(struct fourier_b200_rfft_double *plan, const double *x_dev,
                                        const double *y_dev, size_t y_rows, size_t in_len, const double *window_dev,
                                        size_t hop, int detrend, double *out_dev, size_t batch, void *cuda_stream);

/* ---- analytic signal and envelope of real rows (Hilbert transform) ----
 * On a real plan of length N >= 1, for `batch` rows of N reals x (row b at element b*N):
 *   y = irfft(G * rfft(x), n = N),  G[k] = -i (0 < k < N/2),  G[0] = 0,  G[N/2] = 0 (N even),
 *   z = x + i y,
 * which is scipy.signal.hilbert(x, axis=-1).  FOURIER_B200_HILBERT_ANALYTIC writes z, N complex values (x[n], y[n])
 * interleaved per row (row b from complex element b*N on); FOURIER_B200_HILBERT_ENVELOPE writes |z[n]| =
 * sqrt(x[n]^2 + y[n]^2), N reals per row (row b from real element b*N on).  The real part of the analytic output is a
 * copy of x, bit for bit, on every path; scipy's equals x only up to rounding (it inverts the whole spectrum).  torch
 * has no Hilbert transform.
 * Launches: 1 on the real_fused path (N = 128 .. 2048 in f32, 128 .. 512 in f64); on real_half (other even N), per
 * scratch chunk of rows (512 MB), 2 plus twice those of the inner complex plan of length N/2 (its forward and its
 * unscaled inverse); on real_full (odd N), per scratch chunk, 3 plus twice those of the inner plan of length N.
 * Refused with cudaErrorInvalidValue and a message naming the argument: a NULL argument and an output other than the
 * two macros (these also when batch == 0, which otherwise succeeds and launches nothing); input and output overlapping,
 * except in == out for the envelope, which runs in place (the analytic signal is out of place only); and a mix of host
 * and device buffers in the synchronous calls.  Device base pointers must be 16-byte aligned
 * (cudaErrorMisalignedAddress).  Host memory is staged through the plan's buffers in whole rows and gives the same bits
 * as device memory.  The _async calls take device memory, are enqueued on `cuda_stream` and never synchronise the
 * host. */
#define FOURIER_B200_HILBERT_ANALYTIC 0
#define FOURIER_B200_HILBERT_ENVELOPE 1
int fourier_b200_hilbert_float(struct fourier_b200_rfft_float *plan, const float *in, void *out, size_t batch,
                               int output);
int fourier_b200_hilbert_double(struct fourier_b200_rfft_double *plan, const double *in, void *out, size_t batch,
                                int output);
int fourier_b200_hilbert_async_float(struct fourier_b200_rfft_float *plan, const float *in_dev, void *out_dev,
                                     size_t batch, int output, void *cuda_stream);
int fourier_b200_hilbert_async_double(struct fourier_b200_rfft_double *plan, const double *in_dev, void *out_dev,
                                      size_t batch, int output, void *cuda_stream);

/* ---- type-IV DCT, MDCT and IMDCT of real rows ----
 * On a real plan of even length N (odd N is refused), h the norm's scale as for the DCT (FOURIER_B200_DCT_NORM_*:
 * 1, 1 / sqrt(2N) or 1 / (2N); type IV has no bin-0 scale), and h' the scale of the norm with backward and forward
 * swapped:
 *   dct4:  y[k] = 2 h sum_{n<N} x[n] cos(pi (2n+1)(2k+1) / (4N)) for `batch` rows of N reals (row b at element b*N),
 *          scipy.fft.dct(x, type=4, norm); its inverse is dct4 with the swapped norm (scipy.fft.idct(type=4)).  in == out
 *          transforms in place.
 *   mdct:  N coefficients per frame of 2N samples every N, times `window` (2N reals):
 *          X_f[k] = 2 h sum_{s<2N} w[s] x~[fN - pad + s] cos(pi/N (s + 1/2 + N/2)(k + 1/2)), k < N, x~ = 0 outside the
 *          row.  center != 0: pad = N and F = ceil(in_len / N) + 1 frames, every sample in two frames; center == 0:
 *          pad = 0 and F = 1 + (in_len - 2N) / N frames (in_len >= 2N), tf.signal.mdct(x, 2N, window_fn,
 *          pad_end=False).  Rows of in_len reals (row b at element b*in_len) -> F frames of N reals per row
 *          (row b at element b*F*N, frame-major).
 *   imdct: y[i] = sum_f w[t - fN] v_f[t - fN], t = i + pad, over the frames f < `frames` with 0 <= t - fN < 2N in
 *          ascending f, v_f[s] = 2 h' sum_k X_f[k] cos(pi/N (s + 1/2 + N/2)(k + 1/2)); no envelope division.  Rows of
 *          frames*N reals -> rows of out_len >= 1 reals (0 where no frame covers t).  With center, out_len = in_len and
 *          a Princen-Bradley window (w[s]^2 + w[s+N]^2 = 1, w symmetric: sine, Vorbis, KBD), imdct(mdct(x)) = x in
 *          every norm.
 * Launches: dct4 and mdct 1 on the real_fused path (N = 128 .. 2048 in f32, 128 .. 512 in f64); on real_half (other
 * even N), per scratch chunk of rows or frames (512 MB), 2 plus those of the inner complex plan of length N/2.  imdct,
 * per run of frames through the plan's scratch: the dct4 of the run's frames, then 1 overlap-add kernel.
 * Refused with cudaErrorInvalidValue and a message naming the argument, also when batch == 0 (which otherwise succeeds
 * and launches nothing): a NULL argument, a norm other than the three macros, in_len == 0, frames == 0 and
 * out_len == 0.  Also refused: an odd plan length, in_len < 2N without center, an output that overlaps the input or the
 * window (dct4: in == out is allowed, a partial overlap is not), and a mix of host and device buffers in the
 * synchronous calls.  Device base pointers must be 16-byte aligned (cudaErrorMisalignedAddress).  Host memory is
 * staged through the plan's buffers (the window once, whole rows) and gives the same bits as device memory.  The
 * _async calls take device memory, are enqueued on `cuda_stream` and never synchronise the host. */
int fourier_b200_dct4_float(struct fourier_b200_rfft_float *plan, const float *in, float *out, size_t batch, int norm);
int fourier_b200_dct4_double(struct fourier_b200_rfft_double *plan, const double *in, double *out, size_t batch,
                             int norm);
int fourier_b200_dct4_async_float(struct fourier_b200_rfft_float *plan, const float *in_dev, float *out_dev,
                                  size_t batch, int norm, void *cuda_stream);
int fourier_b200_dct4_async_double(struct fourier_b200_rfft_double *plan, const double *in_dev, double *out_dev,
                                   size_t batch, int norm, void *cuda_stream);
int fourier_b200_mdct_float(struct fourier_b200_rfft_float *plan, const float *in, size_t in_len, const float *window,
                            int center, int norm, float *out, size_t batch);
int fourier_b200_mdct_double(struct fourier_b200_rfft_double *plan, const double *in, size_t in_len,
                             const double *window, int center, int norm, double *out, size_t batch);
int fourier_b200_mdct_async_float(struct fourier_b200_rfft_float *plan, const float *in_dev, size_t in_len,
                                  const float *window_dev, int center, int norm, float *out_dev, size_t batch,
                                  void *cuda_stream);
int fourier_b200_mdct_async_double(struct fourier_b200_rfft_double *plan, const double *in_dev, size_t in_len,
                                   const double *window_dev, int center, int norm, double *out_dev, size_t batch,
                                   void *cuda_stream);
int fourier_b200_imdct_float(struct fourier_b200_rfft_float *plan, const float *in, size_t frames, const float *window,
                             int center, int norm, float *out, size_t out_len, size_t batch);
int fourier_b200_imdct_double(struct fourier_b200_rfft_double *plan, const double *in, size_t frames,
                              const double *window, int center, int norm, double *out, size_t out_len, size_t batch);
int fourier_b200_imdct_async_float(struct fourier_b200_rfft_float *plan, const float *in_dev, size_t frames,
                                   const float *window_dev, int center, int norm, float *out_dev, size_t out_len,
                                   size_t batch, void *cuda_stream);
int fourier_b200_imdct_async_double(struct fourier_b200_rfft_double *plan, const double *in_dev, size_t frames,
                                    const double *window_dev, int center, int norm, double *out_dev, size_t out_len,
                                    size_t batch, void *cuda_stream);

const char *fourier_b200_last_error(void);
const char *fourier_b200_version(void);

#undef FB200_PLAN_F
#undef FB200_PLAN_D
#undef FB200_F
#undef FB200_D
#ifdef __cplusplus
}
#endif
#endif /* FOURIER_B200_H_ */
