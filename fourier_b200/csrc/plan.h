// plan.h -- host-side plan objects behind the C ABI (include/fourier.h, include/fourier_b200.h).
//
// A Plan<T> is what the reference boxes up as `Box<dyn Fft<Real = T> + Send>`
// (fourier/src/lib.rs:31-60): it owns the twiddle tables and scratch for one transform size and
// exposes the single required operation, transform_in_place / transform with a Transform code
// (fourier-algorithms/src/fft.rs:40-82).  Here the tables and scratch live in HBM, the operation
// is batched, and it is enqueued on a CUDA stream.
#pragma once

#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstddef>
#include <exception>
#include <memory>
#include <new>
#include <string>
#include <vector>

#include "cplx.cuh"
#include "real_kernels.cuh"   // real::SegMap

namespace fb200 {

// Execution strategy chosen at plan time.
enum class Path : int {
  kTrivial = 0,         // N == 1
  kOnChip = 1,          // one shared-memory Stockham FFT per CTA-slice (pow2 N <= on-chip limit)
  kTwoPass = 2,         // four-step, two fused kernels, L2-resident intermediate (large pow2 N)
  kGlobalStages = 3,    // one kernel per Stockham stage over HBM ({2,3}-smooth N, any size)
  kBluestein = 4,       // chirp-z around a pow2 inner plan, separate kernels
  kBluesteinFused = 5,  // chirp-z with the inner FFTs on chip, one kernel
  kCta = 6,             // whole transforms in shared memory, one CTA per group of transforms, all Stockham stages
                        // in one kernel ({2,3}-smooth N, pow2 N between the on-chip and two-pass kernels)
  kThreePass = 7,       // pow2 N above the two-pass kernels: outer column pass + two-pass rows storing transposed
  // real-input plans (RealPlan, real.cu)
  kRealFused = 8,       // N = 2M, M an on-chip size class: one fused on-chip kernel
  kRealHalf = 9,        // other even N: complex plan of length N/2 + one untangle / tangle kernel
  kRealFull = 10,       // odd N: complex plan of length N between two O(N) kernels
};

const char* path_name(Path p);

constexpr size_t kScratchTargetBytes = (size_t)512 << 20;  // per scratch buffer on the general and real paths
constexpr size_t kHostChunkBytes = (size_t)64 << 20;       // host-pointer pipeline granule

constexpr int kMaxPeers = 16;   // ranks of one box (peer-memory exchange, exchange.cu / dist_fft.cu)

// Selection rule of create_fft_f32/f64 (fourier/src/lib.rs:38-42 with autosort/mod.rs:104-117):
// Autosort iff N = 2^a * 3^b (N >= 1), else Bluestein with inner size next_pow2(2N-1).
bool is_23_smooth(size_t n);
size_t bluestein_inner_size(size_t n);  // bluesteins.rs:110

// thread-local error text for the C ABI
void set_last_error(const std::string& s);
const char* last_error();

// Returns the error of a failing CUDA call from the enclosing function, with last_error set to the call and its text.
#define FB_CHECK(expr)                                                                       \
  do {                                                                                       \
    cudaError_t _e = (expr);                                                                 \
    if (_e != cudaSuccess) {                                                                 \
      set_last_error(std::string(#expr) + ": " + cudaGetErrorString(_e));                    \
      return _e;                                                                             \
    }                                                                                        \
  } while (0)

// Scale factor of a Transform code for length n (autosort/mod.rs:381-385, bluesteins.rs:240-258).
template <typename T> T scale_for(int code, size_t n) {
  switch (code) {
    case kIfft: return (T)1 / (T)n;
    case kSqrtScaledFft:
    case kSqrtScaledIfft: return (T)1 / std::sqrt((T)n);
    default: return (T)1;
  }
}

// Multiprocessor count of `device`; 132 (H100 SXM) when the query fails.
inline int sm_count(int device) {
  int sms = 132;
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess) sms = 132;
  return sms;
}

// Grid of the grid-stride kernels (stockham_generic.cu, real.cu): kThreads per CTA, one thread per element up to
// 32 CTAs per SM of a 132-SM H100, grid-stride beyond.
constexpr int kThreads = 256;
inline unsigned grid_for(size_t total) {
  const size_t blocks = (total + kThreads - 1) / kThreads;
  return (unsigned)std::max<size_t>(1, std::min<size_t>(blocks, 132u * 32u));
}

// Makes `dev` the current device for the lifetime of the guard.
struct DeviceGuard {
  int prev = -1;
  bool ok = true;
  explicit DeviceGuard(int dev) {
    if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
    if (prev != dev) ok = cudaSetDevice(dev) == cudaSuccess;
  }
  ~DeviceGuard() {
    int cur = -1;
    if (prev >= 0 && cudaGetDevice(&cur) == cudaSuccess && cur != prev) cudaSetDevice(prev);
  }
};

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) is a per-device setting: done once per kernel AND device (a process
// may hold plans on several GPUs).  `done` is the kernel's own bit mask of prepared devices.  carveout >= 0 also sets
// the kernel's preferred shared-memory carveout (percent, or a cudaSharedmemCarveout value) on the same terms.
template <class Kernel>
inline cudaError_t ensure_dynamic_smem(Kernel kernel, size_t bytes, std::atomic<unsigned long long>& done,
                                       int carveout = -1) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  const unsigned long long bit = 1ull << (dev & 63);
  if (done.load(std::memory_order_acquire) & bit) return cudaSuccess;
  e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  if (e == cudaSuccess && carveout >= 0)
    e = cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, carveout);
  if (e == cudaSuccess) done.fetch_or(bit, std::memory_order_release);
  return e;
}

// Grow-only device allocation.
class DeviceBuffer {
 public:
  DeviceBuffer() = default;
  ~DeviceBuffer();
  DeviceBuffer(const DeviceBuffer&) = delete;
  DeviceBuffer& operator=(const DeviceBuffer&) = delete;
  cudaError_t reserve(size_t bytes);
  void* data() const { return ptr_; }
  size_t bytes() const { return bytes_; }
  void release();

 private:
  void* ptr_ = nullptr;
  size_t bytes_ = 0;
};

// Copies a host table into `buf`, which keeps at least one element so that an empty table still has an address.
template <typename U>
cudaError_t upload(DeviceBuffer& buf, const std::vector<U>& host) {
  cudaError_t e = buf.reserve(std::max<size_t>(host.size(), 1) * sizeof(U));
  if (e != cudaSuccess || host.empty()) return e;
  return cudaMemcpy(buf.data(), host.data(), host.size() * sizeof(U), cudaMemcpyHostToDevice);
}

// create() of Plan and RealPlan: nullptr (and last_error set) when the plan cannot be built; size 0 is refused
// (the reference never returns for 0: autosort/mod.rs:112).
template <class P>
P* create_plan(size_t n, int device, bool allow_fast_paths) {
  if (n == 0) {
    set_last_error("size 0 is not a valid transform length");
    return nullptr;
  }
  P* p = new (std::nothrow) P();
  if (!p) return nullptr;
  cudaError_t e = cudaErrorUnknown;
  try {
    e = p->init(n, device, allow_fast_paths);
  } catch (const std::exception& ex) {   // e.g. bad_alloc while building an N-entry host table
    set_last_error(std::string("plan construction threw: ") + ex.what());
  }
  if (e != cudaSuccess) {
    delete p;
    return nullptr;
  }
  return p;
}

struct PlanInfo {
  size_t size = 0;
  int path = 0;
  size_t inner_size = 0;     // Bluestein inner FFT length, else 0
  int inner_path = 0;
  size_t n1 = 0, n2 = 0;     // two-pass split
  int precision_bytes = 0;   // 4 or 8
  int device = 0;
  size_t table_bytes = 0;    // twiddle / chirp tables resident in HBM
};

template <typename T>
class Plan {
 public:
  using C = cpx<T>;

  // Returns nullptr (and sets last_error) when the plan cannot be built; size 0 is refused.
  static Plan* create(size_t n, int device, bool allow_fast_paths = true) {
    return create_plan<Plan>(n, device, allow_fast_paths);
  }
  ~Plan();

  size_t size() const { return n_; }
  int device() const { return device_; }
  Path path() const { return path_; }
  PlanInfo info() const;

  // Batched transform on device-resident data: `batch` contiguous transforms of size() samples,
  // in == out allowed (in place).  Enqueued on `stream`; not synchronised.
  cudaError_t exec_device(const C* in, C* out, size_t batch, int code, cudaStream_t stream);

  // Same on host memory (the reference ABI's case): staged H2D -> transform -> D2H through the
  // plan's own streams, chunked and pipelined; returns after the result is in `out`.
  cudaError_t exec_host(const C* in, C* out, size_t batch, int code);

  // Distributed six-step transform (dist_fft.cu): batched FFT of `rows` contiguous rows of size() samples whose last
  // register stage stores the result transposed, and optionally twiddled, straight into the destination ranks'
  // buffers: outs[q][c * out_ld + out_off + r] = X_r[q * cb + c] * w_Ntot^{(row0 + r) * (q * cb + c)}, cb = size() / nranks
  // (what launch_exchange() delivers after exec_device() on the same rows).  Two-pass sizes only; `in` is left intact.
  // rows_per_batch != 0 (three-pass path): the rows come in batches of that many, batch b goes out_batch_stride
  // elements further on: outs[q][b * out_batch_stride + c * out_ld + out_off + r % rows_per_batch]; rows_valid != 0:
  // only the first rows_valid rows exist, the rest pads the last tile (read, transformed, not stored).
  cudaError_t exec_rows_exchange(const C* in, size_t rows, bool forward, void* const* outs, int nranks, size_t out_ld,
                                 size_t out_off, int twiddle, unsigned long long row0, unsigned long long n_total,
                                 cudaStream_t stream, size_t rows_per_batch = 0, size_t out_batch_stride = 0,
                                 size_t rows_valid = 0);

  // Number of kernel launches the last exec_* call issued (bench.py reports it).
  unsigned long long launches() const { return launches_; }

  // Name of the kernel that moves (nearly) all of this plan's bytes -- what a profiler will list first.  For the
  // persistent two-pass kernel it is followed by the configuration the plan chose, e.g.
  // "fused::fused_twopass_kernel [1024x1024, 2 groups x 256, TMA staging, ring 4, lag 2]" (the ring and lag of a full
  // batch; exec_twopass shrinks the ring for a small one).
  const char* kernel_name() const;

 private:
  template <class P> friend P* create_plan(size_t, int, bool);
  Plan() = default;
  cudaError_t init(size_t n, int device, bool allow_fast_paths);

  cudaError_t exec_global_stages(const C* in, C* out, size_t batch, int code, cudaStream_t s);
  cudaError_t exec_onchip(const C* in, C* out, size_t batch, int code, cudaStream_t s);
  cudaError_t exec_twopass(const C* in, C* out, size_t batch, int code, cudaStream_t s);
  cudaError_t exec_bluestein(const C* in, C* out, size_t batch, int code, cudaStream_t s);
  cudaError_t exec_bluestein_fused(const C* in, C* out, size_t batch, int code, cudaStream_t s);
  cudaError_t exec_cta(const C* in, C* out, size_t batch, int code, cudaStream_t s, bool chirp);
  cudaError_t exec_bigpow2(const C* in, C* out, size_t batch, int code, cudaStream_t s);

  cudaError_t init_global_stages();
  cudaError_t init_onchip();
  cudaError_t init_twopass();
  cudaError_t init_bigpow2();
  cudaError_t init_threepass_radix3();
  cudaError_t init_cta(size_t len);   // len = n_, or the Bluestein inner size
  cudaError_t init_bluestein(bool allow_fast_paths);
  cudaError_t init_bluestein_fused(const std::vector<double>& chirp_re, const std::vector<double>& chirp_im,
                                   const std::vector<double>& w_re, const std::vector<double>& w_im);

  size_t n_ = 0;
  int device_ = 0;
  Path path_ = Path::kTrivial;
  unsigned long long launches_ = 0;

  // kGlobalStages: radices of the Stockham stages and the full forward table w_N^k, k < N
  std::vector<int> radices_;
  DeviceBuffer wtab_;

  // kOnChip / kTwoPass: see onchip.cu / twopass.cu
  size_t n1_ = 0, n2_ = 0;
  DeviceBuffer tw_a_, tw_b_, tw2_, tw_f_, tw_f2_;   // tw_f_, tw_f2_: stage twiddles of the persistent kernel's two register tiles
  const void* fast_ops_ = nullptr;   // TwoPassOps<T> / OnChipOps<T> of the selected kernel family
  size_t chunk_ = 0;                 // transforms per L2-resident chunk (two-pass)
  const void* fused_ops_ = nullptr;  // FusedOps<T>: persistent single-launch variant
  int ring_ = 0, lag_ = 0, sm_count_ = 132;
  std::string kernel_desc_;          // kernel_name() of the persistent kernel: tile lengths, groups, loads, ring, lag
  int outer_radix3_ = 0;             // kThreePass: 3 / 9 / 27 = the outer pass is a radix-3 DFT (N = 3^b * 2^k), 0 = power of two
  DeviceBuffer counters_, tbase_, tstep_, trace_;

  // kCta (and kBluesteinFused through the CTA kernel): on-chip transform length, radices_ and wtab_ as above
  size_t cta_len_ = 0;
  bool cta_chirp_ = false;

  // kBluestein*: chirp x[i] (N entries), W = FFT_M(wrapped chirp) (M entries), both forward;
  // the inverse direction uses their conjugate-symmetric counterparts computed at plan time.
  size_t m_ = 0;
  std::unique_ptr<Plan<T>> inner_;
  DeviceBuffer chirp_, wf_, wi_;

  // scratch (grow-only) and host staging
  DeviceBuffer work_, work2_;
  DeviceBuffer stage_[3];
  cudaStream_t streams_[3] = {nullptr, nullptr, nullptr};
  cudaEvent_t events_[9] = {};
  cudaError_t host_resources();   // streams and events of the host-pointer path, created once
  void* zc_in_ = nullptr;         // pinned, device-mapped bounce buffers of the smallest host calls (64 KB each)
  void* zc_out_ = nullptr;
};

// onchip.cu: the fused real-input kernels of the on-chip size class of L (onchip_lookup), N = 2L; nullptr when L has
// none.  run(): `in` / `out` are the reals (L complex values per row) and the spectrum (L+1 per row), swapped for the
// inverse; tab = w_N^k, k <= L/2; h = scale / 2 (forward) or scale (inverse).  conv(): y = irfft(rfft(x) . H) of
// real rows, in == out allowed; spec holds `rows` spectrum rows of L+1 bins, row b of the batch uses spectrum row
// ((row0 + b) / per) mod rows; h = 1 / (2N).  lconv(): segments g0 .. g0 + nseg - 1 of the linear convolution map m
// (real::SegMap, DESIGN.md §4.12), out of place; segment g uses spectrum row (g / m.per) mod rows; h = 1 / (2N).
// stft(): the rfft of the windowed frames g0 .. g0 + nframes - 1 of the frame map m (real::FrameMap, DESIGN.md
// §4.13) into consecutive spectrum rows from `out` on.
template <typename T> struct RealOnChipOps {
  int ra, rb;
  int cols;   // FFTs per CTA (the C of real::welch_items)
  cudaError_t (*prepare)();
  cudaError_t (*run)(const void* in, void* out, const void* twa, const cpx<T>* tab, size_t batch, bool fwd, T h,
                     int sms, cudaStream_t);
  cudaError_t (*conv)(const void* in, void* out, const void* twa, const cpx<T>* tab, const cpx<T>* spec, size_t rows,
                      size_t row0, size_t per, size_t batch, T h, int sms, cudaStream_t);
  cudaError_t (*lconv)(const T* in, T* out, const real::SegMap& m, size_t nseg, const void* twa, const cpx<T>* tab,
                       const cpx<T>* spec, size_t rows, T h, int sms, cudaStream_t);
  cudaError_t (*stft)(const T* in, const T* win, void* out, const real::FrameMap& m, size_t nframes, const void* twa,
                      const cpx<T>* tab, int sms, cudaStream_t);
  // mel(): the mel energies of the same frames (DESIGN.md §4.14), n_mels reals per frame from `out` on
  cudaError_t (*mel)(const T* in, const T* win, const T* filters, const real::Band* bands, size_t n_mels, int power,
                     T* out, const real::FrameMap& m, size_t nframes, const void* twa, const cpx<T>* tab, int sms,
                     cudaStream_t);
  // mfcc(): the MFCC / log-mel outputs of the same frames (DESIGN.md §4.18), p.n_out reals per frame from `out` on, or
  // with max_sweep only each frame's log-mel maximum folded into its group's slot (n_mels <= L - 1)
  cudaError_t (*mfcc)(const T* in, const T* win, const T* filters, const real::Band* bands, size_t n_mels, int power,
                      const real::MfccArgs<T>& p, bool max_sweep, T* out, const real::FrameMap& m, size_t nframes,
                      const void* twa, const cpx<T>* tab, int sms, cudaStream_t);
  // welch(): the Welch items w (DESIGN.md §4.15) of the rows of m, from `in` on: each item's partial into part, or, when
  // a row is one item, the row's output into out; base = s / F in device memory, detrend real::kDetrend*
  cudaError_t (*welch)(const T* in, const T* win, const T* base, int detrend, T* part, T* out, const real::FrameMap& m,
                       const real::WelchItems& w, const void* twa, const cpx<T>* tab, int sms, cudaStream_t);
  // dct(): the discrete cosine transform of type 2 or 3 (DESIGN.md §4.16) of `batch` rows of N reals, in == out
  // allowed; wq = W^k, k <= L; h, h0 from real::dct_scales
  cudaError_t (*dct)(const T* in, T* out, int type, const void* twa, const cpx<T>* tab, const cpx<T>* wq, size_t batch,
                     T h, T h0, int sms, cudaStream_t);
  // csd(): welch() on frame pairs (DESIGN.md §4.17): the cross-spectral density (coh false) or coherence items w over
  // cols / 2 pair columns of the rows of m from x on, row b with y row (y_off + b) mod y_rows; out: cpx<T> or T rows
  cudaError_t (*csd)(const T* x, const T* y, size_t y_rows, size_t y_off, const T* win, const T* base, int detrend,
                     bool coh, T* part, void* out, const real::FrameMap& m, const real::WelchItems& w, const void* twa,
                     const cpx<T>* tab, int sms, cudaStream_t);
  // hilbert(): the analytic signal or its envelope (output real::kHilbert*, DESIGN.md §4.19) of `batch` rows of N reals
  // into N complex values or N reals per row, out == in allowed for the envelope; h = 1 / (2N)
  cudaError_t (*hilbert)(const T* in, void* out, int output, const void* twa, const cpx<T>* tab, size_t batch, T h,
                         int sms, cudaStream_t);
  // dct4(): the type-IV DCT (DESIGN.md §4.20) of `batch` rows of N reals, in == out allowed; wq = W^k, k <= L; c from
  // real::dct4_const
  cudaError_t (*dct4)(const T* in, T* out, const void* twa, const cpx<T>* wq, cpx<T> c, size_t batch, int sms,
                      cudaStream_t);
  // mdct(): the MDCT of frames m.g0 .. m.g0 + nframes - 1 of m (real::mdct_map), frame q of the launch writing its N
  // coefficients at out + q N
  cudaError_t (*mdct)(const T* in, const T* win, T* out, const real::FrameMap& m, size_t nframes, const void* twa,
                      const cpx<T>* wq, cpx<T> c, int sms, cudaStream_t);
};
template <typename T> const RealOnChipOps<T>* real_onchip_lookup(size_t l);

// Batched real-input transform of length N (real.cu, DESIGN.md §4.10).  Forward: `batch` rows of N reals -> rows of
// N/2+1 complex bins (numpy's rfft layout); inverse: the other way round (numpy's irfft).  Out of place only.
// convolve_*: both in one call with a pointwise multiply between them (DESIGN.md §4.11), in place allowed.
// linear_convolve_*: linear convolution of rows of any length by overlap-save on the same paths (DESIGN.md §4.12).
template <typename T>
class RealPlan {
 public:
  using C = cpx<T>;

  // nullptr (and last_error set) when the plan cannot be built; size 0 is refused
  static RealPlan* create(size_t n, int device, bool allow_fast_paths = true) {
    return create_plan<RealPlan>(n, device, allow_fast_paths);
  }
  ~RealPlan();

  size_t size() const { return n_; }
  Path path() const { return path_; }
  PlanInfo info() const;

  // Device pointers, enqueued on `stream`, not synchronised.  `forward` selects the direction; a code of the other
  // direction is refused.
  cudaError_t exec_device(bool forward, const void* in, void* out, size_t batch, int code, cudaStream_t stream);
  // Host pointers: staged through the plan's device buffers in chunks, the same device code; returns when `out` is done.
  cudaError_t exec_host(bool forward, const void* in, void* out, size_t batch, int code);

  // Circular convolution (DESIGN.md §4.11): out[b] = irfft(rfft(in[b]) . spec[b mod rows], n = N) for `batch` rows of
  // N reals; `spec` holds rows >= 1 spectra of N/2+1 bins in the rfft layout.  in == out allowed.  Device pointers,
  // enqueued on `stream`, not synchronised.
  cudaError_t convolve_device(const T* in, const C* spec, size_t rows, T* out, size_t batch, cudaStream_t stream) {
    launches_ = 0;
    return convolve_rows(in, spec, rows, 0, 1, out, batch, stream);
  }
  // Host pointers: the spectra are staged once, the rows in chunks as in exec_host; returns when `out` is done.
  cudaError_t convolve_host(const T* in, const C* spec, size_t rows, T* out, size_t batch);

  // Linear convolution by overlap-save (DESIGN.md §4.12): `batch` rows of in_len reals -> rows of
  // real::linear_out_len(mode, in_len, taps) reals, out[b][i] = y_full[off + i], y_full = row b (*) c, where
  // c = irfft(spec[b mod rows], n = N) must vanish beyond its first `taps` samples.  1 <= taps <= N, in_len >= 1 (>= taps
  // for valid), mode real::kLinear*; checked by the caller.  Out of place only.  Device pointers, enqueued on `stream`.
  cudaError_t linear_convolve_device(const T* in, size_t in_len, const C* spec, size_t rows, size_t taps, int mode,
                                     T* out, size_t batch, cudaStream_t stream);
  // Host pointers: the spectra are staged once; whole rows in chunks when a row's input and output fit the staging
  // chunk, else runs of segments of one row with only the input window they read; the same device code and bits.
  cudaError_t linear_convolve_host(const T* in, size_t in_len, const C* spec, size_t rows, size_t taps, int mode,
                                   T* out, size_t batch);

  // Short-time Fourier transform (DESIGN.md §4.13): `batch` rows of in_len reals -> F = real::stft_frames(...) rows of
  // N/2+1 bins per input row, frame-major, frame f = rfft(window . frame f of the row).  hop >= 1, boundary
  // real::kStft*, in_len legal for it; checked by the caller.  Out of place only.  Device pointers, on `stream`.
  cudaError_t stft_device(const T* in, size_t in_len, const T* win, size_t hop, int boundary, C* out, size_t batch,
                          cudaStream_t stream);
  // Inverse: `batch` rows of `frames` spectra -> rows of out_len reals, the windowed overlap-add of the frames' irfft
  // divided by the window envelope (0 where it is below 1e-11); pad = N/2 if center.  Device pointers, on `stream`.
  cudaError_t istft_device(const C* in, size_t frames, const T* win, size_t hop, bool center, T* out, size_t out_len,
                           size_t batch, cudaStream_t stream);
  // Host pointers: the window is staged once, whole rows in chunks through stage_rows; the same device code and bits.
  cudaError_t stft_host(const T* in, size_t in_len, const T* win, size_t hop, int boundary, C* out, size_t batch);
  cudaError_t istft_host(const C* in, size_t frames, const T* win, size_t hop, bool center, T* out, size_t out_len,
                         size_t batch);

  // Mel spectrogram (DESIGN.md §4.14): the frames of stft_device -> n_mels reals each, frame-major,
  // out[b][f][m] = sum_k filters[m][k] |X_{b,f}[k]|^power, filters a row-major (n_mels, N/2+1) matrix, power 1 or 2,
  // n_mels >= 1; checked by the caller with the stft's arguments.  Out of place only.  Device pointers, on `stream`.
  cudaError_t mel_device(const T* in, size_t in_len, const T* win, size_t hop, int boundary, const T* filters,
                         size_t n_mels, int power, T* out, size_t batch, cudaStream_t stream);
  // Host pointers: the window and the filters are staged once, whole rows through stage_rows; the same bits.
  cudaError_t mel_host(const T* in, size_t in_len, const T* win, size_t hop, int boundary, const T* filters,
                       size_t n_mels, int power, T* out, size_t batch);

  // MFCC and log-mel spectrogram (DESIGN.md §4.18): the mels of mel_device -> n_out reals per frame, frame-major,
  // out[b][f][j] = sum_m max(scale ln(max(mel + offset, floor)), theta_g) dct[m][j] + bias (real::MfccArgs; dct nullptr:
  // the identity).  With top_db finite, theta_g = max over clamp group g (top_db_rows consecutive rows, batch a multiple
  // of it) of the logs - top_db, found by a first sweep over the frames; else -inf.  Scalars finite, floor and scale > 0,
  // checked by the caller with the mel spectrogram's arguments.  Out of place only.  Device pointers, on `stream`.
  cudaError_t mfcc_device(const T* in, size_t in_len, const T* win, size_t hop, int boundary, int power,
                          const T* filters, size_t n_mels, double log_offset, double log_floor, double log_scale,
                          double top_db, size_t top_db_rows, const T* dct, size_t n_out, double bias, T* out,
                          size_t batch, cudaStream_t stream);
  // Host pointers: the window, filters and matrix are staged once, whole rows through stage_rows (twice with the clamp);
  // the same bits.
  cudaError_t mfcc_host(const T* in, size_t in_len, const T* win, size_t hop, int boundary, int power, const T* filters,
                        size_t n_mels, double log_offset, double log_floor, double log_scale, double top_db,
                        size_t top_db_rows, const T* dct, size_t n_out, double bias, T* out, size_t batch);

  // Welch power spectral density (DESIGN.md §4.15): `batch` rows of in_len >= N reals -> N/2+1 reals each, out[b][k] =
  // c_k s / F sum_f |rfft(win . (frame f - its mean))[k]|^2 over the F frames of hop `hop` (no padding), the mean only
  // with detrend real::kDetrendConstant, s from scaling real::kWelch* and fs.  Arguments checked by the caller.  Out of
  // place only.  Device pointers, on `stream`, never synchronised: the window sums are formed on the device.
  cudaError_t welch_device(const T* in, size_t in_len, const T* win, size_t hop, int detrend, int scaling, double fs,
                           T* out, size_t batch, cudaStream_t stream);
  // Host pointers: the window is staged once, whole rows through stage_rows; the same bits.
  cudaError_t welch_host(const T* in, size_t in_len, const T* win, size_t hop, int detrend, int scaling, double fs,
                         T* out, size_t batch);

  // Cross-spectral density and coherence (DESIGN.md §4.17): `batch` rows x of in_len >= N reals, row b paired with y row
  // b mod y_rows (y_rows >= 1 rows of in_len reals), both framed, detrended and windowed as welch_device.  coh false:
  // out[b][k] = c_k s / F sum_f conj(X_bf[k]) Y_bf[k], N/2+1 complex values per row; coh true: out[b][k] =
  // |sum_f conj(X) Y|^2 / (sum_f |X|^2 sum_f |Y|^2), N/2+1 reals per row (scaling and fs unused).  y nullptr with coh
  // false and y_rows 1: welch_device.  Arguments checked by the caller.  Out of place only.  Device pointers, on
  // `stream`, never synchronised.
  cudaError_t cross_device(const T* x, const T* y, size_t y_rows, size_t in_len, const T* win, size_t hop, int detrend,
                           bool coh, int scaling, double fs, void* out, size_t batch, cudaStream_t stream);
  // Host pointers: the window is staged once, x rows through stage_rows and each chunk's y rows beside them; the same
  // bits.
  cudaError_t cross_host(const T* x, const T* y, size_t y_rows, size_t in_len, const T* win, size_t hop, int detrend,
                         bool coh, int scaling, double fs, void* out, size_t batch);

  // Discrete cosine transform (DESIGN.md §4.16): `batch` rows of N reals -> rows of N reals, scipy.fft.dct(x, type,
  // norm), type 2 or 3, norm real::kDctNorm*; checked by the caller.  in == out allowed.  Device pointers, on `stream`.
  cudaError_t dct_device(const T* in, T* out, size_t batch, int type, int norm, cudaStream_t stream);
  // Host pointers: whole rows through stage_rows; the same bits.
  cudaError_t dct_host(const T* in, T* out, size_t batch, int type, int norm);

  // Analytic signal (DESIGN.md §4.19): `batch` rows of N reals -> scipy.signal.hilbert of each row, N complex values
  // (x[n], y[n]) per row with the real part a copy of x (output real::kHilbertAnalytic), or its modulus, N reals per row
  // (real::kHilbertEnvelope); checked by the caller.  in == out allowed for the envelope, else out of place.  Device
  // pointers, on `stream`.
  cudaError_t hilbert_device(const T* in, void* out, size_t batch, int output, cudaStream_t stream);
  // Host pointers: whole rows through stage_rows; the same bits.
  cudaError_t hilbert_host(const T* in, void* out, size_t batch, int output);

  // Type-IV DCT and MDCT (DESIGN.md §4.20), even N only; norm real::kDctNorm*, the other arguments checked by the caller.
  // dct4: `batch` rows of N reals -> scipy.fft.dct(x, type=4, norm), in == out allowed.  mdct: rows of in_len samples ->
  // F = mdct_frames(in_len, center) frames of N coefficients per row, frame-major.  imdct: rows of `frames` frames of N
  // coefficients -> rows of out_len samples, the windowed overlap-add of the inverse.  Device pointers, on `stream`.
  cudaError_t dct4_device(const T* in, T* out, size_t batch, int norm, cudaStream_t stream);
  cudaError_t mdct_device(const T* in, size_t in_len, const T* win, bool center, int norm, T* out, size_t batch,
                          cudaStream_t stream);
  cudaError_t imdct_device(const T* in, size_t frames, const T* win, bool center, int norm, T* out, size_t out_len,
                           size_t batch, cudaStream_t stream);
  // Host pointers: the window once, whole rows through stage_rows; the same bits.
  cudaError_t dct4_host(const T* in, T* out, size_t batch, int norm);
  cudaError_t mdct_host(const T* in, size_t in_len, const T* win, bool center, int norm, T* out, size_t batch);
  cudaError_t imdct_host(const T* in, size_t frames, const T* win, bool center, int norm, T* out, size_t out_len,
                         size_t batch);
  // frames of one MDCT row of in_len samples (real::mdct_map)
  size_t mdct_frames(size_t in_len, bool center) const {
    return (size_t)real::mdct_map((long)n_, (long)in_len, center).frames;
  }

  unsigned long long launches() const { return launches_; }
  const char* kernel_name() const { return kernel_desc_.c_str(); }

  // cudaErrorInvalidValue (and last_error set) for an unknown code or one of the other direction
  cudaError_t check_code(bool forward, int code) const;

  // bytes of one input / output row
  size_t row_bytes(bool forward, bool input) const {
    const size_t real = n_ * sizeof(T), spec = (n_ / 2 + 1) * sizeof(C);
    return forward == input ? real : spec;
  }
  // bytes of `rows` spectra of N/2+1 bins: a convolution's spectra, or one istft input row of `rows` frames
  size_t spec_bytes(size_t rows) const { return rows * (n_ / 2 + 1) * sizeof(C); }
  // bytes of one stft output row (a spectrum per frame) and of one mel output row (n_mels reals per frame)
  size_t stft_row_bytes(size_t in_len, size_t hop, int boundary) const {
    return spec_bytes(frame_count(in_len, hop, boundary));
  }
  size_t mel_row_bytes(size_t in_len, size_t hop, int boundary, size_t n_mels) const {
    return frame_count(in_len, hop, boundary) * n_mels * sizeof(T);
  }
  // an MFCC call runs the fused kernel: a fused plan, and n_mels <= L - 1 log-mels fit the park behind the L+1 powers
  bool mfcc_fused(size_t n_mels) const { return path_ == Path::kRealFused && n_mels + 1 <= m_; }

 private:
  template <class P> friend P* create_plan(size_t, int, bool);
  RealPlan() = default;
  cudaError_t init(size_t n, int device, bool allow_fast_paths);
  // frames of one stft / mel row
  size_t frame_count(size_t in_len, size_t hop, int boundary) const {
    return (size_t)real::frame_map((long)n_, (long)in_len, (long)hop, boundary).frames;
  }
  // exec_device after its checks
  cudaError_t rfft_rows(bool forward, const void* in, void* out, size_t batch, int code, cudaStream_t s);
  // convolve_device with row b using spectrum row ((row0 + b) / per) mod rows
  cudaError_t convolve_rows(const T* in, const C* spec, size_t rows, size_t row0, size_t per, T* out, size_t batch,
                            cudaStream_t s);
  // segments m.g0 .. m.g0 + nseg - 1 of a linear convolution: the fused kernel, or chunks of gather, convolve_rows and
  // scatter through seg_
  cudaError_t linear_segments(const T* in, T* out, const real::SegMap& m, size_t nseg, const C* spec, size_t rows,
                              cudaStream_t s);
  // stft_device, istft_device and dct_device after their checks: the fused kernel, or chunks through seg_
  cudaError_t stft_rows(const T* in, size_t in_len, const T* win, size_t hop, int boundary, C* out, size_t batch,
                        cudaStream_t s);
  cudaError_t istft_rows(const C* in, size_t frames, const T* win, size_t hop, bool center, T* out, size_t out_len,
                         size_t batch, cudaStream_t s);
  cudaError_t dct_rows(const T* in, T* out, size_t batch, int type, int norm, cudaStream_t s);
  // hilbert_device after its checks: the fused kernel, or chunks of rows through seg_ (half length) or work_ (full)
  cudaError_t hilbert_rows(const T* in, void* out, size_t batch, int output, cudaStream_t s);
  // dct4_device after its checks: the fused kernel, or chunks of rows through `scratch` (half length)
  cudaError_t dct4_rows(const T* in, T* out, size_t batch, int norm, DeviceBuffer& scratch, cudaStream_t s);
  // mdct_device and imdct_device after their checks: the fused kernel or chunks of frames through seg_; runs of frames
  // (real::istft_runs) through seg_, their DCT-IV by dct4_rows (its scratch work_), then the overlap-add
  cudaError_t mdct_rows(const T* in, size_t in_len, const T* win, bool center, int norm, T* out, size_t batch,
                        cudaStream_t s);
  cudaError_t imdct_rows(const T* in, size_t frames, const T* win, bool center, int norm, T* out, size_t out_len,
                         size_t batch, cudaStream_t s);
  // the band of every filter row into bands_ (one launch)
  cudaError_t mel_bands(const T* filters, size_t n_mels, cudaStream_t s);
  // mel_device after mel_bands: the fused kernel, or chunks of frames through seg_
  cudaError_t mel_rows(const T* in, size_t in_len, const T* win, size_t hop, int boundary, const T* filters,
                       size_t n_mels, int power, T* out, size_t batch, cudaStream_t s);
  // one sweep of an MFCC call after mel_bands over `batch` rows (p.row0 the first one's row in the call): the max sweep
  // (max_sweep) or the output sweep, by the fused kernel or chunks of frames through seg_
  cudaError_t mfcc_rows(const T* in, size_t in_len, const T* win, size_t hop, int boundary, int power,
                        const T* filters, size_t n_mels, const real::MfccArgs<T>& p, bool max_sweep, T* out,
                        size_t batch, cudaStream_t s);
  // the MfccArgs of a call from its double scalars (each rounded to T once) and the slots of its groups in slots_, set
  // to 0 on `s` when the clamp is on (a memset, not counted as a launch)
  cudaError_t mfcc_args(double log_offset, double log_floor, double log_scale, double top_db, size_t top_db_rows,
                        const T* dct, size_t n_out, double bias, size_t batch, cudaStream_t s, real::MfccArgs<T>* p);
  // s / F of a Welch call from the window into welch_base_ (one launch)
  cudaError_t welch_scale(const T* win, int scaling, double fs, size_t frames, cudaStream_t s);
  // cross_device after welch_scale (Welch and csd): row b of x with y row (y_off + b) mod y_rows, or alone (y nullptr:
  // Welch); chunks of rows whose partials fit part_, each through the fused kernel or chunks of frames (x and y frame
  // pairs) through seg_, then the finish
  cudaError_t welch_cross_rows(const T* x, const T* y, size_t y_rows, size_t y_off, size_t in_len, const T* win,
                               size_t hop, int detrend, bool coh, void* out, size_t batch, cudaStream_t s);
  // Frames 0 .. total-1 of m, k per index, in chunks through seg_: per chunk gather(seg, mc, nq) (one launch), the
  // plan's rfft of the chunk's k * nq frames into spec_out + k * q0 spectra or into seg_ behind the frames, then
  // use(spec, q0, nq, extra_region) with `extra` bytes per index behind the spectra (real.cu).
  template <class Gather, class Use>
  cudaError_t frame_chunks(const real::FrameMap& m, size_t total, size_t k, C* spec_out, size_t extra, cudaStream_t s,
                           Gather gather, Use use);
  // The host-pointer loop (real.cu): chunks of rows of in_row / out_row bytes go H2D, through
  // step(dev_in, dev_out, first_row, rows) on host_stream_, and D2H (nothing with out_row 0).
  template <class Step>
  cudaError_t stage_rows(const void* in, void* out, size_t batch, size_t in_row, size_t out_row, Step step);
  // A host-pointer call's constant operands, a and optionally b, go H2D into stage_spec_ on host_stream_, each at a
  // 256-byte-aligned offset; *da and *db are their device copies.  The caller holds the DeviceGuard.
  template <class A, class B = A>
  cudaError_t stage_consts(const A* a, size_t a_bytes, const A** da, const B* b = nullptr, size_t b_bytes = 0,
                           const B** db = nullptr);
  // creates host_stream_ on the first host-pointer call
  cudaError_t open_host_stream();

  size_t n_ = 0, m_ = 0;        // m_ = N/2 (even N)
  int device_ = 0;
  Path path_ = Path::kRealFull;
  // launches() of the last call: each public method sets it to 0 at its start, and every private step adds the launches
  // it makes, 1 per kernel and inner_->launches() after each call of the inner plan
  unsigned long long launches_ = 0;
  int sm_count_ = 132;
  const RealOnChipOps<T>* fused_ = nullptr;
  std::unique_ptr<Plan<T>> inner_;   // length N/2 (kRealHalf) or N (kRealFull)
  DeviceBuffer tab_, twa_;           // w_N^k, k <= N/4 (even N); stage twiddles of the fused kernel
  DeviceBuffer dct_tab_;             // W^k = exp(-i pi k / (2N)), k <= N/2: the twiddles of the DCT
  DeviceBuffer work_;                // one chunk of inner-plan rows
  DeviceBuffer stage_in_, stage_out_;
  DeviceBuffer stage_spec_;          // the constant operands of a host-pointer call: spectra, window, filters
  DeviceBuffer seg_;                 // one chunk of N-real segments or frames (real::FrameMap: the frames' spectra
                                     // and per-frame values behind them)
  DeviceBuffer bands_;               // the filter bands of the last mel call (real::Band per filter row)
  DeviceBuffer slots_;               // the clamp groups' maxima of the last MFCC call (real::MaxKey<T> per group)
  DeviceBuffer welch_base_;          // s / F of the last Welch call (one T)
  DeviceBuffer part_;                // one chunk of rows of Welch partials (N/2+1 reals per item; 2 or 4 planes of
                                     // them for the csd and coherence)
  DeviceBuffer stage_y_;             // the y rows of one host-pointer chunk of a csd or coherence call
  DeviceBuffer stage_dct_;           // the projection matrix of a host-pointer MFCC call
  cudaStream_t host_stream_ = nullptr;
  std::string kernel_desc_;
};

// ---- kernel launchers implemented in the .cu files ------------------------------------------------

// stockham_generic.cu
template <typename T>
cudaError_t launch_stockham_stage(int radix, const cpx<T>* in, cpx<T>* out, const cpx<T>* wtab, size_t n,
                                  size_t sub_size, size_t stride, size_t batch, bool forward, bool last,
                                  T scale, cudaStream_t s);
template <typename T>
cudaError_t launch_scale_copy(const cpx<T>* in, cpx<T>* out, size_t count, T scale, cudaStream_t s);
template <typename T>
cudaError_t launch_chirp_in(const cpx<T>* in, cpx<T>* work, const cpx<T>* chirp, size_t n, size_t m,
                            size_t batch, bool forward, cudaStream_t s);
template <typename T>
cudaError_t launch_pointwise(cpx<T>* work, const cpx<T>* w, size_t m, size_t batch, bool forward,
                             cudaStream_t s);
template <typename T>
cudaError_t launch_chirp_out(const cpx<T>* work, cpx<T>* out, const cpx<T>* chirp, size_t n, size_t m,
                             size_t batch, bool forward, T scale, cudaStream_t s);

// synth.cu: counter-hash synthetic input (same generator as oracle/fourier_oracle.c fo_fill_input_*)
template <typename T>
cudaError_t launch_fill_input(T* out, unsigned long long first_scalar, size_t count,
                              unsigned long long seed, cudaStream_t s);

// synth.cu: helpers of the distributed six-step transform
template <typename T>
cudaError_t launch_transpose(const cpx<T>* in, cpx<T>* out, size_t batch, size_t rows, size_t cols, cudaStream_t s);
template <typename T>
cudaError_t launch_pack(const cpx<T>* in, cpx<T>* out, size_t batch, size_t rows, size_t cols, size_t ld, size_t ibs,
                        size_t obs, int twiddle, unsigned long long row0, unsigned long long col0,
                        unsigned long long n_total, cudaStream_t s);
template <typename T>
cudaError_t launch_swap_leading(const cpx<T>* in, cpx<T>* out, size_t a, size_t b, size_t inner, cudaStream_t s);
template <typename T>
cudaError_t launch_twiddle_rows(cpx<T>* data, size_t rows, size_t cols, unsigned long long row0,
                                unsigned long long n_total, bool forward, cudaStream_t s);

// exchange.cu: exchange step of the distributed transform over NVLink peer memory + CUDA-IPC plumbing
template <typename T>
cudaError_t launch_exchange(const cpx<T>* in, void* const* outs, int nranks, int me, size_t rows, size_t cb, size_t ld,
                            size_t out_ld, size_t out_off, int twiddle, unsigned long long row0,
                            unsigned long long n_total, cudaStream_t s);
cudaError_t peer_alloc(size_t bytes, void** ptr, void* handle64);
cudaError_t peer_open(const void* handle64, void** ptr);
cudaError_t peer_close(void* ptr);
cudaError_t peer_free(void* ptr);

// host math helpers (plan_math.cpp part of plan.cu)
void host_twiddle(size_t k, size_t n, double* re, double* im);            // exp(-2*pi*i*k/n), long-double accurate
void host_fft_pow2(std::vector<double>& re, std::vector<double>& im, bool inverse);  // unscaled, in place

}  // namespace fb200
