// capi.cu -- the C ABI of libfourier.so: the eight reference symbols (include/fourier.h, replacing
// fourier-ffi/src/lib.rs:14-106) and the additive batched / device-pointer entry points
// (include/fourier_b200.h), real-input transforms included.  No torch types, plain pointers and sizes only.
//
// Error convention of the reference symbols (fourier-ffi/src/lib.rs): create returns NULL when the
// constructor fails; transform_* / destroy swallow every failure (catch_unwind) and return nothing.
// Only the C ABI is exported; everything else in the library is built with -fvisibility=hidden.
#pragma GCC visibility push(default)
#include "../../include/fourier_b200.h"
#pragma GCC visibility pop

#include <cmath>
#include <cstdint>
#include <initializer_list>
#include <new>

#include "plan.h"

using fb200::Plan;
using fb200::RealPlan;

namespace {

thread_local int g_device = -1;

int resolve_device() {
  if (g_device >= 0) return g_device;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return -1;
  return dev;
}

// host memory (pageable or pinned) -> false; device / managed memory -> true
bool is_device_pointer(const void* p) {
  cudaPointerAttributes attr;
  if (cudaPointerGetAttributes(&attr, p) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged;
}

// Where the buffers of a synchronous call live: 1 all in device memory, 0 all in host memory, -1 a mix, which is
// refused (last_error set to `mix`).
int residence(std::initializer_list<const void*> bufs, const char* mix) {
  const bool dev = is_device_pointer(*bufs.begin());
  for (auto p = bufs.begin() + 1; p != bufs.end(); ++p)
    if (is_device_pointer(*p) != dev) {
      fb200::set_last_error(mix);
      return -1;
    }
  return dev ? 1 : 0;
}

// The kernels read and write device buffers with 16-byte vector accesses (cpx<double> as double2, f32 pairs as
// float4, TMA tensor maps on the input): a misaligned device pointer would fault and poison the CUDA context, so it
// is refused up front.  (cudaMalloc and torch allocations are 256/512-byte aligned; a slice starting at an odd f32
// sample is not.)  Host pointers are staged through the library's own buffers and may have any alignment.
bool device_pointers_aligned(std::initializer_list<const void*> bufs) {
  uintptr_t bits = 0;
  for (const void* p : bufs) bits |= (uintptr_t)p;
  if (bits & 15) {
    fb200::set_last_error("device buffers must be 16-byte aligned");
    return false;
  }
  return true;
}

// Plan<T> or RealPlan<T> on the calling thread's device
template <class P>
void* create(size_t size, bool fast) {
  const int dev = resolve_device();
  if (dev < 0) {
    fb200::set_last_error("no usable CUDA device (libfourier.so has no CPU fallback)");
    return nullptr;
  }
  try {
    return P::create(size, dev, fast);
  } catch (...) {
    fb200::set_last_error("plan construction threw");
    return nullptr;
  }
}

// returned by run_call's checks() to go on with the call
constexpr int kRun = -1;

// The end of every batched entry point, after its checks that need no plan.  checks() makes the entry point's other
// checks and returns kRun, or else the call's result.  A synchronous call then needs `bufs` all in host or all in
// device memory (else last_error = `mix`), and runs host() on host memory.  Otherwise the device buffers `aligned`
// must be 16-byte aligned, and device(s) runs on the caller's `stream` if async (not synchronised), else on the
// per-thread default stream, synchronised.  An exception becomes "<what> threw".
template <class Checks, class Host, class Device>
int run_call(const char* what, bool async, void* stream, Checks checks, std::initializer_list<const void*> bufs,
             const char* mix, Host host, std::initializer_list<const void*> aligned, Device device) {
  try {
    if (const int rc = checks(); rc != kRun) return rc;
    if (!async) {
      const int dev = residence(bufs, mix);
      if (dev < 0) return (int)cudaErrorInvalidValue;
      if (!dev) return (int)host();
    }
    if (!device_pointers_aligned(aligned)) return (int)cudaErrorMisalignedAddress;
    cudaStream_t s = async ? (cudaStream_t)stream : cudaStreamPerThread;
    cudaError_t e = device(s);
    if (e != cudaSuccess || async) return (int)e;
    return (int)cudaStreamSynchronize(s);
  } catch (...) {
    fb200::set_last_error(std::string(what) + " threw");
    return (int)cudaErrorUnknown;
  }
}

template <typename T>
int fft_exec(const void* plan, const void* in, void* out, size_t batch, int code, bool async, void* stream) {
  if (!plan || !in || !out) { fb200::set_last_error("null argument"); return (int)cudaErrorInvalidValue; }
  auto* p = const_cast<Plan<T>*>(static_cast<const Plan<T>*>(plan));
  using C = typename Plan<T>::C;
  return run_call(
      "transform", async, stream, [] { return kRun; },
      {in, out}, "input and output must both be host or both be device memory",
      [&] { return p->exec_host((const C*)in, (C*)out, batch, code); },
      {in, out}, [&](cudaStream_t s) { return p->exec_device((const C*)in, (C*)out, batch, code, s); });
}

template <typename T>
int rows_exchange(const void* plan, const void* in, size_t rows, int forward, void* const* outs, int nranks,
                  size_t out_ld, size_t out_off, int twiddle, unsigned long long row0, unsigned long long n_total,
                  void* stream) {
  if (!plan || !in || !outs) { fb200::set_last_error("null argument"); return (int)cudaErrorInvalidValue; }
  auto* p = const_cast<Plan<T>*>(static_cast<const Plan<T>*>(plan));
  using C = typename Plan<T>::C;
  try {
    if (!device_pointers_aligned({in})) return (int)cudaErrorMisalignedAddress;
    return (int)p->exec_rows_exchange((const C*)in, rows, forward != 0, outs, nranks, out_ld, out_off, twiddle, row0,
                                      n_total, (cudaStream_t)stream);
  } catch (...) {
    fb200::set_last_error("rows_exchange threw");
    return (int)cudaErrorUnknown;
  }
}

// Plan<T> or RealPlan<T>
template <class P>
int plan_info(const void* plan, fourier_b200_plan_info* out) {
  if (!plan || !out) { fb200::set_last_error("null argument"); return (int)cudaErrorInvalidValue; }
  const auto* p = static_cast<const P*>(plan);
  const fb200::PlanInfo i = p->info();
  out->size = i.size; out->path = i.path; out->inner_size = i.inner_size; out->inner_path = i.inner_path;
  out->n1 = i.n1; out->n2 = i.n2; out->precision_bytes = i.precision_bytes; out->device = i.device;
  out->table_bytes = i.table_bytes; out->last_launches = p->launches();
  return 0;
}

// the byte ranges [a, a + a_bytes) and [b, b + b_bytes) share a byte
bool ranges_meet(const void* a, size_t a_bytes, const void* b, size_t b_bytes) {
  const uintptr_t x = (uintptr_t)a, y = (uintptr_t)b;
  return x < y + b_bytes && y < x + a_bytes;
}

// Real transforms are out of place: the byte ranges [in, in + in_bytes) and [out, out + out_bytes) must not meet.
bool disjoint(const void* in, size_t in_bytes, const void* out, size_t out_bytes) {
  if (ranges_meet(in, in_bytes, out, out_bytes)) {
    fb200::set_last_error("input and output overlap (real transforms are out of place only)");
    return false;
  }
  return true;
}

template <typename T>
int rfft_exec(void* plan, bool forward, const void* in, void* out, size_t batch, int code, bool async, void* stream) {
  if (!plan || !in || !out) { fb200::set_last_error("null argument"); return (int)cudaErrorInvalidValue; }
  auto* p = static_cast<RealPlan<T>*>(plan);
  return run_call(
      "real transform", async, stream,
      [&] {
        if (cudaError_t e = p->check_code(forward, code)) return (int)e;
        if (batch == 0) return (int)p->exec_device(forward, in, out, 0, code, nullptr);
        if (!disjoint(in, batch * p->row_bytes(forward, true), out, batch * p->row_bytes(forward, false)))
          return (int)cudaErrorInvalidValue;
        return kRun;
      },
      {in, out}, "input and output must both be host or both be device memory",
      [&] { return p->exec_host(forward, in, out, batch, code); },
      {in, out}, [&](cudaStream_t s) { return p->exec_device(forward, in, out, batch, code, s); });
}

// Convolution of real rows: in == out allowed, otherwise in, out and spectrum as for rfft_exec.
template <typename T>
int convolve_exec(void* plan, const T* in, const void* spectrum, size_t rows, T* out, size_t batch, bool async,
                  void* stream) {
  if (!plan || !in || !out || !spectrum) { fb200::set_last_error("null argument"); return (int)cudaErrorInvalidValue; }
  if (rows == 0) { fb200::set_last_error("spectrum_rows must be at least 1"); return (int)cudaErrorInvalidValue; }
  auto* p = static_cast<RealPlan<T>*>(plan);
  using C = typename RealPlan<T>::C;
  const C* spec = static_cast<const C*>(spectrum);
  return run_call(
      "convolution", async, stream,
      [&] {
        if (batch == 0) return (int)p->convolve_device(in, spec, rows, out, 0, nullptr);
        const size_t bytes = batch * p->size() * sizeof(T);
        if (in != out && ranges_meet(in, bytes, out, bytes)) {
          fb200::set_last_error("input and output overlap (they must be the same buffer or disjoint)");
          return (int)cudaErrorInvalidValue;
        }
        if (ranges_meet(spectrum, p->spec_bytes(rows), out, bytes)) {
          fb200::set_last_error("spectrum and output overlap");
          return (int)cudaErrorInvalidValue;
        }
        return kRun;
      },
      {in, spectrum, out}, "input, spectrum and output must all be host or all be device memory",
      [&] { return p->convolve_host(in, spec, rows, out, batch); },
      {in, out, spectrum}, [&](cudaStream_t s) { return p->convolve_device(in, spec, rows, out, batch, s); });
}

// Linear convolution of real rows by overlap-save: out of place only; scalar arguments are checked before the plan is
// touched, even for batch == 0.
template <typename T>
int linear_exec(void* plan, const T* in, size_t in_len, const void* spectrum, size_t rows, size_t taps, int mode, T* out,
                size_t batch, bool async, void* stream) {
  if (!plan || !in || !out || !spectrum) { fb200::set_last_error("null argument"); return (int)cudaErrorInvalidValue; }
  const char* bad = rows == 0                                      ? "spectrum_rows must be at least 1"
                    : taps == 0                                    ? "taps must be at least 1"
                    : in_len == 0                                  ? "in_len must be at least 1"
                    : mode < 0 || mode > 2                         ? "unknown mode (FOURIER_B200_LINEAR_FULL, _SAME or _VALID)"
                    : mode == fb200::real::kLinearValid && in_len < taps ? "mode valid needs in_len >= taps"
                                                                   : nullptr;
  if (bad) { fb200::set_last_error(bad); return (int)cudaErrorInvalidValue; }
  auto* p = static_cast<RealPlan<T>*>(plan);
  using C = typename RealPlan<T>::C;
  const C* spec = static_cast<const C*>(spectrum);
  if (taps > p->size()) { fb200::set_last_error("taps must not exceed the plan length N"); return (int)cudaErrorInvalidValue; }
  return run_call(
      "linear convolution", async, stream,
      [&] {
        if (batch == 0) return (int)p->linear_convolve_device(in, in_len, spec, rows, taps, mode, out, 0, nullptr);
        const size_t in_bytes = batch * in_len * sizeof(T);
        const size_t out_bytes =
            batch * (size_t)fb200::real::linear_out_len(mode, (long)in_len, (long)taps) * sizeof(T);
        if (ranges_meet(in, in_bytes, out, out_bytes)) {
          fb200::set_last_error("input and output overlap (linear convolution is out of place only)");
          return (int)cudaErrorInvalidValue;
        }
        if (ranges_meet(spectrum, p->spec_bytes(rows), out, out_bytes)) {
          fb200::set_last_error("spectrum and output overlap");
          return (int)cudaErrorInvalidValue;
        }
        return kRun;
      },
      {in, spectrum, out}, "input, spectrum and output must all be host or all be device memory",
      [&] { return p->linear_convolve_host(in, in_len, spec, rows, taps, mode, out, batch); },
      {in, out, spectrum},
      [&](cudaStream_t s) { return p->linear_convolve_device(in, in_len, spec, rows, taps, mode, out, batch, s); });
}

// The framing checks of stft_exec and mel_exec, in this order: hop, boundary and in_len; then `bad`, the caller's
// refusal of its other scalar arguments (nullptr: none); then in_len against N, the only check that reads the plan.
template <typename T>
bool check_frames(const RealPlan<T>* p, size_t in_len, size_t hop, int boundary, const char* bad) {
  const char* why = hop == 0                          ? "hop must be at least 1"
                    : boundary < 0 || boundary > 2    ? "unknown boundary (FOURIER_B200_STFT_NONE, _ZEROS or _REFLECT)"
                    : in_len == 0                     ? "in_len must be at least 1"
                                                      : bad;
  if (!why) {
    const size_t n = p->size();
    why = boundary == fb200::real::kStftNone && in_len < n             ? "boundary none needs in_len >= N"
          : boundary == fb200::real::kStftReflect && in_len <= n / 2   ? "boundary reflect needs in_len > N/2"
                                                                       : nullptr;
  }
  if (why) fb200::set_last_error(why);
  return !why;
}

// Short-time Fourier transform of real rows: out of place only; the arguments are checked before the plan is touched,
// even for batch == 0, except in_len against N.
template <typename T>
int stft_exec(void* plan, const T* in, size_t in_len, const T* window, size_t hop, int boundary, void* out, size_t batch,
              bool async, void* stream) {
  if (!plan || !in || !window || !out) { fb200::set_last_error("null argument"); return (int)cudaErrorInvalidValue; }
  auto* p = static_cast<RealPlan<T>*>(plan);
  using C = typename RealPlan<T>::C;
  if (!check_frames(p, in_len, hop, boundary, nullptr)) return (int)cudaErrorInvalidValue;
  return run_call(
      "stft", async, stream,
      [&] {
        if (batch == 0) return (int)p->stft_device(in, in_len, window, hop, boundary, (C*)out, 0, nullptr);
        const size_t in_bytes = batch * in_len * sizeof(T), out_bytes = batch * p->stft_row_bytes(in_len, hop, boundary);
        if (ranges_meet(in, in_bytes, out, out_bytes) || ranges_meet(window, p->size() * sizeof(T), out, out_bytes)) {
          fb200::set_last_error("input or window and output overlap (the stft is out of place only)");
          return (int)cudaErrorInvalidValue;
        }
        return kRun;
      },
      {in, window, out}, "input, window and output must all be host or all be device memory",
      [&] { return p->stft_host(in, in_len, window, hop, boundary, (C*)out, batch); },
      {in, out}, [&](cudaStream_t s) { return p->stft_device(in, in_len, window, hop, boundary, (C*)out, batch, s); });
}

// Mel spectrogram of real rows: stft_exec's rules, plus power and n_mels checked before the plan is touched and the
// filters kept apart from the output.
template <typename T>
int mel_exec(void* plan, const T* in, size_t in_len, const T* window, size_t hop, int boundary, int power,
             const T* filters, size_t n_mels, T* out, size_t batch, bool async, void* stream) {
  if (!plan || !in || !window || !filters || !out) {
    fb200::set_last_error("null argument");
    return (int)cudaErrorInvalidValue;
  }
  auto* p = static_cast<RealPlan<T>*>(plan);
  if (!check_frames(p, in_len, hop, boundary,
                    power != 1 && power != 2 ? "power must be 1 or 2"
                    : n_mels == 0            ? "n_mels must be at least 1"
                                             : nullptr))
    return (int)cudaErrorInvalidValue;
  const size_t n = p->size();
  return run_call(
      "mel spectrogram", async, stream,
      [&] {
        if (batch == 0)
          return (int)p->mel_device(in, in_len, window, hop, boundary, filters, n_mels, power, out, 0, nullptr);
        const size_t in_bytes = batch * in_len * sizeof(T);
        const size_t out_bytes = batch * p->mel_row_bytes(in_len, hop, boundary, n_mels);
        if (ranges_meet(in, in_bytes, out, out_bytes) || ranges_meet(window, n * sizeof(T), out, out_bytes) ||
            ranges_meet(filters, n_mels * (n / 2 + 1) * sizeof(T), out, out_bytes)) {
          fb200::set_last_error(
              "input, window or filters and output overlap (the mel spectrogram is out of place only)");
          return (int)cudaErrorInvalidValue;
        }
        return kRun;
      },
      {in, window, filters, out}, "input, window, filters and output must all be host or all be device memory",
      [&] { return p->mel_host(in, in_len, window, hop, boundary, filters, n_mels, power, out, batch); },
      {in, out},
      [&](cudaStream_t s) {
        return p->mel_device(in, in_len, window, hop, boundary, filters, n_mels, power, out, batch, s);
      });
}

// MFCC and log-mel spectrogram of real rows: mel_exec's rules, plus n_out, the matrix and the log, clamp and bias
// scalars checked before the plan is touched; then, with the clamp, the batch against top_db_rows; the window, filters
// and matrix kept apart from the output.
template <typename T>
int mfcc_exec(void* plan, const T* in, size_t in_len, const T* window, size_t hop, int boundary, int power,
              const T* filters, size_t n_mels, double log_offset, double log_floor, double log_scale, double top_db,
              size_t top_db_rows, const T* dct, size_t n_out, double bias, T* out, size_t batch, bool async,
              void* stream) {
  if (!plan || !in || !window || !filters || !out) {
    fb200::set_last_error("null argument");
    return (int)cudaErrorInvalidValue;
  }
  const bool clamp = std::isfinite(top_db);
  auto* p = static_cast<RealPlan<T>*>(plan);
  if (!check_frames(p, in_len, hop, boundary,
                    power != 1 && power != 2                          ? "power must be 1 or 2"
                    : n_mels == 0                                     ? "n_mels must be at least 1"
                    : n_out == 0                                      ? "n_out must be at least 1"
                    : !dct && n_out != n_mels                         ? "dct NULL (the identity) needs n_out == n_mels"
                    : !std::isfinite(log_offset)                      ? "log_offset must be finite"
                    : !std::isfinite(bias)                            ? "bias must be finite"
                    : !(std::isfinite(log_floor) && log_floor > 0)    ? "log_floor must be finite and positive"
                    : !(std::isfinite(log_scale) && log_scale > 0)    ? "log_scale must be finite and positive"
                    : !(top_db >= 0)                                  ? "top_db must be >= 0 (+inf: no clamp)"
                    : top_db_rows == 0                                ? "top_db_rows must be at least 1"
                    : clamp && batch % top_db_rows != 0               ? "batch must be a multiple of top_db_rows"
                                                                      : nullptr))
    return (int)cudaErrorInvalidValue;
  const size_t n = p->size();
  return run_call(
      "mfcc", async, stream,
      [&] {
        if (batch == 0)
          return (int)p->mfcc_device(in, in_len, window, hop, boundary, power, filters, n_mels, log_offset, log_floor,
                                     log_scale, top_db, top_db_rows, dct, n_out, bias, out, 0, nullptr);
        const size_t in_bytes = batch * in_len * sizeof(T);
        const size_t out_bytes = batch * p->mel_row_bytes(in_len, hop, boundary, n_out);
        if (ranges_meet(in, in_bytes, out, out_bytes) || ranges_meet(window, n * sizeof(T), out, out_bytes) ||
            ranges_meet(filters, n_mels * (n / 2 + 1) * sizeof(T), out, out_bytes) ||
            (dct && ranges_meet(dct, n_mels * n_out * sizeof(T), out, out_bytes))) {
          fb200::set_last_error("input, window, filters or dct and output overlap (mfcc is out of place only)");
          return (int)cudaErrorInvalidValue;
        }
        return kRun;
      },
      {in, window, filters, dct ? (const void*)dct : (const void*)out, out},
      "input, window, filters, dct and output must all be host or all be device memory",
      [&] {
        return p->mfcc_host(in, in_len, window, hop, boundary, power, filters, n_mels, log_offset, log_floor, log_scale,
                            top_db, top_db_rows, dct, n_out, bias, out, batch);
      },
      {in, out},
      [&](cudaStream_t s) {
        return p->mfcc_device(in, in_len, window, hop, boundary, power, filters, n_mels, log_offset, log_floor,
                              log_scale, top_db, top_db_rows, dct, n_out, bias, out, batch, s);
      });
}

// Welch power spectral density of real rows: stft_exec's rules with boundary none, plus detrend, scaling and fs checked
// before the plan is touched.
template <typename T>
int welch_exec(void* plan, const T* in, size_t in_len, const T* window, size_t hop, int detrend, int scaling, double fs,
               T* out, size_t batch, bool async, void* stream) {
  if (!plan || !in || !window || !out) { fb200::set_last_error("null argument"); return (int)cudaErrorInvalidValue; }
  auto* p = static_cast<RealPlan<T>*>(plan);
  if (!check_frames(p, in_len, hop, fb200::real::kStftNone,
                    detrend != 0 && detrend != 1    ? "unknown detrend (FOURIER_B200_DETREND_NONE or _CONSTANT)"
                    : scaling != 0 && scaling != 1  ? "unknown scaling (FOURIER_B200_WELCH_DENSITY or _SPECTRUM)"
                    : !(std::isfinite(fs) && fs > 0) ? "fs must be finite and positive"
                                                     : nullptr))
    return (int)cudaErrorInvalidValue;
  const size_t n = p->size();
  return run_call(
      "welch", async, stream,
      [&] {
        if (batch == 0) return (int)p->welch_device(in, in_len, window, hop, detrend, scaling, fs, out, 0, nullptr);
        const size_t in_bytes = batch * in_len * sizeof(T), out_bytes = batch * (n / 2 + 1) * sizeof(T);
        if (ranges_meet(in, in_bytes, out, out_bytes) || ranges_meet(window, n * sizeof(T), out, out_bytes)) {
          fb200::set_last_error("input or window and output overlap (welch is out of place only)");
          return (int)cudaErrorInvalidValue;
        }
        return kRun;
      },
      {in, window, out}, "input, window and output must all be host or all be device memory",
      [&] { return p->welch_host(in, in_len, window, hop, detrend, scaling, fs, out, batch); },
      {in, out},
      [&](cudaStream_t s) { return p->welch_device(in, in_len, window, hop, detrend, scaling, fs, out, batch, s); });
}

// Discrete cosine transform of real rows: type and norm checked before the plan is touched, even for batch == 0; in == out
// allowed, otherwise disjoint.
template <typename T>
int dct_exec(void* plan, const T* in, T* out, size_t batch, int type, int norm, bool async, void* stream) {
  if (!plan || !in || !out) { fb200::set_last_error("null argument"); return (int)cudaErrorInvalidValue; }
  const char* bad = type != 2 && type != 3   ? "unknown type (the DCT types are 2 and 3)"
                    : norm < 0 || norm > 2 ? "unknown norm (FOURIER_B200_DCT_NORM_BACKWARD, _ORTHO or _FORWARD)"
                                           : nullptr;
  if (bad) { fb200::set_last_error(bad); return (int)cudaErrorInvalidValue; }
  auto* p = static_cast<RealPlan<T>*>(plan);
  return run_call(
      "dct", async, stream,
      [&] {
        if (batch == 0) return (int)p->dct_device(in, out, 0, type, norm, nullptr);
        const size_t bytes = batch * p->size() * sizeof(T);
        if (in != out && ranges_meet(in, bytes, out, bytes)) {
          fb200::set_last_error("input and output overlap (they must be the same buffer or disjoint)");
          return (int)cudaErrorInvalidValue;
        }
        return kRun;
      },
      {in, out}, "input and output must both be host or both be device memory",
      [&] { return p->dct_host(in, out, batch, type, norm); },
      {in, out}, [&](cudaStream_t s) { return p->dct_device(in, out, batch, type, norm, s); });
}

// Analytic signal and envelope of real rows: the arguments and the output kind checked before the plan is touched, even
// for batch == 0; the envelope may run in place (in == out), the analytic signal is out of place, and any other overlap
// is refused.
template <typename T>
int hilbert_exec(void* plan, const T* in, void* out, size_t batch, int output, bool async, void* stream) {
  const char* bad = !plan ? "null argument: plan"
                    : !in ? "null argument: in"
                    : !out ? "null argument: out"
                    : output != fb200::real::kHilbertAnalytic && output != fb200::real::kHilbertEnvelope
                        ? "unknown output (FOURIER_B200_HILBERT_ANALYTIC or _ENVELOPE)"
                        : nullptr;
  if (bad) { fb200::set_last_error(bad); return (int)cudaErrorInvalidValue; }
  auto* p = static_cast<RealPlan<T>*>(plan);
  const bool env = output == fb200::real::kHilbertEnvelope;
  return run_call(
      "hilbert", async, stream,
      [&] {
        if (batch == 0) return (int)p->hilbert_device(in, out, 0, output, nullptr);
        const size_t in_bytes = batch * p->size() * sizeof(T), out_bytes = env ? in_bytes : 2 * in_bytes;
        if (!(env && (const void*)in == out) && ranges_meet(in, in_bytes, out, out_bytes)) {
          fb200::set_last_error(env ? "input and output overlap (the envelope runs in place or on disjoint buffers)"
                                    : "input and output overlap (the analytic signal is out of place only)");
          return (int)cudaErrorInvalidValue;
        }
        return kRun;
      },
      {in, out}, "input and output must both be host or both be device memory",
      [&] { return p->hilbert_host(in, out, batch, output); },
      {in, out}, [&](cudaStream_t s) { return p->hilbert_device(in, out, batch, output, s); });
}

// Type-IV DCT, MDCT and IMDCT of real rows (DESIGN.md §4.20): the arguments that need no plan checked first, even for
// batch == 0, each refusal naming its argument; then an odd plan length.
const char* bad_norm(int norm) {
  return norm < 0 || norm > 2 ? "unknown norm (FOURIER_B200_DCT_NORM_BACKWARD, _ORTHO or _FORWARD)" : nullptr;
}
template <typename T> bool even_plan(const RealPlan<T>* p, const char* what) {
  if (p->size() % 2 == 0) return true;
  fb200::set_last_error(std::string(what) + " needs an even plan length N");
  return false;
}

// dct4: in == out allowed, otherwise disjoint
template <typename T>
int dct4_exec(void* plan, const T* in, T* out, size_t batch, int norm, bool async, void* stream) {
  const char* bad = !plan ? "null argument: plan" : !in ? "null argument: in" : !out ? "null argument: out" : bad_norm(norm);
  if (bad) { fb200::set_last_error(bad); return (int)cudaErrorInvalidValue; }
  auto* p = static_cast<RealPlan<T>*>(plan);
  if (!even_plan(p, "the type-IV DCT")) return (int)cudaErrorInvalidValue;
  return run_call(
      "dct4", async, stream,
      [&] {
        if (batch == 0) return (int)p->dct4_device(in, out, 0, norm, nullptr);
        const size_t bytes = batch * p->size() * sizeof(T);
        if (in != out && ranges_meet(in, bytes, out, bytes)) {
          fb200::set_last_error("input and output overlap (they must be the same buffer or disjoint)");
          return (int)cudaErrorInvalidValue;
        }
        return kRun;
      },
      {in, out}, "input and output must both be host or both be device memory",
      [&] { return p->dct4_host(in, out, batch, norm); },
      {in, out}, [&](cudaStream_t s) { return p->dct4_device(in, out, batch, norm, s); });
}

// mdct: out of place only; the window (2N reals) must not overlap the output either
template <typename T>
int mdct_exec(void* plan, const T* in, size_t in_len, const T* window, int center, int norm, T* out, size_t batch,
              bool async, void* stream) {
  const char* bad = !plan ? "null argument: plan" : !in ? "null argument: in" : !window ? "null argument: window"
                    : !out ? "null argument: out" : in_len == 0 ? "in_len must be at least 1" : bad_norm(norm);
  if (bad) { fb200::set_last_error(bad); return (int)cudaErrorInvalidValue; }
  auto* p = static_cast<RealPlan<T>*>(plan);
  if (!even_plan(p, "the MDCT")) return (int)cudaErrorInvalidValue;
  const size_t n = p->size();
  if (!center && in_len < 2 * n) {
    fb200::set_last_error("in_len must be at least 2N without center");
    return (int)cudaErrorInvalidValue;
  }
  return run_call(
      "mdct", async, stream,
      [&] {
        if (batch == 0) return (int)p->mdct_device(in, in_len, window, center != 0, norm, out, 0, nullptr);
        const size_t in_bytes = batch * in_len * sizeof(T);
        const size_t out_bytes = batch * p->mdct_frames(in_len, center != 0) * n * sizeof(T);
        if (ranges_meet(in, in_bytes, out, out_bytes) || ranges_meet(window, 2 * n * sizeof(T), out, out_bytes)) {
          fb200::set_last_error("input or window and output overlap (the mdct is out of place only)");
          return (int)cudaErrorInvalidValue;
        }
        return kRun;
      },
      {in, window, out}, "input, window and output must all be host or all be device memory",
      [&] { return p->mdct_host(in, in_len, window, center != 0, norm, out, batch); },
      {in, out}, [&](cudaStream_t s) { return p->mdct_device(in, in_len, window, center != 0, norm, out, batch, s); });
}

// imdct: out of place only; the window (2N reals) must not overlap the output either
template <typename T>
int imdct_exec(void* plan, const T* in, size_t frames, const T* window, int center, int norm, T* out, size_t out_len,
               size_t batch, bool async, void* stream) {
  const char* bad = !plan ? "null argument: plan" : !in ? "null argument: in" : !window ? "null argument: window"
                    : !out ? "null argument: out" : frames == 0 ? "frames must be at least 1"
                    : out_len == 0 ? "out_len must be at least 1" : bad_norm(norm);
  if (bad) { fb200::set_last_error(bad); return (int)cudaErrorInvalidValue; }
  auto* p = static_cast<RealPlan<T>*>(plan);
  if (!even_plan(p, "the IMDCT")) return (int)cudaErrorInvalidValue;
  const size_t n = p->size();
  return run_call(
      "imdct", async, stream,
      [&] {
        if (batch == 0) return (int)p->imdct_device(in, frames, window, center != 0, norm, out, out_len, 0, nullptr);
        const size_t in_bytes = batch * frames * n * sizeof(T), out_bytes = batch * out_len * sizeof(T);
        if (ranges_meet(in, in_bytes, out, out_bytes) || ranges_meet(window, 2 * n * sizeof(T), out, out_bytes)) {
          fb200::set_last_error("input or window and output overlap (the imdct is out of place only)");
          return (int)cudaErrorInvalidValue;
        }
        return kRun;
      },
      {in, window, out}, "input, window and output must all be host or all be device memory",
      [&] { return p->imdct_host(in, frames, window, center != 0, norm, out, out_len, batch); },
      {in, out},
      [&](cudaStream_t s) { return p->imdct_device(in, frames, window, center != 0, norm, out, out_len, batch, s); });
}

// Cross-spectral density (coh false) and coherence of real rows: welch_exec's rules for x, the window, hop, detrend
// (and for the csd scaling and fs), plus y and y_rows, checked before the plan is touched; y may overlap x.
template <typename T>
int cross_exec(void* plan, const T* x, const T* y, size_t y_rows, size_t in_len, const T* window, size_t hop,
               int detrend, bool coh, int scaling, double fs, void* out, size_t batch, bool async, void* stream) {
  if (!plan || !x || !y || !window || !out) { fb200::set_last_error("null argument"); return (int)cudaErrorInvalidValue; }
  auto* p = static_cast<RealPlan<T>*>(plan);
  if (!check_frames(p, in_len, hop, fb200::real::kStftNone,
                    y_rows == 0                              ? "y_rows must be at least 1"
                    : detrend != 0 && detrend != 1           ? "unknown detrend (FOURIER_B200_DETREND_NONE or _CONSTANT)"
                    : !coh && scaling != 0 && scaling != 1   ? "unknown scaling (FOURIER_B200_WELCH_DENSITY or _SPECTRUM)"
                    : !coh && !(std::isfinite(fs) && fs > 0) ? "fs must be finite and positive"
                                                             : nullptr))
    return (int)cudaErrorInvalidValue;
  const size_t n = p->size();
  const char* what = coh ? "coherence" : "csd";
  return run_call(
      what, async, stream,
      [&] {
        if (batch == 0)
          return (int)p->cross_device(x, y, y_rows, in_len, window, hop, detrend, coh, scaling, fs, out, 0, nullptr);
        const size_t x_bytes = batch * in_len * sizeof(T), y_bytes = y_rows * in_len * sizeof(T);
        const size_t out_bytes = batch * (n / 2 + 1) * (coh ? sizeof(T) : 2 * sizeof(T));
        if (ranges_meet(x, x_bytes, out, out_bytes) || ranges_meet(y, y_bytes, out, out_bytes) ||
            ranges_meet(window, n * sizeof(T), out, out_bytes)) {
          fb200::set_last_error(coh ? "x, y or window and output overlap (coherence is out of place only)"
                                    : "x, y or window and output overlap (csd is out of place only)");
          return (int)cudaErrorInvalidValue;
        }
        return kRun;
      },
      {x, y, window, out}, "x, y, window and output must all be host or all be device memory",
      [&] { return p->cross_host(x, y, y_rows, in_len, window, hop, detrend, coh, scaling, fs, out, batch); },
      {x, y, out},
      [&](cudaStream_t s) {
        return p->cross_device(x, y, y_rows, in_len, window, hop, detrend, coh, scaling, fs, out, batch, s);
      });
}

template <typename T>
int istft_exec(void* plan, const void* in, size_t frames, const T* window, size_t hop, int center, T* out,
               size_t out_len, size_t batch, bool async, void* stream) {
  if (!plan || !in || !window || !out) { fb200::set_last_error("null argument"); return (int)cudaErrorInvalidValue; }
  const char* bad = hop == 0        ? "hop must be at least 1"
                    : frames == 0   ? "frames must be at least 1"
                    : out_len == 0  ? "out_len must be at least 1"
                                    : nullptr;
  if (bad) { fb200::set_last_error(bad); return (int)cudaErrorInvalidValue; }
  auto* p = static_cast<RealPlan<T>*>(plan);
  using C = typename RealPlan<T>::C;
  const C* spec = static_cast<const C*>(in);
  return run_call(
      "istft", async, stream,
      [&] {
        if (batch == 0) return (int)p->istft_device(spec, frames, window, hop, center != 0, out, out_len, 0, nullptr);
        const size_t in_bytes = batch * p->spec_bytes(frames), out_bytes = batch * out_len * sizeof(T);
        if (ranges_meet(in, in_bytes, out, out_bytes) || ranges_meet(window, p->size() * sizeof(T), out, out_bytes)) {
          fb200::set_last_error("input or window and output overlap (the istft is out of place only)");
          return (int)cudaErrorInvalidValue;
        }
        return kRun;
      },
      {in, window, out}, "input, window and output must all be host or all be device memory",
      [&] { return p->istft_host(spec, frames, window, hop, center != 0, out, out_len, batch); },
      {in, out},
      [&](cudaStream_t s) { return p->istft_device(spec, frames, window, hop, center != 0, out, out_len, batch, s); });
}

}  // namespace

using fourier::c::fourier_fft_double;
using fourier::c::fourier_fft_float;

namespace fourier {
namespace c {
extern "C" {

// ---- the eight reference symbols --------------------------------------------------------------------
fourier_fft_float* fourier_create_float(size_t size) {
  return static_cast<fourier_fft_float*>(create<Plan<float>>(size, true));
}
fourier_fft_double* fourier_create_double(size_t size) {
  return static_cast<fourier_fft_double*>(create<Plan<double>>(size, true));
}
void fourier_destroy_float(fourier_fft_float* plan) {
  try { delete reinterpret_cast<Plan<float>*>(plan); } catch (...) {}
}
void fourier_destroy_double(fourier_fft_double* plan) {
  try { delete reinterpret_cast<Plan<double>*>(plan); } catch (...) {}
}
void fourier_transform_in_place_float(const fourier_fft_float* plan, std::complex<float>* data, int t) {
  (void)fft_exec<float>(plan, data, data, 1, t, false, nullptr);
}
void fourier_transform_in_place_double(const fourier_fft_double* plan, std::complex<double>* data, int t) {
  (void)fft_exec<double>(plan, data, data, 1, t, false, nullptr);
}
void fourier_transform_float(const fourier_fft_float* plan, const std::complex<float>* in,
                             std::complex<float>* out, int t) {
  (void)fft_exec<float>(plan, in, out, 1, t, false, nullptr);
}
void fourier_transform_double(const fourier_fft_double* plan, const std::complex<double>* in,
                              std::complex<double>* out, int t) {
  (void)fft_exec<double>(plan, in, out, 1, t, false, nullptr);
}

}  // extern "C"
}  // namespace c
}  // namespace fourier

extern "C" {

// ---- additive entry points --------------------------------------------------------------------------
int fourier_b200_set_device(int device) {
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || device < 0 || device >= count) {
    fb200::set_last_error("invalid device ordinal");
    return (int)cudaErrorInvalidDevice;
  }
  g_device = device;
  return 0;
}
int fourier_b200_get_device(void) { return resolve_device(); }
int fourier_b200_device_count(void) {
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess) { cudaGetLastError(); return 0; }
  return count;
}

int fourier_b200_transform_batch_float(const fourier_fft_float* plan, const void* in, void* out,
                                       size_t batch, int t) {
  return fft_exec<float>(plan, in, out, batch, t, false, nullptr);
}
int fourier_b200_transform_batch_double(const fourier_fft_double* plan, const void* in, void* out,
                                        size_t batch, int t) {
  return fft_exec<double>(plan, in, out, batch, t, false, nullptr);
}
int fourier_b200_transform_batch_async_float(const fourier_fft_float* plan, const void* in, void* out,
                                             size_t batch, int t, void* stream) {
  return fft_exec<float>(plan, in, out, batch, t, true, stream);
}
int fourier_b200_transform_batch_async_double(const fourier_fft_double* plan, const void* in, void* out,
                                              size_t batch, int t, void* stream) {
  return fft_exec<double>(plan, in, out, batch, t, true, stream);
}

int fourier_b200_plan_info_float(const fourier_fft_float* plan, fourier_b200_plan_info* out) {
  return plan_info<Plan<float>>(plan, out);
}
int fourier_b200_plan_info_double(const fourier_fft_double* plan, fourier_b200_plan_info* out) {
  return plan_info<Plan<double>>(plan, out);
}
const char* fourier_b200_path_name(int path) { return fb200::path_name((fb200::Path)path); }
const char* fourier_b200_plan_kernel_float(const fourier_fft_float* plan) {
  return plan ? reinterpret_cast<const Plan<float>*>(plan)->kernel_name() : "";
}
const char* fourier_b200_plan_kernel_double(const fourier_fft_double* plan) {
  return plan ? reinterpret_cast<const Plan<double>*>(plan)->kernel_name() : "";
}

fourier_fft_float* fourier_b200_create_general_float(size_t size) {
  return static_cast<fourier_fft_float*>(create<Plan<float>>(size, false));
}
fourier_fft_double* fourier_b200_create_general_double(size_t size) {
  return static_cast<fourier_fft_double*>(create<Plan<double>>(size, false));
}

int fourier_b200_fill_input_float(void* dev_out, unsigned long long first, size_t count,
                                  unsigned long long seed, void* stream) {
  return (int)fb200::launch_fill_input<float>((float*)dev_out, first, count, seed, (cudaStream_t)stream);
}
int fourier_b200_fill_input_double(void* dev_out, unsigned long long first, size_t count,
                                   unsigned long long seed, void* stream) {
  return (int)fb200::launch_fill_input<double>((double*)dev_out, first, count, seed, (cudaStream_t)stream);
}

int fourier_b200_transpose_float(const void* in, void* out, size_t batch, size_t rows, size_t cols, void* stream) {
  return (int)fb200::launch_transpose<float>((const float2*)in, (float2*)out, batch, rows, cols, (cudaStream_t)stream);
}
int fourier_b200_transpose_double(const void* in, void* out, size_t batch, size_t rows, size_t cols, void* stream) {
  return (int)fb200::launch_transpose<double>((const double2*)in, (double2*)out, batch, rows, cols, (cudaStream_t)stream);
}
int fourier_b200_pack_float(const void* in, void* out, size_t batch, size_t rows, size_t cols, size_t ld, size_t ibs,
                            size_t obs, int twiddle, unsigned long long row0, unsigned long long col0,
                            unsigned long long n_total, void* stream) {
  return (int)fb200::launch_pack<float>((const float2*)in, (float2*)out, batch, rows, cols, ld, ibs, obs, twiddle, row0,
                                        col0, n_total, (cudaStream_t)stream);
}
int fourier_b200_pack_double(const void* in, void* out, size_t batch, size_t rows, size_t cols, size_t ld, size_t ibs,
                             size_t obs, int twiddle, unsigned long long row0, unsigned long long col0,
                             unsigned long long n_total, void* stream) {
  return (int)fb200::launch_pack<double>((const double2*)in, (double2*)out, batch, rows, cols, ld, ibs, obs, twiddle, row0,
                                         col0, n_total, (cudaStream_t)stream);
}
int fourier_b200_exchange_float(const void* in, void* const* outs, int nranks, int me, size_t rows, size_t cb, size_t ld,
                                size_t out_ld, size_t out_off, int twiddle, unsigned long long row0,
                                unsigned long long n_total, void* stream) {
  return (int)fb200::launch_exchange<float>((const float2*)in, outs, nranks, me, rows, cb, ld, out_ld, out_off, twiddle,
                                            row0, n_total, (cudaStream_t)stream);
}
int fourier_b200_exchange_double(const void* in, void* const* outs, int nranks, int me, size_t rows, size_t cb, size_t ld,
                                 size_t out_ld, size_t out_off, int twiddle, unsigned long long row0,
                                 unsigned long long n_total, void* stream) {
  return (int)fb200::launch_exchange<double>((const double2*)in, outs, nranks, me, rows, cb, ld, out_ld, out_off, twiddle,
                                             row0, n_total, (cudaStream_t)stream);
}
int fourier_b200_fft_rows_exchange_float(const fourier_fft_float* plan, const void* in, size_t rows, int forward,
                                         void* const* outs, int nranks, size_t out_ld, size_t out_off, int twiddle,
                                         unsigned long long row0, unsigned long long n_total, void* stream) {
  return rows_exchange<float>(plan, in, rows, forward, outs, nranks, out_ld, out_off, twiddle, row0, n_total, stream);
}
int fourier_b200_fft_rows_exchange_double(const fourier_fft_double* plan, const void* in, size_t rows, int forward,
                                          void* const* outs, int nranks, size_t out_ld, size_t out_off, int twiddle,
                                          unsigned long long row0, unsigned long long n_total, void* stream) {
  return rows_exchange<double>(plan, in, rows, forward, outs, nranks, out_ld, out_off, twiddle, row0, n_total, stream);
}
int fourier_b200_peer_alloc(size_t bytes, void** dev_ptr, void* handle64) { return (int)fb200::peer_alloc(bytes, dev_ptr, handle64); }
int fourier_b200_peer_open(const void* handle64, void** dev_ptr) { return (int)fb200::peer_open(handle64, dev_ptr); }
int fourier_b200_peer_close(void* dev_ptr) { return (int)fb200::peer_close(dev_ptr); }
int fourier_b200_peer_free(void* dev_ptr) { return (int)fb200::peer_free(dev_ptr); }
int fourier_b200_swap_leading_float(const void* in, void* out, size_t a, size_t b, size_t inner, void* stream) {
  return (int)fb200::launch_swap_leading<float>((const float2*)in, (float2*)out, a, b, inner, (cudaStream_t)stream);
}
int fourier_b200_swap_leading_double(const void* in, void* out, size_t a, size_t b, size_t inner, void* stream) {
  return (int)fb200::launch_swap_leading<double>((const double2*)in, (double2*)out, a, b, inner, (cudaStream_t)stream);
}
int fourier_b200_twiddle_rows_float(void* data, size_t rows, size_t cols, unsigned long long row0,
                                    unsigned long long n_total, int forward, void* stream) {
  return (int)fb200::launch_twiddle_rows<float>((float2*)data, rows, cols, row0, n_total, forward != 0, (cudaStream_t)stream);
}
int fourier_b200_twiddle_rows_double(void* data, size_t rows, size_t cols, unsigned long long row0,
                                     unsigned long long n_total, int forward, void* stream) {
  return (int)fb200::launch_twiddle_rows<double>((double2*)data, rows, cols, row0, n_total, forward != 0, (cudaStream_t)stream);
}

// ---- real-input transforms ------------------------------------------------------------------------------
fourier_b200_rfft_float* fourier_b200_rfft_create_float(size_t n) {
  return static_cast<fourier_b200_rfft_float*>(create<RealPlan<float>>(n, true));
}
fourier_b200_rfft_double* fourier_b200_rfft_create_double(size_t n) {
  return static_cast<fourier_b200_rfft_double*>(create<RealPlan<double>>(n, true));
}
void fourier_b200_rfft_destroy_float(fourier_b200_rfft_float* plan) {
  try { delete reinterpret_cast<RealPlan<float>*>(plan); } catch (...) {}
}
void fourier_b200_rfft_destroy_double(fourier_b200_rfft_double* plan) {
  try { delete reinterpret_cast<RealPlan<double>*>(plan); } catch (...) {}
}
int fourier_b200_rfft_forward_float(fourier_b200_rfft_float* plan, const float* in, void* out, size_t batch, int t) {
  return rfft_exec<float>(plan, true, in, out, batch, t, false, nullptr);
}
int fourier_b200_rfft_forward_double(fourier_b200_rfft_double* plan, const double* in, void* out, size_t batch, int t) {
  return rfft_exec<double>(plan, true, in, out, batch, t, false, nullptr);
}
int fourier_b200_rfft_forward_async_float(fourier_b200_rfft_float* plan, const float* in, void* out, size_t batch, int t,
                                          void* stream) {
  return rfft_exec<float>(plan, true, in, out, batch, t, true, stream);
}
int fourier_b200_rfft_forward_async_double(fourier_b200_rfft_double* plan, const double* in, void* out, size_t batch,
                                           int t, void* stream) {
  return rfft_exec<double>(plan, true, in, out, batch, t, true, stream);
}
int fourier_b200_rfft_inverse_float(fourier_b200_rfft_float* plan, const void* in, float* out, size_t batch, int t) {
  return rfft_exec<float>(plan, false, in, out, batch, t, false, nullptr);
}
int fourier_b200_rfft_inverse_double(fourier_b200_rfft_double* plan, const void* in, double* out, size_t batch, int t) {
  return rfft_exec<double>(plan, false, in, out, batch, t, false, nullptr);
}
int fourier_b200_rfft_inverse_async_float(fourier_b200_rfft_float* plan, const void* in, float* out, size_t batch, int t,
                                          void* stream) {
  return rfft_exec<float>(plan, false, in, out, batch, t, true, stream);
}
int fourier_b200_rfft_inverse_async_double(fourier_b200_rfft_double* plan, const void* in, double* out, size_t batch,
                                           int t, void* stream) {
  return rfft_exec<double>(plan, false, in, out, batch, t, true, stream);
}
int fourier_b200_rfft_info_float(const fourier_b200_rfft_float* plan, fourier_b200_plan_info* out) {
  return plan_info<RealPlan<float>>(plan, out);
}
int fourier_b200_rfft_info_double(const fourier_b200_rfft_double* plan, fourier_b200_plan_info* out) {
  return plan_info<RealPlan<double>>(plan, out);
}
const char* fourier_b200_rfft_kernel_float(const fourier_b200_rfft_float* plan) {
  return plan ? reinterpret_cast<const RealPlan<float>*>(plan)->kernel_name() : "";
}
const char* fourier_b200_rfft_kernel_double(const fourier_b200_rfft_double* plan) {
  return plan ? reinterpret_cast<const RealPlan<double>*>(plan)->kernel_name() : "";
}

int fourier_b200_convolve_real_float(fourier_b200_rfft_float* plan, const float* in, const void* spectrum,
                                     size_t spectrum_rows, float* out, size_t batch) {
  return convolve_exec<float>(plan, in, spectrum, spectrum_rows, out, batch, false, nullptr);
}
int fourier_b200_convolve_real_double(fourier_b200_rfft_double* plan, const double* in, const void* spectrum,
                                      size_t spectrum_rows, double* out, size_t batch) {
  return convolve_exec<double>(plan, in, spectrum, spectrum_rows, out, batch, false, nullptr);
}
int fourier_b200_convolve_real_async_float(fourier_b200_rfft_float* plan, const float* in_dev, const void* spectrum_dev,
                                           size_t spectrum_rows, float* out_dev, size_t batch, void* stream) {
  return convolve_exec<float>(plan, in_dev, spectrum_dev, spectrum_rows, out_dev, batch, true, stream);
}
int fourier_b200_convolve_real_async_double(fourier_b200_rfft_double* plan, const double* in_dev,
                                            const void* spectrum_dev, size_t spectrum_rows, double* out_dev,
                                            size_t batch, void* stream) {
  return convolve_exec<double>(plan, in_dev, spectrum_dev, spectrum_rows, out_dev, batch, true, stream);
}

int fourier_b200_linear_convolve_real_float(fourier_b200_rfft_float* plan, const float* in, size_t in_len,
                                            const void* spectrum, size_t spectrum_rows, size_t taps, int mode,
                                            float* out, size_t batch) {
  return linear_exec<float>(plan, in, in_len, spectrum, spectrum_rows, taps, mode, out, batch, false, nullptr);
}
int fourier_b200_linear_convolve_real_double(fourier_b200_rfft_double* plan, const double* in, size_t in_len,
                                             const void* spectrum, size_t spectrum_rows, size_t taps, int mode,
                                             double* out, size_t batch) {
  return linear_exec<double>(plan, in, in_len, spectrum, spectrum_rows, taps, mode, out, batch, false, nullptr);
}
int fourier_b200_linear_convolve_real_async_float(fourier_b200_rfft_float* plan, const float* in_dev, size_t in_len,
                                                  const void* spectrum_dev, size_t spectrum_rows, size_t taps, int mode,
                                                  float* out_dev, size_t batch, void* stream) {
  return linear_exec<float>(plan, in_dev, in_len, spectrum_dev, spectrum_rows, taps, mode, out_dev, batch, true, stream);
}
int fourier_b200_linear_convolve_real_async_double(fourier_b200_rfft_double* plan, const double* in_dev, size_t in_len,
                                                   const void* spectrum_dev, size_t spectrum_rows, size_t taps,
                                                   int mode, double* out_dev, size_t batch, void* stream) {
  return linear_exec<double>(plan, in_dev, in_len, spectrum_dev, spectrum_rows, taps, mode, out_dev, batch, true,
                             stream);
}

int fourier_b200_stft_float(fourier_b200_rfft_float* plan, const float* in, size_t in_len, const float* window,
                            size_t hop, int boundary, void* out, size_t batch) {
  return stft_exec<float>(plan, in, in_len, window, hop, boundary, out, batch, false, nullptr);
}
int fourier_b200_stft_double(fourier_b200_rfft_double* plan, const double* in, size_t in_len, const double* window,
                             size_t hop, int boundary, void* out, size_t batch) {
  return stft_exec<double>(plan, in, in_len, window, hop, boundary, out, batch, false, nullptr);
}
int fourier_b200_stft_async_float(fourier_b200_rfft_float* plan, const float* in_dev, size_t in_len,
                                  const float* window_dev, size_t hop, int boundary, void* out_dev, size_t batch,
                                  void* stream) {
  return stft_exec<float>(plan, in_dev, in_len, window_dev, hop, boundary, out_dev, batch, true, stream);
}
int fourier_b200_stft_async_double(fourier_b200_rfft_double* plan, const double* in_dev, size_t in_len,
                                   const double* window_dev, size_t hop, int boundary, void* out_dev, size_t batch,
                                   void* stream) {
  return stft_exec<double>(plan, in_dev, in_len, window_dev, hop, boundary, out_dev, batch, true, stream);
}
int fourier_b200_istft_float(fourier_b200_rfft_float* plan, const void* in, size_t frames, const float* window,
                             size_t hop, int center, float* out, size_t out_len, size_t batch) {
  return istft_exec<float>(plan, in, frames, window, hop, center, out, out_len, batch, false, nullptr);
}
int fourier_b200_istft_double(fourier_b200_rfft_double* plan, const void* in, size_t frames, const double* window,
                              size_t hop, int center, double* out, size_t out_len, size_t batch) {
  return istft_exec<double>(plan, in, frames, window, hop, center, out, out_len, batch, false, nullptr);
}
int fourier_b200_istft_async_float(fourier_b200_rfft_float* plan, const void* in_dev, size_t frames,
                                   const float* window_dev, size_t hop, int center, float* out_dev, size_t out_len,
                                   size_t batch, void* stream) {
  return istft_exec<float>(plan, in_dev, frames, window_dev, hop, center, out_dev, out_len, batch, true, stream);
}
int fourier_b200_istft_async_double(fourier_b200_rfft_double* plan, const void* in_dev, size_t frames,
                                    const double* window_dev, size_t hop, int center, double* out_dev, size_t out_len,
                                    size_t batch, void* stream) {
  return istft_exec<double>(plan, in_dev, frames, window_dev, hop, center, out_dev, out_len, batch, true, stream);
}

int fourier_b200_mel_spectrogram_float(fourier_b200_rfft_float* plan, const float* in, size_t in_len,
                                       const float* window, size_t hop, int boundary, int power, const float* filters,
                                       size_t n_mels, float* out, size_t batch) {
  return mel_exec<float>(plan, in, in_len, window, hop, boundary, power, filters, n_mels, out, batch, false, nullptr);
}
int fourier_b200_mel_spectrogram_double(fourier_b200_rfft_double* plan, const double* in, size_t in_len,
                                        const double* window, size_t hop, int boundary, int power,
                                        const double* filters, size_t n_mels, double* out, size_t batch) {
  return mel_exec<double>(plan, in, in_len, window, hop, boundary, power, filters, n_mels, out, batch, false, nullptr);
}
int fourier_b200_mel_spectrogram_async_float(fourier_b200_rfft_float* plan, const float* in_dev, size_t in_len,
                                             const float* window_dev, size_t hop, int boundary, int power,
                                             const float* filters_dev, size_t n_mels, float* out_dev, size_t batch,
                                             void* stream) {
  return mel_exec<float>(plan, in_dev, in_len, window_dev, hop, boundary, power, filters_dev, n_mels, out_dev, batch,
                         true, stream);
}
int fourier_b200_mel_spectrogram_async_double(fourier_b200_rfft_double* plan, const double* in_dev, size_t in_len,
                                              const double* window_dev, size_t hop, int boundary, int power,
                                              const double* filters_dev, size_t n_mels, double* out_dev, size_t batch,
                                              void* stream) {
  return mel_exec<double>(plan, in_dev, in_len, window_dev, hop, boundary, power, filters_dev, n_mels, out_dev, batch,
                          true, stream);
}

int fourier_b200_mfcc_float(fourier_b200_rfft_float* plan, const float* in, size_t in_len, const float* window,
                            size_t hop, int boundary, int power, const float* filters, size_t n_mels, double log_offset,
                            double log_floor, double log_scale, double top_db, size_t top_db_rows, const float* dct,
                            size_t n_out, double bias, float* out, size_t batch) {
  return mfcc_exec<float>(plan, in, in_len, window, hop, boundary, power, filters, n_mels, log_offset, log_floor,
                          log_scale, top_db, top_db_rows, dct, n_out, bias, out, batch, false, nullptr);
}
int fourier_b200_mfcc_double(fourier_b200_rfft_double* plan, const double* in, size_t in_len, const double* window,
                             size_t hop, int boundary, int power, const double* filters, size_t n_mels,
                             double log_offset, double log_floor, double log_scale, double top_db, size_t top_db_rows,
                             const double* dct, size_t n_out, double bias, double* out, size_t batch) {
  return mfcc_exec<double>(plan, in, in_len, window, hop, boundary, power, filters, n_mels, log_offset, log_floor,
                           log_scale, top_db, top_db_rows, dct, n_out, bias, out, batch, false, nullptr);
}
int fourier_b200_mfcc_async_float(fourier_b200_rfft_float* plan, const float* in_dev, size_t in_len,
                                  const float* window_dev, size_t hop, int boundary, int power,
                                  const float* filters_dev, size_t n_mels, double log_offset, double log_floor,
                                  double log_scale, double top_db, size_t top_db_rows, const float* dct_dev,
                                  size_t n_out, double bias, float* out_dev, size_t batch, void* stream) {
  return mfcc_exec<float>(plan, in_dev, in_len, window_dev, hop, boundary, power, filters_dev, n_mels, log_offset,
                          log_floor, log_scale, top_db, top_db_rows, dct_dev, n_out, bias, out_dev, batch, true, stream);
}
int fourier_b200_mfcc_async_double(fourier_b200_rfft_double* plan, const double* in_dev, size_t in_len,
                                   const double* window_dev, size_t hop, int boundary, int power,
                                   const double* filters_dev, size_t n_mels, double log_offset, double log_floor,
                                   double log_scale, double top_db, size_t top_db_rows, const double* dct_dev,
                                   size_t n_out, double bias, double* out_dev, size_t batch, void* stream) {
  return mfcc_exec<double>(plan, in_dev, in_len, window_dev, hop, boundary, power, filters_dev, n_mels, log_offset,
                           log_floor, log_scale, top_db, top_db_rows, dct_dev, n_out, bias, out_dev, batch, true,
                           stream);
}

int fourier_b200_welch_float(fourier_b200_rfft_float* plan, const float* in, size_t in_len, const float* window,
                             size_t hop, int detrend, int scaling, double fs, float* out, size_t batch) {
  return welch_exec<float>(plan, in, in_len, window, hop, detrend, scaling, fs, out, batch, false, nullptr);
}
int fourier_b200_welch_double(fourier_b200_rfft_double* plan, const double* in, size_t in_len, const double* window,
                              size_t hop, int detrend, int scaling, double fs, double* out, size_t batch) {
  return welch_exec<double>(plan, in, in_len, window, hop, detrend, scaling, fs, out, batch, false, nullptr);
}
int fourier_b200_welch_async_float(fourier_b200_rfft_float* plan, const float* in_dev, size_t in_len,
                                   const float* window_dev, size_t hop, int detrend, int scaling, double fs,
                                   float* out_dev, size_t batch, void* stream) {
  return welch_exec<float>(plan, in_dev, in_len, window_dev, hop, detrend, scaling, fs, out_dev, batch, true, stream);
}
int fourier_b200_welch_async_double(fourier_b200_rfft_double* plan, const double* in_dev, size_t in_len,
                                    const double* window_dev, size_t hop, int detrend, int scaling, double fs,
                                    double* out_dev, size_t batch, void* stream) {
  return welch_exec<double>(plan, in_dev, in_len, window_dev, hop, detrend, scaling, fs, out_dev, batch, true, stream);
}

int fourier_b200_dct_float(fourier_b200_rfft_float* plan, const float* in, float* out, size_t batch, int type, int norm) {
  return dct_exec<float>(plan, in, out, batch, type, norm, false, nullptr);
}
int fourier_b200_dct_double(fourier_b200_rfft_double* plan, const double* in, double* out, size_t batch, int type,
                            int norm) {
  return dct_exec<double>(plan, in, out, batch, type, norm, false, nullptr);
}
int fourier_b200_dct_async_float(fourier_b200_rfft_float* plan, const float* in_dev, float* out_dev, size_t batch,
                                 int type, int norm, void* stream) {
  return dct_exec<float>(plan, in_dev, out_dev, batch, type, norm, true, stream);
}
int fourier_b200_dct_async_double(fourier_b200_rfft_double* plan, const double* in_dev, double* out_dev, size_t batch,
                                  int type, int norm, void* stream) {
  return dct_exec<double>(plan, in_dev, out_dev, batch, type, norm, true, stream);
}

int fourier_b200_csd_float(fourier_b200_rfft_float* plan, const float* x, const float* y, size_t y_rows, size_t in_len,
                       const float* window, size_t hop, int detrend, int scaling, double fs, void* out, size_t batch) {
  return cross_exec<float>(plan, x, y, y_rows, in_len, window, hop, detrend, false, scaling, fs, out, batch, false,
                           nullptr);
}
int fourier_b200_csd_async_float(fourier_b200_rfft_float* plan, const float* x_dev, const float* y_dev, size_t y_rows,
                             size_t in_len, const float* window_dev, size_t hop, int detrend, int scaling, double fs,
                             void* out_dev, size_t batch, void* stream) {
  return cross_exec<float>(plan, x_dev, y_dev, y_rows, in_len, window_dev, hop, detrend, false, scaling, fs, out_dev,
                           batch, true, stream);
}
int fourier_b200_coherence_float(fourier_b200_rfft_float* plan, const float* x, const float* y, size_t y_rows,
                             size_t in_len, const float* window, size_t hop, int detrend, float* out, size_t batch) {
  return cross_exec<float>(plan, x, y, y_rows, in_len, window, hop, detrend, true, 0, 1.0, out, batch, false, nullptr);
}
int fourier_b200_coherence_async_float(fourier_b200_rfft_float* plan, const float* x_dev, const float* y_dev,
                                   size_t y_rows, size_t in_len, const float* window_dev, size_t hop, int detrend,
                                   float* out_dev, size_t batch, void* stream) {
  return cross_exec<float>(plan, x_dev, y_dev, y_rows, in_len, window_dev, hop, detrend, true, 0, 1.0, out_dev, batch,
                           true, stream);
}
int fourier_b200_csd_double(fourier_b200_rfft_double* plan, const double* x, const double* y, size_t y_rows, size_t in_len,
                       const double* window, size_t hop, int detrend, int scaling, double fs, void* out, size_t batch) {
  return cross_exec<double>(plan, x, y, y_rows, in_len, window, hop, detrend, false, scaling, fs, out, batch, false,
                           nullptr);
}
int fourier_b200_csd_async_double(fourier_b200_rfft_double* plan, const double* x_dev, const double* y_dev, size_t y_rows,
                             size_t in_len, const double* window_dev, size_t hop, int detrend, int scaling, double fs,
                             void* out_dev, size_t batch, void* stream) {
  return cross_exec<double>(plan, x_dev, y_dev, y_rows, in_len, window_dev, hop, detrend, false, scaling, fs, out_dev,
                           batch, true, stream);
}
int fourier_b200_coherence_double(fourier_b200_rfft_double* plan, const double* x, const double* y, size_t y_rows,
                             size_t in_len, const double* window, size_t hop, int detrend, double* out, size_t batch) {
  return cross_exec<double>(plan, x, y, y_rows, in_len, window, hop, detrend, true, 0, 1.0, out, batch, false, nullptr);
}
int fourier_b200_coherence_async_double(fourier_b200_rfft_double* plan, const double* x_dev, const double* y_dev,
                                   size_t y_rows, size_t in_len, const double* window_dev, size_t hop, int detrend,
                                   double* out_dev, size_t batch, void* stream) {
  return cross_exec<double>(plan, x_dev, y_dev, y_rows, in_len, window_dev, hop, detrend, true, 0, 1.0, out_dev, batch,
                           true, stream);
}

int fourier_b200_hilbert_float(fourier_b200_rfft_float* plan, const float* in, void* out, size_t batch, int output) {
  return hilbert_exec<float>(plan, in, out, batch, output, false, nullptr);
}
int fourier_b200_hilbert_double(fourier_b200_rfft_double* plan, const double* in, void* out, size_t batch, int output) {
  return hilbert_exec<double>(plan, in, out, batch, output, false, nullptr);
}
int fourier_b200_hilbert_async_float(fourier_b200_rfft_float* plan, const float* in_dev, void* out_dev, size_t batch,
                                     int output, void* stream) {
  return hilbert_exec<float>(plan, in_dev, out_dev, batch, output, true, stream);
}
int fourier_b200_hilbert_async_double(fourier_b200_rfft_double* plan, const double* in_dev, void* out_dev, size_t batch,
                                      int output, void* stream) {
  return hilbert_exec<double>(plan, in_dev, out_dev, batch, output, true, stream);
}

int fourier_b200_dct4_float(fourier_b200_rfft_float* plan, const float* in, float* out, size_t batch, int norm) {
  return dct4_exec<float>(plan, in, out, batch, norm, false, nullptr);
}
int fourier_b200_dct4_double(fourier_b200_rfft_double* plan, const double* in, double* out, size_t batch, int norm) {
  return dct4_exec<double>(plan, in, out, batch, norm, false, nullptr);
}
int fourier_b200_dct4_async_float(fourier_b200_rfft_float* plan, const float* in_dev, float* out_dev, size_t batch,
                                  int norm, void* stream) {
  return dct4_exec<float>(plan, in_dev, out_dev, batch, norm, true, stream);
}
int fourier_b200_dct4_async_double(fourier_b200_rfft_double* plan, const double* in_dev, double* out_dev, size_t batch,
                                   int norm, void* stream) {
  return dct4_exec<double>(plan, in_dev, out_dev, batch, norm, true, stream);
}

int fourier_b200_mdct_float(fourier_b200_rfft_float* plan, const float* in, size_t in_len, const float* window,
                            int center, int norm, float* out, size_t batch) {
  return mdct_exec<float>(plan, in, in_len, window, center, norm, out, batch, false, nullptr);
}
int fourier_b200_mdct_double(fourier_b200_rfft_double* plan, const double* in, size_t in_len, const double* window,
                             int center, int norm, double* out, size_t batch) {
  return mdct_exec<double>(plan, in, in_len, window, center, norm, out, batch, false, nullptr);
}
int fourier_b200_mdct_async_float(fourier_b200_rfft_float* plan, const float* in_dev, size_t in_len,
                                  const float* window_dev, int center, int norm, float* out_dev, size_t batch,
                                  void* stream) {
  return mdct_exec<float>(plan, in_dev, in_len, window_dev, center, norm, out_dev, batch, true, stream);
}
int fourier_b200_mdct_async_double(fourier_b200_rfft_double* plan, const double* in_dev, size_t in_len,
                                   const double* window_dev, int center, int norm, double* out_dev, size_t batch,
                                   void* stream) {
  return mdct_exec<double>(plan, in_dev, in_len, window_dev, center, norm, out_dev, batch, true, stream);
}

int fourier_b200_imdct_float(fourier_b200_rfft_float* plan, const float* in, size_t frames, const float* window,
                             int center, int norm, float* out, size_t out_len, size_t batch) {
  return imdct_exec<float>(plan, in, frames, window, center, norm, out, out_len, batch, false, nullptr);
}
int fourier_b200_imdct_double(fourier_b200_rfft_double* plan, const double* in, size_t frames, const double* window,
                              int center, int norm, double* out, size_t out_len, size_t batch) {
  return imdct_exec<double>(plan, in, frames, window, center, norm, out, out_len, batch, false, nullptr);
}
int fourier_b200_imdct_async_float(fourier_b200_rfft_float* plan, const float* in_dev, size_t frames,
                                   const float* window_dev, int center, int norm, float* out_dev, size_t out_len,
                                   size_t batch, void* stream) {
  return imdct_exec<float>(plan, in_dev, frames, window_dev, center, norm, out_dev, out_len, batch, true, stream);
}
int fourier_b200_imdct_async_double(fourier_b200_rfft_double* plan, const double* in_dev, size_t frames,
                                    const double* window_dev, int center, int norm, double* out_dev, size_t out_len,
                                    size_t batch, void* stream) {
  return imdct_exec<double>(plan, in_dev, frames, window_dev, center, norm, out_dev, out_len, batch, true, stream);
}

const char* fourier_b200_last_error(void) { return fb200::last_error(); }
const char* fourier_b200_version(void) { return "fourier-b200 0.1.0 (sm_90a)"; }

}  // extern "C"
