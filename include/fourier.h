/*
 * fourier.h -- drop-in C / C++ interface of the H100 FFT engine (libfourier.so).
 *
 * This header declares exactly the C ABI that the reference's `fourier-ffi` crate exports
 * (reference: fourier-ffi/include/fourier.h:30-58, implemented by fourier-ffi/src/lib.rs:14-106)
 * plus a C++ convenience wrapper with the reference's names (fourier-ffi/include/fourier.h:64-128).
 * A program compiled against the reference header links and runs unchanged against this library;
 * see INTEGRATION.md.  Additive, non-reference entry points (batches, device pointers, streams)
 * are in fourier_b200.h.
 *
 *   symbol                                   replaces (reference file:line)
 *   fourier_create_float / _double           fourier-ffi/src/lib.rs:14-20, 61-67  -> fourier::create_fft_f32/f64
 *   fourier_destroy_float / _double          fourier-ffi/src/lib.rs:22-29, 69-76
 *   fourier_transform_in_place_float/_double fourier-ffi/src/lib.rs:31-43, 78-90  -> Fft::transform_in_place
 *   fourier_transform_float / _double        fourier-ffi/src/lib.rs:45-59, 92-106 -> Fft::transform
 *
 * Semantics kept from the reference:
 *   - buffers hold exactly size() interleaved (re, im) samples; `transform` needs in != out;
 *   - create returns NULL on failure (size 0 is refused -- the reference never returns for it);
 *   - transform / destroy never report errors: unknown transform codes or NULL plans are a
 *     silent no-op, as with the swallowed panic in fourier-ffi/src/lib.rs:3-12;
 *   - a plan may move between threads but must not be used by two threads at once
 *     (the reference plan is Send, not Sync: autosort/mod.rs:54,151).
 * Buffers may be host memory (staged over PCIe) or device memory on the plan's GPU.
 */
#ifndef FOURIER_H_
#define FOURIER_H_

#ifdef __cplusplus
#include <complex>
#include <cstddef>
#include <memory>
#define FOURIER_B200_CF ::std::complex<float>
#define FOURIER_B200_CD ::std::complex<double>
#define FOURIER_B200_SIZE ::std::size_t
namespace fourier {
namespace c {
extern "C" {
#else
#include <stddef.h>
#define FOURIER_B200_CF float _Complex
#define FOURIER_B200_CD double _Complex
#define FOURIER_B200_SIZE size_t
#endif

/* Transform codes: fourier-algorithms/src/fft.rs:5-16 via fourier-ffi/src/lib.rs:3-12. */
enum {
  FOURIER_TRANSFORM_FFT = 0,              /* forward, unscaled */
  FOURIER_TRANSFORM_IFFT = 1,             /* inverse, scaled by 1/N */
  FOURIER_TRANSFORM_UNSCALED_IFFT = 2,    /* inverse, unscaled */
  FOURIER_TRANSFORM_SQRT_SCALED_FFT = 3,  /* forward, scaled by 1/sqrt(N) */
  FOURIER_TRANSFORM_SQRT_SCALED_IFFT = 4  /* inverse, scaled by 1/sqrt(N) */
};

/* Opaque plans (the reference's Box<Box<dyn Fft<Real = T> + Send>>). */
struct fourier_fft_float;
struct fourier_fft_double;

#define FOURIER_B200_DECLARE(NAME, CPLX)                                                        \
  struct fourier_fft_##NAME *fourier_create_##NAME(FOURIER_B200_SIZE size);                     \
  void fourier_destroy_##NAME(struct fourier_fft_##NAME *plan);                                 \
  void fourier_transform_in_place_##NAME(const struct fourier_fft_##NAME *plan, CPLX *data,     \
                                         int transform);                                        \
  void fourier_transform_##NAME(const struct fourier_fft_##NAME *plan, const CPLX *input,       \
                                CPLX *output, int transform);

FOURIER_B200_DECLARE(float, FOURIER_B200_CF)
FOURIER_B200_DECLARE(double, FOURIER_B200_CD)

#ifdef __cplusplus
} /* extern "C" */
} /* namespace c */

/* C++ surface with the reference's names: fourier::transform, fourier::fft<float|double>. */
enum class transform : int {
  fft = c::FOURIER_TRANSFORM_FFT,
  ifft = c::FOURIER_TRANSFORM_IFFT,
  unscaled_ifft = c::FOURIER_TRANSFORM_UNSCALED_IFFT,
  sqrt_scaled_fft = c::FOURIER_TRANSFORM_SQRT_SCALED_FFT,
  sqrt_scaled_ifft = c::FOURIER_TRANSFORM_SQRT_SCALED_IFFT,
};

namespace detail {
template <typename T> struct abi;
template <> struct abi<float> {
  using plan = c::fourier_fft_float;
  static plan *create(std::size_t n) { return c::fourier_create_float(n); }
  static void destroy(plan *p) { c::fourier_destroy_float(p); }
  static void in_place(const plan *p, std::complex<float> *x, int t) {
    c::fourier_transform_in_place_float(p, x, t);
  }
  static void out_of_place(const plan *p, const std::complex<float> *i, std::complex<float> *o, int t) {
    c::fourier_transform_float(p, i, o, t);
  }
};
template <> struct abi<double> {
  using plan = c::fourier_fft_double;
  static plan *create(std::size_t n) { return c::fourier_create_double(n); }
  static void destroy(plan *p) { c::fourier_destroy_double(p); }
  static void in_place(const plan *p, std::complex<double> *x, int t) {
    c::fourier_transform_in_place_double(p, x, t);
  }
  static void out_of_place(const plan *p, const std::complex<double> *i, std::complex<double> *o, int t) {
    c::fourier_transform_double(p, i, o, t);
  }
};
}  // namespace detail

/* Owning plan handle; move-only like the reference wrapper. */
template <typename T> struct fft {
  explicit fft(std::size_t size) : impl(detail::abi<T>::create(size), &detail::abi<T>::destroy) {}
  fft() = delete;
  fft(const fft &) = delete;
  fft &operator=(const fft &) = delete;
  fft(fft &&) = default;
  fft &operator=(fft &&) = default;
  ~fft() = default;

  void transform_in_place(std::complex<T> *x, transform t) const {
    detail::abi<T>::in_place(impl.get(), x, static_cast<int>(t));
  }
  void transform(const std::complex<T> *in, std::complex<T> *out, ::fourier::transform t) const {
    detail::abi<T>::out_of_place(impl.get(), in, out, static_cast<int>(t));
  }
  /* handle for the fourier_b200.h extension calls */
  const typename detail::abi<T>::plan *get() const { return impl.get(); }

 private:
  std::unique_ptr<typename detail::abi<T>::plan, void (*)(typename detail::abi<T>::plan *)> impl;
};

}  // namespace fourier
#endif /* __cplusplus */

#endif /* FOURIER_H_ */
