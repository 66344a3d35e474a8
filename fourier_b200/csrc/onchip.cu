// onchip.cu -- plans and launchers for the transforms that fit on chip (onchip_kernels.cuh):
// batched power-of-two FFTs up to 1024 points, the fused Bluestein kernel for N <= 1024 and the fused
// real-input kernels for N = 2L (real.cu drives them).
// Reference counterparts: Autosort for small sizes (autosort/mod.rs:141-166) and
// Bluesteins::transform_in_place / apply (bluesteins.rs:193-259).
#include <algorithm>
#include <cmath>

#include "onchip_configs.cuh"
#include "plan.h"
#include "tables.cuh"  // make_twa

namespace fb200 {

namespace {

template <typename T> struct OnChipOps {
  int ra, rb;
  cudaError_t (*prepare)();
  cudaError_t (*fft)(const cpx<T>*, cpx<T>*, const void* twa, size_t batch, bool fwd, T scale, bool do_scale,
                     int sms, cudaStream_t);
  // Bluestein: nullptr when the size class has no fused kernel
  cudaError_t (*bluestein)(const cpx<T>*, cpx<T>*, const void* twa, const cpx<T>* chirp, const cpx<T>* wm,
                           const cpx<T>* wce, const cpx<T>* wco, size_t n, size_t batch, T scale, int sms,
                           cudaStream_t);
  const RealOnChipOps<T>* real;   // real-input transforms of length 2L on the same tiles
};

// the launchers of one size class K (onchip_configs.cuh)
template <class K>
struct OnChipImpl {
  using T = typename K::T;
  static constexpr int RA = K::RA, RB = K::RB, MINB = K::MINB;
  static constexpr bool kHasBluestein = K::kHasBluestein;
  template <bool FWD> using Cfg = typename K::template Cfg<FWD>;
  using BCfg = typename K::BCfg;
  static constexpr size_t smem_fft = Cfg<true>::EX_BYTES + Cfg<true>::TWA_BYTES;
  static constexpr size_t smem_welch = smem_fft + onchip::WelchBody<Cfg<true>>::ACC_BYTES;
  // The Welch kernel's CTAs per SM: the class's, or fewer where its accumulators leave shared memory for fewer (228 KB
  // per H100 SM, 1 KB of it reserved per CTA).  That is f32 L = 128 only: 3 instead of 4, which also lifts its register
  // cap from 64 to 80, at which it does not spill.
  static constexpr int MINB_WELCH = std::min<int>(MINB, (int)((228u << 10) / (smem_welch + 1024)));
  // The csd and coherence kernels' the same way: csd's accumulators are Welch's size, the coherence's twice that
  // (DESIGN.md §4.17 has the CTAs per SM this gives).
  template <bool COH> using Csd = onchip::CsdBody<Cfg<true>, COH>;
  static constexpr size_t smem_csd(bool coh) { return smem_fft + (coh ? Csd<true>::ACC_BYTES : Csd<false>::ACC_BYTES); }
  static constexpr int minb_csd(bool coh) { return std::min<int>(MINB, (int)((228u << 10) / (smem_csd(coh) + 1024))); }
  static constexpr size_t smem_blue() {
    return BCfg::EX_BYTES + BCfg::TWA_BYTES +
           sizeof(cpx<T>) * (4 * (size_t)BCfg::L + (K::LOCAL_STASH ? 0 : (size_t)K::E * BCfg::THREADS));
  }

  // the fft / real / conv kernels: the exchange and the stage twiddles in shared memory, groups of C transforms
  // grid-stride over at most sms * MINB * 4 CTAs
  template <class Args> static cudaError_t allow_smem(void (*kernel)(Args)) {
    return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_fft);
  }
  template <class Args>
  static cudaError_t launch(void (*kernel)(Args), const Args& a, size_t batch, int sms, cudaStream_t s) {
    const size_t groups = (batch + Cfg<true>::C - 1) / Cfg<true>::C;
    const unsigned grid = (unsigned)std::min<size_t>(groups, (size_t)sms * MINB * 4);
    kernel<<<grid, Cfg<true>::THREADS, smem_fft, s>>>(a);
    return cudaGetLastError();
  }

  static cudaError_t prepare() {
    cudaError_t e;
    if ((e = allow_smem(onchip::onchip_fft_kernel<Cfg<true>, MINB>))) return e;
    if ((e = allow_smem(onchip::onchip_fft_kernel<Cfg<false>, MINB>))) return e;
    if constexpr (kHasBluestein) {
      if ((e = cudaFuncSetAttribute(onchip::bluestein_fused_kernel<BCfg, 1, K::LOCAL_STASH>,
                                    cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_blue()))) return e;
    }
    return cudaSuccess;
  }
  static cudaError_t fft(const cpx<T>* in, cpx<T>* out, const void* twa, size_t batch, bool fwd, T scale,
                         bool do_scale, int sms, cudaStream_t s) {
    if (fwd)
      return launch(onchip::onchip_fft_kernel<Cfg<true>, MINB>,
                    {in, out, (const TwPair<T>*)twa, (long)batch, scale, do_scale}, batch, sms, s);
    return launch(onchip::onchip_fft_kernel<Cfg<false>, MINB>,
                  {in, out, (const TwPair<T>*)twa, (long)batch, scale, do_scale}, batch, sms, s);
  }
  static cudaError_t bluestein(const cpx<T>* in, cpx<T>* out, const void* twa, const cpx<T>* chirp,
                               const cpx<T>* wm, const cpx<T>* wce, const cpx<T>* wco, size_t n, size_t batch,
                               T scale, int sms, cudaStream_t s) {
    if constexpr (kHasBluestein) {
      const size_t groups = (batch + BCfg::C - 1) / BCfg::C;
      const unsigned grid = (unsigned)std::min<size_t>(groups, (size_t)sms * 2);
      typename onchip::BluesteinBody<BCfg>::Args a = {in, out, (const TwPair<T>*)twa, chirp, wm, wce, wco,
                                                      (long)n, (long)batch, scale};
      onchip::bluestein_fused_kernel<BCfg, 1, K::LOCAL_STASH><<<grid, BCfg::THREADS, smem_blue(), s>>>(a);
      return cudaGetLastError();
    } else {
      return cudaErrorNotSupported;
    }
  }
  static cudaError_t real_prepare() {
    cudaError_t e;
    if ((e = allow_smem(onchip::onchip_real_kernel<Cfg<true>, MINB>))) return e;
    if ((e = allow_smem(onchip::onchip_real_kernel<Cfg<false>, MINB>))) return e;
    if ((e = allow_smem(onchip::onchip_conv_kernel<Cfg<true>, MINB>))) return e;
    if ((e = allow_smem(onchip::onchip_lconv_kernel<Cfg<true>, MINB>))) return e;
    if ((e = allow_smem(onchip::onchip_stft_kernel<Cfg<true>, MINB>))) return e;
    if ((e = allow_smem(onchip::onchip_mel_kernel<Cfg<true>, MINB>))) return e;
    if ((e = allow_smem(onchip::onchip_mfcc_kernel<Cfg<true>, MINB, true>))) return e;
    if ((e = allow_smem(onchip::onchip_mfcc_kernel<Cfg<true>, MINB, false>))) return e;
    if ((e = allow_smem(onchip::onchip_dct_kernel<Cfg<true>, MINB, 2>))) return e;
    if ((e = allow_smem(onchip::onchip_dct_kernel<Cfg<true>, MINB, 3>))) return e;
    if ((e = allow_smem(onchip::onchip_hilbert_kernel<Cfg<true>, MINB, false>))) return e;
    if ((e = allow_smem(onchip::onchip_hilbert_kernel<Cfg<true>, MINB, true>))) return e;
    if ((e = allow_smem(onchip::onchip_dct4_kernel<Cfg<true>, MINB>))) return e;
    if ((e = allow_smem(onchip::onchip_mdct_kernel<Cfg<true>, MINB>))) return e;
    if ((e = cudaFuncSetAttribute(onchip::onchip_csd_kernel<Cfg<true>, minb_csd(false), false>,
                                  cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_csd(false)))) return e;
    if ((e = cudaFuncSetAttribute(onchip::onchip_csd_kernel<Cfg<true>, minb_csd(true), true>,
                                  cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_csd(true)))) return e;
    return cudaFuncSetAttribute(onchip::onchip_welch_kernel<Cfg<true>, MINB_WELCH>,
                                cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_welch);
  }
  // the csd (coh false) or coherence items of w over C/2 pair columns, as welch(); row b of m pairs with y row
  // (y_off + b) mod y_rows
  static cudaError_t csd(const T* x, const T* y, size_t y_rows, size_t y_off, const T* win, const T* base, int detrend,
                         bool coh, T* part, void* out, const real::FrameMap& m, const real::WelchItems& w,
                         const void* twa, const cpx<T>* tab, int sms, cudaStream_t s) {
    onchip::CsdArgs<Cfg<true>> a;
    static_cast<typename onchip::RealBody<Cfg<true>>::Args&>(a) = {
        nullptr, nullptr, (const TwPair<T>*)twa, tab, 0, (T)0.5};
    a.x = x;
    a.win = win;
    a.m = m;
    a.part = part;
    a.psd = (T*)out;
    a.base = base;
    a.w = w;
    a.detrend = detrend;
    a.y = y;
    a.y_rows = (long)y_rows;
    a.y_off = (long)y_off;
    a.y_rcp = 1.0 / (double)y_rows;
    if (coh) {
      const unsigned grid = (unsigned)std::min<size_t>((size_t)w.groups, (size_t)sms * minb_csd(true) * 4);
      onchip::onchip_csd_kernel<Cfg<true>, minb_csd(true), true><<<grid, Cfg<true>::THREADS, smem_csd(true), s>>>(a);
    } else {
      const unsigned grid = (unsigned)std::min<size_t>((size_t)w.groups, (size_t)sms * minb_csd(false) * 4);
      onchip::onchip_csd_kernel<Cfg<true>, minb_csd(false), false><<<grid, Cfg<true>::THREADS, smem_csd(false), s>>>(a);
    }
    return cudaGetLastError();
  }
  // the items of w, groups grid-stride over at most sms * MINB_WELCH * 4 CTAs, as launch() does
  static cudaError_t welch(const T* in, const T* win, const T* base, int detrend, T* part, T* out,
                           const real::FrameMap& m, const real::WelchItems& w, const void* twa, const cpx<T>* tab, int sms,
                           cudaStream_t s) {
    typename onchip::WelchBody<Cfg<true>>::Args a;
    static_cast<typename onchip::RealBody<Cfg<true>>::Args&>(a) = {
        nullptr, nullptr, (const TwPair<T>*)twa, tab, 0, (T)0.5};
    a.x = in;
    a.win = win;
    a.m = m;
    a.part = part;
    a.psd = out;
    a.base = base;
    a.w = w;
    a.detrend = detrend;
    const unsigned grid = (unsigned)std::min<size_t>((size_t)w.groups, (size_t)sms * MINB_WELCH * 4);
    onchip::onchip_welch_kernel<Cfg<true>, MINB_WELCH><<<grid, Cfg<true>::THREADS, smem_welch, s>>>(a);
    return cudaGetLastError();
  }
  static cudaError_t dct(const T* in, T* out, int type, const void* twa, const cpx<T>* tab, const cpx<T>* wq,
                         size_t batch, T h, T h0, int sms, cudaStream_t s) {
    typename onchip::Dct2Body<Cfg<true>>::Args a;
    static_cast<typename onchip::RealBody<Cfg<true>>::Args&>(a) = {
        nullptr, nullptr, (const TwPair<T>*)twa, tab, (long)batch, h};
    a.x = in;
    a.y = out;
    a.wq = wq;
    a.h0 = h0;
    if (type == 2) return launch(onchip::onchip_dct_kernel<Cfg<true>, MINB, 2>, a, batch, sms, s);
    return launch(onchip::onchip_dct_kernel<Cfg<true>, MINB, 3>, a, batch, sms, s);
  }
  static cudaError_t hilbert(const T* in, void* out, int output, const void* twa, const cpx<T>* tab, size_t batch, T h,
                             int sms, cudaStream_t s) {
    onchip::HilbertArgs<Cfg<true>> a;
    static_cast<typename onchip::ConvBody<Cfg<true>>::Args&>(a) = {
        (const cpx<T>*)in, nullptr, (const TwPair<T>*)twa, tab, nullptr, 1, 0, (long)batch, h, 1};
    a.y = out;
    if (output == real::kHilbertEnvelope)
      return launch(onchip::onchip_hilbert_kernel<Cfg<true>, MINB, true>, a, batch, sms, s);
    return launch(onchip::onchip_hilbert_kernel<Cfg<true>, MINB, false>, a, batch, sms, s);
  }
  static cudaError_t dct4(const T* in, T* out, const void* twa, const cpx<T>* wq, cpx<T> c, size_t batch, int sms,
                          cudaStream_t s) {
    typename onchip::Dct4Body<Cfg<true>>::Args a;
    static_cast<typename onchip::RealBody<Cfg<true>>::Args&>(a) = {
        nullptr, nullptr, (const TwPair<T>*)twa, nullptr, (long)batch, (T)1};
    a.x = in;
    a.y = out;
    a.wq = wq;
    a.c = c;
    return launch(onchip::onchip_dct4_kernel<Cfg<true>, MINB>, a, batch, sms, s);
  }
  static cudaError_t mdct(const T* in, const T* win, T* out, const real::FrameMap& m, size_t nframes, const void* twa,
                          const cpx<T>* wq, cpx<T> c, int sms, cudaStream_t s) {
    typename onchip::MdctBody<Cfg<true>>::Args a;
    static_cast<typename onchip::RealBody<Cfg<true>>::Args&>(a) = {
        nullptr, nullptr, (const TwPair<T>*)twa, nullptr, (long)nframes, (T)1};
    a.x = in;
    a.y = out;
    a.wq = wq;
    a.c = c;
    a.win = win;
    a.m = m;
    return launch(onchip::onchip_mdct_kernel<Cfg<true>, MINB>, a, nframes, sms, s);
  }
  static cudaError_t mel(const T* in, const T* win, const T* filters, const real::Band* bands, size_t n_mels, int power,
                         T* out, const real::FrameMap& m, size_t nframes, const void* twa, const cpx<T>* tab, int sms,
                         cudaStream_t s) {
    typename onchip::MelBody<Cfg<true>>::Args a;
    static_cast<typename onchip::RealBody<Cfg<true>>::Args&>(a) = {
        nullptr, nullptr, (const TwPair<T>*)twa, tab, (long)nframes, (T)0.5};
    a.x = in;
    a.win = win;
    a.m = m;
    a.mel = out;
    a.filters = filters;
    a.bands = bands;
    a.n_mels = (long)n_mels;
    a.power = power;
    return launch(onchip::onchip_mel_kernel<Cfg<true>, MINB>, a, nframes, sms, s);
  }
  static cudaError_t mfcc(const T* in, const T* win, const T* filters, const real::Band* bands, size_t n_mels,
                          int power, const real::MfccArgs<T>& p, bool max_sweep, T* out, const real::FrameMap& m,
                          size_t nframes, const void* twa, const cpx<T>* tab, int sms, cudaStream_t s) {
    onchip::MfccArgs<Cfg<true>> a;
    static_cast<typename onchip::RealBody<Cfg<true>>::Args&>(a) = {
        nullptr, nullptr, (const TwPair<T>*)twa, tab, (long)nframes, (T)0.5};
    a.x = in;
    a.win = win;
    a.m = m;
    a.mel = out;
    a.filters = filters;
    a.bands = bands;
    a.n_mels = (long)n_mels;
    a.power = power;
    a.p = p;
    if (max_sweep) return launch(onchip::onchip_mfcc_kernel<Cfg<true>, MINB, true>, a, nframes, sms, s);
    return launch(onchip::onchip_mfcc_kernel<Cfg<true>, MINB, false>, a, nframes, sms, s);
  }
  static cudaError_t stft(const T* in, const T* win, void* out, const real::FrameMap& m, size_t nframes,
                          const void* twa, const cpx<T>* tab, int sms, cudaStream_t s) {
    typename onchip::StftBody<Cfg<true>>::Args a;
    static_cast<typename onchip::RealBody<Cfg<true>>::Args&>(a) = {
        nullptr, (cpx<T>*)out, (const TwPair<T>*)twa, tab, (long)nframes, (T)0.5};
    a.x = in;
    a.win = win;
    a.m = m;
    return launch(onchip::onchip_stft_kernel<Cfg<true>, MINB>, a, nframes, sms, s);
  }
  static cudaError_t conv(const void* in, void* out, const void* twa, const cpx<T>* tab, const cpx<T>* spec,
                          size_t rows, size_t row0, size_t per, size_t batch, T h, int sms, cudaStream_t s) {
    return launch(onchip::onchip_conv_kernel<Cfg<true>, MINB>,
                  {(const cpx<T>*)in, (cpx<T>*)out, (const TwPair<T>*)twa, tab, spec, (long)rows, (long)row0, (long)batch, h,
                   (long)per},
                  batch, sms, s);
  }
  static cudaError_t lconv(const T* in, T* out, const real::SegMap& m, size_t nseg, const void* twa, const cpx<T>* tab,
                           const cpx<T>* spec, size_t rows, T h, int sms, cudaStream_t s) {
    typename onchip::LinConvBody<Cfg<true>>::Args a;
    static_cast<typename onchip::ConvBody<Cfg<true>>::Args&>(a) = {
        nullptr, nullptr, (const TwPair<T>*)twa, tab, spec, (long)rows, m.g0, (long)nseg, h, m.per};
    a.x = in;
    a.y = out;
    a.m = m;
    return launch(onchip::onchip_lconv_kernel<Cfg<true>, MINB>, a, nseg, sms, s);
  }
  static cudaError_t real(const void* in, void* out, const void* twa, const cpx<T>* tab, size_t batch, bool fwd, T h,
                          int sms, cudaStream_t s) {
    if (fwd)
      return launch(onchip::onchip_real_kernel<Cfg<true>, MINB>,
                    {(const cpx<T>*)in, (cpx<T>*)out, (const TwPair<T>*)twa, tab, (long)batch, h}, batch, sms, s);
    return launch(onchip::onchip_real_kernel<Cfg<false>, MINB>,
                  {(const cpx<T>*)in, (cpx<T>*)out, (const TwPair<T>*)twa, tab, (long)batch, h}, batch, sms, s);
  }
  static const OnChipOps<T>* ops() {
    static const RealOnChipOps<T> r = {RA, RB, Cfg<true>::C, &real_prepare, &real, &conv, &lconv, &stft, &mel, &mfcc,
                                      &welch, &dct, &csd, &hilbert, &dct4, &mdct};
    static const OnChipOps<T> o = {RA, RB, &prepare, &fft, kHasBluestein ? &bluestein : nullptr, &r};
    return &o;
  }
};

// the size class of length l (onchip_configs.cuh), nullptr when there is none
template <typename T> const OnChipOps<T>* onchip_lookup(size_t l) {
  const OnChipOps<T>* o = nullptr;
  onchip::visit_onchip<T>(l, [&](auto k) { o = OnChipImpl<decltype(k)>::ops(); });
  return o;
}

}  // namespace

template <typename T>
cudaError_t Plan<T>::init_onchip() {
  const OnChipOps<T>* ops = onchip_lookup<T>(n_);
  if (!ops) return cudaErrorNotSupported;
  FB_CHECK(ops->prepare());
  FB_CHECK(upload(tw_a_, twopass::make_twa<T>(ops->ra, ops->rb)));
  fast_ops_ = ops;
  sm_count_ = sm_count(device_);
  return cudaSuccess;
}

template <typename T>
cudaError_t Plan<T>::exec_onchip(const C* in, C* out, size_t batch, int code, cudaStream_t s) {
  const auto* ops = static_cast<const OnChipOps<T>*>(fast_ops_);
  const bool fwd = transform_is_forward(code);
  const bool do_scale = code != kFft && code != kUnscaledIfft;
  FB_CHECK(ops->fft(in, out, tw_a_.data(), batch, fwd, scale_for<T>(code, n_), do_scale, sm_count_, s));
  launches_ += 1;
  return cudaSuccess;
}

// Tables of the fused Bluestein kernel (one set per direction), built from the same chirp and W that
// init_bluestein() computes in double precision.
template <typename T>
cudaError_t Plan<T>::init_bluestein_fused(const std::vector<double>& chirp_re, const std::vector<double>& chirp_im,
                                          const std::vector<double>& w_re, const std::vector<double>& w_im) {
  const size_t l = m_ / 2;
  const OnChipOps<T>* ops = onchip_lookup<T>(l);
  if (!ops || !ops->bluestein) return cudaErrorNotSupported;
  FB_CHECK(ops->prepare());
  FB_CHECK(upload(tw_a_, twopass::make_twa<T>(ops->ra, ops->rb)));
  // layout per direction d (0 forward, 1 inverse): [chirp | wm | wce | wco], L entries each
  std::vector<cpx<T>> tab(2 * 4 * l, mk<T>((T)0, (T)0));
  for (int d = 0; d < 2; ++d) {
    const double sgn = d == 0 ? 1.0 : -1.0;   // the inverse direction conjugates chirp and W
    cpx<T>* t = tab.data() + (size_t)d * 4 * l;
    for (size_t i = 0; i < l; ++i) {
      if (i < n_) t[i] = mk<T>((T)chirp_re[i], (T)(sgn * chirp_im[i]));
      double re, im;
      host_twiddle(i, m_, &re, &im);
      t[l + i] = mk<T>((T)re, (T)im);                                    // w_M^i (same for both directions)
      t[2 * l + i] = mk<T>((T)w_re[2 * i], (T)(-sgn * w_im[2 * i]));          // conj(W_dir[2k])
      t[3 * l + i] = mk<T>((T)w_re[2 * i + 1], (T)(-sgn * w_im[2 * i + 1]));  // conj(W_dir[2k+1])
    }
  }
  FB_CHECK(upload(tbase_, tab));
  fast_ops_ = ops;
  sm_count_ = sm_count(device_);
  return cudaSuccess;
}

template <typename T>
cudaError_t Plan<T>::exec_bluestein_fused(const C* in, C* out, size_t batch, int code, cudaStream_t s) {
  const auto* ops = static_cast<const OnChipOps<T>*>(fast_ops_);
  const bool fwd = transform_is_forward(code);
  const T scale = scale_for<T>(code, n_) / (T)m_;
  const size_t l = m_ / 2;
  const C* t = (const C*)tbase_.data() + (fwd ? 0 : 4 * l);
  FB_CHECK(ops->bluestein(in, out, tw_a_.data(), t, t + l, t + 2 * l, t + 3 * l, n_, batch, scale, sm_count_, s));
  launches_ += 1;
  return cudaSuccess;
}

template <typename T>
const RealOnChipOps<T>* real_onchip_lookup(size_t m) {
  const OnChipOps<T>* ops = onchip_lookup<T>(m);
  return ops ? ops->real : nullptr;
}

template const RealOnChipOps<float>* real_onchip_lookup<float>(size_t);
template const RealOnChipOps<double>* real_onchip_lookup<double>(size_t);
template cudaError_t Plan<float>::init_onchip();
template cudaError_t Plan<double>::init_onchip();
template cudaError_t Plan<float>::exec_onchip(const C*, C*, size_t, int, cudaStream_t);
template cudaError_t Plan<double>::exec_onchip(const C*, C*, size_t, int, cudaStream_t);
template cudaError_t Plan<float>::init_bluestein_fused(const std::vector<double>&, const std::vector<double>&,
                                                       const std::vector<double>&, const std::vector<double>&);
template cudaError_t Plan<double>::init_bluestein_fused(const std::vector<double>&, const std::vector<double>&,
                                                        const std::vector<double>&, const std::vector<double>&);
template cudaError_t Plan<float>::exec_bluestein_fused(const C*, C*, size_t, int, cudaStream_t);
template cudaError_t Plan<double>::exec_bluestein_fused(const C*, C*, size_t, int, cudaStream_t);

}  // namespace fb200
