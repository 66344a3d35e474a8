// onchip_configs.cuh -- the size classes of the on-chip kernels (onchip_kernels.cuh) per precision and transform length
// L, in one place for the library (onchip_lookup in onchip.cu) and the CPU emulators (tools/emulate*.cu).
#pragma once

#include <cstddef>

#include "onchip_kernels.cuh"

namespace fb200 {
namespace onchip {

// One size class: L = RA * RB points, E per thread; the fft / real / conv / lconv / stft kernels run WARPS warps per CTA
// and at least MINB CTAs per SM.  BWARPS > 0 marks a class of the fused Bluestein kernel (square tiles only), with
// BWARPS warps per CTA; LOCAL_STASH keeps its even half in a per-thread array instead of shared memory.
template <typename T_, int RA_, int RB_, int E_, int WARPS_, int MINB_, int BWARPS_ = 0, bool LOCAL_STASH_ = false>
struct OnChipClass {
  using T = T_;
  static constexpr int RA = RA_, RB = RB_, E = E_, WARPS = WARPS_, MINB = MINB_, BWARPS = BWARPS_, L = RA * RB;
  static constexpr bool LOCAL_STASH = LOCAL_STASH_, kHasBluestein = BWARPS > 0;
  static_assert(!kHasBluestein || (RA == RB && E == RA), "the fused Bluestein kernel runs square tiles");
  template <bool FWD> using Cfg = OnChipCfg<T, RA, RB, E, WARPS, FWD>;
  using BCfg = OnChipCfg<T, RA, RB, E, BWARPS, true>;   // the fused Bluestein kernel's (kHasBluestein only)
};

// visit_onchip<T>(l, f) calls f with a value of the size class of length l (false when there is none).
// f32 L = 1024: the Bluestein kernel keeps the even half per thread, which allows 16 warps per SM (a shared-memory stash
// allows only 11).
template <class F> bool visit_onchip_f32(size_t l, F&& f) {
  switch (l) {
    case 64: f(OnChipClass<float, 8, 8, 8, 8, 4, 8>{}); return true;
    case 128: f(OnChipClass<float, 8, 16, 16, 8, 4>{}); return true;
    case 256: f(OnChipClass<float, 16, 16, 16, 8, 3, 8>{}); return true;
    case 512: f(OnChipClass<float, 16, 32, 32, 8, 2>{}); return true;
    case 1024: f(OnChipClass<float, 32, 32, 32, 8, 2, 16, true>{}); return true;
    default: return false;
  }
}
template <class F> bool visit_onchip_f64(size_t l, F&& f) {
  switch (l) {
    case 64: f(OnChipClass<double, 8, 8, 8, 8, 3, 8>{}); return true;
    case 128: f(OnChipClass<double, 8, 16, 16, 8, 2>{}); return true;
    case 256: f(OnChipClass<double, 16, 16, 16, 8, 1, 8>{}); return true;
    default: return false;
  }
}
template <typename T, class F> bool visit_onchip(size_t l, F&& f) {
  if constexpr (sizeof(T) == 4) return visit_onchip_f32(l, f);
  else return visit_onchip_f64(l, f);
}

}  // namespace onchip
}  // namespace fb200
