// fused_configs.cuh -- the configurations of the persistent two-pass kernel (fused_kernels.cuh) per transform size, in
// one place for the library (fused_lookup in twopass.cu) and the CPU emulator (tools/emulate.cu).
//
// FusedConfig<T, LOG2N>: the configuration of N = 2^LOG2N (HAS = false where there is none).  A configuration with
// pair items (PairCfg) runs its Cfg::Unpaired with FOURIER_B200_PAIR=0.  Cfg is the kernel configuration,
// RING / LAG its default ring and lag.
// Ring (intermediates kept in L2) = 32 MB / transform size, lag = ring / 2: the ring must stay well inside the
// H100's 50 MB L2 next to the prefetched input tiles.  The ring may have any size >= 2.  Measured on one H100 SXM
// (700 W limit, power-capped near 1.3 GHz in that run): N = 2^20 f32 ring 4 against 8 and N = 2^16 f64 ring 32
// against 64 gave +20 % and +13 %.
#pragma once

#include "fused_kernels.cuh"

namespace fb200 {
namespace fused {

template <typename T, int LOG2N> struct FusedConfig { static constexpr bool HAS = false; };

#define FB_FUSED_CONFIG(T_, LOG2N_, ...)                                                                \
  template <> struct FusedConfig<T_, LOG2N_> {                                                          \
    static constexpr bool HAS = true;                                                                   \
    using Cfg = __VA_ARGS__;                                                                            \
    static constexpr int RING = (int)((32l << 20) / (Cfg::N * (long)sizeof(cpx<T_>))), LAG = RING / 2; \
  };

// template arguments: <T, RA, C, G, PAD1, EXB, DIRECT, RB, RA2, RB2, E1, E2, C1, TABG>
// 1024 x 1024: two 256-thread groups, TMA staging, one shared exchange buffer taken under a lock; pair items
// (FOURIER_B200_PAIR=0: one item per group)
FB_FUSED_CONFIG(float, 20, PairCfg<FusedCfg<float, 32, 8, 2, 8, 1>>)
// 512 (32 x 16) x 1024 (32 x 32), 16-column pass-1 tiles: two 256-thread groups; tile tables read from L2
FB_FUSED_CONFIG(float, 19, FusedCfg<float, 32, 8, 2, 0, 1, false, 16, 32, 32, 32, 32, 16, true>)
// 512 x 512 with 32 x 16 register tiles: three 128-thread groups with TMA staging
FB_FUSED_CONFIG(float, 18, FusedCfg<float, 32, 8, 3, 8, 3, false, 16>)
// 256 (16 x 16, 16 per thread) x 512 (32 x 16, 32 per thread): three 128-thread groups
FB_FUSED_CONFIG(float, 17, FusedCfg<float, 16, 8, 3, 8, 3, false, 16, 32, 16, 16, 32>)
// 256 x 256 with 16 x 16 register tiles, four 128-thread groups, 64-byte tile rows as at 2^20
FB_FUSED_CONFIG(float, 16, FusedCfg<float, 16, 8, 4, 8, 4>)
// 128 (16 x 8, 16 per thread) x 256 (16 x 16, 32 per thread): six 64-thread groups
FB_FUSED_CONFIG(float, 15, FusedCfg<float, 16, 8, 6, 8, 6, false, 8, 16, 16, 16, 32>)
// 128 x 128 with 16 x 8 register tiles: eight 64-thread groups
FB_FUSED_CONFIG(float, 14, FusedCfg<float, 16, 8, 8, 8, 8, false, 8>)
// 64 (8 x 8, 8 per thread) x 128 (16 x 8, 16 per thread): eight 64-thread groups
FB_FUSED_CONFIG(float, 13, FusedCfg<float, 8, 8, 8, 8, 8, false, 8, 16, 8, 8, 16>)
// f64 256 x 256: three 128-thread groups with TMA staging
FB_FUSED_CONFIG(double, 16, FusedCfg<double, 16, 8, 3, 4, 3>)
// f64 128 x 128 with 16 x 8 register tiles: four 64-thread groups with TMA staging
FB_FUSED_CONFIG(double, 14, FusedCfg<double, 16, 8, 4, 4, 4, false, 8>)
// f64 64 (8 x 8) x 128 (16 x 8): eight 64-thread groups loading directly
FB_FUSED_CONFIG(double, 13, FusedCfg<double, 8, 8, 8, 4, 8, true, 8, 16, 8, 8, 16>)
// f64 64 x 64 with 8 x 8 register tiles: eight 64-thread groups loading directly
FB_FUSED_CONFIG(double, 12, FusedCfg<double, 8, 8, 8, 4, 8, true>)

#undef FB_FUSED_CONFIG

// for_each_fused_size<T>(f) calls f(std::integral_constant<int, LOG2N>{}) for every N = 2^LOG2N with a configuration
// above, smallest first: the size list of the library's fused_lookup and of the emulator.
template <typename T, class F> void for_each_fused_size(F&& f) {
  static_for<1, 31>([&](auto k) {
    if constexpr (FusedConfig<T, decltype(k)::value>::HAS) f(k);
  });
}

}  // namespace fused
}  // namespace fb200
