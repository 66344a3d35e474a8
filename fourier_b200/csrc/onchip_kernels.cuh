// onchip_kernels.cuh -- transforms that fit on chip: one warp (or a fraction of a warp) owns a whole
// FFT of length L = RA*RB, so the single exchange of the TileFFT stays inside the warp
// (__syncwarp only, no CTA barrier) and every warp of the SM runs independently.
//
//   * onchip_fft_kernel:      batched power-of-two FFT, N = L in {64 .. 1024}: global -> registers ->
//                             one warp-private shared-memory exchange -> registers -> global.
//   * onchip_real_kernel:     real-input transforms of length 2L (forward and inverse) on the same tiles.
//   * onchip_conv_kernel:     y = irfft(rfft(x) . H) of real rows of length 2L, both transforms in one kernel.
//   * onchip_lconv_kernel:    linear convolution of real rows of any length by overlap-save on the same phases.
//   * onchip_stft_kernel:     windowed frames of real rows of any length through the forward real-input phases.
//   * onchip_mel_kernel:      the stft's frames to mel energies: power and filter bank on chip.
//   * onchip_mfcc_kernel:     the mel energies on to their logs, a clamp and a projection (MFCC, log-mel) on chip.
//   * onchip_dct_kernel:      discrete cosine transforms (types II and III) of real rows of length 2L.
//   * onchip_hilbert_kernel:  the analytic signal (Hilbert transform) or its envelope of real rows of length 2L.
//     (these nine run the phases of FftBody / RealBody / ConvBody / LinConvBody / StftBody / MelBody / MfccBody /
//     Dct2Body / Dct3Body / HilbertBody through run_onchip_groups, tilefft.cuh)
//   * onchip_welch_kernel:    detrended, windowed frames to Welch's averaged power spectrum, summed on chip
//                             (WelchBody through run_welch_groups, below).
//   * onchip_csd_kernel:      Welch's frames of two signals in pairs to their cross-spectral density or coherence
//                             (CsdBody through run_welch_groups, below).
//   * bluestein_fused_kernel: the whole chirp-z transform of the reference (bluesteins.rs:218-259) for
//                             N <= L, M = 2L, in one kernel and without touching HBM in between.
//
// Bluestein on M = 2L with half of the input zero (N <= L always holds: M = next_pow2(2N-1) >= 2N):
//   FFT_M(pad(a))[2k]   = FFT_L(a)[k],         FFT_M(pad(a))[2k+1] = FFT_L(a * w_M^n)[k]
//   IFFT_M(Z)[n], n < L = IFFT_L(Z_even)[n] + w_M^{-n} * IFFT_L(Z_odd)[n]
// so the two padded length-M transforms of the reference become four length-L transforms (10% fewer
// butterflies, and the 1024-point register tile of the two-pass kernel is reused as is).  The inverse
// transforms are computed as conj(FFT(conj(.))) with the conjugations folded into the pointwise
// multiplies, so only the forward tile is instantiated.
#pragma once

#include "real_kernels.cuh"
#include "tilefft.cuh"

namespace fb200 {
namespace onchip {

// Exchange layout for "u fast" scatter AND gather (lanes run along the FFT in both stages).
// (when several FFTs share a half-warp their blocks must not start on the same bank: +8 if the block
// size is a multiple of 16 words)
template <int RA, int RB>
using WarpLayout = ExLayout<RA + 1, 1, RB * (RA + 1) + ((RB * (RA + 1)) % 16 == 0 ? 8 : 0)>;

template <typename T, int RA, int RB, int E, int WARPS, bool FWD>
struct OnChipCfg {
  using Tile = TileFFT<T, RA, RB, E, (WARPS * 32) / ((RA * RB) / E), FWD>;
  using Lay = WarpLayout<RA, RB>;
  static constexpr int L = RA * RB, TP = L / E, THREADS = WARPS * 32, C = THREADS / TP;
  static_assert(TP <= 32, "one FFT must fit inside a warp");
  // rounded up: the twiddle pairs behind it are read with 128-bit (f32) / 2 x 128-bit (f64) loads
  static constexpr size_t EX_BYTES = ((sizeof(cpx<T>) * (size_t)Tile::template smem_elems<Lay>() + 127) / 128) * 128;
  static constexpr size_t TWA_BYTES = sizeof(TwPair<T>) * (RA / 2) * RB;
};

// ---- plain batched FFT ----------------------------------------------------------------------------------------
template <class Cfg> struct FftBody {
  using Tile = typename Cfg::Tile;
  using V = typename Tile::V;
  using T = decltype(V::x);
  struct Args { const V* in; V* out; const TwPair<T>* twa; long batch; T scale; int do_scale; };

  // group `grp` = C consecutive transforms; transforms beyond the batch are clamped on load and
  // masked on store, so every lane keeps executing the warp-level synchronisation.
  static FB_HD void phase1(Tile& f, const Args& a, long grp, int t, V* smem, const TwPair<T>* twa) {
    const int col = Tile::template col_of<true>(t), u = Tile::template u_of<true>(t);
    long b = grp * Cfg::C + col;
    if (b >= a.batch) b = a.batch - 1;
    const V* p = a.in + b * Cfg::L + u;
#pragma unroll
    for (int q = 0; q < Tile::NA; ++q)
#pragma unroll
      for (int i = 0; i < Tile::RA; ++i) f.v[q * Tile::RA + i] = p[Tile::TP * q + Tile::RB * i];
    f.template stage_a<true>(t, twa);
    f.template scatter<true, typename Cfg::Lay>(t, smem);
  }
  static FB_HD void phase2(Tile& f, const Args& a, long grp, int t, const V* smem) {
    const int col = Tile::template col_of<true>(t), u = Tile::template u_of<true>(t);
    f.template gather<true, typename Cfg::Lay>(t, smem);
    f.stage_b();
    const long b = grp * Cfg::C + col;
    if (b >= a.batch) return;
    V* p = a.out + b * Cfg::L;
    static_for<0, Tile::NB>([&](auto Cc) FB_LAMBDA {
      constexpr int c = decltype(Cc)::value;
      static_for<0, Tile::RB>([&](auto Rr) FB_LAMBDA {
        constexpr int r = decltype(Rr)::value;
        V val = f.v[c * Tile::RB + bitrev(r, ilog2(Tile::RB))];
        if (a.do_scale) val = cscale(val, a.scale);
        p[(u + Tile::TP * c) + Tile::RA * r] = val;
      });
    });
  }

  // phase protocol (tilefft.cuh)
  static constexpr int kPhases = 2;
  template <int P> static FB_HD void phase(Tile& f, const Args& a, long grp, int t, V* smem, const TwPair<T>* twa) {
    if constexpr (P == 0) phase1(f, a, grp, t, smem, twa);
    else phase2(f, a, grp, t, smem);
  }
};

template <class Cfg, int MINB>
__global__ void __launch_bounds__(Cfg::THREADS, MINB) onchip_fft_kernel(const typename FftBody<Cfg>::Args a) {
  run_onchip_groups<Cfg, FftBody<Cfg>>(a);
}

// ---- fused real-input transforms, N = 2L (real_kernels.cuh) ----------------------------------------------------
// Forward: the 2L reals of a row are loaded as L complex values with FftBody's loads and run through the tile; the
// spectrum Z is parked in natural order in the FFT's own block of the exchange buffer, and each lane untangles the
// pairs (k, L-k), k = u + TP*j, into the L+1 bins of the row (lane u = 0 also the self-paired k = L/2).
// Inverse: the lane that owns stage-A position n forms Z'[n] from X[n] and X[L-n] in registers; the tile's own store
// writes z' as interleaved reals.  One launch, one trip through HBM.
template <class Cfg> struct RealBody {
  using Tile = typename Cfg::Tile;
  using V = typename Tile::V;
  using T = decltype(V::x);
  using Fft = FftBody<Cfg>;
  static constexpr int L = Cfg::L, TP = Tile::TP, RA = Tile::RA, RB = Tile::RB, E = Tile::E;
  struct Args { const V* in; V* out; const TwPair<T>* twa; const V* tab; long batch; T h; };

  // the FFT `col` of the CTA keeps Z in natural order at smem[col * SC + k], k < L (inside its exchange block)
  static FB_HD int park(int t) { return Tile::template col_of<true>(t) * Cfg::Lay::SC; }

  static FB_HD void fwd_phase1(Tile& f, const Args& a, long grp, int t, V* smem, const TwPair<T>* twa) {
    const typename Fft::Args fa = {a.in, nullptr, twa, a.batch, (T)1, 0};
    Fft::phase1(f, fa, grp, t, smem, twa);
  }
  static FB_HD void fwd_gather(Tile& f, int t, const V* smem) {
    f.template gather<true, typename Cfg::Lay>(t, smem);
    f.stage_b();
  }
  static FB_HD void fwd_park(const Tile& f, int t, V* smem) {
    const int u = Tile::template u_of<true>(t);
    V* z = smem + park(t);
    static_for<0, Tile::NB>([&](auto Cc) FB_LAMBDA {
      constexpr int c = decltype(Cc)::value;
      static_for<0, RB>([&](auto Rr) FB_LAMBDA {
        constexpr int r = decltype(Rr)::value;
        z[(u + TP * c) + RA * r] = f.v[c * RB + bitrev(r, ilog2(RB))];
      });
    });
  }
  static FB_HD void fwd_store(const Args& a, long grp, int t, const V* smem) {
    const int u = Tile::template u_of<true>(t);
    const long b = grp * Cfg::C + Tile::template col_of<true>(t);
    if (b >= a.batch) return;
    const V* z = smem + park(t);
    V* x = a.out + b * (L + 1);
#pragma unroll
    for (int j = 0; j < E / 2; ++j) real::untangle(z, x, (long)L, (long)(u + TP * j), a.tab, a.h);
    if (u == 0) real::untangle(z, x, (long)L, (long)(L / 2), a.tab, a.h);
  }

  static FB_HD void inv_phase1(Tile& f, const Args& a, long grp, int t, V* smem, const TwPair<T>* twa) {
    const int u = Tile::template u_of<true>(t);
    long b = grp * Cfg::C + Tile::template col_of<true>(t);
    if (b >= a.batch) b = a.batch - 1;
    const V* x = a.in + b * (L + 1);
#pragma unroll
    for (int q = 0; q < Tile::NA; ++q)
#pragma unroll
      for (int i = 0; i < RA; ++i) f.v[q * RA + i] = real::tangle_one(x, (long)L, (long)(u + TP * q + RB * i), a.tab, a.h);
    f.template stage_a<true>(t, twa);
    f.template scatter<true, typename Cfg::Lay>(t, smem);
  }
  static FB_HD void inv_phase2(Tile& f, const Args& a, long grp, int t, const V* smem) {
    const typename Fft::Args fa = {nullptr, a.out, nullptr, a.batch, (T)1, 0};
    Fft::phase2(f, fa, grp, t, smem);
  }

  // phase protocol (tilefft.cuh): forward load + stage A, stage B, park, untangle; inverse tangle + stage A, stage B
  static constexpr int kPhases = Tile::FWD ? 4 : 2;
  template <int P> static FB_HD void phase(Tile& f, const Args& a, long grp, int t, V* smem, const TwPair<T>* twa) {
    if constexpr (Tile::FWD) {
      if constexpr (P == 0) fwd_phase1(f, a, grp, t, smem, twa);
      else if constexpr (P == 1) fwd_gather(f, t, smem);
      else if constexpr (P == 2) fwd_park(f, t, smem);
      else fwd_store(a, grp, t, smem);
    } else {
      if constexpr (P == 0) inv_phase1(f, a, grp, t, smem, twa);
      else inv_phase2(f, a, grp, t, smem);
    }
  }
};

template <class Cfg, int MINB>
__global__ void __launch_bounds__(Cfg::THREADS, MINB) onchip_real_kernel(const typename RealBody<Cfg>::Args a) {
  run_onchip_groups<Cfg, RealBody<Cfg>>(a);
}

// ---- fused convolution of real rows, y = irfft(rfft(x) . H), N = 2L (real_kernels.cuh, DESIGN.md §4.11) ----------
// The forward phase is RealBody's: Z parked in natural order in the FFT's own exchange block.  Each lane then runs
// real::conv_pair on the pairs it owns (k = u + TP*j, lane u = 0 also k = L/2), in place on the park.  The inverse
// FFT of Z' runs on the same forward tile as conj(FFT(conj Z')), as bluestein_fused_kernel does: the stage-A reads
// conjugate, and so does the store.  Row b uses spectrum row ((row0 + b) / per) mod rows.
template <class Cfg> struct ConvBody {
  using Tile = typename Cfg::Tile;   // FWD = true
  using V = typename Tile::V;
  using T = decltype(V::x);
  using Fft = FftBody<Cfg>;
  using Real = RealBody<Cfg>;
  static constexpr int L = Cfg::L, TP = Tile::TP, RA = Tile::RA, RB = Tile::RB, E = Tile::E;
  // per: rows of the batch per spectrum row step (the segments of one row, LinConvBody); 1 for circular convolution
  struct Args { const V* in; V* out; const TwPair<T>* twa; const V* tab; const V* spec; long rows, row0, batch; T h;
                long per = 1; };

  static FB_HD void fwd_phase1(Tile& f, const Args& a, long grp, int t, V* smem, const TwPair<T>* twa) {
    const typename Fft::Args fa = {a.in, nullptr, twa, a.batch, (T)1, 0};
    Fft::phase1(f, fa, grp, t, smem, twa);
  }
  // untangle . H . tangle of the lane's pairs, written back into the park
  static FB_HD void pairs(const Args& a, long grp, int t, V* smem) {
    const int u = Tile::template u_of<true>(t);
    const long b = grp * Cfg::C + Tile::template col_of<true>(t);
    if (b >= a.batch) return;
    V* z = smem + Real::park(t);
    const V* hs = a.spec + (((a.row0 + b) / a.per) % a.rows) * (L + 1);
#pragma unroll 4
    for (int j = 0; j < E / 2; ++j) real::conv_pair(z, hs, (long)L, (long)(u + TP * j), a.tab, a.h);
    if (u == 0) real::conv_pair(z, hs, (long)L, (long)(L / 2), a.tab, a.h);
  }
  // conj Z' from the park in stage-A input order, stage A; the scatter (which overwrites the park) comes after a
  // __syncwarp
  static FB_HD void inv_stage_a(Tile& f, int t, const V* smem, const TwPair<T>* twa) {
    const int u = Tile::template u_of<true>(t);
    const V* z = smem + Real::park(t);
#pragma unroll
    for (int q = 0; q < Tile::NA; ++q)
#pragma unroll
      for (int i = 0; i < RA; ++i) f.v[q * RA + i] = cconj(z[u + TP * q + RB * i]);
    f.template stage_a<true>(t, twa);
  }
  static FB_HD void inv_scatter(const Tile& f, int t, V* smem) { f.template scatter<true, typename Cfg::Lay>(t, smem); }
  static FB_HD void inv_store(Tile& f, const Args& a, long grp, int t, const V* smem) {
    const int u = Tile::template u_of<true>(t);
    f.template gather<true, typename Cfg::Lay>(t, smem);
    f.stage_b();
    const long b = grp * Cfg::C + Tile::template col_of<true>(t);
    if (b >= a.batch) return;
    V* p = a.out + b * L;
    static_for<0, Tile::NB>([&](auto Cc) FB_LAMBDA {
      constexpr int c = decltype(Cc)::value;
      static_for<0, RB>([&](auto Rr) FB_LAMBDA {
        constexpr int r = decltype(Rr)::value;
        p[(u + TP * c) + RA * r] = cconj(f.v[c * RB + bitrev(r, ilog2(RB))]);
      });
    });
  }

  // phase protocol (tilefft.cuh): RealBody's forward up to the park, the pairs, then the inverse on the forward tile
  static constexpr int kPhases = 7;
  template <int P> static FB_HD void phase(Tile& f, const Args& a, long grp, int t, V* smem, const TwPair<T>* twa) {
    if constexpr (P == 0) fwd_phase1(f, a, grp, t, smem, twa);
    else if constexpr (P == 1) Real::fwd_gather(f, t, smem);
    else if constexpr (P == 2) Real::fwd_park(f, t, smem);
    else if constexpr (P == 3) pairs(a, grp, t, smem);
    else if constexpr (P == 4) inv_stage_a(f, t, smem, twa);
    else if constexpr (P == 5) inv_scatter(f, t, smem);
    else inv_store(f, a, grp, t, smem);
  }
};

template <class Cfg, int MINB>
__global__ void __launch_bounds__(Cfg::THREADS, MINB) onchip_conv_kernel(const typename ConvBody<Cfg>::Args a) {
  run_onchip_groups<Cfg, ConvBody<Cfg>>(a);
}

// ---- fused linear convolution of real rows by overlap-save, N = 2L (real::SegMap, DESIGN.md §4.12) ---------------
// ConvBody's phases 1-5 as they are, on groups of C consecutive segments instead of rows.
//   * load (phase 0): each lane reads its tile values' reals as scalars, issuing no read outside the row's [lo, hi)
//     (zeros there), pairs them into complex values, runs stage A and scatters;
//   * store (phases 6-8): RealBody's gather and park put the inverse's output in natural order into the FFT's park,
//     and the TP lanes of the FFT store only the segment's kept outputs [lo, hi) from it, consecutive lanes writing
//     consecutive samples, conjugating on the way out as ConvBody's store does.
// Masking the store per tile register instead, or unrolling the store loop 1, 4 or 8 deep, makes ptxas spill a few
// bytes at the f32 L = 128 and L = 1024 register caps; unrolled 2 deep no instance spills.
// Segment q of the launch uses spectrum row ((g0 + q) / per) mod rows (ConvBody::pairs with row0 = g0).
template <class Cfg> struct LinConvBody {
  using Conv = ConvBody<Cfg>;
  using Real = RealBody<Cfg>;
  using Tile = typename Cfg::Tile;   // FWD = true
  using V = typename Tile::V;
  using T = decltype(V::x);
  static constexpr int L = Cfg::L, TP = Tile::TP, RA = Tile::RA, RB = Tile::RB;
  // Conv::Args with in = out = nullptr, row0 = m.g0, per = m.per, batch = segments of the launch
  struct Args : Conv::Args { const T* x; T* y; real::SegMap m; };

  static FB_HD void load(Tile& f, const Args& a, long grp, int t, V* smem, const TwPair<T>* twa) {
    const int u = Tile::template u_of<true>(t);
    long q = grp * Cfg::C + Tile::template col_of<true>(t);
    if (q >= a.batch) q = a.batch - 1;
    const real::SegMap::Window w = a.m.in_window(q);
    const T* src = a.x + w.base;
    const unsigned n = w.hi - w.lo;
    const long g = a.m.g0 + q;
#pragma unroll
    for (int qa = 0; qa < Tile::NA; ++qa)
#pragma unroll
      for (int i = 0; i < RA; ++i) {
        // d = p - lo: one unsigned compare against hi - lo; a signed offset, so that the constant part folds into the
        // load's immediate
        const int d = 2 * (u + TP * qa + RB * i) - w.lo;
        f.v[qa * RA + i] = mk<T>((unsigned)d < n ? real::lin_ld(src + d, g) : (T)0,
                                 (unsigned)(d + 1) < n ? real::lin_ld(src + (d + 1), g) : (T)0);
      }
    f.template stage_a<true>(t, twa);
    f.template scatter<true, typename Cfg::Lay>(t, smem);
  }
  // the park holds Z'' = FFT(conj Z') in natural order; the output is conj Z'' as interleaved reals
  static FB_HD void store(const Args& a, long grp, int t, const V* smem) {
    const int u = Tile::template u_of<true>(t);
    const long q = grp * Cfg::C + Tile::template col_of<true>(t);
    if (q >= a.batch) return;
    const real::SegMap::Window w = a.m.out_window(q);
    T* dst = a.y + w.base;
    const long g = a.m.g0 + q;
    const T* z = reinterpret_cast<const T*>(smem + Real::park(t));
#pragma unroll 2
    for (int p = w.lo + u; p < w.hi; p += TP) real::lin_st(dst + (p - w.lo), (p & 1) ? -z[p] : z[p], g);
  }

  // phase protocol (tilefft.cuh): load + stage A + scatter; ConvBody's phases 1-5; gather + stage B, park, store
  static constexpr int kPhases = 9;
  template <int P> static FB_HD void phase(Tile& f, const Args& a, long grp, int t, V* smem, const TwPair<T>* twa) {
    if constexpr (P == 0) load(f, a, grp, t, smem, twa);
    else if constexpr (P <= 5) Conv::template phase<P>(f, a, grp, t, smem, twa);
    else if constexpr (P == 6) Real::fwd_gather(f, t, smem);
    else if constexpr (P == 7) Real::fwd_park(f, t, smem);
    else store(a, grp, t, smem);
  }
};

template <class Cfg, int MINB>
__global__ void __launch_bounds__(Cfg::THREADS, MINB) onchip_lconv_kernel(const typename LinConvBody<Cfg>::Args a) {
  run_onchip_groups<Cfg, LinConvBody<Cfg>>(a);
}

// ---- fused short-time Fourier transform of real rows, N = 2L (real::FrameMap, DESIGN.md §4.13) -------------------
// RealBody's forward on groups of C consecutive frames instead of rows, with its own load:
//   * load (phase 0): the TP lanes of an FFT read the frame's N reals as scalars, consecutive lanes taking consecutive
//     samples, multiply them by the window w[p] and write them into the FFT's park.  A frame inside the row reads
//     row[t0 + p] unmasked; only a frame that reaches past either end maps each sample through FrameMap::Edge (zero or
//     mirrored), so no read leaves [0, L);
//   * phases 1-2: the frame as L complex values from the park in stage-A input order, stage A; the scatter (which
//     overwrites the park) after a __syncwarp;
//   * phases 3-5: RealBody's gather + stage B, park and untangle store, frame q of the launch writing spectrum row q of
//     `out` (frames are spectrum rows, frame-major).
// Loading the tile's registers straight from the row, as LinConvBody does, needs the window's N reals beside the
// frame's: ptxas then spilled 650-700 bytes at the f32 L = 512 and 1024 register caps.  Staged through the park, no
// instance spills.
template <class Cfg> struct StftBody {
  using Real = RealBody<Cfg>;
  using Tile = typename Cfg::Tile;   // FWD = true
  using V = typename Tile::V;
  using T = decltype(V::x);
  static constexpr int L = Cfg::L, TP = Tile::TP, RA = Tile::RA, RB = Tile::RB;
  // Real::Args with in = nullptr, out = the spectrum of frame g0, batch = frames of the launch
  struct Args : Real::Args { const T* x; const T* win; real::FrameMap m; };

  static FB_HD void load(const Args& a, long grp, int t, V* smem) {
    const int u = Tile::template u_of<true>(t);
    long q = grp * Cfg::C + Tile::template col_of<true>(t);
    if (q >= a.batch) q = a.batch - 1;
    const long g = a.m.g0 + q, b = a.m.row_of(g), t0 = a.m.start(g, b);
    const T* row = a.x + (b - a.m.r0) * a.m.in_ld;
    T* z = reinterpret_cast<T*>(smem + Real::park(t));
    if (t0 >= 0 && t0 + 2 * L <= a.m.len) {
      const T* src = row + t0;
#pragma unroll 2
      for (int p = u; p < 2 * L; p += TP) z[p] = real::lin_ld(src + p, g) * a.win[p];
    } else {
      // 32-bit offsets from an anchor sample c of the row (see FrameMap::edge)
      const real::FrameMap::Edge e = a.m.edge(t0);
      const T* src = row + e.c;
#pragma unroll 2
      for (int p = u; p < 2 * L; p += TP) {
        const int d = e.map(e.d0 + p);
        z[p] = e.in(d) ? real::lin_ld(src + d, g) * a.win[p] : (T)0;
      }
    }
  }
  static FB_HD void load_stage_a(Tile& f, int t, const V* smem, const TwPair<T>* twa) {
    const int u = Tile::template u_of<true>(t);
    const V* z = smem + Real::park(t);
#pragma unroll
    for (int q = 0; q < Tile::NA; ++q)
#pragma unroll
      for (int i = 0; i < RA; ++i) f.v[q * RA + i] = z[u + TP * q + RB * i];
    f.template stage_a<true>(t, twa);
  }

  // phase protocol (tilefft.cuh): load into the park; stage A; scatter; RealBody's gather + stage B, park, store
  static constexpr int kPhases = 6;
  template <int P> static FB_HD void phase(Tile& f, const Args& a, long grp, int t, V* smem, const TwPair<T>* twa) {
    if constexpr (P == 0) load(a, grp, t, smem);
    else if constexpr (P == 1) load_stage_a(f, t, smem, twa);
    else if constexpr (P == 2) f.template scatter<true, typename Cfg::Lay>(t, smem);
    else Real::template phase<P - 2>(f, a, grp, t, smem, twa);
  }
};

template <class Cfg, int MINB>
__global__ void __launch_bounds__(Cfg::THREADS, MINB) onchip_stft_kernel(const typename StftBody<Cfg>::Args a) {
  run_onchip_groups<Cfg, StftBody<Cfg>>(a);
}

// ---- fused mel spectrogram of real rows, N = 2L (real::band_scan / mel_dot, DESIGN.md §4.14) ---------------------
// StftBody's phases 0-4 as they are (the windowed frame through stage A, the scatter, RealBody's gather + stage B and
// park), then:
//   * powers (phase 5): each lane untangles the pairs it owns, k = u + TP*j (lane u = 0 also k = L/2), and keeps
//     |X[k]|^p and |X[L-k]|^p in its own tile registers;
//   * park powers (phase 6): the L+1 powers go into the FFT's park as reals (it holds 2L; no lane reads Z any more);
//   * mels (phase 7): lane u of the FFT sums mels m = u, u + TP, ... over their bands of the parked powers and stores
//     them to row q of `mel`, consecutive lanes writing consecutive mels.
// Only the mel energies reach HBM: n_mels reals per frame instead of N/2+1 complex bins.
template <class Cfg> struct MelBody {
  using Stft = StftBody<Cfg>;
  using Real = RealBody<Cfg>;
  using Tile = typename Cfg::Tile;   // FWD = true
  using V = typename Tile::V;
  using T = decltype(V::x);
  static constexpr int L = Cfg::L, TP = Tile::TP, E = Tile::E;
  // Stft::Args with out = nullptr; frame q of the launch writes mel[q * n_mels ..]
  struct Args : Stft::Args { T* mel; const T* filters; const real::Band* bands; long n_mels; int power; };

  static FB_HD void powers(Tile& f, const Args& a, int t, const V* smem) {
    const int u = Tile::template u_of<true>(t);
    const V* z = smem + Real::park(t);
#pragma unroll
    for (int j = 0; j < E / 2; ++j) f.v[j] = real::power_pair(z, L, u + TP * j, a.tab, a.h, a.power);
    if (u == 0) f.v[E / 2] = real::power_pair(z, L, L / 2, a.tab, a.h, a.power);
  }
  static FB_HD void park_powers(const Tile& f, int t, V* smem) {
    const int u = Tile::template u_of<true>(t);
    T* pw = reinterpret_cast<T*>(smem + Real::park(t));
#pragma unroll
    for (int j = 0; j < E / 2; ++j) {
      pw[u + TP * j] = f.v[j].x;
      pw[L - (u + TP * j)] = f.v[j].y;
    }
    if (u == 0) pw[L / 2] = f.v[E / 2].x;
  }
  static FB_HD void mels(const Args& a, long grp, int t, const V* smem) {
    const int u = Tile::template u_of<true>(t);
    const long q = grp * Cfg::C + Tile::template col_of<true>(t);
    if (q >= a.batch) return;
    const T* pw = reinterpret_cast<const T*>(smem + Real::park(t));
    T* y = a.mel + q * a.n_mels;
    const long g = a.m.g0 + q;
    // The empty asm makes these three pointers opaque here, so the lane's first weight, band and power addresses are
    // formed in this phase: hoisted out of the group loop they stayed live through stage A, and ptxas spilled 24 bytes
    // at the f32 L = 128 register cap.
    const T* filters = a.filters;
    const real::Band* bands = a.bands;
#ifdef __CUDA_ARCH__
    asm volatile("" : "+l"(filters), "+l"(bands), "+l"(pw));
#endif
    for (long m = u; m < a.n_mels; m += TP)
      real::lin_st(y + m, real::mel_dot(filters, bands, (long)(L + 1), m, [&](long k) { return pw[k]; }), g);
  }

  // phase protocol (tilefft.cuh): StftBody's load, stage A, scatter, gather + stage B and park; powers, park powers, mels
  static constexpr int kPhases = 8;
  template <int P> static FB_HD void phase(Tile& f, const Args& a, long grp, int t, V* smem, const TwPair<T>* twa) {
    if constexpr (P <= 4) Stft::template phase<P>(f, a, grp, t, smem, twa);
    else if constexpr (P == 5) powers(f, a, t, smem);
    else if constexpr (P == 6) park_powers(f, t, smem);
    else mels(a, grp, t, smem);
  }
};

template <class Cfg, int MINB>
__global__ void __launch_bounds__(Cfg::THREADS, MINB) onchip_mel_kernel(const typename MelBody<Cfg>::Args a) {
  run_onchip_groups<Cfg, MelBody<Cfg>>(a);
}

// ---- fused MFCC and log-mel spectrogram of real rows, N = 2L (real::log_mel / mfcc_dot, DESIGN.md §4.18) -----------
// MelBody's phases 0-6 as they are (the frame through the FFT, the untangle and the L+1 powers parked as reals), then:
//   * log-mels (phase 7): lane u of the FFT forms mels m = u, u + TP, ... with real::mel_dot and their logs.  The output
//     sweep parks them in the park's free L-1 reals behind the powers (n_mels <= L-1; no lane reads those in this phase).
//     The max sweep (MAX) parks instead the key of each lane's largest log-mel, at real L+1+u;
//   * project (phase 8): lane u computes outputs j = u, u + TP, ... < n_out from the parked log-mels, clamped to its
//     row's group threshold, reading dct[m][j] (consecutive lanes on consecutive addresses) and storing out[q][j].
//     The max sweep's phase 8 instead: lane 0 of the FFT folds the largest of the TP keys into the group slot, one fold
//     per frame (a fold per lane made the max sweep four times slower than the output sweep at f32 N = 512).
// MelBody::Args with mel = the output (n_out reals per frame, unused by the max sweep), for both sweeps
template <class Cfg> struct MfccArgs : MelBody<Cfg>::Args { real::MfccArgs<typename MelBody<Cfg>::T> p; };
template <class Cfg, bool MAX> struct MfccBody {
  using Mel = MelBody<Cfg>;
  using Real = RealBody<Cfg>;
  using Tile = typename Cfg::Tile;   // FWD = true
  using V = typename Tile::V;
  using T = decltype(V::x);
  static constexpr int L = Cfg::L, TP = Tile::TP;
  using Args = MfccArgs<Cfg>;

  static FB_HD void log_mels(const Args& a, long grp, int t, V* smem) {
    const int u = Tile::template u_of<true>(t);
    const long q = grp * Cfg::C + Tile::template col_of<true>(t);
    if (q >= a.batch) return;
    T* pw = reinterpret_cast<T*>(smem + Real::park(t));
    // opaque as in MelBody::mels: formed here, not hoisted through the FFT phases
    const T* filters = a.filters;
    const real::Band* bands = a.bands;
#ifdef __CUDA_ARCH__
    asm volatile("" : "+l"(filters), "+l"(bands), "+l"(pw));
#endif
    real::MaxKey<T> hi = 0;
    for (long m = u; m < a.n_mels; m += TP) {
      const T v = real::log_mel(real::mel_dot(filters, bands, (long)(L + 1), m, [&](long k) { return pw[k]; }), a.p);
      if constexpr (MAX) {
        const real::MaxKey<T> k = real::max_key(v);
        hi = k > hi ? k : hi;
      } else {
        pw[L + 1 + m] = v;
      }
    }
    if constexpr (MAX) memcpy(pw + L + 1 + u, &hi, sizeof hi);
  }
  static FB_HD void fold(const Args& a, long grp, int t, const V* smem) {
    const long q = grp * Cfg::C + Tile::template col_of<true>(t);
    if (q >= a.batch || Tile::template u_of<true>(t) != 0) return;
    const T* keys = reinterpret_cast<const T*>(smem + Real::park(t)) + (L + 1);
#ifdef __CUDA_ARCH__
    asm volatile("" : "+l"(keys));
#endif
    real::MaxKey<T> hi = 0;
    for (int v = 0; v < TP; ++v) {
      real::MaxKey<T> k;
      memcpy(&k, keys + v, sizeof k);
      hi = k > hi ? k : hi;
    }
    real::max_fold(a.p.slots + real::clamp_group(a.p, a.m.row_of(a.m.g0 + q)), hi);
  }
  static FB_HD void project(const Args& a, long grp, int t, const V* smem) {
    const int u = Tile::template u_of<true>(t);
    const long q = grp * Cfg::C + Tile::template col_of<true>(t);
    if (q >= a.batch) return;
    const long g = a.m.g0 + q;
    const T* lm = reinterpret_cast<const T*>(smem + Real::park(t)) + (L + 1);
#ifdef __CUDA_ARCH__
    asm volatile("" : "+l"(lm));
#endif
    const T theta = real::clamp_threshold(a.p, a.m.row_of(g));
    T* y = a.mel + q * a.p.n_out;
    for (long j = u; j < a.p.n_out; j += TP)
      real::lin_st(y + j, real::mfcc_dot(a.p, a.n_mels, j, [&](long m) { return real::clamp_db(lm[m], theta); }), g);
  }

  // phase protocol (tilefft.cuh): MelBody's load, stage A, scatter, gather + stage B, park, powers and park powers;
  // log-mels; project (output sweep) or fold (max sweep)
  static constexpr int kPhases = 9;
  template <int P> static FB_HD void phase(Tile& f, const Args& a, long grp, int t, V* smem, const TwPair<T>* twa) {
    if constexpr (P <= 6) Mel::template phase<P>(f, a, grp, t, smem, twa);
    else if constexpr (P == 7) log_mels(a, grp, t, smem);
    else if constexpr (MAX) fold(a, grp, t, smem);
    else project(a, grp, t, smem);
  }
};

template <class Cfg, int MINB, bool MAX>
__global__ void __launch_bounds__(Cfg::THREADS, MINB) onchip_mfcc_kernel(const typename MfccBody<Cfg, MAX>::Args a) {
  run_onchip_groups<Cfg, MfccBody<Cfg, MAX>>(a);
}

// ---- fused Welch power spectral density of real rows, N = 2L (real::WelchItems, DESIGN.md §4.15) -----------------
// Groups are the items of real::WelchItems, run in rounds of C frames, frame f of an item in column f mod C.  Per frame:
//   * load (phase 0): the TP lanes of an FFT read the frame's N raw samples as StftBody's load does (a frame always lies
//     inside its row, L >= N), park them and put each lane's sum of its own samples, in ascending p, in `sums`;
//   * detrend (phase 1): each lane forms the frame mean from the TP lane sums in lane order (0 with detrend none) and
//     rewrites its own parked samples as (x - mu) w[p], so the mean is taken off before the window;
//   * phases 2-5: StftBody's stage A, scatter, gather + stage B and park;
//   * accumulate (phase 6): each lane forms |X[k]|^2 and |X[L-k]|^2 of the pairs it owns (real::power_pair, lane u = 0
//     also k = L/2) and adds them to its column's row of L+1 accumulators in shared memory (stores them in round 0).
// After the last round a CTA barrier, then the flush: thread o of the CTA sums bin k of an item over the item's columns
// in ascending order and writes the item's partial, or, when a row is one item, the row's output through welch_out.
// The lane sums go through shared memory rather than warp shuffles so that the CPU emulator runs these phases as they
// are.  Shared memory behind the exchange and the stage twiddles: C rows of L+1 accumulators, then one lane sum per
// thread.
template <class Cfg> struct WelchBody {
  using Stft = StftBody<Cfg>;
  using Real = RealBody<Cfg>;
  using Tile = typename Cfg::Tile;   // FWD = true
  using V = typename Tile::V;
  using T = decltype(V::x);
  static constexpr int L = Cfg::L, TP = Tile::TP, E = Tile::E, C = Cfg::C, THREADS = Cfg::THREADS, BINS = L + 1;
  static constexpr size_t ACC_BYTES = sizeof(T) * ((size_t)C * BINS + THREADS);
  // Stft::Args with out = nullptr (m: the frames of the launch's rows, rows in_ld apart from x); part: a partial of
  // BINS reals per item of the launch, psd: BINS reals per row, base: s / F (welch_base) in device memory
  struct Args : Stft::Args { T* part; T* psd; const T* base; real::WelchItems w; int detrend; };

  // The empty asm makes a 64-bit value (the group, the round, a pointer) opaque where a phase uses it, so that what the
  // phase derives from it (the item, row and frame of real::WelchItems::slot, addresses) is not hoisted out of the round
  // loop and kept live through the FFT phases: that spilled 16-84 bytes at the register caps.
  template <typename U> static FB_HD void opaque(U& v) {
    static_assert(sizeof(U) == 8, "64-bit values only");
#ifdef __CUDA_ARCH__
    asm volatile("" : "+l"(v));
#endif
    (void)v;
  }
  static FB_HD bool slot(const Args& a, long g, long r, int t, long& i, long& b, long& f) {
    opaque(g);
    return a.w.slot(g, Tile::template col_of<true>(t), r, i, b, f);
  }

  static FB_HD void load(const Args& a, long g, long r, int t, V* smem, T* acc) {
    const int u = Tile::template u_of<true>(t);
    long i, b, f;
    slot(a, g, r, t, i, b, f);
    const long fg = b * a.w.frames + f;
    const T* src = a.x + b * a.m.in_ld + f * a.m.hop;
    load_frame(src, fg, u, t, smem, acc);
  }
  // the frame of N raw samples from src into the park of thread t (lane u), and its lane sum behind the C rows of
  // accumulators; fg: the frame of the launch, for the access log
  static FB_HD void load_frame(const T* src, long fg, int u, int t, V* smem, T* acc) {
    T* z = reinterpret_cast<T*>(smem + Real::park(t));
    opaque(z);
    T s = 0;
#pragma unroll 2
    for (int p = u; p < 2 * L; p += TP) {
      const T x = real::lin_ld(src + p, fg);
      z[p] = x;
      s += x;
    }
    acc[C * BINS + t] = s;
  }
  static FB_HD void detrend(const Args& a, int t, V* smem, const T* acc) {
    const int u = Tile::template u_of<true>(t), col = Tile::template col_of<true>(t);
    T mu = 0;
    if (a.detrend == real::kDetrendConstant) {
      const T* sums = acc + C * BINS + col * TP;
      T s = 0;
      for (int v = 0; v < TP; ++v) s += sums[v];
      mu = s / (T)(2 * L);
    }
    T* z = reinterpret_cast<T*>(smem + Real::park(t));
    const T* win = a.win;
    opaque(z);
    opaque(win);
#pragma unroll 2
    for (int p = u; p < 2 * L; p += TP) z[p] = (z[p] - mu) * win[p];
  }
  static FB_HD void accumulate(const Args& a, long g, long r, int t, const V* smem, T* acc) {
    const int u = Tile::template u_of<true>(t), col = Tile::template col_of<true>(t);
    long i, b, f;
    if (!slot(a, g, r, t, i, b, f)) return;
    const V* z = smem + Real::park(t);
    const V* tab = a.tab;
    T* y = acc + col * BINS;
    opaque(z);
    opaque(tab);
    opaque(y);
#pragma unroll 4
    for (int j = 0; j < E / 2; ++j) {
      const int k = u + TP * j;
      const V p = real::power_pair(z, L, k, tab, a.h, 2);
      y[k] = r == 0 ? p.x : y[k] + p.x;
      y[L - k] = r == 0 ? p.y : y[L - k] + p.y;
    }
    if (u == 0) {
      const V p = real::power_pair(z, L, L / 2, tab, a.h, 2);
      y[L / 2] = r == 0 ? p.x : y[L / 2] + p.x;
    }
  }
  // the item sums of group g, after a CTA barrier; thread t takes outputs t, t + THREADS, ...
  static FB_HD void flush(const Args& a, long g, int t, const T* acc) {
    const int outs = (int)a.w.per_group * BINS;
    for (int o = t; o < outs; o += THREADS) {
      const int q = o / BINS, k = o - q * BINS;
      const long i = g * a.w.per_group + q;
      if (i >= a.w.total()) return;
      const long cnt = a.w.count(i), used = cnt < C ? cnt : C;
      const T* y = acc + q * a.w.block * BINS + k;
      T s = 0;
      for (long c = 0; c < used; ++c) s += y[c * BINS];
      if (a.w.items == 1) real::lin_st(a.psd + i * BINS + k, real::welch_out(s, *a.base, 2L * L, (long)k), i);
      else real::lin_st(a.part + i * BINS + k, s, i);
    }
  }

  // phase protocol of run_welch_groups: load, detrend, StftBody's stage A, scatter, gather + stage B, park; accumulate
  static constexpr int kPhases = 7;
  template <int P>
  static FB_HD void phase(Tile& f, const Args& a, long g, long r, int t, V* smem, T* acc, const TwPair<T>* twa) {
    if constexpr (P == 0) load(a, g, r, t, smem, acc);
    else if constexpr (P == 1) detrend(a, t, smem, acc);
    else if constexpr (P <= 5) Stft::template phase<P - 1>(f, a, 0, t, smem, twa);
    else accumulate(a, g, r, t, smem, acc);
  }
  // the barrier after phase P: the threads of one FFT share a warp
  static constexpr bool pair_barrier(int) { return false; }
};

// ---- fused cross-spectral density and coherence of real rows, N = 2L (DESIGN.md §4.17) ----------------------------
// WelchBody's rounds on frame pairs: pair column c of the tile holds the x frame in FFT column 2c and the y frame in
// column 2c+1, so a round runs C/2 frame pairs and the items are real::WelchItems over C/2 pair columns.  Per frame pair:
//   * load and detrend (phases 0-1): WelchBody's, each column from its own row (x row b, y row (y_off + b) mod y_rows);
//   * phases 2-5: StftBody's stage A, scatter, gather + stage B and park, per column as in Welch;
//   * cross (phase 6): the 2 TP lanes of a pair split its bin pairs (k = u + TP j, j even in the x column, odd in the
//     y column; lane u = 0 of the x column also k = L/2), untangle X and Y of each from both parks (real::spec_pair)
//     and add real::cross_terms to the pair column's PLANES planes of L+1 accumulators (stores them in round 0).
// Phase 6 reads the partner column's park: with TP <= 16 both columns sit in one warp and __syncwarp orders it; at
// TP = 32 (f32 L = 1024) they are two warps, and a barrier over the pair's 64 threads follows the park (phase 5) and
// the cross phase (before the next round's load overwrites the parks).  The flush sums each plane of an item over its
// pair columns in ascending order into the item's partial, or, when a row is one item, writes the row's output.
// Shared memory behind the exchange and the stage twiddles: C/2 pair columns of PLANES (L+1) accumulators, then one lane
// sum per thread (where WelchBody's load and detrend keep it).
// WelchBody::Args (x, part, psd, base, w over C/2 pair columns, detrend) plus the y rows: row b of the launch pairs
// with y row (y_off + b) mod y_rows, y_rcp = 1 / y_rows; psd: the csd's N/2+1 complex values per row (cpx<T>), or the
// coherence's N/2+1 reals
template <class Cfg> struct CsdArgs : WelchBody<Cfg>::Args {
  const typename WelchBody<Cfg>::T* y;
  long y_rows, y_off;
  double y_rcp;
};
template <class Cfg, bool COH> struct CsdBody {
  using Welch = WelchBody<Cfg>;
  using Stft = StftBody<Cfg>;
  using Real = RealBody<Cfg>;
  using Tile = typename Cfg::Tile;   // FWD = true
  using V = typename Tile::V;
  using T = decltype(V::x);
  static constexpr int L = Cfg::L, TP = Tile::TP, E = Tile::E, C = Cfg::C, THREADS = Cfg::THREADS, BINS = L + 1;
  static constexpr int PLANES = COH ? real::kCoherencePlanes : real::kCsdPlanes, PAIRS = C / 2;
  static constexpr size_t ACC_BYTES = sizeof(T) * ((size_t)PAIRS * PLANES * BINS + THREADS);
  static_assert(C % 2 == 0 && E % 4 == 0 && (2 * TP <= 32 || TP == 32), "a frame pair is one warp or two");
  using Args = CsdArgs<Cfg>;

  template <typename U> static FB_HD void opaque(U& v) { Welch::opaque(v); }
  // Welch's load and detrend find the lane sums behind C (L+1) reals
  static FB_HD T* sums_base(T* acc) { return acc + ((size_t)PAIRS * PLANES * BINS - (size_t)C * BINS); }
  static FB_HD bool slot(const Args& a, long g, long r, int t, long& i, long& b, long& f) {
    Welch::opaque(g);
    return a.w.slot(g, Tile::template col_of<true>(t) >> 1, r, i, b, f);
  }
  static FB_HD void load(const Args& a, long g, long r, int t, V* smem, T* acc) {
    const int u = Tile::template u_of<true>(t);
    long i, b, f;
    slot(a, g, r, t, i, b, f);
    const T* row = a.x + b * a.m.in_ld;
    if (Tile::template col_of<true>(t) & 1) {
      const long yb = a.y_off + b;
      row = a.y + (yb - real::div_rcp(yb, a.y_rows, a.y_rcp) * a.y_rows) * a.m.in_ld;
    }
    Welch::load_frame(row + f * a.m.hop, b * a.w.frames + f, u, t, smem, sums_base(acc));
  }
  static FB_HD void cross(const Args& a, long g, long r, int t, const V* smem, T* acc) {
    const int u = Tile::template u_of<true>(t), col = Tile::template col_of<true>(t), side = col & 1;
    long i, b, f;
    if (!slot(a, g, r, t, i, b, f)) return;
    const V* zx = smem + (col - side) * Cfg::Lay::SC;
    const V* zy = zx + Cfg::Lay::SC;
    const V* tab = a.tab;
    T* y = acc + (col >> 1) * PLANES * BINS;
    Welch::opaque(zx);
    Welch::opaque(zy);
    Welch::opaque(tab);
    Welch::opaque(y);
    auto add = [&](int k, V xv, V yv) FB_LAMBDA {
      T d[real::kCoherencePlanes];
      real::cross_terms(xv, yv, d);
#pragma unroll
      for (int q = 0; q < PLANES; ++q) y[q * BINS + k] = r == 0 ? d[q] : y[q * BINS + k] + d[q];
    };
#pragma unroll 2
    for (int jj = 0; jj < E / 4; ++jj) {
      const int k = u + TP * (2 * jj + side);
      V xk, xm, yk, ym;
      real::spec_pair(zx, L, k, tab, a.h, xk, xm);
      real::spec_pair(zy, L, k, tab, a.h, yk, ym);
      add(k, xk, yk);
      add(L - k, xm, ym);
    }
    if (u == 0 && side == 0) {
      V xk, xm, yk, ym;
      real::spec_pair(zx, L, L / 2, tab, a.h, xk, xm);
      real::spec_pair(zy, L, L / 2, tab, a.h, yk, ym);
      add(L / 2, xk, yk);
    }
  }
  // the item sums of group g, after a CTA barrier; thread t takes outputs t, t + THREADS, ...
  static FB_HD void flush(const Args& a, long g, int t, const T* acc) {
    const int outs = (int)a.w.per_group * BINS;
    for (int o = t; o < outs; o += THREADS) {
      const int q = o / BINS, k = o - q * BINS;
      const long i = g * a.w.per_group + q;
      if (i >= a.w.total()) return;
      const long cnt = a.w.count(i), used = cnt < PAIRS ? cnt : PAIRS;
      const T* y = acc + q * a.w.block * PLANES * BINS + k;
      T s[PLANES];
#pragma unroll
      for (int j = 0; j < PLANES; ++j) s[j] = 0;
      for (long c = 0; c < used; ++c)
#pragma unroll
        for (int j = 0; j < PLANES; ++j) s[j] += y[(c * PLANES + j) * BINS];
      if (a.w.items > 1) {
#pragma unroll
        for (int j = 0; j < PLANES; ++j) real::lin_st(a.part + (i * PLANES + j) * BINS + k, s[j], i);
      } else if constexpr (COH) {
        real::lin_st(a.psd + i * BINS + k, real::coherence_out(s[0], s[1], s[2], s[3]), i);
      } else {
        real::spec_st(reinterpret_cast<V*>(a.psd) + i * BINS + k, real::csd_out(s[0], s[1], *a.base, 2L * L, (long)k));
      }
    }
  }

  // phase protocol of run_welch_groups: WelchBody's load and detrend, StftBody's stage A, scatter, gather + stage B,
  // park; cross
  static constexpr int kPhases = 7;
  template <int P>
  static FB_HD void phase(Tile& f, const Args& a, long g, long r, int t, V* smem, T* acc, const TwPair<T>* twa) {
    if constexpr (P == 0) load(a, g, r, t, smem, acc);
    else if constexpr (P == 1) Welch::detrend(a, t, smem, sums_base(acc));
    else if constexpr (P <= 5) Stft::template phase<P - 1>(f, a, 0, t, smem, twa);
    else cross(a, g, r, t, smem, acc);
  }
  // the barrier after phase P over a frame pair in two warps (see above); __syncwarp otherwise
  static constexpr bool pair_barrier(int p) { return TP == 32 && (p == 5 || p == 6); }
};

// The device driver of WelchBody and CsdBody: run_onchip_groups' set-up, then per group its rounds, each phase followed
// by __syncwarp (or, where Body::pair_barrier asks, a barrier over the 64 threads of a frame pair), and the flush
// between two CTA barriers (the accumulators of every column are complete before it, and it has read them before the
// next group's round 0 stores).  tools/emulate_common.h has the CPU drivers.
template <class Cfg, class Body> __device__ __forceinline__ void run_welch_groups(const typename Body::Args& a) {
  using Tile = typename Cfg::Tile;
  using T = typename Body::T;
  extern __shared__ __align__(128) unsigned char onchip_smem[];
  typename Tile::V* exch = reinterpret_cast<typename Tile::V*>(onchip_smem);
  TwPair<T>* twa = reinterpret_cast<TwPair<T>*>(onchip_smem + Cfg::EX_BYTES);
  T* acc = reinterpret_cast<T*>(onchip_smem + Cfg::EX_BYTES + Cfg::TWA_BYTES);
  for (int i = threadIdx.x; i < (Tile::RA / 2) * Tile::RB; i += Cfg::THREADS) twa[i] = a.twa[i];
  __syncthreads();
  Tile f;
  // One loop over (group, round), carrying only g and r: whatever a phase derives from g is formed again where it is
  // used (g is opaque at the top of every iteration), so the FFT phases have the registers the stft kernel has.
  long g = blockIdx.x;
  int r = 0;
  while (g < a.w.groups) {
    Body::opaque(g);
    static_for<0, Body::kPhases>([&](auto P) FB_LAMBDA {
      Body::template phase<decltype(P)::value>(f, a, g, r, threadIdx.x, exch, acc, twa);
      if constexpr (Body::pair_barrier(decltype(P)::value))
        asm volatile("bar.sync %0, 64;" ::"r"(1 + (int)threadIdx.x / 64) : "memory");
      else
        __syncwarp();
    });
    if (++r == a.w.rounds(g)) {
      __syncthreads();
      Body::flush(a, g, threadIdx.x, acc);
      __syncthreads();
      g += gridDim.x;
      r = 0;
    }
  }
}

template <class Cfg, int MINB>
__global__ void __launch_bounds__(Cfg::THREADS, MINB) onchip_welch_kernel(const typename WelchBody<Cfg>::Args a) {
  run_welch_groups<Cfg, WelchBody<Cfg>>(a);
}
template <class Cfg, int MINB, bool COH>
__global__ void __launch_bounds__(Cfg::THREADS, MINB) onchip_csd_kernel(const typename CsdBody<Cfg, COH>::Args a) {
  run_welch_groups<Cfg, CsdBody<Cfg, COH>>(a);
}

// ---- fused discrete cosine transforms of real rows, N = 2L (real::dct2_pair / dct3_pair, DESIGN.md §4.16) --------
// Type 2 (Dct2Body):
//   * load (phase 0): lane u of the FFT reads the row as pairs (x[2j], x[2j+1]), j = u, u + TP, ..., and writes them
//     into the FFT's park as reals in Makhoul's order, v[j] = x[2j] and v[N-1-j] = x[2j+1];
//   * phases 1-4: StftBody's stage A from the park, the scatter, RealBody's gather + stage B and park;
//   * pairs (phase 5): each lane forms the four outputs y[k], y[N-k], y[L-k], y[L+k] of the pairs it owns,
//     k = u + TP*j, into tile registers 2j and 2j+1; lane u = 0's pair k = 0 gives only y[0] and y[L], so its register 1
//     takes y[L/2] and y[3L/2] of the self-paired k = L/2;
//   * park (phase 6): the N outputs go into the FFT's park as reals (no lane reads Z any more);
//   * store (phase 7): consecutive lanes write consecutive outputs of the row.
// Type 3 (Dct3Body):
//   * load (phase 0): the row's N reals into the park, one complex value (two reals) per lane and step;
//   * pairs (phase 1): each lane forms Z'[k] and Z'[L-k] of the pairs it owns, k = u + TP*j, from x[k], x[N-k], x[L-k]
//     and x[L+k] in the park, into tile registers 2j and 2j+1 (lane u = 0: Z'[0] and the self-paired Z'[L/2]);
//   * park (phase 2): Z' into the park in natural order;
//   * phases 3-4: ConvBody's stage A on conj Z' from the park and its scatter: the inverse runs on the forward tile as
//     conj(FFT(conj .));
//   * phases 5-6: RealBody's gather + stage B and park: the park holds conj u as interleaved reals;
//   * store (phase 7): lane u writes (y[2j], y[2j+1]) = (u[j], u[N-1-j]), j = u, u + TP, ..., as one complex value.
// Forming Z'[n] straight in the stage-A registers instead, from the four inputs of each of the lane's E positions, made
// ptxas spill 360-380 bytes at the f32 L = 512 and 1024 register caps (and 20-104 bytes at L = 128).
// A row is read completely into the park before any of its outputs is stored, and only its own FFT reads it (a column
// past the batch transforms zeros and stores nothing), so in == out is safe.
template <class Cfg> struct Dct2Body {
  using Stft = StftBody<Cfg>;
  using Real = RealBody<Cfg>;
  using Tile = typename Cfg::Tile;   // FWD = true
  using V = typename Tile::V;
  using T = decltype(V::x);
  static constexpr int L = Cfg::L, TP = Tile::TP, E = Tile::E;
  // Real::Args with in = out = nullptr and h the pair step's scale; x, y: rows of N = 2L reals (x == y allowed); wq: W^k,
  // k <= L; h0: the scale of bin 0 (real::dct_scales)
  struct Args : Real::Args { const T* x; T* y; const V* wq; T h0; };

  static FB_HD long row(long grp, int t) { return grp * Cfg::C + Tile::template col_of<true>(t); }

  static FB_HD void load(const Args& a, long grp, int t, V* smem) {
    const int u = Tile::template u_of<true>(t);
    const long b = row(grp, t);
    T* z = reinterpret_cast<T*>(smem + Real::park(t));
    if (b >= a.batch) {
      for (int p = u; p < 2 * L; p += TP) z[p] = (T)0;
      return;
    }
    const V* src = reinterpret_cast<const V*>(a.x + b * (2 * L));
#pragma unroll 2
    for (int j = u; j < L; j += TP) {
      const V s = real::lin_ld(src + j, b);
      z[j] = s.x;
      z[2 * L - 1 - j] = s.y;
    }
  }
  static FB_HD void pairs(Tile& f, const Args& a, int t, const V* smem) {
    const int u = Tile::template u_of<true>(t);
    const V* z = smem + Real::park(t);
#pragma unroll
    for (int j = 0; j < E / 2; ++j) {
      const int k = u + TP * j;
      real::dct2_pair(z[k], z[(L - k) & (L - 1)], (long)L, (long)k, a.tab, a.wq, a.h, a.h0, f.v[2 * j], f.v[2 * j + 1]);
    }
    if (u == 0) {
      V hi;
      real::dct2_pair(z[L / 2], z[L / 2], (long)L, (long)(L / 2), a.tab, a.wq, a.h, a.h0, f.v[1], hi);
    }
  }
  static FB_HD void park_out(const Tile& f, int t, V* smem) {
    const int u = Tile::template u_of<true>(t);
    T* y = reinterpret_cast<T*>(smem + Real::park(t));
#pragma unroll
    for (int j = 0; j < E / 2; ++j) {
      const int k = u + TP * j;
      const V lo = f.v[2 * j], hi = f.v[2 * j + 1];
      if (k == 0) {
        y[0] = lo.x;
        y[L] = lo.y;
        y[L / 2] = hi.x;
        y[3 * L / 2] = hi.y;
      } else {
        y[k] = lo.x;
        y[2 * L - k] = lo.y;
        y[L - k] = hi.x;
        y[L + k] = hi.y;
      }
    }
  }
  static FB_HD void store(const Args& a, long grp, int t, const V* smem) {
    const int u = Tile::template u_of<true>(t);
    const long b = row(grp, t);
    if (b >= a.batch) return;
    const T* y = reinterpret_cast<const T*>(smem + Real::park(t));
    T* dst = a.y + b * (2 * L);
#pragma unroll 2
    for (int p = u; p < 2 * L; p += TP) real::lin_st(dst + p, y[p], b);
  }

  // phase protocol (tilefft.cuh): load into the park; StftBody's stage A and scatter; RealBody's gather + stage B and
  // park; pairs, park, store
  static constexpr int kPhases = 8;
  template <int P> static FB_HD void phase(Tile& f, const Args& a, long grp, int t, V* smem, const TwPair<T>* twa) {
    if constexpr (P == 0) load(a, grp, t, smem);
    else if constexpr (P == 1) Stft::load_stage_a(f, t, smem, twa);
    else if constexpr (P == 2) f.template scatter<true, typename Cfg::Lay>(t, smem);
    else if constexpr (P == 3) Real::fwd_gather(f, t, smem);
    else if constexpr (P == 4) Real::fwd_park(f, t, smem);
    else if constexpr (P == 5) pairs(f, a, t, smem);
    else if constexpr (P == 6) park_out(f, t, smem);
    else store(a, grp, t, smem);
  }
};

template <class Cfg> struct Dct3Body {
  using Dct2 = Dct2Body<Cfg>;
  using Conv = ConvBody<Cfg>;
  using Real = RealBody<Cfg>;
  using Tile = typename Cfg::Tile;   // FWD = true
  using V = typename Tile::V;
  using T = decltype(V::x);
  static constexpr int L = Cfg::L, TP = Tile::TP, E = Tile::E;
  using Args = typename Dct2::Args;

  static FB_HD void load(const Args& a, long grp, int t, V* smem) {
    const int u = Tile::template u_of<true>(t);
    const long b = Dct2::row(grp, t);
    V* z = smem + Real::park(t);
    if (b >= a.batch) {
      for (int j = u; j < L; j += TP) z[j] = mk<T>((T)0, (T)0);
      return;
    }
    const V* src = reinterpret_cast<const V*>(a.x + b * (2 * L));
#pragma unroll 2
    for (int j = u; j < L; j += TP) z[j] = real::lin_ld(src + j, b);
  }
  // Z'[k] and Z'[L-k] of the pairs the lane owns into tile registers 2j and 2j+1 (lane u = 0: Z'[0] and Z'[L/2])
  static FB_HD void pairs(Tile& f, const Args& a, int t, const V* smem) {
    const int u = Tile::template u_of<true>(t);
    const T* x = reinterpret_cast<const T*>(smem + Real::park(t));
#pragma unroll
    for (int j = 0; j < E / 2; ++j)
      real::dct3_pair(x, (long)L, (long)(u + TP * j), a.tab, a.wq, a.h, a.h0, f.v[2 * j], f.v[2 * j + 1]);
    if (u == 0) {
      V q;
      real::dct3_pair(x, (long)L, (long)(L / 2), a.tab, a.wq, a.h, a.h0, f.v[1], q);
    }
  }
  static FB_HD void park_pairs(const Tile& f, int t, V* smem) {
    const int u = Tile::template u_of<true>(t);
    V* z = smem + Real::park(t);
#pragma unroll
    for (int j = 0; j < E / 2; ++j) {
      const int k = u + TP * j;
      z[k] = f.v[2 * j];
      z[k == 0 ? L / 2 : L - k] = f.v[2 * j + 1];
    }
  }
  static FB_HD void store(const Args& a, long grp, int t, const V* smem) {
    const int u = Tile::template u_of<true>(t);
    const long b = Dct2::row(grp, t);
    if (b >= a.batch) return;
    const T* r = reinterpret_cast<const T*>(smem + Real::park(t));
    V* dst = reinterpret_cast<V*>(a.y + b * (2 * L));
    // u[p] = r[p] (p even), -r[p] (p odd); j and N-1-j have opposite parities
#pragma unroll 2
    for (int j = u; j < L; j += TP) {
      const T lo = r[j], hi = r[2 * L - 1 - j];
      real::lin_st(dst + j, (j & 1) ? mk<T>(-lo, hi) : mk<T>(lo, -hi), b);
    }
  }

  // phase protocol (tilefft.cuh): load into the park; pairs, park Z'; ConvBody's conj stage A and scatter; RealBody's
  // gather + stage B and park; store
  static constexpr int kPhases = 8;
  template <int P> static FB_HD void phase(Tile& f, const Args& a, long grp, int t, V* smem, const TwPair<T>* twa) {
    if constexpr (P == 0) load(a, grp, t, smem);
    else if constexpr (P == 1) pairs(f, a, t, smem);
    else if constexpr (P == 2) park_pairs(f, t, smem);
    else if constexpr (P == 3) Conv::inv_stage_a(f, t, smem, twa);
    else if constexpr (P == 4) Conv::inv_scatter(f, t, smem);
    else if constexpr (P == 5) Real::fwd_gather(f, t, smem);
    else if constexpr (P == 6) Real::fwd_park(f, t, smem);
    else store(a, grp, t, smem);
  }
};

// the body of DCT type TYPE (2 or 3)
template <class Cfg, int TYPE> struct DctBodyOf { using type = Dct2Body<Cfg>; };
template <class Cfg> struct DctBodyOf<Cfg, 3> { using type = Dct3Body<Cfg>; };
template <class Cfg, int TYPE> using DctBody = typename DctBodyOf<Cfg, TYPE>::type;

template <class Cfg, int MINB, int TYPE>
__global__ void __launch_bounds__(Cfg::THREADS, MINB) onchip_dct_kernel(const typename Dct2Body<Cfg>::Args a) {
  run_onchip_groups<Cfg, DctBody<Cfg, TYPE>>(a);
}

// ---- fused type-IV DCT and MDCT of real rows, N = 2L (real::dct4_pre / dct4_post / mdct_fold, DESIGN.md §4.20) -------
// Dct4Body, on rows of N reals:
//   * load (phase 0): consecutive lanes of the FFT read consecutive samples of the row and park x[2j] and x[2j+1] as
//     z[j].x and z[L-1-j].y (reals 2j and N-1-2j), so that the park holds z[n] = (x[2n], x[N-1-2n]);
//   * pre (phase 1): each lane multiplies the park's positions n = u, u + TP, ... by W^{2n} in place;
//   * phases 2-5: StftBody's stage A from the park, the scatter, RealBody's gather + stage B and park: the park holds
//     Z in natural order;
//   * post (phase 6): each lane forms (y[2k], y[N-1-2k]) of its positions k = u + TP*j from Z[k] into tile register j;
//   * park (phase 7): those pairs into the park as reals (no lane reads Z any more);
//   * store (phase 8): consecutive lanes write consecutive complex values (two reals) of the row.
// The twiddles are applied in passes over the park, with each step's index formed in its own loop iteration, as
// Dct2Body's pairs are.  Applying them in the stage-A registers and to the stage-B registers instead kept the twiddle
// indices and table reads live through the FFT phases: ptxas spilled 24-270 bytes at the f32 L = 128, 512 and 1024
// register caps.
// A row is read completely into the park before any output is stored, and only its own FFT reads it (a column past the
// batch transforms zeros and stores nothing), so in == out is safe.
// MdctBody, on groups of C consecutive frames (real::mdct_map): its load (phase 0) reads the frame's 2N samples as
// StftBody's does (unmasked inside the row, through FrameMap::Edge at its ends, so no read leaves [0, L)), windows and
// folds them, and parks the N folded values in Dct4Body's packing; frame q of the launch writes output row q (frame-major,
// N reals per frame).  The rest is Dct4Body's.
template <class Cfg> struct Dct4Body {
  using Stft = StftBody<Cfg>;
  using Real = RealBody<Cfg>;
  using Tile = typename Cfg::Tile;   // FWD = true
  using V = typename Tile::V;
  using T = decltype(V::x);
  static constexpr int L = Cfg::L, TP = Tile::TP, E = Tile::E;
  // Real::Args with in = out = nullptr; x, y: rows of N = 2L reals (x == y allowed); wq: W^k, k <= L; c: the post
  // step's constant (real::dct4_const)
  struct Args : Real::Args { const T* x; T* y; const V* wq; V c; };

  static FB_HD long row(long grp, int t) { return grp * Cfg::C + Tile::template col_of<true>(t); }

  static FB_HD void load(const Args& a, long grp, int t, V* smem) {
    const int u = Tile::template u_of<true>(t);
    const long b = row(grp, t);
    T* z = reinterpret_cast<T*>(smem + Real::park(t));
    if (b >= a.batch) {
      for (int p = u; p < 2 * L; p += TP) z[p] = (T)0;
      return;
    }
    const T* src = a.x + b * (2 * L);
    // sample p at real p (even) or N - p (odd) of the park
#pragma unroll 2
    for (int p = u; p < 2 * L; p += TP) z[(p & 1) ? 2 * L - p : p] = real::lin_ld(src + p, b);
  }
  // z[n] *= W^{2n} at the lane's positions, in place
  static FB_HD void pre(const Args& a, int t, V* smem) {
    const int u = Tile::template u_of<true>(t);
    V* z = smem + Real::park(t);
#pragma unroll 4
    for (int j = 0; j < E; ++j) {
      const int n = u + TP * j;
      const V v = z[n];
      z[n] = real::dct4_pre(v.x, v.y, a.wq, (long)(2 * L), (long)n);
    }
  }
  // (y[2k], y[N-1-2k]) of the lane's positions k = u + TP*j into tile register j
  static FB_HD void post(Tile& f, const Args& a, int t, const V* smem) {
    const int u = Tile::template u_of<true>(t);
    const V* z = smem + Real::park(t);
#pragma unroll
    for (int j = 0; j < E; ++j) {
      const int k = u + TP * j;
      f.v[j] = real::dct4_post(z[k], a.c, a.wq, (long)(2 * L), (long)k);
    }
  }
  static FB_HD void park_out(const Tile& f, int t, V* smem) {
    const int u = Tile::template u_of<true>(t);
    T* y = reinterpret_cast<T*>(smem + Real::park(t));
#pragma unroll
    for (int j = 0; j < E; ++j) {
      const int k = u + TP * j;
      y[2 * k] = f.v[j].x;
      y[2 * L - 1 - 2 * k] = f.v[j].y;
    }
  }
  // out: the row's N reals
  static FB_HD void store(T* out, long g, int t, const V* smem) {
    const int u = Tile::template u_of<true>(t);
    const V* y = smem + Real::park(t);
    V* dst = reinterpret_cast<V*>(out);
#pragma unroll 2
    for (int j = u; j < L; j += TP) real::lin_st(dst + j, y[j], g);
  }

  // phase protocol (tilefft.cuh): load into the park; pre-twiddle in the park; StftBody's stage A and scatter;
  // RealBody's gather + stage B and park; post into registers, park, store
  static constexpr int kPhases = 9;
  template <int P> static FB_HD void phase(Tile& f, const Args& a, long grp, int t, V* smem, const TwPair<T>* twa) {
    if constexpr (P == 0) load(a, grp, t, smem);
    else if constexpr (P == 1) pre(a, t, smem);
    else if constexpr (P == 2) Stft::load_stage_a(f, t, smem, twa);
    else if constexpr (P == 3) f.template scatter<true, typename Cfg::Lay>(t, smem);
    else if constexpr (P == 4) Real::fwd_gather(f, t, smem);
    else if constexpr (P == 5) Real::fwd_park(f, t, smem);
    else if constexpr (P == 6) post(f, a, t, smem);
    else if constexpr (P == 7) park_out(f, t, smem);
    else {
      const long b = row(grp, t);
      if (b < a.batch) store(a.y + b * (2 * L), b, t, smem);
    }
  }
};

template <class Cfg> struct MdctBody {
  using Dct4 = Dct4Body<Cfg>;
  using Real = RealBody<Cfg>;
  using Tile = typename Cfg::Tile;   // FWD = true
  using V = typename Tile::V;
  using T = decltype(V::x);
  static constexpr int L = Cfg::L, TP = Tile::TP;
  // Dct4::Args with x = the rows, y = the output of frame g0, batch = frames of the launch; plus the window (2N reals)
  // and the frame map (real::mdct_map)
  struct Args : Dct4::Args { const T* win; real::FrameMap m; };

  static FB_HD void load(const Args& a, long grp, int t, V* smem) {
    const int u = Tile::template u_of<true>(t);
    long q = Dct4::row(grp, t);
    if (q >= a.batch) q = a.batch - 1;
    const long g = a.m.g0 + q, b = a.m.row_of(g), t0 = a.m.start(g, b);
    const T* row = a.x + (b - a.m.r0) * a.m.in_ld;
    T* z = reinterpret_cast<T*>(smem + Real::park(t));
    constexpr int N = 2 * L;
    // folded value n of the frame into the park: n even at n, n odd at N - n (z[j] = (u[2j], u[N-1-2j]))
    auto put = [&](int n, T f0, T f1) FB_LAMBDA { z[(n & 1) ? N - n : n] = real::mdct_fold(f0, f1, (long)n, (long)N); };
    if (t0 >= 0 && t0 + 2 * N <= a.m.len) {
      const T* src = row + t0;
#pragma unroll 2
      for (int n = u; n < N; n += TP) {
        long s0, s1;
        real::mdct_fold_pos(n, N, s0, s1);
        put(n, real::lin_ld(src + s0, g) * a.win[s0], real::lin_ld(src + s1, g) * a.win[s1]);
      }
    } else {
      // 32-bit offsets from an anchor sample c of the row (see FrameMap::edge)
      const real::FrameMap::Edge e = a.m.edge(t0);
      const T* src = row + e.c;
#pragma unroll 2
      for (int n = u; n < N; n += TP) {
        long s0, s1;
        real::mdct_fold_pos(n, N, s0, s1);
        const int d0 = e.map(e.d0 + (int)s0), d1 = e.map(e.d0 + (int)s1);
        put(n, e.in(d0) ? real::lin_ld(src + d0, g) * a.win[s0] : (T)0,
            e.in(d1) ? real::lin_ld(src + d1, g) * a.win[s1] : (T)0);
      }
    }
  }

  // phase protocol (tilefft.cuh): the frame folded into the park; Dct4Body's phases 1-7; store
  static constexpr int kPhases = Dct4::kPhases;
  template <int P> static FB_HD void phase(Tile& f, const Args& a, long grp, int t, V* smem, const TwPair<T>* twa) {
    if constexpr (P == 0) load(a, grp, t, smem);
    else if constexpr (P < kPhases - 1) Dct4::template phase<P>(f, a, grp, t, smem, twa);
    else {
      const long q = Dct4::row(grp, t);
      if (q < a.batch) Dct4::store(a.y + q * (2 * L), a.m.g0 + q, t, smem);
    }
  }
};

template <class Cfg, int MINB>
__global__ void __launch_bounds__(Cfg::THREADS, MINB) onchip_dct4_kernel(const typename Dct4Body<Cfg>::Args a) {
  run_onchip_groups<Cfg, Dct4Body<Cfg>>(a);
}
template <class Cfg, int MINB>
__global__ void __launch_bounds__(Cfg::THREADS, MINB) onchip_mdct_kernel(const typename MdctBody<Cfg>::Args a) {
  run_onchip_groups<Cfg, MdctBody<Cfg>>(a);
}

// ---- fused analytic signal and envelope of real rows, N = 2L (real::hilbert_pair, DESIGN.md §4.19) -----------------
// ConvBody's phases 0-5 as they are, with the pair step real::hilbert_pair (a fixed multiplier, no spectrum read) in
// phase 3.  Then:
//   * store (phase 6): ConvBody's gather + stage B leave y at the lane's stage-B positions p as conj(y[2p], y[2p+1]);
//     the lane re-reads x[2p], x[2p+1] from the row (which the load just brought into L2) and writes, per position,
//     (x[2p], y[2p]), (x[2p+1], y[2p+1]) as one 16-byte store in f32 (ANALYTIC), or the two moduli (ENV).
// The re-reads go G positions at a time ahead of their stores, so a lane has G loads in flight rather than one.  Every
// lane reads x only at the positions it stores, each before its store, and in and y are not __restrict__, so the
// envelope may run in place (y == in).
template <class Cfg> struct HilbertArgs : ConvBody<Cfg>::Args { void* y; };
template <class Cfg, bool ENV> struct HilbertBody {
  using Conv = ConvBody<Cfg>;
  using Real = RealBody<Cfg>;
  using Tile = typename Cfg::Tile;   // FWD = true
  using V = typename Tile::V;
  using T = decltype(V::x);
  static constexpr int L = Cfg::L, TP = Tile::TP, RA = Tile::RA, RB = Tile::RB, E = Tile::E;
  static constexpr int G = sizeof(T) == 4 && !ENV ? 8 : 4;
  static_assert(RB % G == 0, "the re-reads go G stage-B registers at a time");
  // Conv::Args with in = the rows (L complex values each), out = spec = nullptr, rows = per = 1 and h = 1 / (2N); y: the
  // output rows, N complex values (analytic) or N reals (ENV) each
  using Args = HilbertArgs<Cfg>;

  static FB_HD void pairs(const Args& a, long grp, int t, V* smem) {
    const int u = Tile::template u_of<true>(t);
    const long b = grp * Cfg::C + Tile::template col_of<true>(t);
    if (b >= a.batch) return;
    V* z = smem + Real::park(t);
#pragma unroll 4
    for (int j = 0; j < E / 2; ++j) real::hilbert_pair(z, (long)L, (long)(u + TP * j), a.tab, a.h);
    if (u == 0) real::hilbert_pair(z, (long)L, (long)(L / 2), a.tab, a.h);
  }
  static FB_HD void store(Tile& f, const Args& a, long grp, int t, const V* smem) {
    const int u = Tile::template u_of<true>(t);
    f.template gather<true, typename Cfg::Lay>(t, smem);
    f.stage_b();
    const long b = grp * Cfg::C + Tile::template col_of<true>(t);
    if (b >= a.batch) return;
    const V* x = a.in + b * L;
    V* y = reinterpret_cast<V*>(a.y) + (ENV ? b * L : b * 2 * L);
    static_for<0, Tile::NB>([&](auto Cc) FB_LAMBDA {
      constexpr int c = decltype(Cc)::value;
      static_for<0, RB / G>([&](auto Gg) FB_LAMBDA {
        constexpr int r0 = decltype(Gg)::value * G;
        V xs[G];
        static_for<0, G>([&](auto Rr) FB_LAMBDA {
          constexpr int i = decltype(Rr)::value;
          xs[i] = real::lin_ld(x + (u + TP * c) + RA * (r0 + i), b);
        });
        static_for<0, G>([&](auto Rr) FB_LAMBDA {
          constexpr int i = decltype(Rr)::value;
          const int p = (u + TP * c) + RA * (r0 + i);
          const V v = cconj(f.v[c * RB + bitrev(r0 + i, ilog2(RB))]);
          if constexpr (ENV)
            real::lin_st(y + p, mk<T>(real::hilbert_mod(xs[i].x, v.x), real::hilbert_mod(xs[i].y, v.y)), b);
          else
            real::analytic_st2(y + 2 * p, xs[i], v, b);
        });
      });
    });
  }

  // phase protocol (tilefft.cuh): ConvBody's phases 0-5 with the pair step of phase 3 replaced; store
  static constexpr int kPhases = 7;
  template <int P> static FB_HD void phase(Tile& f, const Args& a, long grp, int t, V* smem, const TwPair<T>* twa) {
    if constexpr (P == 3) pairs(a, grp, t, smem);
    else if constexpr (P < 6) Conv::template phase<P>(f, a, grp, t, smem, twa);
    else store(f, a, grp, t, smem);
  }
};

template <class Cfg, int MINB, bool ENV>
__global__ void __launch_bounds__(Cfg::THREADS, MINB) onchip_hilbert_kernel(const HilbertArgs<Cfg> a) {
  run_onchip_groups<Cfg, HilbertBody<Cfg, ENV>>(a);
}

// ---- fused Bluestein -------------------------------------------------------------------------------------------
// conj(a) * b
template <typename V> FB_HD V cmul_conja(V a, V b) { return cmulc(b, a); }

template <class Cfg> struct BluesteinBody {
  using Tile = typename Cfg::Tile;   // FWD = true
  using V = typename Tile::V;
  using T = decltype(V::x);
  static constexpr int L = Cfg::L, RA = Tile::RA, RB = Tile::RB, TP = Tile::TP, E = Tile::E;
  static_assert(Tile::NA * RA == E && Tile::NB * RB == E, "tile shape");
  struct Args {
    const V* in; V* out;
    const TwPair<T>* twa;
    const V* chirp;   // [L]  c[n] = exp(-+ i pi n^2 / N) for n < N, 0 beyond   (direction-specific table)
    const V* wm;      // [L]  w_M^n, M = 2L
    const V* wce;     // [L]  conj(W[2k])   W = FFT_M(wrapped conj chirp)      (direction-specific)
    const V* wco;     // [L]  conj(W[2k+1])
    long n, batch;
    T scale;          // Transform scale / M
  };

  // position n (stage-A input order) held in f.v[q*RA + i] by the thread with offset u
  static FB_HD int pos_in(int u, int q, int i) { return u + TP * q + RB * i; }
  // position (stage-B output order) of f.v[c*RB + bitrev(r)]
  static FB_HD int pos_out(int u, int c, int r) { return (u + TP * c) + RA * r; }

  // x * chirp (odd = false) or x * chirp * w_M^n (odd = true) into stage-A input order, then stage A
  template <bool ODD>
  static FB_HD void load_half(Tile& f, const Args& a, long b, int t, V* smem, const TwPair<T>* twa,
                              const V* chirp, const V* wm) {
    const int u = Tile::template u_of<true>(t);
    const V* p = a.in + b * a.n;
    static_for<0, Tile::NA>([&](auto Q) FB_LAMBDA {
      constexpr int q = decltype(Q)::value;
      static_for<0, RA>([&](auto I) FB_LAMBDA {
        constexpr int i = decltype(I)::value;
        const int n = pos_in(u, q, i);
        V v = mk<T>((T)0, (T)0);
        if (n < a.n) {
          v = cmul(p[n], chirp[n]);
          if (ODD) v = cmul(v, wm[n]);
        }
        f.v[q * RA + i] = v;
      });
    });
    f.template stage_a<true>(t, twa);
    f.template scatter<true, typename Cfg::Lay>(t, smem);
  }

  // finish the forward FFT and multiply by conj(W) in the conjugate domain.  The outputs sit at
  // bit-reversed register positions while the next stage A wants natural order: for the square tiles
  // used here (RA == RB, one butterfly per thread and stage) output r of this FFT is input i = r of
  // the next one, so the reordering is an in-register swap of (r, bitrev r) pairs -- pure renaming.
  static FB_HD void middle(Tile& f, int t, V* smem, const V* wc) {
    static_assert(RA == RB && Tile::NA == 1 && Tile::NB == 1, "fused Bluestein uses square tiles");
    const int u = Tile::template u_of<true>(t);
    f.template gather<true, typename Cfg::Lay>(t, smem);
    f.stage_b();
    static_for<0, RB>([&](auto Rr) FB_LAMBDA {
      constexpr int r = decltype(Rr)::value;
      constexpr int q = bitrev(r, ilog2(RB));
      if constexpr (r == q) {
        f.v[r] = cmul_conja(f.v[r], wc[pos_out(u, 0, r)]);          // conj(A[k] * W[k])
      } else if constexpr (r < q) {
        const V lo = cmul_conja(f.v[q], wc[pos_out(u, 0, r)]);      // value of output r lives at position q
        const V hi = cmul_conja(f.v[r], wc[pos_out(u, 0, q)]);
        f.v[r] = lo;
        f.v[q] = hi;
      }
    });
  }
  static FB_HD void second_fft_start(Tile& f, int t, V* smem, const TwPair<T>* twa) {
    f.template stage_a<true>(t, twa);
    f.template scatter<true, typename Cfg::Lay>(t, smem);
  }
  static FB_HD void second_fft_finish(Tile& f, int t, const V* smem) {
    f.template gather<true, typename Cfg::Lay>(t, smem);
    f.stage_b();
  }
  // out[n] = scale * c[n] * (e[n] + conj(w_M^n) * o[n]),  e = conj(E'), o = conj(O')
  // `stash` holds E' of the even half, thread-private: register i of thread t at stash[i*THREADS + t]
  static FB_HD void stash_even(const Tile& f, int t, V* stash) {
    static_for<0, E>([&](auto I) FB_LAMBDA { constexpr int i = decltype(I)::value; stash[i * Cfg::THREADS + t] = f.v[i]; });
  }
  static FB_HD void combine_store_local(const V (&keep)[E], const Tile& f, const Args& a, long b, int t, const V* chirp,
                                        const V* wm) {
    const int u = Tile::template u_of<true>(t);
    V* p = a.out + b * a.n;
    static_for<0, Tile::NB>([&](auto Cc) FB_LAMBDA {
      constexpr int c = decltype(Cc)::value;
      static_for<0, RB>([&](auto Rr) FB_LAMBDA {
        constexpr int r = decltype(Rr)::value;
        const int n = pos_out(u, c, r);
        if (n < a.n) {
          constexpr int idx = c * RB + bitrev(r, ilog2(RB));
          const V o = cmul(f.v[idx], wm[n]);
          p[n] = cscale(cmul_conja(cadd(keep[idx], o), chirp[n]), a.scale);
        }
      });
    });
  }
  static FB_HD void combine_store(const V* stash, const Tile& f, const Args& a, long b, int t, const V* chirp,
                                  const V* wm) {
    const int u = Tile::template u_of<true>(t);
    V* p = a.out + b * a.n;
    static_for<0, Tile::NB>([&](auto Cc) FB_LAMBDA {
      constexpr int c = decltype(Cc)::value;
      static_for<0, RB>([&](auto Rr) FB_LAMBDA {
        constexpr int r = decltype(Rr)::value;
        const int n = pos_out(u, c, r);
        if (n < a.n) {
          constexpr int idx = c * RB + bitrev(r, ilog2(RB));
          const V o = cmul(f.v[idx], wm[n]);              // O' * w  == conj(o * conj(w))
          const V sum = cadd(stash[idx * Cfg::THREADS + t], o);              // conj(e + conj(w) o)
          p[n] = cscale(cmul_conja(sum, chirp[n]), a.scale);
        }
      });
    });
  }
};

template <class Cfg, int MINB, bool LOCAL_STASH = false>
__global__ void __launch_bounds__(Cfg::THREADS, MINB)
bluestein_fused_kernel(const typename BluesteinBody<Cfg>::Args a) {
  using Body = BluesteinBody<Cfg>;
  using V = typename Cfg::Tile::V;
  using T = decltype(V::x);
  constexpr int L = Cfg::L;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  V* exch = reinterpret_cast<V*>(smem_raw);
  TwPair<T>* twa = reinterpret_cast<TwPair<T>*>(smem_raw + Cfg::EX_BYTES);
  V* tabs = reinterpret_cast<V*>(smem_raw + Cfg::EX_BYTES + Cfg::TWA_BYTES);
  V* chirp = tabs; V* wm = tabs + L; V* wce = tabs + 2 * L; V* wco = tabs + 3 * L;
  V* stash_smem = tabs + 4 * L;   // [E][THREADS] (unused with LOCAL_STASH)
  // LOCAL_STASH: E' of the even half waits in a per-thread array instead (registers if they fit, else
  // thread-local memory behind L1/L2): frees 8 KB of shared memory per warp -> more resident warps.
  V keep[LOCAL_STASH ? Cfg::Tile::E : 1];
  for (int i = threadIdx.x; i < (Cfg::Tile::RA / 2) * Cfg::Tile::RB; i += Cfg::THREADS) twa[i] = a.twa[i];
  for (int i = threadIdx.x; i < L; i += Cfg::THREADS) {
    chirp[i] = a.chirp[i]; wm[i] = a.wm[i]; wce[i] = a.wce[i]; wco[i] = a.wco[i];
  }
  __syncthreads();
  const int t = threadIdx.x;
  const int col = Cfg::Tile::template col_of<true>(t);
  const long groups = (a.batch + Cfg::C - 1) / Cfg::C;
  typename Cfg::Tile f;
  for (long grp = blockIdx.x; grp < groups; grp += gridDim.x) {
    const long b_real = grp * Cfg::C + col;
    const long b = b_real < a.batch ? b_real : a.batch - 1;
    // even half: E' = FFT(conj(FFT(x c) W_even)), parked in shared memory while the odd half runs
    Body::template load_half<false>(f, a, b, t, exch, twa, chirp, wm);
    __syncwarp();
    Body::middle(f, t, exch, wce);
    __syncwarp();
    Body::second_fft_start(f, t, exch, twa);
    __syncwarp();
    Body::second_fft_finish(f, t, exch);
    if constexpr (LOCAL_STASH) {
      static_for<0, Cfg::Tile::E>([&](auto I) FB_LAMBDA { constexpr int i = decltype(I)::value; keep[i] = f.v[i]; });
    } else {
      Body::stash_even(f, t, stash_smem);
    }
    __syncwarp();
    // odd half
    Body::template load_half<true>(f, a, b, t, exch, twa, chirp, wm);
    __syncwarp();
    Body::middle(f, t, exch, wco);
    __syncwarp();
    Body::second_fft_start(f, t, exch, twa);
    __syncwarp();
    Body::second_fft_finish(f, t, exch);
    if (b_real < a.batch) {
      if constexpr (LOCAL_STASH) Body::combine_store_local(keep, f, a, b, t, chirp, wm);
      else Body::combine_store(stash_smem, f, a, b, t, chirp, wm);
    }
    __syncwarp();
  }
}

}  // namespace onchip
}  // namespace fb200
