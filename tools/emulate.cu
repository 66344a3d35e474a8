// emulate.cu -- runs the fused kernels' device code on the CPU, thread by thread and phase by phase
// (the code in tilefft.cuh / twopass_kernels.cuh is __host__ __device__), and checks the result
// against a double-precision FFT.  There is no GPU in the build container, so this is how index maps,
// twiddle tables and shared-memory layouts are verified before a kernel ever runs on the GPU.
// It also reports shared-memory bank conflicts of the exchange (64-bit/128-bit access model).
// Build: nvcc -std=c++17 -O1 --expt-relaxed-constexpr -I fourier_b200/csrc tools/emulate.cu \
//             fourier_b200/csrc/host_math.cu (host only, never run on the device)
#include "emulate_common.h"

#include "cta_kernels.cuh"
#include "dist_kernels.cuh"
#include "fused_configs.cuh"
#include "fused_kernels.cuh"
#include "outer_kernels.cuh"
#include "twopass_kernels.cuh"

using namespace fb200::twopass;

template <typename T> static const char* prec() { return sizeof(T) == 4 ? "f32" : "f64"; }

// Bank-conflict report for the exchange of a tile: scatter with mapping UF_A, gather with col-fast.
template <class Tile, class LAY, int UF_A, int UF_B = 0>
static void report_conflicts(const char* name) {
  using V = typename Tile::V;
  constexpr int B = (int)sizeof(V);
  int worst_w = 1, worst_r = 1;
  for (int warp = 0; warp < Tile::THREADS / 32; ++warp) {
    for (int a = 0; a < Tile::NA; ++a)
      for (int p = 0; p < Tile::RA; ++p) {
        std::vector<long> idx;
        for (int l = 0; l < 32; ++l) {
          const int t = warp * 32 + l;
          idx.push_back((long)(Tile::template u_of<UF_A>(t) + Tile::TP * a) * LAY::SJ + (long)p * LAY::SP +
                        (long)Tile::template col_of<UF_A>(t) * LAY::SC);
        }
        worst_w = std::max(worst_w, conflict_degree<B>(idx));
      }
    for (int c = 0; c < Tile::NB; ++c)
      for (int j = 0; j < Tile::RB; ++j) {
        std::vector<long> idx;
        for (int l = 0; l < 32; ++l) {
          const int t = warp * 32 + l;
          idx.push_back((long)j * LAY::SJ + (long)(Tile::template u_of<UF_B>(t) + Tile::TP * c) * LAY::SP +
                        (long)Tile::template col_of<UF_B>(t) * LAY::SC);
        }
        worst_r = std::max(worst_r, conflict_degree<B>(idx));
      }
  }
  printf("  %-8s threads %4d smem %6zu B  exchange conflicts: write x%d, read x%d\n", name, Tile::THREADS,
         sizeof(V) * Tile::template smem_elems<LAY>(), worst_w, worst_r);
}

template <typename T, class Cfg>
static int check(const char* name, double tol) {
  const long N = Cfg::N, N1 = Cfg::N1, N2 = Cfg::N2;
  const int batch = 2;
  printf("%s: N=%ld = %ld x %ld\n", name, N, N1, N2);
  report_conflicts<typename Cfg::template Tile1<true>, typename Cfg::Lay1, false>("pass 1");
  report_conflicts<typename Cfg::template Tile2<true>, typename Cfg::Lay2, true>("pass 2");
  int bad = 0;
  for (int fwd = 1; fwd >= 0; --fwd) {
    std::vector<cpx<T>> x((size_t)N * batch), scratch((size_t)N * batch), out((size_t)N * batch);
    fill<T>(x, 7 + fwd);
    const auto* ops = Cfg::ops();
    auto twa1 = make_twa<T>(ops->ra1, ops->rb1), twa2 = make_twa<T>(ops->ra2, ops->rb2);
    std::vector<cpx<T>> tw2(N);
    for (long k1 = 0; k1 < N1; ++k1)
      for (long c = 0; c < N2; ++c) {
        double re, im;
        host_twiddle((size_t)(k1 * c), (size_t)N, &re, &im);
        tw2[k1 * N2 + c] = mk<T>((T)re, (T)im);
      }
    const T scale = (T)0.5;
    if (fwd) {
      run_body<typename Cfg::template Body1<true>, typename Cfg::template Tile1<true>, typename Cfg::Lay1>(
          Cfg::template args1<true>(x.data(), scratch.data(), twa1.data(), tw2.data()), batch * (N2 / Cfg::template Tile1<true>::C));
      run_body<typename Cfg::template Body2<true>, typename Cfg::template Tile2<true>, typename Cfg::Lay2>(
          Cfg::template args2<true>(scratch.data(), out.data(), twa2.data(), scale, true), batch * (N1 / Cfg::template Tile2<true>::C));
    } else {
      run_body<typename Cfg::template Body1<false>, typename Cfg::template Tile1<false>, typename Cfg::Lay1>(
          Cfg::template args1<false>(x.data(), scratch.data(), twa1.data(), tw2.data()), batch * (N2 / Cfg::template Tile1<false>::C));
      run_body<typename Cfg::template Body2<false>, typename Cfg::template Tile2<false>, typename Cfg::Lay2>(
          Cfg::template args2<false>(scratch.data(), out.data(), twa2.data(), scale, true), batch * (N1 / Cfg::template Tile2<false>::C));
    }
    double worst = 0;
    for (int b = 0; b < batch; ++b) {
      std::vector<double> re(N), im(N);
      for (long i = 0; i < N; ++i) { re[i] = x[(size_t)b * N + i].x; im[i] = x[(size_t)b * N + i].y; }
      host_fft_pow2(re, im, !fwd);
      double maxref = 0, maxerr = 0;
      for (long i = 0; i < N; ++i) {
        const double rr = re[i] * 0.5, ii = im[i] * 0.5;
        maxref = std::max(maxref, std::hypot(rr, ii));
        maxerr = std::max(maxerr, std::hypot(out[(size_t)b * N + i].x - rr, out[(size_t)b * N + i].y - ii));
      }
      worst = std::max(worst, maxerr / maxref);
    }
    printf("  %s: max rel err vs f64 FFT %.3e (tol %.1e) %s\n", fwd ? "forward" : "inverse", worst, tol,
           worst < tol ? "OK" : "FAIL");
    bad += !(worst < tol);
  }
  return bad;
}

// ---- on-chip kernels (onchip_kernels.cuh) -------------------------------------------------------------------------
// size class K of onchip_configs.cuh
template <class K>
static int check_onchip(const char* name, double tol) {
  using T = typename K::T;
  constexpr int RA = K::RA, RB = K::RB;
  int bad = 0;
  for (int fwd = 1; fwd >= 0; --fwd) {
    const long L = RA * RB, batch = 5;   // 5 is not a multiple of the transforms per CTA: exercises the tail
    std::vector<cpx<T>> x((size_t)L * batch), out((size_t)L * batch);
    fill<T>(x, 21 + fwd);
    auto twa = make_twa<T>(RA, RB);
    auto run = [&](auto cfg_tag) {
      using Cfg = decltype(cfg_tag);
      using Body = onchip::FftBody<Cfg>;
      run_body<Body, typename Cfg::Tile, typename Cfg::Lay>({x.data(), out.data(), twa.data(), batch, (T)0.5, 1},
                                                            (batch + Cfg::C - 1) / Cfg::C, twa.data());
      report_conflicts<typename Cfg::Tile, typename Cfg::Lay, true, true>("exchange");
    };
    if (fwd) run(typename K::template Cfg<true>{}); else run(typename K::template Cfg<false>{});
    double worst = 0;
    for (long b = 0; b < batch; ++b) {
      std::vector<double> re(L), im(L);
      for (long i = 0; i < L; ++i) { re[i] = x[b * L + i].x; im[i] = x[b * L + i].y; }
      host_fft_pow2(re, im, !fwd);
      double mr = 0, me = 0;
      for (long i = 0; i < L; ++i) {
        mr = std::max(mr, std::hypot(re[i], im[i]) * 0.5);
        me = std::max(me, std::hypot(out[b * L + i].x - 0.5 * re[i], out[b * L + i].y - 0.5 * im[i]));
      }
      worst = std::max(worst, me / mr);
    }
    printf("%s L=%d %s: max rel err %.3e %s\n", name, RA * RB, fwd ? "forward" : "inverse", worst, worst < tol ? "OK" : "FAIL");
    bad += !(worst < tol);
  }
  return bad;
}

// the fused Bluestein kernel of size class K (onchip_configs.cuh), at its warps per CTA and with its stash of the even
// half: shared memory (stash_even, combine_store) or, with LOCAL_STASH, a per-thread array (combine_store_local)
template <class K>
static int check_bluestein(const char* name, long n, double tol) {
  using T = typename K::T;
  using Cfg = typename K::BCfg;
  using Body = onchip::BluesteinBody<Cfg>;
  using V = cpx<T>;
  constexpr int R = K::RA, E = K::E;
  const long L = R * R, M = 2 * L, batch = 3;
  int bad = 0;
  for (int inverse = 0; inverse < 2; ++inverse) {
    // tables exactly as Plan<T>::init_bluestein / init_bluestein_fused build them
    std::vector<double> cr(n), ci(n), wr(M, 0.0), wi(M, 0.0);
    for (long i = 0; i < n; ++i) {
      const size_t idx = (size_t)(((unsigned __int128)i * i) % (2 * (unsigned __int128)n));
      host_twiddle(idx, 2 * n, &cr[i], &ci[i]);
      wr[i] = cr[i]; wi[i] = -ci[i];
      if (i) { wr[M - i] = cr[i]; wi[M - i] = -ci[i]; }
    }
    host_fft_pow2(wr, wi, false);
    const double sgn = inverse ? -1.0 : 1.0;
    std::vector<V> chirp(L, mk<T>(0, 0)), wm(L), wce(L), wco(L);
    for (long i = 0; i < L; ++i) {
      if (i < n) chirp[i] = mk<T>((T)cr[i], (T)(sgn * ci[i]));
      double re, im;
      host_twiddle(i, M, &re, &im);
      wm[i] = mk<T>((T)re, (T)im);
      wce[i] = mk<T>((T)wr[2 * i], (T)(-sgn * wi[2 * i]));
      wco[i] = mk<T>((T)wr[2 * i + 1], (T)(-sgn * wi[2 * i + 1]));
    }
    auto twa = make_twa<T>(R, R);
    std::vector<V> x((size_t)n * batch), out((size_t)n * batch);
    fill<T>(x, 31 + inverse);
    typename Body::Args a = {x.data(), out.data(), twa.data(), chirp.data(), wm.data(), wce.data(), wco.data(), n, batch,
                             (T)(1.0 / M)};
    std::vector<V> exch(Cfg::Tile::template smem_elems<typename Cfg::Lay>());
    std::vector<V> stash((size_t)E * Cfg::THREADS);
    struct Keep { V v[E]; };
    std::vector<Keep> keep(Cfg::THREADS);
    std::vector<typename Cfg::Tile> thr(Cfg::THREADS);
    const long groups = (batch + Cfg::C - 1) / Cfg::C;
    auto all = [&](auto fn) { for (int t = 0; t < Cfg::THREADS; ++t) fn(t); };
    for (long g = 0; g < groups; ++g) {
      auto bidx = [&](int t) { long b = g * Cfg::C + Cfg::Tile::template col_of<true>(t); return b; };
      auto bcl = [&](int t) { long b = bidx(t); return b < batch ? b : batch - 1; };
      for (int odd = 0; odd < 2; ++odd) {
        all([&](int t) { if (odd) Body::template load_half<true>(thr[t], a, bcl(t), t, exch.data(), twa.data(), chirp.data(), wm.data());
                         else Body::template load_half<false>(thr[t], a, bcl(t), t, exch.data(), twa.data(), chirp.data(), wm.data()); });
        all([&](int t) { Body::middle(thr[t], t, exch.data(), odd ? wco.data() : wce.data()); });
        all([&](int t) { Body::second_fft_start(thr[t], t, exch.data(), twa.data()); });
        all([&](int t) { Body::second_fft_finish(thr[t], t, exch.data()); });
        if (!odd) all([&](int t) {
          if constexpr (K::LOCAL_STASH) { for (int i = 0; i < E; ++i) keep[t].v[i] = thr[t].v[i]; }
          else Body::stash_even(thr[t], t, stash.data());
        });
      }
      all([&](int t) {
        if (bidx(t) >= batch) return;
        if constexpr (K::LOCAL_STASH) Body::combine_store_local(keep[t].v, thr[t], a, bcl(t), t, chirp.data(), wm.data());
        else Body::combine_store(stash.data(), thr[t], a, bcl(t), t, chirp.data(), wm.data());
      });
    }
    double worst = 0;
    for (long b = 0; b < batch; ++b) {
      double mr = 0, me = 0;
      for (long k = 0; k < n; ++k) {
        double sr = 0, si = 0;
        for (long j = 0; j < n; ++j) {
          double re, im;
          host_twiddle((size_t)((k * j) % n), (size_t)n, &re, &im);
          if (inverse) im = -im;
          sr += x[b * n + j].x * re - x[b * n + j].y * im;
          si += x[b * n + j].x * im + x[b * n + j].y * re;
        }
        mr = std::max(mr, std::hypot(sr, si));
        me = std::max(me, std::hypot(out[b * n + k].x - sr, out[b * n + k].y - si));
      }
      worst = std::max(worst, me / mr);
    }
    printf("%s N=%ld (L=%ld) %s: %d warps, %s stash, max rel err vs naive f64 DFT %.3e %s\n", name, n, L,
           inverse ? "inverse" : "forward", Cfg::THREADS / 32, K::LOCAL_STASH ? "per-thread" : "shared", worst,
           worst < tol ? "OK" : "FAIL");
    bad += !(worst < tol);
  }
  return bad;
}

// ---- persistent kernel: the consumer arithmetic (fused::FusedMath) with the producer / TMA side replaced by
// plain copies: staging = what the TMA box (pass 1) or the bulk copy (pass 2) would deliver --------------------------
template <class Cfg>
static int check_fused(const char* name, double tol) {
  using T = typename Cfg::T;
  using V = cpx<T>;
  constexpr long N = Cfg::N, N1 = Cfg::N1, N2 = Cfg::N2;
  constexpr int C = Cfg::C, C1 = Cfg::C1, GT = Cfg::GT;
  printf("%s: persistent-kernel arithmetic, N=%ld = %ld x %ld, blocked intermediate%s\n", name, N, N1, N2, Cfg::DIRECT ? ", direct loads" : "");
  report_conflicts<typename Cfg::template Tile1<true>, typename Cfg::Lay1, kMapCF>("pass 1");
  report_conflicts<typename Cfg::template Tile2<true>, typename Cfg::Lay2, fused::FusedMath<Cfg, true>::kMap2>("pass 2");
  {  // staging reads of pass 2 (the other staging / table reads are contiguous by construction)
    using Tile = typename Cfg::template Tile2<true>;
    int worst = 1;
    for (int warp = 0; warp < GT / 32; ++warp)
      for (int i = 0; i < Tile::RA; ++i) {
        std::vector<long> idx;
        for (int l = 0; l < 32; ++l) {
          const int t = warp * 32 + l;
          constexpr int M = fused::FusedMath<Cfg, true>::kMap2;
          const long u = Tile::template u_of<M>(t), col = Tile::template col_of<M>(t), n = u + (long)Tile::RB * i;
          idx.push_back((n / 8) * 64 + col * 8 + n % 8);
        }
        worst = std::max(worst, conflict_degree<(int)sizeof(V)>(idx));
      }
    printf("  pass 2 staging reads: conflicts x%d %s\n", worst, worst == 1 ? "" : "FAIL");
    if (worst != 1) return 1;
  }
  {  // LSU cost model of the two accesses the blocked layout changes: 128-byte lines touched by one warp-wide
     // pass-1 store, and different stage twiddles one warp loads in pass 2 (identical addresses broadcast)
    using Tile = typename Cfg::template Tile1<true>;
    using TileB = typename Cfg::template Tile2<true>;
    constexpr int M = fused::FusedMath<Cfg, true>::kMap2;
    long lines = 0, twiddles = 0;
    for (int warp = 0; warp < GT / 32; ++warp) {
      std::vector<long> seen_l, seen_t;
      for (int l = 0; l < 32; ++l) {
        const int t = warp * 32 + l;
        const long col = Tile::template col_of<kMapCF>(t), p = Tile::template u_of<kMapCF>(t);
        const long e = (p >> 3) * (N2 * 8) + (col >> 3) * 64 + (p & 7) * 8 + (col & 7);   // output r = 0
        const long line = e * (long)sizeof(V) / 128, tw = TileB::template u_of<M>(t);
        if (std::find(seen_l.begin(), seen_l.end(), line) == seen_l.end()) seen_l.push_back(line);
        if (std::find(seen_t.begin(), seen_t.end(), tw) == seen_t.end()) seen_t.push_back(tw);
      }
      lines += (long)seen_l.size();
      twiddles += (long)seen_t.size();
    }
    printf("  per warp: %.1f lines of 128 B per pass-1 store instruction (%d B stored), %.1f different pass-2 stage twiddles\n",
           (double)lines / (GT / 32), 32 * (int)sizeof(V), (double)twiddles / (GT / 32));
  }
  auto twa_pairs = make_twa<T>(Cfg::RA, Cfg::RB), twa2_pairs = make_twa<T>(Cfg::RA2, Cfg::RB2);
  std::vector<TwPair<T>> twa(twa_pairs.size()), twa2(twa2_pairs.size());     // the kernel re-lays the tables out in 8-byte planes
  for (int i = 0; i < (int)twa_pairs.size(); ++i) fused::FusedMath<Cfg, true>::relayout_twa(twa.data(), twa_pairs.data(), i, (int)twa_pairs.size());
  for (int i = 0; i < (int)twa2_pairs.size(); ++i) fused::FusedMath<Cfg, true>::relayout_twa(twa2.data(), twa2_pairs.data(), i, (int)twa2_pairs.size());
  std::vector<V> tbase, tstep;
  make_factored_twiddles<T>((size_t)N, (size_t)N2, Cfg::RA, Cfg::RB, C1, tbase, tstep, true);
  int bad = 0;
  for (int fwd = 1; fwd >= 0; --fwd) {
    std::vector<V> x(N), scratch(N), out(N), staging(std::max((size_t)C1 * N1, (size_t)C * N2)), tab((size_t)Cfg::TAB_ELEMS);
    std::vector<V> exch(Cfg::EX_ELEMS);
    fill<T>(x, 41 + fwd);
    const T scale = (T)0.5;
    auto run_tile = [&](auto fwd_tag, auto pass_tag, int tile) {
      constexpr bool FWD = decltype(fwd_tag)::value;
      constexpr int PASS = decltype(pass_tag)::value;
      using Math = fused::FusedMath<Cfg, FWD>;
      using P = typename Math::template Pass<PASS>;
      std::vector<typename P::Tile> thr(GT);
      // direct mode: the threads read global memory themselves (same pointers as the kernel computes)
      const V* src = !Cfg::DIRECT ? staging.data() : PASS == 1 ? x.data() + (size_t)tile * C1
                                                                : scratch.data() + (size_t)tile * C * N2;
      for (int t = 0; t < GT; ++t) { P::load(thr[t], t, src); P::stage_a(thr[t], t, PASS == 1 ? twa.data() : twa2.data()); }
      for (int t = 0; t < GT; ++t) P::scatter(thr[t], t, exch.data());
      for (int t = 0; t < GT; ++t) {
        P::gather(thr[t], t, exch.data());
        thr[t].stage_b();
        if constexpr (PASS == 1) Math::store1(thr[t], t, scratch.data(), tile, tab.data(), tab.data() + Cfg::TAB_BASE);
        else Math::store2(thr[t], t, out.data(), tile, true, scale);
      }
    };
    using One = std::integral_constant<int, 1>;
    using Two = std::integral_constant<int, 2>;
    for (int tile = 0; tile < Cfg::T1; ++tile) {        // pass 1: TMA box = rows n1, columns tile*C .. +C
      for (long r = 0; r < N1; ++r)
        for (int c = 0; c < C1; ++c) staging[r * C1 + c] = x[r * N2 + (long)tile * C1 + c];
      for (int i = 0; i < Cfg::TAB_BASE; ++i) tab[i] = tbase[(size_t)tile * Cfg::TAB_BASE + i];
      for (int i = 0; i < Cfg::TAB_STEP; ++i) tab[Cfg::TAB_BASE + i] = tstep[(size_t)tile * Cfg::TAB_STEP + i];
      if (fwd) run_tile(std::true_type{}, One{}, tile); else run_tile(std::false_type{}, One{}, tile);
    }
    for (int tile = 0; tile < Cfg::T2; ++tile) {        // pass 2: bulk copy of C*N2 contiguous samples
      for (long i = 0; i < (long)C * N2; ++i) staging[i] = scratch[(size_t)tile * C * N2 + i];
      if (fwd) run_tile(std::true_type{}, Two{}, tile); else run_tile(std::false_type{}, Two{}, tile);
    }
    std::vector<double> re(N), im(N);
    for (long i = 0; i < N; ++i) { re[i] = x[i].x; im[i] = x[i].y; }
    host_fft_pow2(re, im, !fwd);
    double maxref = 0, maxerr = 0;
    for (long i = 0; i < N; ++i) {
      maxref = std::max(maxref, std::hypot(re[i], im[i]) * 0.5);
      maxerr = std::max(maxerr, std::hypot(out[i].x - 0.5 * re[i], out[i].y - 0.5 * im[i]));
    }
    printf("  %s: max rel err vs f64 FFT %.3e (tol %.1e) %s\n", fwd ? "forward" : "inverse", maxerr / maxref, tol,
           maxerr / maxref < tol ? "OK" : "FAIL");
    bad += !(maxerr / maxref < tol);
  }
  return bad;
}

// ---- work queue of the fused kernel: order and dependency properties ---------------------------------------------
// One queue (T1 pass-1 and T2 pass-2 tiles per transform, `batch` transforms, ring / lag as launched): every tile
// appears exactly once; pass 2 of b comes after all pass-1 tiles of b; pass 1 of b + ring comes after all pass-2
// tiles of b (the slot is free); and in the steady state both gaps of DESIGN.md 4.2 hold exactly.  `gaps` counts the
// steady-state gaps checked.
static bool check_queue_order(int t1, int t2, int batch, int ring, int lag, long* gaps) {
  const long total = (long)batch * (t1 + t2);
  std::vector<long> pos1((size_t)batch * t1, -1), pos2((size_t)batch * t2, -1);
  for (long w = 0; w < total; ++w) {
    const fused::WorkItem it = fused::decode_work(w, batch, lag, t1, t2);
    if (it.pass == 1 && it.b >= 0 && it.b < batch && it.tile >= 0 && it.tile < t1 && pos1[(size_t)it.b * t1 + it.tile] < 0)
      pos1[(size_t)it.b * t1 + it.tile] = w;
    else if (it.pass == 2 && it.b >= 0 && it.b < batch && it.tile >= 0 && it.tile < t2 && pos2[(size_t)it.b * t2 + it.tile] < 0)
      pos2[(size_t)it.b * t2 + it.tile] = w;
    else return false;   // out of range or duplicate (so, with `total` items, some tile is missing)
  }
  if (fused::decode_work(total, batch, lag, t1, t2).pass >= 0) return false;   // exhausted marker
  std::vector<long> first1(batch), last1(batch), first2(batch), last2(batch);
  for (int b = 0; b < batch; ++b) {
    first1[b] = *std::min_element(pos1.begin() + (size_t)b * t1, pos1.begin() + (size_t)(b + 1) * t1);
    last1[b] = *std::max_element(pos1.begin() + (size_t)b * t1, pos1.begin() + (size_t)(b + 1) * t1);
    first2[b] = *std::min_element(pos2.begin() + (size_t)b * t2, pos2.begin() + (size_t)(b + 1) * t2);
    last2[b] = *std::max_element(pos2.begin() + (size_t)b * t2, pos2.begin() + (size_t)(b + 1) * t2);
  }
  for (int b = 0; b < batch; ++b) {
    if (!(last1[b] < first2[b])) return false;                          // pass 2 of b only depends on earlier items
    if (b >= ring && !(last2[b - ring] < first1[b])) return false;      // slot reuse: pass 1 of b after pass 2 of b-ring
    if (b >= lag && b + lag < batch) {                                  // steady state: pass-2 gap
      if (first2[b] - last1[b] != (long)lag * (t1 + t2) + 1) return false;
      ++*gaps;
    }
    if (b >= ring) {                                                    // steady state: slot-reuse gap
      if (first1[b] - last2[b - ring] != (long)(ring - lag - 1) * (t1 + t2) + 1) return false;
      ++*gaps;
    }
  }
  return true;
}

// The queue of one persistent configuration (fused_configs.cuh: the library's table): its (T1, T2) at its default
// ring / lag and at rings 2, 3, 5 and 24 with every lag, over a range of batches, and the ring / lag the launch
// actually uses (fused::launch_ring, the rule the library runs) for every batch 1 .. 3 x ring.  With pair items
// (PairCfg) the queue holds T1 / 2 and T2 / 2 items per transform, two tiles each.
template <class Conf>
static int check_queue(const char* name) {
  using Cfg = typename Conf::Cfg;
  constexpr int t1 = Cfg::PAIR ? Cfg::T1 / 2 : Cfg::T1, t2 = Cfg::PAIR ? Cfg::T2 / 2 : Cfg::T2;
  const int ring0 = Conf::RING, lag0 = Conf::LAG;
  int layouts = 0, bad = 0;
  long gaps = 0;
  auto one = [&](int batch, int ring, int lag) {
    ++layouts;
    if (!check_queue_order(t1, t2, batch, ring, lag, &gaps)) {
      printf("  queue order FAILED %s T1=%d T2=%d batch=%d ring=%d lag=%d\n", name, t1, t2, batch, ring, lag);
      ++bad;
    }
  };
  std::vector<std::pair<int, int>> rings = {{ring0, lag0}};
  for (int ring : {2, 3, 5, 24})
    for (int lag = 1; lag < ring; ++lag) rings.push_back({ring, lag});
  for (auto rl : rings)
    for (int batch : {1, 2, 3, rl.second, rl.second + 1, rl.first, rl.first + 1, 2 * rl.first + rl.second + 3})
      one(batch, rl.first, rl.second);
  int shrunk = 0;
  for (int batch = 1; batch <= 3 * ring0; ++batch) {
    const fused::RingLag rl = fused::launch_ring(ring0, lag0, batch);
    const bool ok = rl.ring >= 2 && rl.ring <= ring0 && rl.lag >= 1 && rl.lag < rl.ring &&
                    (rl.ring == ring0 || rl.ring >= batch);   // a shrunk ring holds the whole batch
    if (!ok) { printf("  ring shrink FAILED %s batch=%d: ring %d lag %d\n", name, batch, rl.ring, rl.lag); ++bad; }
    shrunk += rl.ring < ring0;
    one(batch, rl.ring, rl.lag);
  }
  printf("fused work queue %s%s (T1 %d, T2 %d; ring %d, lag %d; rings 2, 3, 5, 24; launch rings of batches 1..%d, %d "
         "shrunk): %d layouts, %ld steady-state gaps, permutation / dependency-order / gap properties %s\n",
         name, Cfg::PAIR ? ", pair items" : "", t1, t2, ring0, lag0, 3 * ring0, shrunk, layouts, gaps, bad ? "FAILED" : "OK");
  return bad;
}

// ---- CTA-level shared-memory Stockham kernel (cta_kernels.cuh): every step for every thread, barrier = loop end ----
template <typename T>
static int check_cta(const char* name, int n, bool chirp_mode, double tol) {
  using V = cpx<T>;
  int len = n;
  if (chirp_mode) { len = 1; while (len < 2 * n - 1) len *= 2; }
  cta::Args<T> a;
  if (!cta::factorize((size_t)len, a.st)) { printf("%s N=%d: cannot factorize\n", name, n); return 1; }
  const int group = std::max(1, (int)(32768 / sizeof(V)) / len), batch = group + 1;   // a full and a partial group
  std::vector<V> wtab = cta::make_stage_twiddles<T>((size_t)len, a.st, host_twiddle);
  std::vector<V> chirp(n), wf(len), x((size_t)batch * n), out((size_t)batch * n);
  if (chirp_mode) {
    std::vector<double> wr(len, 0.0), wi(len, 0.0);
    for (int i = 0; i < n; ++i) {
      double re, im;
      host_twiddle((size_t)(((unsigned long long)i * i) % (2ull * n)), 2 * (size_t)n, &re, &im);
      chirp[i] = mk<T>((T)re, (T)im);
      wr[i] = re; wi[i] = -im;
      if (i) { wr[len - i] = re; wi[len - i] = -im; }
    }
    host_fft_pow2(wr, wi, false);
    for (int i = 0; i < len; ++i) wf[i] = mk<T>((T)wr[i], (T)wi[i]);
  }
  fill<T>(x, 77 + n);
  a.in = x.data(); a.out = out.data(); a.wtab = wtab.data(); a.chirp = chirp.data(); a.wf = wf.data();
  a.batch = batch; a.n = n; a.len = len; a.group = group; a.pad = a.st.radix[0] % 2 == 0 ? 1 : 0;
  printf("%s N=%d%s: on-chip length %d, stages", name, n, chirp_mode ? " (chirp-z)" : "", len);
  for (int i = 0; i < a.st.count; ++i) printf(" %d", a.st.radix[i]);
  printf(", %d transforms per CTA iteration\n", group);
  // bank conflicts of the shared-memory accesses, worst warp-wide instruction per stage
  {
    int sub = len, stride = 1;
    for (int sidx = 0; sidx < a.st.count; ++sidx) {
      const int R = a.st.radix[sidx], per = len / R, m = sub / R;
      int worst_r = 1, worst_w = 1;
      for (int warp = 0; warp < std::min(cta::kThreads, group * per) / 32; ++warp)
        for (int k = 0; k < R; ++k) {
          std::vector<long> ri, wi2;
          for (int l = 0; l < 32; ++l) {
            const int g = warp * 32 + l, tl = g / per, q = g - tl * per, i = q / stride, j = q - i * stride;
            const int er = tl * len + (k * m + i) * stride + j, ew = tl * len + (i * R + k) * stride + j;
            ri.push_back(a.pad ? cta::padded(er) : er);
            wi2.push_back(a.pad ? cta::padded(ew) : ew);
          }
          worst_r = std::max(worst_r, conflict_degree<(int)sizeof(V)>(ri));
          worst_w = std::max(worst_w, conflict_degree<(int)sizeof(V)>(wi2));
        }
      printf("  stage %d (radix %2d, stride %5d): shared read conflicts x%d, write x%d\n", sidx, R, stride, worst_r, worst_w);
      sub /= R; stride *= R;
    }
  }
  int bad = 0;
  std::vector<V> buf0((size_t)cta::padded(group * len) + 1), buf1(buf0.size());
  for (int dir = 1; dir >= 0; --dir) {
    a.scale = (T)(chirp_mode ? 0.5 / len : 0.5);
    for (long first = 0; first < batch; first += group) {
      const int cnt = (int)std::min<long>(group, batch - first);
      auto run = [&](auto D, auto Cm) {
        using P = cta::Program<T, decltype(D)::value, decltype(Cm)::value>;
        for (int st = 0; st < P::steps(a); ++st)
          for (int tid = 0; tid < cta::kThreads; ++tid) P::step(a, st, tid, cta::kThreads, first, cnt, buf0.data(), buf1.data());
      };
      if (dir && chirp_mode) run(std::true_type{}, std::true_type{});
      else if (dir) run(std::true_type{}, std::false_type{});
      else if (chirp_mode) run(std::false_type{}, std::true_type{});
      else run(std::false_type{}, std::false_type{});
    }
    double worst = 0;
    for (int b = 0; b < batch; ++b) {
      double me = 0, mr = 0;
      for (int k = 0; k < n; ++k) {
        double sr = 0, si = 0;
        for (int j = 0; j < n; ++j) {
          double re, im;
          host_twiddle((size_t)(((unsigned long long)j * k) % n), (size_t)n, &re, &im);
          if (!dir) im = -im;
          const double xr = x[(size_t)b * n + j].x, xi = x[(size_t)b * n + j].y;
          sr += xr * re - xi * im; si += xr * im + xi * re;
        }
        sr *= 0.5; si *= 0.5;
        me = std::max(me, std::hypot(out[(size_t)b * n + k].x - sr, out[(size_t)b * n + k].y - si));
        mr = std::max(mr, std::hypot(sr, si));
      }
      worst = std::max(worst, me / mr);
    }
    printf("  %s: max rel err vs naive f64 DFT %.3e %s\n", dir ? "forward" : "inverse", worst, worst < tol ? "OK" : "FAIL");
    bad += !(worst < tol);
  }
  return bad;
}

// ---- row FFTs with the exchange folded into the store of pass 2 (dist_kernels.cuh) -----------------------------
// pass 1 of the configuration as it is, then RowsExchangeBody with P destination buffers in host memory; reference:
// dst_q[c * out_ld + out_off + r] = FFT(row r)[q * cb + c] * w_Ntot^{(row0 + r) * (q * cb + c)}
// WIDE: the tile of twice as many transforms that dist_fft.cu also uses, else the configuration's pass-2 tile
// (dist::ExchangeShape)
template <typename T, class Cfg, int TW, bool WIDE>
static int check_rows_exchange(const char* name, int P, double tol) {
  using SW = dist::ExchangeShape<Cfg, WIDE, T>;
  constexpr bool FWD = TW != 2;
  const long N = Cfg::N, N1 = Cfg::N1, N2 = Cfg::N2;
  using Tile = TileFFT<T, SW::RA, SW::RB, SW::E, SW::C, FWD>;
  using LayX = ExLayout<SW::RA * SW::C + SW::PAD, SW::C, 1>;
  report_conflicts<Tile, LayX, true>("exchange tile");
  using Body = dist::RowsExchangeBody<Tile, LayX, Cfg::N1, Cfg::N2, TW>;
  const long rows = 2 * Tile::C, cb = N / P;
  const unsigned long long row0 = 12345, n_total = (unsigned long long)N * 4096, out_off = 3 * rows, out_ld = 5 * rows;
  std::vector<cpx<T>> x((size_t)N * rows), scratch((size_t)N * rows);
  fill<T>(x, 21 + TW);
  const auto* ops = Cfg::ops();
  auto twa1 = make_twa<T>(ops->ra1, ops->rb1), twa2 = make_twa<T>(ops->ra2, ops->rb2);
  std::vector<cpx<T>> tw2(N);
  for (long k1 = 0; k1 < N1; ++k1)
    for (long c = 0; c < N2; ++c) {
      double re, im;
      host_twiddle((size_t)(k1 * c), (size_t)N, &re, &im);
      tw2[k1 * N2 + c] = mk<T>((T)re, (T)im);
    }
  run_body<typename Cfg::template Body1<FWD>, typename Cfg::template Tile1<FWD>, typename Cfg::Lay1>(
      Cfg::template args1<FWD>(x.data(), scratch.data(), twa1.data(), tw2.data()), rows * (N2 / Cfg::template Tile1<FWD>::C));
  std::vector<std::vector<cpx<T>>> dst(P, std::vector<cpx<T>>((size_t)cb * out_ld, mk<T>((T)777, (T)777)));
  typename Body::Args a;
  a.scratch = scratch.data(); a.twa = twa2.data();
  for (int q = 0; q < kMaxPeers; ++q) a.outs.p[q] = q < P ? dst[q].data() : nullptr;
  a.out_ld = out_ld; a.out_off = out_off; a.row0 = row0; a.n_total = n_total; a.groups = (unsigned)(rows / Tile::C);
  a.r0 = 0; a.out_bs = 0; a.rb_shift = 63; a.rpb = 0; a.rows_valid = ~0ull;
  a.cb_shift = 0;
  while ((1L << a.cb_shift) < cb) ++a.cb_shift;
  run_body<Body, Tile, LayX>(a, (long)a.groups * N1);
  double worst = 0, maxref = 0;
  for (long r = 0; r < rows; ++r) {
    std::vector<double> re(N), im(N);
    for (long i = 0; i < N; ++i) { re[i] = x[(size_t)r * N + i].x; im[i] = x[(size_t)r * N + i].y; }
    host_fft_pow2(re, im, !FWD);
    for (long k = 0; k < N; ++k) {
      double wr = 1, wi = 0;
      if (TW) {
        const unsigned long long m = (row0 + r) * (unsigned long long)k % n_total;
        const double ang = 2 * M_PI * (double)m / (double)n_total;
        wr = std::cos(ang); wi = TW == 1 ? -std::sin(ang) : std::sin(ang);
      }
      const double rr = re[k] * wr - im[k] * wi, ii = re[k] * wi + im[k] * wr;
      const cpx<T> got = dst[k / cb][(size_t)(k % cb) * out_ld + out_off + r];
      maxref = std::max(maxref, std::hypot(rr, ii));
      worst = std::max(worst, std::hypot(got.x - rr, got.y - ii));
    }
  }
  // nothing outside the chunk's columns may be written
  long stray = 0;
  for (int q = 0; q < P; ++q)
    for (long c = 0; c < cb; ++c)
      for (long j = 0; j < (long)out_ld; ++j)
        if ((j < (long)out_off || j >= (long)out_off + rows) && dst[q][(size_t)c * out_ld + j].x != (T)777) ++stray;
  const double rel = worst / maxref;
  printf("%s rows+exchange (P=%d, twiddle %d): max rel err %.3e (tol %.1e), stray stores %ld %s\n", name, P, TW, rel, tol, stray,
         rel < tol && stray == 0 ? "OK" : "FAIL");
  return !(rel < tol && stray == 0);
}

// ---- three-pass path (bigpow2.cu): outer column pass + two-pass rows with the transposed store ---------------------
// Col: the outer pass (outer::visit_column), Cfg: the two-pass configuration of the rows
template <typename T, class Col, class Cfg, bool FWD>
static int check_threepass(const char* name, double tol) {
  using SO = typename Col::Shape;
  const long Na = SO::L, Nb = Cfg::N, N = Na * Nb;
  using TileO = typename Col::template Tile<FWD>;
  using LayO = typename Col::Lay;
  using BodyO = typename Col::template Body<FWD>;
  const long B = 2;   // two long transforms in one call
  std::vector<cpx<T>> x(B * N), work(B * N), scratch(B * N), out(B * N);
  fill<T>(x, 31 + FWD);
  auto twao = make_twa<T>(SO::RA, SO::RB);
  typename BodyO::Args ao;
  ao.in = x.data(); ao.out = work.data(); ao.twa = twao.data(); ao.nb = Nb; ao.n_total = N; ao.tiles = (unsigned)(Nb / SO::C);
  ao.scale = (T)0.5;
  run_body<BodyO, TileO, LayO>(ao, B * (Nb / SO::C));
  const auto* ops = Cfg::ops();
  auto twa1 = make_twa<T>(ops->ra1, ops->rb1), twa2 = make_twa<T>(ops->ra2, ops->rb2);
  std::vector<cpx<T>> tw2(Nb);
  for (long k1 = 0; k1 < Cfg::N1; ++k1)
    for (long c = 0; c < Cfg::N2; ++c) {
      double re, im;
      host_twiddle((size_t)(k1 * c), (size_t)Nb, &re, &im);
      tw2[k1 * Cfg::N2 + c] = mk<T>((T)re, (T)im);
    }
  run_body<typename Cfg::template Body1<FWD>, typename Cfg::template Tile1<FWD>, typename Cfg::Lay1>(
      Cfg::template args1<FWD>(work.data(), scratch.data(), twa1.data(), tw2.data()), B * Na * (Cfg::N2 / Cfg::template Tile1<FWD>::C));
  using Tile = typename Cfg::template Tile2<FWD>;
  using Body = dist::RowsExchangeBody<Tile, typename Cfg::Lay2, Cfg::N1, Cfg::N2, 0>;
  typename Body::Args a;
  a.scratch = scratch.data(); a.twa = twa2.data();
  for (int q = 0; q < kMaxPeers; ++q) a.outs.p[q] = q == 0 ? out.data() : nullptr;
  a.out_ld = Na; a.out_off = 0; a.row0 = 0; a.n_total = 0; a.groups = (unsigned)(B * Na / Tile::C);
  a.r0 = 0; a.out_bs = N; a.rb_shift = 0; a.rpb = 0; a.rows_valid = ~0ull;
  while ((1L << a.rb_shift) < Na) ++a.rb_shift;
  a.cb_shift = 0;
  while ((1L << a.cb_shift) < Nb) ++a.cb_shift;
  run_body<Body, Tile, typename Cfg::Lay2>(a, (long)a.groups * Cfg::N1);
  double maxref = 0, maxerr = 0;
  for (long bb = 0; bb < B; ++bb) {
    std::vector<double> re(N), im(N);
    for (long i = 0; i < N; ++i) { re[i] = x[bb * N + i].x; im[i] = x[bb * N + i].y; }
    host_fft_pow2(re, im, !FWD);
    for (long i = 0; i < N; ++i) {
      maxref = std::max(maxref, std::hypot(re[i] * 0.5, im[i] * 0.5));
      maxerr = std::max(maxerr, std::hypot(out[bb * N + i].x - re[i] * 0.5, out[bb * N + i].y - im[i] * 0.5));
    }
  }
  printf("%s three-pass %ld x %ld (%s): max rel err %.3e (tol %.1e) %s\n", name, Na, Nb, FWD ? "forward" : "inverse",
         maxerr / maxref, tol, maxerr / maxref < tol ? "OK" : "FAIL");
  return !(maxerr / maxref < tol);
}

// ---- three-pass path with an outer radix-3 / 9 / 27 pass (N = 3^b * 2^k, bigpow2.cu) ---------------------------------
template <typename T, int B, class Cfg, bool FWD>
static int check_threepass_radix3(const char* name, double tol) {
  const long Nb = Cfg::N, N = B * Nb, BATCH = 2;
  using Tile = typename Cfg::template Tile2<FWD>;
  const long rows = BATCH * B, rows_pad = (rows + Tile::C - 1) / Tile::C * Tile::C;
  std::vector<cpx<T>> x(BATCH * N), work(rows_pad * Nb, mk<T>((T)NAN, (T)NAN)), scratch(rows_pad * Nb), out(BATCH * N, mk<T>((T)777, (T)777));
  fill<T>(x, 41 + B);
  using BodyO = outer::Radix3ColumnBody<T, B, FWD>;
  typename BodyO::Args ao;
  ao.in = x.data(); ao.out = work.data(); ao.nb = Nb; ao.n_total = N; ao.count = BATCH * Nb; ao.scale = (T)0.5;
  for (long i = 0; i < BATCH * Nb + 7; ++i) BodyO::run(ao, i);          // a few threads beyond the end, as the grid has
  const auto* ops = Cfg::ops();
  auto twa1 = make_twa<T>(ops->ra1, ops->rb1), twa2 = make_twa<T>(ops->ra2, ops->rb2);
  std::vector<cpx<T>> tw2(Nb);
  for (long k1 = 0; k1 < Cfg::N1; ++k1)
    for (long c = 0; c < Cfg::N2; ++c) {
      double re, im;
      host_twiddle((size_t)(k1 * c), (size_t)Nb, &re, &im);
      tw2[k1 * Cfg::N2 + c] = mk<T>((T)re, (T)im);
    }
  run_body<typename Cfg::template Body1<FWD>, typename Cfg::template Tile1<FWD>, typename Cfg::Lay1>(
      Cfg::template args1<FWD>(work.data(), scratch.data(), twa1.data(), tw2.data()), rows_pad * (Cfg::N2 / Cfg::template Tile1<FWD>::C));
  using Body = dist::RowsExchangeBody<Tile, typename Cfg::Lay2, Cfg::N1, Cfg::N2, 0>;
  typename Body::Args a;
  a.scratch = scratch.data(); a.twa = twa2.data();
  for (int q = 0; q < kMaxPeers; ++q) a.outs.p[q] = q == 0 ? out.data() : nullptr;
  a.out_ld = B; a.out_off = 0; a.row0 = 0; a.n_total = 0; a.groups = (unsigned)(rows_pad / Tile::C);
  a.r0 = 0; a.out_bs = N; a.rb_shift = 63; a.rpb = B; a.rows_valid = rows;
  a.cb_shift = 0;
  while ((1L << a.cb_shift) < Nb) ++a.cb_shift;
  run_body<Body, Tile, typename Cfg::Lay2>(a, (long)a.groups * Cfg::N1);
  double maxref = 0, maxerr = 0;
  for (long bb = 0; bb < BATCH; ++bb) {                                   // naive DFT of a few outputs + an FFT-free check
    std::vector<double> re(N), im(N);
    for (long i = 0; i < N; ++i) { re[i] = x[bb * N + i].x; im[i] = x[bb * N + i].y; }
    for (long k = 0; k < N; k += (k < 40 ? 1 : N / 97 + 1)) {
      double sr = 0, si = 0;
      for (long n = 0; n < N; ++n) {
        const double ang = (FWD ? -2.0 : 2.0) * M_PI * (double)((k * n) % N) / (double)N;
        sr += re[n] * std::cos(ang) - im[n] * std::sin(ang);
        si += re[n] * std::sin(ang) + im[n] * std::cos(ang);
      }
      maxref = std::max(maxref, std::hypot(sr * 0.5, si * 0.5));
      maxerr = std::max(maxerr, std::hypot(out[bb * N + k].x - sr * 0.5, out[bb * N + k].y - si * 0.5));
    }
  }
  long untouched = 0, nans = 0;
  for (auto& v : out) { untouched += v.x == (T)777; nans += std::isnan(v.x); }
  printf("%s three-pass %d x %ld (%s): max rel err %.3e (tol %.1e), unwritten %ld, nan %ld %s\n", name, B, Nb, FWD ? "forward" : "inverse",
         maxerr / maxref, tol, untouched, nans, maxerr / maxref < tol && untouched == 0 && nans == 0 ? "OK" : "FAIL");
  return !(maxerr / maxref < tol && untouched == 0 && nans == 0);
}

// ---- the configurations of the library's tables -------------------------------------------------------------------
// f with the two-pass configuration of N = 2^log2n (twopass::visit_config); a size without one is a failure
template <typename T, class F> static int with_config(int log2n, F&& f) {
  int bad = -1;
  visit_config<T>((size_t)1 << log2n, [&](auto g) { bad = f(g); });
  if (bad < 0) printf("%s 2^%d: no two-pass configuration FAIL\n", prec<T>(), log2n);
  return bad < 0 ? 1 : bad;
}

// every two-pass configuration
template <typename T> static int check_twopass(double tol) {
  int bad = 0;
  for (int k = 1; k <= 30; ++k)
    visit_config<T>((size_t)1 << k, [&](auto g) {
      char name[32];
      snprintf(name, sizeof name, "%s 2^%d", prec<T>(), k);
      bad += check<T, decltype(g)>(name, tol);
    });
  return bad;
}

template <typename T, int TW, bool WIDE = false> static int rows_exchange(int log2n, int P, double tol) {
  char name[32];
  snprintf(name, sizeof name, "%s 2^%d%s", prec<T>(), log2n, WIDE ? " wide" : "");
  return with_config<T>(log2n, [&](auto g) { return check_rows_exchange<T, decltype(g), TW, WIDE>(name, P, tol); });
}

// the outer pass of every length (outer::visit_column), both directions, before rows of N = 2^log2nb
template <typename T> static int threepass(int log2nb, double tol) {
  int bad = 0;
  for (int a = 1; a <= 30; ++a)
    outer::visit_column<T>(a, [&](auto col) {
      char name[32];
      snprintf(name, sizeof name, "%s 2^%d", prec<T>(), a + log2nb);
      bad += with_config<T>(log2nb, [&](auto g) {
        return check_threepass<T, decltype(col), decltype(g), true>(name, tol) +
               check_threepass<T, decltype(col), decltype(g), false>(name, tol);
      });
    });
  return bad;
}

template <typename T, int B, bool FWD> static int threepass_radix3(int log2nb, double tol) {
  char name[32];
  snprintf(name, sizeof name, "%s %d*2^%d", prec<T>(), B, log2nb);
  return with_config<T>(log2nb, [&](auto g) { return check_threepass_radix3<T, B, decltype(g), FWD>(name, tol); });
}

// the fused Bluestein kernel of the size class of M = next_pow2(2N - 1) = 2L; a class without one is a failure
template <typename T> static int bluestein(long n, double tol) {
  size_t m = 1;
  while (m < (size_t)(2 * n - 1)) m *= 2;
  int bad = -1;
  onchip::visit_onchip<T>(m / 2, [&](auto k) {
    if constexpr (decltype(k)::kHasBluestein) {
      char name[32];
      snprintf(name, sizeof name, "bluestein %s", prec<T>());
      bad = check_bluestein<decltype(k)>(name, n, tol);
    }
  });
  if (bad < 0) printf("bluestein %s N=%ld: no fused Bluestein class FAIL\n", prec<T>(), n);
  return bad < 0 ? 1 : bad;
}

// the persistent kernel of N = 2^LOG2N (fused_configs.cuh); pair items (PairCfg) change only which tiles a group
// claims, so a paired configuration runs as its Unpaired one
template <typename T, int LOG2N> static int check_persistent(double tol) {
  char name[64];
  snprintf(name, sizeof name, "fused %s 2^%d", prec<T>(), LOG2N);
  return check_fused<typename fused::FusedConfig<T, LOG2N>::Cfg::Unpaired>(name, tol);
}

// the work queue of the default configuration of N = 2^LOG2N, and with pair items also the one item per group that
// FOURIER_B200_PAIR=0 selects
template <typename T, int LOG2N> static int check_queues() {
  using D = fused::FusedConfig<T, LOG2N>;
  char name[64];
  snprintf(name, sizeof name, "%s 2^%d", prec<T>(), LOG2N);
  int bad = check_queue<D>(name);
  if constexpr (D::Cfg::PAIR) {
    struct Single : D { using Cfg = typename D::Cfg::Unpaired; };
    snprintf(name, sizeof name, "%s 2^%d (FOURIER_B200_PAIR=0)", prec<T>(), LOG2N);
    bad += check_queue<Single>(name);
  }
  return bad;
}

int main() {
  int bad = 0;
  bad += threepass_radix3<float, 3, true>(11, 2e-6);
  bad += threepass_radix3<float, 9, false>(11, 2e-6);
  bad += threepass_radix3<float, 27, true>(11, 2e-6);
  bad += threepass_radix3<double, 27, false>(9, 1e-14);
  bad += threepass_radix3<double, 3, true>(9, 1e-14);
  bad += threepass<float>(11, 2e-6);
  bad += threepass<double>(9, 5e-15);
  bad += rows_exchange<float, 1>(11, 4, 2e-6);
  bad += rows_exchange<float, 1>(14, 8, 2e-6);
  bad += rows_exchange<float, 2>(14, 2, 2e-6);
  bad += rows_exchange<float, 0>(15, 8, 2e-6);
  bad += rows_exchange<float, 1>(16, 1, 2e-6);
  bad += rows_exchange<double, 1>(9, 4, 5e-15);
  bad += rows_exchange<double, 2>(12, 16, 5e-15);
  // tiles of twice as many transforms (256-byte store runs)
  bad += rows_exchange<float, 1, true>(14, 8, 2e-6);
  bad += rows_exchange<float, 2, true>(16, 4, 2e-6);
  bad += rows_exchange<double, 1, true>(13, 2, 5e-15);
  bad += rows_exchange<double, 0, true>(16, 8, 5e-15);
  bad += check_cta<float>("cta f32", 243, false, 2e-6);
  bad += check_cta<float>("cta f32", 729, false, 2e-6);
  bad += check_cta<float>("cta f32", 2187, false, 3e-6);
  bad += check_cta<float>("cta f32", 96, false, 2e-6);
  bad += check_cta<float>("cta f32", 1536, false, 2e-6);
  bad += check_cta<float>("cta f32", 2048, false, 2e-6);
  bad += check_cta<float>("cta f32", 6, false, 2e-6);
  bad += check_cta<float>("cta f32", 9, false, 2e-6);
  bad += check_cta<double>("cta f64", 768, false, 5e-15);
  bad += check_cta<double>("cta f64", 81, false, 5e-15);
  bad += check_cta<double>("cta f64", 1458, false, 5e-15);
  bad += check_cta<float>("cta f32", 1418, true, 3e-6);
  bad += check_cta<float>("cta f32", 3125, true, 4e-6);
  bad += check_cta<double>("cta f64", 1009, true, 1e-13);
  bad += check_cta<double>("cta f64", 5, true, 1e-13);
  bad += check_twopass<float>(2e-6);
  bad += check_twopass<double>(5e-15);
  for_each_onchip<float>([&](auto k) { bad += check_onchip<decltype(k)>("onchip f32", 2e-6); });
  for_each_onchip<double>([&](auto k) { bad += check_onchip<decltype(k)>("onchip f64", 5e-15); });
  for (long n : {1009L, 513L, 255L, 37L}) bad += bluestein<float>(n, 3e-6);
  for (long n : {191L, 61L}) bad += bluestein<double>(n, 1e-13);
  fused::for_each_fused_size<float>([&](auto k) { bad += check_persistent<float, decltype(k)::value>(2e-6); });
  fused::for_each_fused_size<double>([&](auto k) { bad += check_persistent<double, decltype(k)::value>(5e-15); });
  fused::for_each_fused_size<float>([&](auto k) { bad += check_queues<float, decltype(k)::value>(); });
  fused::for_each_fused_size<double>([&](auto k) { bad += check_queues<double, decltype(k)::value>(); });
  printf(bad ? "EMULATION FAILED (%d)\n" : "EMULATION OK\n", bad);
  return bad ? 1 : 0;
}
