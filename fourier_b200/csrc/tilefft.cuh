// tilefft.cuh -- the building block of the fused kernels: a tile of C independent length-L FFTs
// (L = RA*RB), E samples per thread in registers, ONE shared-memory exchange.
//
//   stage A:  n = j + RB*i   DFT_RA over i (registers)  ->  Y[j][p], times w_L^{j*p}
//   exchange: Y through shared memory (32x32-style transpose per FFT)
//   stage B:  DFT_RB over j (registers)                 ->  X[p + RA*r]
//
// This replaces RA*RB/8.. passes of the reference's stage loop (radix_R_wide / radix_R_narrow,
// fourier-algorithms/src/autosort/mod.rs:211-284: one full sweep over the array per radix-4/8
// stage) by a single read and a single write of the tile: for L = 1024 the reference streams the
// data 4 times (radices 4,8,8,4), here it is loaded once into registers and stored once.
//
// Thread <-> data mapping.  TP = L/E threads cooperate on one FFT.  A thread owns NA = E/RA stage-A
// butterflies (j = u + TP*a) and NB = E/RB stage-B butterflies (p = u + TP*c).  Which of the two
// tile coordinates runs along the lanes of a warp is chosen per access so that global memory is
// always touched in >= 64..128-byte contiguous pieces:
//   "col fast" (CF): lane -> FFT index inside the tile (used when consecutive FFTs are adjacent in
//                    memory: column tiles of the four-step algorithm)
//   "u fast"   (UF): lane -> position inside one FFT (used when one FFT is contiguous in memory)
//   "block fast" (BF): lane -> (position mod 8, FFT index mod 4), for tiles of 8 FFTs stored in 8 x 8 blocks
//                    [position / 8][FFT][position mod 8] (the blocked intermediate of the persistent kernel):
//                    a warp reads 256 contiguous bytes and only 8 different stage twiddles (broadcast)
// The mapping is a template argument MAP of each access: kMapCF = 0 (false), kMapUF = 1 (true), kMapBF = 2.
//
// Every member is __host__ __device__, so the CPU emulators (tools/emulate*.cu) run the identical code thread by
// thread on the CPU.
//
// Phase protocol.  A kernel body built on these tiles (FftBody, RealBody, ConvBody in onchip_kernels.cuh,
// twopass::TileBody, dist::RowsExchangeBody, outer::ColumnBody) states once what runs between two barriers, and in
// what order:
//   static constexpr int kPhases;
//   template <int P> static FB_HD void phase(Tile& f, const Args& a, long grp, int t, V* smem, const TwPair<T>* twa);
// for P = 0 .. kPhases-1, thread t of group (tile) grp, exchange buffer smem, stage twiddles twa in shared memory (the
// bodies that read theirs from Args ignore it).  The caller puts a barrier between consecutive phases: the device
// drivers below, and the CPU driver of tools/emulate_common.h, which runs each phase for every thread before the next.
#pragma once

#include "cplx.cuh"

namespace fb200 {

// Global store with an L2 eviction hint: 0 = default, 1 = streaming / evict-first (data that is not
// read again: the transform output), 2 = evict-last (data that should stay in L2: the intermediate).
template <int HINT, typename V> FB_HD void st_hint(V* p, const V& v) {
#if defined(__CUDA_ARCH__)
  if constexpr (HINT == 0) {
    *p = v;
  } else if constexpr (sizeof(V) == 8) {
    if constexpr (HINT == 1) {
      asm volatile("st.global.cs.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(v.x), "f"(v.y) : "memory");
    } else {
      asm volatile(
          "{\n\t.reg .b64 pol;\n\tcreatepolicy.fractional.L2::evict_last.b64 pol, 1.0;\n\t"
          "st.global.L2::cache_hint.v2.f32 [%0], {%1, %2}, pol;\n\t}" ::"l"(p), "f"(v.x), "f"(v.y) : "memory");
    }
  } else {
    if constexpr (HINT == 1) {
      asm volatile("st.global.cs.v2.f64 [%0], {%1, %2};" ::"l"(p), "d"(v.x), "d"(v.y) : "memory");
    } else {
      asm volatile(
          "{\n\t.reg .b64 pol;\n\tcreatepolicy.fractional.L2::evict_last.b64 pol, 1.0;\n\t"
          "st.global.L2::cache_hint.v2.f64 [%0], {%1, %2}, pol;\n\t}" ::"l"(p), "d"(v.x), "d"(v.y) : "memory");
    }
  }
#else
  *p = v;
#endif
}

// Global load with a cache hint: 0 = default, 1 = streaming (.cs: read once, evict first), 2 = L2 only (.cg:
// data other SMs rewrite during the kernel must not be served from a stale L1 line).
template <int HINT, typename V> FB_HD V ld_hint(const V* p) {
#if defined(__CUDA_ARCH__)
  if constexpr (HINT == 1) return __ldcs(p);
  else if constexpr (HINT == 2) return __ldcg(p);
  else return *p;
#else
  return *p;
#endif
}

// Two consecutive twiddles, loaded with one 128-bit (f32) / two 128-bit (f64) instructions.
template <typename T> struct alignas(2 * sizeof(cpx<T>)) TwPair { cpx<T> a, b; };

// The same table in 8-byte planes, for mappings in which many lanes of a warp read the SAME pair (col fast, block
// fast): a 16-byte shared-memory load costs a wavefront per quarter-warp even when its lanes hit one address
// (4 per LDS.128 in pass 1, f64 pairs 8), an 8-byte load of <= 16 distinct
// words costs one in total.  f32: [a (count cpx)][b (count cpx)];  f64: [a.x][a.y][b.x][b.y] (count doubles each).
template <typename T> struct TwPlanes;
template <> struct TwPlanes<float> {
  static FB_HD void put(void* planes, int count, int idx, const TwPair<float>& w) {
    cpx<float>* p = static_cast<cpx<float>*>(planes);
    p[idx] = w.a; p[count + idx] = w.b;
  }
  static FB_HD TwPair<float> get(const void* planes, int count, int idx) {
    const cpx<float>* p = static_cast<const cpx<float>*>(planes);
    TwPair<float> w; w.a = p[idx]; w.b = p[count + idx];
    return w;
  }
};
template <> struct TwPlanes<double> {
  static FB_HD void put(void* planes, int count, int idx, const TwPair<double>& w) {
    double* p = static_cast<double*>(planes);
    p[idx] = w.a.x; p[count + idx] = w.a.y; p[2 * count + idx] = w.b.x; p[3 * count + idx] = w.b.y;
  }
  static FB_HD TwPair<double> get(const void* planes, int count, int idx) {
    const double* p = static_cast<const double*>(planes);
    TwPair<double> w;
    w.a = mk<double>(p[idx], p[count + idx]);
    w.b = mk<double>(p[2 * count + idx], p[3 * count + idx]);
    return w;
  }
};

// Table layout for the stage-A twiddles w_L^{j*p}: pair index (p/2)*RB + j holds p even / p odd.
// Lanes that differ in j read consecutive pairs (UF); lanes that share j broadcast (CF).
template <int RA, int RB> FB_HD int twa_index(int j, int p_half) { return p_half * RB + j; }

// Shared-memory layout of the exchange: Y[j][p] of FFT `col` at j*SJ + p*SP + col*SC (in elements).
template <int SJ_, int SP_, int SC_> struct ExLayout {
  static constexpr int SJ = SJ_, SP = SP_, SC = SC_;
  template <int RA, int RB, int C> static constexpr int elems() { return (RB - 1) * SJ + (RA - 1) * SP + (C - 1) * SC + 1; }
};

constexpr int kMapCF = 0, kMapUF = 1, kMapBF = 2;

template <typename T, int RA_, int RB_, int E_, int C_, bool FWD_>
struct TileFFT {
  static constexpr int RA = RA_, RB = RB_, E = E_, C = C_;
  static constexpr int L = RA * RB;
  static constexpr int TP = L / E;          // threads per FFT
  static constexpr int NA = E / RA;         // stage-A butterflies per thread
  static constexpr int NB = E / RB;         // stage-B butterflies per thread
  static constexpr int THREADS = TP * C;
  static constexpr bool FWD = FWD_;
  static_assert(E % RA == 0 && E % RB == 0 && L % E == 0, "bad tile shape");
  static_assert(RB % TP == 0 || TP % RB == 0, "bad tile shape");

  // shared-memory footprint of the exchange in elements for layout LAY
  template <class LAY> static constexpr int smem_elems() { return LAY::template elems<RA, RB, C>(); }

  using V = cpx<T>;
  V v[E];

  template <int MAP> static FB_HD int col_of(int t) {
    if constexpr (MAP == kMapBF) return ((t & 31) >> 3) + 4 * ((t >> 5) & 1);
    else return MAP == kMapUF ? t / TP : t % C;
  }
  template <int MAP> static FB_HD int u_of(int t) {
    if constexpr (MAP == kMapBF) return ((t >> 6) << 3) + (t & 7);
    else return MAP == kMapUF ? t % TP : t / C;
  }
  // BF covers the tile exactly once iff there are 8 FFTs per tile and 8 positions per pair of warps
  static constexpr bool kBlockFastOk = C == 8 && TP % 8 == 0 && THREADS % 64 == 0 && THREADS / 64 * 8 == TP;

  // global -> registers.  Sample n of FFT `col` lives at base[col*CS + n*NS].
  template <int UF, long NS, long CS, int HINT = 0> FB_HD void load(int t, const V* __restrict__ base) {
    const int col = col_of<UF>(t), u = u_of<UF>(t);
    const V* p = base + (long)col * CS + (long)u * NS;
#pragma unroll
    for (int a = 0; a < NA; ++a)
#pragma unroll
      for (int i = 0; i < RA; ++i) {
        if constexpr (HINT == 0) v[a * RA + i] = p[(long)(TP * a + RB * i) * NS];
        else v[a * RA + i] = ld_hint<HINT>(p + (long)(TP * a + RB * i) * NS);
      }
  }

  // Same with strides known only at run time (outer column pass of the three-pass path, outer_kernels.cuh).
  template <int MAP> FB_HD void load_rt(int t, const V* __restrict__ base, long ns, long cs) {
    const int col = col_of<MAP>(t), u = u_of<MAP>(t);
    const V* p = base + (long)col * cs + (long)u * ns;
#pragma unroll
    for (int a = 0; a < NA; ++a)
#pragma unroll
      for (int i = 0; i < RA; ++i) v[a * RA + i] = p[(long)(TP * a + RB * i) * ns];
  }

  // Same for a tile of C = 8 FFTs stored in 8 x 8 blocks: sample n of FFT `col` at (n / 8) * 64 + col * 8 + n % 8.
  template <int MAP, int HINT = 0> FB_HD void load_blocked(int t, const V* __restrict__ base) {
    static_assert(C == 8 && RB % 8 == 0 && TP % 8 == 0, "blocked tiles hold 8 FFTs");
    const int col = col_of<MAP>(t), u = u_of<MAP>(t);
    const V* p = base + (u >> 3) * 64 + col * 8 + (u & 7);
#pragma unroll
    for (int a = 0; a < NA; ++a)
#pragma unroll
      for (int i = 0; i < RA; ++i) v[a * RA + i] = ld_hint<HINT>(p + (TP * a + RB * i) * 8);   // (.. / 8) blocks of 64
  }

  // DFT_RA over i for each owned j, then the stage twiddle w_L^{j*p} (skipped for p == 0).
  // PLANES: `twa` is the table in the 8-byte-plane layout (TwPlanes) instead of an array of pairs.
  template <int UF, bool PLANES = false> FB_HD void stage_a(int t, const TwPair<T>* __restrict__ twa) {
    const int u = u_of<UF>(t);
    static_for<0, NA>([&](auto A) FB_LAMBDA {
      constexpr int a = decltype(A)::value;
      dif2<RA, a * RA, FWD, T, E>(v);
      const int j = u + TP * a;
      static_for<0, RA / 2>([&](auto H) FB_LAMBDA {
        constexpr int h = decltype(H)::value;
        const TwPair<T> w = PLANES ? TwPlanes<T>::get(twa, (RA / 2) * RB, twa_index<RA, RB>(j, h))
                                   : twa[twa_index<RA, RB>(j, h)];
        if constexpr (h != 0) v[a * RA + bitrev(2 * h, ilog2(RA))] = ctw<FWD>(v[a * RA + bitrev(2 * h, ilog2(RA))], w.a);
        v[a * RA + bitrev(2 * h + 1, ilog2(RA))] = ctw<FWD>(v[a * RA + bitrev(2 * h + 1, ilog2(RA))], w.b);
      });
    });
  }

  // registers -> shared (layout LAY)
  template <int UF, class LAY> FB_HD void scatter(int t, V* smem) const {
    constexpr int SJ = LAY::SJ, SP = LAY::SP, SC = LAY::SC;
    const int col = col_of<UF>(t), u = u_of<UF>(t);
    static_for<0, NA>([&](auto A) FB_LAMBDA {
      constexpr int a = decltype(A)::value;
      V* s = smem + (u + TP * a) * SJ + col * SC;
      static_for<0, RA>([&](auto P) FB_LAMBDA {
        constexpr int p = decltype(P)::value;
        s[p * SP] = v[a * RA + bitrev(p, ilog2(RA))];
      });
    });
  }

  // shared -> registers for stage B: thread owns p = u + TP*c, reads all j
  template <int UF, class LAY> FB_HD void gather(int t, const V* smem) {
    constexpr int SJ = LAY::SJ, SP = LAY::SP, SC = LAY::SC;
    const int col = col_of<UF>(t), u = u_of<UF>(t);
#pragma unroll
    for (int c = 0; c < NB; ++c) {
      const V* s = smem + (u + TP * c) * SP + col * SC;
#pragma unroll
      for (int j = 0; j < RB; ++j) v[c * RB + j] = s[j * SJ];
    }
  }

  FB_HD void stage_b() {
    static_for<0, NB>([&](auto Cc) FB_LAMBDA {
      constexpr int c = decltype(Cc)::value;
      dif2<RB, c * RB, FWD, T, E>(v);
    });
  }

  // registers -> global.  Output k = p + RA*r of FFT `col` goes to base[col*CS + k*KS], optionally
  // multiplied by the inter-pass twiddle tw2[col*CS + k*KS] (same layout as the destination) and by
  // a real scale factor.
  template <int UF, long KS, long CS, bool TW2, bool SCALE, int HINT = 0>
  FB_HD void store(int t, V* __restrict__ base, const V* __restrict__ tw2, T scale) const {
    const int col = col_of<UF>(t), u = u_of<UF>(t);
    static_for<0, NB>([&](auto Cc) FB_LAMBDA {
      constexpr int c = decltype(Cc)::value;
      const long off = (long)col * CS + (long)(u + TP * c) * KS;
      if constexpr (TW2) {
        // Inter-pass twiddles come from L2: fetch them in batches of TWB so that a batch costs one
        // round trip instead of one per value (the values of a batch are all loaded before first use).
        constexpr int TWB = RB < 8 ? RB : 8;
        V w[TWB];
#pragma unroll
        for (int q = 0; q < TWB; ++q) w[q] = tw2[off + (long)(RA * q) * KS];
        static_for<0, RB / TWB>([&](auto G) FB_LAMBDA {
          constexpr int g = decltype(G)::value;
          V wn[TWB];
          if constexpr ((g + 1) * TWB < RB) {
#pragma unroll
            for (int q = 0; q < TWB; ++q) wn[q] = tw2[off + (long)(RA * ((g + 1) * TWB + q)) * KS];
          }
          static_for<0, TWB>([&](auto Q) FB_LAMBDA {
            constexpr int r = g * TWB + decltype(Q)::value;
            V val = ctw<FWD>(v[c * RB + bitrev(r, ilog2(RB))], w[decltype(Q)::value]);
            if constexpr (SCALE) val = cscale(val, scale);
            st_hint<HINT>(&base[off + (long)(RA * r) * KS], val);
          });
          if constexpr ((g + 1) * TWB < RB) {
#pragma unroll
            for (int q = 0; q < TWB; ++q) w[q] = wn[q];
          }
        });
      } else {
        static_for<0, RB>([&](auto Rr) FB_LAMBDA {
          constexpr int r = decltype(Rr)::value;
          V val = v[c * RB + bitrev(r, ilog2(RB))];
          if constexpr (SCALE) val = cscale(val, scale);
          st_hint<HINT>(&base[off + (long)(RA * r) * KS], val);
        });
      }
    });
  }

  // Pass-1 store with the inter-pass twiddle in factored form, both factors in shared memory:
  //   w_N^{n2*(p + RA*r)} = base[n2][p] * step[n2][r],  base = w_N^{n2*p},  step = w_N^{RA*n2*r}.
  // sbase is laid out [col][p], sstep [r][col] (lanes that differ in col read adjacent words, lanes that
  // differ in p broadcast).  Costs one extra complex multiply per sample and no global-memory load.
  // BLOCK_ROW > 0: the destination is the blocked intermediate [k / 8][tile][k % 8][col] with BLOCK_ROW
  // elements per k-block row (= 64 * tiles per row) and `base` pointing at the tile's block of row 0: the 4
  // consecutive k of a warp and its 8 columns form one 256-byte run.
  // BASE_PCOL: sbase is laid out [p][col] instead of [col][p] (conflict-free for lanes = 8 columns x 4 p).
  template <long KS, long CS, int HINT, long BLOCK_ROW = 0, bool BASE_PCOL = false>
  FB_HD void store_factored(int t, V* __restrict__ base, const V* sbase, const V* sstep) const {
    const int col = col_of<false>(t), u = u_of<false>(t);
    static_assert(BLOCK_ROW == 0 || ((C == 8 || C == 16) && RA % 8 == 0), "blocked intermediate: 8 or 16 columns per tile");
    static_for<0, NB>([&](auto Cc) FB_LAMBDA {
      constexpr int c = decltype(Cc)::value;
      const int p = u + TP * c;
      // blocked: column block col / 8 (64 elements apart), row p % 8 of the block, column col % 8
      const long off = BLOCK_ROW ? (long)(p >> 3) * BLOCK_ROW + (col >> 3) * 64 + (p & 7) * 8 + (col & 7)
                                 : (long)col * CS + (long)p * KS;
      const V wb = BASE_PCOL ? sbase[p * C + col] : sbase[col * RA + p];
      static_for<0, RB>([&](auto Rr) FB_LAMBDA {
        constexpr int r = decltype(Rr)::value;
        const V w = cmul(wb, sstep[r * C + col]);
        constexpr long step = BLOCK_ROW ? (long)(RA * r / 8) * BLOCK_ROW : (long)(RA * r) * KS;
        st_hint<HINT>(&base[off + step], ctw<FWD>(v[c * RB + bitrev(r, ilog2(RB))], w));
      });
    });
  }
};

// ---- device drivers of the phase protocol -------------------------------------------------------------------------
// On-chip kernels (onchip_kernels.cuh): the stage twiddles are copied to shared memory behind the exchange buffer, then
// the CTA loops grid-stride over groups of Cfg::C transforms, each phase followed by __syncwarp (the last one too: the
// next group reuses the exchange buffer).
template <class Cfg, class Body> __device__ __forceinline__ void run_onchip_groups(const typename Body::Args& a) {
  using Tile = typename Cfg::Tile;
  using T = typename Body::T;
  extern __shared__ __align__(128) unsigned char onchip_smem[];
  typename Tile::V* exch = reinterpret_cast<typename Tile::V*>(onchip_smem);
  TwPair<T>* twa = reinterpret_cast<TwPair<T>*>(onchip_smem + Cfg::EX_BYTES);
  for (int i = threadIdx.x; i < (Tile::RA / 2) * Tile::RB; i += Cfg::THREADS) twa[i] = a.twa[i];
  __syncthreads();
  const long groups = (a.batch + Cfg::C - 1) / Cfg::C;
  Tile f;
  for (long grp = blockIdx.x; grp < groups; grp += gridDim.x) {
    static_for<0, Body::kPhases>([&](auto P) FB_LAMBDA {
      Body::template phase<decltype(P)::value>(f, a, grp, threadIdx.x, exch, twa);
      __syncwarp();
    });
  }
}

// Single-tile CTA kernels: CTA blockIdx.x runs the phases of its tile, with __syncthreads between them.
template <class Tile, class Body> __device__ __forceinline__ void run_cta_tile(const typename Body::Args& a) {
  extern __shared__ __align__(16) unsigned char tile_smem[];
  typename Tile::V* smem = reinterpret_cast<typename Tile::V*>(tile_smem);
  Tile f;
  static_for<0, Body::kPhases>([&](auto P) FB_LAMBDA {
    if constexpr (decltype(P)::value > 0) __syncthreads();
    Body::template phase<decltype(P)::value>(f, a, blockIdx.x, threadIdx.x, smem, nullptr);
  });
}

}  // namespace fb200
