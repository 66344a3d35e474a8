// dist_kernels.cuh -- pass 2 of the two-pass row FFT with the exchange of the distributed six-step transform
// (fourier_b200/distributed.py, BASELINE configs[4]) folded into its store.
//
// The stand-alone exchange (exchange.cu) re-reads the finished FFT rows from HBM, transposes them through shared
// memory and stores them into the peers.  Here the last register stage of the row FFT stores its results STRAIGHT
// into the destination ranks' buffers over NVLink, in the final layout, with the inter-step twiddle applied on
// the way -- one HBM sweep and one kernel less per exchange, and the NVLink transfer overlaps the butterflies.
//
//   rows r = 0 .. rows-1 of length N (this rank's rows of the row-distributed matrix), X_r = FFT_N(row r)
//   dst_q[c * out_ld + out_off + r] = X_r[q * cb + c] * w_Ntot^{(row0 + r) * (q * cb + c)},   cb = N / P
//   (rows in batches of R: dst_q[(r / R) * out_bs + c * out_ld + out_off + r % R], the three-pass path of bigpow2.cu)
//
// which is exactly what fourier_b200_exchange_* delivers after a batched FFT of the rows.  The store is contiguous
// along r (the batch), so one tile takes the SAME intermediate row k1 of C ADJACENT TRANSFORMS (instead of C adjacent
// rows of one transform, twopass_kernels.cuh Body2): loads are C contiguous runs of N2 samples, stores are C-sample
// (64 / 128-byte) pieces, one per output k = k1 + N1 * k2, whose destination rank is k / cb.
// Every member is __host__ __device__; the two phases follow tilefft.cuh's protocol.
#pragma once

#include <cmath>
#include <type_traits>

#include "plan.h"
#include "tilefft.cuh"
#include "twopass_kernels.cuh"

namespace fb200 {
namespace dist {

struct PeerPtrs { void* p[kMaxPeers]; };

FB_HD void unit_root(unsigned long long m, unsigned long long n_total, double* re, double* im) {
  // exp(+2 pi i m / n_total)
  const double x = 2.0 * (double)m / (double)n_total;
#if defined(__CUDA_ARCH__)
  sincospi(x, im, re);
#else
  *re = std::cos(3.14159265358979323846 * x);
  *im = std::sin(3.14159265358979323846 * x);
#endif
}

// TW: 0 = no twiddle, 1 = w = exp(-2 pi i m / Ntot) (forward), 2 = exp(+2 pi i m / Ntot) (inverse)
template <class Tile, class LAY, long N1, long N2, int TW>
struct RowsExchangeBody {
  using V = typename Tile::V;
  using T = decltype(V::x);
  static constexpr long N = N1 * N2;
  static constexpr int C = Tile::C;
  struct Args {
    const V* scratch;              // intermediate A[b][k1][n2] of the chunk (output of pass 1)
    const TwPair<T>* twa;          // stage twiddles of the tile
    PeerPtrs outs;                 // destination buffers, one per rank
    unsigned long long out_ld;     // row length of the destination matrices
    unsigned long long out_off;    // destination column of the chunk's first transform
    unsigned long long row0;       // global row index of the chunk's first transform (twiddle)
    unsigned long long n_total;    // Ntot of the twiddle
    unsigned long long r0;         // index of the chunk's first transform among the rows of the call
    unsigned long long out_bs;     // three-pass path (bigpow2.cu): rows come in batches of 2^rb_shift (one batch = one
    int rb_shift;                  //   long transform), batch b is stored out_bs elements further on; 63 = one batch
    unsigned long long rpb;        // != 0: batches of rpb rows, not a power of two (outer radix 3 / 9 / 27)
    unsigned long long rows_valid; // rows of the call that exist: the last tile may be padding (nothing is stored for it)
    unsigned groups;               // transforms of the chunk / C
    int cb_shift;                  // log2(cb): destination rank of output k is k >> cb_shift
  };
  // block -> (k1, group of C transforms); consecutive blocks store adjacent pieces of the same destination rows
  static FB_HD void phase1(Tile& f, const Args& a, long block, int t, V* smem) {
    const long g = block % a.groups, k1 = block / a.groups;
    const V* src = a.scratch + g * (C * N) + k1 * N2;
    f.template load<kMapUF, 1, N>(t, src);
    f.template stage_a<kMapUF>(t, a.twa);
    f.template scatter<kMapUF, LAY>(t, smem);
  }
  static FB_HD void phase2(Tile& f, const Args& a, long block, int t, const V* smem) {
    constexpr int RA = Tile::RA, RB = Tile::RB, TP = Tile::TP, NB = Tile::NB;
    const long g = block % a.groups, k1 = block / a.groups;
    f.template gather<kMapCF, LAY>(t, smem);
    f.stage_b();
    const int col = Tile::template col_of<kMapCF>(t), u = Tile::template u_of<kMapCF>(t);
    const unsigned long long r = (unsigned long long)g * C + col;          // transform of the chunk
    const unsigned long long rc = a.r0 + r;                                // ... of the call
    const unsigned long long bidx = a.rpb ? rc / a.rpb : rc >> a.rb_shift;
    const unsigned long long dcol = bidx * a.out_bs + a.out_off + (a.rpb ? rc - bidx * a.rpb : rc & ((1ull << a.rb_shift) - 1));
    const bool valid = rc < a.rows_valid;
    const unsigned long long mask = (1ull << a.cb_shift) - 1;
    [[maybe_unused]] double sr = 1.0, si = 0.0;
    [[maybe_unused]] unsigned long long rg = 0;
    if constexpr (TW != 0) {
      rg = (a.row0 + rc) % a.n_total;
      unit_root(rg * (unsigned long long)(N1 * RA) % a.n_total, a.n_total, &sr, &si);
      if (TW == 1) si = -si;
    }
    static_for<0, NB>([&](auto Cc) FB_LAMBDA {
      constexpr int c = decltype(Cc)::value;
      const unsigned long long k0 = (unsigned long long)k1 + (unsigned long long)N1 * (u + TP * c);
      [[maybe_unused]] double wr = 1.0, wi = 0.0;
      if constexpr (TW != 0) {
        unit_root(rg * k0 % a.n_total, a.n_total, &wr, &wi);   // rg, k0 < 2^32 (checked by the launcher)
        if (TW == 1) wi = -wi;
      }
      static_for<0, RB>([&](auto Rr) FB_LAMBDA {
        constexpr int rr = decltype(Rr)::value;
        const unsigned long long k = k0 + (unsigned long long)(N1 * RA) * rr;
        V val = f.v[c * RB + bitrev(rr, ilog2(RB))];
        if constexpr (TW != 0) {
          val = cmul(val, mk<T>((T)wr, (T)wi));
          const double nr = wr * sr - wi * si;
          wi = wr * si + wi * sr;
          wr = nr;
        }
        V* dst = reinterpret_cast<V*>(a.outs.p[k >> a.cb_shift]);
        if (valid) dst[(k & mask) * a.out_ld + dcol] = val;
      });
    });
  }

  // phase protocol (tilefft.cuh); the stage twiddles come from Args
  static constexpr int kPhases = 2;
  template <int P> static FB_HD void phase(Tile& f, const Args& a, long block, int t, V* smem, const TwPair<T>*) {
    if constexpr (P == 0) phase1(f, a, block, t, smem);
    else phase2(f, a, block, t, smem);
  }
};

template <class Body, class Tile, int MINB>
__global__ void __launch_bounds__(Tile::THREADS, MINB) rows_exchange_kernel(const typename Body::Args a) {
  run_cta_tile<Tile, Body>(a);
}

// Tiles of twice as many transforms where the configuration's pass-2 tile has 16 (f32) / 8 (f64): a warp's store is then
// one 256-byte run instead of two 128-byte pieces.  WideShape<S, T>::type is the wide tile of pass-2 shape S (S itself
// where there is none); the paddings are the bank-conflict-free ones (tools/emulate.cu).
template <class S, typename T> struct WideShape { using type = S; };
template <> struct WideShape<twopass::Shape<8, 16, 16, 16, 2>, float> { using type = twopass::Shape<8, 16, 16, 32, 2>; };
template <> struct WideShape<twopass::Shape<16, 16, 16, 16, 1>, float> { using type = twopass::Shape<16, 16, 16, 32, 1>; };
template <> struct WideShape<twopass::Shape<8, 16, 16, 8, 1>, double> { using type = twopass::Shape<8, 16, 16, 16, 1>; };
template <> struct WideShape<twopass::Shape<16, 16, 16, 8, 1>, double> { using type = twopass::Shape<16, 16, 16, 16, 1>; };
// the tile shape of the exchange for two-pass configuration G: its wide tile (WIDE) or its pass-2 tile
template <class G, bool WIDE, typename T>
using ExchangeShape = typename std::conditional<WIDE, typename WideShape<typename G::Shape2, T>::type, typename G::Shape2>::type;

}  // namespace dist
}  // namespace fb200
