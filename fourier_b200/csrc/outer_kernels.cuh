// outer_kernels.cuh -- outer column pass of the three-pass path for power-of-two N beyond the two-pass kernels
// (f32 N >= 2^21, f64 N >= 2^17; csrc/bigpow2.cu).
//
//   N = Na * Nb, n = na * Nb + nb, k = ka + Na * kb              (the four-step split once more, around the two-pass path)
//   outer pass (this kernel):   A[ka][nb] = scale * w_N^{nb * ka} * sum_{na} x[na][nb] w_Na^{na * ka}
//   rows (Plan(Nb)::exec_rows_exchange with one destination):  X[ka + Na * kb] = sum_{nb} A[ka][nb] w_Nb^{nb * kb}
//
// One CTA = one tile of C adjacent columns nb, every sample read once into registers (C * 8-byte pieces, row pitch Nb)
// and written once to the same position of the output; the register tile is the one of the two-pass kernels
// (tilefft.cuh), both stages "col fast".  The twiddle w_N^{nb * ka} is not a table (N entries would be as large as
// the data): per thread the outputs ka = p + RA * r form a geometric sequence, i.e. two sincospi in double (index
// reduced exactly) and a recurrence in double, rounded to T per use -- as accurate as a table rounded once.
// The reference streams the whole array once per radix-4/8 stage (autosort/mod.rs:338-379: 10+ sweeps at N = 2^24);
// this pass and the row pass sweep HBM once each.
#pragma once

#include "dist_kernels.cuh"
#include "tilefft.cuh"
#include "twopass_kernels.cuh"

namespace fb200 {
namespace outer {

template <class Tile, class LAY>
struct ColumnBody {
  using V = typename Tile::V;
  using T = decltype(V::x);
  static constexpr int C = Tile::C;
  static constexpr bool FWD = Tile::FWD;
  struct Args {
    const V* in; V* out; const TwPair<T>* twa;
    unsigned long long nb;        // row length = pitch of the samples of one column
    unsigned long long n_total;   // N = L * nb
    unsigned tiles;               // nb / C
    T scale;
  };
  static FB_HD void phase1(Tile& f, const Args& a, long block, int t, V* smem) {
    const long tile = block % a.tiles, b = block / a.tiles;
    f.template load_rt<kMapCF>(t, a.in + b * (long)a.n_total + tile * C, (long)a.nb, 1);
    f.template stage_a<kMapCF>(t, a.twa);
    f.template scatter<kMapCF, LAY>(t, smem);
  }
  static FB_HD void phase2(Tile& f, const Args& a, long block, int t, const V* smem) {
    constexpr int RA = Tile::RA, RB = Tile::RB, TP = Tile::TP, NB = Tile::NB;
    const long tile = block % a.tiles, b = block / a.tiles;
    f.template gather<kMapCF, LAY>(t, smem);
    f.stage_b();
    const int col = Tile::template col_of<kMapCF>(t), u = Tile::template u_of<kMapCF>(t);
    const unsigned long long n2 = (unsigned long long)tile * C + col;       // column index nb of this thread
    V* dst = a.out + b * (long)a.n_total + n2;
    double sr, si;
    dist::unit_root(n2 * RA % a.n_total, a.n_total, &sr, &si);              // n2 * ka < N <= 2^32: no overflow
    if (FWD) si = -si;
    static_for<0, NB>([&](auto Cc) FB_LAMBDA {
      constexpr int c = decltype(Cc)::value;
      const unsigned long long p = u + TP * c;
      double wr, wi;
      dist::unit_root(n2 * p % a.n_total, a.n_total, &wr, &wi);
      if (FWD) wi = -wi;
      wr *= (double)a.scale; wi *= (double)a.scale;
      static_for<0, RB>([&](auto Rr) FB_LAMBDA {
        constexpr int r = decltype(Rr)::value;
        const V val = cmul(f.v[c * RB + bitrev(r, ilog2(RB))], mk<T>((T)wr, (T)wi));
        dst[(p + (unsigned long long)(RA * r)) * a.nb] = val;
        const double nr = wr * sr - wi * si;
        wi = wr * si + wi * sr;
        wr = nr;
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
__global__ void __launch_bounds__(Tile::THREADS, MINB) column_kernel(const typename Body::Args a) {
  run_cta_tile<Tile, Body>(a);
}

// The outer pass of length Na = S::L: register tile Shape S (twopass_kernels.cuh) over C = S::C columns per CTA, at
// least MINB CTAs per SM.
template <typename T_, class S, int MINB_> struct ColumnCfg {
  using T = T_;
  using Shape = S;
  static constexpr int MINB = MINB_;
  template <bool FWD> using Tile = TileFFT<T, S::RA, S::RB, S::E, S::C, FWD>;
  using Lay = ExLayout<S::RA * S::C + S::PAD, S::C, 1>;
  template <bool FWD> using Body = ColumnBody<Tile<FWD>, Lay>;
};

// visit_column<T>(log2_na, f) calls f with a value of the outer pass of length 2^log2_na (false when there is none):
// the pass-1 shapes of the two-pass configurations, whose paddings keep the exchange bank-conflict free.
template <class F> bool visit_column_f32(int log2_na, F&& f) {
  using twopass::Shape;
  switch (log2_na) {
    case 5: f(ColumnCfg<float, Shape<4, 8, 8, 32, 0>, 4>{}); return true;
    case 6: f(ColumnCfg<float, Shape<8, 8, 8, 32, 0>, 4>{}); return true;
    case 7: f(ColumnCfg<float, Shape<8, 16, 16, 16, 0>, 4>{}); return true;
    case 8: f(ColumnCfg<float, Shape<16, 16, 16, 16, 0>, 2>{}); return true;
    case 9: f(ColumnCfg<float, Shape<16, 32, 32, 8, 8>, 2>{}); return true;
    case 10: f(ColumnCfg<float, Shape<32, 32, 32, 8, 8>, 2>{}); return true;
    default: return false;
  }
}
template <class F> bool visit_column_f64(int log2_na, F&& f) {
  using twopass::Shape;
  switch (log2_na) {
    case 4: f(ColumnCfg<double, Shape<4, 4, 4, 16, 0>, 4>{}); return true;
    case 5: f(ColumnCfg<double, Shape<4, 8, 8, 16, 0>, 4>{}); return true;
    case 6: f(ColumnCfg<double, Shape<8, 8, 8, 16, 0>, 4>{}); return true;
    case 7: f(ColumnCfg<double, Shape<8, 16, 16, 8, 4>, 2>{}); return true;
    case 8: f(ColumnCfg<double, Shape<16, 16, 16, 8, 4>, 2>{}); return true;
    default: return false;
  }
}
template <typename T, class F> bool visit_column(int log2_na, F&& f) {
  if constexpr (sizeof(T) == 4) return visit_column_f32(log2_na, f);
  else return visit_column_f64(log2_na, f);
}

// Outer pass of length B = 3, 9 or 27 for N = B * Nb (Nb a two-pass power of two): the radix-3 stages of the
// reference (autosort/mod.rs:20-21, butterfly.rs:9-22) taken FIRST, as one in-register DFT_B per column -- one thread
// per column nb, so every access of a warp is a 256-byte run -- followed by the twiddle w_N^{nb * ka} (one sincospi
// in double per thread, powers by recurrence) and the scale.  The rows then run as in the power-of-two case.
template <typename T, int B, bool FWD_>
struct Radix3ColumnBody {
  using V = cpx<T>;
  static constexpr bool FWD = FWD_;
  struct Args {
    const V* in; V* out;
    unsigned long long nb;        // row length = pitch of the samples of one column
    unsigned long long n_total;   // N = B * nb
    unsigned long long count;     // columns of the call (batch * nb)
    T scale;
  };
  static FB_HD void run(const Args& a, unsigned long long idx) {
    if (idx >= a.count) return;
    const unsigned long long b = idx / a.nb, col = idx - b * a.nb;
    const V* src = a.in + b * a.n_total + col;
    V x[B];
#pragma unroll
    for (int i = 0; i < B; ++i) x[i] = src[(unsigned long long)i * a.nb];
    if constexpr (B == 3) dft3<FWD, T>(x);
    else if constexpr (B == 9) dft9<FWD, T>(x);
    else dft27<FWD, T>(x);
    double sr, si;
    dist::unit_root(col, a.n_total, &sr, &si);
    if (FWD) si = -si;
    double wr = (double)a.scale, wi = 0.0;
    V* dst = a.out + b * a.n_total + col;
    static_for<0, B>([&](auto K) FB_LAMBDA {
      constexpr int ka = decltype(K)::value;
      dst[(unsigned long long)ka * a.nb] = cmul(x[ka], mk<T>((T)wr, (T)wi));
      const double nr = wr * sr - wi * si;
      wi = wr * si + wi * sr;
      wr = nr;
    });
  }
};

template <class Body>
__global__ void __launch_bounds__(256) radix3_column_kernel(const typename Body::Args a) {
  Body::run(a, (unsigned long long)blockIdx.x * 256 + threadIdx.x);
}

}  // namespace outer
}  // namespace fb200
