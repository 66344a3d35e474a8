// emulate_conv.cu -- runs the device code of the convolution of real rows, y = irfft(rfft(x) . H) (DESIGN.md §4.11),
// on the CPU, thread by thread and phase by phase (real::conv_pair in real_kernels.cuh and ConvBody in
// onchip_kernels.cuh are __host__ __device__), against a direct circular convolution in double:
//   * the fused on-chip conv kernel for every on-chip size class of both precisions, with F = 3 spectrum rows, a
//     batch of 5 and a batch that is not a multiple of the rows per CTA, starting at spectrum row 0 and 2;
//   * real::conv_pair alone (the half-length path's conv_pair_kernel), for even and odd M = N/2.
// H is the rfft of random real taps h, with random imaginary parts added to bins 0 and N/2 (they must not count).
// Every spectrum access goes through FB_SPEC_ACCESS, which records its address and width (emulate_common.h): the
// check fails on any access wider than one complex value, misaligned, or outside H, and when no odd row of H (8 bytes
// off a 16-byte boundary for f32) was read.  It also reports the bank-conflict degree of the pair step's write-back
// into the park and of the stage-A reads of Z' from it.
// Build: nvcc -std=c++17 -O1 --expt-relaxed-constexpr -I fourier_b200/csrc tools/emulate_conv.cu \
//             fourier_b200/csrc/host_math.cu (host only, never run on the device)
#include "emulate_common.h"

// F rows of taps h (double) and their spectra H = rfft(h) rounded to T, bins 0 and N/2 (N even) with random
// imaginary parts
template <typename T>
static void make_filters(long n, long rows, unsigned long long& seed, std::vector<double>& h, Buf<cpx<T>>& H) {
  const long bins = n / 2 + 1;
  h.resize(rows * n);
  for (auto& v : h) v = rnd(seed);
  for (long f = 0; f < rows; ++f)
    for (long k = 0; k < bins; ++k) {
      double a = 0, c = 0;
      for (long j = 0; j < n; ++j) {
        double wr, wi;
        host_twiddle((size_t)((k * j) % n), (size_t)n, &wr, &wi);
        a += h[f * n + j] * wr; c += h[f * n + j] * wi;
      }
      if (k == 0 || 2 * k == n) c = rnd(seed);
      H[f * bins + k] = mk<T>((T)a, (T)c);
    }
}

// max over rows of max |y - x (*) h| / max |x (*) h|, the circular convolution in double; row b uses h row
// (row0 + b) mod rows
static double conv_err(const std::vector<double>& x, const std::vector<double>& h, const std::vector<double>& y, long n,
                       long batch, long rows, long row0) {
  double worst = 0;
  for (long b = 0; b < batch; ++b) {
    const double* hf = h.data() + ((row0 + b) % rows) * n;
    double e = 0, r = 0;
    for (long i = 0; i < n; ++i) {
      double s = 0;
      for (long m = 0; m < n; ++m) s += x[b * n + m] * hf[(i - m + n) % n];
      e = std::max(e, std::fabs(y[b * n + i] - s));
      r = std::max(r, std::fabs(s));
    }
    worst = std::max(worst, std::isnan(e) ? INFINITY : e / r);
  }
  return worst;
}

// ---- fused on-chip conv kernel --------------------------------------------------------------------------------------
template <class K>
static int check_fused(const char* name, double tol) {
  using T = typename K::T;
  constexpr int RA = K::RA, RB = K::RB, E = K::E;
  using V = cpx<T>;
  using Cfg = typename K::template Cfg<true>;
  using Body = onchip::ConvBody<Cfg>;
  using Tile = typename Cfg::Tile;
  constexpr long L = RA * RB, N = 2 * L, rows = 3;
  int bad = 0;
  const auto twa = twopass::make_twa<T>(RA, RB);
  const auto tab = pair_table<T>(L);
  unsigned long long seed = 1313 + L;
  std::vector<double> h;
  Buf<V> H(rows * (L + 1));
  make_filters<T>(N, rows, seed, h, H);
  for (long batch : {5L, (long)Cfg::C + 3}) {   // neither a multiple of the rows per CTA
    for (long row0 : {0L, 2L}) {
      Buf<T> x(N * batch), y(N * batch);
      std::vector<double> xd(N * batch), yd(N * batch);
      for (long i = 0; i < N * batch; ++i) { x[i] = (T)rnd(seed); xd[i] = x[i]; y[i] = (T)NAN; }
      run_body<Body, Tile, typename Cfg::Lay>({reinterpret_cast<const V*>(x.p), reinterpret_cast<V*>(y.p), twa.data(),
                                               tab.data(), H.p, rows, row0, batch, (T)(1.0 / (2 * N))},
                                              (batch + Cfg::C - 1) / Cfg::C, twa.data());
      for (long i = 0; i < N * batch; ++i) yd[i] = y[i];
      const double worst = conv_err(xd, h, yd, N, batch, rows, row0);
      printf("%s N=%ld F=%ld batch=%ld row0=%ld: max rel err vs direct circular convolution %.3e %s\n", name, N, rows,
             batch, row0, worst, worst < tol ? "OK" : "FAIL");
      bad += !(worst < tol);
      bad += check_access("H", H.p, rows, (L + 1) * sizeof(V), (int)sizeof(V));
    }
  }
  // bank conflicts: the pair step writes z[k] ascending and z[L-k] descending back into the park; the inverse reads
  // Z' in stage-A order
  int worst_w = 1, worst_r = 1;
  for (int warp = 0; warp < Cfg::THREADS / 32; ++warp) {
    for (int j = 0; j < E / 2; ++j) {
      std::vector<long> up, down;
      for (int l = 0; l < 32; ++l) {
        const int t = warp * 32 + l;
        const long k = Tile::template u_of<true>(t) + Tile::TP * j;
        up.push_back(Body::Real::park(t) + k);
        down.push_back(k == 0 ? -1 : Body::Real::park(t) + L - k);   // lane k = 0 takes its own branch
      }
      worst_w = std::max({worst_w, conflict_degree<(int)sizeof(V)>(up), conflict_degree<(int)sizeof(V)>(down)});
    }
    for (int q = 0; q < Tile::NA; ++q)
      for (int i = 0; i < RA; ++i) {
        std::vector<long> idx;
        for (int l = 0; l < 32; ++l) {
          const int t = warp * 32 + l;
          idx.push_back(Body::Real::park(t) + Tile::template u_of<true>(t) + Tile::TP * q + RB * i);
        }
        worst_r = std::max(worst_r, conflict_degree<(int)sizeof(V)>(idx));
      }
  }
  printf("  conv     threads %4d  exchange conflicts: write-back x%d, stage-A read x%d\n", Cfg::THREADS, worst_w,
         worst_r);
  return bad;
}

// ---- real::conv_pair alone, in place on Z = FFT_M(z) (the half-length path) -----------------------------------------
template <typename T>
static int check_pair(const char* name, long m, double tol) {
  using V = cpx<T>;
  const long n = 2 * m, batch = 5, rows = 3, row0 = 1;
  const auto tab = pair_table<T>(m);
  unsigned long long seed = 5151 + m;
  std::vector<double> h, x(n * batch);
  Buf<V> H(rows * (m + 1));
  make_filters<T>(n, rows, seed, h, H);
  for (auto& v : x) v = (T)rnd(seed);
  std::vector<V> z = packed_fft<T>(x, m, batch);
  for (long b = 0; b < batch; ++b)
    for (long k = 0; k <= m / 2; ++k)
      real::conv_pair(z.data() + b * m, H.p + ((row0 + b) % rows) * (m + 1), m, k, tab.data(), (T)(1.0 / (2 * n)));
  const std::vector<double> y = packed_ifft<T>(z, m, batch);   // unscaled inverse, interleaved
  const double worst = conv_err(x, h, y, n, batch, rows, row0);
  printf("%s conv_pair N=%ld (M=%ld): max rel err vs direct circular convolution %.3e %s\n", name, n, m, worst,
         worst < tol ? "OK" : "FAIL");
  int bad = !(worst < tol);
  bad += check_access("H", H.p, rows, (m + 1) * sizeof(V), (int)sizeof(V));
  return bad;
}

int main() {
  int bad = 0;
  // every on-chip size class (onchip_configs.cuh): L = M = N/2
  for_each_onchip<float>([&](auto k) { bad += check_fused<decltype(k)>("fused f32", 2e-6); });
  for_each_onchip<double>([&](auto k) { bad += check_fused<decltype(k)>("fused f64", 1e-13); });
  for (long m : {1L, 2L, 3L, 512L, 1000L, 1009L}) {
    bad += check_pair<float>("pair f32", m, 2e-6);
    bad += check_pair<double>("pair f64", m, 1e-13);
  }
  printf(bad ? "EMULATION FAILED (%d)\n" : "EMULATION OK\n", bad);
  return bad ? 1 : 0;
}
