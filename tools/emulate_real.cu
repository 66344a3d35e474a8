// emulate_real.cu -- runs the device code of the real-input transforms on the CPU, thread by thread and phase by
// phase (real_kernels.cuh and RealBody in onchip_kernels.cuh are __host__ __device__), against a double-precision
// DFT:
//   * the fused on-chip real kernel, forward and inverse, for every on-chip size class of both precisions;
//   * the untangle / tangle steps of the half-length path, for even and odd M = N/2.
// Every spectrum access goes through FB_SPEC_ACCESS, which records its address and width (emulate_common.h): the
// check fails on any access wider than one complex value or not aligned to its width (f32 spectrum rows of odd index
// start 8 bytes off a 16-byte boundary).  It also reports the bank-conflict degree of the forward kernel's
// natural-order park and of the untangle's ascending / descending reads.
// Build: nvcc -std=c++17 -O1 --expt-relaxed-constexpr -I fourier_b200/csrc tools/emulate_real.cu \
//             fourier_b200/csrc/host_math.cu (host only, never run on the device)
#include "emulate_common.h"

// numpy.fft.rfft of the reals x[0 .. n) times s, in double
static void ref_rfft(const double* x, long n, double s, std::vector<double>& re, std::vector<double>& im) {
  std::vector<double> wr, wi;
  twiddles(n, wr, wi);
  re.assign(n / 2 + 1, 0); im.assign(n / 2 + 1, 0);
  for (long k = 0; k <= n / 2; ++k) {
    double a = 0, b = 0;
    for (long j = 0; j < n; ++j) { const long q = (k * j) % n; a += x[j] * wr[q]; b += x[j] * wi[q]; }
    re[k] = a * s; im[k] = b * s;
  }
}

// N * numpy.fft.irfft(X, n) times s, in double (imaginary parts of bin 0 and, n even, bin n/2 ignored)
static void ref_irfft(const double* xr, const double* xi, long n, double s, std::vector<double>& y) {
  std::vector<double> wr, wi;
  twiddles(n, wr, wi);
  y.assign(n, 0);
  for (long j = 0; j < n; ++j) {
    double a = xr[0];
    for (long k = 1; 2 * k < n; ++k) {
      const long q = (k * j) % n;   // Re(X[k] * conj(w^{kj}))
      a += 2 * (xr[k] * wr[q] + xi[k] * wi[q]);
    }
    if (n % 2 == 0) a += xr[n / 2] * ((j % 2) ? -1.0 : 1.0);
    y[j] = a * s;
  }
}

// max |got - ref| / max |ref|
static double rel(const std::vector<double>& got, const std::vector<double>& ref) {
  double e = 0, r = 0;
  for (size_t i = 0; i < ref.size(); ++i) { e = std::max(e, std::fabs(got[i] - ref[i])); r = std::max(r, std::fabs(ref[i])); }
  return std::isnan(e) ? INFINITY : e / r;
}

// ---- fused on-chip real kernel ------------------------------------------------------------------------------------
template <class K>
static int check_fused(const char* name, double tol) {
  using T = typename K::T;
  constexpr int RA = K::RA, RB = K::RB, E = K::E;
  using V = cpx<T>;
  constexpr long L = RA * RB, N = 2 * L, batch = 5;   // 5: not a multiple of the transforms per CTA
  const double s = 0.5;
  int bad = 0;
  auto twa = twopass::make_twa<T>(RA, RB);
  const auto tab = pair_table<T>(L);
  unsigned long long seed = 977 + L;
  {  // forward
    using Cfg = typename K::template Cfg<true>;
    using Body = onchip::RealBody<Cfg>;
    Buf<T> x(N * batch);
    for (long i = 0; i < N * batch; ++i) x[i] = (T)rnd(seed);
    Buf<V> out((L + 1) * batch);
    for (long i = 0; i < (L + 1) * batch; ++i) out[i] = mk<T>((T)NAN, (T)NAN);
    run_body<Body, typename Cfg::Tile, typename Cfg::Lay>(
        {reinterpret_cast<const V*>(x.p), out.p, twa.data(), tab.data(), batch, (T)(s / 2)}, (batch + Cfg::C - 1) / Cfg::C,
        twa.data());
    double worst = 0;
    bool zero_imag = true;
    for (long b = 0; b < batch; ++b) {
      std::vector<double> xd(N), re, im, got, ref;
      for (long i = 0; i < N; ++i) xd[i] = x[b * N + i];
      ref_rfft(xd.data(), N, s, re, im);
      for (long k = 0; k <= L; ++k) {
        const V v = out[b * (L + 1) + k];
        got.push_back(v.x); got.push_back(v.y); ref.push_back(re[k]); ref.push_back(im[k]);
      }
      worst = std::max(worst, rel(got, ref));
      for (long k : {0L, L}) { const V v = out[b * (L + 1) + k]; zero_imag &= v.y == 0 && !std::signbit(v.y); }
    }
    printf("%s N=%ld forward: max rel err vs f64 DFT %.3e, Im X[0], Im X[N/2] == +0: %s %s\n", name, N, worst,
           zero_imag ? "yes" : "no", worst < tol && zero_imag ? "OK" : "FAIL");
    bad += !(worst < tol && zero_imag);
    bad += check_access("forward spectrum", out.p, batch, (L + 1) * sizeof(V), (int)sizeof(V));

    // bank conflicts: natural-order park (write), untangle reads z[k] ascending and z[L-k] descending
    using Tile = typename Cfg::Tile;
    int worst_w = 1, worst_r = 1;
    for (int warp = 0; warp < Cfg::THREADS / 32; ++warp) {
      for (int c = 0; c < Tile::NB; ++c)
        for (int r = 0; r < RB; ++r) {
          std::vector<long> idx;
          for (int l = 0; l < 32; ++l) {
            const int t = warp * 32 + l;
            idx.push_back(Body::park(t) + (Tile::template u_of<true>(t) + Tile::TP * c) + RA * r);
          }
          worst_w = std::max(worst_w, conflict_degree<(int)sizeof(V)>(idx));
        }
      for (int j = 0; j < E / 2; ++j) {
        std::vector<long> up, down;
        for (int l = 0; l < 32; ++l) {
          const int t = warp * 32 + l;
          const long k = Tile::template u_of<true>(t) + Tile::TP * j;
          up.push_back(Body::park(t) + k);
          down.push_back(k == 0 ? -1 : Body::park(t) + L - k);   // lane k = 0 takes its own branch
        }
        worst_r = std::max({worst_r, conflict_degree<(int)sizeof(V)>(up), conflict_degree<(int)sizeof(V)>(down)});
      }
    }
    printf("  park     threads %4d  exchange conflicts: write x%d, read x%d\n", Cfg::THREADS, worst_w, worst_r);
  }
  {  // inverse (Ifft: s = 1/N), random imaginary parts in bins 0 and N/2
    using Cfg = typename K::template Cfg<false>;
    using Body = onchip::RealBody<Cfg>;
    Buf<V> x((L + 1) * batch);
    for (long i = 0; i < (L + 1) * batch; ++i) x[i] = mk<T>((T)rnd(seed), (T)rnd(seed));
    Buf<T> y(N * batch);
    for (long i = 0; i < N * batch; ++i) y[i] = (T)NAN;
    run_body<Body, typename Cfg::Tile, typename Cfg::Lay>(
        {x.p, reinterpret_cast<V*>(y.p), twa.data(), tab.data(), batch, (T)(1.0 / N)}, (batch + Cfg::C - 1) / Cfg::C,
        twa.data());
    double worst = 0;
    for (long b = 0; b < batch; ++b) {
      std::vector<double> xr(L + 1), xi(L + 1), got(N), ref;
      for (long k = 0; k <= L; ++k) { xr[k] = x[b * (L + 1) + k].x; xi[k] = x[b * (L + 1) + k].y; }
      ref_irfft(xr.data(), xi.data(), N, 1.0 / N, ref);
      for (long i = 0; i < N; ++i) got[i] = y[b * N + i];
      worst = std::max(worst, rel(got, ref));
    }
    printf("%s N=%ld inverse: max rel err vs f64 DFT %.3e %s\n", name, N, worst, worst < tol ? "OK" : "FAIL");
    bad += !(worst < tol);
    bad += check_access("inverse spectrum", x.p, batch, (L + 1) * sizeof(V), (int)sizeof(V));
  }
  return bad;
}

// ---- untangle / tangle steps of the half-length path ---------------------------------------------------------------
template <typename T>
static int check_steps(const char* name, long m, double tol) {
  using V = cpx<T>;
  const long n = 2 * m, batch = 3;
  const double s = 1.0 / std::sqrt((double)n);   // SqrtScaledFft / SqrtScaledIfft
  const auto tab = pair_table<T>(m);
  unsigned long long seed = 4242 + m;
  int bad = 0;
  {  // forward: Z = FFT_M(z) in double, rounded to T; untangle; compare with rfft
    std::vector<double> x(n * batch);
    for (auto& v : x) v = (T)rnd(seed);
    std::vector<V> z = packed_fft<T>(x, m, batch);
    Buf<V> out((m + 1) * batch);
    for (long i = 0; i < (m + 1) * batch; ++i) out[i] = mk<T>((T)NAN, (T)NAN);
    for (long b = 0; b < batch; ++b)
      for (long k = 0; k <= m / 2; ++k) real::untangle(z.data() + b * m, out.p + b * (m + 1), m, k, tab.data(), (T)(s / 2));
    double worst = 0;
    bool zero_imag = true;
    for (long b = 0; b < batch; ++b) {
      std::vector<double> re, im, got, ref;
      ref_rfft(x.data() + b * n, n, s, re, im);
      for (long k = 0; k <= m; ++k) {
        const V v = out[b * (m + 1) + k];
        got.push_back(v.x); got.push_back(v.y); ref.push_back(re[k]); ref.push_back(im[k]);
      }
      worst = std::max(worst, rel(got, ref));
      for (long k : {0L, m}) { const V v = out[b * (m + 1) + k]; zero_imag &= v.y == 0 && !std::signbit(v.y); }
    }
    printf("%s untangle N=%ld (M=%ld): max rel err vs f64 DFT %.3e, Im X[0], Im X[N/2] == +0: %s %s\n", name, n, m,
           worst, zero_imag ? "yes" : "no", worst < tol && zero_imag ? "OK" : "FAIL");
    bad += !(worst < tol && zero_imag);
    bad += check_access("untangle spectrum", out.p, batch, (m + 1) * sizeof(V), (int)sizeof(V));
  }
  {  // inverse: tangle; unscaled IFFT_M in double; compare with irfft (random imaginary parts in bins 0 and M)
    Buf<V> x((m + 1) * batch);
    for (long i = 0; i < (m + 1) * batch; ++i) x[i] = mk<T>((T)rnd(seed), (T)rnd(seed));
    std::vector<V> z(m * batch, mk<T>((T)NAN, (T)NAN));
    for (long b = 0; b < batch; ++b)
      for (long k = 0; k <= m / 2; ++k) real::tangle(x.p + b * (m + 1), z.data() + b * m, m, k, tab.data(), (T)s);
    const std::vector<double> y = packed_ifft<T>(z, m, batch);
    double worst = 0;
    for (long b = 0; b < batch; ++b) {
      std::vector<double> got(y.begin() + b * n, y.begin() + (b + 1) * n), ref, xr(m + 1), xi(m + 1);
      for (long k = 0; k <= m; ++k) { xr[k] = x[b * (m + 1) + k].x; xi[k] = x[b * (m + 1) + k].y; }
      ref_irfft(xr.data(), xi.data(), n, s, ref);
      worst = std::max(worst, rel(got, ref));
    }
    printf("%s tangle N=%ld (M=%ld): max rel err vs f64 DFT %.3e %s\n", name, n, m, worst, worst < tol ? "OK" : "FAIL");
    bad += !(worst < tol);
    bad += check_access("tangle spectrum", x.p, batch, (m + 1) * sizeof(V), (int)sizeof(V));
  }
  return bad;
}

int main() {
  int bad = 0;
  // every on-chip size class (onchip_configs.cuh): L = M = N/2
  for_each_onchip<float>([&](auto k) { bad += check_fused<decltype(k)>("fused f32", 2e-6); });
  for_each_onchip<double>([&](auto k) { bad += check_fused<decltype(k)>("fused f64", 5e-15); });
  for (long m : {1L, 2L, 3L, 512L, 1000L, 1009L}) {
    bad += check_steps<float>("steps f32", m, 2e-6);
    bad += check_steps<double>("steps f64", m, 2e-14);   // the reference is a direct DFT in double: ~sqrt(N) eps
  }
  printf(bad ? "EMULATION FAILED (%d)\n" : "EMULATION OK\n", bad);
  return bad ? 1 : 0;
}
