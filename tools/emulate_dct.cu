// emulate_dct.cu -- runs the device code of the discrete cosine transforms on the CPU, thread by thread and phase by
// phase (Dct2Body / Dct3Body in onchip_kernels.cuh and the real::dct* steps of real_kernels.cuh are __host__
// __device__), against a direct O(N^2) DCT-II / DCT-III in double:
//   * both fused bodies for every on-chip size class of both precisions, all three norms, a batch that leaves a partial
//     group, and in place against out of place (bit for bit);
//   * every input read and output write goes through FB_LIN_ACCESS: reads must lie in the row of their transform and
//     every output must be written exactly once;
//   * the shared-memory bank conflicts of the new load, pair, park and store phases;
//   * the element steps of the other paths (permute, untangle, tangle, unpermute at half length; permute, post, pre,
//     unpermute at full length) for N = 1, 2, 96 and 97 over two chunks of rows, the inner FFT done in double.
// Build: nvcc -std=c++17 -O1 --expt-relaxed-constexpr -I fourier_b200/csrc tools/emulate_dct.cu \
//             fourier_b200/csrc/host_math.cu (host only, never run on the device)
static void lin_record(int write, const void* p, long g);
#ifdef __CUDA_ARCH__
#define FB_LIN_ACCESS(w, p, g)
#else
#define FB_LIN_ACCESS(w, p, g) lin_record((w), (const void*)(p), (long)(g))
#endif
#include "emulate_common.h"

struct LinAccess { int write; uintptr_t addr; long g; };
static std::vector<LinAccess> g_lin;
__attribute__((unused)) static void lin_record(int write, const void* p, long g) { g_lin.push_back({write, (uintptr_t)p, g}); }

static const char* kNorms[] = {"backward", "ortho", "forward"};

// scipy.fft.dct(x, type, norm) of one row in double, directly
static std::vector<double> ref_dct(const std::vector<double>& x, int type, int norm) {
  const long n = (long)x.size();
  double h, h0;
  real::dct_scales(type, norm, n, h, h0);
  std::vector<double> c(4 * n), y(n, 0.0);
  const double pi = std::acos(-1.0);
  for (long i = 0; i < 4 * n; ++i) c[i] = std::cos(pi * (double)i / (2.0 * n));   // cos(2 pi i / (4N))
  for (long k = 0; k < n; ++k) {
    double s = 0;
    if (type == 2) {
      for (long j = 0; j < n; ++j) s += x[j] * c[(k * (2 * j + 1)) % (4 * n)];
      y[k] = 2 * (k == 0 ? h0 : h) * s;
    } else {
      for (long j = 1; j < n; ++j) s += x[j] * c[(j * (2 * k + 1)) % (4 * n)];
      y[k] = h0 * x[0] + 2 * h * s;
    }
  }
  return y;
}

static double rel(const std::vector<double>& got, const std::vector<double>& ref) {
  double e = 0, r = 0;
  for (size_t i = 0; i < ref.size(); ++i) { e = std::max(e, std::fabs(got[i] - ref[i])); r = std::max(r, std::fabs(ref[i])); }
  return std::isnan(e) ? INFINITY : e / std::max(r, 1e-300);
}

template <typename T> static std::vector<cpx<T>> dct_table(long n) {
  std::vector<cpx<T>> w(n / 2 + 1);
  for (long k = 0; k <= n / 2; ++k) {
    double re, im;
    host_twiddle((size_t)k, (size_t)(4 * n), &re, &im);
    w[k] = mk<T>((T)re, (T)im);
  }
  return w;
}

// ---- fused bodies ---------------------------------------------------------------------------------------------------
template <class K, int TYPE> static int check_fused(const char* name, double tol) {
  using T = typename K::T;
  using V = cpx<T>;
  using Cfg = typename K::template Cfg<true>;
  using Body = onchip::DctBody<Cfg, TYPE>;
  constexpr long L = Cfg::L, N = 2 * L, batch = Cfg::C + 3;   // a full group and a partial one
  const long groups = (batch + Cfg::C - 1) / Cfg::C;
  const auto twa = twopass::make_twa<T>(K::RA, K::RB);
  const auto tab = pair_table<T>(L);
  const auto wq = dct_table<T>(N);
  int bad = 0;
  unsigned long long seed = 31 * L + TYPE;
  for (int norm = 0; norm < 3; ++norm) {
    double h, h0;
    real::dct_scales(TYPE, norm, N, h, h0);
    Buf<T> x(N * batch), y(N * batch), z(N * batch);
    for (long i = 0; i < N * batch; ++i) { x[i] = (T)rnd(seed); y[i] = (T)NAN; z[i] = x[i]; }
    typename Body::Args a;
    static_cast<typename onchip::RealBody<Cfg>::Args&>(a) = {nullptr, nullptr, twa.data(), tab.data(), batch, (T)h};
    a.x = x.p; a.y = y.p; a.wq = wq.data(); a.h0 = (T)h0;
    g_lin.clear();
    run_body<Body, typename Cfg::Tile, typename Cfg::Lay>(a, groups, twa.data());
    // accesses: reads inside the row of their transform, every output once
    long outside = 0, not_once = 0;
    std::vector<int> writes(N * batch, 0);
    for (const LinAccess& e : g_lin) {
      const uintptr_t base = e.write ? (uintptr_t)y.p : (uintptr_t)x.p;
      // reads are complex values; type 2 writes reals, type 3 complex values
      const long bytes = e.write && TYPE == 2 ? (long)sizeof(T) : (long)sizeof(V);
      const long off = (long)(e.addr - base);
      if (off < e.g * N * (long)sizeof(T) || off + bytes > (e.g + 1) * N * (long)sizeof(T)) { ++outside; continue; }
      if (e.write)
        for (long i = off / (long)sizeof(T); i < (off + bytes) / (long)sizeof(T); ++i) ++writes[i];
    }
    for (int w : writes) not_once += w != 1;
    double worst = 0;
    for (long b = 0; b < batch; ++b) {
      std::vector<double> xd(x.p + b * N, x.p + (b + 1) * N), got(y.p + b * N, y.p + (b + 1) * N);
      worst = std::max(worst, rel(got, ref_dct(xd, TYPE, norm)));
    }
    // in place: the same bits
    a.x = z.p; a.y = z.p;
    run_body<Body, typename Cfg::Tile, typename Cfg::Lay>(a, groups, twa.data());
    g_lin.clear();
    const bool same = std::equal(y.p, y.p + N * batch, z.p);
    const bool ok = worst < tol && !outside && !not_once && same;
    printf("%s type=%d N=%ld batch=%ld norm=%s: max rel err %.3e, outside row %ld, not once %ld, in place %s %s\n", name,
           TYPE, N, batch, kNorms[norm], worst, outside, not_once, same ? "same" : "differs", ok ? "OK" : "FAIL");
    bad += !ok;
  }
  return bad;
}

// bank conflicts of the DCT's own phases (the FFT phases are the stft's)
template <class K> static void conflicts() {
  using T = typename K::T;
  using V = cpx<T>;
  using Cfg = typename K::template Cfg<true>;
  using Tile = typename Cfg::Tile;
  using Real = onchip::RealBody<Cfg>;
  constexpr int L = Cfg::L, TP = Tile::TP, E = Tile::E, B = (int)sizeof(T), BV = (int)sizeof(V);
  // one access per lane of a warp: f(t) -> element index (reals or complex values, -1 for none)
  auto worst = [&](int bytes, auto f, int steps) {
    int w = 1;
    for (int warp = 0; warp < Cfg::THREADS / 32; ++warp)
      for (int s = 0; s < steps; ++s) {
        std::vector<long> idx;
        for (int l = 0; l < 32; ++l) idx.push_back(f(warp * 32 + l, s));
        w = std::max(w, bytes == B ? conflict_degree<B>(idx) : conflict_degree<BV>(idx));
      }
    return w;
  };
  auto u = [](int t) { return Tile::template u_of<true>(t); };
  auto pr = [](int t) { return 2L * Real::park(t); };   // the park in reals
  const int lsteps = L / TP, nsteps = 2 * L / TP, psteps = E / 2;
  // type 2: load writes v[j], v[N-1-j]; pairs read Z[k], Z[L-k]; park writes y[k], y[N-k], y[L-k], y[L+k]; store reads
  const int l2 = std::max(worst(B, [&](int t, int s) { return pr(t) + u(t) + TP * s; }, lsteps),
                          worst(B, [&](int t, int s) { return pr(t) + 2 * L - 1 - (u(t) + TP * s); }, lsteps));
  auto kk = [&](int t, int s) { return u(t) + TP * s; };
  const int p2 = std::max(worst(BV, [&](int t, int s) { return Real::park(t) + kk(t, s); }, psteps),
                          worst(BV, [&](int t, int s) { return kk(t, s) ? Real::park(t) + L - kk(t, s) : -1; }, psteps));
  int k2 = 1;
  for (int d : {0, 1, 2, 3})
    k2 = std::max(k2, worst(B, [&](int t, int s) {
      const long k = kk(t, s);
      if (k == 0) return -1L;
      return pr(t) + (d == 0 ? k : d == 1 ? 2 * L - k : d == 2 ? L - k : L + k);
    }, psteps));
  const int s2 = worst(B, [&](int t, int s) { return pr(t) + u(t) + TP * s; }, nsteps);
  // type 3: load writes complex values j; pairs read x[k], x[N-k], x[L-k], x[L+k]; park writes Z'[k], Z'[L-k]; store
  // reads r[j], r[N-1-j]
  const int l3 = worst(BV, [&](int t, int s) { return Real::park(t) + u(t) + TP * s; }, lsteps);
  int q3 = 1;
  for (int d : {0, 1, 2, 3})
    q3 = std::max(q3, worst(B, [&](int t, int s) {
      const long k = kk(t, s);
      if (k == 0) return -1L;
      return pr(t) + (d == 0 ? k : d == 1 ? 2 * L - k : d == 2 ? L - k : L + k);
    }, psteps));
  const int w3 = std::max(worst(BV, [&](int t, int s) { return Real::park(t) + kk(t, s); }, psteps),
                          worst(BV, [&](int t, int s) { return kk(t, s) ? Real::park(t) + L - kk(t, s) : -1; }, psteps));
  const int s3 = std::max(worst(B, [&](int t, int s) { return pr(t) + u(t) + TP * s; }, lsteps),
                          worst(B, [&](int t, int s) { return pr(t) + 2 * L - 1 - (u(t) + TP * s); }, lsteps));
  printf("  %s L=%d threads %d conflicts: type 2 load x%d, pairs read x%d, park x%d, store x%d; "
         "type 3 load x%d, pairs read x%d, park x%d, store x%d\n",
         sizeof(T) == 4 ? "f32" : "f64", L, Cfg::THREADS, l2, p2, k2, s2, l3, q3, w3, s3);
}

// ---- the other paths' element steps ---------------------------------------------------------------------------------
// direct DFT of each row of `in` (len complex values), forward or unscaled inverse, in double, rounded to T
template <typename V> static void dft_rows(std::vector<V>& v, long len, long rows, bool inverse) {
  using T = decltype(V::x);
  std::vector<double> wr, wi;
  twiddles(len, wr, wi);
  std::vector<V> out(v.size());
  for (long b = 0; b < rows; ++b)
    for (long k = 0; k < len; ++k) {
      double a = 0, c = 0;
      for (long j = 0; j < len; ++j) {
        const V s = v[b * len + j];
        const double tr = wr[(k * j) % len], ti = inverse ? -wi[(k * j) % len] : wi[(k * j) % len];
        a += s.x * tr - s.y * ti; c += s.x * ti + s.y * tr;
      }
      out[b * len + k] = mk<T>((T)a, (T)c);
    }
  v = out;
}

// dct_device's chunk loop on real_half (even N) or real_full (odd N), chunk rows at a time
template <typename T> static std::vector<T> other_path(const std::vector<T>& x, long n, long batch, long chunk, int type,
                                                       int norm) {
  using V = cpx<T>;
  double hd, h0d;
  real::dct_scales(type, norm, n, hd, h0d);
  const T h = (T)hd, h0 = (T)h0d;
  const auto wq = dct_table<T>(n);
  std::vector<T> y(n * batch, (T)NAN);
  const long m = n / 2;
  const auto tab = pair_table<T>(std::max(m, 1L));
  for (long b0 = 0; b0 < batch; b0 += chunk) {
    const long nb = std::min(chunk, batch - b0);
    const T* in = x.data() + b0 * n;
    T* out = y.data() + b0 * n;
    if (n % 2 == 0) {
      std::vector<V> seg(m * nb);
      if (type == 2) {
        T* s = reinterpret_cast<T*>(seg.data());
        for (long g = 0; g < n * nb; ++g) s[g] = in[(g / n) * n + real::dct_src(n, g % n)];
        dft_rows(seg, m, nb, false);
        for (long b = 0; b < nb; ++b)
          for (long k = 0; k <= m / 2; ++k) {
            const V* z = seg.data() + b * m;
            T* yb = out + b * n;
            V lo, hi;
            real::dct2_pair(z[k], z[k ? m - k : 0], m, k, tab.data(), wq.data(), h, h0, lo, hi);
            yb[k] = lo.x;
            if (k == 0) { yb[m] = lo.y; continue; }
            yb[n - k] = lo.y;
            if (m - k == k) continue;
            yb[m - k] = hi.x;
            yb[m + k] = hi.y;
          }
      } else {
        for (long b = 0; b < nb; ++b)
          for (long k = 0; k <= m / 2; ++k) {
            V p, q;
            real::dct3_pair(in + b * n, m, k, tab.data(), wq.data(), h, h0, p, q);
            seg[b * m + k] = p;
            if (k > 0 && m - k != k) seg[b * m + m - k] = q;
          }
        dft_rows(seg, m, nb, true);
        const T* s = reinterpret_cast<const T*>(seg.data());
        for (long g = 0; g < n * nb; ++g) out[g] = s[(g / n) * n + real::dct_pos(n, g % n)];
      }
    } else {
      std::vector<V> seg(n * nb);
      if (type == 2) {
        for (long g = 0; g < n * nb; ++g) seg[g] = mk<T>(in[(g / n) * n + real::dct_src(n, g % n)], (T)0);
        dft_rows(seg, n, nb, false);
        for (long b = 0; b < nb; ++b)
          for (long k = 0; k <= n / 2; ++k) real::dct2_post(seg.data() + b * n, out + b * n, n, k, wq.data(), h, h0, b);
      } else {
        for (long g = 0; g < n * nb; ++g) seg[g] = real::dct3_pre(in + (g / n) * n, n, g % n, wq.data(), h, h0);
        dft_rows(seg, n, nb, true);
        for (long g = 0; g < n * nb; ++g) out[g] = seg[(g / n) * n + real::dct_pos(n, g % n)].x;
      }
    }
  }
  return y;
}

template <typename T> static int check_other(const char* name, long n, double tol) {
  const long batch = 5, chunk = 3;   // two chunks
  unsigned long long seed = 77 + n;
  std::vector<T> x(n * batch);
  for (auto& v : x) v = (T)rnd(seed);
  int bad = 0;
  for (int type : {2, 3})
    for (int norm = 0; norm < 3; ++norm) {
      g_lin.clear();
      const std::vector<T> y = other_path(x, n, batch, chunk, type, norm);
      g_lin.clear();
      double worst = 0;
      for (long b = 0; b < batch; ++b) {
        std::vector<double> xd(x.begin() + b * n, x.begin() + (b + 1) * n), got(y.begin() + b * n, y.begin() + (b + 1) * n);
        worst = std::max(worst, rel(got, ref_dct(xd, type, norm)));
      }
      const bool ok = worst < tol;
      printf("elements %s %s N=%ld type=%d norm=%s chunks=2: max rel err %.3e %s\n", name, n % 2 ? "full" : "half", n,
             type, kNorms[norm], worst, ok ? "OK" : "FAIL");
      bad += !ok;
    }
  return bad;
}

int main() {
  int bad = 0;
  for_each_onchip<float>([&](auto k) {
    bad += check_fused<decltype(k), 2>("fused f32", 1e-5);
    bad += check_fused<decltype(k), 3>("fused f32", 1e-5);
    conflicts<decltype(k)>();
  });
  for_each_onchip<double>([&](auto k) {
    bad += check_fused<decltype(k), 2>("fused f64", 1e-12);
    bad += check_fused<decltype(k), 3>("fused f64", 1e-12);
    conflicts<decltype(k)>();
  });
  for (long n : {1L, 2L, 96L, 97L}) {
    bad += check_other<float>("f32", n, 1e-5);
    bad += check_other<double>("f64", n, 1e-12);
  }
  printf(bad ? "EMULATION FAILED (%d)\n" : "EMULATION OK\n", bad);
  return bad ? 1 : 0;
}
