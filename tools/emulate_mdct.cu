// emulate_mdct.cu -- runs the device code of the type-IV DCT and the MDCT on the CPU, thread by thread and phase by phase
// (Dct4Body / MdctBody in onchip_kernels.cuh and the real::dct4* / mdct* / imdct* steps of real_kernels.cuh are
// __host__ __device__), against the direct formulas in double:
//   * Dct4Body for every on-chip size class of both precisions, all three norms, a batch of C + 3 rows, and in place
//     against out of place (bit for bit);
//   * MdctBody with center on and off, at row lengths of the shortest legal length, 2N + 1, a multiple of N and three
//     frames plus a remainder, on batches that leave a partial group of frames;
//   * every input read and output write goes through FB_LIN_ACCESS: reads must lie in the row of their transform (frame)
//     and every output must be written exactly once;
//   * the shared-memory bank conflicts of the new load, pre-twiddle, post and store phases;
//   * the element steps of the other paths (pre-twiddle, post, fold gather) for N = 2, 4 and 96 over two chunks, the
//     inner FFT done in double, and imdct_add_one over the real::istft_runs cuts of several scratch sizes (the bits of
//     every output must not depend on the cut).
// Build: nvcc -std=c++17 -O1 --expt-relaxed-constexpr -I fourier_b200/csrc tools/emulate_mdct.cu \
//             fourier_b200/csrc/host_math.cu (host only, never run on the device)
static void lin_record(int write, const void* p, long g);
#ifdef __CUDA_ARCH__
#define FB_LIN_ACCESS(w, p, g)
#else
#define FB_LIN_ACCESS(w, p, g) lin_record((w), (const void*)(p), (long)(g))
#endif
#include "emulate_common.h"

#include <cstring>

struct LinAccess { int write; uintptr_t addr; long g; };
static std::vector<LinAccess> g_lin;
__attribute__((unused)) static void lin_record(int write, const void* p, long g) { g_lin.push_back({write, (uintptr_t)p, g}); }

static const char* kNorms[] = {"backward", "ortho", "forward"};

static double scale_of(int norm, long n) {
  double h, h0;
  real::dct_scales(4, norm, n, h, h0);
  return h;
}

// scipy.fft.dct(x, type=4, norm) of one row in double, directly
static std::vector<double> ref_dct4(const std::vector<double>& x, int norm) {
  const long n = (long)x.size();
  const double h = scale_of(norm, n), pi = std::acos(-1.0);
  std::vector<double> c(8 * n), y(n, 0.0);
  for (long i = 0; i < 8 * n; ++i) c[i] = std::cos(pi * (double)i / (4.0 * n));   // cos(2 pi i / (8N))
  for (long k = 0; k < n; ++k) {
    double s = 0;
    for (long j = 0; j < n; ++j) s += x[j] * c[((2 * j + 1) * (2 * k + 1)) % (8 * n)];
    y[k] = 2 * h * s;
  }
  return y;
}

// the MDCT of one row of L samples in double, directly: F frames of N coefficients
static std::vector<double> ref_mdct(const std::vector<double>& x, const std::vector<double>& w, long n, bool center,
                                    int norm) {
  const real::FrameMap m = real::mdct_map(n, (long)x.size(), center);
  const double h = scale_of(norm, n), pi = std::acos(-1.0);
  std::vector<double> c(8 * n), y(m.frames * n, 0.0);
  for (long i = 0; i < 8 * n; ++i) c[i] = std::cos(pi * (double)i / (4.0 * n));
  for (long f = 0; f < m.frames; ++f)
    for (long k = 0; k < n; ++k) {
      double s = 0;
      for (long p = 0; p < 2 * n; ++p) {
        const long t = f * n - m.pad + p;
        if (t < 0 || t >= (long)x.size()) continue;
        s += w[p] * x[t] * c[((2 * p + 1 + n) * (2 * k + 1)) % (8 * n)];   // cos(pi/N (p + 1/2 + N/2)(k + 1/2))
      }
      y[f * n + k] = 2 * h * s;
    }
  return y;
}

static double rel(const double* got, const double* ref, long cnt) {
  double e = 0, r = 0;
  for (long i = 0; i < cnt; ++i) { e = std::max(e, std::fabs(got[i] - ref[i])); r = std::max(r, std::fabs(ref[i])); }
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
template <typename T> static cpx<T> dct4_c(int norm, long n) {
  double re, im;
  real::dct4_const(norm, n, re, im);
  return mk<T>((T)re, (T)im);
}

// Checks the access log: every read (a real) lies in [row(g) * in_row, (row(g) + 1) * in_row) elements of `in`, every
// write (a complex value) wholly within out_row elements of its g in `out`, and every element of `out` (count
// elements) is written exactly once.  Returns (outside, not once).
template <typename T, class RowOf>
static void check_log(const T* in, long in_row, const T* out, long out_row, long count, RowOf row_of, long& outside,
                      long& not_once) {
  outside = not_once = 0;
  std::vector<int> writes(count, 0);
  for (const LinAccess& e : g_lin) {
    const uintptr_t base = e.write ? (uintptr_t)out : (uintptr_t)in;
    const long row = e.write ? e.g : row_of(e.g), width = e.write ? out_row : in_row;
    const long off = (long)(e.addr - base);
    // the loads read reals, the fused store writes complex values (two reals); the whole access must lie in the row
    const long bytes = e.write ? (long)sizeof(cpx<T>) : (long)sizeof(T);
    if (off < row * width * (long)sizeof(T) || off + bytes > (row + 1) * width * (long)sizeof(T)) {
      ++outside;
      continue;
    }
    if (e.write)
      for (long i = off / (long)sizeof(T); i < std::min((off + bytes) / (long)sizeof(T), count); ++i) ++writes[i];
  }
  for (int w : writes) not_once += w != 1;
  g_lin.clear();
}

// ---- fused bodies ---------------------------------------------------------------------------------------------------
template <class K> static int check_dct4(const char* name, double tol) {
  using T = typename K::T;
  using Cfg = typename K::template Cfg<true>;
  using Body = onchip::Dct4Body<Cfg>;
  constexpr long L = Cfg::L, N = 2 * L, batch = Cfg::C + 3;   // a full group and a partial one
  const long groups = (batch + Cfg::C - 1) / Cfg::C;
  const auto twa = twopass::make_twa<T>(K::RA, K::RB);
  const auto wq = dct_table<T>(N);
  int bad = 0;
  unsigned long long seed = 41 * L + 4;
  for (int norm = 0; norm < 3; ++norm) {
    Buf<T> x(N * batch), y(N * batch), z(N * batch);
    for (long i = 0; i < N * batch; ++i) { x[i] = (T)rnd(seed); y[i] = (T)NAN; z[i] = x[i]; }
    typename Body::Args a;
    static_cast<typename onchip::RealBody<Cfg>::Args&>(a) = {nullptr, nullptr, twa.data(), nullptr, batch, (T)1};
    a.x = x.p; a.y = y.p; a.wq = wq.data(); a.c = dct4_c<T>(norm, N);
    g_lin.clear();
    run_body<Body, typename Cfg::Tile, typename Cfg::Lay>(a, groups, twa.data());
    long outside, not_once;
    // reads: reals inside their row; writes: complex values inside their row, every real once
    check_log(x.p, N, y.p, N, N * batch, [](long g) { return g; }, outside, not_once);
    double worst = 0;
    for (long b = 0; b < batch; ++b) {
      std::vector<double> xd(x.p + b * N, x.p + (b + 1) * N), got(y.p + b * N, y.p + (b + 1) * N);
      const std::vector<double> ref = ref_dct4(xd, norm);
      worst = std::max(worst, rel(got.data(), ref.data(), N));
    }
    a.x = z.p; a.y = z.p;
    run_body<Body, typename Cfg::Tile, typename Cfg::Lay>(a, groups, twa.data());
    g_lin.clear();
    const bool same = std::memcmp(y.p, z.p, N * batch * sizeof(T)) == 0;
    const bool ok = worst < tol && !outside && !not_once && same;
    printf("fused dct4 %s N=%ld batch=%ld norm=%s: max rel err %.3e, outside row %ld, not once %ld, in place %s %s\n",
           name, N, batch, kNorms[norm], worst, outside, not_once, same ? "same" : "differs", ok ? "OK" : "FAIL");
    bad += !ok;
  }
  return bad;
}

template <class K> static int check_mdct(const char* name, double tol) {
  using T = typename K::T;
  using Cfg = typename K::template Cfg<true>;
  using Body = onchip::MdctBody<Cfg>;
  constexpr long L = Cfg::L, N = 2 * L;
  const auto twa = twopass::make_twa<T>(K::RA, K::RB);
  const auto wq = dct_table<T>(N);
  std::vector<T> win(2 * N);
  std::vector<double> wd(2 * N);
  for (long p = 0; p < 2 * N; ++p) {
    win[p] = (T)std::sin(std::acos(-1.0) * (p + 0.5) / (2.0 * N));
    wd[p] = (double)win[p];
  }
  int bad = 0;
  unsigned long long seed = 43 * L + 7;
  for (int center = 1; center >= 0; --center)
    for (long len : {center ? 1L : 2 * N, 2 * N + 1, 4 * N, (center ? 3 : 4) * N + N / 2 + 5}) {
      const real::FrameMap m0 = real::mdct_map(N, len, center);
      // the fewest rows whose frames leave a partial group, at least one full group
      long batch = 1;
      while (batch * m0.frames <= Cfg::C || (batch * m0.frames) % Cfg::C == 0) ++batch;
      const long total = batch * m0.frames, groups = (total + Cfg::C - 1) / Cfg::C;
      const int norm = (int)((len + center) % 3);
      Buf<T> x(len * batch), y(total * N);
      for (long i = 0; i < len * batch; ++i) x[i] = (T)rnd(seed);
      for (long i = 0; i < total * N; ++i) y[i] = (T)NAN;
      typename Body::Args a;
      static_cast<typename onchip::RealBody<Cfg>::Args&>(a) = {nullptr, nullptr, twa.data(), nullptr, total, (T)1};
      a.x = x.p; a.y = y.p; a.wq = wq.data(); a.c = dct4_c<T>(norm, N); a.win = win.data(); a.m = m0;
      g_lin.clear();
      run_body<Body, typename Cfg::Tile, typename Cfg::Lay>(a, groups, twa.data());
      long outside, not_once;
      const long frames = m0.frames;
      check_log(x.p, len, y.p, N, total * N, [&](long g) { return g / frames; }, outside, not_once);
      double worst = 0;
      for (long b = 0; b < batch; ++b) {
        std::vector<double> xd(x.p + b * len, x.p + (b + 1) * len), got(y.p + b * frames * N, y.p + (b + 1) * frames * N);
        const std::vector<double> ref = ref_mdct(xd, wd, N, center, norm);
        worst = std::max(worst, rel(got.data(), ref.data(), frames * N));
      }
      const bool ok = worst < tol && !outside && !not_once;
      printf("fused mdct %s N=%ld center=%d L=%ld frames=%ld batch=%ld norm=%s: max rel err %.3e, outside row %ld, "
             "not once %ld %s\n", name, N, center, len, frames, batch, kNorms[norm], worst, outside, not_once,
             ok ? "OK" : "FAIL");
      bad += !ok;
    }
  return bad;
}

// bank conflicts of the new phases (the FFT phases are the stft's)
template <class K> static void conflicts() {
  using T = typename K::T;
  using V = cpx<T>;
  using Cfg = typename K::template Cfg<true>;
  using Tile = typename Cfg::Tile;
  using Real = onchip::RealBody<Cfg>;
  constexpr int L = Cfg::L, N = 2 * L, TP = Tile::TP, E = Tile::E, B = (int)sizeof(T),
                BV = (int)sizeof(V);
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
  // the loads: sample (dct4) or folded value (mdct) n = u + TP s at real n (even) or N - n (odd)
  const int ld = worst(B, [&](int t, int s) { const long n = u(t) + TP * s; return pr(t) + ((n & 1) ? N - n : n); },
                       N / TP);
  // pre: complex values n = u + TP j, read and written in place; post: Z[k], k = u + TP j, read as complex values,
  // then the pairs written as reals 2k and N-1-2k
  const int pre = worst(BV, [&](int t, int s) { return Real::park(t) + u(t) + TP * s; }, E);
  const int po = std::max({worst(BV, [&](int t, int s) { return Real::park(t) + u(t) + TP * s; }, E),
                           worst(B, [&](int t, int s) { return pr(t) + 2L * (u(t) + TP * s); }, E),
                           worst(B, [&](int t, int s) { return pr(t) + N - 1 - 2L * (u(t) + TP * s); }, E)});
  // store: complex values j = u + TP s
  const int st = worst(BV, [&](int t, int s) { return Real::park(t) + u(t) + TP * s; }, L / TP);
  printf("  %s L=%d threads %d conflicts: load x%d, pre x%d, post x%d, store x%d\n",
         sizeof(T) == 4 ? "f32" : "f64", L, Cfg::THREADS, ld, pre, po, st);
}

// ---- the other paths' element steps ---------------------------------------------------------------------------------
// the forward FFT of each row of `v` (len complex values) in double, rounded to T
template <typename V> static void dft_rows(std::vector<V>& v, long len, long rows) {
  using T = decltype(V::x);
  std::vector<double> wr, wi;
  twiddles(len, wr, wi);
  std::vector<V> out(v.size());
  for (long b = 0; b < rows; ++b)
    for (long k = 0; k < len; ++k) {
      double a = 0, c = 0;
      for (long j = 0; j < len; ++j) {
        const V s = v[b * len + j];
        const double tr = wr[(k * j) % len], ti = wi[(k * j) % len];
        a += s.x * tr - s.y * ti; c += s.x * ti + s.y * tr;
      }
      out[b * len + k] = mk<T>((T)a, (T)c);
    }
  v = out;
}

// dct4_rows' chunk loop on real_half, `chunk` rows at a time: pre, FFT, post
template <typename T> static std::vector<T> other_dct4(const T* x, long n, long batch, long chunk, int norm) {
  using V = cpx<T>;
  const auto wq = dct_table<T>(n);
  const V c = dct4_c<T>(norm, n);
  const long m = n / 2;
  std::vector<T> y(n * batch, (T)NAN);
  for (long b0 = 0; b0 < batch; b0 += chunk) {
    const long nb = std::min(chunk, batch - b0);
    std::vector<V> z(m * nb);
    for (long g = 0; g < m * nb; ++g) {
      const long b = g / m, k = g - b * m;
      const T* r = x + (b0 + b) * n;
      z[g] = real::dct4_pre(r[2 * k], r[n - 1 - 2 * k], wq.data(), n, k);
    }
    dft_rows(z, m, nb);
    for (long g = 0; g < m * nb; ++g) {
      const long b = g / m, k = g - b * m;
      const V p = real::dct4_post(z[g], c, wq.data(), n, k);
      y[(b0 + b) * n + 2 * k] = p.x;
      y[(b0 + b) * n + n - 1 - 2 * k] = p.y;
    }
  }
  return y;
}

template <typename T> static int check_other(const char* name, long n, double tol) {
  using V = cpx<T>;
  int bad = 0;
  unsigned long long seed = 91 + n;
  const long m = n / 2;
  const auto wq = dct_table<T>(n);
  // dct4 over two chunks of rows
  {
    const long batch = 5, chunk = 3;
    std::vector<T> x(n * batch);
    for (auto& v : x) v = (T)rnd(seed);
    for (int norm = 0; norm < 3; ++norm) {
      const std::vector<T> y = other_dct4(x.data(), n, batch, chunk, norm);
      double worst = 0;
      for (long b = 0; b < batch; ++b) {
        std::vector<double> xd(x.begin() + b * n, x.begin() + (b + 1) * n), got(y.begin() + b * n, y.begin() + (b + 1) * n);
        const std::vector<double> ref = ref_dct4(xd, norm);
        worst = std::max(worst, rel(got.data(), ref.data(), n));
      }
      const bool ok = worst < tol;
      printf("elements %s dct4 N=%ld norm=%s chunks=2: max rel err %.3e %s\n", name, n, kNorms[norm], worst,
             ok ? "OK" : "FAIL");
      bad += !ok;
    }
  }
  // mdct: the fold gather, FFT and post over two chunks of frames; then the imdct through the runs of several caps
  std::vector<T> win(2 * n);
  std::vector<double> wd(2 * n);
  for (long p = 0; p < 2 * n; ++p) {
    win[p] = (T)std::sin(std::acos(-1.0) * (p + 0.5) / (2.0 * n));
    wd[p] = (double)win[p];
  }
  for (int center = 1; center >= 0; --center) {
    const long len = 3 * n + n / 2 + 1, batch = 2;
    const int norm = center ? real::kDctNormOrtho : real::kDctNormBackward;
    const real::FrameMap m0 = real::mdct_map(n, len, center);
    const long frames = m0.frames, total = batch * frames, chunk = total / 2 + 1;
    std::vector<T> x(len * batch), X(total * n, (T)NAN);
    for (auto& v : x) v = (T)rnd(seed);
    const V c = dct4_c<T>(norm, n);
    g_lin.clear();
    for (long q0 = 0; q0 < total; q0 += chunk) {
      const long nq = std::min(chunk, total - q0);
      real::FrameMap mc = m0;
      mc.g0 = q0;
      std::vector<V> z(m * nq);
      for (long g = 0; g < m * nq; ++g) {
        const long q = g / m, k = g - q * m;
        z[g] = real::dct4_pre(real::mdct_fold_one(mc, x.data(), win.data(), q, 2 * k),
                              real::mdct_fold_one(mc, x.data(), win.data(), q, n - 1 - 2 * k), wq.data(), n, k);
      }
      dft_rows(z, m, nq);
      for (long g = 0; g < m * nq; ++g) {
        const long q = g / m, k = g - q * m;
        const V p = real::dct4_post(z[g], c, wq.data(), n, k);
        X[(q0 + q) * n + 2 * k] = p.x;
        X[(q0 + q) * n + n - 1 - 2 * k] = p.y;
      }
    }
    long outside = 0;
    for (const LinAccess& e : g_lin) {
      const long off = (long)(e.addr - (uintptr_t)x.data()) / (long)sizeof(T), row = e.g / frames;
      outside += e.write || off < row * len || off >= (row + 1) * len;
    }
    g_lin.clear();
    double worst = 0;
    for (long b = 0; b < batch; ++b) {
      std::vector<double> xd(x.begin() + b * len, x.begin() + (b + 1) * len);
      std::vector<double> got(X.begin() + b * frames * n, X.begin() + (b + 1) * frames * n);
      const std::vector<double> ref = ref_mdct(xd, wd, n, center, norm);
      worst = std::max(worst, rel(got.data(), ref.data(), frames * n));
    }
    bool ok = worst < tol && !outside;
    printf("elements %s mdct N=%ld center=%d L=%ld frames=%ld chunks=2: max rel err %.3e, outside row %ld %s\n", name, n,
           center, len, frames, worst, outside, ok ? "OK" : "FAIL");
    bad += !ok;
    // imdct: v = DCT-IV(X) with the swapped norm in double, then the overlap-add over the runs of each cap
    std::vector<T> v(total * n);
    for (long f = 0; f < total; ++f) {
      std::vector<double> xf(X.begin() + f * n, X.begin() + (f + 1) * n);
      const std::vector<double> r = ref_dct4(xf, real::dct_swapped_norm(norm));
      for (long k = 0; k < n; ++k) v[f * n + k] = (T)r[k];
    }
    real::FrameMap mi = real::mdct_map(n, 2 * n, center);
    mi.frames = frames;
    mi.rcp = 1.0 / (double)frames;
    const long out_len = center ? len : (frames + 1) * n;
    std::vector<T> first;
    bool same = true;
    long caps = 0, not_once = 0;
    for (size_t cap : {(size_t)1000000, (size_t)total, (size_t)frames, (size_t)3, (size_t)2}) {
      const size_t capf = real::istft_scratch_frames(cap, 2 * n, n, frames);
      std::vector<T> y(out_len * batch, (T)NAN);
      std::vector<int> writes(out_len * batch, 0);
      real::istft_runs(2 * n, n, (size_t)mi.pad, frames, out_len, batch, capf,
                       [&](size_t gs, size_t ge, size_t b0, size_t nb, size_t i0, size_t i1) -> int {
                         std::vector<T> seg(v.begin() + gs * n, v.begin() + ge * n);
                         for (size_t r = 0; r < nb; ++r)
                           for (size_t i = i0; i < i1; ++i) {
                             real::imdct_add_one(mi, seg.data(), win.data(), (long)gs, y.data() + (b0 + r) * out_len,
                                                 (long)(b0 + r), (long)i);
                             ++writes[(b0 + r) * out_len + i];
                           }
                         return 0;
                       });
      for (int w : writes) not_once += w != 1;
      if (first.empty()) first = y;
      else same &= std::memcmp(first.data(), y.data(), y.size() * sizeof(T)) == 0;
      ++caps;
    }
    g_lin.clear();
    // with center and the sine window the round trip gives x back; without, the interior (covered by two frames)
    double rt = 0, rx = 0;
    for (long b = 0; b < batch; ++b)
      for (long i = center ? 0 : n; i < (center ? len : frames * n); ++i) {
        rt = std::max(rt, std::fabs((double)first[b * out_len + i] - (double)x[b * len + i]));
        rx = std::max(rx, std::fabs((double)x[b * len + i]));
      }
    rt /= rx;
    ok = same && !not_once && rt < tol;
    printf("elements %s imdct N=%ld center=%d caps=%ld: outputs %s, not once %ld, round trip max rel err %.3e %s\n", name,
           n, center, caps, same ? "same" : "differ", not_once, rt, ok ? "OK" : "FAIL");
    bad += !ok;
  }
  return bad;
}

int main() {
  int bad = 0;
  for_each_onchip<float>([&](auto k) {
    bad += check_dct4<decltype(k)>("f32", 1e-5);
    bad += check_mdct<decltype(k)>("f32", 1e-5);
    conflicts<decltype(k)>();
  });
  for_each_onchip<double>([&](auto k) {
    bad += check_dct4<decltype(k)>("f64", 1e-12);
    bad += check_mdct<decltype(k)>("f64", 1e-12);
    conflicts<decltype(k)>();
  });
  for (long n : {2L, 4L, 96L}) {
    bad += check_other<float>("f32", n, 1e-5);
    bad += check_other<double>("f64", n, 1e-12);
  }
  printf(bad ? "EMULATION FAILED (%d)\n" : "EMULATION OK\n", bad);
  return bad ? 1 : 0;
}
