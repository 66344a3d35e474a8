// emulate_hilbert.cu -- runs the device code of the analytic signal and envelope on the CPU, thread by thread and phase
// by phase (HilbertBody in onchip_kernels.cuh and the real::hilbert* steps of real_kernels.cuh are __host__ __device__),
// against a direct DFT -> G -> inverse DFT in double:
//   * the fused body for every on-chip size class of both precisions, both outputs, a batch that leaves a partial group;
//     the analytic signal's real part must be the input bit for bit, and the envelope in place must give the bits of the
//     envelope out of place;
//   * every input read and output write goes through FB_LIN_ACCESS: reads must lie in the row of their transform and
//     every output must be written exactly once;
//   * the shared-memory bank conflicts of the new pair phase (the store phase reads shared memory only in ConvBody's
//     gather);
//   * the element steps of the other paths (hilbert_pair at half length, hilbert_bin at full length, the output step) for
//     N = 1, 2, 96 and 97 over two chunks of rows, the inner FFT done in double.
// Build: nvcc -std=c++17 -O1 --expt-relaxed-constexpr -I fourier_b200/csrc tools/emulate_hilbert.cu \
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

static const char* kOutputs[] = {"analytic", "envelope"};

// y of scipy.signal.hilbert for each of `batch` rows of n reals, in double: y = Re IDFT(G . DFT(x)) / n
static std::vector<double> ref_hilbert(const std::vector<double>& x, long n, long batch) {
  std::vector<double> wr, wi, y(n * batch);
  twiddles(n, wr, wi);
  std::vector<double> xr(n), xi(n);
  for (long b = 0; b < batch; ++b) {
    const double* r = x.data() + b * n;
    for (long k = 0; k < n; ++k) {
      double a = 0, c = 0;
      for (long j = 0; j < n; ++j) { a += r[j] * wr[(k * j) % n]; c += r[j] * wi[(k * j) % n]; }
      // times G: -i below n/2, +i above, 0 at 0 and n/2
      const double s = k == 0 || 2 * k == n ? 0.0 : 2 * k < n ? 1.0 : -1.0;
      xr[k] = s * c;
      xi[k] = -s * a;
    }
    for (long j = 0; j < n; ++j) {
      double a = 0;
      for (long k = 0; k < n; ++k) a += xr[k] * wr[(k * j) % n] + xi[k] * wi[(k * j) % n];   // Re(X[k] conj(w^kj))
      y[b * n + j] = a / (double)n;
    }
  }
  return y;
}

// worst over rows of max |got - want| / max |want|, for output `output` of rows x (reals) and y (the reference)
static double row_err(const double* got, const std::vector<double>& x, const std::vector<double>& y, long n, long batch,
                      int output) {
  double worst = 0;
  for (long b = 0; b < batch; ++b) {
    double e = 0, r = 0;
    for (long j = 0; j < n; ++j) {
      const double xv = x[b * n + j], yv = y[b * n + j];
      if (output == real::kHilbertAnalytic) {
        const double* g = got + 2 * (b * n + j);
        e = std::max(e, std::hypot(g[0] - xv, g[1] - yv));
      } else {
        e = std::max(e, std::fabs(got[b * n + j] - std::hypot(xv, yv)));
      }
      r = std::max(r, std::hypot(xv, yv));
    }
    worst = std::max(worst, std::isnan(e) ? INFINITY : e / std::max(r, 1e-300));
  }
  return worst;
}

// the real parts of the analytic output equal the input bit for bit
template <typename T> static bool real_part_exact(const T* out, const T* x, long count) {
  for (long i = 0; i < count; ++i)
    if (std::memcmp(out + 2 * i, x + i, sizeof(T))) return false;
  return true;
}

// ---- fused bodies ---------------------------------------------------------------------------------------------------
template <class K, bool ENV> static int check_fused(const char* name, double tol) {
  using T = typename K::T;
  using V = cpx<T>;
  using Cfg = typename K::template Cfg<true>;
  using Body = onchip::HilbertBody<Cfg, ENV>;
  constexpr long L = Cfg::L, N = 2 * L, batch = Cfg::C + 3;   // a full group and a partial one
  constexpr int output = ENV ? real::kHilbertEnvelope : real::kHilbertAnalytic;
  constexpr long out_row = ENV ? N : 2 * N;   // reals per output row
  const long groups = (batch + Cfg::C - 1) / Cfg::C;
  const auto twa = twopass::make_twa<T>(K::RA, K::RB);
  const auto tab = pair_table<T>(L);
  unsigned long long seed = 41 * L + sizeof(T);
  Buf<T> x(N * batch), y(out_row * batch), z(N * batch);
  for (long i = 0; i < N * batch; ++i) { x[i] = (T)rnd(seed); z[i] = x[i]; }
  for (long i = 0; i < out_row * batch; ++i) y[i] = (T)NAN;
  typename Body::Args a;
  static_cast<typename onchip::ConvBody<Cfg>::Args&>(a) = {reinterpret_cast<const V*>(x.p), nullptr, twa.data(),
                                                           tab.data(), nullptr, 1, 0, batch, (T)(1.0 / (2.0 * N)), 1};
  a.y = y.p;
  g_lin.clear();
  run_body<Body, typename Cfg::Tile, typename Cfg::Lay>(a, groups, twa.data());
  // accesses: reads inside the input row of their transform, every output real written once
  long outside = 0, not_once = 0;
  std::vector<int> writes(out_row * batch, 0);
  for (const LinAccess& e : g_lin) {
    const uintptr_t base = e.write ? (uintptr_t)y.p : (uintptr_t)x.p;
    const long row = (e.write ? out_row : N) * (long)sizeof(T), off = (long)(e.addr - base);
    if (off < e.g * row || off + (long)sizeof(V) > (e.g + 1) * row) { ++outside; continue; }
    if (e.write)
      for (long i = off / (long)sizeof(T); i < (off + (long)sizeof(V)) / (long)sizeof(T); ++i) ++writes[i];
  }
  for (int w : writes) not_once += w != 1;
  std::vector<double> xd(x.p, x.p + N * batch), got(y.p, y.p + out_row * batch);
  const double err = row_err(got.data(), xd, ref_hilbert(xd, N, batch), N, batch, output);
  // the analytic signal's real part is x; the envelope in place has the bits of the envelope out of place
  bool exact = true;
  if (ENV) {
    a.in = reinterpret_cast<const V*>(z.p);
    a.y = z.p;
    run_body<Body, typename Cfg::Tile, typename Cfg::Lay>(a, groups, twa.data());
    exact = std::equal(y.p, y.p + N * batch, z.p);
  } else {
    exact = real_part_exact(y.p, x.p, N * batch);
  }
  g_lin.clear();
  const bool ok = err < tol && !outside && !not_once && exact;
  printf("%s output=%s N=%ld batch=%ld: max rel err %.3e, outside row %ld, not once %ld, %s %s %s\n", name,
         kOutputs[output], N, batch, err, outside, not_once, ENV ? "in place" : "real part",
         exact ? (ENV ? "same" : "exact") : (ENV ? "differs" : "inexact"), ok ? "OK" : "FAIL");
  return !ok;
}

// bank conflicts of the pair phase: each lane reads and writes Z[k] and Z[L-k] of its pairs k = u + TP*j in the park
template <class K> static void conflicts() {
  using T = typename K::T;
  using V = cpx<T>;
  using Cfg = typename K::template Cfg<true>;
  using Tile = typename Cfg::Tile;
  using Real = onchip::RealBody<Cfg>;
  constexpr int L = Cfg::L, TP = Tile::TP, E = Tile::E;
  auto worst = [&](auto f) {
    int w = 1;
    for (int warp = 0; warp < Cfg::THREADS / 32; ++warp)
      for (int s = 0; s < E / 2; ++s) {
        std::vector<long> idx;
        for (int l = 0; l < 32; ++l) idx.push_back(f(warp * 32 + l, s));
        w = std::max(w, conflict_degree<(int)sizeof(V)>(idx));
      }
    return w;
  };
  auto k = [](int t, int s) { return (long)(Tile::template u_of<true>(t) + TP * s); };
  const int lo = worst([&](int t, int s) { return Real::park(t) + k(t, s); });
  const int hi = worst([&](int t, int s) { return k(t, s) ? Real::park(t) + L - k(t, s) : -1L; });
  printf("  %s L=%d threads %d conflicts: pairs Z[k] x%d, Z[L-k] x%d\n", sizeof(T) == 4 ? "f32" : "f64", L,
         Cfg::THREADS, lo, hi);
}

// ---- the other paths' element steps ---------------------------------------------------------------------------------
// direct DFT of each row of v (len complex values), forward or unscaled inverse, in double, rounded to T
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

// hilbert_device's chunk loop on real_half (even N) or real_full (odd N), chunk rows at a time; out holds N complex
// values (analytic) or N reals (envelope) per row
template <typename T> static std::vector<T> other_path(const std::vector<T>& x, long n, long batch, long chunk,
                                                       int output) {
  using V = cpx<T>;
  const long per = output == real::kHilbertAnalytic ? 2 * n : n, m = n / 2;
  std::vector<T> y(per * batch, (T)NAN);
  const auto tab = pair_table<T>(std::max(m, 1L));
  for (long b0 = 0; b0 < batch; b0 += chunk) {
    const long nb = std::min(chunk, batch - b0);
    const T* in = x.data() + b0 * n;
    T* out = y.data() + b0 * per;
    if (n % 2 == 0) {
      std::vector<V> seg(m * nb);
      std::memcpy(seg.data(), in, n * nb * sizeof(T));
      dft_rows(seg, m, nb, false);
      for (long b = 0; b < nb; ++b)
        for (long k = 0; k <= m / 2; ++k) real::hilbert_pair(seg.data() + b * m, m, k, tab.data(), (T)(1.0 / (2.0 * n)));
      dft_rows(seg, m, nb, true);
      const T* s = reinterpret_cast<const T*>(seg.data());
      for (long g = 0; g < n * nb; ++g) real::hilbert_out_one(in[g], s[g], out, g, output, g / n);
    } else {
      std::vector<V> seg(n * nb);
      for (long g = 0; g < n * nb; ++g) seg[g] = mk<T>(in[g], (T)0);
      dft_rows(seg, n, nb, false);
      for (long g = 0; g < n * nb; ++g) seg[g] = real::hilbert_bin(seg[g], n, g % n, (T)(1.0 / n));
      dft_rows(seg, n, nb, true);
      for (long g = 0; g < n * nb; ++g) real::hilbert_out_one(in[g], seg[g].x, out, g, output, g / n);
    }
  }
  return y;
}

template <typename T> static int check_other(const char* name, long n, double tol) {
  const long batch = 5, chunk = 3;   // two chunks
  unsigned long long seed = 91 + n;
  std::vector<T> x(n * batch);
  for (auto& v : x) v = (T)rnd(seed);
  const std::vector<double> xd(x.begin(), x.end()), ref = ref_hilbert(xd, n, batch);
  int bad = 0;
  for (int output : {(int)real::kHilbertAnalytic, (int)real::kHilbertEnvelope}) {
    g_lin.clear();
    const std::vector<T> y = other_path(x, n, batch, chunk, output);
    g_lin.clear();
    const std::vector<double> got(y.begin(), y.end());
    const double err = row_err(got.data(), xd, ref, n, batch, output);
    const bool exact = output != real::kHilbertAnalytic || real_part_exact(y.data(), x.data(), n * batch);
    const bool ok = err < tol && exact;
    printf("elements %s %s N=%ld output=%s chunks=2: max rel err %.3e, real part %s %s\n", name, n % 2 ? "full" : "half",
           n, kOutputs[output], err, exact ? "exact" : "inexact", ok ? "OK" : "FAIL");
    bad += !ok;
  }
  return bad;
}

int main() {
  int bad = 0;
  for_each_onchip<float>([&](auto k) {
    bad += check_fused<decltype(k), false>("fused f32", 1e-5);
    bad += check_fused<decltype(k), true>("fused f32", 1e-5);
    conflicts<decltype(k)>();
  });
  for_each_onchip<double>([&](auto k) {
    bad += check_fused<decltype(k), false>("fused f64", 1e-12);
    bad += check_fused<decltype(k), true>("fused f64", 1e-12);
    conflicts<decltype(k)>();
  });
  for (long n : {1L, 2L, 96L, 97L}) {
    bad += check_other<float>("f32", n, 1e-5);
    bad += check_other<double>("f64", n, 1e-12);
  }
  printf(bad ? "EMULATION FAILED (%d)\n" : "EMULATION OK\n", bad);
  return bad ? 1 : 0;
}
