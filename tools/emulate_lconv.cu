// emulate_lconv.cu -- runs the device code of the linear convolution of real rows by overlap-save (DESIGN.md §4.12) on
// the CPU, thread by thread and phase by phase (LinConvBody in onchip_kernels.cuh, real::SegMap, gather_one and
// scatter_one in real_kernels.cuh are __host__ __device__), against a direct linear convolution in double:
//   * the fused kernel for every on-chip size class of both precisions, K in {1, 2, 33, N/2, N-1, N}, modes full, same
//     and valid, rows of L in {1, S-1, S, S+1, 3S+7} samples (S = N - K + 1), F = 3 spectrum rows, a batch of 5 rows,
//     and one batch per class whose segments leave a partial group;
//   * the gather / scatter maps of the half-length and full-length paths for an even and an odd N, over two chunks of
//     segments, and over the host path's runs of segments of one row staged with only their input window.
// Every input read and output write goes through FB_LIN_ACCESS: the check fails on a read outside [0, L) of the
// segment's row, a write outside its output row, and an output written zero times or twice.  It also reports the
// bank-conflict degree of the shared phases (the pair step's write-back into the park, the stage-A reads of Z') and of
// the store's reads of the park.
// Build: nvcc -std=c++17 -O1 --expt-relaxed-constexpr -I fourier_b200/csrc tools/emulate_lconv.cu \
//             fourier_b200/csrc/host_math.cu (host only, never run on the device)
#include <cstdint>
#include <vector>

static void lin_record(int write, const void* p, long g);
#ifdef __CUDA_ARCH__
#define FB_LIN_ACCESS(w, p, g)
#else
#define FB_LIN_ACCESS(w, p, g) lin_record((w), (const void*)(p), (long)(g))
#endif

#include "emulate_common.h"

// ---- access log: checked as it happens ------------------------------------------------------------------------------
struct LinCheck {
  bool on = false;
  uintptr_t x = 0, y = 0;
  long esz = 0, in_len = 0, out_len = 0, per = 1;
  long bad_reads = 0, bad_writes = 0;
  std::vector<int> writes;
};
static LinCheck g_chk;

static void lin_record(int write, const void* p, long g) {
  if (!g_chk.on) return;
  const long row = g / g_chk.per;
  const intptr_t d = (intptr_t)p - (intptr_t)(write ? g_chk.y : g_chk.x);
  const long e = (long)(d / g_chk.esz);
  const long len = write ? g_chk.out_len : g_chk.in_len;
  if (d % g_chk.esz || d < 0 || e < row * len || e >= (row + 1) * len) {
    ++(write ? g_chk.bad_writes : g_chk.bad_reads);
    return;
  }
  if (write) ++g_chk.writes[e];
}

template <typename T> static void check_begin(const T* x, const T* y, long in_len, long out_len, long per, long batch) {
  g_chk.on = true;
  g_chk.x = (uintptr_t)x; g_chk.y = (uintptr_t)y;
  g_chk.esz = sizeof(T); g_chk.in_len = in_len; g_chk.out_len = out_len; g_chk.per = per;
  g_chk.bad_reads = g_chk.bad_writes = 0;
  g_chk.writes.assign(out_len * batch, 0);
}
// -> reads outside the row, writes outside the row, outputs written zero times, outputs written more than once
static void check_end(long& reads, long& writes, long& missing, long& twice) {
  g_chk.on = false;
  reads = g_chk.bad_reads; writes = g_chk.bad_writes; missing = twice = 0;
  for (int c : g_chk.writes) { missing += c == 0; twice += c > 1; }
}

// a tap of magnitude in [0.5, 1): the error of an FFT convolution scales with the whole filter, and a row of one output
// (L = 1, mode same) is a single tap times x[0], so no tap may be much smaller than the others
static double tap(unsigned long long& seed) {
  const double r = rnd(seed);
  return r < 0 ? -0.5 + 0.5 * r : 0.5 + 0.5 * r;
}

// F rows of K taps h (double, zero beyond K) and H = rfft(h, n = N) rounded to T
template <typename T>
static void make_taps(long n, long k, long rows, unsigned long long& seed, std::vector<double>& h, Buf<cpx<T>>& H) {
  const long bins = n / 2 + 1;
  h.assign(rows * k, 0.0);
  for (auto& v : h) v = tap(seed);
  for (long f = 0; f < rows; ++f)
    for (long b = 0; b < bins; ++b) {
      double a = 0, c = 0;
      for (long j = 0; j < k; ++j) {
        double wr, wi;
        host_twiddle((size_t)((b * j) % n), (size_t)n, &wr, &wi);
        a += h[f * k + j] * wr; c += h[f * k + j] * wi;
      }
      H[f * bins + b] = mk<T>((T)a, (T)c);
    }
}

// max over rows of max |y - ref| / max |ref|, ref = the linear convolution of row b with h row b mod rows, outputs
// [off, off + out_len) of the full result
static double lin_err(const std::vector<double>& x, const std::vector<double>& h, const std::vector<double>& y, long L,
                      long k, long off, long out_len, long batch, long rows) {
  double worst = 0;
  for (long b = 0; b < batch; ++b) {
    const double* hf = h.data() + (b % rows) * k;
    double e = 0, r = 0;
    for (long i = 0; i < out_len; ++i) {
      const long t = off + i;
      double s = 0;
      for (long m = std::max(0L, t - L + 1); m < k && m <= t; ++m) s += x[b * L + t - m] * hf[m];
      e = std::max(e, std::fabs(y[b * out_len + i] - s));
      r = std::max(r, std::fabs(s));
    }
    worst = std::max(worst, std::isnan(e) ? INFINITY : e / std::max(r, 1e-300));
  }
  return worst;
}

static const char* kModes[3] = {"full", "same", "valid"};

// the row lengths of one K: 1, S-1, S, S+1, 3S+7 (distinct, >= 1, >= K for valid)
static std::vector<long> row_lengths(long s, long k, int mode) {
  std::vector<long> ls;
  for (long l : {1L, s - 1, s, s + 1, 3 * s + 7})
    if (l >= 1 && (mode != real::kLinearValid || l >= k) && std::find(ls.begin(), ls.end(), l) == ls.end())
      ls.push_back(l);
  return ls;
}

static int report(const char* what, double worst, double tol, long reads, long writes, long missing, long twice) {
  const bool ok = worst < tol && !reads && !writes && !missing && !twice;
  printf("%s: max rel err %.3e, reads outside row %ld, writes outside row %ld, unwritten %ld, written twice %ld %s\n",
         what, worst, reads, writes, missing, twice, ok ? "OK" : "FAIL");
  return !ok;
}

// ---- fused on-chip linear convolution kernel -----------------------------------------------------------------------
template <class K>
static int check_fused(const char* name, double tol) {
  using T = typename K::T;
  constexpr int RA = K::RA, RB = K::RB, E = K::E;
  using V = cpx<T>;
  using Cfg = typename K::template Cfg<true>;
  using Body = onchip::LinConvBody<Cfg>;
  using Tile = typename Cfg::Tile;
  constexpr long L = RA * RB, N = 2 * L, rows = 3;
  int bad = 0;
  const auto twa = twopass::make_twa<T>(RA, RB);
  const auto tab = pair_table<T>(L);
  unsigned long long seed = 2929 + L;
  auto run = [&](long k, int mode, long in_len, long batch, const std::vector<double>& h, const Buf<V>& H) {
    const real::SegMap m = real::linear_map(N, k, mode, in_len);
    const long nseg = batch * m.per;
    Buf<T> x(in_len * batch), y(m.out_len * batch);
    std::vector<double> xd(in_len * batch), yd(m.out_len * batch);
    for (long i = 0; i < in_len * batch; ++i) { x[i] = (T)rnd(seed); xd[i] = x[i]; }
    for (long i = 0; i < m.out_len * batch; ++i) y[i] = (T)NAN;
    typename Body::Args a;
    static_cast<typename onchip::ConvBody<Cfg>::Args&>(a) = {nullptr, nullptr, twa.data(), tab.data(), H.p, rows, m.g0,
                                                             nseg, (T)(1.0 / (2 * N)), m.per};
    a.x = x.p; a.y = y.p; a.m = m;
    check_begin(x.p, y.p, in_len, m.out_len, m.per, batch);
    run_body<Body, Tile, typename Cfg::Lay>(a, (nseg + Cfg::C - 1) / Cfg::C, twa.data());
    long reads, writes, missing, twice;
    check_end(reads, writes, missing, twice);
    for (long i = 0; i < m.out_len * batch; ++i) yd[i] = y[i];
    const double worst = lin_err(xd, h, yd, in_len, k, m.off, m.out_len, batch, rows);
    char what[160];
    snprintf(what, sizeof what, "%s N=%ld K=%ld %s L=%ld F=%ld batch=%ld segments=%ld", name, N, k, kModes[mode], in_len,
             rows, batch, nseg);
    return report(what, worst, tol, reads, writes, missing, twice);
  };
  for (long k : {1L, 2L, 33L, N / 2, N - 1, N}) {
    std::vector<double> h;
    Buf<V> H(rows * (L + 1));
    make_taps<T>(N, k, rows, seed, h, H);
    for (int mode = 0; mode < 3; ++mode)
      for (long in_len : row_lengths(N - k + 1, k, mode)) bad += run(k, mode, in_len, 5, h, H);
    if (k == 33) {   // C + 3 rows of two segments: the last group is partial
      const long s = N - k + 1;
      bad += run(k, real::kLinearFull, s + 1, Cfg::C + 3, h, H);
    }
  }
  // bank conflicts of the shared phases (ConvBody's): the pair step's write-back and the stage-A reads of Z'
  int worst_w = 1, worst_r = 1;
  for (int warp = 0; warp < Cfg::THREADS / 32; ++warp) {
    for (int j = 0; j < E / 2; ++j) {
      std::vector<long> up, down;
      for (int l = 0; l < 32; ++l) {
        const int t = warp * 32 + l;
        const long k = Tile::template u_of<true>(t) + Tile::TP * j;
        up.push_back(Body::Real::park(t) + k);
        down.push_back(k == 0 ? -1 : Body::Real::park(t) + L - k);
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
  // the store's reads of the park as reals: lane u of an FFT reads real lo + u + TP*i, for any lo
  int worst_s = 1;
  for (int warp = 0; warp < Cfg::THREADS / 32; ++warp)
    for (int lo : {0, 1, 32, 33}) {
      std::vector<long> idx;
      for (int l = 0; l < 32; ++l) {
        const int t = warp * 32 + l;
        idx.push_back(2 * Body::Real::park(t) + lo + Tile::template u_of<true>(t));
      }
      worst_s = std::max(worst_s, conflict_degree<(int)sizeof(T)>(idx));
    }
  printf("  lconv    threads %4d  exchange conflicts: write-back x%d, stage-A read x%d, store read x%d\n", Cfg::THREADS,
         worst_w, worst_r, worst_s);
  return bad;
}

// ---- gather / scatter maps of the half-length and full-length paths ------------------------------------------------
// seg -> the circular convolution of each segment with its taps, in double (what convolve_rows computes)
static void circular(std::vector<double>& seg, const real::SegMap& m, long nseg, const std::vector<double>& h,
                     long rows) {
  std::vector<double> tmp(m.n);
  for (long q = 0; q < nseg; ++q) {
    const double* hf = h.data() + (((m.g0 + q) / m.per) % rows) * m.k;
    double* z = seg.data() + q * m.n;
    for (long p = 0; p < m.n; ++p) {
      double s = 0;
      for (long j = 0; j < m.k; ++j) s += z[((p - j) % m.n + m.n) % m.n] * hf[j];
      tmp[p] = s;
    }
    std::copy(tmp.begin(), tmp.end(), z);
  }
}

static int check_maps(long n) {
  int bad = 0;
  const long rows = 3, batch = 5;
  unsigned long long seed = 4343 + n;
  for (long k : {1L, 2L, 33L, n / 2, n - 1, n})
    for (int mode = 0; mode < 3; ++mode)
      for (long in_len : row_lengths(n - k + 1, k, mode)) {
        std::vector<double> h(rows * k);
        for (auto& v : h) v = tap(seed);
        const real::SegMap m = real::linear_map(n, k, mode, in_len);
        const long nseg = batch * m.per;
        std::vector<double> x(in_len * batch), y(m.out_len * batch, NAN), seg(nseg * n);
        for (auto& v : x) v = rnd(seed);
        // device path: two chunks of segments (the second starting at global segment g0 = nseg / 2)
        check_begin(x.data(), y.data(), in_len, m.out_len, m.per, batch);
        for (long c0 : {0L, nseg / 2}) {
          real::SegMap mc = m;
          mc.g0 = c0;
          const long nq = c0 == 0 ? nseg / 2 : nseg - nseg / 2;
          std::vector<double> part(nq * n);
          for (long q = 0; q < nq; ++q)
            for (long p = 0; p < n; ++p) real::gather_one(mc, x.data(), part.data(), q, p);
          circular(part, mc, nq, h, rows);
          for (long q = 0; q < nq; ++q)
            for (long p = 0; p < n; ++p) real::scatter_one(mc, part.data(), y.data(), q, p);
        }
        long reads, writes, missing, twice;
        check_end(reads, writes, missing, twice);
        double worst = lin_err(x, h, y, in_len, k, m.off, m.out_len, batch, rows);
        // host path: runs of at most 2 segments of one row, only the input window [lo, hi) staged
        std::vector<double> yh(m.out_len * batch, NAN);
        long holes = 0;
        for (long b = 0; b < batch; ++b)
          for (long j0 = 0; j0 < m.per; j0 += 2) {
            const long j1 = std::min(m.per, j0 + 2);
            real::SegMap mp = m;
            mp.g0 = b * m.per + j0; mp.r0 = b; mp.out_lo = j0 * m.s;
            mp.lo = std::max(0L, m.off + j0 * m.s - (m.k - 1));
            mp.hi = std::min(in_len, m.off + j1 * m.s);
            const long out_hi = std::min(m.out_len, j1 * m.s);
            std::vector<double> win(x.begin() + b * in_len + std::min(mp.lo, mp.hi), x.begin() + b * in_len + mp.hi);
            std::vector<double> part((j1 - j0) * n), o(out_hi - mp.out_lo, NAN);
            for (long q = 0; q < j1 - j0; ++q)
              for (long p = 0; p < n; ++p) real::gather_one(mp, win.data(), part.data(), q, p);
            circular(part, mp, j1 - j0, h, rows);
            for (long q = 0; q < j1 - j0; ++q)
              for (long p = 0; p < n; ++p) real::scatter_one(mp, part.data(), o.data(), q, p);
            for (long i = 0; i < (long)o.size(); ++i) {
              holes += std::isnan(o[i]);
              yh[b * m.out_len + mp.out_lo + i] = o[i];
            }
          }
        bool same = true;
        for (long i = 0; i < m.out_len * batch; ++i) same &= yh[i] == y[i];
        char what[160];
        snprintf(what, sizeof what, "maps N=%ld K=%ld %s L=%ld F=%ld batch=%ld segments=%ld host runs %s", n, k,
                 kModes[mode], in_len, rows, batch, nseg, same && !holes ? "same" : "DIFFER");
        bad += report(what, worst, 1e-12, reads, writes, missing, twice);
        bad += !(same && !holes);
      }
  return bad;
}

int main() {
  int bad = 0;
  // every on-chip size class (onchip_configs.cuh): L = N/2
  for_each_onchip<float>([&](auto k) { bad += check_fused<decltype(k)>("fused f32", 1e-5); });
  for_each_onchip<double>([&](auto k) { bad += check_fused<decltype(k)>("fused f64", 1e-12); });
  for (long n : {96L, 97L}) bad += check_maps(n);
  printf(bad ? "EMULATION FAILED (%d)\n" : "EMULATION OK\n", bad);
  return bad ? 1 : 0;
}
