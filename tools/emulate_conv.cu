// emulate_conv.cu -- runs the device code of the convolution of real rows, y = irfft(rfft(x) . H) (DESIGN.md §4.11),
// on the CPU, thread by thread and phase by phase (real::conv_pair in real_kernels.cuh and ConvBody in
// onchip_kernels.cuh are __host__ __device__), against a direct circular convolution in double:
//   * the fused on-chip conv kernel for every on-chip size class of both precisions, with F = 3 spectrum rows, a
//     batch of 5 and a batch that is not a multiple of the rows per CTA, starting at spectrum row 0 and 2;
//   * real::conv_pair alone (the half-length path's conv_pair_kernel), for even and odd M = N/2.
// H is the rfft of random real taps h, with random imaginary parts added to bins 0 and N/2 (they must not count).
// Every spectrum access goes through FB_SPEC_ACCESS, which records its address and width: the check fails on any
// access wider than one complex value, misaligned, or outside H, and when no odd row of H (8 bytes off a 16-byte
// boundary for f32) was read.  It also reports the bank-conflict degree of the pair step's write-back into the park
// and of the stage-A reads of Z' from it.
// Build: nvcc -std=c++17 -O1 --expt-relaxed-constexpr -I fourier_b200/csrc tools/emulate_conv.cu \
//             fourier_b200/csrc/host_math.cu (host only, never run on the device)
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>

static void spec_record(const void* p, int bytes);
#ifdef __CUDA_ARCH__
#define FB_SPEC_ACCESS(p, bytes)
#else
#define FB_SPEC_ACCESS(p, bytes) spec_record((const void*)(p), (int)(bytes))
#endif

#include "onchip_kernels.cuh"
#include "plan.h"
#include "tables.cuh"

using namespace fb200;

// ---- spectrum access log ------------------------------------------------------------------------------------------
struct Access { uintptr_t addr; int bytes; };
static std::vector<Access> g_access;
__attribute__((unused)) static void spec_record(const void* p, int bytes) { g_access.push_back({(uintptr_t)p, bytes}); }

// Checks the log against H = [base, base + rows * row_bytes): every access inside it, aligned to its width, at most
// `widest_allowed` bytes wide, and some at odd rows.  Prints one line; returns the number of failures.
static int check_access(const void* base, size_t rows, size_t row_bytes, int widest_allowed) {
  size_t odd = 0, outside = 0, misaligned = 0;
  int widest = 0;
  const uintptr_t b = (uintptr_t)base;
  for (const Access& a : g_access) {
    widest = std::max(widest, a.bytes);
    if (a.addr < b || a.addr + a.bytes > b + rows * row_bytes) { ++outside; continue; }
    if (a.addr % a.bytes) ++misaligned;
    if (((a.addr - b) / row_bytes) % 2 == 1) ++odd;
  }
  const bool ok = !g_access.empty() && widest <= widest_allowed && !outside && !misaligned && odd > 0;
  printf("  H accesses: %zu (%zu at odd rows), widest %d B, misaligned %zu, outside %zu %s\n", g_access.size(), odd,
         widest, misaligned, outside, ok ? "OK" : "FAIL");
  g_access.clear();
  return !ok;
}

// 16-byte aligned storage (what cudaMalloc gives), so that the row offsets are the ones a device buffer would have
template <typename V> struct Buf {
  std::vector<double2> raw;
  V* p;
  explicit Buf(size_t n) : raw((n * sizeof(V) + 15) / 16 + 1), p(reinterpret_cast<V*>(raw.data())) {}
  V& operator[](size_t i) { return p[i]; }
};

static double rnd(unsigned long long& s) {
  s = s * 6364136223846793005ull + 1442695040888963407ull;
  return (double)(s >> 11) / 9007199254740992.0 * 2 - 1;
}

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

// degree of one warp-wide shared access (lanes served in groups of 128 bytes; identical addresses broadcast;
// inactive lanes < 0)
template <int B> static int conflict_degree(const std::vector<long>& idx) {
  const int group = 128 / B;
  int worst = 1;
  for (size_t g = 0; g + group <= idx.size(); g += group) {
    int count[32] = {0};
    std::vector<long> seen;
    for (int l = 0; l < group; ++l) {
      const long e = idx[g + l];
      if (e < 0 || std::find(seen.begin(), seen.end(), e) != seen.end()) continue;
      seen.push_back(e);
      worst = std::max(worst, ++count[(int)((e * B / 4) % 32)]);
    }
  }
  return worst;
}

template <typename T> static std::vector<cpx<T>> pair_table(long m) {
  std::vector<cpx<T>> tab(m / 2 + 1);
  for (long k = 0; k <= m / 2; ++k) {
    double re, im;
    host_twiddle((size_t)k, (size_t)(2 * m), &re, &im);
    tab[k] = mk<T>((T)re, (T)im);
  }
  return tab;
}

// ---- fused on-chip conv kernel --------------------------------------------------------------------------------------
template <typename T, int RA, int RB, int E, int WARPS>
static int check_fused(const char* name, double tol) {
  using V = cpx<T>;
  using Cfg = onchip::OnChipCfg<T, RA, RB, E, WARPS, true>;
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
      const typename Body::Args a = {reinterpret_cast<const V*>(x.p), reinterpret_cast<V*>(y.p), twa.data(), tab.data(),
                                     H.p, rows, row0, batch, (T)(1.0 / (2 * N))};
      std::vector<V> smem(Tile::template smem_elems<typename Cfg::Lay>());
      std::vector<Tile> thr(Cfg::THREADS);
      for (long g = 0; g < (batch + Cfg::C - 1) / Cfg::C; ++g) {
        for (int t = 0; t < Cfg::THREADS; ++t) Body::fwd_phase1(thr[t], a, g, t, smem.data(), twa.data());
        for (int t = 0; t < Cfg::THREADS; ++t) Body::Real::fwd_gather(thr[t], t, smem.data());
        for (int t = 0; t < Cfg::THREADS; ++t) Body::Real::fwd_park(thr[t], t, smem.data());
        for (int t = 0; t < Cfg::THREADS; ++t) Body::pairs(a, g, t, smem.data());
        for (int t = 0; t < Cfg::THREADS; ++t) Body::inv_stage_a(thr[t], t, smem.data(), twa.data());
        for (int t = 0; t < Cfg::THREADS; ++t) Body::inv_scatter(thr[t], t, smem.data());
        for (int t = 0; t < Cfg::THREADS; ++t) Body::inv_store(thr[t], a, g, t, smem.data());
      }
      for (long i = 0; i < N * batch; ++i) yd[i] = y[i];
      const double worst = conv_err(xd, h, yd, N, batch, rows, row0);
      printf("%s N=%ld F=%ld batch=%ld row0=%ld: max rel err vs direct circular convolution %.3e %s\n", name, N, rows,
             batch, row0, worst, worst < tol ? "OK" : "FAIL");
      bad += !(worst < tol);
      bad += check_access(H.p, rows, (L + 1) * sizeof(V), (int)sizeof(V));
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
  std::vector<double> h, x(n * batch), y(n * batch);
  Buf<V> H(rows * (m + 1));
  make_filters<T>(n, rows, seed, h, H);
  for (auto& v : x) v = (T)rnd(seed);
  std::vector<double> wr(m), wi(m);
  for (long j = 0; j < m; ++j) host_twiddle((size_t)j, (size_t)m, &wr[j], &wi[j]);
  std::vector<V> z(m * batch);
  for (long b = 0; b < batch; ++b)
    for (long k = 0; k < m; ++k) {
      double a = 0, c = 0;
      for (long j = 0; j < m; ++j) {
        const double zr = x[b * n + 2 * j], zi = x[b * n + 2 * j + 1], tr = wr[(k * j) % m], ti = wi[(k * j) % m];
        a += zr * tr - zi * ti; c += zr * ti + zi * tr;
      }
      z[b * m + k] = mk<T>((T)a, (T)c);
    }
  for (long b = 0; b < batch; ++b)
    for (long k = 0; k <= m / 2; ++k)
      real::conv_pair(z.data() + b * m, H.p + ((row0 + b) % rows) * (m + 1), m, k, tab.data(), (T)(1.0 / (2 * n)));
  for (long b = 0; b < batch; ++b)   // unscaled inverse FFT_M in double, interleaved
    for (long j = 0; j < m; ++j) {
      double a = 0, c = 0;
      for (long k = 0; k < m; ++k) {
        const V v = z[b * m + k];
        const double tr = wr[(k * j) % m], ti = -wi[(k * j) % m];
        a += v.x * tr - v.y * ti; c += v.x * ti + v.y * tr;
      }
      y[b * n + 2 * j] = a; y[b * n + 2 * j + 1] = c;
    }
  const double worst = conv_err(x, h, y, n, batch, rows, row0);
  printf("%s conv_pair N=%ld (M=%ld): max rel err vs direct circular convolution %.3e %s\n", name, n, m, worst,
         worst < tol ? "OK" : "FAIL");
  int bad = !(worst < tol);
  bad += check_access(H.p, rows, (m + 1) * sizeof(V), (int)sizeof(V));
  return bad;
}

int main() {
  int bad = 0;
  // the on-chip size classes of onchip_lookup (onchip.cu): L = M = N/2
  bad += check_fused<float, 8, 8, 8, 8>("fused f32", 2e-6);
  bad += check_fused<float, 8, 16, 16, 8>("fused f32", 2e-6);
  bad += check_fused<float, 16, 16, 16, 8>("fused f32", 2e-6);
  bad += check_fused<float, 16, 32, 32, 8>("fused f32", 2e-6);
  bad += check_fused<float, 32, 32, 32, 8>("fused f32", 2e-6);
  bad += check_fused<double, 8, 8, 8, 8>("fused f64", 1e-13);
  bad += check_fused<double, 8, 16, 16, 8>("fused f64", 1e-13);
  bad += check_fused<double, 16, 16, 16, 8>("fused f64", 1e-13);
  for (long m : {1L, 2L, 3L, 512L, 1000L, 1009L}) {
    bad += check_pair<float>("pair f32", m, 2e-6);
    bad += check_pair<double>("pair f64", m, 1e-13);
  }
  printf(bad ? "EMULATION FAILED (%d)\n" : "EMULATION OK\n", bad);
  return bad ? 1 : 0;
}
