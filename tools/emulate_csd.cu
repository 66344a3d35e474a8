// emulate_csd.cu -- runs the device code of the cross-spectral density and coherence of real rows (DESIGN.md §4.17) on
// the CPU, warp by warp and phase by phase (CsdBody in onchip_kernels.cuh through the CPU driver run_warp_body, which
// keeps the kernel's barriers between warps; real::WelchItems, spec_pair, cross_terms, csd_out, coherence_out,
// cross_accumulate_one, csd_finish_one and coherence_finish_one in real_kernels.cuh are __host__ __device__), against
// direct sums in double:
//   * the fused kernel and the finish of both outputs for every on-chip size class of both precisions: detrend none and
//     constant, the csd with density (fs = 2.5) and spectrum scaling, hops 1, N/4, N and N+3, rows of F = 1, F < C/2,
//     F = B-1, B, B+1 and 2B+3 frames at hop N/4 (B = real::welch_block(F, C/2)), F < C/2 and B+1 at the other hops,
//     y_rows 1 and y_rows = batch.  The inputs carry a random DC offset; y is a filtered copy of x plus independent
//     noise, so no bin's coherence is near 0/0.  The batches of short rows leave a partial group;
//   * for N = 96 and 97 the accumulate and finish element functions of the other paths over two chunks of frames, one
//     item straddling the cut, against the direct sums.
// Every x and y read and every partial and output write is logged: the check fails on a read outside the frame's own x
// row (b) or y row (b mod y_rows), and on a partial or output written zero times or twice.  It also reports the
// bank-conflict degree of the cross phase's park reads and accumulator updates and of the flush's reads.
// Build: nvcc -std=c++17 -O1 --expt-relaxed-constexpr -I fourier_b200/csrc tools/emulate_csd.cu \
//             fourier_b200/csrc/host_math.cu (host only, never run on the device)
#include <complex>
#include <cstdint>
#include <string>
#include <vector>

static void lin_record(int write, const void* p, long g);
#ifdef __CUDA_ARCH__
#define FB_LIN_ACCESS(w, p, g)
#else
#define FB_LIN_ACCESS(w, p, g) lin_record((w), (const void*)(p), (long)(g))
#endif

#include "emulate_common.h"

// ---- access log: checked as it happens --------------------------------------------------------------------------------
// reads: g is the frame of the launch, whose row b = g / frames must hold the sample (x row b or y row b mod y_rows);
// writes: into the partials or the (real) output; the csd's complex output is written through spec_st (g_access)
struct CsdCheck {
  bool on = false;
  uintptr_t x = 0, y = 0, part = 0, out = 0;
  long esz = 0, in_len = 0, frames = 1, y_rows = 1, n_part = 0, n_out = 0;
  long bad_reads = 0, bad_writes = 0, x_reads = 0, y_reads = 0;
  std::vector<int> part_writes, out_writes;
};
static CsdCheck g_chk;

static bool in_row(uintptr_t base, const void* p, long row) {
  const intptr_t d = (intptr_t)p - (intptr_t)base;
  const long e = (long)(d / g_chk.esz);
  return d >= 0 && d % g_chk.esz == 0 && e >= row * g_chk.in_len && e < (row + 1) * g_chk.in_len;
}
static void lin_record(int write, const void* p, long g) {
  if (!g_chk.on) return;
  if (!write) {
    const long b = g / g_chk.frames;
    if (in_row(g_chk.x, p, b)) ++g_chk.x_reads;
    else if (in_row(g_chk.y, p, b % g_chk.y_rows)) ++g_chk.y_reads;
    else ++g_chk.bad_reads;
    return;
  }
  const intptr_t dp = (intptr_t)p - (intptr_t)g_chk.part, dq = (intptr_t)p - (intptr_t)g_chk.out;
  if (g_chk.part && dp >= 0 && dp % g_chk.esz == 0 && dp / g_chk.esz < g_chk.n_part) ++g_chk.part_writes[dp / g_chk.esz];
  else if (dq >= 0 && dq % g_chk.esz == 0 && dq / g_chk.esz < g_chk.n_out) ++g_chk.out_writes[dq / g_chk.esz];
  else ++g_chk.bad_writes;
}
// the csd's output writes from the spectrum log: each complex element once
static void count_spec_writes(size_t csz) {
  for (const Access& a : g_access) {
    const intptr_t d = (intptr_t)a.addr - (intptr_t)g_chk.out;
    if (d >= 0 && d % (intptr_t)csz == 0 && d / (intptr_t)csz < g_chk.n_out && a.bytes == (int)csz)
      ++g_chk.out_writes[d / csz];
    else ++g_chk.bad_writes;
  }
  g_access.clear();
}
static long not_once() {
  long bad = g_chk.bad_writes;
  for (int c : g_chk.part_writes) bad += c != 1;
  for (int c : g_chk.out_writes) bad += c != 1;
  return bad;
}

static const char* kDetrend[2] = {"none", "constant"};
using cd = std::complex<double>;

// rfft(w . (frame - mean)) of one frame in double, directly
static void frame_spectrum(const double* x, const std::vector<double>& w, const std::vector<double>& wr,
                           const std::vector<double>& wi, long n, bool detrend, cd* s) {
  double mu = 0;
  if (detrend) {
    for (long p = 0; p < n; ++p) mu += x[p];
    mu /= (double)n;
  }
  std::vector<double> u(n);
  for (long p = 0; p < n; ++p) u[p] = (x[p] - mu) * w[p];
  for (long k = 0; k <= n / 2; ++k) {
    double re = 0, im = 0;
    for (long p = 0, j = 0; p < n; ++p, j = j + k >= n ? j + k - n : j + k) { re += u[p] * wr[j]; im += u[p] * wi[j]; }
    s[k] = cd(re, im);
  }
}

// ---- fused on-chip kernel and the finish -------------------------------------------------------------------------------
template <class K, bool COH>
static int run_fused(const char* name, double tol, double& worst_seen) {
  using T = typename K::T;
  constexpr int RA = K::RA, RB = K::RB;
  using V = cpx<T>;
  using Cfg = typename K::template Cfg<true>;
  using Body = onchip::CsdBody<Cfg, COH>;
  using Tile = typename Cfg::Tile;
  constexpr long L = RA * RB, N = 2 * L, bins = L + 1, C = Cfg::C, PAIRS = C / 2, PL = Body::PLANES;
  int bad = 0, partial = 0;
  const auto twa = twopass::make_twa<T>(RA, RB);
  const auto tab = pair_table<T>(L);
  std::vector<double> wr, wi;
  twiddles(N, wr, wi);
  unsigned long long seed = 9127 + N + (COH ? 1 : 0);
  Buf<T> win(N);
  std::vector<double> wd(N);
  double sw = 0, sw2 = 0;
  for (long p = 0; p < N; ++p) {
    win[p] = (T)(0.5 + 0.5 * rnd(seed));
    wd[p] = win[p];
    sw += wd[p];
    sw2 += wd[p] * wd[p];
  }
  std::vector<std::pair<long, long>> cases;
  for (long hop : {1L, N / 4, N, N + 3}) {
    const long f_small = PAIRS / 2 + 1, b_long = real::welch_block(PAIRS + 1, PAIRS);
    if (hop == N / 4)
      for (long f : {1L, f_small, b_long - 1, b_long, b_long + 1, 2 * b_long + 3}) cases.push_back({hop, f});
    else
      for (long f : {f_small, b_long + 1}) cases.push_back({hop, f});
  }
  for (const auto& hc : cases) {
    const long hop = hc.first, F = hc.second, in_len = N + (F - 1) * hop + hop / 2;
    const real::FrameMap m = real::frame_map(N, in_len, hop, real::kStftNone);
    if (m.frames != F) { printf("fused %s N=%ld: F=%ld gave %ld frames FAIL\n", name, N, F, m.frames); ++bad; continue; }
    const real::WelchItems w1 = real::welch_items(F, PAIRS, 1);
    const long batch = w1.per_group > 1 ? w1.per_group + 1 : 2;
    Buf<T> x(in_len * batch), y(in_len * batch);
    const double dc = 3.0 * rnd(seed);
    for (long i = 0; i < in_len * batch; ++i) x[i] = (T)(dc + rnd(seed));
    for (long i = 0; i < in_len * batch; ++i) {
      const long t = i % in_len;
      y[i] = (T)(0.6 * (x[i] - dc) + (t > 0 ? 0.3 * (x[i - 1] - dc) : 0.0) + 0.5 * rnd(seed) - dc / 2);
    }
    const real::WelchItems w = real::welch_items(F, PAIRS, batch);
    // (detrend, scaling, y_rows): csd density with fs = 2.5 or spectrum; the coherence ignores the scaling
    for (int v = 0; v < 2; ++v) {
      const int detrend = v == 0 ? real::kDetrendConstant : real::kDetrendNone;
      const int scaling = v == 0 ? real::kWelchDensity : real::kWelchSpectrum;
      const double fs = v == 0 ? 2.5 : 1.0;
      const long y_rows = v == 0 ? 1 : batch;
      // the direct sums of conj(X) Y, |X|^2 and |Y|^2
      std::vector<cd> sxy(batch * bins, 0.0);
      std::vector<double> sxx(batch * bins, 0.0), syy(batch * bins, 0.0);
      std::vector<double> xd(N), yd(N);
      std::vector<cd> X(bins), Y(bins);
      for (long b = 0; b < batch; ++b)
        for (long f = 0; f < F; ++f) {
          for (long p = 0; p < N; ++p) {
            xd[p] = x[b * in_len + f * hop + p];
            yd[p] = y[(b % y_rows) * in_len + f * hop + p];
          }
          frame_spectrum(xd.data(), wd, wr, wi, N, detrend == real::kDetrendConstant, X.data());
          frame_spectrum(yd.data(), wd, wr, wi, N, detrend == real::kDetrendConstant, Y.data());
          for (long k = 0; k < bins; ++k) {
            sxy[b * bins + k] += std::conj(X[k]) * Y[k];
            sxx[b * bins + k] += std::norm(X[k]);
            syy[b * bins + k] += std::norm(Y[k]);
          }
        }
      const T base = (T)real::welch_base(sw, sw2, scaling, fs, F);
      Buf<T> part(w.total() * PL * bins);
      Buf<V> out_c(batch * bins);
      Buf<T> out_r(batch * bins);
      for (long i = 0; i < w.total() * PL * bins; ++i) part[i] = (T)NAN;
      for (long i = 0; i < batch * bins; ++i) { out_c[i] = mk<T>((T)NAN, (T)NAN); out_r[i] = (T)NAN; }
      onchip::CsdArgs<Cfg> a;
      static_cast<typename onchip::RealBody<Cfg>::Args&>(a) = {nullptr, nullptr, twa.data(), tab.data(), 0, (T)0.5};
      a.x = x.p; a.win = win.p; a.m = m;
      a.part = part.p; a.psd = COH ? out_r.p : (T*)out_c.p; a.base = &base; a.w = w; a.detrend = detrend;
      a.y = y.p; a.y_rows = y_rows; a.y_off = 0; a.y_rcp = 1.0 / (double)y_rows;
      g_chk.on = true;
      g_chk.x = (uintptr_t)x.p; g_chk.y = (uintptr_t)y.p;
      g_chk.part = w.items > 1 ? (uintptr_t)part.p : 0; g_chk.out = COH ? (uintptr_t)out_r.p : (uintptr_t)out_c.p;
      g_chk.esz = sizeof(T); g_chk.in_len = in_len; g_chk.frames = F; g_chk.y_rows = y_rows;
      g_chk.n_part = w.items > 1 ? w.total() * PL * bins : 0; g_chk.n_out = batch * bins;
      g_chk.bad_reads = g_chk.bad_writes = g_chk.x_reads = g_chk.y_reads = 0;
      g_chk.part_writes.assign(g_chk.n_part, 0);
      g_chk.out_writes.assign(g_chk.n_out, 0);
      g_access.clear();
      if (!COH) g_chk.esz = sizeof(T);
      run_warp_body<Body, Tile, typename Cfg::Lay>(a, twa.data());
      if (w.items > 1)   // cross_finish_kernel
        for (long b = 0; b < batch; ++b)
          for (long k = 0; k < bins; ++k) {
            if (COH) real::coherence_finish_one(part.p, w.items, N, out_r.p, b, k);
            else real::csd_finish_one(part.p, w.items, N, base, out_c.p, b, k);
          }
      if (!COH) count_spec_writes(sizeof(V));
      g_chk.on = false;
      const long extra = not_once();
      const bool reads_ok = !g_chk.bad_reads && g_chk.x_reads > 0 && g_chk.y_reads > 0;
      const double s = real::welch_base(sw, sw2, scaling, fs, F);
      double worst = 0;
      bool edges = true;
      for (long b = 0; b < batch; ++b) {
        double e = 0, r = 0;
        for (long k = 0; k < bins; ++k) {
          if (COH) {
            const double ref = std::norm(sxy[b * bins + k]) / (sxx[b * bins + k] * syy[b * bins + k]);
            const double got = out_r[b * bins + k];
            e = std::max(e, std::isnan(got) ? INFINITY : std::fabs(got - ref));
            r = 1;
          } else {
            const cd ref = (double)real::welch_factor(N, k) * s * sxy[b * bins + k];
            const V g = out_c[b * bins + k];
            e = std::max(e, std::isnan(g.x) || std::isnan(g.y) ? INFINITY : std::abs(cd(g.x, g.y) - ref));
            r = std::max(r, std::abs(ref));
            if ((k == 0 || k == L) && (g.y != 0 || std::signbit(g.y))) edges = false;
          }
        }
        worst = std::max(worst, e / std::max(r, 1e-300));
      }
      worst_seen = std::max(worst_seen, worst);
      const bool part_group = w.total() % w.per_group != 0;
      partial += part_group;
      const bool ok = worst < tol && reads_ok && !extra && edges;
      printf("fused %s %s N=%ld H=%ld L=%ld batch=%ld y_rows=%ld F=%ld B=%ld items=%ld per_group=%ld detrend=%s "
             "scaling=%s%s: max %s err %.3e, outside row %ld, not once %ld, im edges %s %s\n",
             COH ? "coherence" : "csd", name, N, hop, in_len, batch, y_rows, F, w.block, w.items, w.per_group,
             kDetrend[detrend], COH ? "none" : scaling == real::kWelchDensity ? "density" : "spectrum",
             part_group ? " partial" : "", COH ? "abs" : "rel", worst, g_chk.bad_reads, extra, edges ? "+0" : "BAD",
             ok ? "OK" : "FAIL");
      bad += !ok;
    }
  }
  if (!partial) { printf("fused %s N=%ld: no batch left a partial group FAIL\n", name, N); ++bad; }
  // shared-memory bank conflicts per warp: the cross phase's park reads (lane u of column c reads z[k] of both parks
  // of its pair, k = u + TP (2 jj + side)), its accumulator updates (planes of L+1 per pair column) and the flush's
  // reads (thread o reads bin o mod (L+1) of each plane of an item's pair columns)
  int worst_z = 1, worst_a = 1, worst_f = 1;
  for (int warp = 0; warp < Cfg::THREADS / 32; ++warp) {
    auto lane_t = [&](int l) { return warp * 32 + l; };
    auto u_of = [&](int l) { return (long)Tile::template u_of<true>(lane_t(l)); };
    auto col_of = [&](int l) { return (long)Tile::template col_of<true>(lane_t(l)); };
    for (int jj = 0; jj < Tile::E / 4; ++jj) {
      std::vector<long> zk, zm, up, down;
      for (int l = 0; l < 32; ++l) {
        const long c = col_of(l), side = c & 1, k = u_of(l) + Tile::TP * (2 * jj + side);
        const long park = (c - side) * Cfg::Lay::SC;
        zk.push_back(park + k);
        zm.push_back(park + L - k);
        up.push_back((c >> 1) * PL * bins + k);
        down.push_back((c >> 1) * PL * bins + L - k);
      }
      worst_z = std::max({worst_z, conflict_degree<(int)sizeof(V)>(zk), conflict_degree<(int)sizeof(V)>(zm)});
      worst_a = std::max({worst_a, conflict_degree<(int)sizeof(T)>(up), conflict_degree<(int)sizeof(T)>(down)});
    }
    for (int c = 0; c < PAIRS; ++c) {
      std::vector<long> idx;
      for (int l = 0; l < 32; ++l) idx.push_back(c * PL * bins + lane_t(l) % bins);
      worst_f = std::max(worst_f, conflict_degree<(int)sizeof(T)>(idx));
    }
  }
  printf("  %s threads %4d  conflicts: park read x%d; accumulate x%d; flush read x%d\n", COH ? "coherence" : "csd",
         Cfg::THREADS, worst_z, worst_a, worst_f);
  return bad;
}

// ---- the other paths' accumulate and finish elements, N = 96 and 97 ---------------------------------------------------
static int check_elements(long n, bool coh) {
  using V = cpx<double>;
  const long bins = n / 2 + 1, F = 7, rows = 2, total = rows * F;
  const int planes = coh ? real::kCoherencePlanes : real::kCsdPlanes;
  const real::WelchItems w = real::welch_items(F, 1, rows);
  unsigned long long seed = 5501 + n;
  // the x spectra, then the y spectra, as seg_ holds them
  Buf<V> spec(2 * total * bins);
  for (long i = 0; i < 2 * total * bins; ++i) spec[i] = mk<double>(rnd(seed), rnd(seed));
  const V* sx = spec.p;
  const V* sy = spec.p + total * bins;
  const double base = 0.375;
  std::vector<double> part(w.total() * planes * bins, NAN), yr(rows * bins, NAN);
  Buf<V> yc(rows * bins);
  g_access.clear();
  // two chunks of frames, [0, 5) and [5, 14): the second item of row 0 spans both
  for (long q0 : {0L, 5L}) {
    const long nq = q0 == 0 ? 5 : total - 5;
    for (long i = 0; i < w.total(); ++i)
      for (long k = 0; k < bins; ++k) {
        const long b = i / w.items;
        real::cross_accumulate_one(sx + q0 * bins, sy + q0 * bins, bins, q0, nq,
                                   b * F + (i - b * w.items) * w.block, w.count(i), planes, part.data(), i, k);
      }
  }
  int bad = check_access(coh ? "coherence spectra" : "csd spectra", spec.p, 2 * total, bins * sizeof(V), (int)sizeof(V));
  for (long b = 0; b < rows; ++b)
    for (long k = 0; k < bins; ++k) {
      if (coh) real::coherence_finish_one(part.data(), w.items, n, yr.data(), b, k);
      else real::csd_finish_one(part.data(), w.items, n, base, yc.p, b, k);
    }
  g_access.clear();
  double e = 0, r = 0;
  for (long b = 0; b < rows; ++b)
    for (long k = 0; k < bins; ++k) {
      cd s = 0;
      double xx = 0, yy = 0;
      for (long f = 0; f < F; ++f) {
        const V a = sx[(b * F + f) * bins + k], c = sy[(b * F + f) * bins + k];
        s += std::conj(cd(a.x, a.y)) * cd(c.x, c.y);
        xx += a.x * a.x + a.y * a.y;
        yy += c.x * c.x + c.y * c.y;
      }
      if (coh) {
        const double ref = std::norm(s) / (xx * yy), got = yr[b * bins + k];
        e = std::max(e, std::isnan(got) ? INFINITY : std::fabs(got - ref));
        r = 1;
      } else {
        cd ref = (double)real::welch_factor(n, k) * base * s;
        if (k == 0 || 2 * k == n) ref = cd(ref.real(), 0.0);
        const V g = yc[b * bins + k];
        e = std::max(e, std::isnan(g.x) || std::isnan(g.y) ? INFINITY : std::abs(cd(g.x, g.y) - ref));
        r = std::max(r, std::abs(ref));
      }
    }
  const bool ok = e / r < 1e-12 && w.items == 2;
  printf("elements %s N=%ld F=%ld B=%ld items=%ld chunks=2: max err %.3e %s\n", coh ? "coherence" : "csd", n, F,
         w.block, w.items, e / r, ok ? "OK" : "FAIL");
  return bad + !ok;
}

int main() {
  int bad = 0;
  double w32[2] = {0, 0}, w64[2] = {0, 0};
  // every on-chip size class (onchip_configs.cuh): L = N/2.  The f32 coherence is held to 5e-5: a ratio of sums of
  // products, it carries the FFT's relative error of each frame's weaker bins, which grows with N (1.6e-5 measured at
  // N = 512 to 2048 on rows of 3 to 17 frames).
  for_each_onchip<float>([&](auto k) {
    bad += run_fused<decltype(k), false>("f32", 1e-5, w32[0]);
    bad += run_fused<decltype(k), true>("f32", 5e-5, w32[1]);
  });
  for_each_onchip<double>([&](auto k) {
    bad += run_fused<decltype(k), false>("f64", 1e-12, w64[0]);
    bad += run_fused<decltype(k), true>("f64", 1e-12, w64[1]);
  });
  printf("worst: csd f32 %.3e f64 %.3e (relative to the row's max |P|); coherence f32 %.3e f64 %.3e (absolute)\n",
         w32[0], w64[0], w32[1], w64[1]);
  for (long n : {96L, 97L})
    for (bool coh : {false, true}) bad += check_elements(n, coh);
  printf(bad ? "EMULATION FAILED (%d)\n" : "EMULATION OK\n", bad);
  return bad ? 1 : 0;
}
