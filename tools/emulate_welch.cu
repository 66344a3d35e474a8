// emulate_welch.cu -- runs the device code of the Welch power spectral density of real rows (DESIGN.md §4.15) on the
// CPU, thread by thread and phase by phase (WelchBody in onchip_kernels.cuh through the CPU driver run_welch_body;
// real::WelchItems, welch_out, welch_accumulate_one and welch_finish_one in real_kernels.cuh are __host__ __device__),
// against direct sums in double:
//   * the fused kernel and the finish for every on-chip size class of both precisions, detrend none and constant,
//     scaling density with fs = 1 and 2.5 and spectrum, hops 1, N/4, N/2, N and N+3, and rows of F = 1, F < C,
//     F = B-1, B, B+1 and 2B+3 frames (B = real::welch_block(F, C)) at hop N/4, F < C and B+1 at the other hops.  The
//     batches of short rows leave a partial group.  The reference is a direct windowed DFT of every frame, the mean
//     taken off first, |.|^2 averaged with the one-sided factor and the scale;
//   * for N = 96 and 97 the accumulate and finish element functions of the other paths over two chunks of frames,
//     against the direct sum of the frames' powers.
// Every input read and every partial and output write goes through FB_LIN_ACCESS: the check fails on a read outside
// the frame's row and on a partial or output written zero times or twice.  It also reports the bank-conflict degree of
// the shared accesses: the park write and stage-A read of the load, the accumulator update and the flush's reads.
// Build: nvcc -std=c++17 -O1 --expt-relaxed-constexpr -I fourier_b200/csrc tools/emulate_welch.cu \
//             fourier_b200/csrc/host_math.cu (host only, never run on the device)
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

// ---- access log: checked as it happens ------------------------------------------------------------------------------
// reads: g is the frame of the launch, whose row g / frames must hold the sample; writes: into the partials or the output
struct WelchCheck {
  bool on = false;
  uintptr_t x = 0, part = 0, out = 0;
  long esz = 0, in_len = 0, frames = 1, n_part = 0, n_out = 0;
  long bad_reads = 0, bad_writes = 0;
  std::vector<int> part_writes, out_writes;
};
static WelchCheck g_chk;

static void lin_record(int write, const void* p, long g) {
  if (!g_chk.on) return;
  if (!write) {
    const intptr_t d = (intptr_t)p - (intptr_t)g_chk.x;
    const long e = (long)(d / g_chk.esz), row = g / g_chk.frames;
    if (d % g_chk.esz || d < 0 || e < row * g_chk.in_len || e >= (row + 1) * g_chk.in_len) ++g_chk.bad_reads;
    return;
  }
  const intptr_t dp = (intptr_t)p - (intptr_t)g_chk.part, dq = (intptr_t)p - (intptr_t)g_chk.out;
  if (g_chk.part && dp >= 0 && dp % g_chk.esz == 0 && dp / g_chk.esz < g_chk.n_part) ++g_chk.part_writes[dp / g_chk.esz];
  else if (dq >= 0 && dq % g_chk.esz == 0 && dq / g_chk.esz < g_chk.n_out) ++g_chk.out_writes[dq / g_chk.esz];
  else ++g_chk.bad_writes;
}
static long not_once() {
  long bad = g_chk.bad_writes;
  for (int c : g_chk.part_writes) bad += c != 1;
  for (int c : g_chk.out_writes) bad += c != 1;
  return bad;
}

static const char* kDetrend[2] = {"none", "constant"};
static const char* kScaling[2] = {"density", "spectrum"};

// |rfft(w . (frame - mean))|^2 of one frame in double, directly
static void frame_powers(const double* x, const std::vector<double>& w, const std::vector<double>& wr,
                         const std::vector<double>& wi, long n, bool detrend, double* pw) {
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
    pw[k] = re * re + im * im;
  }
}

// ---- fused on-chip Welch kernel and the finish ------------------------------------------------------------------------
template <class K>
static int check_fused(const char* name, double tol) {
  using T = typename K::T;
  constexpr int RA = K::RA, RB = K::RB;
  using V = cpx<T>;
  using Cfg = typename K::template Cfg<true>;
  using Body = onchip::WelchBody<Cfg>;
  using Tile = typename Cfg::Tile;
  constexpr long L = RA * RB, N = 2 * L, bins = L + 1, C = Cfg::C;
  int bad = 0, partial = 0;
  const auto twa = twopass::make_twa<T>(RA, RB);
  const auto tab = pair_table<T>(L);
  std::vector<double> wr, wi;
  twiddles(N, wr, wi);
  unsigned long long seed = 7717 + N;
  Buf<T> win(N);
  std::vector<double> wd(N);
  double sw = 0, sw2 = 0;
  for (long p = 0; p < N; ++p) {
    win[p] = (T)(0.5 + 0.5 * rnd(seed));
    wd[p] = win[p];
    sw += wd[p];
    sw2 += wd[p] * wd[p];
  }
  // (hop, F): every frame count at hop N/4, F < C and B+1 at the others
  std::vector<std::pair<long, long>> cases;
  for (long hop : {1L, N / 4, N / 2, N, N + 3}) {
    const long fs_small = C / 2 + 1, b_long = real::welch_block(C + 1, C);
    if (hop == N / 4)
      for (long f : {1L, fs_small, b_long - 1, b_long, b_long + 1, 2 * b_long + 3}) cases.push_back({hop, f});
    else
      for (long f : {fs_small, b_long + 1}) cases.push_back({hop, f});
  }
  for (const auto& hc : cases) {
    const long hop = hc.first, F = hc.second, in_len = N + (F - 1) * hop + hop / 2;
    const real::FrameMap m = real::frame_map(N, in_len, hop, real::kStftNone);
    if (m.frames != F) { printf("fused %s N=%ld: F=%ld gave %ld frames FAIL\n", name, N, F, m.frames); ++bad; continue; }
    const real::WelchItems w1 = real::welch_items(F, C, 1);
    // short rows: one row more than fills whole groups, so the last group is partial; long rows: 2 rows
    const long batch = w1.per_group > 1 ? w1.per_group + 1 : 2;
    Buf<T> x(in_len * batch);
    std::vector<double> xd(in_len * batch);
    const double dc = 3.0 * rnd(seed);
    for (long i = 0; i < in_len * batch; ++i) { x[i] = (T)(dc + rnd(seed)); xd[i] = x[i]; }
    // the direct sums of the frames' powers, per detrend
    std::vector<double> sum[2] = {std::vector<double>(batch * bins, 0.0), std::vector<double>(batch * bins, 0.0)};
    std::vector<double> pw(bins);
    for (int d = 0; d < 2; ++d)
      for (long b = 0; b < batch; ++b)
        for (long f = 0; f < F; ++f) {
          frame_powers(xd.data() + b * in_len + f * hop, wd, wr, wi, N, d == 1, pw.data());
          for (long k = 0; k < bins; ++k) sum[d][b * bins + k] += pw[k];
        }
    const real::WelchItems w = real::welch_items(F, C, batch);
    for (int detrend = 0; detrend < 2; ++detrend)
      for (int sc = 0; sc < 3; ++sc) {
        const int scaling = sc == 2 ? real::kWelchSpectrum : real::kWelchDensity;
        const double fs = sc == 1 ? 2.5 : 1.0;
        const T base = (T)real::welch_base(sw, sw2, scaling, fs, F);
        Buf<T> part(w.total() * bins), y(batch * bins);
        for (long i = 0; i < w.total() * bins; ++i) part[i] = (T)NAN;
        for (long i = 0; i < batch * bins; ++i) y[i] = (T)NAN;
        typename Body::Args a;
        static_cast<typename onchip::RealBody<Cfg>::Args&>(a) = {nullptr, nullptr, twa.data(), tab.data(), 0, (T)0.5};
        a.x = x.p; a.win = win.p; a.m = m;
        a.part = part.p; a.psd = y.p; a.base = &base; a.w = w; a.detrend = detrend;
        g_chk.on = true;
        g_chk.x = (uintptr_t)x.p; g_chk.part = w.items > 1 ? (uintptr_t)part.p : 0; g_chk.out = (uintptr_t)y.p;
        g_chk.esz = sizeof(T); g_chk.in_len = in_len; g_chk.frames = F;
        g_chk.n_part = w.items > 1 ? w.total() * bins : 0; g_chk.n_out = batch * bins;
        g_chk.bad_reads = g_chk.bad_writes = 0;
        g_chk.part_writes.assign(g_chk.n_part, 0);
        g_chk.out_writes.assign(g_chk.n_out, 0);
        run_welch_body<Body, Tile, typename Cfg::Lay>(a, twa.data());
        if (w.items > 1)   // welch_finish_kernel
          for (long b = 0; b < batch; ++b)
            for (long k = 0; k < bins; ++k) real::welch_finish_one(part.p, w.items, N, base, y.p, b, k);
        g_chk.on = false;
        const long extra = not_once();
        const double s = real::welch_base(sw, sw2, scaling, fs, F);
        double worst = 0;
        for (long b = 0; b < batch; ++b) {
          double e = 0, r = 0;
          for (long k = 0; k < bins; ++k) {
            const double ref = real::welch_factor(N, k) * s * sum[detrend][b * bins + k], got = y[b * bins + k];
            e = std::max(e, std::isnan(got) ? INFINITY : std::fabs(got - ref));
            r = std::max(r, std::fabs(ref));
          }
          worst = std::max(worst, e / std::max(r, 1e-300));
        }
        const bool part_group = w.total() % w.per_group != 0;
        partial += part_group;
        const bool ok = worst < tol && !g_chk.bad_reads && !extra;
        printf("fused %s N=%ld H=%ld L=%ld batch=%ld F=%ld B=%ld items=%ld per_group=%ld detrend=%s scaling=%s fs=%g%s: "
               "max rel err %.3e, outside row %ld, not once %ld %s\n",
               name, N, hop, in_len, batch, F, w.block, w.items, w.per_group, kDetrend[detrend], kScaling[scaling], fs,
               part_group ? " partial" : "", worst, g_chk.bad_reads, extra, ok ? "OK" : "FAIL");
        bad += !ok;
      }
  }
  if (!partial) { printf("fused %s N=%ld: no batch left a partial group FAIL\n", name, N); ++bad; }
  // shared-memory bank conflicts per warp: the load's park write (lane u writes sample u + TP*j) and stage-A read, the
  // accumulator update (lane u updates u + TP*j and L - u - TP*j of its column's row, lane 0 also L/2) and the flush's
  // reads (thread o reads bin o mod (L+1) of an item's columns)
  int worst_w = 1, worst_r = 1, worst_a = 1, worst_f = 1;
  for (int warp = 0; warp < Cfg::THREADS / 32; ++warp) {
    auto lane_t = [&](int l) { return warp * 32 + l; };
    auto u_of = [&](int l) { return Tile::template u_of<true>(lane_t(l)); };
    auto col_of = [&](int l) { return (long)Tile::template col_of<true>(lane_t(l)); };
    auto park2 = [&](int l) { return 2L * Body::Real::park(lane_t(l)); };
    for (int j = 0; j < 2 * L / Tile::TP; ++j) {
      std::vector<long> idx;
      for (int l = 0; l < 32; ++l) idx.push_back(park2(l) + u_of(l) + Tile::TP * j);
      worst_w = std::max(worst_w, conflict_degree<(int)sizeof(T)>(idx));
    }
    for (int q = 0; q < Tile::NA; ++q)
      for (int i = 0; i < RA; ++i) {
        std::vector<long> idx;
        for (int l = 0; l < 32; ++l) idx.push_back(Body::Real::park(lane_t(l)) + u_of(l) + Tile::TP * q + RB * i);
        worst_r = std::max(worst_r, conflict_degree<(int)sizeof(V)>(idx));
      }
    for (int j = 0; j < Tile::E / 2; ++j) {
      std::vector<long> up, down;
      for (int l = 0; l < 32; ++l) {
        up.push_back(col_of(l) * bins + u_of(l) + Tile::TP * j);
        down.push_back(col_of(l) * bins + L - (u_of(l) + Tile::TP * j));
      }
      worst_a = std::max({worst_a, conflict_degree<(int)sizeof(T)>(up), conflict_degree<(int)sizeof(T)>(down)});
    }
    for (int c = 0; c < C; ++c) {
      std::vector<long> idx;
      for (int l = 0; l < 32; ++l) idx.push_back(c * bins + lane_t(l) % bins);
      worst_f = std::max(worst_f, conflict_degree<(int)sizeof(T)>(idx));
    }
  }
  printf("  welch    threads %4d  conflicts: park write x%d, stage-A read x%d; accumulate x%d; flush read x%d\n",
         Cfg::THREADS, worst_w, worst_r, worst_a, worst_f);
  return bad;
}

// ---- the other paths' accumulate and finish elements, N = 96 and 97 ---------------------------------------------------
static int check_elements(long n) {
  using V = cpx<double>;
  const long bins = n / 2 + 1, F = 7, rows = 2, total = rows * F;
  const real::WelchItems w = real::welch_items(F, 1, rows);
  unsigned long long seed = 4409 + n;
  Buf<V> spec(total * bins);
  for (long i = 0; i < total * bins; ++i) spec[i] = mk<double>(rnd(seed), rnd(seed));
  const double base = 0.375;
  std::vector<double> part(w.total() * bins, NAN), y(rows * bins, NAN);
  g_access.clear();
  // two chunks of frames, [0, 5) and [5, 14): the second item of row 0 spans both
  for (long q0 : {0L, 5L}) {
    const long nq = q0 == 0 ? 5 : total - 5;
    for (long i = 0; i < w.total(); ++i)
      for (long k = 0; k < bins; ++k) {
        const long b = i / w.items;
        real::welch_accumulate_one(spec.p + q0 * bins, bins, q0, nq, b * F + (i - b * w.items) * w.block, w.count(i),
                                   part.data(), i, k);
      }
  }
  for (long b = 0; b < rows; ++b)
    for (long k = 0; k < bins; ++k) real::welch_finish_one(part.data(), w.items, n, base, y.data(), b, k);
  int bad = check_access("welch spectra", spec.p, total, bins * sizeof(V), (int)sizeof(V));
  double e = 0, r = 0;
  for (long b = 0; b < rows; ++b)
    for (long k = 0; k < bins; ++k) {
      double s = 0;
      for (long f = 0; f < F; ++f) {
        const V v = spec[(b * F + f) * bins + k];
        s += v.x * v.x + v.y * v.y;
      }
      const double ref = real::welch_factor(n, k) * base * s, got = y[b * bins + k];
      e = std::max(e, std::isnan(got) ? INFINITY : std::fabs(got - ref));
      r = std::max(r, std::fabs(ref));
    }
  const bool ok = e / r < 1e-12 && w.items == 2;
  printf("elements N=%ld F=%ld B=%ld items=%ld chunks=2: max rel err %.3e %s\n", n, F, w.block, w.items, e / r,
         ok ? "OK" : "FAIL");
  return bad + !ok;
}

int main() {
  int bad = 0;
  // every on-chip size class (onchip_configs.cuh): L = N/2
  for_each_onchip<float>([&](auto k) { bad += check_fused<decltype(k)>("f32", 1e-5); });
  for_each_onchip<double>([&](auto k) { bad += check_fused<decltype(k)>("f64", 1e-12); });
  for (long n : {96L, 97L}) bad += check_elements(n);
  printf(bad ? "EMULATION FAILED (%d)\n" : "EMULATION OK\n", bad);
  return bad ? 1 : 0;
}
