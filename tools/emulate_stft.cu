// emulate_stft.cu -- runs the device code of the short-time Fourier transform of real rows (DESIGN.md §4.13) on the
// CPU, thread by thread and phase by phase (StftBody in onchip_kernels.cuh; real::FrameMap, gather_frame_one,
// overlap_add_one and istft_runs in real_kernels.cuh are __host__ __device__ or host code), against direct sums in
// double:
//   * the fused forward kernel for every on-chip size class of both precisions, boundaries none / zeros / reflect,
//     hops 1, 37, N/4, N and N+3, rows of the smallest legal length, N, N+1 and three frames plus a remainder, against
//     a direct windowed DFT of the frame (every frame up to 12 per row, else the first and last 3 and every F/4-th);
//     one batch per class leaves a partial group;
//   * the gather of the other forward paths and the overlap-add of the inverse for N = 96 and 97, element by element,
//     the inverse over runs cut by scratches of several sizes, whose bits must not depend on the cut.
// Every input read and output write goes through FB_LIN_ACCESS and every spectrum write through FB_SPEC_ACCESS: the
// check fails on a read outside [0, L) of the frame's row, a bin or output written zero times or twice, and a spectrum
// access that is misaligned or wider than one complex value.  It also reports the bank-conflict degree of the load
// phases' shared accesses: the windowed reals written into the park and the stage-A reads of them.
// Build: nvcc -std=c++17 -O1 --expt-relaxed-constexpr -I fourier_b200/csrc tools/emulate_stft.cu \
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
// reads: g is the global frame, whose row g / frames must hold the sample; writes (overlap-add): g is the output row
struct StftCheck {
  bool on = false;
  uintptr_t x = 0, y = 0;
  long esz = 0, in_len = 0, out_len = 0, frames = 1;
  long bad_reads = 0, bad_writes = 0;
  std::vector<int> writes;
};
static StftCheck g_chk;

static void lin_record(int write, const void* p, long g) {
  if (!g_chk.on) return;
  const long row = write ? g : g / g_chk.frames;
  const intptr_t d = (intptr_t)p - (intptr_t)(write ? g_chk.y : g_chk.x);
  const long e = (long)(d / g_chk.esz);
  const long len = write ? g_chk.out_len : g_chk.in_len;
  if (d % g_chk.esz || d < 0 || e < row * len || e >= (row + 1) * len) {
    ++(write ? g_chk.bad_writes : g_chk.bad_reads);
    return;
  }
  if (write) ++g_chk.writes[e];
}

template <typename T>
static void check_begin(const T* x, const T* y, long in_len, long out_len, long frames, long rows) {
  g_chk.on = true;
  g_chk.x = (uintptr_t)x; g_chk.y = (uintptr_t)y;
  g_chk.esz = sizeof(T); g_chk.in_len = in_len; g_chk.out_len = out_len; g_chk.frames = frames;
  g_chk.bad_reads = g_chk.bad_writes = 0;
  g_chk.writes.assign(out_len * rows, 0);
}
static void check_end(long& reads, long& writes, long& missing, long& twice) {
  g_chk.on = false;
  reads = g_chk.bad_reads; writes = g_chk.bad_writes; missing = twice = 0;
  for (int c : g_chk.writes) { missing += c == 0; twice += c > 1; }
}

static const char* kBoundary[3] = {"none", "zeros", "reflect"};

// the padded row of the definition: sample t of [-pad, L + pad), 0 or mirrored outside [0, L)
static double padded(const std::vector<double>& x, long b, long len, long t, int boundary) {
  if (t >= 0 && t < len) return x[b * len + t];
  if (boundary != real::kStftReflect) return 0.0;
  return x[b * len + (t < 0 ? -t : 2 * (len - 1) - t)];
}

// the row lengths of one boundary and hop: the smallest legal, N, N+1, and N - 2 pad + 3H + H/2 (three frames plus a
// remainder), distinct
static std::vector<long> row_lengths(long n, long hop, int boundary) {
  const long pad = boundary == real::kStftNone ? 0 : n / 2;
  const long least = boundary == real::kStftNone ? n : boundary == real::kStftZeros ? 1 : n / 2 + 1;
  std::vector<long> ls;
  for (long l : {least, n, n + 1, std::max(least, n - 2 * pad + 3 * hop + hop / 2)})
    if (std::find(ls.begin(), ls.end(), l) == ls.end()) ls.push_back(l);
  return ls;
}

// outside: input reads (or overlap-add writes) outside their row; extra: bins or outputs not written exactly once,
// stray spectrum accesses, or gathered elements that differ from the definition
static int report(const char* what, double worst, double tol, long outside, long extra) {
  const bool ok = worst < tol && !outside && !extra;
  printf("%s: max rel err %.3e, outside row %ld, not once %ld %s\n", what, worst, outside, extra, ok ? "OK" : "FAIL");
  return !ok;
}

// ---- fused on-chip stft kernel -------------------------------------------------------------------------------------
template <class K>
static int check_fused(const char* name, double tol) {
  using T = typename K::T;
  constexpr int RA = K::RA, RB = K::RB;
  using V = cpx<T>;
  using Cfg = typename K::template Cfg<true>;
  using Body = onchip::StftBody<Cfg>;
  using Tile = typename Cfg::Tile;
  constexpr long L = RA * RB, N = 2 * L, bins = L + 1;
  int bad = 0, partial = 0;
  const auto twa = twopass::make_twa<T>(RA, RB);
  const auto tab = pair_table<T>(L);
  std::vector<double> wr, wi;
  twiddles(N, wr, wi);
  unsigned long long seed = 7177 + N;
  Buf<T> win(N);
  std::vector<double> wd(N);
  for (long p = 0; p < N; ++p) { win[p] = (T)(0.5 + 0.5 * rnd(seed)); wd[p] = win[p]; }
  auto run = [&](int boundary, long hop, long in_len, long batch) {
    const real::FrameMap m = real::frame_map(N, in_len, hop, boundary);
    const long nf = batch * m.frames;
    Buf<T> x(in_len * batch);
    Buf<V> y(nf * bins);
    std::vector<double> xd(in_len * batch);
    for (long i = 0; i < in_len * batch; ++i) { x[i] = (T)rnd(seed); xd[i] = x[i]; }
    for (long i = 0; i < nf * bins; ++i) y[i] = mk<T>((T)NAN, (T)NAN);
    typename Body::Args a;
    static_cast<typename onchip::RealBody<Cfg>::Args&>(a) = {nullptr, y.p, twa.data(), tab.data(), nf, (T)0.5};
    a.x = x.p; a.win = win.p; a.m = m;
    check_begin(x.p, (const T*)nullptr, in_len, 0, m.frames, 0);
    g_access.clear();
    run_body<Body, Tile, typename Cfg::Lay>(a, (nf + Cfg::C - 1) / Cfg::C, twa.data());
    long reads, writes, missing, twice;
    check_end(reads, writes, missing, twice);
    // every bin of every frame written exactly once, each access one aligned complex value
    std::vector<int> count(nf * bins, 0);
    long stray = 0;
    for (const Access& ac : g_access) {
      const intptr_t d = (intptr_t)ac.addr - (intptr_t)y.p;
      if (d < 0 || d % sizeof(V) || d / (intptr_t)sizeof(V) >= nf * bins) { ++stray; continue; }
      ++count[d / sizeof(V)];
    }
    for (int c : count) stray += c != 1;
    bad += check_access("stft spectrum", y.p, nf, bins * sizeof(V), (int)sizeof(V));
    // the direct windowed DFT of (a sample of) the frames
    const long stride = m.frames <= 12 ? 1 : m.frames / 4;
    double worst = 0;
    std::vector<double> u(N);
    for (long b = 0; b < batch; ++b)
      for (long f = 0; f < m.frames; ++f) {
        if (!(f < 3 || f >= m.frames - 3 || f % stride == 0)) continue;
        for (long p = 0; p < N; ++p) u[p] = padded(xd, b, in_len, f * hop - m.pad + p, boundary) * wd[p];
        double e = 0, r = 0;
        for (long k = 0; k < bins; ++k) {
          double re = 0, im = 0;
          for (long p = 0, j = 0; p < N; ++p, j = j + k >= N ? j + k - N : j + k) { re += u[p] * wr[j]; im += u[p] * wi[j]; }
          const V got = y[(b * m.frames + f) * bins + k];
          e = std::max(e, std::hypot(got.x - re, got.y - im));
          r = std::max(r, std::hypot(re, im));
        }
        worst = std::max(worst, std::isnan(e) ? INFINITY : e / std::max(r, 1e-300));
      }
    partial += nf % Cfg::C != 0;
    char what[160];
    snprintf(what, sizeof what, "fused %s N=%ld %s H=%ld L=%ld batch=%ld frames=%ld%s", name, N, kBoundary[boundary],
             hop, in_len, batch, m.frames, nf % Cfg::C ? " partial" : "");
    return report(what, worst, tol, reads, stray);
  };
  for (int boundary = 0; boundary < 3; ++boundary)
    for (long hop : {1L, 37L, N / 4, N, N + 3})
      for (long in_len : row_lengths(N, hop, boundary)) bad += run(boundary, hop, in_len, 2);
  if (!partial) bad += run(real::kStftReflect, N / 4, N + 1, 3);   // 3 rows of 5 frames
  // the load phase's writes of the frame's reals into the park (lane u of an FFT writes real u + TP*j) and the
  // stage-A reads of it as complex values
  int worst_w = 1, worst_r = 1;
  for (int warp = 0; warp < Cfg::THREADS / 32; ++warp) {
    for (int j = 0; j < 2 * L / Tile::TP; ++j) {
      std::vector<long> idx;
      for (int l = 0; l < 32; ++l) {
        const int t = warp * 32 + l;
        idx.push_back(2 * Body::Real::park(t) + Tile::template u_of<true>(t) + Tile::TP * j);
      }
      worst_w = std::max(worst_w, conflict_degree<(int)sizeof(T)>(idx));
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
  printf("  stft     threads %4d  load conflicts: park write x%d, stage-A read x%d\n", Cfg::THREADS, worst_w, worst_r);
  return bad;
}

// ---- gather and overlap-add of the other paths ---------------------------------------------------------------------
static int check_maps(long n) {
  int bad = 0;
  unsigned long long seed = 5151 + n;
  std::vector<double> win(n);
  for (auto& v : win) v = 0.5 + 0.5 * rnd(seed);
  const long batch = 3;
  for (int boundary = 0; boundary < 3; ++boundary)
    for (long hop : {1L, 37L, n / 4, n, n + 3})
      for (long in_len : row_lengths(n, hop, boundary)) {
        // gather: two chunks of frames, element by element against the definition
        const real::FrameMap m = real::frame_map(n, in_len, hop, boundary);
        const long nf = batch * m.frames;
        std::vector<double> x(in_len * batch), seg(nf * n, NAN);
        for (auto& v : x) v = rnd(seed);
        check_begin(x.data(), (const double*)nullptr, in_len, 0, m.frames, 0);
        for (long c0 : {0L, nf / 2}) {
          real::FrameMap mc = m;
          mc.g0 = c0;
          const long nq = c0 == 0 ? nf / 2 : nf - nf / 2;
          for (long q = 0; q < nq; ++q)
            for (long p = 0; p < n; ++p) real::gather_frame_one(mc, x.data(), win.data(), seg.data() + c0 * n, q, p);
        }
        long reads, writes, missing, twice, differ = 0;
        check_end(reads, writes, missing, twice);
        for (long g = 0; g < nf; ++g)
          for (long p = 0; p < n; ++p)
            differ += !(seg[g * n + p] ==
                        padded(x, g / m.frames, in_len, (g % m.frames) * hop - m.pad + p, boundary) * win[p]);
        char what[160];
        snprintf(what, sizeof what, "gather N=%ld %s H=%ld L=%ld batch=%ld frames=%ld", n, kBoundary[boundary], hop,
                 in_len, batch, m.frames);
        bad += report(what, differ ? 1.0 : 0.0, 0.5, reads, differ);
      }
  // overlap-add of random frames, center and not, out_len past the last frame, runs cut by several scratch sizes
  for (int center = 0; center < 2; ++center)
    for (long hop : {1L, 37L, n / 4, n, n + 3})
      for (long frames : {1L, 2L, 7L}) {
        real::FrameMap m = real::frame_map(n, n, hop, real::kStftNone);
        m.pad = center ? n / 2 : 0;
        m.frames = frames;
        m.rcp = 1.0 / (double)frames;
        const long out_len = std::max(1L, hop * (frames - 1) + n - 2 * m.pad + hop / 2 + 3);
        std::vector<double> v(batch * frames * n);
        for (auto& e : v) e = rnd(seed);
        // the direct sum of the definition
        std::vector<double> ref(batch * out_len);
        for (long b = 0; b < batch; ++b)
          for (long i = 0; i < out_len; ++i) {
            const long t = i + m.pad;
            double num = 0, den = 0;
            for (long f = 0; f < frames; ++f)
              if (t - f * hop >= 0 && t - f * hop < n) {
                num += win[t - f * hop] * v[(b * frames + f) * n + t - f * hop];
                den += win[t - f * hop] * win[t - f * hop];
              }
            ref[b * out_len + i] = den >= 1e-11 ? num / den : 0.0;
          }
        std::vector<double> first;
        const size_t back = real::istft_back((size_t)n, (size_t)hop);
        for (size_t target : {(size_t)1 << 30, (size_t)frames, back + 2, (size_t)1}) {
          const size_t cap = real::istft_scratch_frames(target, (size_t)n, (size_t)hop, (size_t)frames);
          std::vector<double> y(batch * out_len, NAN), seg;
          long runs = 0;
          check_begin((const double*)nullptr, y.data(), 0, out_len, frames, batch);
          real::istft_runs((size_t)n, (size_t)hop, (size_t)m.pad, (size_t)frames, (size_t)out_len, (size_t)batch, cap,
                           [&](size_t gs, size_t ge, size_t b0, size_t nb, size_t i0, size_t i1) {
                             ++runs;
                             seg.assign(v.begin() + gs * n, v.begin() + ge * n);   // what the run's irfft leaves
                             for (size_t r = 0; r < nb; ++r)
                               for (size_t i = i0; i < i1; ++i)
                                 real::overlap_add_one(m, seg.data(), win.data(), (long)gs, y.data() + (b0 + r) * out_len,
                                                       (long)(b0 + r), (long)i);
                             return 0;
                           });
          long reads, writes, missing, twice;
          check_end(reads, writes, missing, twice);
          double worst = 0, r = 0;
          for (long i = 0; i < batch * out_len; ++i) {
            worst = std::max(worst, std::isnan(y[i]) ? INFINITY : std::fabs(y[i] - ref[i]));
            r = std::max(r, std::fabs(ref[i]));
          }
          worst /= std::max(r, 1e-300);
          bool same = true;
          if (first.empty()) first = y;
          for (long i = 0; i < batch * out_len; ++i) same &= y[i] == first[i];
          char what[192];
          snprintf(what, sizeof what, "overlap-add N=%ld center=%d H=%ld frames=%ld out_len=%ld scratch=%zu runs=%ld %s",
                   n, center, hop, frames, out_len, cap, runs, same ? "same bits" : "DIFFERENT BITS");
          bad += report(what, worst, 1e-12, writes, missing + twice);
          bad += !same;
        }
      }
  return bad;
}

int main() {
  int bad = 0;
  // every on-chip size class (onchip_configs.cuh): L = N/2
  for_each_onchip<float>([&](auto k) { bad += check_fused<decltype(k)>("f32", 1e-5); });
  for_each_onchip<double>([&](auto k) { bad += check_fused<decltype(k)>("f64", 1e-12); });
  for (long n : {96L, 97L}) bad += check_maps(n);
  printf(bad ? "EMULATION FAILED (%d)\n" : "EMULATION OK\n", bad);
  return bad ? 1 : 0;
}
