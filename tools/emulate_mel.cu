// emulate_mel.cu -- runs the device code of the mel spectrogram of real rows (DESIGN.md §4.14) on the CPU, thread by
// thread and phase by phase (MelBody in onchip_kernels.cuh; real::band_scan, band_merge, mel_dot, power_pair and
// mel_spectrum_one in real_kernels.cuh are __host__ __device__), against direct sums in double:
//   * the fused kernel for every on-chip size class of both precisions, boundaries none / zeros / reflect, hops 1, N/4
//     and N+3, powers 1 and 2, and three filter banks: an HTK triangular bank of 80 mels, one dense random row, and
//     N/2+6 rows that are all zero, a single weight at bin 0, a single weight at bin N/2, negative weights over a
//     random band, or a single weight elsewhere.  The reference is a direct windowed DFT of the frame, |.|^p and the
//     bank (every frame of rows up to 12 frames, else the first and last 3 and every F/4-th);
//   * for N = 96 and 97 the per-output function of mel_spectra_kernel over two chunks of frames, and the band rule of
//     mel_bands_kernel (a scan every 256th weight per thread, merged) on the same banks.
// Every input read and output write goes through FB_LIN_ACCESS and every weight read through FB_MEL_ACCESS: the check
// fails on a read outside the frame's row, an output written zero times or twice, a weight read outside its mel's
// band or the matrix, and a zero filter row whose output is not exactly 0.  It also reports the bank-conflict degree
// of the shared accesses: StftBody's load phases, the power write into the park and, for the HTK bank, the mel phase's
// reads of the parked powers.
// Build: nvcc -std=c++17 -O1 --expt-relaxed-constexpr -I fourier_b200/csrc tools/emulate_mel.cu \
//             fourier_b200/csrc/host_math.cu (host only, never run on the device)
#include <cstdint>
#include <string>
#include <vector>

static void lin_record(int write, const void* p, long g);
static void mel_record(const void* p, long m);
#ifdef __CUDA_ARCH__
#define FB_LIN_ACCESS(w, p, g)
#define FB_MEL_ACCESS(p, m)
#else
#define FB_LIN_ACCESS(w, p, g) lin_record((w), (const void*)(p), (long)(g))
#define FB_MEL_ACCESS(p, m) mel_record((const void*)(p), (long)(m))
#endif

#include "emulate_common.h"

// ---- access log: checked as it happens ------------------------------------------------------------------------------
// reads: g is the global frame, whose row g / frames must hold the sample; writes: g is the frame, n_mels outputs each
struct MelCheck {
  bool on = false;
  uintptr_t x = 0, y = 0, w = 0;
  long esz = 0, in_len = 0, n_mels = 0, frames = 1, bins = 0, y_first = 0;
  long bad_reads = 0, bad_writes = 0, bad_weights = 0;
  std::vector<int> writes;
  std::vector<real::Band> band;   // the bands of the definition, computed directly
};
static MelCheck g_chk;

static void lin_record(int write, const void* p, long g) {
  if (!g_chk.on) return;
  const intptr_t d = (intptr_t)p - (intptr_t)(write ? g_chk.y : g_chk.x);
  const long e = (long)(d / g_chk.esz);
  if (write) {
    const long row = g - g_chk.y_first;
    if (d % g_chk.esz || d < 0 || e < row * g_chk.n_mels || e >= (row + 1) * g_chk.n_mels) { ++g_chk.bad_writes; return; }
    ++g_chk.writes[e];
  } else {
    const long row = g / g_chk.frames;
    if (d % g_chk.esz || d < 0 || e < row * g_chk.in_len || e >= (row + 1) * g_chk.in_len) ++g_chk.bad_reads;
  }
}
static void mel_record(const void* p, long m) {
  if (!g_chk.on) return;
  const intptr_t d = (intptr_t)p - (intptr_t)g_chk.w;
  const long e = (long)(d / g_chk.esz), k = e - m * g_chk.bins;
  if (d % g_chk.esz || d < 0 || m < 0 || m >= g_chk.n_mels || k < g_chk.band[m].lo || k >= g_chk.band[m].hi)
    ++g_chk.bad_weights;
}

static const char* kBoundary[3] = {"none", "zeros", "reflect"};

// ---- filter banks, (n_mels, bins) row-major in double ----------------------------------------------------------------
struct Bank {
  std::string name;
  long n_mels;
  std::vector<double> w;
};

// torchaudio.functional.melscale_fbanks(bins, 0, sr / 2, n_mels, sr, norm=None, mel_scale="htk"), transposed
static Bank htk_bank(long bins, long n_mels, double sr) {
  Bank b{"htk", n_mels, std::vector<double>(n_mels * bins, 0.0)};
  auto mel = [](double f) { return 2595.0 * std::log10(1.0 + f / 700.0); };
  auto hz = [](double m) { return 700.0 * (std::pow(10.0, m / 2595.0) - 1.0); };
  std::vector<double> f(n_mels + 2);
  for (long i = 0; i < n_mels + 2; ++i) f[i] = hz(mel(0.0) + (mel(sr / 2) - mel(0.0)) * (double)i / (double)(n_mels + 1));
  for (long k = 0; k < bins; ++k) {
    const double fk = (sr / 2) * (double)k / (double)(bins - 1);
    for (long m = 0; m < n_mels; ++m) {
      const double down = (fk - f[m]) / (f[m + 1] - f[m]), up = (f[m + 2] - fk) / (f[m + 2] - f[m + 1]);
      b.w[m * bins + k] = std::max(0.0, std::min(down, up));
    }
  }
  return b;
}
static Bank dense_bank(long bins, unsigned long long& seed) {
  Bank b{"dense", 1, std::vector<double>(bins)};
  for (auto& v : b.w) v = rnd(seed);
  return b;
}
// rows m = 5i: zero, 5i+1: one weight at bin 0, 5i+2: one at bin N/2, 5i+3: negative weights over a random band,
// 5i+4: one weight at bin m mod bins; bins + 5 rows
static Bank special_bank(long bins, unsigned long long& seed) {
  Bank b{"special", bins + 5, std::vector<double>((bins + 5) * bins, 0.0)};
  for (long m = 0; m < b.n_mels; ++m) {
    double* r = b.w.data() + m * bins;
    switch (m % 5) {
      case 1: r[0] = 1.0 + rnd(seed); break;
      case 2: r[bins - 1] = 1.0 + rnd(seed); break;
      case 3: {
        long lo = (long)((0.5 + 0.5 * rnd(seed)) * bins) % bins, hi = lo + 1 + (long)((0.5 + 0.5 * rnd(seed)) * 9);
        for (long k = lo; k < std::min(hi, bins); ++k) r[k] = -(0.25 + 0.5 * (0.5 + 0.5 * rnd(seed)));
        break;
      }
      case 4: r[m % bins] = 0.5; break;
      default: break;
    }
  }
  return b;
}

// the bands of the definition, directly: first non-zero to one past the last, {bins, 0} when there is none
template <typename T> static std::vector<real::Band> direct_bands(const std::vector<T>& w, long n_mels, long bins) {
  std::vector<real::Band> out(n_mels, real::Band{(int)bins, 0});
  for (long m = 0; m < n_mels; ++m)
    for (long k = 0; k < bins; ++k)
      if (w[m * bins + k] != (T)0) {
        if (out[m].lo == (int)bins) out[m].lo = (int)k;
        out[m].hi = (int)k + 1;
      }
  return out;
}
// the bands as mel_bands_kernel forms them: thread t of the CTA scans every 256th weight from t, merged
template <typename T> static std::vector<real::Band> kernel_bands(const T* w, long n_mels, long bins) {
  std::vector<real::Band> out(n_mels);
  for (long m = 0; m < n_mels; ++m) {
    real::Band b = real::band_scan(w + m * bins, bins, 0L, 256L);
    for (long t = 1; t < 256; ++t) b = real::band_merge(b, real::band_scan(w + m * bins, bins, t, 256L));
    out[m] = b;
  }
  return out;
}
static bool same_bands(const std::vector<real::Band>& a, const std::vector<real::Band>& b) {
  if (a.size() != b.size()) return false;
  for (size_t i = 0; i < a.size(); ++i)
    if (a[i].lo != b[i].lo || a[i].hi != b[i].hi) return false;
  return true;
}

// the padded row of the definition: sample t of [-pad, L + pad), 0 or mirrored outside [0, L)
static double padded(const std::vector<double>& x, long b, long len, long t, int boundary) {
  if (t >= 0 && t < len) return x[b * len + t];
  if (boundary != real::kStftReflect) return 0.0;
  return x[b * len + (t < 0 ? -t : 2 * (len - 1) - t)];
}

static int report(const char* what, double worst, double tol, long outside, long extra, long weights, long zero_rows) {
  const bool ok = worst < tol && !outside && !extra && !weights && !zero_rows;
  printf("%s: max rel err %.3e, outside row %ld, not once %ld, outside band %ld, zero rows not 0 %ld %s\n", what, worst,
         outside, extra, weights, zero_rows, ok ? "OK" : "FAIL");
  return !ok;
}

template <typename T> static void check_begin(const T* x, const T* y, const T* w, long in_len, long n_mels, long frames,
                                              long bins, long nf, const std::vector<real::Band>& band) {
  g_chk.on = true;
  g_chk.x = (uintptr_t)x; g_chk.y = (uintptr_t)y; g_chk.w = (uintptr_t)w;
  g_chk.esz = sizeof(T); g_chk.in_len = in_len; g_chk.n_mels = n_mels; g_chk.frames = frames; g_chk.bins = bins;
  g_chk.y_first = 0;
  g_chk.bad_reads = g_chk.bad_writes = g_chk.bad_weights = 0;
  g_chk.writes.assign(nf * n_mels, 0);
  g_chk.band = band;
}
static long check_end() {
  g_chk.on = false;
  long extra = g_chk.bad_writes;
  for (int c : g_chk.writes) extra += c != 1;
  return extra;
}

// ---- fused on-chip mel kernel --------------------------------------------------------------------------------------
template <class K>
static int check_fused(const char* name, double tol) {
  using T = typename K::T;
  constexpr int RA = K::RA, RB = K::RB;
  using V = cpx<T>;
  using Cfg = typename K::template Cfg<true>;
  using Body = onchip::MelBody<Cfg>;
  using Tile = typename Cfg::Tile;
  constexpr long L = RA * RB, N = 2 * L, bins = L + 1;
  int bad = 0, partial = 0;
  const auto twa = twopass::make_twa<T>(RA, RB);
  const auto tab = pair_table<T>(L);
  std::vector<double> wr, wi;
  twiddles(N, wr, wi);
  unsigned long long seed = 9391 + N;
  Buf<T> win(N);
  std::vector<double> wd(N);
  for (long p = 0; p < N; ++p) { win[p] = (T)(0.5 + 0.5 * rnd(seed)); wd[p] = win[p]; }
  std::vector<Bank> banks = {htk_bank(bins, 80, 16000.0), dense_bank(bins, seed), special_bank(bins, seed)};
  const long batch = 2;
  for (int boundary = 0; boundary < 3; ++boundary)
    for (long hop : {1L, N / 4, N + 3}) {
      const long pad = boundary == real::kStftNone ? 0 : N / 2;
      const long least = boundary == real::kStftNone ? N : boundary == real::kStftZeros ? 1 : N / 2 + 1;
      const long in_len = std::max(least, N - 2 * pad + 3 * hop + hop / 2);
      const real::FrameMap m = real::frame_map(N, in_len, hop, boundary);
      const long nf = batch * m.frames;
      Buf<T> x(in_len * batch);
      std::vector<double> xd(in_len * batch);
      for (long i = 0; i < in_len * batch; ++i) { x[i] = (T)rnd(seed); xd[i] = x[i]; }
      // the direct spectra of the sampled frames
      const long stride = m.frames <= 12 ? 1 : m.frames / 4;
      std::vector<long> sampled;
      for (long f = 0; f < m.frames; ++f)
        if (f < 3 || f >= m.frames - 3 || f % stride == 0) sampled.push_back(f);
      std::vector<double> pow2(batch * sampled.size() * bins);
      std::vector<double> u(N);
      for (long b = 0; b < batch; ++b)
        for (size_t s = 0; s < sampled.size(); ++s) {
          const long f = sampled[s];
          for (long p = 0; p < N; ++p) u[p] = padded(xd, b, in_len, f * hop - m.pad + p, boundary) * wd[p];
          for (long k = 0; k < bins; ++k) {
            double re = 0, im = 0;
            for (long p = 0, j = 0; p < N; ++p, j = j + k >= N ? j + k - N : j + k) { re += u[p] * wr[j]; im += u[p] * wi[j]; }
            pow2[(b * sampled.size() + s) * bins + k] = re * re + im * im;
          }
        }
      for (const Bank& bank : banks)
        for (int power : {1, 2}) {
          // hops 1 and N+3: the HTK bank at power 2 and the special bank at power 1 only
          if (hop != N / 4 && !((bank.name == "htk" && power == 2) || (bank.name == "special" && power == 1))) continue;
          const long nm = bank.n_mels;
          std::vector<T> wt(nm * bins);
          for (long i = 0; i < nm * bins; ++i) wt[i] = (T)bank.w[i];
          Buf<T> filt(nm * bins);
          for (long i = 0; i < nm * bins; ++i) filt[i] = wt[i];
          const std::vector<real::Band> band = direct_bands(wt, nm, bins);
          const std::vector<real::Band> kband = kernel_bands(filt.p, nm, bins);
          Buf<T> y(nf * nm);
          for (long i = 0; i < nf * nm; ++i) y[i] = (T)NAN;
          typename Body::Args a;
          static_cast<typename onchip::RealBody<Cfg>::Args&>(a) = {nullptr, nullptr, twa.data(), tab.data(), nf, (T)0.5};
          a.x = x.p; a.win = win.p; a.m = m;
          a.mel = y.p; a.filters = filt.p; a.bands = kband.data(); a.n_mels = nm; a.power = power;
          check_begin(x.p, y.p, filt.p, in_len, nm, m.frames, bins, nf, band);
          run_body<Body, Tile, typename Cfg::Lay>(a, (nf + Cfg::C - 1) / Cfg::C, twa.data());
          const long extra = check_end() + !same_bands(band, kband);
          // against bank . |X|^p in double, relative to the row's max
          double worst = 0;
          for (long b = 0; b < batch; ++b) {
            double e = 0, r = 0;
            for (size_t s = 0; s < sampled.size(); ++s) {
              const double* pw = pow2.data() + (b * sampled.size() + s) * bins;
              for (long mm = 0; mm < nm; ++mm) {
                double ref = 0;
                for (long k = 0; k < bins; ++k) ref += (double)wt[mm * bins + k] * (power == 2 ? pw[k] : std::sqrt(pw[k]));
                const double got = y[(b * m.frames + sampled[s]) * nm + mm];
                e = std::max(e, std::isnan(got) ? INFINITY : std::fabs(got - ref));
                r = std::max(r, std::fabs(ref));
              }
            }
            worst = std::max(worst, e / std::max(r, 1e-300));
          }
          long zero_rows = 0;
          for (long mm = 0; mm < nm; ++mm)
            if (band[mm].lo >= band[mm].hi)
              for (long g = 0; g < nf; ++g) zero_rows += !(y[g * nm + mm] == (T)0);
          partial += nf % Cfg::C != 0;
          char what[224];
          snprintf(what, sizeof what, "fused %s N=%ld %s H=%ld L=%ld batch=%ld frames=%ld bank=%s mels=%ld p=%d%s", name,
                   N, kBoundary[boundary], hop, in_len, batch, m.frames, bank.name.c_str(), nm, power,
                   nf % Cfg::C ? " partial" : "");
          bad += report(what, worst, tol, g_chk.bad_reads, extra, g_chk.bad_weights, zero_rows);
        }
    }
  if (!partial) { printf("fused %s N=%ld: no batch left a partial group FAIL\n", name, N); ++bad; }
  // shared-memory bank conflicts per warp: StftBody's load phases (the frame's reals into the park, the stage-A reads),
  // the power write into the park (lane u writes u + TP*j and L - u - TP*j, lane 0 also L/2), and the mel phase's reads
  // of the parked powers for the HTK bank (lane u reads power lo_m + s of mel m = u + TP*i at step s of its sum)
  int worst_w = 1, worst_r = 1, worst_p = 1, worst_m = 1;
  const std::vector<real::Band> hb = direct_bands(std::vector<T>(banks[0].w.begin(), banks[0].w.end()), 80, bins);
  for (int warp = 0; warp < Cfg::THREADS / 32; ++warp) {
    auto lane_t = [&](int l) { return warp * 32 + l; };
    auto u_of = [&](int l) { return Tile::template u_of<true>(lane_t(l)); };
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
        up.push_back(park2(l) + u_of(l) + Tile::TP * j);
        down.push_back(park2(l) + L - (u_of(l) + Tile::TP * j));
      }
      worst_p = std::max({worst_p, conflict_degree<(int)sizeof(T)>(up), conflict_degree<(int)sizeof(T)>(down)});
    }
    std::vector<long> mid;
    for (int l = 0; l < 32; ++l) mid.push_back(u_of(l) == 0 ? park2(l) + L / 2 : -1);
    worst_p = std::max(worst_p, conflict_degree<(int)sizeof(T)>(mid));
    for (int i = 0; i * Tile::TP < 80; ++i)
      for (int s = 0; s < (int)bins; ++s) {
        std::vector<long> idx;
        bool any = false;
        for (int l = 0; l < 32; ++l) {
          const long mm = u_of(l) + Tile::TP * i;
          const bool on = mm < 80 && hb[mm].lo + s < hb[mm].hi;
          idx.push_back(on ? park2(l) + hb[mm].lo + s : -1);
          any |= on;
        }
        if (any) worst_m = std::max(worst_m, conflict_degree<(int)sizeof(T)>(idx));
      }
  }
  printf("  mel      threads %4d  load conflicts: park write x%d, stage-A read x%d; power write x%d; mel read x%d "
         "(HTK, 80 mels)\n", Cfg::THREADS, worst_w, worst_r, worst_p, worst_m);
  return bad;
}

// ---- the spectrum path's per-output function and the band rule, N = 96 and 97 ----------------------------------------
static int check_spectra(long n) {
  int bad = 0;
  using V = cpx<double>;
  const long bins = n / 2 + 1, nf = 7;
  unsigned long long seed = 6263 + n;
  std::vector<Bank> banks = {htk_bank(bins, 80, 16000.0), dense_bank(bins, seed), special_bank(bins, seed)};
  Buf<V> spec(nf * bins);
  for (long i = 0; i < nf * bins; ++i) spec[i] = mk<double>(rnd(seed), rnd(seed));
  for (const Bank& bank : banks) {
    const long nm = bank.n_mels;
    Buf<double> filt(nm * bins);
    for (long i = 0; i < nm * bins; ++i) filt[i] = bank.w[i];
    const std::vector<real::Band> band = direct_bands(bank.w, nm, bins), kband = kernel_bands(filt.p, nm, bins);
    const bool same = same_bands(band, kband);
    printf("bands N=%ld bank=%s mels=%ld: %s\n", n, bank.name.c_str(), nm, same ? "OK" : "FAIL");
    bad += !same;
    for (int power : {1, 2}) {
      std::vector<double> y(nf * nm, NAN);
      check_begin((const double*)nullptr, y.data(), filt.p, 0, nm, 1, bins, nf, band);
      g_access.clear();
      // two chunks of frames: [0, 3) and [3, nf), each with its spectra and output rows from its first frame on
      for (long c0 : {0L, 3L}) {
        const long nq = c0 == 0 ? 3 : nf - 3;
        for (long q = 0; q < nq; ++q)
          for (long mm = 0; mm < nm; ++mm)
            real::mel_spectrum_one(spec.p + c0 * bins, filt.p, kband.data(), bins, nm, power, y.data() + c0 * nm, q, mm,
                                   c0 + q);
      }
      const long extra = check_end();
      bad += check_access("mel spectra", spec.p, nf, bins * sizeof(V), (int)sizeof(V));
      double e = 0, r = 0;
      long zero_rows = 0;
      for (long g = 0; g < nf; ++g)
        for (long mm = 0; mm < nm; ++mm) {
          double ref = 0;
          for (long k = 0; k < bins; ++k) {
            const V v = spec[g * bins + k];
            const double p2 = v.x * v.x + v.y * v.y;
            ref += bank.w[mm * bins + k] * (power == 2 ? p2 : std::sqrt(p2));
          }
          const double got = y[g * nm + mm];
          e = std::max(e, std::isnan(got) ? INFINITY : std::fabs(got - ref));
          r = std::max(r, std::fabs(ref));
          if (band[mm].lo >= band[mm].hi) zero_rows += got != 0.0;
        }
      char what[160];
      snprintf(what, sizeof what, "spectra N=%ld bank=%s mels=%ld p=%d chunks=2", n, bank.name.c_str(), nm, power);
      bad += report(what, e / std::max(r, 1e-300), 1e-12, 0, extra, g_chk.bad_weights, zero_rows);
    }
  }
  return bad;
}

int main() {
  int bad = 0;
  // every on-chip size class (onchip_configs.cuh): L = N/2
  for_each_onchip<float>([&](auto k) { bad += check_fused<decltype(k)>("f32", 1e-5); });
  for_each_onchip<double>([&](auto k) { bad += check_fused<decltype(k)>("f64", 1e-12); });
  for (long n : {96L, 97L}) bad += check_spectra(n);
  printf(bad ? "EMULATION FAILED (%d)\n" : "EMULATION OK\n", bad);
  return bad ? 1 : 0;
}
