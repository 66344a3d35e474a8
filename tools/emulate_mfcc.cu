// emulate_mfcc.cu -- runs the device code of the MFCC and log-mel spectrogram of real rows (DESIGN.md §4.18) on the
// CPU, thread by thread and phase by phase (MfccBody in onchip_kernels.cuh, both instantiations; real::log_mel, max_key,
// max_fold, clamp_threshold, clamp_db and mfcc_dot in real_kernels.cuh are __host__ __device__), against direct sums in
// double:
//   * the fused kernel for every on-chip size class of both precisions, boundaries none / zeros / reflect, hops 1, N/4
//     and N+3, powers 1 and 2, three banks (an HTK bank of 40 mels, an HTK bank of exactly L-1 mels, and the 40-mel bank
//     with an all-zero row), projections dct NULL, n_out 13 and n_out 2 TP + 3, bias 0 and 1.5, the clamp off and
//     binding (the rows' last third is 60 dB quieter, top_db 30), clamp groups of 1 and 2 rows.  The reference is a
//     direct windowed DFT of the frame, |.|^p, the bank, the log, the clamp at the group's threshold and the projection
//     (every frame of rows up to 12 frames, else the first and last 3 and every F/4-th);
//   * every run with the clamp also runs the max sweep (MAX) first, and an identity run (dct NULL, bias 0, no clamp)
//     gives the log-mels themselves: each group slot must equal the maximum of its rows' log-mels exactly (and, where
//     every frame is sampled, the direct maximum to the tolerance), and an all-zero filter row must give exactly
//     log_scale ln(max(log_offset, log_floor));
//   * for N = 96 and 97 the element steps of mfcc_frames_kernel (both forms) over two chunks of frames, the first chunk
//     ending inside a row, on mels from mel_spectrum_one.
// Every input read and output write goes through FB_LIN_ACCESS, every weight read through FB_MEL_ACCESS and every matrix
// read through FB_DCT_ACCESS: the check fails on a read outside the frame's row, an output written zero times or twice, a
// weight read outside its mel's band, and a matrix read outside [0, n_mels n_out).  It also reports the bank-conflict
// degree of the new phases' shared accesses: the log-mel write into the park and the projection's log-mel read.
// Build: nvcc -std=c++17 -O1 --expt-relaxed-constexpr -I fourier_b200/csrc tools/emulate_mfcc.cu \
//             fourier_b200/csrc/host_math.cu (host only, never run on the device)
#include <cstdint>
#include <string>
#include <vector>

static void lin_record(int write, const void* p, long g);
static void mel_record(const void* p, long m);
static void dct_record(const void* p);
#ifdef __CUDA_ARCH__
#define FB_LIN_ACCESS(w, p, g)
#define FB_MEL_ACCESS(p, m)
#define FB_DCT_ACCESS(p)
#else
#define FB_LIN_ACCESS(w, p, g) lin_record((w), (const void*)(p), (long)(g))
#define FB_MEL_ACCESS(p, m) mel_record((const void*)(p), (long)(m))
#define FB_DCT_ACCESS(p) dct_record((const void*)(p))
#endif

#include "emulate_common.h"

// ---- access log: checked as it happens ------------------------------------------------------------------------------
// reads: g is the global frame, whose row g / frames must hold the sample; writes: g is the frame, n_out outputs each
struct MfccCheck {
  bool on = false;
  uintptr_t x = 0, y = 0, w = 0, d = 0;
  long esz = 0, in_len = 0, n_out = 0, n_mels = 0, frames = 1, bins = 0;
  long bad_reads = 0, bad_writes = 0, bad_weights = 0, bad_dct = 0;
  std::vector<int> writes;
  std::vector<real::Band> band;
};
static MfccCheck g_chk;

static void lin_record(int write, const void* p, long g) {
  if (!g_chk.on) return;
  const intptr_t d = (intptr_t)p - (intptr_t)(write ? g_chk.y : g_chk.x);
  const long e = (long)(d / g_chk.esz);
  if (write) {
    if (d % g_chk.esz || d < 0 || e < g * g_chk.n_out || e >= (g + 1) * g_chk.n_out) { ++g_chk.bad_writes; return; }
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
static void dct_record(const void* p) {
  if (!g_chk.on) return;
  const intptr_t d = (intptr_t)p - (intptr_t)g_chk.d;
  if (d % g_chk.esz || d < 0 || d / g_chk.esz >= g_chk.n_mels * g_chk.n_out) ++g_chk.bad_dct;
}

static const char* kBoundary[3] = {"none", "zeros", "reflect"};

// torchaudio.functional.melscale_fbanks(bins, 0, sr / 2, n_mels, sr, norm=None, mel_scale="htk"), transposed
static std::vector<double> htk_bank(long bins, long n_mels, double sr) {
  std::vector<double> w(n_mels * bins, 0.0);
  auto mel = [](double f) { return 2595.0 * std::log10(1.0 + f / 700.0); };
  auto hz = [](double m) { return 700.0 * (std::pow(10.0, m / 2595.0) - 1.0); };
  std::vector<double> f(n_mels + 2);
  for (long i = 0; i < n_mels + 2; ++i) f[i] = hz(mel(sr / 2) * (double)i / (double)(n_mels + 1));
  for (long k = 0; k < bins; ++k) {
    const double fk = (sr / 2) * (double)k / (double)(bins - 1);
    for (long m = 0; m < n_mels; ++m) {
      const double down = (fk - f[m]) / (f[m + 1] - f[m]), up = (f[m + 2] - fk) / (f[m + 2] - f[m + 1]);
      w[m * bins + k] = std::max(0.0, std::min(down, up));
    }
  }
  return w;
}
template <typename T> static std::vector<real::Band> direct_bands(const T* w, long n_mels, long bins) {
  std::vector<real::Band> out(n_mels, real::Band{(int)bins, 0});
  for (long m = 0; m < n_mels; ++m)
    for (long k = 0; k < bins; ++k)
      if (w[m * bins + k] != (T)0) {
        if (out[m].lo == (int)bins) out[m].lo = (int)k;
        out[m].hi = (int)k + 1;
      }
  return out;
}
static double padded(const std::vector<double>& x, long b, long len, long t, int boundary) {
  if (t >= 0 && t < len) return x[b * len + t];
  if (boundary != real::kStftReflect) return 0.0;
  return x[b * len + (t < 0 ? -t : 2 * (len - 1) - t)];
}

// the parameters of one run; the projection matrix is random in [-1, 1)
struct Run { long n_out; bool dct; double bias; bool clamp; long rows; };

template <typename T> static real::MfccArgs<T> mfcc_args(const Run& r, const T* dct, real::MaxKey<T>* slots) {
  real::MfccArgs<T> p;
  p.offset = (T)0;
  p.floor = (T)1e-10;
  p.scale = (T)(10.0 / std::log(10.0));
  p.top_db = (T)30.0;
  p.bias = (T)r.bias;
  p.dct = r.dct ? dct : nullptr;
  p.n_out = r.n_out;
  p.rows = r.clamp ? r.rows : 0;
  p.row0 = 0;
  p.rows_rcp = r.clamp ? 1.0 / (double)r.rows : 0.0;
  p.slots = slots;
  return p;
}

// ---- fused on-chip MFCC kernel -------------------------------------------------------------------------------------
template <class K>
static int check_fused(const char* name, double tol, double& worst_all) {
  using T = typename K::T;
  constexpr int RA = K::RA, RB = K::RB;
  using Cfg = typename K::template Cfg<true>;
  using Out = onchip::MfccBody<Cfg, false>;
  using Max = onchip::MfccBody<Cfg, true>;
  using Tile = typename Cfg::Tile;
  constexpr long L = RA * RB, N = 2 * L, bins = L + 1, TP = Tile::TP;
  int bad = 0, partial = 0;
  const auto twa = twopass::make_twa<T>(RA, RB);
  const auto tab = pair_table<T>(L);
  std::vector<double> wr, wi;
  twiddles(N, wr, wi);
  unsigned long long seed = 7717 + N;
  Buf<T> win(N);
  std::vector<double> wd(N);
  for (long p = 0; p < N; ++p) { win[p] = (T)(0.5 + 0.5 * rnd(seed)); wd[p] = win[p]; }
  struct BankDef { const char* name; long n_mels; std::vector<double> w; };
  std::vector<BankDef> banks = {{"htk", 40, htk_bank(bins, 40, 16000.0)}, {"full", L - 1, htk_bank(bins, L - 1, 16000.0)},
                                {"zero-row", 40, htk_bank(bins, 40, 16000.0)}};
  for (long k = 0; k < bins; ++k) banks[2].w[7 * bins + k] = 0.0;
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
      for (long i = 0; i < in_len * batch; ++i) {
        const double quiet = (i % in_len) >= 2 * in_len / 3 ? 1e-3 : 1.0;   // 60 dB quieter for the last third
        x[i] = (T)(quiet * rnd(seed));
        xd[i] = x[i];
      }
      const long stride = m.frames <= 12 ? 1 : m.frames / 4;
      std::vector<long> sampled;
      for (long f = 0; f < m.frames; ++f)
        if (f < 3 || f >= m.frames - 3 || f % stride == 0) sampled.push_back(f);
      const bool all_sampled = (long)sampled.size() == m.frames;
      std::vector<double> pow2(batch * sampled.size() * bins), u(N);
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
      int i = 0;
      for (const BankDef& bank : banks)
        for (int power : {1, 2}) {
          // hops 1 and N+3: two runs only; hop N/4: every projection with the clamp off and binding
          const int idx = i++;
          if (hop != N / 4 && idx > 1) continue;
          const long nm = bank.n_mels;
          const long outs[3] = {nm, 13, 2 * TP + 3};
          const Run run = {outs[idx % 3], idx % 3 != 0, idx % 2 ? 1.5 : 0.0, hop != N / 4 ? idx == 0 : (idx / 3) % 2 == 1,
                           1 + idx % 2};
          Buf<T> filt(nm * bins);
          for (long k = 0; k < nm * bins; ++k) filt[k] = (T)bank.w[k];
          const std::vector<real::Band> band = direct_bands(filt.p, nm, bins);
          Buf<T> dct(nm * run.n_out);
          for (long k = 0; k < nm * run.n_out; ++k) dct[k] = (T)rnd(seed);
          std::vector<real::MaxKey<T>> slots(batch / run.rows, 0);
          auto launch = [&](auto body, const real::MfccArgs<T>& p, T* y) {
            using Body = decltype(body);
            onchip::MfccArgs<Cfg> a;
            static_cast<typename onchip::RealBody<Cfg>::Args&>(a) = {nullptr, nullptr, twa.data(), tab.data(), nf, (T)0.5};
            a.x = x.p; a.win = win.p; a.m = m;
            a.mel = y; a.filters = filt.p; a.bands = band.data(); a.n_mels = nm; a.power = power; a.p = p;
            run_body<Body, Tile, typename Cfg::Lay>(a, (nf + Cfg::C - 1) / Cfg::C, twa.data());
          };
          auto begin = [&](const T* y, long n_out) {
            g_chk.on = true;
            g_chk.x = (uintptr_t)x.p; g_chk.y = (uintptr_t)y; g_chk.w = (uintptr_t)filt.p; g_chk.d = (uintptr_t)dct.p;
            g_chk.esz = sizeof(T); g_chk.in_len = in_len; g_chk.n_out = n_out; g_chk.n_mels = nm;
            g_chk.frames = m.frames; g_chk.bins = bins; g_chk.band = band;
            g_chk.writes.assign(nf * n_out, 0);
          };
          g_chk.bad_reads = g_chk.bad_writes = g_chk.bad_weights = g_chk.bad_dct = 0;
          // the log-mels themselves (identity, no clamp), and the max sweep's slots against their group maxima
          Buf<T> lm(nf * nm);
          for (long k = 0; k < nf * nm; ++k) lm[k] = (T)NAN;
          Run ident = {nm, false, 0.0, false, 1};
          begin(lm.p, nm);
          launch(Out{}, mfcc_args<T>(ident, dct.p, nullptr), lm.p);
          long extra = 0;
          for (int c : g_chk.writes) extra += c != 1;
          long slot_bad = 0;
          const T floor_out = real::log_mel((T)0, mfcc_args<T>(ident, dct.p, nullptr));
          long zero_rows = 0;
          for (long mm = 0; mm < nm; ++mm)
            if (band[mm].lo >= band[mm].hi)
              for (long g = 0; g < nf; ++g) zero_rows += !(lm[g * nm + mm] == floor_out);
          if (run.clamp) {
            begin(nullptr, run.n_out);
            g_chk.on = true;
            launch(Max{}, mfcc_args<T>(run, dct.p, slots.data()), nullptr);
            for (size_t g = 0; g < slots.size(); ++g) {
              T hi = -(T)INFINITY;
              for (long k = (long)g * run.rows * m.frames * nm; k < ((long)g + 1) * run.rows * m.frames * nm; ++k)
                hi = std::max(hi, lm[k]);
              slot_bad += real::key_value<T>(slots[g]) != hi;
            }
          }
          // the output sweep
          Buf<T> y(nf * run.n_out);
          for (long k = 0; k < nf * run.n_out; ++k) y[k] = (T)NAN;
          begin(y.p, run.n_out);
          launch(Out{}, mfcc_args<T>(run, dct.p, slots.data()), y.p);
          g_chk.on = false;
          for (int c : g_chk.writes) extra += c != 1;
          extra += g_chk.bad_writes;
          // against the direct sums in double, relative to the row's max |out|; the threshold from the slot
          double worst = 0;
          for (long b = 0; b < batch; ++b) {
            const double theta = run.clamp ? (double)real::key_value<T>(slots[b / run.rows]) - 30.0 : -INFINITY;
            double e = 0, r = 0, direct_max = -INFINITY;
            for (size_t s = 0; s < sampled.size(); ++s) {
              const double* pw = pow2.data() + (b * sampled.size() + s) * bins;
              std::vector<double> lc(nm);
              for (long mm = 0; mm < nm; ++mm) {
                double mel = 0;
                for (long k = 0; k < bins; ++k) mel += (double)filt[mm * bins + k] * (power == 2 ? pw[k] : std::sqrt(pw[k]));
                const double l = 10.0 / std::log(10.0) * std::log(std::max(mel, 1e-10));
                direct_max = std::max(direct_max, l);
                lc[mm] = std::max(l, theta);
              }
              for (long j = 0; j < run.n_out; ++j) {
                double ref = run.bias;
                if (run.dct) for (long mm = 0; mm < nm; ++mm) ref += lc[mm] * (double)dct[mm * run.n_out + j];
                else ref += lc[j];
                const double got = y[(b * m.frames + sampled[s]) * run.n_out + j];
                e = std::max(e, std::isnan(got) ? INFINITY : std::fabs(got - ref));
                r = std::max(r, std::fabs(ref));
              }
            }
            worst = std::max(worst, e / std::max(r, 1e-300));
            if (run.clamp && all_sampled && run.rows == 1)
              slot_bad += std::fabs((double)real::key_value<T>(slots[b]) - direct_max) > tol * std::fabs(direct_max);
          }
          worst_all = std::max(worst_all, worst);
          partial += nf % Cfg::C != 0;
          const bool ok = worst < tol && !g_chk.bad_reads && !extra && !g_chk.bad_weights && !g_chk.bad_dct &&
                          !slot_bad && !zero_rows;
          printf("fused %s N=%ld %s H=%ld L=%ld batch=%ld frames=%ld bank=%s mels=%ld p=%d out=%ld%s bias=%g clamp=%s "
                 "rows=%ld%s: max rel err %.3e, outside row %ld, not once %ld, outside band %ld, dct outside %ld, "
                 "slots off %ld, zero rows off %ld %s\n",
                 name, N, kBoundary[boundary], hop, in_len, batch, m.frames, bank.name, nm, power, run.n_out,
                 run.dct ? "" : " (identity)", run.bias, run.clamp ? "on" : "off", run.rows,
                 nf % Cfg::C ? " partial" : "", worst, g_chk.bad_reads, extra, g_chk.bad_weights, g_chk.bad_dct,
                 slot_bad, zero_rows, ok ? "OK" : "FAIL");
          bad += !ok;
        }
    }
  if (!partial) { printf("fused %s N=%ld: no batch left a partial group FAIL\n", name, N); ++bad; }
  // shared-memory bank conflicts per warp of the new phases: the log-mel write (lane u writes park real L+1+u+TP*i) and
  // the projection's log-mel read (the TP lanes of an FFT all read park real L+1+m)
  int worst_w = 1, worst_r = 1;
  for (int warp = 0; warp < Cfg::THREADS / 32; ++warp) {
    std::vector<long> wi_, ri;
    for (int l = 0; l < 32; ++l) {
      const int t = warp * 32 + l;
      const long base = 2L * Out::Real::park(t) + L + 1;
      wi_.push_back(base + Tile::template u_of<true>(t));
      ri.push_back(base);
    }
    worst_w = std::max(worst_w, conflict_degree<(int)sizeof(T)>(wi_));
    worst_r = std::max(worst_r, conflict_degree<(int)sizeof(T)>(ri));
  }
  printf("  mfcc     threads %4d  conflicts: log-mel write x%d; projection read x%d\n", Cfg::THREADS, worst_w, worst_r);
  return bad;
}

// ---- the element steps of mfcc_frames_kernel, N = 96 and 97: two chunks of frames --------------------------------------
static int check_chunks(long n) {
  using V = cpx<double>;
  const long bins = n / 2 + 1, nm = 40, frames = 4, rows = 2, nf = rows * frames, n_out = 13, threads = 256;
  unsigned long long seed = 5501 + n;
  const std::vector<double> w = htk_bank(bins, nm, 16000.0);
  const std::vector<real::Band> band = direct_bands(w.data(), nm, bins);
  Buf<V> spec(nf * bins);
  for (long i = 0; i < nf * bins; ++i) spec[i] = mk<double>(rnd(seed), rnd(seed));
  for (long i = 3 * bins; i < nf * bins; ++i) spec[i] = mk<double>(spec[i].x * 1e-4, spec[i].y * 1e-4);
  Buf<double> dct(nm * n_out);
  for (long i = 0; i < nm * n_out; ++i) dct[i] = rnd(seed);
  Run run = {n_out, true, 0.5, true, rows};
  std::vector<real::MaxKey<double>> slots(1, 0);
  real::MfccArgs<double> p = mfcc_args<double>(run, dct.p, slots.data());
  p.top_db = 20.0;
  std::vector<double> mel(nf * nm), y(nf * n_out, NAN);
  g_chk.on = false;
  for (int max_sweep = 1; max_sweep >= 0; --max_sweep)
    for (long c0 : {0L, 3L}) {   // chunks [0, 3) and [3, nf): the first ends inside row 0
      const long nq = c0 == 0 ? 3 : nf - 3;
      for (long q = 0; q < nq; ++q)
        for (long mm = 0; mm < nm; ++mm)
          real::mel_spectrum_one(spec.p + c0 * bins, w.data(), band.data(), bins, nm, 2, mel.data() + c0 * nm, q, mm,
                                 c0 + q);
      for (long q = 0; q < nq; ++q) {
        double* x = mel.data() + (c0 + q) * nm;
        const long b = (c0 + q) / frames;
        if (max_sweep) {
          for (long t = 0; t < threads; ++t) {
            real::MaxKey<double> hi = 0;
            for (long mm = t; mm < nm; mm += threads) hi = std::max(hi, real::max_key(real::log_mel(x[mm], p)));
            if (t < nm) real::max_fold(p.slots + real::clamp_group(p, b), hi);
          }
        } else {
          const double theta = real::clamp_threshold(p, b);
          for (long mm = 0; mm < nm; ++mm) x[mm] = real::clamp_db(real::log_mel(x[mm], p), theta);
          for (long j = 0; j < n_out; ++j) y[(c0 + q) * n_out + j] = real::mfcc_dot(p, nm, j, [&](long k) { return x[k]; });
        }
      }
    }
  // reference in double from the same spectra
  double hi = -INFINITY, e = 0, r = 0;
  std::vector<double> lm(nf * nm);
  for (long g = 0; g < nf; ++g)
    for (long mm = 0; mm < nm; ++mm) {
      double s = 0;
      for (long k = 0; k < bins; ++k) s += w[mm * bins + k] * (spec[g * bins + k].x * spec[g * bins + k].x +
                                                               spec[g * bins + k].y * spec[g * bins + k].y);
      lm[g * nm + mm] = 10.0 / std::log(10.0) * std::log(std::max(s, 1e-10));
      hi = std::max(hi, lm[g * nm + mm]);
    }
  long clamped = 0;
  for (long g = 0; g < nf; ++g)
    for (long j = 0; j < n_out; ++j) {
      double ref = 0.5;
      for (long mm = 0; mm < nm; ++mm) {
        clamped += j == 0 && lm[g * nm + mm] < hi - 20.0;
        ref += std::max(lm[g * nm + mm], hi - 20.0) * dct[mm * n_out + j];
      }
      e = std::max(e, std::isnan(y[g * n_out + j]) ? INFINITY : std::fabs(y[g * n_out + j] - ref));
      r = std::max(r, std::fabs(ref));
    }
  const double slot_err = std::fabs(real::key_value<double>(slots[0]) - hi) / std::fabs(hi);
  const bool ok = e / r < 1e-12 && slot_err < 1e-12 && clamped > 0;
  printf("chunks N=%ld frames=%ld rows=%ld chunks=2: max rel err %.3e, slot rel err %.3e, clamped %ld %s\n", n, nf,
         rows, e / r, slot_err, clamped, ok ? "OK" : "FAIL");
  return !ok;
}

int main() {
  int bad = 0;
  double worst32 = 0, worst64 = 0;
  // every on-chip size class (onchip_configs.cuh): L = N/2
  for_each_onchip<float>([&](auto k) { bad += check_fused<decltype(k)>("f32", 1e-5, worst32); });
  for_each_onchip<double>([&](auto k) { bad += check_fused<decltype(k)>("f64", 1e-12, worst64); });
  printf("worst rel err: f32 %.3e, f64 %.3e\n", worst32, worst64);
  for (long n : {96L, 97L}) bad += check_chunks(n);
  printf(bad ? "EMULATION FAILED (%d)\n" : "EMULATION OK\n", bad);
  return bad ? 1 : 0;
}
