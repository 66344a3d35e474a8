// emulate_common.h -- the harness the CPU emulators (tools/emulate*.cu) share: they run the kernels' __host__ __device__
// bodies thread by thread and phase by phase on the CPU and check them against references in double.
//   * run_body: the CPU driver of tilefft.cuh's phase protocol, so an emulator runs exactly the phases of the kernel;
//   * for_each_onchip: the on-chip size classes the library selects from;
//   * the input generator, 16-byte-aligned buffers and the bank-conflict model of shared-memory accesses;
//   * the spectrum access hook (FB_SPEC_ACCESS, defined before the kernel headers) and check_access;
//   * the w_N^k pair table and the direct transforms of packed reals of the real-input emulators.
// Include it before any kernel header.
#pragma once

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

#include "onchip_configs.cuh"
#include "plan.h"
#include "tables.cuh"

using namespace fb200;

// ---- CPU driver of the phase protocol (tilefft.cuh) ---------------------------------------------------------------
// Groups (CTA tiles) 0 .. groups-1 of Body one after the other; each phase runs for every thread before the next one
// starts, which is the barrier.  twa: the stage twiddles an on-chip kernel copies to shared memory (ignored by the
// bodies that read theirs from Args).
template <class Body, class Tile, class LAY>
static void run_body(const typename Body::Args& a, long groups, const TwPair<typename Body::T>* twa = nullptr) {
  std::vector<typename Tile::V> smem(Tile::template smem_elems<LAY>());
  std::vector<Tile> thr(Tile::THREADS);
  for (long g = 0; g < groups; ++g)
    static_for<0, Body::kPhases>([&](auto P) {
      for (int t = 0; t < Tile::THREADS; ++t) Body::template phase<decltype(P)::value>(thr[t], a, g, t, smem.data(), twa);
    });
}

// The CPU driver of run_welch_groups (onchip_kernels.cuh): per group of a.w its rounds, each phase for every thread
// before the next, then the flush for every thread, which is the CTA barrier on both sides.  acc: the accumulators
// and lane sums the device keeps behind the exchange buffer and the stage twiddles.
template <class Body, class Tile, class LAY>
static void run_welch_body(const typename Body::Args& a, const TwPair<typename Body::T>* twa) {
  using T = typename Body::T;
  std::vector<typename Tile::V> smem(Tile::template smem_elems<LAY>());
  std::vector<T> acc(Body::ACC_BYTES / sizeof(T));
  std::vector<Tile> thr(Tile::THREADS);
  for (long g = 0; g < a.w.groups; ++g) {
    for (long r = 0; r < a.w.rounds(g); ++r)
      static_for<0, Body::kPhases>([&](auto P) {
        for (int t = 0; t < Tile::THREADS; ++t)
          Body::template phase<decltype(P)::value>(thr[t], a, g, r, t, smem.data(), acc.data(), twa);
      });
    for (int t = 0; t < Tile::THREADS; ++t) Body::flush(a, g, t, acc.data());
  }
}

// The CPU driver of run_welch_groups that also mirrors its barriers between warps (CsdBody): per group, each warp in
// ascending order runs its own (round, phase) steps, lane by lane per phase (the __syncwarp), until it has run a phase
// that Body::pair_barrier marks (the barrier over a frame pair's two warps) or the group ends; the warps take turns
// until all have finished the group, then the flush runs for every thread (the CTA barrier).  A warp that read another
// warp's shared memory without a barrier ordering the two would see it stale here.
template <class Body, class Tile, class LAY>
static void run_warp_body(const typename Body::Args& a, const TwPair<typename Body::T>* twa) {
  using T = typename Body::T;
  std::vector<typename Tile::V> smem(Tile::template smem_elems<LAY>());
  std::vector<T> acc(Body::ACC_BYTES / sizeof(T));
  std::vector<Tile> thr(Tile::THREADS);
  constexpr int warps = (Tile::THREADS + 31) / 32;
  for (long g = 0; g < a.w.groups; ++g) {
    const long steps = a.w.rounds(g) * Body::kPhases;
    std::vector<long> pos(warps, 0);
    for (bool left = true; left;) {
      left = false;
      for (int w = 0; w < warps; ++w) {
        for (bool stop = false; !stop && pos[w] < steps; ++pos[w]) {
          const long r = pos[w] / Body::kPhases;
          const int p = (int)(pos[w] % Body::kPhases);
          static_for<0, Body::kPhases>([&](auto P) {
            if (decltype(P)::value != p) return;
            for (int t = 32 * w; t < std::min(32 * (w + 1), Tile::THREADS); ++t)
              Body::template phase<decltype(P)::value>(thr[t], a, g, r, t, smem.data(), acc.data(), twa);
          });
          stop = Body::pair_barrier(p);
        }
        left |= pos[w] < steps;
      }
    }
    for (int t = 0; t < Tile::THREADS; ++t) Body::flush(a, g, t, acc.data());
  }
}

// every on-chip size class of precision T (onchip_configs.cuh), smallest first: f(class)
template <typename T, class F> static void for_each_onchip(F&& f) {
  for (size_t l = 1; l <= ((size_t)1 << 16); l *= 2) onchip::visit_onchip<T>(l, f);
}

// ---- inputs -------------------------------------------------------------------------------------------------------
// uniform in [-1, 1), from a 64-bit LCG
static double rnd(unsigned long long& s) {
  s = s * 6364136223846793005ull + 1442695040888963407ull;
  return (double)(s >> 11) / 9007199254740992.0 * 2 - 1;
}

template <typename T> static void fill(std::vector<cpx<T>>& x, unsigned seed) {
  unsigned long long s = seed * 2654435761ull + 12345;
  for (auto& v : x) {
    v.x = (T)rnd(s);
    v.y = (T)rnd(s);
  }
}

// 16-byte aligned storage (what cudaMalloc gives), so that the row offsets are the ones a device buffer would have
template <typename V> struct Buf {
  std::vector<double2> raw;
  V* p;
  explicit Buf(size_t n) : raw((n * sizeof(V) + 15) / 16 + 1), p(reinterpret_cast<V*>(raw.data())) {}
  V& operator[](size_t i) { return p[i]; }
};

// ---- shared-memory bank conflicts ---------------------------------------------------------------------------------
// worst-case degree of one warp-wide shared access, element size B bytes: lanes are served in groups of 128 bytes
// worth of lanes (half-warp for 8 B, quarter-warp for 16 B); distinct addresses in the same bank conflict, identical
// addresses broadcast; inactive lanes have index < 0
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

// ---- spectrum access log ------------------------------------------------------------------------------------------
struct Access { uintptr_t addr; int bytes; };
static std::vector<Access> g_access;
__attribute__((unused)) static void spec_record(const void* p, int bytes) { g_access.push_back({(uintptr_t)p, bytes}); }

// Checks the log against the spectrum [base, base + rows * row_bytes): every access inside it, aligned to its width,
// at most `widest_allowed` bytes wide, and (two rows or more) some at odd rows.  Prints one line, "<what> accesses:
// ...", clears the log and returns the number of failures.
__attribute__((unused)) static int check_access(const char* what, const void* base, size_t rows, size_t row_bytes,
                                                int widest_allowed) {
  size_t odd = 0, outside = 0, misaligned = 0;
  int widest = 0;
  const uintptr_t b = (uintptr_t)base;
  for (const Access& a : g_access) {
    widest = std::max(widest, a.bytes);
    if (a.addr < b || a.addr + a.bytes > b + rows * row_bytes) { ++outside; continue; }
    if (a.addr % a.bytes) ++misaligned;
    if (((a.addr - b) / row_bytes) % 2 == 1) ++odd;
  }
  const bool ok = !g_access.empty() && widest <= widest_allowed && !outside && !misaligned && (rows < 2 || odd > 0);
  printf("  %s accesses: %zu (%zu at odd rows), widest %d B, misaligned %zu, outside %zu %s\n", what, g_access.size(),
         odd, widest, misaligned, outside, ok ? "OK" : "FAIL");
  g_access.clear();
  return !ok;
}

// ---- real-input transforms: tables and direct references ----------------------------------------------------------
// w[j] = exp(-2 pi i j / n)
__attribute__((unused)) static void twiddles(long n, std::vector<double>& wr, std::vector<double>& wi) {
  wr.resize(n); wi.resize(n);
  for (long j = 0; j < n; ++j) host_twiddle((size_t)j, (size_t)n, &wr[j], &wi[j]);
}

// the pair table of real_kernels.cuh for N = 2M: w_N^k, k <= M/2
template <typename T> static std::vector<cpx<T>> pair_table(long m) {
  std::vector<cpx<T>> tab(m / 2 + 1);
  for (long k = 0; k <= m / 2; ++k) {
    double re, im;
    host_twiddle((size_t)k, (size_t)(2 * m), &re, &im);
    tab[k] = mk<T>((T)re, (T)im);
  }
  return tab;
}

// Z = FFT_M(z) of each of `batch` rows of 2M reals x packed as z[j] = x[2j] + i x[2j+1], in double, rounded to T
template <typename T> static std::vector<cpx<T>> packed_fft(const std::vector<double>& x, long m, long batch) {
  const long n = 2 * m;
  std::vector<double> wr, wi;
  twiddles(m, wr, wi);
  std::vector<cpx<T>> z(m * batch);
  for (long b = 0; b < batch; ++b)
    for (long k = 0; k < m; ++k) {
      double a = 0, c = 0;
      for (long j = 0; j < m; ++j) {
        const double zr = x[b * n + 2 * j], zi = x[b * n + 2 * j + 1], tr = wr[(k * j) % m], ti = wi[(k * j) % m];
        a += zr * tr - zi * ti; c += zr * ti + zi * tr;
      }
      z[b * m + k] = mk<T>((T)a, (T)c);
    }
  return z;
}

// the unscaled inverse FFT_M of each of `batch` rows of Z, in double, as 2M interleaved reals per row
template <typename T> static std::vector<double> packed_ifft(const std::vector<cpx<T>>& z, long m, long batch) {
  const long n = 2 * m;
  std::vector<double> wr, wi, y(n * batch);
  twiddles(m, wr, wi);
  for (long b = 0; b < batch; ++b)
    for (long j = 0; j < m; ++j) {
      double a = 0, c = 0;
      for (long k = 0; k < m; ++k) {
        const cpx<T> v = z[b * m + k];
        const double tr = wr[(k * j) % m], ti = -wi[(k * j) % m];
        a += v.x * tr - v.y * ti; c += v.x * ti + v.y * tr;
      }
      y[b * n + 2 * j] = a; y[b * n + 2 * j + 1] = c;
    }
  return y;
}
