// fused_kernels.cuh -- the flagship kernel: both passes of the four-step FFT in ONE persistent,
// warp-specialised launch.
//
//   * one CTA per SM: G consumer groups, each processing one TileFFT tile in registers at a time, and
//     one producer warp (a first version let thread 0 of each group produce: the ~3000 cycles of
//     queue/TMA work per tile then sat on the critical path of its group's first barrier);
//   * the producer waits until its group has emptied the staging buffer, then claims an item of a global
//     work queue (atomic counter) whose order interleaves pass-1 tiles of transform s with pass-2 tiles
//     of transform s-LAG, waits for the tile's dependencies, and brings the tile into the group's
//     shared-memory staging buffer with TMA: a 2-D tensor-map box for the
//     strided column tiles of pass 1 (cp.async.bulk.tensor), plain bulk copies for the contiguous
//     row tiles of pass 2 (cp.async.bulk) -- completion is signalled on an mbarrier (full[g]);
//   * a consumer group waits on full[g], pulls its 32 (16) samples per thread out of the staging
//     buffer, releases it (empty[g]) so the next tile's TMA overlaps ALL of the remaining work,
//     runs stage A, exchanges through a shared buffer (one buffer, taken under a lock: the
//     exchange is ~10% of a tile), runs stage B and stores straight from registers;
//   * the intermediate A[k1][n2] lives in a ring of RING transforms (any RING >= 2; slot = b % RING)
//     that stays in the 50 MB L2: pass-1 tiles of transform b may only start once pass 2 of transform
//     b-RING has consumed the slot (done2), pass-2 tiles of b once all pass-1 tiles of b are stored (done1).
//     The scheme cannot deadlock: every dependency points to an earlier queue position; the tile a group
//     computes in registers waits on nothing; and a producer claims only into an empty staging buffer, so
//     the earliest claimed but unfinished item depends only on finished items and has a buffer to land in.
//     A group holds at most two claimed items (registers, staging), so about 2 x G x SMs queue positions
//     are in flight, and the ring must cover that window for the dependency waits to stay short.
//
// HBM therefore sees each sample exactly twice (one read, one write); there are no launch gaps or
// partial waves, and memory latency is hidden by the TMA prefetch instead of by occupancy.
#pragma once

#include <cuda.h>

#include <cstdint>

#include "tilefft.cuh"

namespace fb200 {
namespace fused {

// ---- PTX wrappers ---------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded spin: a protocol bug must abort the kernel (trap), never hang the GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  for (unsigned spins = 0; !mbar_try_wait(bar, parity); ++spins)
    if (spins > (1u << 22)) __trap();
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int x, int y, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
      ::"r"(smem_u32(dst)), "l"(map), "r"(x), "r"(y), "r"(smem_u32(bar))
      : "memory");
}
// same, with an L2 evict-first hint: the transform input is read exactly once
__device__ __forceinline__ void tma_load_2d_first(void* dst, const CUtensorMap* map, int x, int y, uint64_t* bar) {
  asm volatile(
      "{\n\t.reg .b64 pol;\n\tcreatepolicy.fractional.L2::evict_first.b64 pol, 1.0;\n\t"
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%2, %3}], "
      "[%4], pol;\n\t}"
      ::"r"(smem_u32(dst)), "l"(map), "r"(x), "r"(y), "r"(smem_u32(bar))
      : "memory");
}
// brings a box of the tensor into L2 only (no shared-memory destination, no completion signal)
__device__ __forceinline__ void tma_prefetch_2d(const CUtensorMap* map, int x, int y) {
  asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global.tile [%0, {%1, %2}];" ::"l"(map), "r"(x), "r"(y) : "memory");
}
__device__ __forceinline__ void bulk_load(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ unsigned ld_acquire(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_release_add(unsigned* p, unsigned v) {
  asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned atom_add_acq_rel_cta_shared(unsigned* p, unsigned v) {
  unsigned old;
  asm volatile("atom.acq_rel.cta.shared::cta.add.u32 %0, [%1], %2;" : "=r"(old) : "r"(smem_u32(p)), "r"(v) : "memory");
  return old;
}
__device__ __forceinline__ void st_release_cta_shared(unsigned* p, unsigned v) {
  asm volatile("st.release.cta.shared::cta.u32 [%0], %1;" ::"r"(smem_u32(p)), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned ld_acquire_cta_shared(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.cta.shared::cta.u32 %0, [%1];" : "=r"(v) : "r"(smem_u32(p)) : "memory");
  return v;
}
__device__ __forceinline__ void spin_until_ge(const unsigned* p, unsigned target) {
  for (unsigned spins = 0; ld_acquire(p) < target; ++spins) {
    if (spins > (1u << 24)) __trap();
    __nanosleep(64);
  }
}
__device__ __forceinline__ void group_sync(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// ---- work queue ---------------------------------------------------------------------------------------------
struct WorkItem { int pass, b, tile, slot; };  // pass: 1, 2, or -1 = queue exhausted; slot = b % ring

// Queue order: slot s = 0 .. B+LAG-1 holds [pass-1 tiles of transform s] then [pass-2 tiles of s-LAG].
__host__ __device__ inline WorkItem decode_work(long w, int batch, int lag, int t1, int t2) {
  WorkItem it = {-1, 0, 0, 0};
  const long total = (long)batch * (t1 + t2);
  if (w >= total) return it;
  const int d = lag < batch ? lag : batch;
  const long pro = (long)d * t1;
  if (w < pro) { it.pass = 1; it.b = (int)(w / t1); it.tile = (int)(w % t1); return it; }
  w -= pro;
  const long steady = (long)(batch - d) * (t1 + t2);
  if (w < steady) {
    const int s = d + (int)(w / (t1 + t2));
    const int r = (int)(w % (t1 + t2));
    if (r < t1) { it.pass = 1; it.b = s; it.tile = r; }
    else { it.pass = 2; it.b = s - d; it.tile = r - t1; }
    return it;
  }
  w -= steady;
  it.pass = 2; it.b = (batch - d) + (int)(w / t2); it.tile = (int)(w % t2);
  return it;
}

// Ring and lag of one launch.  A batch that fills only part of the plan's ring gets a smaller ring: it is halved
// while half of it still holds the whole batch (so a shrunk ring never wraps), down to 2 slots, and the lag stays
// below the ring.
struct RingLag { int ring, lag; };
__host__ __device__ inline RingLag launch_ring(int ring, int lag, long batch) {
  while (ring > 2 && (long)(ring / 2) >= batch) ring = ring / 2 > 2 ? ring / 2 : 2;
  RingLag r = {ring, lag < ring - 1 ? lag : ring - 1};
  return r;
}

template <typename T> struct FusedArgs {
  const cpx<T>* in;
  cpx<T>* out;
  cpx<T>* scratch;            // RING transforms
  const TwPair<T>* twa;       // stage-A twiddles of the pass-1 register tile (length N1)
  const TwPair<T>* twa2;      // ... of the pass-2 register tile (length N2; same table when the tiles are equal)
  const cpx<T>* tbase;        // [tile][col][p]  w_N^{n2*p}        (pass-1 tile tables, contiguous per tile)
  const cpx<T>* tstep;        // [tile][r][col]  w_N^{R*n2*r}
  unsigned* counters;         // [0] queue head, [1 .. 1+B) done1, [1+B .. 1+2B) done2
  int batch, ring, lag;
  T scale;
  int do_scale;
  long long* trace;           // optional phase timestamps of CTA 0 (debugging / DESIGN.md timeline), else nullptr
  uint32_t trace_from;        // first tile of each warp the trace records (kTraceTiles from there)
};

// Configuration: N = N1 * N2 (two register-tile lengths, see RB_ / RA2_ ... below), tiles of C = 8 FFTs, G consumer groups per CTA, EXB exchange buffers (group g uses
// g % EXB, under a lock when shared); the staging buffer is released as soon as the samples are in registers.
// The intermediate is stored in 8 x 8 blocks [k1 / 8][n2 / 8][k1 % 8][n2 % 8]: a pass-1 tile writes 256-byte runs (a
// warp's store = 4 consecutive k1 x 8 columns; row-major A[k1][n2] gave four 64-byte pieces and twice the LSU
// wavefronts), and a pass-2 tile (8 rows k1) is
// still one contiguous bulk copy; its threads pick their samples with the block-fast mapping (tilefft.cuh), under
// which a warp needs only 8 different stage twiddles (broadcast loads).  The base table of the factored inter-pass
// twiddle is [tile][p][col] (conflict-free for lanes = 8 columns x 4 p).
// DIRECT_: no shared-memory staging: the consumers load their samples from global memory straight into registers
//          (pass 1: the input, which the producer lane has prefetched into L2 one tile period ahead with
//          cp.async.bulk.prefetch.tensor; pass 2: the L2-resident intermediate, ld.global.cg), one exchange buffer
//          per group and no lock.  Meant for f64, where four 128-thread groups can hide the load latency; the f32
//          configurations with two 256-thread groups stage through shared memory.
// RB_: second radix of the register tile when the tile length L = R_ * RB_ is not a square (L = 128 = 16 x 8,
//      512 = 32 x 16): N = L^2 = 2^14, 2^18.
// C1_: columns per pass-1 tile (8, or 16 = two 8 x 8 block columns: then the strided input is read in 128-byte pieces
//      and a 512-point pass-1 tile has as many threads as a 1024-point pass-2 tile: 2^19 = 512 x 1024).
// TABG_: the factored-twiddle tables of a pass-1 tile are read from global memory (L2-resident, 6 KB per tile) instead
//      of travelling into shared memory with the tile: for the one configuration whose shared memory is full (2^19).
// RA2_, RB2_, E1_, E2_: a different register tile for pass 2 (N2 = RA2_ * RB2_ != N1 = R_ * RB_: the odd powers of
//      two, e.g. 2^15 = 128 x 256); E1_ / E2_ samples per thread chosen so that both tiles have the same number of
//      threads per FFT (TP = N1 / E1 = N2 / E2), i.e. the same group size.
template <typename T_, int R_, int C_, int G_, int PAD1_, int EXB_ = 1, bool DIRECT_ = false, int RB_ = R_,
          int RA2_ = R_, int RB2_ = RB_, int E1_ = (R_ > RB_ ? R_ : RB_), int E2_ = (RA2_ > RB2_ ? RA2_ : RB2_),
          int C1_ = C_, bool TABG_ = false>
struct FusedCfg {
  using T = T_;
  static constexpr bool DIRECT = DIRECT_, TABG = TABG_;
  static_assert(!DIRECT_ || EXB_ == G_, "direct loads: one exchange buffer per group");
  static constexpr int RA = R_, RB = RB_, RA2 = RA2_, RB2 = RB2_, C = C_, C1 = C1_, G = G_, EXB = EXB_;
  static constexpr long N1 = (long)RA * RB, N2 = (long)RA2 * RB2, N = N1 * N2;
  template <bool FWD> using Tile1 = TileFFT<T, RA, RB, E1_, C1, FWD>;    // pass 1: C1 columns, FFT length N1
  template <bool FWD> using Tile2 = TileFFT<T, RA2, RB2, E2_, C, FWD>;   // pass 2: C rows, FFT length N2
  static_assert(Tile1<true>::THREADS == Tile2<true>::THREADS, "both register tiles must use the same group size");
  using Lay1 = ExLayout<RA * C1 + PAD1_, C1, 1>;                   // pass 1: scatter and gather col-fast
  // pass 2: scatter block-fast (row stride = 2 mod 16 for 8-byte, odd for 16-byte elements: conflict-free for
  // lanes = 8 positions x 4 FFTs), gather col-fast
  using Lay2 = ExLayout<RA2 * C + (sizeof(T_) == 4 ? 2 : 1), C, 1>;
  static_assert(C_ == 8 && (C1_ == 8 || C1_ == 16) && RB_ % 8 == 0 && RB2_ % 8 == 0, "the blocked intermediate: 8 x 8 blocks");
  static constexpr int GT = Tile1<true>::THREADS;     // threads per group
  static constexpr int CONSUMERS = G * GT;
  // setmaxnreg is a warpgroup-wide instruction: consumers and producers must not share a group of four warps
  static_assert(CONSUMERS % 128 == 0, "the consumer threads must fill whole warpgroups");
  static constexpr int AUX = ((G + 1 + 3) / 4) * 128;  // G producer warps + 1 signaller warp, in whole warpgroups
  static constexpr int THREADS = CONSUMERS + AUX;
  // Register budget.  Registers are handed out per 4 warps, so a 17th warp costs as much as 4; the
  // producer warpgroup therefore gives its registers back (setmaxnreg.dec) and the consumers take
  // them (setmaxnreg.inc): LAUNCH_REGS per thread at launch, REGS_CONSUMER / REGS_PRODUCER afterwards.
  static constexpr int LAUNCH_REGS = ((65536 / THREADS) / 8) * 8;
  static constexpr int REGS_PRODUCER = 24;
  static constexpr int REGS_CONSUMER_RAW = ((LAUNCH_REGS * THREADS - REGS_PRODUCER * AUX) / CONSUMERS / 8) * 8;
  static constexpr int REGS_CONSUMER = REGS_CONSUMER_RAW > 232 ? 232 : REGS_CONSUMER_RAW;
  static constexpr int T1 = (int)(N2 / C1), T2 = (int)(N1 / C);
  static constexpr uint32_t TILE1_BYTES = (uint32_t)(sizeof(cpx<T>) * C1 * N1), TILE2_BYTES = (uint32_t)(sizeof(cpx<T>) * C * N2);
  static constexpr int TAB_BASE = C1 * RA, TAB_STEP = C1 * RB, TAB_ELEMS = TAB_BASE + TAB_STEP;   // [base | step] of a tile
  static constexpr uint32_t TAB_BASE_BYTES = (uint32_t)(sizeof(cpx<T>) * TAB_BASE), TAB_STEP_BYTES = (uint32_t)(sizeof(cpx<T>) * TAB_STEP);
  static constexpr uint32_t TAB_BYTES = TABG ? 0 : TAB_BASE_BYTES + TAB_STEP_BYTES;   // travelling with a tile
  static constexpr int EX1 = Tile1<true>::template smem_elems<Lay1>(), EX2 = Tile2<true>::template smem_elems<Lay2>();
  static constexpr int EX_ELEMS = EX1 > EX2 ? EX1 : EX2;
  static constexpr size_t EX_BYTES = ((sizeof(cpx<T>) * EX_ELEMS + 127) / 128) * 128;
  static constexpr int TWA1_PAIRS = (RA / 2) * RB, TWA2_PAIRS = (RA2 / 2) * RB2;
  static constexpr bool SAME_TILE = RA == RA2 && RB == RB2 && E1_ == E2_;   // one stage-twiddle table serves both passes
  static constexpr size_t TWA1_BYTES = sizeof(TwPair<T>) * TWA1_PAIRS,
                          TWA_BYTES = TWA1_BYTES + (SAME_TILE ? 0 : sizeof(TwPair<T>) * TWA2_PAIRS);
  static constexpr size_t BUF_BYTES = DIRECT ? 0 : (size_t)(TILE1_BYTES > TILE2_BYTES ? TILE1_BYTES : TILE2_BYTES);   // staging
  // layout: staging[G] | exchange[EXB] | twa (tile 1, tile 2) | tile tables [G][2 (double buffer)][base, step] | control
  static constexpr size_t OFF_EX = (size_t)G * BUF_BYTES;
  static constexpr size_t OFF_TWA = OFF_EX + (size_t)EXB * EX_BYTES;
  static constexpr size_t OFF_TAB = OFF_TWA + TWA_BYTES;
  static constexpr size_t OFF_CTL = OFF_TAB + (size_t)G * 2 * TAB_BYTES;
  static constexpr size_t SMEM_BYTES = OFF_CTL + 2048 /* control block: G * sizeof(GroupCtl) + locks */;
  static constexpr int BOX_ROWS = N1 < 256 ? (int)N1 : 256;   // TMA box limit: 256 per dimension
  static_assert(SMEM_BYTES <= 232448, "exceeds the 227 KB of shared memory per CTA");
  static constexpr bool PAIR = false;
  using Unpaired = FusedCfg;
};

// Pair items: one producer lane per CTA claims two adjacent tiles at a time (pass-1 tiles 2j, 2j+1 or pass-2 tiles
// 2i, 2i+1) and loads tile 2 x item + g into the staging buffer of group g, once both groups have emptied theirs.  The
// two groups then load and store the two halves of the same 128-byte lines of HBM at about the same time, where
// single items leave each half to a different SM at an unrelated moment (DESIGN.md 4.2, 5).  Everything a group
// does is unchanged: its staging layout, its tile, its counters.
template <class Base> struct PairCfg : Base {
  static_assert(Base::G == 2 && !Base::DIRECT && Base::T1 % 2 == 0 && Base::T2 % 2 == 0, "pairs: two staged groups");
  static constexpr bool PAIR = true;
  using Unpaired = Base;
};

constexpr int kStoreRing = 16;

struct GroupCtl {            // per-group control block in shared memory
  uint64_t full;             // TMA for the group's next tile has landed
  uint64_t empty;            // every thread of the group is done with the staging buffer
  WorkItem desc;             // the tile the staging buffer holds / will hold
  unsigned loaded;           // warps of the group that are done with the ring rows of the current pass-2 tile
  unsigned stored_warps;     // warps of the group that have issued the stores of the current pass-1 tile
  unsigned stored_seq;       // pass-1 tiles of this group whose stores have all been issued
  unsigned finished;         // the group has left its tile loop
  unsigned acked;            // pass-1 tiles of this group the signaller has published (back-pressure)
  int store_b[kStoreRing];   // transform index of pass-1 tile number n at [n % kStoreRing]
};

// Direct loads: a pass-2 tile reports its ring slot as consumed (done2) once every warp of the group has loaded and
// discarded the slot's rows.  Each warp's discards are ordered before its lane 0's acq_rel count in shared memory
// (__syncwarp), and the last warp of the group publishes with a gpu-scope release: a pass-1 tile of b + RING that sees
// done2[b] complete stores into the slot only after all of them.  Called by every thread of the group.
__device__ __forceinline__ void report_consumed(GroupCtl* ctl, unsigned* done2_b, int warps) {
  __syncwarp();
  if ((threadIdx.x & 31) == 0 && atom_add_acq_rel_cta_shared(&ctl->loaded, 1u) == (unsigned)warps - 1) {
    ctl->loaded = 0;
    red_release_add(done2_b, 1u);
  }
}

// Issues the loads of one work item into the group's staging buffer (one thread of the group).
template <class Cfg>
__device__ __forceinline__ void issue_tile(const WorkItem& wi, const CUtensorMap* in_map,
                                           const FusedArgs<typename Cfg::T>& a, cpx<typename Cfg::T>* dst,
                                           cpx<typename Cfg::T>* tab, GroupCtl* ctl) {
  using V = cpx<typename Cfg::T>;
  constexpr int C = Cfg::C;
  WorkItem d = wi;
  d.slot = wi.b % a.ring;
  ctl->desc = d;
  if (wi.pass < 0) { mbar_arrive(&ctl->full); return; }
  if constexpr (Cfg::DIRECT) {
    // nothing to stage, the consumers read global memory themselves; only the tile tables of a pass-1 tile travel
    if (wi.pass == 2) { mbar_arrive(&ctl->full); return; }
    if constexpr (Cfg::TABG) { mbar_arrive(&ctl->full); return; }
    mbar_arrive_expect_tx(&ctl->full, Cfg::TAB_BYTES);
    bulk_load(tab, a.tbase + (size_t)wi.tile * Cfg::TAB_BASE, Cfg::TAB_BASE_BYTES, &ctl->full);
    bulk_load(tab + Cfg::TAB_BASE, a.tstep + (size_t)wi.tile * Cfg::TAB_STEP, Cfg::TAB_STEP_BYTES, &ctl->full);
    return;
  }
  // (the group's reads of `dst` are ordered before this refill by the empty-mbarrier wait of the caller)
  if (wi.pass == 1) {
    mbar_arrive_expect_tx(&ctl->full, Cfg::TILE1_BYTES + Cfg::TAB_BYTES);
    constexpr int BOX = Cfg::BOX_ROWS;
    const int x = wi.tile * Cfg::C1 * 2;  // in scalars of T
#pragma unroll
    for (int r0 = 0; r0 < (int)Cfg::N1; r0 += BOX)
      tma_load_2d_first(dst + (size_t)r0 * Cfg::C1, in_map, x, (int)((long)wi.b * Cfg::N1 + r0), &ctl->full);
    if constexpr (!Cfg::TABG) {
      bulk_load(tab, a.tbase + (size_t)wi.tile * Cfg::TAB_BASE, Cfg::TAB_BASE_BYTES, &ctl->full);
      bulk_load(tab + Cfg::TAB_BASE, a.tstep + (size_t)wi.tile * Cfg::TAB_STEP, Cfg::TAB_STEP_BYTES, &ctl->full);
    }
  } else {
    mbar_arrive_expect_tx(&ctl->full, Cfg::TILE2_BYTES);
    const V* src = a.scratch + (size_t)d.slot * Cfg::N + (size_t)wi.tile * C * Cfg::N2;
    constexpr uint32_t PIECE = 16384;
#pragma unroll
    for (uint32_t o = 0; o < Cfg::TILE2_BYTES; o += PIECE)
      bulk_load((unsigned char*)dst + o, (const unsigned char*)src + o,
                Cfg::TILE2_BYTES - o < PIECE ? Cfg::TILE2_BYTES - o : PIECE, &ctl->full);
  }
}

// Address of the counter a work item depends on (nullptr: no dependency) and the value it must reach.
template <class Cfg>
__device__ __forceinline__ const unsigned* dep_counter(const WorkItem& wi, const FusedArgs<typename Cfg::T>& a,
                                                       unsigned* target) {
  if (wi.pass == 1 && wi.b >= a.ring) { *target = (unsigned)Cfg::T2; return a.counters + 1 + a.batch + (wi.b - a.ring); }
  if (wi.pass == 2) { *target = (unsigned)Cfg::T1; return a.counters + 1 + wi.b; }
  *target = 0;
  return nullptr;
}

// The arithmetic of one consumer thread between the barriers of the kernel, per pass (Pass<1>: column tiles on
// Tile1, Pass<2>: row tiles on Tile2).  __host__ __device__: the kernel below and tools/emulate.cu (CPU, thread by
// thread) run exactly this code.
template <class Cfg, bool FWD> struct FusedMath {
  using T = typename Cfg::T;
  using V = cpx<T>;
  using Tile1 = typename Cfg::template Tile1<FWD>;
  using Tile2 = typename Cfg::template Tile2<FWD>;
  static constexpr int C = Cfg::C;
  static constexpr long N = Cfg::N, N1 = Cfg::N1, N2 = Cfg::N2;
  static_assert(Tile2::kBlockFastOk, "pass-2 tile shape does not fit the block-fast mapping");

  template <int PASS, int DUMMY = 0> struct Pass;

  // ---- pass 1: staging = [n1][C] (TMA box), or with DIRECT C columns of x in global memory (row stride N2, read
  // once); everything col-fast; store = inter-pass twiddle (factored, tables tb = [base | step]) into the blocked
  // ring slot (kept in L2)
  template <int DUMMY> struct Pass<1, DUMMY> {
    using Tile = Tile1;
    static FB_HD void load(Tile& f, int t, const V* stage) {
      if constexpr (Cfg::DIRECT) f.template load<kMapCF, N2, 1, 1>(t, stage);
      else f.template load<kMapCF, Cfg::C1, 1>(t, stage);
    }
    static FB_HD void stage_a(Tile& f, int t, const TwPair<T>* twa) { f.template stage_a<kMapCF, true>(t, twa); }
    static FB_HD void scatter(const Tile& f, int t, V* exch) { f.template scatter<kMapCF, typename Cfg::Lay1>(t, exch); }
    static FB_HD void gather(Tile& f, int t, const V* exch) { f.template gather<kMapCF, typename Cfg::Lay1>(t, exch); }
  };
  // ---- pass 2: staging (or, DIRECT, the L2-resident ring: rewritten by other SMs during the kernel, L2 only) = the
  // tile's 8 x 8 blocks; block-fast up to the exchange, col-fast after it; transposed streaming store X[k1 + N1 * k2]
  template <int DUMMY> struct Pass<2, DUMMY> {
    using Tile = Tile2;
    static FB_HD void load(Tile& f, int t, const V* stage) {
      if constexpr (Cfg::DIRECT) f.template load_blocked<kMapBF, 2>(t, stage);
      else f.template load_blocked<kMapBF>(t, stage);
    }
    static FB_HD void stage_a(Tile& f, int t, const TwPair<T>* twa) { f.template stage_a<kMapBF, true>(t, twa); }
    static FB_HD void scatter(const Tile& f, int t, V* exch) { f.template scatter<kMapBF, typename Cfg::Lay2>(t, exch); }
    static FB_HD void gather(Tile& f, int t, const V* exch) { f.template gather<kMapCF, typename Cfg::Lay2>(t, exch); }
  };
  static constexpr int kMap2 = kMapBF;
  // `twa`: stage twiddles in the 8-byte-plane layout (TwPlanes): in both mappings 4 or 8 lanes share a pair.
  // Plane layout of the pair tables of the two tiles, entry i of tile `which`:
  static FB_HD void relayout_twa(void* planes, const TwPair<T>* src, int i, int pairs) {
    TwPlanes<T>::put(planes, pairs, i, src[i]);
  }
  static FB_HD void store1(const Tile1& f, int t, V* slot_base, int tile, const V* tbase, const V* tstep) {
    f.template store_factored<N2, 1, 2, N2 * 8, true>(t, slot_base + (size_t)tile * (8 * Cfg::C1), tbase, tstep);
  }
  static FB_HD void store2(const Tile2& f, int t, V* out_b, int tile, bool do_scale, T scale) {
    V* dst = out_b + (size_t)tile * C;
    if (do_scale) f.template store<kMapCF, N1, 1, false, true, 1>(t, dst, nullptr, scale);
    else f.template store<kMapCF, N1, 1, false, false, 1>(t, dst, nullptr, scale);
  }
};

constexpr int kTraceTiles = 64, kTracePhases = 8;
#define FB_TRACE(phase)                                                                                   \
  do {                                                                                                    \
    if (a.trace && blockIdx.x == 0 && (t & 31) == 0 && k - a.trace_from < kTraceTiles)                    \
      a.trace[(((long)g * (GT / 32) + (t >> 5)) * kTraceTiles + (k - a.trace_from)) * kTracePhases + (phase)] = \
          clock64();                                                                                      \
  } while (0)

#define FB_PTRACE(phase)                                                                                  \
  do {                                                                                                    \
    if (a.trace && blockIdx.x == 0 && it - a.trace_from < kTraceTiles)                                    \
      a.trace[(((long)(Cfg::CONSUMERS / 32) + g) * kTraceTiles + (it - a.trace_from)) * kTracePhases + (phase)] = \
          clock64();                                                                                      \
  } while (0)

template <class Cfg, bool FWD>
__global__ void __launch_bounds__(Cfg::THREADS, 1)
fused_twopass_kernel(const __grid_constant__ CUtensorMap in_map, const FusedArgs<typename Cfg::T> a) {
  using T = typename Cfg::T;
  using V = cpx<T>;
  constexpr int G = Cfg::G, GT = Cfg::GT, C = Cfg::C;
  constexpr long N = Cfg::N, N2 = Cfg::N2;
  constexpr int T1 = Cfg::T1, T2 = Cfg::T2;
  using Math = FusedMath<Cfg, FWD>;

  // No integer round-trip on this pointer: the compiler must keep the shared address space, otherwise
  // every staging/exchange access becomes a generic LD/ST (seen in the first profile of this kernel).
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  unsigned char* base = smem_raw;
  unsigned char* staging = base;                                             // [G][BUF_BYTES]
  unsigned char* exch_pool = base + Cfg::OFF_EX;
  TwPair<T>* twa1 = reinterpret_cast<TwPair<T>*>(base + Cfg::OFF_TWA);
  TwPair<T>* twa2 = Cfg::SAME_TILE ? twa1 : reinterpret_cast<TwPair<T>*>(base + Cfg::OFF_TWA + Cfg::TWA1_BYTES);
  V* tabs = reinterpret_cast<V*>(base + Cfg::OFF_TAB);                       // [G][2][base | step]
  GroupCtl* ctl_all = reinterpret_cast<GroupCtl*>(base + Cfg::OFF_CTL);
  int* locks = reinterpret_cast<int*>(ctl_all + G);   // one per exchange buffer

  const int tid = threadIdx.x;
  if (tid == 0) {
    for (int g = 0; g < G; ++g) {
      mbar_init(&ctl_all[g].full, 1);
      mbar_init(&ctl_all[g].empty, GT);
      ctl_all[g].loaded = 0;
      ctl_all[g].stored_warps = 0;
      ctl_all[g].stored_seq = 0;
      ctl_all[g].finished = 0;
      ctl_all[g].acked = 0;
    }
    for (int i = 0; i < Cfg::EXB; ++i) locks[i] = 0;
    fence_barrier_init();
  }
  // stage-A twiddles of both register tiles live in shared memory (8-byte planes)
  for (int i = tid; i < Cfg::TWA1_PAIRS; i += Cfg::THREADS) Math::relayout_twa(twa1, a.twa, i, Cfg::TWA1_PAIRS);
  if constexpr (!Cfg::SAME_TILE)
    for (int i = tid; i < Cfg::TWA2_PAIRS; i += Cfg::THREADS) Math::relayout_twa(twa2, a.twa2, i, Cfg::TWA2_PAIRS);
  __syncthreads();

  unsigned* queue = a.counters;
  unsigned* done1 = a.counters + 1;
  unsigned* done2 = a.counters + 1 + a.batch;

  if (tid >= Cfg::CONSUMERS) {
    // =============================== producer warpgroup =======================================================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(Cfg::REGS_PRODUCER));
    const int pw = (tid - Cfg::CONSUMERS) >> 5;
    if ((tid & 31) != 0) return;
    if constexpr (Cfg::PAIR) {
      if (pw == 0) {
        // ---- the producer of both groups (pair items): the same just-in-time claim, for a tile per group.  The CTA
        // holds at most two claimed, unfinished items (one in both groups' registers, one staged or in flight), every
        // dependency points to an earlier queue position, and the lane claims only once both staging buffers are
        // empty: the argument of the header comment holds item by item.
        const int g = 0;   // (trace row)
        uint32_t n_p1 = 0;
        for (uint32_t it = 0;; ++it) {
          FB_PTRACE(0);
          if (it > 0)
            for (int h = 0; h < G; ++h) mbar_wait(&ctl_all[h].empty, (it - 1) & 1);
          FB_PTRACE(2);
          const WorkItem wi = decode_work((long)atomicAdd(queue, 1u), a.batch, a.lag, T1 / 2, T2 / 2);
          unsigned target;
          const unsigned* dep = dep_counter<Cfg>(wi, a, &target);   // counted in tiles, as for single items
          if (dep) { spin_until_ge(dep, target); fence_proxy_async(); }
          FB_PTRACE(1);
          for (int h = 0; h < G; ++h) {
            WorkItem wh = wi;
            wh.tile = 2 * wi.tile + h;
            issue_tile<Cfg>(wh, &in_map, a, reinterpret_cast<V*>(staging + (size_t)h * Cfg::BUF_BYTES),
                            tabs + (size_t)h * 2 * Cfg::TAB_ELEMS + (size_t)(n_p1 & 1) * Cfg::TAB_ELEMS, &ctl_all[h]);
          }
          FB_PTRACE(3);
          n_p1 += wi.pass == 1;
          if (wi.pass < 0) break;
        }
        return;
      }
      if (pw < G) return;
    }
    if (pw < G) {
      // ---- producer of group pw: wait until the group has emptied its staging buffer, only then claim a queue
      // item, wait for its dependencies (blocking is fine here: nothing a consumer needs is held back by it),
      // refill the staging buffer by TMA.  Claiming just in time keeps a group at two claimed but unfinished
      // items (one in registers, one in staging or in flight): every item claimed ahead of that widens the
      // window of queue positions in flight, and with it the ring the dependency waits need to stay short.
      const int g = pw;
      GroupCtl* ctl = &ctl_all[g];
      V* stage_g = reinterpret_cast<V*>(staging + (size_t)g * Cfg::BUF_BYTES);
      V* tab_g = tabs + (size_t)g * 2 * Cfg::TAB_ELEMS;
      uint32_t n_p1 = 0;
      for (uint32_t it = 0;; ++it) {
        FB_PTRACE(0);
        if (it > 0) mbar_wait(&ctl->empty, (it - 1) & 1);
        FB_PTRACE(2);
        const WorkItem wi = decode_work((long)atomicAdd(queue, 1u), a.batch, a.lag, T1, T2);
        unsigned target;
        const unsigned* dep = dep_counter<Cfg>(wi, a, &target);
        if (dep) { spin_until_ge(dep, target); fence_proxy_async(); }
        FB_PTRACE(1);
        if constexpr (Cfg::DIRECT) {
          // The group started on the previous item when `empty` landed, so it will ask for this tile at most one tile
          // period from now (less by the dependency wait above): long enough for HBM -> L2 in the steady state,
          // short enough that the prefetched tiles of all groups (132 x G x 64 KB) do not crowd the intermediate
          // out of L2.
          if (wi.pass == 1) {
#pragma unroll
            for (int r0 = 0; r0 < (int)Cfg::N1; r0 += Cfg::BOX_ROWS)
              tma_prefetch_2d(&in_map, wi.tile * Cfg::C1 * 2, (int)((long)wi.b * Cfg::N1 + r0));
          }
        }
        issue_tile<Cfg>(wi, &in_map, a, stage_g, tab_g + (size_t)(n_p1 & 1) * Cfg::TAB_ELEMS, ctl);
        FB_PTRACE(3);
        n_p1 += wi.pass == 1;
        if (wi.pass < 0) break;
      }
    } else if (pw == G) {
      // ---- signaller: publishes finished pass-1 tiles.  The gpu-scope release fence costs ~2500 cycles; on a
      // consumer thread it delayed that thread's warp, and with it the whole group at its next barrier.
      unsigned seen[G];
#pragma unroll
      for (int g = 0; g < G; ++g) seen[g] = 0;
      for (unsigned idle = 0;;) {
        unsigned seq[G];
        bool all_done = true, work = false;
#pragma unroll
        for (int g = 0; g < G; ++g) {
          const unsigned fin = ld_acquire_cta_shared(&ctl_all[g].finished);   // read before seq: no tile is missed
          seq[g] = ld_acquire_cta_shared(&ctl_all[g].stored_seq);
          work = work || seen[g] < seq[g];
          all_done = all_done && fin && seen[g] == seq[g];
        }
        if (work) {
          __threadfence();   // every store the groups issued for tiles < seq[g] is visible gpu-wide after this
#pragma unroll
          for (int g = 0; g < G; ++g) {
            for (; seen[g] < seq[g]; ++seen[g]) atomicAdd(&done1[ctl_all[g].store_b[seen[g] % kStoreRing]], 1u);
            st_release_cta_shared(&ctl_all[g].acked, seen[g]);
          }
          idle = 0;
        } else {
          if (all_done) break;
          __nanosleep(100);
          if (++idle > (1u << 26)) __trap();
        }
      }
    }
    return;
  }

  // ======================================= consumer groups =====================================================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(Cfg::REGS_CONSUMER));
  const int g = tid / GT;
  const int t = tid - g * GT;
  V* stage_g = reinterpret_cast<V*>(staging + (size_t)g * Cfg::BUF_BYTES);
  V* tab_g = tabs + (size_t)g * 2 * Cfg::TAB_ELEMS;
  GroupCtl* ctl = &ctl_all[g];
  const int bar_id = 1 + g;
  V* exch = reinterpret_cast<V*>(exch_pool + (size_t)(g % Cfg::EXB) * Cfg::EX_BYTES);
  int* lock = &locks[g % Cfg::EXB];
  constexpr bool kLocked = Cfg::EXB < G;   // several groups share one exchange buffer
  uint32_t k_p1 = 0;   // pass-1 tiles consumed so far by this group: selects the tile-table buffer

  for (uint32_t k = 0;; ++k) {
    FB_TRACE(0);
    // one lane per warp polls (every poll is a shared-memory transaction on the LSU pipe the kernel is bound by);
    // __syncwarp orders the other lanes' reads of the staged data after its acquire
    if ((t & 31) == 0) mbar_wait(&ctl->full, k & 1);
    __syncwarp();
    const WorkItem wi = ctl->desc;
    if (wi.pass < 0) break;
    FB_TRACE(1);
    if (a.trace && blockIdx.x == 0 && t == 0 && k - a.trace_from < kTraceTiles)
      a.trace[((long)g * (GT / 32) * kTraceTiles + (k - a.trace_from)) * kTracePhases + 7] = wi.pass;
    const V* ring_rows = a.scratch + (size_t)wi.slot * N + (size_t)wi.tile * C * N2;   // pass 2: the tile's rows

    // One tile, from its samples to its stores; the whole group takes the same branch (wi is the group's item), so
    // the named barriers inside are reached by all of its threads.  P = Math::Pass<1> or Pass<2>.
    auto tile_body = [&](auto pass_tag) FB_LAMBDA {
      constexpr int PASS = decltype(pass_tag)::value;
      using P = typename Math::template Pass<PASS>;
      constexpr uint32_t TILE_BYTES = PASS == 1 ? Cfg::TILE1_BYTES : Cfg::TILE2_BYTES;
      // ---- staging (or global memory) -> registers; the staging buffer is free again as soon as every thread has
      // its samples ----
      typename P::Tile f;
      if constexpr (Cfg::DIRECT) P::load(f, t, PASS == 1 ? a.in + (size_t)wi.b * N + (size_t)wi.tile * Cfg::C1 : ring_rows);
      else P::load(f, t, stage_g);
      mbar_arrive(&ctl->empty);
      if constexpr (!Cfg::DIRECT && PASS == 2) {
        // The intermediate rows this tile just consumed are dead: drop them from L2 instead of letting the
        // cache write them back to HBM later (the slot is completely rewritten before it is read again).
        const unsigned char* rows = reinterpret_cast<const unsigned char*>(ring_rows);
        for (uint32_t o = (uint32_t)t * 128u; o < TILE_BYTES; o += (uint32_t)GT * 128u)
          asm volatile("discard.global.L2 [%0], 128;" ::"l"(rows + o) : "memory");
        // the last warp of the group to have pulled its samples reports the ring slot as consumed by this
        // tile -- promptly and from the consumer side (a lazy report by the producer could deadlock it
        // against its own dependency wait).  Each warp issues its discards before its count (__syncwarp), but the
        // report stays relaxed: report_consumed() here (gpu-scope release) made the f32 2^20 kernel 4.3 % slower,
        // a release after stage A 7.3 % (DESIGN.md 4.2).  So only timing orders these discards before the stores of
        // the pass-1 tile of b + RING, which sees done2, loads its input and computes a whole tile first.
        __syncwarp();
        if ((t & 31) == 0 && atomicAdd(&ctl->loaded, 1u) == GT / 32 - 1) { ctl->loaded = 0; atomicAdd(&done2[wi.b], 1u); }
      }
      FB_TRACE(2);

      P::stage_a(f, t, PASS == 1 ? twa1 : twa2);

      // ---- exchange through the shared buffer (under the CTA-wide lock when the groups share one) --------------
      if (kLocked && t == 0) {
        unsigned spins = 0;
        while (atomicCAS(lock, 0, 1) != 0) if (++spins > (1u << 26)) __trap();
      }
      FB_TRACE(3);
      group_sync(bar_id, GT);
      if constexpr (Cfg::DIRECT && PASS == 2) {
        // every warp of the group is past stage A, i.e. all loads of the tile have completed: drop its rows from L2,
        // then report the slot as consumed (not before: a pass-1 tile of b + RING may store into these rows as soon
        // as done2 is complete, and a discard landing after those stores would throw them away)
        const unsigned char* rows = reinterpret_cast<const unsigned char*>(ring_rows);
        for (uint32_t o = (uint32_t)t * 128u; o < TILE_BYTES; o += (uint32_t)GT * 128u)
          asm volatile("discard.global.L2 [%0], 128;" ::"l"(rows + o) : "memory");
        report_consumed(ctl, &done2[wi.b], GT / 32);
      }
      P::scatter(f, t, exch);
      FB_TRACE(4);
      group_sync(bar_id, GT);
      P::gather(f, t, exch);
      if constexpr (kLocked) {
        group_sync(bar_id, GT);
        if (t == 0) { __threadfence_block(); atomicExch(lock, 0); }
      }
      FB_TRACE(5);

      // ---- stage B and the stores -------------------------------------------------------------------------------
      f.stage_b();
      if constexpr (PASS == 1) {
        const V* tb = Cfg::TABG ? a.tbase + (size_t)wi.tile * Cfg::TAB_BASE : tab_g + (size_t)(k_p1 & 1) * Cfg::TAB_ELEMS;
        const V* ts = Cfg::TABG ? a.tstep + (size_t)wi.tile * Cfg::TAB_STEP : tb + Cfg::TAB_BASE;
        ++k_p1;
        Math::store1(f, t, a.scratch + (size_t)wi.slot * N, wi.tile, tb, ts);
        // report "stores issued"; the last warp of the group hands the tile to the signaller warp
        __syncwarp();
        if ((t & 31) == 0 && atom_add_acq_rel_cta_shared(&ctl->stored_warps, 1u) == GT / 32 - 1) {
          ctl->stored_warps = 0;
          for (unsigned spins = 0; k_p1 - ld_acquire_cta_shared(&ctl->acked) > (unsigned)kStoreRing; ++spins) {
            if (spins > (1u << 24)) __trap();   // the signaller is more than kStoreRing tiles behind: wait
            __nanosleep(100);
          }
          ctl->store_b[(k_p1 - 1) % kStoreRing] = wi.b;
          st_release_cta_shared(&ctl->stored_seq, k_p1);
        }
      } else {
        Math::store2(f, t, a.out + (size_t)wi.b * N, wi.tile, a.do_scale != 0, a.scale);
      }
      FB_TRACE(6);
    };
    if (wi.pass == 1) tile_body(std::integral_constant<int, 1>{});
    else tile_body(std::integral_constant<int, 2>{});
  }
  group_sync(bar_id, GT);
  if (t == 0) st_release_cta_shared(&ctl->finished, 1u);
}

}  // namespace fused
}  // namespace fb200
