// hbm_pattern.cu -- the HBM access pattern of the persistent two-pass kernel at f32 2^20 (csrc/fused_kernels.cuh),
// as a pure copy: no FFT, no L2 ring.  Run by tools/hbm_pattern_bench.py, which compiles it.
//
// A batch of 1024 x 1024 complex-f32 transforms is copied tile by tile.  A tile is 8 columns x 1024 rows (64 KB):
// the kernel's pass-1 load (a TMA box per 256 rows, evict-first, into a shared-memory staging buffer) and, because
// X[k1 + 1024 k2] for 8 consecutive k1 is the same 8 x 1024 footprint, also its pass-2 store (st.global.cs, 64 bytes
// per row, 8 KB apart).  One CTA per SM, two 256-thread consumer groups and producer lanes, items claimed just in
// time from an atomic queue in transform-major order, as in the kernel.  Variants:
//   group8: an item is one tile of one group; boxes 8 columns wide (64 B per row) -- the kernel today;
//   pair16: an item is two adjacent tiles of one CTA, loaded as boxes 16 columns wide (one 128-byte line per box row);
//           group g stores tile 2j + g, so both halves of every output line are stored by one SM at the same time;
//   pair8:  the same pairs, loaded as boxes 8 columns wide (separates the box width from the pairing).
// The output is checked to equal the input after each variant's first run.
//
// usage: hbm_pattern [batch] [rounds]     prints one line per round and variant: "time <variant> <round> <ms per copy>"
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdio>
#include <cstdlib>

#include "fused_kernels.cuh"

using namespace fb200::fused;

namespace {

constexpr int N1 = 1024, N2 = 1024;            // rows x columns of one transform
constexpr long N = (long)N1 * N2;
constexpr int GT = 256, G = 2;                  // consumer groups of 256 threads
constexpr int THREADS = G * GT + 128;           // + a producer warpgroup (setmaxnreg works on whole warpgroups)
constexpr int REGS_PRODUCER = 24, REGS_CONSUMER = 112;   // as in the kernel: the producers hand their registers over
constexpr int BOX_ROWS = 256;
constexpr int TILES = N2 / 8;                   // 8-column tiles per transform
constexpr uint32_t TILE_BYTES = 8u * 8u * N1;   // 64 KB
constexpr size_t SMEM = 2 * TILE_BYTES + 1024;

enum Mode { kGroup8 = 0, kPair16 = 1, kPair8 = 2 };

struct Ctl {
  uint64_t full[G], empty[G];
  int item[G];
};

template <int MODE>
__global__ void __launch_bounds__(THREADS, 1)
copy_kernel(const __grid_constant__ CUtensorMap map8, const __grid_constant__ CUtensorMap map16, float2* out,
            unsigned* queue, int batch) {
  constexpr bool PAIR = MODE != kGroup8;
  extern __shared__ __align__(1024) unsigned char smem[];
  float2* stage = reinterpret_cast<float2*>(smem);
  Ctl* ctl = reinterpret_cast<Ctl*>(smem + 2 * TILE_BYTES);
  const int tid = threadIdx.x;
  if (tid == 0) {
    for (int g = 0; g < G; ++g) {
      mbar_init(&ctl->full[g], 1);
      mbar_init(&ctl->empty[g], PAIR ? G * GT : GT);
    }
    fence_barrier_init();
  }
  __syncthreads();
  const long items = (long)batch * (PAIR ? TILES / 2 : TILES);

  if (tid >= G * GT) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(REGS_PRODUCER));
    // producer lane of group pw (group8: lanes 0 and 1), or of the CTA (pairs: lane 0)
    const int pw = tid - G * GT;
    if (pw >= (PAIR ? 1 : G)) return;
    float2* dst = stage + (size_t)pw * (TILE_BYTES / sizeof(float2));
    for (uint32_t it = 0;; ++it) {
      if (it > 0) mbar_wait(&ctl->empty[pw], (it - 1) & 1);
      const long w = (long)atomicAdd(queue, 1u);
      if (w >= items) { ctl->item[pw] = -1; mbar_arrive(&ctl->full[pw]); break; }
      ctl->item[pw] = (int)w;
      const int per = PAIR ? TILES / 2 : TILES;
      const int b = (int)(w / per), j = (int)(w % per);
      mbar_arrive_expect_tx(&ctl->full[pw], PAIR ? 2 * TILE_BYTES : TILE_BYTES);
      for (int r0 = 0; r0 < N1; r0 += BOX_ROWS) {
        const int y = b * N1 + r0;
        if (MODE == kGroup8) {
          tma_load_2d_first(dst + (size_t)r0 * 8, &map8, j * 16, y, &ctl->full[pw]);
        } else if (MODE == kPair16) {
          tma_load_2d_first(stage + (size_t)r0 * 16, &map16, j * 32, y, &ctl->full[0]);
        } else {
          for (int h = 0; h < 2; ++h)
            tma_load_2d_first(stage + (size_t)h * (TILE_BYTES / sizeof(float2)) + (size_t)r0 * 8, &map8,
                              (2 * j + h) * 16, y, &ctl->full[0]);
        }
      }
    }
    return;
  }

  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(REGS_CONSUMER));
  const int g = tid / GT, t = tid % GT;
  const int bar = PAIR ? 0 : g;   // the barriers this group waits on and releases
  const int col = t % 8, row0 = t / 8;
  for (uint32_t k = 0;; ++k) {
    if ((t & 31) == 0) mbar_wait(&ctl->full[bar], k & 1);
    __syncwarp();
    const int w = ctl->item[bar];
    if (w < 0) break;
    float2 v[N1 / 32];
    const float2* src;
    int pitch, b, tile;
    if (MODE == kGroup8) { src = stage + (size_t)g * (TILE_BYTES / sizeof(float2)); pitch = 8; b = w / TILES; tile = w % TILES; }
    else if (MODE == kPair16) { src = stage + 8 * g; pitch = 16; b = w / (TILES / 2); tile = 2 * (w % (TILES / 2)) + g; }
    else { src = stage + (size_t)g * (TILE_BYTES / sizeof(float2)); pitch = 8; b = w / (TILES / 2); tile = 2 * (w % (TILES / 2)) + g; }
#pragma unroll
    for (int i = 0; i < N1 / 32; ++i) v[i] = src[(size_t)(row0 + 32 * i) * pitch + col];
    mbar_arrive(&ctl->empty[bar]);
    float2* dst = out + (size_t)b * N + (size_t)tile * 8 + col;
#pragma unroll
    for (int i = 0; i < N1 / 32; ++i)
      asm volatile("st.global.cs.v2.f32 [%0], {%1, %2};" ::"l"(dst + (size_t)(row0 + 32 * i) * N2), "f"(v[i].x),
                   "f"(v[i].y)
                   : "memory");
  }
}

__global__ void fill_kernel(float2* x, size_t n) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const uint32_t h = (uint32_t)i * 2654435761u ^ (uint32_t)(i >> 32);
    x[i] = make_float2((float)(h & 0xffff), (float)(h >> 16));
  }
}

__global__ void diff_kernel(const float2* a, const float2* b, size_t n, unsigned long long* bad) {
  unsigned long long c = 0;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    c += a[i].x != b[i].x || a[i].y != b[i].y;
  if (c) atomicAdd(bad, c);
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

#define CK(x)                                                                              \
  do {                                                                                     \
    cudaError_t e_ = (x);                                                                  \
    if (e_ != cudaSuccess) {                                                               \
      fprintf(stderr, "%s:%d: %s: %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_)); \
      exit(2);                                                                             \
    }                                                                                      \
  } while (0)

// the kernel's input tensor map (csrc/twopass.cu), with boxes `cols` columns wide
CUtensorMap make_map(EncodeTiledFn enc, const float2* in, int batch, int cols) {
  CUtensorMap m;
  const cuuint64_t gdim[2] = {(cuuint64_t)(2 * N2), (cuuint64_t)batch * N1};
  const cuuint64_t gstride[1] = {(cuuint64_t)(N2 * sizeof(float2))};
  const cuuint32_t box[2] = {(cuuint32_t)(2 * cols), (cuuint32_t)BOX_ROWS};
  const cuuint32_t estr[2] = {1, 1};
  if (enc(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)in, gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
          CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS) {
    fprintf(stderr, "cuTensorMapEncodeTiled failed\n");
    exit(2);
  }
  return m;
}

}  // namespace

int main(int argc, char** argv) {
  const int batch = argc > 1 ? atoi(argv[1]) : 4096;
  const int rounds = argc > 2 ? atoi(argv[2]) : 5;
  constexpr int kReps = 3;   // copies per timed window
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q));
  if (!p || q != cudaDriverEntryPointSuccess) { fprintf(stderr, "no cuTensorMapEncodeTiled\n"); return 2; }
  const EncodeTiledFn enc = (EncodeTiledFn)p;
  int sms = 0;
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));

  const size_t n = (size_t)batch * N, bytes = n * sizeof(float2);
  float2 *in = nullptr, *out = nullptr;
  unsigned* queue = nullptr;
  unsigned long long* bad = nullptr;
  CK(cudaMalloc(&in, bytes));
  CK(cudaMalloc(&out, bytes));
  CK(cudaMalloc(&queue, sizeof(unsigned)));
  CK(cudaMalloc(&bad, sizeof(unsigned long long)));
  fill_kernel<<<4 * sms, 1024>>>(in, n);
  CK(cudaGetLastError());
  const CUtensorMap m8 = make_map(enc, in, batch, 8), m16 = make_map(enc, in, batch, 16);
  CK(cudaFuncSetAttribute(copy_kernel<kGroup8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM));
  CK(cudaFuncSetAttribute(copy_kernel<kPair16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM));
  CK(cudaFuncSetAttribute(copy_kernel<kPair8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM));

  const char* names[4] = {"group8", "pair16", "pair8", "contiguous"};
  auto run = [&](int v) {
    if (v == 3) { CK(cudaMemcpyAsync(out, in, bytes, cudaMemcpyDeviceToDevice)); return; }
    CK(cudaMemsetAsync(queue, 0, sizeof(unsigned)));
    if (v == 0) copy_kernel<kGroup8><<<sms, THREADS, SMEM>>>(m8, m16, out, queue, batch);
    if (v == 1) copy_kernel<kPair16><<<sms, THREADS, SMEM>>>(m8, m16, out, queue, batch);
    if (v == 2) copy_kernel<kPair8><<<sms, THREADS, SMEM>>>(m8, m16, out, queue, batch);
    CK(cudaGetLastError());
  };
  // every variant once on a poisoned output, checked: warm-up and proof that it copies every byte
  for (int v = 0; v < 4; ++v) {
    CK(cudaMemset(out, 0xff, bytes));
    CK(cudaMemset(bad, 0, sizeof(unsigned long long)));
    run(v);
    diff_kernel<<<4 * sms, 1024>>>(in, out, n, bad);
    unsigned long long h = 0;
    CK(cudaMemcpy(&h, bad, sizeof h, cudaMemcpyDeviceToHost));
    printf("check %s: %llu mismatches\n", names[v], h);
    if (h) return 1;
  }
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  for (int r = 0; r < rounds; ++r)
    for (int i = 0; i < 4; ++i) {
      const int v = (i + r) % 4;   // rotate the order from round to round
      CK(cudaEventRecord(e0));
      for (int k = 0; k < kReps; ++k) run(v);
      CK(cudaEventRecord(e1));
      CK(cudaEventSynchronize(e1));
      float ms = 0;
      CK(cudaEventElapsedTime(&ms, e0, e1));
      printf("time %s %d %.4f\n", names[v], r, ms / kReps);
    }
  fflush(stdout);
  return 0;
}
