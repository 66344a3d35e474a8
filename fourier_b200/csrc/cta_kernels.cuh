// cta_kernels.cuh -- one CTA owns whole transforms in shared memory: the Stockham autosort stage loop of the
// reference (fourier-algorithms/src/autosort/mod.rs:211-284,313-404: read (k*m+i)*stride+j, DFT_R, post-twiddle
// w_S^{i*k}, write (i*R+k)*stride+j, ping-pong between two buffers) with ALL stages inside one kernel:
// the first stage reads global memory, the last one writes it, everything in between stays in shared memory.
// HBM sees each sample once in and once out, whatever the number of stages.
//
// Serves every size the register-tile kernels do not: {2,3}-smooth N that are not a power of two (radix-3 is a
// first-class stage of the reference: mod.rs:20-21, butterfly.rs:9-22; its benches run 243 / 729 / 2187), powers of
// two between the on-chip and the two-pass kernels, and -- CHIRP mode -- the reference's Bluestein chirp-z
// (bluesteins.rs:218-259) for inner sizes M above the warp-level fused kernel: x*chirp (zero-padded to M) -> FFT_M
// -> *W -> IFFT_M -> *chirp*scale, the two pointwise products folded into the first loads of the two transforms and
// the last into the final store; the padded length-M intermediates never leave the SM.
//
// Layout: a group of `group` transforms of length `len` lives in a buffer of group*len samples, element e at word
// e + (e >> 5) (one pad element per 32: the scattered writes (i*R+k)*stride+j of the early stages, stride < 32,
// then spread over all banks -- checked by tools/emulate.cu).  One thread = one radix-R butterfly at a time;
// consecutive threads take consecutive q = i*stride + j, so shared-memory reads and the global loads / stores of
// the first / last stage are contiguous.
//
// Every function is __host__ __device__: tools/emulate.cu runs the same code thread by thread on the CPU.
#pragma once

#include <vector>

#include "cplx.cuh"

namespace fb200 {
namespace cta {

constexpr int kMaxStages = 16;
constexpr int kThreads = 256;

struct Stages {
  int count;
  int radix[kMaxStages];
  int tw_off[kMaxStages];        // first entry of the stage's twiddle block in Args::wtab
  unsigned magic[kMaxStages];    // ceil(2^32 / stride): q / stride == (q * magic) >> 32 for q * stride < 2^32
};

// Twiddles of stage s (sub-size S = R*m): block [k-1][i] = w_S^{i*k}, k = 1..R-1, i < m -- transposed so that the
// threads of a warp (consecutive q = i*stride + j: `stride` lanes share one i, then the next i) read one or two
// contiguous runs per k; the reference's per-stage layout is [i][k] (autosort/mod.rs:24-46), which a warp would
// gather with up to 32 different cache lines per load.  The last stage (S == R) has no twiddles.
inline int twiddle_entries(size_t len, const Stages& st) {
  size_t sub = len, total = 0;
  for (int s = 0; s < st.count; ++s) {
    const size_t r = (size_t)st.radix[s];
    if (sub != r) total += (r - 1) * (sub / r);
    sub /= r;
  }
  return (int)total;
}

FB_HD int padded(int e) { return e + (e >> 5); }
FB_HD int buffer_elems(int group, int len) { return padded(group * len) + 1; }

// Stage radices of a {2,3}-smooth length: 16s, then one of 8 / 4 / 2, then 9s, then a 3 (the reference factors
// [4, 8.., 4.., 3.., 2..], autosort/mod.rs:104-117; wider butterflies = fewer sweeps over shared memory).
// Returns false when len is not {2,3}-smooth or needs more than kMaxStages stages.
inline bool factorize(size_t len, Stages& st) {
  st.count = 0;
  for (int i = 0; i < kMaxStages; ++i) st.radix[i] = 0;
  if (len < 2) return false;
  int twos = 0, threes = 0;
  while (len % 2 == 0) { len /= 2; ++twos; }
  while (len % 3 == 0) { len /= 3; ++threes; }
  if (len != 1) return false;
  const size_t full = ((size_t)1 << twos) * [&] { size_t p = 1; for (int i = 0; i < threes; ++i) p *= 3; return p; }();
  auto push = [&](int r) { if (st.count < kMaxStages) st.radix[st.count] = r; ++st.count; };
  while (twos >= 4) { push(16); twos -= 4; }
  if (twos == 3) push(8);
  if (twos == 2) push(4);
  if (twos == 1) push(2);
  while (threes >= 2) { push(9); threes -= 2; }
  if (threes == 1) push(3);
  if (st.count > kMaxStages) return false;
  size_t sub = full, stride = 1;
  int off = 0;
  for (int s = 0; s < st.count; ++s) {
    const size_t r = (size_t)st.radix[s];
    st.tw_off[s] = off;
    st.magic[s] = stride == 1 ? 0u : (unsigned)((((unsigned long long)1 << 32) + stride - 1) / stride);
    if (sub != r) off += (int)((r - 1) * (sub / r));
    sub /= r;
    stride *= r;
  }
  return true;
}

// Host side: the twiddle blocks of every stage, `tw(idx, size, &re, &im)` = exp(-2 pi i idx / size) in double.
template <typename T, class TW>
inline std::vector<cpx<T>> make_stage_twiddles(size_t len, const Stages& st, TW&& tw) {
  std::vector<cpx<T>> out((size_t)twiddle_entries(len, st));
  size_t sub = len;
  for (int s = 0; s < st.count; ++s) {
    const size_t r = (size_t)st.radix[s], m = sub / r;
    if (sub != r)
      for (size_t k = 1; k < r; ++k)
        for (size_t i = 0; i < m; ++i) {
          double re, im;
          tw(i * k, sub, &re, &im);
          out[(size_t)st.tw_off[s] + (k - 1) * m + i] = mk<T>((T)re, (T)im);
        }
    sub /= r;
  }
  return out;
}

// DFT of R register values, natural order in and out; R in {2, 3, 4, 8, 9, 16}.
template <int R, bool FWD, typename T> FB_HD void dft_natural(cpx<T> (&x)[R]) {
  if constexpr (R == 3) {
    dft3<FWD, T>(x);
  } else if constexpr (R == 9) {
    dft9<FWD, T>(x);
  } else {
    dft_pow2<R, FWD, T>(x);
    cpx<T> y[R];
    static_for<0, R>([&](auto K) FB_LAMBDA { constexpr int k = decltype(K)::value; y[k] = x[rev<R>(k)]; });
    static_for<0, R>([&](auto K) FB_LAMBDA { constexpr int k = decltype(K)::value; x[k] = y[k]; });
  }
}

// Where a stage reads from / writes to.
enum : int {
  kInGlobal = 0,       // the user's input
  kInShared = 1,       // the other ping-pong buffer
  kInGlobalChirp = 2,  // CHIRP: x[e] * chirp[e] for e < n, 0 up to len
  kInSharedW = 3,      // CHIRP: buffer[e] * W[e]
};
enum : int {
  kOutShared = 0,
  kOutGlobal = 1,       // the user's output (times scale)
  kOutGlobalChirp = 2,  // CHIRP: out[e] = v * chirp[e] * scale for e < n
};

template <typename T> struct Args {
  const cpx<T>* in;
  cpx<T>* out;
  const cpx<T>* wtab;    // per-stage twiddle blocks (Stages::tw_off, twiddle_entries), forward
  const cpx<T>* chirp;   // CHIRP: forward chirp, n entries
  const cpx<T>* wf;      // CHIRP: W = FFT_len(wrapped conjugate chirp), len entries, forward direction
  long batch;
  int n;                 // user transform length
  int len;               // length of the transforms computed on chip (n, or the Bluestein inner size M)
  int group;             // transforms per CTA iteration
  int pad;               // buffers use the padded layout (needed iff the first radix is even)
  T scale;
  Stages st;
};

// One stage of the group's transforms for thread `tid` of `nthreads`: FWD = direction of this FFT's twiddles,
// DIR = direction of the user's transform (chirp / W conjugation in CHIRP mode).  `tw` = the stage's twiddle block.
// Index arithmetic (the first version of this kernel issued more integer than floating-point instructions): with per = len / R the R inputs of butterfly q sit at q + k*per and its outputs
// at w0 + k*stride, w0 = i*R*stride + j -- both linear in k; the pad term e >> 5 is linear too whenever per
// (stride) is a multiple of 32, and absent when the buffers are not padded at all (PAD = false: first radix odd,
// whose stride-1 writes are conflict-free as they are).  The source / destination kind is tested once per
// butterfly, outside the unrolled element loops.
template <typename T, int R, bool FWD, bool DIR, bool PAD>
FB_HD void run_stage(const Args<T>& a, int tid, int nthreads, long first, int cnt, int sub, int stride, unsigned magic,
                     const cpx<T>* tw, int in_mode, int out_mode, const cpx<T>* sin, cpx<T>* sout) {
  using V = cpx<T>;
  const int per = a.len / R, m = sub / R;
  const bool lin_r = !PAD || (per & 31) == 0, lin_w = !PAD || (stride & 31) == 0;
  const int dr = PAD ? per + (per >> 5) : per, dw = PAD ? stride + (stride >> 5) : stride;
  // butterflies of the whole group, transform-major: g = tl * per + q (tl and q advance without a division)
  int tl = tid / per, q = tid - tl * per;
  const int dtl = nthreads / per, dq = nthreads - dtl * per;
  for (; tl < cnt; ) {
    const int i = stride == 1 ? q : (int)(((unsigned long long)(unsigned)q * magic) >> 32);
    const int j = q - i * stride;
    const long b = first + tl;
    V x[R];
    if (in_mode == kInShared || in_mode == kInSharedW) {
      const int base = tl * a.len + q;
      if (lin_r) {
        const V* p = sin + (PAD ? padded(base) : base);
        static_for<0, R>([&](auto K) FB_LAMBDA { constexpr int k = decltype(K)::value; x[k] = p[k * dr]; });
      } else {
        static_for<0, R>([&](auto K) FB_LAMBDA { constexpr int k = decltype(K)::value; x[k] = sin[padded(base + k * per)]; });
      }
      if (in_mode == kInSharedW) {
        const V* w = a.wf + q;
        static_for<0, R>([&](auto K) FB_LAMBDA { constexpr int k = decltype(K)::value; x[k] = ctw<DIR>(x[k], w[k * per]); });
      }
    } else {
      const V* p = a.in + b * a.n + q;
      if (in_mode == kInGlobal) {
        static_for<0, R>([&](auto K) FB_LAMBDA { constexpr int k = decltype(K)::value; x[k] = p[k * per]; });
      } else {
        const V* c = a.chirp + q;
        static_for<0, R>([&](auto K) FB_LAMBDA {
          constexpr int k = decltype(K)::value;
          x[k] = q + k * per < a.n ? ctw<DIR>(p[k * per], c[k * per]) : mk<T>((T)0, (T)0);
        });
      }
    }
    dft_natural<R, FWD, T>(x);
    if (sub != R) {
      const V* t = tw + i;
      static_for<1, R>([&](auto K) FB_LAMBDA {
        constexpr int k = decltype(K)::value;
        x[k] = ctw<FWD>(x[k], t[(k - 1) * m]);      // w_S^{i*k}
      });
    }
    const int w0 = i * R * stride + j;
    if (out_mode == kOutShared) {
      const int base = tl * a.len + w0;
      if (lin_w) {
        V* p = sout + (PAD ? padded(base) : base);
        static_for<0, R>([&](auto K) FB_LAMBDA { constexpr int k = decltype(K)::value; p[k * dw] = x[k]; });
      } else {
        static_for<0, R>([&](auto K) FB_LAMBDA { constexpr int k = decltype(K)::value; sout[padded(base + k * stride)] = x[k]; });
      }
    } else {
      V* p = a.out + b * a.n + w0;
      if (out_mode == kOutGlobal) {
        static_for<0, R>([&](auto K) FB_LAMBDA { constexpr int k = decltype(K)::value; p[k * stride] = cscale(x[k], a.scale); });
      } else {
        const V* c = a.chirp + w0;
        static_for<0, R>([&](auto K) FB_LAMBDA {
          constexpr int k = decltype(K)::value;
          if (w0 + k * stride < a.n) p[k * stride] = cscale(ctw<DIR>(x[k], c[k * stride]), a.scale);
        });
      }
    }
    tl += dtl; q += dq;
    if (q >= per) { q -= per; ++tl; }
  }
}

template <typename T, bool FWD, bool DIR>
FB_HD void dispatch_stage(int radix, const Args<T>& a, int tid, int nthreads, long first, int cnt, int sub, int stride,
                          unsigned magic, const cpx<T>* tw, int in_mode, int out_mode, const cpx<T>* sin, cpx<T>* sout) {
#define FB_CTA_STAGE(R)                                                                                              \
  do {                                                                                                             \
    if (a.pad) run_stage<T, R, FWD, DIR, true>(a, tid, nthreads, first, cnt, sub, stride, magic, tw, in_mode, out_mode, sin, sout);  \
    else run_stage<T, R, FWD, DIR, false>(a, tid, nthreads, first, cnt, sub, stride, magic, tw, in_mode, out_mode, sin, sout);       \
  } while (0)
  switch (radix) {
    case 2: FB_CTA_STAGE(2); break;
    case 3: FB_CTA_STAGE(3); break;
    case 4: FB_CTA_STAGE(4); break;
    case 8: FB_CTA_STAGE(8); break;
    case 9: FB_CTA_STAGE(9); break;
    default: FB_CTA_STAGE(16); break;
  }
#undef FB_CTA_STAGE
}

// The stage program of one group, as (transform number, stage) steps separated by CTA barriers.  Plain mode: one
// FFT in direction DIR.  CHIRP mode: FFT_len forward, then FFT_len inverse.  Step s of `steps()`; the caller puts
// a barrier between consecutive steps (tools/emulate.cu: a loop over the threads).
template <typename T, bool DIR, bool CHIRP> struct Program {
  static FB_HD int steps(const Args<T>& a) { return CHIRP ? 2 * a.st.count : a.st.count; }
  static FB_HD void step(const Args<T>& a, int s, int tid, int nthreads, long first, int cnt, cpx<T>* buf0, cpx<T>* buf1) {
    const int nst = a.st.count;
    const int k = s < nst ? s : s - nst;          // stage within its transform
    int sub = a.len, stride = 1;
    for (int q = 0; q < k; ++q) { sub /= a.st.radix[q]; stride *= a.st.radix[q]; }
    const bool first_stage = k == 0, last_stage = k == nst - 1;
    const unsigned magic = a.st.magic[k];
    const cpx<T>* tw = a.wtab + a.st.tw_off[k];
    const cpx<T>* sin = (s & 1) ? buf0 : buf1;    // step s writes buf[s & 1]
    cpx<T>* sout = (s & 1) ? buf1 : buf0;
    if constexpr (!CHIRP) {
      dispatch_stage<T, DIR, DIR>(a.st.radix[k], a, tid, nthreads, first, cnt, sub, stride, magic, tw,
                                  first_stage ? kInGlobal : kInShared, last_stage ? kOutGlobal : kOutShared, sin, sout);
    } else if (s < nst) {
      dispatch_stage<T, true, DIR>(a.st.radix[k], a, tid, nthreads, first, cnt, sub, stride, magic, tw,
                                   first_stage ? kInGlobalChirp : kInShared, kOutShared, sin, sout);
    } else {
      dispatch_stage<T, false, DIR>(a.st.radix[k], a, tid, nthreads, first, cnt, sub, stride, magic, tw,
                                    first_stage ? kInSharedW : kInShared, last_stage ? kOutGlobalChirp : kOutShared,
                                    sin, sout);
    }
  }
};

template <typename T, bool DIR, bool CHIRP>
__global__ void __launch_bounds__(kThreads)
cta_fft_kernel(const Args<T> a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  cpx<T>* buf0 = reinterpret_cast<cpx<T>*>(smem_raw);
  cpx<T>* buf1 = buf0 + buffer_elems(a.group, a.len);
  using P = Program<T, DIR, CHIRP>;
  const int steps = P::steps(a);
  for (long first = (long)blockIdx.x * a.group; first < a.batch; first += (long)gridDim.x * a.group) {
    const int cnt = (int)(a.batch - first < a.group ? a.batch - first : a.group);
    for (int s = 0; s < steps; ++s) {
      P::step(a, s, threadIdx.x, kThreads, first, cnt, buf0, buf1);
      __syncthreads();
    }
  }
}

}  // namespace cta
}  // namespace fb200
