// cplx.cuh -- complex arithmetic and register-resident butterflies shared by every kernel.
//
// Replaces the reference's macro "vector ISA" (fourier-algorithms/src/vector/generic.rs:5-62,
// vector/avx.rs:6-193) and its butterfly macros (autosort/butterfly.rs:3-65).  Unlike the
// reference (mul, mul, addsub -- no FMA) the products here are left to contract into FFMA/DFMA;
// parity with the reference is tolerance-based (SURVEY.md 8c) and FMA only tightens the error.
//
// Everything is __host__ __device__ so the same code runs under the CPU emulation used by
// tests/test_kernel_emulation.py (tools/emulate.cu) -- there is no GPU in the build container.
#pragma once

#include <cuda_runtime.h>

#include <type_traits>

#include "twiddle_consts.h"

#define FB_HD __host__ __device__ __forceinline__
// The compile-time loops below run generic lambdas; if the inliner's budget runs out in a large
// translation unit a lambda becomes a real call, its by-reference capture of the register array forces
// that array into local memory (seen as a 296-byte stack frame in one kernel).  Never let that happen.
#define FB_LAMBDA __attribute__((always_inline))

namespace fb200 {

template <typename T> struct C2;
template <> struct C2<float> { using type = float2; };
template <> struct C2<double> { using type = double2; };
template <typename T> using cpx = typename C2<T>::type;

template <typename T> FB_HD cpx<T> mk(T re, T im) { cpx<T> r; r.x = re; r.y = im; return r; }

// complex<float> arithmetic is scalar FP32: Hopper has no packed two-lane FADD2 / FFMA2, and the products below
// contract into FFMA.
FB_HD float2 cadd(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
FB_HD float2 csub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
FB_HD float2 cmul(float2 a, float2 b) { return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }
FB_HD float2 cmulc(float2 a, float2 b) { return make_float2(a.x * b.x + a.y * b.y, a.y * b.x - a.x * b.y); }
FB_HD float2 cscale(float2 a, float s) { return make_float2(a.x * s, a.y * s); }

FB_HD double2 cadd(double2 a, double2 b) { return make_double2(a.x + b.x, a.y + b.y); }
FB_HD double2 csub(double2 a, double2 b) { return make_double2(a.x - b.x, a.y - b.y); }
FB_HD double2 cmul(double2 a, double2 b) { return make_double2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }
FB_HD double2 cmulc(double2 a, double2 b) { return make_double2(a.x * b.x + a.y * b.y, a.y * b.x - a.x * b.y); }
FB_HD double2 cscale(double2 a, double s) { return make_double2(a.x * s, a.y * s); }

template <typename V> FB_HD V cconj(V a) { V r; r.x = a.x; r.y = -a.y; return r; }
// multiply by -i (forward quarter turn) / +i
template <typename V> FB_HD V cmul_mi(V a) { V r; r.x = a.y; r.y = -a.x; return r; }
template <typename V> FB_HD V cmul_pi(V a) { V r; r.x = -a.y; r.y = a.x; return r; }
// a * w where w is a forward-table twiddle; inverse transforms use the conjugate
template <bool FWD, typename V> FB_HD V ctw(V a, V w) { return FWD ? cmul(a, w) : cmulc(a, w); }

template <int I, int N, typename F> FB_HD void static_for(F&& f) {
  if constexpr (I < N) {
    f(std::integral_constant<int, I>{});
    static_for<I + 1, N>(f);
  }
}

__host__ __device__ constexpr int ilog2(int n) { return n <= 1 ? 0 : 1 + ilog2(n / 2); }
__host__ __device__ constexpr int bitrev(int k, int bits) {
  int r = 0;
  for (int b = 0; b < bits; ++b) r |= ((k >> b) & 1) << (bits - 1 - b);
  return r;
}

// a * w_N^K with w_N = exp(-2*pi*i/N) (FWD) or its conjugate; N | 64, K compile-time.
template <int N, int K, bool FWD, typename T> FB_HD cpx<T> mul_w(cpx<T> a) {
  static_assert(64 % N == 0, "compile-time twiddles cover N | 64");
  constexpr int k = ((K % N) + N) % N;
  if constexpr (k == 0) {
    return a;
  } else if constexpr (4 * k == N) {
    return FWD ? cmul_mi(a) : cmul_pi(a);
  } else if constexpr (2 * k == N) {
    return mk<T>(-a.x, -a.y);
  } else if constexpr (4 * k == 3 * N) {
    return FWD ? cmul_pi(a) : cmul_mi(a);
  } else {
    constexpr T c = (T)kCos64[k * (64 / N)];
    constexpr T s = (T)kSin64[k * (64 / N)];  // forward w = (c, -s)
    constexpr T wy = FWD ? -s : s;
    return cmul(a, mk<T>(c, wy));             // constants: both operand pairs fold at compile time
  }
}

// In-register radix-2 decimation-in-frequency FFT of x[BASE .. BASE+LEN).  Result is bit-reversed:
// X[k] ends up in x[BASE + bitrev(k, log2 LEN)].
template <int LEN, int BASE, bool FWD, typename T, int TOTAL>
FB_HD void dif2(cpx<T> (&x)[TOTAL]) {
  if constexpr (LEN >= 2) {
    constexpr int H = LEN / 2;
    static_for<0, H>([&](auto J) FB_LAMBDA {
      constexpr int j = decltype(J)::value;
      cpx<T> a = x[BASE + j], b = x[BASE + j + H];
      x[BASE + j] = cadd(a, b);
      x[BASE + j + H] = mul_w<LEN, j, FWD, T>(csub(a, b));
    });
    dif2<H, BASE, FWD, T, TOTAL>(x);
    dif2<H, BASE + H, FWD, T, TOTAL>(x);
  }
}

// DFT of R register values (R in {2,4,8,16,32,64}); X[k] is at x[rev<R>(k)] afterwards.
template <int R, bool FWD, typename T> FB_HD void dft_pow2(cpx<T> (&x)[R]) { dif2<R, 0, FWD, T, R>(x); }
template <int R> __host__ __device__ constexpr int rev(int k) { return bitrev(k, ilog2(R)); }

// Radix-3 butterfly, natural order in and out (reference: autosort/butterfly.rs:9-22).
template <bool FWD, typename T> FB_HD void dft3(cpx<T> (&x)[3]) {
  constexpr T h = (T)0.86602540378443864676372317075294;  // sqrt(3)/2
  cpx<T> s = cadd(x[1], x[2]);
  cpx<T> d = cscale(csub(x[1], x[2]), h);
  cpx<T> t = mk<T>(x[0].x - (T)0.5 * s.x, x[0].y - (T)0.5 * s.y);
  cpx<T> r = FWD ? cmul_mi(d) : cmul_pi(d);
  x[0] = cadd(x[0], s);
  x[1] = cadd(t, r);
  x[2] = csub(t, r);
}

// Radix-9 butterfly, natural order in and out: 3 x 3 Cooley-Tukey on radix-3 butterflies.
template <bool FWD, typename T> FB_HD void dft9(cpx<T> (&x)[9]) {
  // n = 3*n1 + n2, k = k1 + 3*k2;  w_9^1, w_9^2, w_9^4 (forward = exp(-2 pi i k / 9))
  constexpr T c1 = (T)0.76604444311897803520239265055542, s1 = (T)0.64278760968653932632264340990726;
  constexpr T c2 = (T)0.17364817766693034885171662676931, s2 = (T)0.98480775301220805936674302458952;
  constexpr T c4 = (T)-0.93969262078590838405410927732473, s4 = (T)0.34202014332566873304409961468226;
  cpx<T> a[3][3];
#pragma unroll
  for (int n2 = 0; n2 < 3; ++n2) {
    cpx<T> t[3] = {x[n2], x[3 + n2], x[6 + n2]};
    dft3<FWD, T>(t);
    a[n2][0] = t[0]; a[n2][1] = t[1]; a[n2][2] = t[2];
  }
  const T sg = FWD ? (T)-1 : (T)1;
  a[1][1] = cmul(a[1][1], mk<T>(c1, sg * s1));
  a[1][2] = cmul(a[1][2], mk<T>(c2, sg * s2));
  a[2][1] = cmul(a[2][1], mk<T>(c2, sg * s2));
  a[2][2] = cmul(a[2][2], mk<T>(c4, sg * s4));
#pragma unroll
  for (int k1 = 0; k1 < 3; ++k1) {
    cpx<T> t[3] = {a[0][k1], a[1][k1], a[2][k1]};
    dft3<FWD, T>(t);
    x[k1] = t[0]; x[k1 + 3] = t[1]; x[k1 + 6] = t[2];
  }
}

// Radix-27 butterfly, natural order in and out: 3 x 9 Cooley-Tukey (n = 9*n1 + n2, k = k1 + 3*k2) on the radix-3 and
// radix-9 butterflies; twiddles w_27^{n2*k1}, n2 < 9, k1 < 3.  Outer pass of the {2,3}-smooth path (smooth3.cu).
template <bool FWD, typename T> FB_HD void dft27(cpx<T> (&x)[27]) {
  constexpr double c27[17] = {1.0, 0.97304487057982383883288517278469592, 0.89363264032341224819257418686665512,
      0.76604444311897803520239265055541667, 0.59715859170278616485185216058395977, 0.39607976603915682369604339160974457,
      0.1736481776669303488517166267693148, -0.058144828910475828538748016847071524, -0.28680323271109025310328017316715794,
      -0.5, -0.68624163786873358572960499961753798, -0.83548781141293641965382617001958359,
      -0.93969262078590838405410927732473147, -0.99323835774194298854789555219370434, -0.99323835774194298854789555219370434,
      -0.93969262078590838405410927732473147, -0.83548781141293641965382617001958359};
  constexpr double s27[17] = {0.0, 0.2306158707424401784501983492929391, 0.44879918020046217278504033473314362,
      0.64278760968653932632264340990726343, 0.80212319275504378508329489193392513, 0.9182161068802740147589614153146366,
      0.98480775301220805936674302458952301, 0.99830815827126820804782070878327753, 0.95798951231548887443737476695675462,
      0.86602540378443864676372317075293618, 0.72737364157304869598717641766381552, 0.54950897807080603526278037405013392,
      0.34202014332566873304409961468225958, 0.11609291412523022967566652338071147, -0.11609291412523022967566652338071147,
      -0.34202014332566873304409961468225958, -0.54950897807080603526278037405013392};
  cpx<T> a[3][9];   // a[k1][n2]
  static_for<0, 9>([&](auto N2) FB_LAMBDA {
    constexpr int n2 = decltype(N2)::value;
    cpx<T> t[3] = {x[n2], x[9 + n2], x[18 + n2]};
    dft3<FWD, T>(t);
    a[0][n2] = t[0];
    if constexpr (n2 == 0) {
      a[1][n2] = t[1]; a[2][n2] = t[2];
    } else {
      a[1][n2] = cmul(t[1], mk<T>((T)c27[n2], (T)(FWD ? -s27[n2] : s27[n2])));
      a[2][n2] = cmul(t[2], mk<T>((T)c27[2 * n2], (T)(FWD ? -s27[2 * n2] : s27[2 * n2])));
    }
  });
  static_for<0, 3>([&](auto K1) FB_LAMBDA {
    constexpr int k1 = decltype(K1)::value;
    dft9<FWD, T>(a[k1]);
    static_for<0, 9>([&](auto K2) FB_LAMBDA { x[k1 + 3 * decltype(K2)::value] = a[k1][decltype(K2)::value]; });
  });
}

// Scale mode of a Transform code (fourier-algorithms/src/fft.rs:5-16, autosort/mod.rs:381-385).
enum : int { kFft = 0, kIfft = 1, kUnscaledIfft = 2, kSqrtScaledFft = 3, kSqrtScaledIfft = 4 };
inline bool transform_is_forward(int code) { return code == kFft || code == kSqrtScaledFft; }

}  // namespace fb200
