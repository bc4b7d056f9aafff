// In-register DFT butterflies of the longitude FFT (fft.cu), generic over the complex value type:
//   float2  one complex number (host emulation, runtime-plan kernels)
//   cpair   the same complex element of TWO latitude rows, real parts in one register pair and imaginary parts in another; every
//           add / mul / fma acts on both rows (two scalar instructions on sm_90a, which has no packed fp32 arithmetic).
// Everything is written with explicit fused multiply-adds and "+ (-i) b" forms so that no negation or multiplication by 0 / 1
// is ever materialised in either instantiation.
#pragma once
#include <cuda_runtime.h>
#include "fft_roots.cuh"

#ifndef HD
#define HD __host__ __device__ __forceinline__
#endif

namespace b200sht {

// ---- real scalar of two rows
struct pr { float2 v; };
struct __align__(16) cpair { pr x, y; };   // (re row A, re row B), (im row A, im row B)

HD pr make_pr(float a, float b) { pr r; r.v = make_float2(a, b); return r; }
HD pr operator+(pr a, pr b) { return make_pr(a.v.x + b.v.x, a.v.y + b.v.y); }
HD pr operator-(pr a, pr b) { return make_pr(a.v.x - b.v.x, a.v.y - b.v.y); }
HD pr operator*(pr a, pr b) { return make_pr(a.v.x * b.v.x, a.v.y * b.v.y); }
// a * s and a * s + c with a scalar factor shared by both rows
HD pr rmul(pr a, float s) { return make_pr(a.v.x * s, a.v.y * s); }
HD pr rfma(pr a, float s, pr c) { return make_pr(a.v.x * s + c.v.x, a.v.y * s + c.v.y); }
HD pr rfma(pr a, pr s, pr c) { return make_pr(a.v.x * s.v.x + c.v.x, a.v.y * s.v.y + c.v.y); }
HD float rmul(float a, float s) { return a * s; }
HD float rfma(float a, float s, float c) { return a * s + c; }

template <class C, class Re> HD C mk(Re x, Re y) { C r; r.x = x; r.y = y; return r; }

// ---- complex helpers (C = float2 or cpair)
template <class C> HD C cadd(C a, C b) { return mk<C>(a.x + b.x, a.y + b.y); }
template <class C> HD C csub(C a, C b) { return mk<C>(a.x - b.x, a.y - b.y); }
template <class C> HD C cadd_mi(C a, C b) { return mk<C>(a.x + b.y, a.y - b.x); }   // a + (-i) b
template <class C> HD C csub_mi(C a, C b) { return mk<C>(a.x - b.y, a.y + b.x); }   // a - (-i) b
template <class C> HD C cscale(C a, float s) { return mk<C>(rmul(a.x, s), rmul(a.y, s)); }
template <class C> HD C caxpy(C a, float s, C c) { return mk<C>(rfma(a.x, s, c.x), rfma(a.y, s, c.y)); }   // a * s + c
// a * w for a twiddle shared by both rows
template <class C> HD C cmulw(C a, float2 w) { return mk<C>(rfma(a.y, -w.y, rmul(a.x, w.x)), rfma(a.y, w.x, rmul(a.x, w.y))); }

HD float2 cmul(float2 a, float2 b) { return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }

template <int R>
struct Butterfly;

template <>
struct Butterfly<2> {
  template <class C> HD static void run(C* v, const float2*, int) {
    const C a = v[0], b = v[1];
    v[0] = cadd(a, b);
    v[1] = csub(a, b);
  }
};

template <class C> HD void dft4(C& a0, C& a1, C& a2, C& a3) {
  const C t0 = cadd(a0, a2), t1 = csub(a0, a2), t2 = cadd(a1, a3), d = csub(a1, a3);
  a0 = cadd(t0, t2);
  a2 = csub(t0, t2);
  a1 = cadd_mi(t1, d);
  a3 = csub_mi(t1, d);
}

template <>
struct Butterfly<4> {
  template <class C> HD static void run(C* v, const float2*, int) { dft4(v[0], v[1], v[2], v[3]); }
};

template <>
struct Butterfly<8> {
  template <class C> HD static void run(C* v, const float2*, int) {
    const float h = 0.70710678118654752440f;
    C b0 = cadd(v[0], v[4]), b4 = csub(v[0], v[4]);
    C b1 = cadd(v[1], v[5]), d5 = csub(v[1], v[5]);
    C b2 = cadd(v[2], v[6]), d6 = csub(v[2], v[6]);
    C b3 = cadd(v[3], v[7]), d7 = csub(v[3], v[7]);
    dft4(b0, b1, b2, b3);  // even outputs X[0], X[2], X[4], X[6]
    // odd outputs: DFT4 of (b4, W8 d5, -i d6, W8^3 d7), W8 = (1 - i)/sqrt2, W8^3 = (-1 - i)/sqrt2
    const C b5 = mk<C>(rmul(d5.x + d5.y, h), rmul(d5.y - d5.x, h));
    const C b7 = mk<C>(rmul(d7.y - d7.x, h), rmul(d7.x + d7.y, -h));
    const C t0 = cadd_mi(b4, d6), t1 = csub_mi(b4, d6), t2 = cadd(b5, b7), d = csub(b5, b7);
    v[0] = b0; v[2] = b1; v[4] = b2; v[6] = b3;
    v[1] = cadd(t0, t2);
    v[5] = csub(t0, t2);
    v[3] = cadd_mi(t1, d);
    v[7] = csub_mi(t1, d);
  }
};

template <>
struct Butterfly<3> {
  template <class C> HD static void run(C* v, const float2*, int) {
    const float s = 0.86602540378443864676f;
    const C t = cadd(v[1], v[2]), u = cscale(csub(v[1], v[2]), s);
    const C m = caxpy(t, -0.5f, v[0]);
    v[0] = cadd(v[0], t);
    v[1] = cadd_mi(m, u);
    v[2] = csub_mi(m, u);
  }
};

template <>
struct Butterfly<5> {
  template <class C> HD static void run(C* v, const float2*, int) {
    const float c1 = 0.30901699437494742410f, c2 = -0.80901699437494742410f;
    const float s1 = 0.95105651629515357212f, s2 = 0.58778525229247312917f;
    const C t1 = cadd(v[1], v[4]), t2 = cadd(v[2], v[3]), t3 = csub(v[1], v[4]), t4 = csub(v[2], v[3]);
    const C m1 = caxpy(t2, c2, caxpy(t1, c1, v[0]));
    const C m2 = caxpy(t2, c1, caxpy(t1, c2, v[0]));
    const C n1 = caxpy(t4, s2, cscale(t3, s1));
    const C n2 = caxpy(t4, -s1, cscale(t3, s2));
    v[0] = cadd(v[0], cadd(t1, t2));
    v[1] = cadd_mi(m1, n1);
    v[4] = csub_mi(m1, n1);
    v[2] = cadd_mi(m2, n2);
    v[3] = csub_mi(m2, n2);
  }
};

// generic O(R^2) butterfly for the rare odd primes (twiddles from the length-N table; R | N)
template <int R>
struct Butterfly {
  template <class C> HD static void run(C* v, const float2* tw, int N) {
    C o[R];
    const int step = N / R;
#pragma unroll
    for (int q = 0; q < R; ++q) {
      C acc = v[0];
#pragma unroll
      for (int r = 1; r < R; ++r) acc = cadd(acc, cmulw(v[r], tw[((r * q) % R) * step]));
      o[q] = acc;
    }
#pragma unroll
    for (int q = 0; q < R; ++q) v[q] = o[q];
  }
};

// multiplication by the constant unit root exp(-2 pi i t / R); quarter turns cost no multiplication
template <int R, class C> HD C cmul_root(C a, int t) {
  if ((4 * t) % R == 0) {
    const int qt = (4 * t) / R % 4;
    if (qt == 0) return a;
    if (qt == 1) return mk<C>(a.y, rmul(a.x, -1.f));                  // * (-i)
    if (qt == 2) return mk<C>(rmul(a.x, -1.f), rmul(a.y, -1.f));
    return mk<C>(rmul(a.y, -1.f), a.x);                               // * (+i)
  }
  return cmulw(a, unit_root<R>(t));
}

// Cooley-Tukey composite in registers: R = R1 * R2, input index n = R2 n1 + n2, output index k = k1 + R1 k2.
template <int R1, int R2>
struct Composite {
  template <class C> HD static void run(C* v) {
    constexpr int R = R1 * R2;
    C t[R];
#pragma unroll
    for (int n2 = 0; n2 < R2; ++n2) {
      C u[R1];
#pragma unroll
      for (int n1 = 0; n1 < R1; ++n1) u[n1] = v[R2 * n1 + n2];
      Butterfly<R1>::run(u, nullptr, 0);
#pragma unroll
      for (int k1 = 0; k1 < R1; ++k1) t[n2 * R1 + k1] = cmul_root<R>(u[k1], n2 * k1);
    }
#pragma unroll
    for (int k1 = 0; k1 < R1; ++k1) {
      C u[R2];
#pragma unroll
      for (int n2 = 0; n2 < R2; ++n2) u[n2] = t[n2 * R1 + k1];
      Butterfly<R2>::run(u, nullptr, 0);
#pragma unroll
      for (int k2 = 0; k2 < R2; ++k2) v[k1 + R1 * k2] = u[k2];
    }
  }
};
template <> struct Butterfly<6> { template <class C> HD static void run(C* v, const float2*, int) { Composite<2, 3>::run(v); } };
template <> struct Butterfly<9> { template <class C> HD static void run(C* v, const float2*, int) { Composite<3, 3>::run(v); } };
template <> struct Butterfly<10> { template <class C> HD static void run(C* v, const float2*, int) { Composite<2, 5>::run(v); } };
template <> struct Butterfly<12> { template <class C> HD static void run(C* v, const float2*, int) { Composite<4, 3>::run(v); } };
template <> struct Butterfly<15> { template <class C> HD static void run(C* v, const float2*, int) { Composite<3, 5>::run(v); } };
template <> struct Butterfly<16> { template <class C> HD static void run(C* v, const float2*, int) { Composite<4, 4>::run(v); } };

}  // namespace b200sht
