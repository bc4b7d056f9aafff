// Radix-8 stage of the tensor-core longitude DFT (dft.cu), written once for three value types:
//   float   host emulation (b200sht_debug_dft_host) and scalar device code
//   pr      the same quantity of TWO latitude rows in one 64-bit register pair: every operation acts on both rows
//
// Factorisation of the length-N real transform, N = 8 * N2 (reference semantics: torch.fft.rfft / irfft(norm="forward") as called
// by torch_harmonics.RealSHT / InverseRealSHT; call sites makani/models/common/spectral_convolution.py:239,253):
//   longitude j = N2 * j1 + j2  (j1 < 8, j2 < N2),   order m = c + 8 * m2  (class c < 8, m2 < M2 = ceil(mmax / 8))
//   exp(2 pi i m j / N) = exp(2 pi i c j1 / 8) * exp(2 pi i c j2 / N) * exp(2 pi i m2 j2 / N2)
//                         radix-8 butterfly      twiddle tw(c, j2)      class-independent matrix E[m2][j2]  -> tensor cores
// synthesis:  V[c][j2] = sum_m2 Z[c + 8 m2] E[m2][j2]   (GEMM),  U = tw * V,  x[N2 j1 + j2] = Re sum_c U[c] exp(2 pi i c j1 / 8)
// analysis :  Y[c][j2] = sum_j1 x[N2 j1 + j2] exp(-2 pi i c j1 / 8),  Y' = conj(tw) * Y,  X[c + 8 m2] = sum_j2 conj(E[m2][j2]) Y'[c][j2]  (GEMM)
// Both GEMMs use E[m2][N2 - j2] = conj(E[m2][j2]): only j2 <= N2 / 2 enters the GEMM, each lane / thread carries j2 and its
// partner N2 - j2 (cosine and sine sums S1..S4, resp. the even / odd combinations Ye, Yo).
#pragma once
#include "fft_butterfly.cuh"

namespace b200sht {

constexpr float kSqrtHalf = 0.70710678118654752440f;

HD float re_zero(float) { return 0.f; }
HD pr re_zero(pr) { return make_pr(0.f, 0.f); }
HD float rneg(float a) { return -a; }
HD pr rneg(pr a) { return rmul(a, -1.f); }
HD float radd(float a, float b) { return a + b; }
HD float rsub(float a, float b) { return a - b; }
HD pr radd(pr a, pr b) { return a + b; }
HD pr rsub(pr a, pr b) { return a - b; }

// twiddles of the partner column j2' = N2 - j2:  tw(c, j2') = exp(i pi c / 4) * conj(tw(c, j2))
HD void dft_partner_twiddles(const float2* tw /*[8], tw[0] unused*/, float2* tp /*[8]*/) {
  const float h = kSqrtHalf;
  tp[0] = make_float2(1.f, 0.f);
  tp[1] = make_float2(h * (tw[1].x + tw[1].y), h * (tw[1].x - tw[1].y));
  tp[2] = make_float2(tw[2].y, tw[2].x);
  tp[3] = make_float2(h * (tw[3].y - tw[3].x), h * (tw[3].x + tw[3].y));
  tp[4] = make_float2(-tw[4].x, tw[4].y);
  tp[5] = make_float2(-h * (tw[5].x + tw[5].y), h * (tw[5].y - tw[5].x));
  tp[6] = make_float2(-tw[6].y, -tw[6].x);
  tp[7] = make_float2(h * (tw[7].x - tw[7].y), -h * (tw[7].x + tw[7].y));
}

// ---------------------------------------------------------------------------------------------- synthesis
// vr / vi: V[c] of one column j (8 classes);  tw[c] = exp(2 pi i c j / N) (tw[0] ignored);  x[j1] = Re sum_c tw[c] V[c] exp(2 pi i c j1 / 8)
template <class Re>
HD void dft_syn_radix8(const Re* vr, const Re* vi, const float2* tw, Re* x) {
  // U = tw * V: real parts of all classes, imaginary parts of c = 1,2,3,5,6,7
  Re ur[8], ui[8];
  ur[0] = vr[0];
#pragma unroll
  for (int c = 1; c < 8; ++c) {
    ur[c] = rfma(vi[c], -tw[c].y, rmul(vr[c], tw[c].x));
    if (c != 4) ui[c] = rfma(vi[c], tw[c].x, rmul(vr[c], tw[c].y));
  }
  const Re p1 = radd(ur[1], ur[7]), p2 = radd(ur[2], ur[6]), p3 = radd(ur[3], ur[5]);
  const Re q1 = rsub(ui[1], ui[7]), q2 = rsub(ui[2], ui[6]), q3 = rsub(ui[3], ui[5]);
  const Re a = radd(ur[0], ur[4]), b = rsub(ur[0], ur[4]);
  const Re sP = radd(p1, p3), dP = rsub(p1, p3), sQ = radd(q1, q3), dQ = rsub(q1, q3);
  const Re e0 = radd(a, p2), e1 = rsub(a, p2), o0 = rsub(b, q2), o1 = radd(b, q2);
  const Re t1 = rsub(dP, sQ), t3 = radd(dP, sQ);
  x[0] = radd(e0, sP);
  x[4] = rsub(e0, sP);
  x[2] = rsub(e1, dQ);
  x[6] = radd(e1, dQ);
  x[1] = rfma(t1, kSqrtHalf, o0);
  x[5] = rfma(t1, -kSqrtHalf, o0);
  x[3] = rfma(t3, -kSqrtHalf, o1);
  x[7] = rfma(t3, kSqrtHalf, o1);
}

// ----------------------------------------------------------------------------------------------- analysis
// x[j1] = eight real samples of one column j;  tw[c] = exp(+2 pi i c j / N);  out: Y'[c] = conj(tw[c]) sum_j1 x[j1] exp(-2 pi i c j1 / 8)
template <class Re>
HD void dft_ana_radix8(const Re* x, const float2* tw, Re* yr, Re* yi) {
  const Re a0 = radd(x[0], x[4]), a1 = rsub(x[0], x[4]), a2 = radd(x[2], x[6]), a3 = rsub(x[2], x[6]);
  const Re b0 = radd(x[1], x[5]), b1 = rsub(x[1], x[5]), b2 = radd(x[3], x[7]), b3 = rsub(x[3], x[7]);
  const Re sa = radd(a0, a2), sb = radd(b0, b2);
  const Re y0 = radd(sa, sb), y4 = rsub(sa, sb);
  const Re y2r = rsub(a0, a2), y2i = rsub(b2, b0);                 // Y2 = (a0 - a2) - i (b0 - b2)
  const Re hm = rmul(rsub(b1, b3), kSqrtHalf), hp = rmul(radd(b1, b3), kSqrtHalf);
  const Re y1r = radd(a1, hm), y1i = rneg(radd(a3, hp));           // Y1 = a1 + h (b1 - b3) - i (a3 + h (b1 + b3))
  const Re y3r = rsub(a1, hm), y3i = rsub(a3, hp);                 // Y3 = a1 - h (b1 - b3) + i (a3 - h (b1 + b3))
  // Y'[c] = Y[c] (tc - i ts): re = Yr tc + Yi ts, im = Yi tc - Yr ts;  Y[8 - c] = conj Y[c]
  yr[0] = y0;
  yi[0] = re_zero(y0);
  yr[4] = rmul(y4, tw[4].x);
  yi[4] = rmul(y4, -tw[4].y);
#define B200_TW(c, R_, I_)                          \
  yr[c] = rfma(I_, tw[c].y, rmul(R_, tw[c].x));     \
  yi[c] = rfma(R_, -tw[c].y, rmul(I_, tw[c].x));
  B200_TW(1, y1r, y1i)
  B200_TW(2, y2r, y2i)
  B200_TW(3, y3r, y3i)
  {
    const Re n3 = rneg(y3i), n2 = rneg(y2i), n1 = rneg(y1i);
    B200_TW(5, y3r, n3)
    B200_TW(6, y2r, n2)
    B200_TW(7, y1r, n1)
  }
#undef B200_TW
}

}  // namespace b200sht
