// Associated-Legendre stage of the SHT: table precompute, fp32 CUDA-core contractions (strict mode) and the
// packed <-> torch layout converters.
//
// Replaces, in torch-harmonics (third-party, pinned 887006c6..., not vendored in /root/reference):
//   legendre precompute (`_precompute_legpoly`)  -> build_table_kernel   (SURVEY.md Appendix A recurrence)
//   RealSHT.forward einsum  "...km,mlk->...lm"   -> legendre_analysis_simt_kernel
//   InverseRealSHT.forward  "...lm,mlk->...km"   -> legendre_synthesis_simt_kernel
// Reference call sites: /root/reference/makani/models/common/spectral_convolution.py:239-253.
#include "common.cuh"
#include <cmath>
#include <vector>

namespace b200sht {

// ------------------------------------------------------------------------------------------ table build
// Orthonormal associated Legendre functions for fixed order m at x = cos(theta): writes P[m][l] for l < lmax
// with stride `stride` between degrees.  fp64 recurrence, fp32 storage.
HD void legendre_column(int m, int lmax, double x, int csphase, float* out, size_t stride) {
  const double sgn = (csphase && (m & 1)) ? -1.0 : 1.0;
  double pmm = 0.28209479177387814347;  // 1/sqrt(4 pi)
  const double s2 = (1.0 + x) * (1.0 - x);
  for (int l = 1; l <= m; ++l) pmm *= sqrt((2.0 * l + 1.0) * s2 / (2.0 * l));
  for (int l = 0; l < m && l < lmax; ++l) out[(size_t)l * stride] = 0.f;
  if (m >= lmax) return;
  out[(size_t)m * stride] = (float)(sgn * pmm);
  if (m + 1 >= lmax) return;
  double p2 = pmm;                                   // P[m][l-2]
  double p1 = sqrt(2.0 * (m + 1) + 1.0) * x * pmm;   // P[m][l-1]
  out[(size_t)(m + 1) * stride] = (float)(sgn * p1);
  for (int l = m + 2; l < lmax; ++l) {
    const double a = sqrt((2.0 * l - 1.0) / (double)(l - m) * (2.0 * l + 1.0) / (double)(l + m));
    const double b = sqrt((double)(l + m - 1) / (double)(l - m) * (2.0 * l + 1.0) / (2.0 * l - 3.0) *
                          (double)(l - m - 1) / (double)(l + m));
    const double p0 = x * a * p1 - b * p2;
    out[(size_t)l * stride] = (float)(sgn * p0);
    p2 = p1;
    p1 = p0;
  }
}

// Tables of the vector SHT for order m at x = cos(theta), fp64 recurrence, fp32 storage, exact zeros for l < m:
//   D[l] = dP_l^m(cos theta) / dtheta,   Q[l] = m P_l^m(cos theta) / sin(theta)   (orthonormal P, optional Condon-Shortley phase).
// Pole-safe without a division by sin(theta): for m >= 1 the recurrence runs on P / sin(theta) (seeded with sin^(m-1) theta), and
//   D_l = l cos(theta) P_l / sin(theta) - sqrt((2l+1)/(2l-1) (l-m)(l+m)) P_{l-1} / sin(theta),
// for m = 0 it runs on P_l^1 (no phase) and D_l = -sqrt(l (l+1)) P_l^1.
HD void legendre_vector_column(int m, int lmax, double x, int csphase, float* D, float* Q, size_t stride) {
  const double s = sqrt((1.0 + x) * (1.0 - x));
  const double sgn = (csphase && (m & 1)) ? -1.0 : 1.0;
  for (int l = 0; l < m && l < lmax; ++l) D[(size_t)l * stride] = Q[(size_t)l * stride] = 0.f;
  if (m >= lmax) return;
  const int mu = m == 0 ? 1 : m;   // order of the recurrence
  double cur = 0.28209479177387814347;
  for (int l = 1; l <= mu; ++l) cur *= sqrt((2.0 * l + 1.0) / (2.0 * l)) * ((m == 0 || l > 1) ? s : 1.0);
  double prev = 0.0;
  if (m == 0) D[0] = Q[0] = 0.f;
  for (int l = mu; l < lmax; ++l) {
    if (l > mu) {
      const double nxt = (l == mu + 1) ? sqrt(2.0 * mu + 3.0) * x * cur
                                       : x * sqrt((2.0 * l - 1.0) / (double)(l - mu) * (2.0 * l + 1.0) / (double)(l + mu)) * cur -
                                             sqrt((double)(l + mu - 1) / (double)(l - mu) * (2.0 * l + 1.0) / (2.0 * l - 3.0) * (double)(l - mu - 1) /
                                                  (double)(l + mu)) * prev;
      prev = cur;
      cur = nxt;
    }
    if (m == 0) {
      D[(size_t)l * stride] = (float)(-sqrt((double)l * (l + 1)) * cur);
      Q[(size_t)l * stride] = 0.f;
    } else {
      const double a = sqrt((2.0 * l + 1.0) / (2.0 * l - 1.0) * (double)(l - m) * (double)(l + m));
      D[(size_t)l * stride] = (float)(sgn * (l * x * cur - a * prev));
      Q[(size_t)l * stride] = (float)(sgn * m * cur);
    }
  }
}

__global__ void round_tf32_kernel(const float* __restrict__ src, float* __restrict__ dst, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = tf32_rn(src[i]);
}

// 3 x TF32: an fp32 operand v enters a TF32 MMA as trunc(v) (the tensor core ignores the 13 low mantissa bits); the residual
// v - trunc(v) is exact in fp32 and is fed to a second MMA, rounded to nearest TF32 here (its own truncation would add a 2^-21 bias).
__global__ void tf32_residual_kernel(const float4* __restrict__ src, float4* __restrict__ dst, size_t n4) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  const float4 v = src[i];
  float4 r;
  r.x = tf32_rn(v.x - __uint_as_float(__float_as_uint(v.x) & 0xffffe000u));
  r.y = tf32_rn(v.y - __uint_as_float(__float_as_uint(v.y) & 0xffffe000u));
  r.z = tf32_rn(v.z - __uint_as_float(__float_as_uint(v.z) & 0xffffe000u));
  r.w = tf32_rn(v.w - __uint_as_float(__float_as_uint(v.w) & 0xffffe000u));
  dst[i] = r;
}
// n floats, n % 4 == 0, both pointers 16-byte aligned
int tf32_residual(const float* src, float* dst, size_t n, cudaStream_t st) {
  const size_t n4 = n / 4;
  if (n4 == 0) return 0;
  tf32_residual_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, st>>>(reinterpret_cast<const float4*>(src), reinterpret_cast<float4*>(dst), n4);
  B200_CHECK_LAUNCH();
  return 0;
}
__global__ void table_lo_kernel(const float* __restrict__ full, const float* __restrict__ hi, float* __restrict__ lo, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) lo[i] = tf32_rn(full[i] - hi[i]);
}
int table_residual(const float* full, const float* hi, float* lo, size_t n, cudaStream_t st) {
  table_lo_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(full, hi, lo, n);
  B200_CHECK_LAUNCH();
  return 0;
}

int round_table_tf32(const float* src, float* dst, size_t n, cudaStream_t st) {
  round_tf32_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(src, dst, n);
  B200_CHECK_LAUNCH();
  return 0;
}

__global__ void build_table_kernel(float* __restrict__ table, const double* __restrict__ cost, int nlat, int kp, int lmax,
                                   int mmax, int csphase, int m0) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  const int m = blockIdx.y;
  if (k >= kp) return;
  float* out = table + (size_t)m * lmax * kp + k;
  if (k >= nlat) {
    for (int l = 0; l < lmax; ++l) out[(size_t)l * kp] = 0.f;
    return;
  }
  legendre_column(m0 + m, lmax, cost[k], csphase, out, kp);
}

// vector plan: table[m] = D rows [0, L) then Q rows [L, 2L) of the global order m0 + m   (L = lmax / 2)
__global__ void build_vector_table_kernel(float* __restrict__ table, const double* __restrict__ cost, int nlat, int kp, int L, int csphase,
                                          int m0) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  const int m = blockIdx.y;
  if (k >= kp) return;
  float* D = table + (size_t)m * 2 * L * kp + k;
  float* Q = D + (size_t)L * kp;
  if (k >= nlat) {
    for (int l = 0; l < L; ++l) D[(size_t)l * kp] = Q[(size_t)l * kp] = 0.f;
    return;
  }
  legendre_vector_column(m0 + m, L, cost[k], csphase, D, Q, kp);
}

int build_table(Plan* pl, const double* d_cost, cudaStream_t st) {
  dim3 grid(ceil_div(pl->kp, 128), pl->mmax);
  if (pl->vector)
    build_vector_table_kernel<<<grid, 128, 0, st>>>(pl->d_table, d_cost, pl->nlat, pl->kp, pl->lmax / 2, pl->csphase, pl->m0);
  else
    build_table_kernel<<<grid, 128, 0, st>>>(pl->d_table, d_cost, pl->nlat, pl->kp, pl->lmax, pl->mmax, pl->csphase, pl->m0);
  B200_CHECK_LAUNCH();
  return 0;
}

// ---------------------------------------------------------------------------- packed index helpers
// jp: flattened padded (p, b, cp) index of a packed spec row;  returns the flattened (p, b, c) latspec row or -1.
__device__ __forceinline__ int jp_to_j(int jp, int B, int C, int cp) {
  const int c = jp % cp;
  const int pb = jp / cp;
  return (c < C) ? pb * C + c : -1;
}

// --------------------------------------------------------------------------------- SIMT contractions
constexpr int TS = 64;   // tile edge
constexpr int TK = 16;   // k slab

// spec[l][m][jp] = sum_k P[m][l][k] * X[m][j][k]      grid: (jp tiles, l tiles, m)
// Only rows k < nlat are read: the latitude padding [nlat, kp) of X may hold anything, as for the tensor-core engine.
__global__ void __launch_bounds__(256) legendre_analysis_simt_kernel(const float* __restrict__ P, const float* __restrict__ X,
                                                                     float* __restrict__ spec, int L, int M, int nlat, int kp, int B,
                                                                     int C, int cp, int m0) {
  __shared__ float As[TK][TS + 4];
  __shared__ float Bs[TK][TS + 4];
  const int m = blockIdx.z;
  const int l0 = lstart(m0 + m) + blockIdx.y * TS;
  if (l0 >= L) return;
  const int JP = 2 * B * cp, J = 2 * B * C;
  const int jp0 = blockIdx.x * TS;
  const int t = threadIdx.x;
  const int lrow = t >> 2, kq = (t & 3) * 4;
  const int ty = t >> 4, tx = t & 15;

  const int la = l0 + lrow;
  const float* arow = (la < L) ? P + ((size_t)m * L + la) * kp : nullptr;
  const int jb = (jp0 + lrow < JP) ? jp_to_j(jp0 + lrow, B, C, cp) : -1;
  const float* brow = (jb >= 0) ? X + ((size_t)m * J + jb) * kp : nullptr;

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int k0 = 0; k0 < nlat; k0 += TK) {
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
    const int k = k0 + kq;
    if (k + 4 <= nlat) {  // a whole quad of latitudes in range (rows are 16-byte aligned: kp % 8 == 0)
      if (arow) a = __ldg(reinterpret_cast<const float4*>(arow + k));
      if (brow) b = __ldg(reinterpret_cast<const float4*>(brow + k));
    } else if (k < nlat) {  // the quad holding the last latitude: the rows beyond nlat stay zero
      float av[4] = {0.f, 0.f, 0.f, 0.f}, bv[4] = {0.f, 0.f, 0.f, 0.f};
      for (int q = 0; k + q < nlat; ++q) {
        if (arow) av[q] = __ldg(arow + k + q);
        if (brow) bv[q] = __ldg(brow + k + q);
      }
      a = make_float4(av[0], av[1], av[2], av[3]);
      b = make_float4(bv[0], bv[1], bv[2], bv[3]);
    }
    __syncthreads();
    As[kq + 0][lrow] = a.x; As[kq + 1][lrow] = a.y; As[kq + 2][lrow] = a.z; As[kq + 3][lrow] = a.w;
    Bs[kq + 0][lrow] = b.x; Bs[kq + 1][lrow] = b.y; Bs[kq + 2][lrow] = b.z; Bs[kq + 3][lrow] = b.w;
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < TK; ++kk) {
      const float4 av = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
      const float4 bv = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
      const float aa[4] = {av.x, av.y, av.z, av.w};
      const float bb[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(aa[i], bb[j], acc[i][j]);
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int l = l0 + ty * 4 + i;
    if (l >= L) continue;
    float* orow = spec + ((size_t)l * M + m) * JP;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int jp = jp0 + tx * 4 + j;
      if (jp < JP) orow[jp] = acc[i][j];
    }
  }
}

// Z[m][j][k] = sum_{l >= lstart(m)} P[m][l][k] * spec[l][m][jp]     grid: (jp tiles, k tiles, m)
__global__ void __launch_bounds__(256) legendre_synthesis_simt_kernel(const float* __restrict__ P, const float* __restrict__ spec,
                                                                      float* __restrict__ Z, int L, int M, int kp, int B, int C,
                                                                      int cp, int m0) {
  __shared__ float As[TK][TS + 4];  // [l][k]
  __shared__ float Bs[TK][TS + 4];  // [l][jp]
  const int m = blockIdx.z;
  const int JP = 2 * B * cp, J = 2 * B * C;
  const int k0 = blockIdx.y * TS;
  const int jp0 = blockIdx.x * TS;
  const int t = threadIdx.x;
  const int lrow = t >> 4, cq = (t & 15) * 4;  // 16 l-rows x 16 float4 columns
  const int ty = t >> 4, tx = t & 15;

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int l0 = lstart(m0 + m); l0 < L; l0 += TK) {
    const int l = l0 + lrow;
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
    if (l < L) {
      if (k0 + cq < kp) a = __ldg(reinterpret_cast<const float4*>(P + ((size_t)m * L + l) * kp + k0 + cq));
      if (jp0 + cq < JP) b = __ldg(reinterpret_cast<const float4*>(spec + ((size_t)l * M + m) * JP + jp0 + cq));  // JP % 8 == 0
    }
    __syncthreads();
    *reinterpret_cast<float4*>(&As[lrow][cq]) = a;
    *reinterpret_cast<float4*>(&Bs[lrow][cq]) = b;
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < TK; ++kk) {
      const float4 av = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
      const float4 bv = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
      const float aa[4] = {av.x, av.y, av.z, av.w};
      const float bb[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(aa[i], bb[j], acc[i][j]);
    }
  }
  // rows i -> k (contiguous in Z), cols j -> jp
  const int k = k0 + ty * 4;
  if (k >= kp) return;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int jp = jp0 + tx * 4 + j;
    if (jp >= JP) continue;
    const int jj = jp_to_j(jp, B, C, cp);
    if (jj < 0) continue;
    *reinterpret_cast<float4*>(Z + ((size_t)m * J + jj) * kp + k) = make_float4(acc[0][j], acc[1][j], acc[2][j], acc[3][j]);
  }
}

int legendre_analysis_simt(const Plan* pl, const float* X, float* spec, int B, int C, cudaStream_t st) {
  const int cp = round_up(C, 4);
  const int JP = 2 * B * cp;
  dim3 grid(ceil_div(JP, TS), ceil_div(pl->lmax, TS), pl->mmax);
  legendre_analysis_simt_kernel<<<grid, 256, 0, st>>>(pl->d_table, X, spec, pl->lmax, pl->mmax, pl->nlat, pl->kp, B, C, cp, pl->m0);
  B200_CHECK_LAUNCH();
  return 0;
}

int legendre_synthesis_simt(const Plan* pl, const float* spec, float* Z, int B, int C, cudaStream_t st) {
  const int cp = round_up(C, 4);
  const int JP = 2 * B * cp;
  dim3 grid(ceil_div(JP, TS), ceil_div(pl->kp, TS), pl->mmax);
  legendre_synthesis_simt_kernel<<<grid, 256, 0, st>>>(pl->d_table, spec, Z, pl->lmax, pl->mmax, pl->kp, B, C, cp, pl->m0);
  B200_CHECK_LAUNCH();
  return 0;
}

// -------------------------------------------------------------------------------- pack / unpack
// spec [L][M][2][B][cp]  <->  coeffs complex64 [B*C][L][M].   block: 32 m x 32 c tile of one (l, b)
__global__ void __launch_bounds__(256) spec_unpack_kernel(const float* __restrict__ spec, float2* __restrict__ coeffs, int L, int M,
                                                          int B, int C, int cp, int mo, int dense) {
  __shared__ float tile[2][32][33];
  const int l = blockIdx.z / B, b = blockIdx.z % B;
  const int m0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 8 rows of 32
  const int JP = 2 * B * cp;
  for (int mm = ty; mm < 32; mm += 8) {
    const int m = m0 + mm, c = c0 + tx;
    float re = 0.f, im = 0.f;
    if (m < M && c < C && (dense || l >= mo + m)) {  // exact zeros for l < m (global order mo + m)
      const float* row = spec + ((size_t)l * M + m) * JP;
      re = row[(0 * B + b) * cp + c];
      im = row[(1 * B + b) * cp + c];
    }
    tile[0][mm][tx] = re;
    tile[1][mm][tx] = im;
  }
  __syncthreads();
  for (int cc = ty; cc < 32; cc += 8) {
    const int c = c0 + cc, m = m0 + tx;
    if (c < C && m < M) coeffs[((size_t)(b * C + c) * L + l) * M + m] = make_float2(tile[0][tx][cc], tile[1][tx][cc]);
  }
}

__global__ void __launch_bounds__(256) spec_pack_kernel(const float2* __restrict__ coeffs, float* __restrict__ spec, int L, int M, int B,
                                                        int C, int cp, int mo, int dense) {
  __shared__ float tile[2][32][33];
  const int l = blockIdx.z / B, b = blockIdx.z % B;
  const int m0 = blockIdx.x * 32, c0 = blockIdx.y * 32;  // c0 runs over cp
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int JP = 2 * B * cp;
  for (int cc = ty; cc < 32; cc += 8) {
    const int c = c0 + cc, m = m0 + tx;
    float2 v = make_float2(0.f, 0.f);
    if (c < C && m < M) v = coeffs[((size_t)(b * C + c) * L + l) * M + m];
    tile[0][tx][cc] = v.x;
    tile[1][tx][cc] = v.y;
  }
  __syncthreads();
  for (int mm = ty; mm < 32; mm += 8) {
    const int m = m0 + mm, c = c0 + tx;
    if (m < M && c < cp && (dense || l >= lstart(mo + m))) {
      float* row = spec + ((size_t)l * M + m) * JP;
      row[(0 * B + b) * cp + c] = tile[0][mm][tx];
      row[(1 * B + b) * cp + c] = tile[1][mm][tx];
    }
  }
}

int spec_unpack(const Plan* pl, const float* spec, void* coeffs, int B, int C, cudaStream_t st) {
  const int cp = round_up(C, 4);
  dim3 grid(ceil_div(pl->mmax, 32), ceil_div(C, 32), pl->lmax * B);
  B200_REQUIRE(grid.z <= 65535, "spec_unpack: lmax*B=%u exceeds grid limit", grid.z);
  spec_unpack_kernel<<<grid, 256, 0, st>>>(spec, static_cast<float2*>(coeffs), pl->lmax, pl->mmax, B, C, cp, pl->m0, pl->dense);
  B200_CHECK_LAUNCH();
  return 0;
}

int spec_pack(const Plan* pl, const void* coeffs, float* spec, int B, int C, cudaStream_t st) {
  const int cp = round_up(C, 4);
  dim3 grid(ceil_div(pl->mmax, 32), ceil_div(cp, 32), pl->lmax * B);
  B200_REQUIRE(grid.z <= 65535, "spec_pack: lmax*B=%u exceeds grid limit", grid.z);
  spec_pack_kernel<<<grid, 256, 0, st>>>(static_cast<const float2*>(coeffs), spec, pl->lmax, pl->mmax, B, C, cp, pl->m0, pl->dense);
  B200_CHECK_LAUNCH();
  return 0;
}

// ------------------------------------------------------------------------------- vector SHT boundary
// stacked vector spec [2L][M][2][B][cp] (cp = round_up(2C, 4); column 2c + component, component 0 = theta, 1 = phi; rows l hold the
// D contractions, rows L + l the Q contractions)  <->  (S, T) complex64 [B*C][2][L][M] (exact zeros for l < m):
//   unpack:  S = f (D x_theta - i Q x_phi),   T = f (-i Q x_theta - D x_phi)
//   pack:    D_theta = f S,  D_phi = -f T,  Q_theta = i f T,  Q_phi = i f S
// f = 1 / (l (l + 1)) (0 at l = 0) when `scaled`, else 1.  pack(scaled) is the adjoint of unpack(scaled): the forward transform ends in
// unpack(1) and its adjoint starts with pack(1); the inverse transform starts with pack(0) and its adjoint ends in unpack(0).
// Local order m is the global order mo + m (the plan's order offset): only the l >= mo + m test depends on it.
// block: 32 orders x 16 vector channels (32 spec columns) of one (l, b)
__global__ void __launch_bounds__(256) vector_spec_unpack_kernel(const float* __restrict__ spec, float2* __restrict__ coeffs, int L, int M, int B,
                                                                 int C, int cp, int mo, int scaled) {
  __shared__ float tile[4][32][33];   // D re, D im, Q re, Q im  x  [m][column]
  const int l = blockIdx.z / B, b = blockIdx.z % B;
  const int m0 = blockIdx.x * 32, c0 = blockIdx.y * 16;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const size_t JP = 2 * (size_t)B * cp, pstride = (size_t)B * cp;
  const int j = 2 * c0 + tx;
  for (int mm = ty; mm < 32; mm += 8) {
    const int m = m0 + mm;
    float v[4] = {0.f, 0.f, 0.f, 0.f};
    if (m < M && j < 2 * C && l >= mo + m) {
      const float* d = spec + ((size_t)l * M + m) * JP + (size_t)b * cp + j;
      const float* q = d + (size_t)L * M * JP;
      v[0] = d[0]; v[1] = d[pstride]; v[2] = q[0]; v[3] = q[pstride];
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) tile[i][mm][tx] = v[i];
  }
  __syncthreads();
  const float f = scaled ? (l > 0 ? 1.f / ((float)l * (float)(l + 1)) : 0.f) : 1.f;
  for (int cc = ty; cc < 16; cc += 8) {
    const int c = c0 + cc, m = m0 + tx;
    if (c >= C || m >= M) continue;
    const int jt = 2 * cc, jf = 2 * cc + 1;
    const float2 S = make_float2(f * (tile[0][tx][jt] + tile[3][tx][jf]), f * (tile[1][tx][jt] - tile[2][tx][jf]));
    const float2 T = make_float2(f * (tile[3][tx][jt] - tile[0][tx][jf]), f * (-tile[2][tx][jt] - tile[1][tx][jf]));
    float2* out = coeffs + ((size_t)(b * C + c) * 2 * L + l) * M + m;
    out[0] = S;
    out[(size_t)L * M] = T;
  }
}

// writes every entry of the stacked spec (zeros for l < mo + m and in the channel padding): the Legendre kernels read all rows
// l >= lstart(mo + m)
__global__ void __launch_bounds__(256) vector_spec_pack_kernel(const float2* __restrict__ coeffs, float* __restrict__ spec, int L, int M, int B,
                                                               int C, int cp, int mo, int scaled) {
  __shared__ float tile[4][32][33];
  const int l = blockIdx.z / B, b = blockIdx.z % B;
  const int m0 = blockIdx.x * 32, c0 = blockIdx.y * 16;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const size_t JP = 2 * (size_t)B * cp, pstride = (size_t)B * cp;
  const float f = scaled ? (l > 0 ? 1.f / ((float)l * (float)(l + 1)) : 0.f) : 1.f;
  for (int cc = ty; cc < 16; cc += 8) {
    const int c = c0 + cc, m = m0 + tx;
    float2 S = make_float2(0.f, 0.f), T = S;
    if (c < C && m < M && l >= mo + m) {
      const float2* in = coeffs + ((size_t)(b * C + c) * 2 * L + l) * M + m;
      S = in[0];
      T = in[(size_t)L * M];
      S.x *= f; S.y *= f; T.x *= f; T.y *= f;
    }
    const int jt = 2 * cc, jf = 2 * cc + 1;
    tile[0][tx][jt] = S.x;  tile[1][tx][jt] = S.y;  tile[2][tx][jt] = -T.y; tile[3][tx][jt] = T.x;
    tile[0][tx][jf] = -T.x; tile[1][tx][jf] = -T.y; tile[2][tx][jf] = -S.y; tile[3][tx][jf] = S.x;
  }
  __syncthreads();
  for (int mm = ty; mm < 32; mm += 8) {
    const int m = m0 + mm, j = 2 * c0 + tx;
    if (m >= M || j >= cp) continue;
    float* d = spec + ((size_t)l * M + m) * JP + (size_t)b * cp + j;
    float* q = d + (size_t)L * M * JP;
    d[0] = tile[0][mm][tx]; d[pstride] = tile[1][mm][tx]; q[0] = tile[2][mm][tx]; q[pstride] = tile[3][mm][tx];
  }
}

int vector_spec_convert(const Plan* pl, float* spec, void* coeffs, int B, int C, int to_packed, int scaled, cudaStream_t st) {
  const int L = pl->lmax / 2, cp = round_up(2 * C, 4);
  dim3 grid(ceil_div(pl->mmax, 32), to_packed ? ceil_div(cp, 32) : ceil_div(C, 16), L * B);
  B200_REQUIRE(grid.z <= 65535, "vector spec conversion: lmax*B=%u exceeds grid limit", grid.z);
  if (to_packed)
    vector_spec_pack_kernel<<<grid, 256, 0, st>>>(static_cast<const float2*>(coeffs), spec, L, pl->mmax, B, C, cp, pl->m0, scaled);
  else
    vector_spec_unpack_kernel<<<grid, 256, 0, st>>>(spec, static_cast<float2*>(coeffs), L, pl->mmax, B, C, cp, pl->m0, scaled);
  B200_CHECK_LAUNCH();
  return 0;
}

// latspec [M][2][R][kp]  <->  complex64 [R][nlat][M]   (the layout the distributed transposes exchange).  block: 32 k x 32 m of one row r
__global__ void __launch_bounds__(256) latspec_convert_kernel(float* __restrict__ lat, float2* __restrict__ coeffs, int M, int R, int nlat, int kp,
                                                              int to_packed) {
  __shared__ float tile[2][32][33];
  const int r = blockIdx.z;
  const int k0 = blockIdx.x * 32, m0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  if (!to_packed) {
    for (int mm = ty; mm < 32; mm += 8) {
      const int m = m0 + mm, k = k0 + tx;
      float re = 0.f, im = 0.f;
      if (m < M && k < nlat) {
        re = lat[(((size_t)m * 2 + 0) * R + r) * kp + k];
        im = lat[(((size_t)m * 2 + 1) * R + r) * kp + k];
      }
      tile[0][mm][tx] = re;
      tile[1][mm][tx] = im;
    }
    __syncthreads();
    for (int kk = ty; kk < 32; kk += 8) {
      const int k = k0 + kk, m = m0 + tx;
      if (k < nlat && m < M) coeffs[((size_t)r * nlat + k) * M + m] = make_float2(tile[0][tx][kk], tile[1][tx][kk]);
    }
  } else {
    for (int kk = ty; kk < 32; kk += 8) {
      const int k = k0 + kk, m = m0 + tx;
      float2 v = make_float2(0.f, 0.f);
      if (k < nlat && m < M) v = coeffs[((size_t)r * nlat + k) * M + m];
      tile[0][tx][kk] = v.x;
      tile[1][tx][kk] = v.y;
    }
    __syncthreads();
    for (int mm = ty; mm < 32; mm += 8) {
      const int m = m0 + mm, k = k0 + tx;
      if (m < M && k < kp) {  // the k padding is written as zeros
        lat[(((size_t)m * 2 + 0) * R + r) * kp + k] = tile[0][mm][tx];
        lat[(((size_t)m * 2 + 1) * R + r) * kp + k] = tile[1][mm][tx];
      }
    }
  }
}

int latspec_convert(const Plan* pl, float* lat, void* coeffs, int B, int C, int to_packed, cudaStream_t st) {
  dim3 grid(ceil_div(pl->kp, 32), ceil_div(pl->mmax, 32), B * C);
  B200_REQUIRE(grid.z <= 65535, "latspec_convert: B*C=%u exceeds grid limit", grid.z);
  latspec_convert_kernel<<<grid, 256, 0, st>>>(lat, static_cast<float2*>(coeffs), pl->mmax, B * C, pl->nlat, pl->kp, to_packed);
  B200_CHECK_LAUNCH();
  return 0;
}

// bias gradient: gbias[c] = sum_{b,k} latspec[m=0][re][b*C+c][k]
__global__ void bias_grad_kernel(const float* __restrict__ X, float* __restrict__ gbias, int B, int C, int kp, int nlat) {
  const int c = blockIdx.x;
  float s = 0.f;
  for (int b = 0; b < B; ++b) {
    const float* row = X + ((size_t)(b * C + c)) * kp;
    for (int k = threadIdx.x; k < nlat; k += blockDim.x) s += row[k];
  }
  __shared__ float red[32];
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = (threadIdx.x < (blockDim.x >> 5)) ? red[threadIdx.x] : 0.f;
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (threadIdx.x == 0) gbias[c] = v;
  }
}

int bias_grad(const Plan* pl, const float* X, float* gbias, int B, int C, cudaStream_t st) {
  bias_grad_kernel<<<C, 256, 0, st>>>(X, gbias, B, C, pl->kp, pl->nlat);
  B200_CHECK_LAUNCH();
  return 0;
}

}  // namespace b200sht

// Debug: the table recurrence on the host (same code as the device kernel) for CPU tests.
extern "C" int b200sht_debug_table_host(int nlat, int lmax, int mmax, const double* cost, int csphase, float* table /*[mmax][lmax][nlat]*/) {
  for (int m = 0; m < mmax; ++m)
    for (int k = 0; k < nlat; ++k)
      b200sht::legendre_column(m, lmax, cost[k], csphase, table + (size_t)m * lmax * nlat + k, nlat);
  return 0;
}

extern "C" int b200sht_debug_vector_table_host(int nlat, int lmax, int mmax, const double* cost, int csphase, float* D /*[mmax][lmax][nlat]*/,
                                               float* Q /*[mmax][lmax][nlat]*/) {
  if (nlat < 1 || lmax < 1 || mmax < 1 || !cost || !D || !Q) return B200SHT_ERR_INVALID;
  for (int m = 0; m < mmax; ++m)
    for (int k = 0; k < nlat; ++k) {
      const size_t o = (size_t)m * lmax * nlat + k;
      b200sht::legendre_vector_column(m, lmax, cost[k], csphase, D + o, Q + o, nlat);
    }
  return 0;
}
