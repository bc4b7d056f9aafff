// Neighbourhood attention on the sphere (torch_harmonics.NeighborhoodAttentionS2): each output point attends to the input points of its DISCO
// support, with the quadrature-weighted softmax of include/b200sht.h.  The neighbourhood is a K = 1 DISCO plan (disco_plan.cuh) whose value at
// (t, i, j) is the quadrature weight w_i = 2 pi w_in[i] / nlon_in:
//
//   N(t, p) = { (i, (j + s p) mod nlon_in) : (i, j) in S(t) },   l_n = scale <q_h(t, p), k_h(n)>
//   y_h(t, p) = sum_n w_i exp(l_n) v_h(n) / sum_n w_i exp(l_n),   lse_h(t, p) = log sum_n w_i exp(l_n)
//
// Operands are point-major and channel-contiguous: q (B, nlat_out nlon_out, H EK), k (B, nlat_in nlon_in, H EK), v (B, nlat_in nlon_in, H EV),
// head h at channels [h E, (h + 1) E).  The support of t in input row i is an arc j in [-off, n - 1 - off] (mod nlon_in), n the row's point count
// and off = (n - 1) / 2 (the whole ring when n = nlon_in), so the columns output point p reads in row i are [s p - off, s p - off + n).
//
// Forward and query-side backward: one CTA per (output latitude t, tile of output longitudes, b * H + h), one thread per output longitude.  For
// each input row of t's band the CTA stages the window of K and V columns its tile reads (shared by up to n threads), in chunks near the poles.
// Forward: online softmax with a running max and sum in fp32.  Query side: alpha from lse, D = <dy, y>, dl = alpha (<dy, v_n> - D),
// dq = scale sum dl k_n; D is written for the key/value side.
// Key/value side: one CTA per (input latitude i, tile of input longitudes, b * H + h), one thread per input point n.  For each output row t that
// reaches i (the plan's input-latitude ordering) it stages the window of q (scaled), dy, lse and D that its tile's points gather from:
// dv_n = sum alpha_pn dy_p and dk_n = sum dl_pn scale q_p.  Every output element is summed by one thread in a fixed order: no atomics, and the
// results are bit-identical run to run.  The logits of the three kernels are the same fma sequence on the same fp32 operands, so the backward
// recomputes the forward's logits bit for bit.
#include "disco_plan.cuh"
#include <algorithm>
#include <cmath>

namespace b200sht {

constexpr int kAttnThreads = 128;              // forward / query side: output longitudes per CTA
constexpr int kAttnKVThreads = 64;             // key/value side: input longitudes per CTA
constexpr int kAttnStageBytes = 48 * 1024;     // staged K / V columns (forward, query side)
constexpr int kAttnKVStageBytes = 32 * 1024;   // staged q / dy / lse / D columns (key/value side)
constexpr int kAttnMaxE = 64;                  // largest head dimension

struct AttnArgs {
  const float *q, *k, *v, *y, *lse, *dy;
  float *out, *out_lse, *dq, *dk, *dv, *D;
  int H, EK, EV, CK, CV;
  int nlat_in, nlon_in, nlat_out, nlon_out, s, Kp;
  float scale;
  const int* rowptr; const int2* band; const float* val;
  int SK, SV, CW;
};

// r[c] = mul g[c] for c < E (0 beyond)
template <int EM, bool VEC>
__device__ __forceinline__ void load_row(float (&r)[EM], const float* g, int E, float mul) {
  if (VEC) {
#pragma unroll
    for (int c4 = 0; c4 < EM / 4; ++c4) {
      float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
      if (4 * c4 < E) x = __ldg(reinterpret_cast<const float4*>(g) + c4);
      r[4 * c4 + 0] = x.x * mul; r[4 * c4 + 1] = x.y * mul; r[4 * c4 + 2] = x.z * mul; r[4 * c4 + 3] = x.w * mul;
    }
  } else {
#pragma unroll
    for (int c = 0; c < EM; ++c) r[c] = c < E ? __ldg(g + c) * mul : 0.f;
  }
}

// sum_c a[c] b[c] over c < E, fma in channel order (the same sequence in every kernel)
template <int EM, bool VEC>
__device__ __forceinline__ float dot_rs(const float (&a)[EM], const float* b, int E) {
  float acc = 0.f;
  if (VEC) {
#pragma unroll
    for (int c4 = 0; c4 < EM / 4; ++c4) {
      if (4 * c4 < E) {
        const float4 x = reinterpret_cast<const float4*>(b)[c4];
        acc = fmaf(a[4 * c4 + 0], x.x, acc); acc = fmaf(a[4 * c4 + 1], x.y, acc);
        acc = fmaf(a[4 * c4 + 2], x.z, acc); acc = fmaf(a[4 * c4 + 3], x.w, acc);
      }
    }
  } else {
#pragma unroll
    for (int c = 0; c < EM; ++c)
      if (c < E) acc = fmaf(a[c], b[c], acc);
  }
  return acc;
}

template <int EM, bool VEC>
__device__ __forceinline__ float dot_ss(const float* a, const float* b, int E) {
  float acc = 0.f;
  if (VEC) {
#pragma unroll
    for (int c4 = 0; c4 < EM / 4; ++c4) {
      if (4 * c4 < E) {
        const float4 x = reinterpret_cast<const float4*>(a)[c4], y = reinterpret_cast<const float4*>(b)[c4];
        acc = fmaf(x.x, y.x, acc); acc = fmaf(x.y, y.y, acc); acc = fmaf(x.z, y.z, acc); acc = fmaf(x.w, y.w, acc);
      }
    }
  } else {
#pragma unroll
    for (int c = 0; c < EM; ++c)
      if (c < E) acc = fmaf(a[c], b[c], acc);
  }
  return acc;
}

// acc[c] += w b[c] for c < E
template <int EM, bool VEC>
__device__ __forceinline__ void axpy(float (&acc)[EM], float w, const float* b, int E) {
  if (VEC) {
#pragma unroll
    for (int c4 = 0; c4 < EM / 4; ++c4) {
      if (4 * c4 < E) {
        const float4 x = reinterpret_cast<const float4*>(b)[c4];
        acc[4 * c4 + 0] = fmaf(w, x.x, acc[4 * c4 + 0]); acc[4 * c4 + 1] = fmaf(w, x.y, acc[4 * c4 + 1]);
        acc[4 * c4 + 2] = fmaf(w, x.z, acc[4 * c4 + 2]); acc[4 * c4 + 3] = fmaf(w, x.w, acc[4 * c4 + 3]);
      }
    }
  } else {
#pragma unroll
    for (int c = 0; c < EM; ++c)
      if (c < E) acc[c] = fmaf(w, b[c], acc[c]);
  }
}

template <int EM>
__device__ __forceinline__ void store_row(float* g, const float (&r)[EM], int E, float mul) {
#pragma unroll
  for (int c = 0; c < EM; ++c)
    if (c < E) g[c] = r[c] * mul;
}

// columns (c0 + w) mod nlon, w in [w0, w0 + cw), of one row of a point-major tensor (row base `src`, C channels per point, E of them from
// channel offset 0 of `src`) -> dst[w - w0][0 .. E) with row stride S; multiplied by `mul`
template <bool VEC>
__device__ __forceinline__ void stage_cols(float* dst, int S, const float* src, int C, int E, int nlon, int c0, int w0, int cw, float mul) {
  if (VEC) {
    const int per = E / 4;
    for (int e = threadIdx.x; e < cw * per; e += blockDim.x) {
      const int w = e / per, c4 = e - w * per;
      const int col = (c0 + w0 + w) % nlon;
      const float4 x = __ldg(reinterpret_cast<const float4*>(src + (size_t)col * C) + c4);
      reinterpret_cast<float4*>(dst + (size_t)w * S)[c4] = make_float4(x.x * mul, x.y * mul, x.z * mul, x.w * mul);
    }
  } else {
    for (int e = threadIdx.x; e < cw * E; e += blockDim.x) {
      const int w = e / E, c = e - w * E;
      const int col = (c0 + w0 + w) % nlon;
      dst[(size_t)w * S + c] = __ldg(src + (size_t)col * C + c) * mul;
    }
  }
}

__device__ __forceinline__ int mod_pos(int x, int n) { x %= n; return x < 0 ? x + n : x; }

// Forward (QUERY = false) and query-side backward (QUERY = true) share the walk over t's band.
template <int EM, bool VEC, bool QUERY>
__global__ void __launch_bounds__(kAttnThreads, 1) attn_query_kernel(AttnArgs a) {
  extern __shared__ __align__(16) float sm[];
  float* ks = sm;                                   // [CW][SK]
  float* vs = sm + (size_t)a.CW * a.SK;             // [CW][SV]

  const int t = blockIdx.x, p0 = blockIdx.y * blockDim.x, bh = blockIdx.z;
  const int b = bh / a.H, h = bh - b * a.H;
  const int lp = threadIdx.x, np = min((int)blockDim.x, a.nlon_out - p0);
  const bool live = lp < np;
  const size_t opt = (size_t)b * a.nlat_out * a.nlon_out + (size_t)t * a.nlon_out + p0 + (live ? lp : 0);   // output point
  const size_t oh = ((size_t)b * a.H + h) * a.nlat_out * a.nlon_out + (size_t)t * a.nlon_out + p0 + (live ? lp : 0);

  float q[EM], acc[EM], dyr[EM];
  load_row<EM, VEC>(q, a.q + opt * a.CK + h * a.EK, a.EK, a.scale);
#pragma unroll
  for (int c = 0; c < EM; ++c) acc[c] = 0.f;
  float m = -INFINITY, l = 0.f, lse = 0.f, Dp = 0.f;
  if (QUERY) {
    load_row<EM, VEC>(dyr, a.dy + opt * a.CV + h * a.EV, a.EV, 1.f);
    float yr[EM];
    load_row<EM, VEC>(yr, a.y + opt * a.CV + h * a.EV, a.EV, 1.f);
    Dp = dot_rs<EM, VEC>(dyr, yr, a.EV);
    lse = __ldg(a.lse + oh);
  }

  const int* rp = a.rowptr + (size_t)t * (a.nlat_in + 1);
  const int2 band = a.band[t];
  const size_t in_b = (size_t)b * a.nlat_in * a.nlon_in;
  for (int i = band.x; i < band.y; ++i) {
    const int q0 = rp[i], n = rp[i + 1] - q0;
    if (n == 0) continue;
    const float w = __ldg(a.val + (size_t)q0 * a.Kp);
    const int off = (n - 1) / 2;
    const int Wd = a.s * (np - 1) + n;
    const int c0 = mod_pos(a.s * p0 - off, a.nlon_in);
    const float* krow = a.k + (in_b + (size_t)i * a.nlon_in) * a.CK + h * a.EK;
    const float* vrow = a.v + (in_b + (size_t)i * a.nlon_in) * a.CV + h * a.EV;
    for (int w0 = 0; w0 < Wd; w0 += a.CW) {
      const int cw = min(a.CW, Wd - w0);
      __syncthreads();   // the previous chunk is consumed
      stage_cols<VEC>(ks, a.SK, krow, a.CK, a.EK, a.nlon_in, c0, w0, cw, 1.f);
      stage_cols<VEC>(vs, a.SV, vrow, a.CV, a.EV, a.nlon_in, c0, w0, cw, 1.f);
      __syncthreads();
      if (!live) continue;
      const int ua = max(w0, a.s * lp), ub = min(w0 + cw, a.s * lp + n);
      for (int u = ua; u < ub; ++u) {
        const float* kr = ks + (size_t)(u - w0) * a.SK;
        const float* vr = vs + (size_t)(u - w0) * a.SV;
        const float lg = dot_rs<EM, VEC>(q, kr, a.EK);
        if (QUERY) {
          const float al = w * expf(lg - lse);
          const float dl = al * (dot_rs<EM, VEC>(dyr, vr, a.EV) - Dp);
          axpy<EM, VEC>(acc, dl, kr, a.EK);
        } else {
          if (lg > m) {
            const float c = expf(m - lg);
            l *= c;
#pragma unroll
            for (int e = 0; e < EM; ++e) acc[e] *= c;
            m = lg;
          }
          const float e = w * expf(lg - m);
          l += e;
          axpy<EM, VEC>(acc, e, vr, a.EV);
        }
      }
    }
  }
  if (!live) return;
  if (QUERY) {
    store_row<EM>(a.dq + opt * a.CK + h * a.EK, acc, a.EK, a.scale);
    a.D[oh] = Dp;
  } else {
    store_row<EM>(a.out + opt * a.CV + h * a.EV, acc, a.EV, 1.f / l);
    a.out_lse[oh] = m + logf(l);
  }
}

// floor(x / s) for x >= -s * nlon_out
__device__ __forceinline__ int floor_div(int x, int s, int nlon_out) { return (x + s * nlon_out) / s - nlon_out; }

template <int EM, bool VEC>
__global__ void __launch_bounds__(kAttnKVThreads, 1) attn_kv_kernel(AttnArgs a) {
  extern __shared__ __align__(16) float sm[];
  float* kn = sm;                                          // [blockDim][SK] the thread's own k_n
  float* vn = kn + (size_t)blockDim.x * a.SK;              // [blockDim][SV] the thread's own v_n
  float* qs = vn + (size_t)blockDim.x * a.SV;              // [CW][SK] scale q_p
  float* ds = qs + (size_t)a.CW * a.SK;                    // [CW][SV] dy_p
  float* ls = ds + (size_t)a.CW * a.SV;                    // [CW] lse_p
  float* Ds = ls + a.CW;                                   // [CW] D_p

  const int i = blockIdx.x, j0 = blockIdx.y * blockDim.x, bh = blockIdx.z;
  const int b = bh / a.H, h = bh - b * a.H;
  const int lj = threadIdx.x, nj = min((int)blockDim.x, a.nlon_in - j0);
  const bool live = lj < nj;
  const int jp = j0 + (live ? lj : 0);
  const size_t ipt = (size_t)b * a.nlat_in * a.nlon_in + (size_t)i * a.nlon_in + jp;
  {
    float r[EM];
    load_row<EM, VEC>(r, a.k + ipt * a.CK + h * a.EK, a.EK, 1.f);
#pragma unroll
    for (int c = 0; c < EM; ++c)
      if (c < a.EK) kn[(size_t)lj * a.SK + c] = r[c];
    load_row<EM, VEC>(r, a.v + ipt * a.CV + h * a.EV, a.EV, 1.f);
#pragma unroll
    for (int c = 0; c < EM; ++c)
      if (c < a.EV) vn[(size_t)lj * a.SV + c] = r[c];
  }
  const float* kr = kn + (size_t)lj * a.SK;
  const float* vr = vn + (size_t)lj * a.SV;
  float dk[EM], dv[EM];
#pragma unroll
  for (int c = 0; c < EM; ++c) dk[c] = dv[c] = 0.f;

  const int* rp = a.rowptr + (size_t)i * (a.nlat_out + 1);
  const int2 band = a.band[i];
  const float w = band.y > band.x ? __ldg(a.val + (size_t)rp[band.x] * a.Kp) : 0.f;
  const size_t out_b = (size_t)b * a.nlat_out * a.nlon_out;
  const size_t lse_b = ((size_t)b * a.H + h) * a.nlat_out * a.nlon_out;
  for (int t = band.x; t < band.y; ++t) {
    const int n = rp[t + 1] - rp[t];
    if (n == 0) continue;
    const int off = (n - 1) / 2;
    // output longitudes p whose neighbourhood holds column j': s p in [j' - (n - 1 - off), j' + off]
    const int P0 = floor_div(j0 - (n - 1 - off) + a.s - 1, a.s, a.nlon_out);
    const int Wp = floor_div(j0 + nj - 1 + off, a.s, a.nlon_out) - P0 + 1;
    const int pa = floor_div(jp - (n - 1 - off) + a.s - 1, a.s, a.nlon_out) - P0;
    const int pb = floor_div(jp + off, a.s, a.nlon_out) - P0 + 1;
    const int c0 = mod_pos(P0, a.nlon_out);
    const size_t orow = out_b + (size_t)t * a.nlon_out;
    const size_t lrow = lse_b + (size_t)t * a.nlon_out;
    for (int w0 = 0; w0 < Wp; w0 += a.CW) {
      const int cw = min(a.CW, Wp - w0);
      __syncthreads();
      stage_cols<VEC>(qs, a.SK, a.q + orow * a.CK + h * a.EK, a.CK, a.EK, a.nlon_out, c0, w0, cw, a.scale);
      stage_cols<VEC>(ds, a.SV, a.dy + orow * a.CV + h * a.EV, a.CV, a.EV, a.nlon_out, c0, w0, cw, 1.f);
      for (int e = threadIdx.x; e < cw; e += blockDim.x) {
        const int col = (c0 + w0 + e) % a.nlon_out;
        ls[e] = __ldg(a.lse + lrow + col);
        Ds[e] = __ldg(a.D + lrow + col);
      }
      __syncthreads();
      if (!live) continue;
      const int ua = max(w0, pa), ub = min(w0 + cw, pb);
      for (int u = ua; u < ub; ++u) {
        const float* qr = qs + (size_t)(u - w0) * a.SK;
        const float* dr = ds + (size_t)(u - w0) * a.SV;
        const float lg = dot_ss<EM, VEC>(qr, kr, a.EK);
        const float al = w * expf(lg - ls[u - w0]);
        const float dl = al * (dot_ss<EM, VEC>(dr, vr, a.EV) - Ds[u - w0]);
        axpy<EM, VEC>(dv, al, dr, a.EV);
        axpy<EM, VEC>(dk, dl, qr, a.EK);
      }
    }
  }
  if (!live) return;
  store_row<EM>(a.dk + ipt * a.CK + h * a.EK, dk, a.EK, 1.f);
  store_row<EM>(a.dv + ipt * a.CV + h * a.EV, dv, a.EV, 1.f);
}

// ------------------------------------------------------------------------------------------------------------------------- launches
template <int EM, bool VEC, bool QUERY> struct AttnQueryTag {};
template <int EM, bool VEC> struct AttnKVTag {};

static bool aligned16f(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// shared-memory row stride: float4 rows with an odd count of float4 (conflict-free 16-byte loads across threads), scalar rows of odd length
static int smem_stride(int E, bool vec) { return vec ? 4 * ((E / 4) | 1) : (E | 1); }

template <int EM, bool VEC, bool QUERY>
static int launch_query(AttnArgs a, int B, cudaStream_t st) {
  a.SK = smem_stride(a.EK, VEC); a.SV = smem_stride(a.EV, VEC);
  a.CW = std::max(1, kAttnStageBytes / ((a.SK + a.SV) * 4));
  const int threads = std::min(kAttnThreads, round_up(a.nlon_out, 32));
  const size_t smem = (size_t)a.CW * (a.SK + a.SV) * 4;
  B200_CHECK_CUDA((ensure_dynamic_smem<AttnQueryTag<EM, VEC, QUERY>>(attn_query_kernel<EM, VEC, QUERY>, smem)));
  dim3 grid(a.nlat_out, ceil_div(a.nlon_out, threads), B * a.H);
  attn_query_kernel<EM, VEC, QUERY><<<grid, threads, smem, st>>>(a);
  B200_CHECK_LAUNCH();
  return B200SHT_OK;
}

template <int EM, bool VEC>
static int launch_kv(AttnArgs a, int B, cudaStream_t st) {
  a.SK = smem_stride(a.EK, VEC); a.SV = smem_stride(a.EV, VEC);
  a.CW = std::max(1, kAttnKVStageBytes / ((a.SK + a.SV + 2) * 4));
  const int threads = std::min(kAttnKVThreads, round_up(a.nlon_in, 32));
  const size_t smem = ((size_t)threads * (a.SK + a.SV) + (size_t)a.CW * (a.SK + a.SV + 2)) * 4;
  B200_CHECK_CUDA((ensure_dynamic_smem<AttnKVTag<EM, VEC>>(attn_kv_kernel<EM, VEC>, smem)));
  dim3 grid(a.nlat_in, ceil_div(a.nlon_in, threads), B * a.H);
  attn_kv_kernel<EM, VEC><<<grid, threads, smem, st>>>(a);
  B200_CHECK_LAUNCH();
  return B200SHT_OK;
}

// kind 0 forward, 1 query side, 2 key/value side
template <bool VEC>
static int dispatch_em(int kind, int em, const AttnArgs& a, int B, cudaStream_t st) {
#define B200_ATTN_CASE(EM)                                          \
  case EM:                                                          \
    if (kind == 0) return launch_query<EM, VEC, false>(a, B, st);   \
    if (kind == 1) return launch_query<EM, VEC, true>(a, B, st);    \
    return launch_kv<EM, VEC>(a, B, st);
  switch (em) {
    B200_ATTN_CASE(4)
    B200_ATTN_CASE(8)
    B200_ATTN_CASE(16)
    B200_ATTN_CASE(32)
    default:
    B200_ATTN_CASE(64)
  }
#undef B200_ATTN_CASE
}

static int attn_check(const char* who, const b200sht_disco_plan* pl, int B, int H, int EK, int EV) {
  B200_REQUIRE(pl, "%s: null plan", who);
  B200_REQUIRE(pl->K == 1, "%s: the neighbourhood plan must have K = 1 (got %d)", who, pl->K);
  B200_REQUIRE(B > 0 && H > 0 && EK > 0 && EV > 0, "%s: bad batch %d / heads %d / head dims %d, %d", who, B, H, EK, EV);
  B200_REQUIRE((long long)B * H <= 65535, "%s: B * heads = %lld is too many for one launch", who, (long long)B * H);
  if (EK > kAttnMaxE || EV > kAttnMaxE) {
    set_error("%s: head dims %d, %d exceed %d", who, EK, EV, kAttnMaxE);
    return B200SHT_ERR_UNSUPPORTED;
  }
  return B200SHT_OK;
}

static AttnArgs attn_args(const b200sht_disco_plan* pl, int H, int EK, int EV, float scale) {
  AttnArgs a;
  memset(&a, 0, sizeof(a));
  a.H = H; a.EK = EK; a.EV = EV; a.CK = H * EK; a.CV = H * EV;
  a.nlat_in = pl->nlat_in; a.nlon_in = pl->nlon_in; a.nlat_out = pl->nlat_out; a.nlon_out = pl->nlon_out;
  a.s = pl->pscale; a.Kp = pl->Kp; a.scale = scale;
  return a;
}

static int head_em(int EK, int EV) {
  const int e = std::max(EK, EV);
  return e <= 4 ? 4 : e <= 8 ? 8 : e <= 16 ? 16 : e <= 32 ? 32 : 64;
}

static bool vec_ok(int EK, int EV, std::initializer_list<const void*> ptrs) {
  if (EK % 4 || EV % 4) return false;
  for (const void* p : ptrs)
    if (!aligned16f(p)) return false;
  return true;
}

int attention_forward(const b200sht_disco_plan* pl, const float* q, const float* k, const float* v, float* y, float* lse, int B, int H, int EK,
                      int EV, float scale, cudaStream_t st) {
  if (int rc = attn_check("attention_forward", pl, B, H, EK, EV)) return rc;
  B200_REQUIRE(q && k && v && y && lse, "attention_forward: null argument");
  AttnArgs a = attn_args(pl, H, EK, EV, scale);
  a.q = q; a.k = k; a.v = v; a.out = y; a.out_lse = lse;
  a.rowptr = pl->d_fwd_rowptr; a.band = pl->d_fwd_band; a.val = pl->d_fwd_val;
  const int em = head_em(EK, EV);
  return vec_ok(EK, EV, {q, k, v, y}) ? dispatch_em<true>(0, em, a, B, st) : dispatch_em<false>(0, em, a, B, st);
}

int attention_backward(const b200sht_disco_plan* pl, const float* q, const float* k, const float* v, const float* y, const float* lse,
                       const float* dy, float* dq, float* dk, float* dv, float* D, int B, int H, int EK, int EV, float scale, cudaStream_t st) {
  if (int rc = attn_check("attention_backward", pl, B, H, EK, EV)) return rc;
  B200_REQUIRE(q && k && v && y && lse && dy && dq && dk && dv && D, "attention_backward: null argument");
  AttnArgs a = attn_args(pl, H, EK, EV, scale);
  a.q = q; a.k = k; a.v = v; a.y = y; a.lse = lse; a.dy = dy; a.dq = dq; a.dk = dk; a.dv = dv; a.D = D;
  const int em = head_em(EK, EV);
  const bool vec = vec_ok(EK, EV, {q, k, v, y, dy, dq, dk, dv});
  a.rowptr = pl->d_fwd_rowptr; a.band = pl->d_fwd_band; a.val = pl->d_fwd_val;
  int rc = vec ? dispatch_em<true>(1, em, a, B, st) : dispatch_em<false>(1, em, a, B, st);
  if (rc) return rc;
  a.rowptr = pl->d_adj_rowptr; a.band = pl->d_adj_band; a.val = pl->d_adj_val;
  return vec ? dispatch_em<true>(2, em, a, B, st) : dispatch_em<false>(2, em, a, B, st);
}

}  // namespace b200sht
