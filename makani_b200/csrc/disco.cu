// DISCO convolution on the sphere (torch_harmonics.DiscreteContinuousConvS2): the two sparse contractions with the filter tensor psi.
//
//   forward  X[b,c,k,t,p]  = sum_{i,j} psi[k,t,i,j] x[b,c,i,(j + pscale p) mod nlon_in]                    x -> X
//   adjoint  dx[b,c,i,j']  = sum_{k,t,p,j : (j + pscale p) mod nlon_in = j'} psi[k,t,i,j] dX[b,c,k,t,p]     dX -> dx
//
// The plan holds psi twice, as points (one support point carrying its K values, padded to Kp = K rounded up to 4):
//   by output latitude t (forward), sorted by (i, j), with a row pointer per (t, i): the rows of t's band are contiguous;
//   by input latitude i (adjoint), sorted by (t, j), with a row pointer per (i, t).
// Forward: one CTA per (t, chunk of R rows of B*C, tile of output longitudes).  It stages the band of input rows t touches (SR rows at a time)
// and t's points (PC at a time) in shared memory; each thread owns NP output longitudes of one row and KP fp32 accumulators for each, so
// a point costs NP shared loads of x, KP/4 broadcast float4 loads of psi and NP*KP FMAs.  K > 32 runs in launches of 32 kernel functions.
// Adjoint: one CTA per (i, chunk of rows, tile of input longitudes).  It stages the band of dX rows that reach i (all K or KC at a time)
// and i's points; a thread owns NJ input longitudes j' = res + pscale u and gathers, for each point (t, j) with j = res (mod pscale), the
// K values dX[k, t, (u - j / pscale) mod nlon_out].  Every output element is summed by one thread in a fixed order: no atomics, and the
// results are bit-identical run to run.
#include "disco_plan.cuh"
#include <algorithm>
#include <type_traits>
#include <vector>

namespace b200sht {

constexpr int kDiscoThreads = 256;
constexpr int kDiscoPC = 256;               // points staged at a time
constexpr int kDiscoStageBytes = 64 * 1024; // staged x rows (forward) or dX rows (adjoint)
constexpr int kDiscoMaxKC = 32;             // kernel functions per forward launch / per adjoint pass
constexpr int kDiscoNJ = 4;                 // adjoint: input longitudes per thread

struct DiscoFwdArgs {
  const void* x; float* X; int dtype, BC;
  int nlat_in, nlon_in, nlat_out, nlon_out, K, Kp, pscale;
  int k0, KC, R, TPR, SR, vec;
  const int* rowptr; const int2* band; const int2* pos; const float* val;
};

struct DiscoAdjArgs {
  const float* dX; void* dx; int dtype, BC;
  int nlat_in, nlon_in, nlat_out, nlon_out, K, Kp, pscale;
  int KC, R, TPJ, ST, vec;
  const int* rowptr; const int2* band; const int2* pos; const float* val;
};

// rows [row0, row0 + n) of `src` (n elements, contiguous) -> fp32 in shared memory; 16-byte loads when vec
__device__ __forceinline__ void stage_rows(float* dst, const void* src, long long off, int n, int dtype, int vec) {
  if (dtype == B200SHT_F32) {
    const float* s = static_cast<const float*>(src) + off;
    if (vec) {
      const float4* s4 = reinterpret_cast<const float4*>(s);
      float4* d4 = reinterpret_cast<float4*>(dst);
      for (int e = threadIdx.x; e < n / 4; e += blockDim.x) d4[e] = __ldg(s4 + e);
    } else {
      for (int e = threadIdx.x; e < n; e += blockDim.x) dst[e] = __ldg(s + e);
    }
  } else {
    const __nv_bfloat16* s = static_cast<const __nv_bfloat16*>(src) + off;
    if (vec) {
      const uint4* s8 = reinterpret_cast<const uint4*>(s);
      float4* d4 = reinterpret_cast<float4*>(dst);
      for (int e = threadIdx.x; e < n / 8; e += blockDim.x) {
        uint4 u = __ldg(s8 + e);
        const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
        float2 a = __bfloat1622float2(h[0]), b = __bfloat1622float2(h[1]), c = __bfloat1622float2(h[2]), d = __bfloat1622float2(h[3]);
        d4[2 * e] = make_float4(a.x, a.y, b.x, b.y);
        d4[2 * e + 1] = make_float4(c.x, c.y, d.x, d.y);
      }
    } else {
      for (int e = threadIdx.x; e < n; e += blockDim.x) dst[e] = __bfloat162float(s[e]);
    }
  }
}

template <int KP, int NP>
__global__ void __launch_bounds__(kDiscoThreads, 2) disco_forward_kernel(DiscoFwdArgs a) {
  extern __shared__ __align__(16) unsigned char smem[];
  float* pv = reinterpret_cast<float*>(smem);                       // [PC][KP]
  int2* pp = reinterpret_cast<int2*>(pv + kDiscoPC * KP);           // [PC] (row offset in xs, j)
  float* xs = reinterpret_cast<float*>(pp + kDiscoPC);              // [R][SR][nlon_in]

  const int t = blockIdx.x;
  const int r = threadIdx.x / a.TPR, g = threadIdx.x % a.TPR;
  const int row = blockIdx.y * a.R + r;
  const int pbase = blockIdx.z * a.TPR * NP + g;
  int pofs[NP];
#pragma unroll
  for (int u = 0; u < NP; ++u) pofs[u] = a.pscale * min(pbase + u * a.TPR, a.nlon_out - 1);
  float acc[NP][KP];
#pragma unroll
  for (int u = 0; u < NP; ++u)
#pragma unroll
    for (int k = 0; k < KP; ++k) acc[u][k] = 0.f;

  const int* rp = a.rowptr + (size_t)t * (a.nlat_in + 1);
  const int2 band = a.band[t];
  const float* xr = xs + (size_t)r * a.SR * a.nlon_in;
  for (int s0 = band.x; s0 < band.y; s0 += a.SR) {
    const int s1 = min(s0 + a.SR, band.y);
    __syncthreads();   // the previous stage is consumed
    for (int rr = 0; rr < a.R; ++rr) {
      const int rw = blockIdx.y * a.R + rr;
      if (rw < a.BC)
        stage_rows(xs + (size_t)rr * a.SR * a.nlon_in, a.x, ((long long)rw * a.nlat_in + s0) * a.nlon_in, (s1 - s0) * a.nlon_in, a.dtype, a.vec);
    }
    const int qa = rp[s0], qb = rp[s1];
    for (int c0 = qa; c0 < qb; c0 += kDiscoPC) {
      const int nc = min(kDiscoPC, qb - c0);
      if (c0 != qa) __syncthreads();
      for (int e = threadIdx.x; e < nc * KP; e += blockDim.x) {
        const int q = e / KP, kk = e % KP;
        pv[e] = kk < a.KC ? __ldg(a.val + (size_t)(c0 + q) * a.Kp + a.k0 + kk) : 0.f;
      }
      for (int q = threadIdx.x; q < nc; q += blockDim.x) {
        const int2 ij = a.pos[c0 + q];
        pp[q] = make_int2((ij.x - s0) * a.nlon_in, ij.y);
      }
      __syncthreads();
      for (int q = 0; q < nc; ++q) {
        const int2 pq = pp[q];
        float xv[NP];
#pragma unroll
        for (int u = 0; u < NP; ++u) {
          int c = pq.y + pofs[u];
          c -= c >= a.nlon_in ? a.nlon_in : 0;
          xv[u] = xr[pq.x + c];
        }
        const float4* w4 = reinterpret_cast<const float4*>(pv + q * KP);
#pragma unroll
        for (int k4 = 0; k4 < KP / 4; ++k4) {
          const float4 w = w4[k4];
#pragma unroll
          for (int u = 0; u < NP; ++u) {
            acc[u][4 * k4 + 0] = fmaf(w.x, xv[u], acc[u][4 * k4 + 0]);
            acc[u][4 * k4 + 1] = fmaf(w.y, xv[u], acc[u][4 * k4 + 1]);
            acc[u][4 * k4 + 2] = fmaf(w.z, xv[u], acc[u][4 * k4 + 2]);
            acc[u][4 * k4 + 3] = fmaf(w.w, xv[u], acc[u][4 * k4 + 3]);
          }
        }
      }
    }
  }
  if (row >= a.BC) return;
#pragma unroll
  for (int u = 0; u < NP; ++u) {
    const int p = pbase + u * a.TPR;
    if (p >= a.nlon_out) continue;
#pragma unroll
    for (int k = 0; k < KP; ++k)
      if (k < a.KC) a.X[(((size_t)row * a.K + a.k0 + k) * a.nlat_out + t) * a.nlon_out + p] = acc[u][k];
  }
}

__global__ void __launch_bounds__(kDiscoThreads) disco_adjoint_kernel(DiscoAdjArgs a) {
  extern __shared__ __align__(16) unsigned char smem[];
  float* pv = reinterpret_cast<float*>(smem);                       // [PC][KC]
  int4* pp = reinterpret_cast<int4*>(pv + kDiscoPC * kDiscoMaxKC);  // [PC] (row offset in ds, j mod pscale, j / pscale)
  float* ds = reinterpret_cast<float*>(pp + kDiscoPC);              // [R][KC][ST][nlon_out]

  const int i = blockIdx.x;
  const int r = threadIdx.x / a.TPJ, g = threadIdx.x % a.TPJ;
  const int row = blockIdx.y * a.R + r;
  const int cbase = blockIdx.z * a.TPJ * kDiscoNJ + g;
  int res[kDiscoNJ], uu[kDiscoNJ];
#pragma unroll
  for (int n = 0; n < kDiscoNJ; ++n) {
    const int c = min(cbase + n * a.TPJ, a.nlon_in - 1);   // column c holds j' = res + pscale u with (res, u) = divmod(c, nlon_out)
    res[n] = c / a.nlon_out;
    uu[n] = c - res[n] * a.nlon_out;
  }
  float acc[kDiscoNJ] = {};

  const int* rp = a.rowptr + (size_t)i * (a.nlat_out + 1);
  const int2 band = a.band[i];
  const size_t slab = (size_t)a.ST * a.nlon_out;
  for (int k0 = 0; k0 < a.K; k0 += a.KC) {
    const int kc = min(a.KC, a.K - k0);
    for (int s0 = band.x; s0 < band.y; s0 += a.ST) {
      const int s1 = min(s0 + a.ST, band.y);
      __syncthreads();
      for (int rr = 0; rr < a.R; ++rr) {
        const int rw = blockIdx.y * a.R + rr;
        if (rw >= a.BC) continue;
        for (int kk = 0; kk < kc; ++kk)
          stage_rows(ds + ((size_t)rr * a.KC + kk) * slab, a.dX, (((long long)rw * a.K + k0 + kk) * a.nlat_out + s0) * a.nlon_out,
                     (s1 - s0) * a.nlon_out, B200SHT_F32, a.vec);
      }
      const int qa = rp[s0], qb = rp[s1];
      for (int c0 = qa; c0 < qb; c0 += kDiscoPC) {
        const int nc = min(kDiscoPC, qb - c0);
        if (c0 != qa) __syncthreads();
        for (int e = threadIdx.x; e < nc * kc; e += blockDim.x) {
          const int q = e / kc, kk = e % kc;
          pv[q * a.KC + kk] = __ldg(a.val + (size_t)(c0 + q) * a.Kp + k0 + kk);
        }
        for (int q = threadIdx.x; q < nc; q += blockDim.x) {
          const int2 tj = a.pos[c0 + q];
          const int jq = tj.y / a.pscale;
          pp[q] = make_int4((tj.x - s0) * a.nlon_out, tj.y - jq * a.pscale, jq, 0);
        }
        __syncthreads();
        const float* dr = ds + (size_t)r * a.KC * slab;
        for (int q = 0; q < nc; ++q) {
          const int4 pq = pp[q];
          int pidx[kDiscoNJ];
          bool any = false;
#pragma unroll
          for (int n = 0; n < kDiscoNJ; ++n) {
            int p = uu[n] - pq.z;
            p += p < 0 ? a.nlon_out : 0;
            pidx[n] = pq.y == res[n] ? pq.x + p : -1;
            any |= pidx[n] >= 0;
          }
          if (!any) continue;
          const float* v = pv + q * a.KC;
          for (int kk = 0; kk < kc; ++kk) {
            const float w = v[kk];
            const float* d = dr + kk * slab;
#pragma unroll
            for (int n = 0; n < kDiscoNJ; ++n)
              if (pidx[n] >= 0) acc[n] = fmaf(w, d[pidx[n]], acc[n]);
          }
        }
      }
    }
  }
  if (row >= a.BC) return;
#pragma unroll
  for (int n = 0; n < kDiscoNJ; ++n) {
    const int c = cbase + n * a.TPJ;
    if (c >= a.nlon_in) continue;
    const size_t o = ((size_t)row * a.nlat_in + i) * a.nlon_in + res[n] + (size_t)a.pscale * uu[n];
    if (a.dtype == B200SHT_F32) static_cast<float*>(a.dx)[o] = acc[n];
    else static_cast<__nv_bfloat16*>(a.dx)[o] = __float2bfloat16_rn(acc[n]);
  }
}

// ------------------------------------------------------------------------------------------------------------------------- plan
struct DiscoEntry { int t, col, k; double v; };

int disco_plan_create(b200sht_disco_plan** out, int nlat_in, int nlon_in, int nlat_out, int nlon_out, int K, long long nnz, const int* ker,
                      const int* lat_out, const int* col_in, const double* vals, cudaStream_t st) {
  B200_REQUIRE(out, "disco_plan_create: null plan pointer");
  *out = nullptr;
  B200_REQUIRE(nlat_in > 0 && nlon_in > 0 && nlat_out > 0 && nlon_out > 0 && K > 0 && nnz >= 0,
               "disco_plan_create: bad sizes (nlat_in %d nlon_in %d nlat_out %d nlon_out %d K %d nnz %lld)", nlat_in, nlon_in, nlat_out, nlon_out, K, nnz);
  B200_REQUIRE(nlon_in % nlon_out == 0, "disco_plan_create: nlon_in %d is not a multiple of nlon_out %d", nlon_in, nlon_out);
  B200_REQUIRE(nnz == 0 || (ker && lat_out && col_in && vals), "disco_plan_create: null entry array");
  if ((long long)nlon_in * 4 > kDiscoStageBytes || (long long)nlon_out * 4 > kDiscoStageBytes) {
    set_error("disco_plan_create: nlon_in %d / nlon_out %d exceed the staged row length (%d floats)", nlon_in, nlon_out, kDiscoStageBytes / 4);
    return B200SHT_ERR_UNSUPPORTED;
  }
  const long long ncol = (long long)nlat_in * nlon_in;
  std::vector<DiscoEntry> e((size_t)nnz);
  for (long long n = 0; n < nnz; ++n) {
    B200_REQUIRE(ker[n] >= 0 && ker[n] < K && lat_out[n] >= 0 && lat_out[n] < nlat_out && col_in[n] >= 0 && col_in[n] < ncol,
                 "disco_plan_create: entry %lld (k %d, t %d, col %d) out of range", n, ker[n], lat_out[n], col_in[n]);
    e[n] = {lat_out[n], col_in[n], ker[n], vals[n]};
  }
  std::stable_sort(e.begin(), e.end(), [](const DiscoEntry& a, const DiscoEntry& b) { return a.t != b.t ? a.t < b.t : a.col < b.col; });

  const int Kp = round_up(K, 4);
  std::vector<int> pt_t, pt_col;
  std::vector<double> acc;
  for (size_t n = 0; n < e.size(); ++n) {
    if (n == 0 || e[n].t != e[n - 1].t || e[n].col != e[n - 1].col) {
      pt_t.push_back(e[n].t);
      pt_col.push_back(e[n].col);
      acc.resize(acc.size() + Kp, 0.0);
    }
    acc[(pt_t.size() - 1) * Kp + e[n].k] += e[n].v;   // duplicate entries are summed in fp64
  }
  const size_t npts = pt_t.size();
  std::vector<int> f_rowptr((size_t)nlat_out * (nlat_in + 1)), a_rowptr((size_t)nlat_in * (nlat_out + 1));
  std::vector<int2> f_band(nlat_out, make_int2(0, 0)), a_band(nlat_in, make_int2(0, 0)), f_pos(npts), a_pos(npts);
  std::vector<float> f_val(npts * Kp), a_val(npts * Kp);
  for (size_t q = 0; q < npts; ++q) {
    f_pos[q] = make_int2(pt_col[q] / nlon_in, pt_col[q] % nlon_in);
    for (int k = 0; k < Kp; ++k) f_val[q * Kp + k] = (float)acc[q * Kp + k];
  }
  {
    size_t q = 0;
    for (int t = 0; t < nlat_out; ++t) {
      const size_t q0 = q;
      for (int i = 0; i <= nlat_in; ++i) {
        while (q < npts && pt_t[q] == t && f_pos[q].x < i) ++q;
        f_rowptr[(size_t)t * (nlat_in + 1) + i] = (int)q;
      }
      if (q > q0) f_band[t] = make_int2(f_pos[q0].x, f_pos[q - 1].x + 1);
    }
  }
  // adjoint copy: the same points ordered by (i, t, j)
  std::vector<int> ord(npts);
  for (size_t q = 0; q < npts; ++q) ord[q] = (int)q;
  std::stable_sort(ord.begin(), ord.end(), [&](int a, int b) { return f_pos[a].x != f_pos[b].x ? f_pos[a].x < f_pos[b].x : pt_t[a] < pt_t[b]; });
  for (size_t n = 0; n < npts; ++n) {
    const int q = ord[n];
    a_pos[n] = make_int2(pt_t[q], f_pos[q].y);
    std::copy(f_val.begin() + (size_t)q * Kp, f_val.begin() + (size_t)(q + 1) * Kp, a_val.begin() + n * Kp);
  }
  {
    size_t n = 0;
    for (int i = 0; i < nlat_in; ++i) {
      const size_t n0 = n;
      for (int t = 0; t <= nlat_out; ++t) {
        while (n < npts && f_pos[ord[n]].x == i && a_pos[n].x < t) ++n;
        a_rowptr[(size_t)i * (nlat_out + 1) + t] = (int)n;
      }
      if (n > n0) a_band[i] = make_int2(a_pos[n0].x, a_pos[n - 1].x + 1);
    }
  }

  b200sht_disco_plan* pl = new b200sht_disco_plan();
  memset(static_cast<DiscoPlan*>(pl), 0, sizeof(DiscoPlan));
  pl->nlat_in = nlat_in; pl->nlon_in = nlon_in; pl->nlat_out = nlat_out; pl->nlon_out = nlon_out;
  pl->K = K; pl->Kp = Kp; pl->pscale = nlon_in / nlon_out; pl->nnz = nnz; pl->npts = (long long)npts;
  cudaError_t err = cudaSuccess;
  auto upload = [&](auto** dst, const auto& v) {
    using T = typename std::decay_t<decltype(v)>::value_type;
    const size_t b = std::max<size_t>(v.size(), 1) * sizeof(T);
    if (err == cudaSuccess) err = cudaMalloc(reinterpret_cast<void**>(dst), b);
    if (err == cudaSuccess && !v.empty()) err = cudaMemcpyAsync(*dst, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice, st);
    pl->bytes += b;
  };
  upload(&pl->d_fwd_rowptr, f_rowptr); upload(&pl->d_fwd_band, f_band); upload(&pl->d_fwd_pos, f_pos); upload(&pl->d_fwd_val, f_val);
  upload(&pl->d_adj_rowptr, a_rowptr); upload(&pl->d_adj_band, a_band); upload(&pl->d_adj_pos, a_pos); upload(&pl->d_adj_val, a_val);
  if (err == cudaSuccess) err = cudaStreamSynchronize(st);   // the host staging vectors go out of scope
  if (err != cudaSuccess) {
    set_error("disco_plan_create: %s", cudaGetErrorString(err));
    cudaFree(pl->d_fwd_rowptr); cudaFree(pl->d_fwd_band); cudaFree(pl->d_fwd_pos); cudaFree(pl->d_fwd_val);
    cudaFree(pl->d_adj_rowptr); cudaFree(pl->d_adj_band); cudaFree(pl->d_adj_pos); cudaFree(pl->d_adj_val);
    delete pl;
    return err == cudaErrorMemoryAllocation ? B200SHT_ERR_NOMEM : B200SHT_ERR_CUDA;
  }
  *out = pl;
  return B200SHT_OK;
}

int disco_plan_destroy(b200sht_disco_plan* pl) {
  if (!pl) return B200SHT_OK;
  cudaFree(pl->d_fwd_rowptr); cudaFree(pl->d_fwd_band); cudaFree(pl->d_fwd_pos); cudaFree(pl->d_fwd_val);
  cudaFree(pl->d_adj_rowptr); cudaFree(pl->d_adj_band); cudaFree(pl->d_adj_pos); cudaFree(pl->d_adj_val);
  delete pl;
  return B200SHT_OK;
}

long long disco_plan_query(const b200sht_disco_plan* pl, int what) {
  if (!pl) return -1;
  switch (what) {
    case 0: return pl->nlat_in;
    case 1: return pl->nlon_in;
    case 2: return pl->nlat_out;
    case 3: return pl->nlon_out;
    case 4: return pl->K;
    case 5: return pl->nnz;
    case 6: return pl->npts;
    case 7: return (long long)pl->bytes;
    case 8: return pl->pscale;
    default: return -1;
  }
}

// ------------------------------------------------------------------------------------------------------------------------- launches
template <int KP> struct DiscoFwdTag {};   // one cache of the shared-memory attribute per instantiation
struct DiscoAdjTag {};

template <int KP>
static int launch_forward(const DiscoFwdArgs& a0, cudaStream_t st) {
  constexpr int NP = KP <= 16 ? 4 : 2;
  DiscoFwdArgs a = a0;
  const int groups = ceil_div(a.nlon_out, NP);
  a.TPR = std::min(kDiscoThreads, round_up(groups, 32));
  a.R = std::max(1, std::min(kDiscoThreads / a.TPR, a.BC));
  while (a.R > 1 && (long long)a.R * a.nlon_in * 4 > kDiscoStageBytes) --a.R;
  a.SR = std::max(1, kDiscoStageBytes / (a.R * a.nlon_in * 4));
  const size_t smem = (size_t)kDiscoPC * KP * 4 + (size_t)kDiscoPC * sizeof(int2) + (size_t)a.R * a.SR * a.nlon_in * 4;
  B200_CHECK_CUDA((ensure_dynamic_smem<DiscoFwdTag<KP>>(disco_forward_kernel<KP, NP>, smem)));
  B200_REQUIRE(ceil_div(a.BC, a.R) <= 65535, "disco_forward: B*C = %d rows is too many for one launch", a.BC);
  dim3 grid(a.nlat_out, ceil_div(a.BC, a.R), ceil_div(a.nlon_out, a.TPR * NP));
  disco_forward_kernel<KP, NP><<<grid, a.R * a.TPR, smem, st>>>(a);
  B200_CHECK_LAUNCH();
  return B200SHT_OK;
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

int disco_forward(const b200sht_disco_plan* pl, const void* x, int dtype, int B, int C, float* X, cudaStream_t st) {
  B200_REQUIRE(pl && x && X, "disco_forward: null argument");
  B200_REQUIRE(dtype == B200SHT_F32 || dtype == B200SHT_BF16, "disco_forward: dtype %d is neither fp32 nor bf16", dtype);
  B200_REQUIRE(B > 0 && C > 0, "disco_forward: bad batch %d / channels %d", B, C);
  DiscoFwdArgs a;
  a.x = x; a.X = X; a.dtype = dtype; a.BC = B * C;
  a.nlat_in = pl->nlat_in; a.nlon_in = pl->nlon_in; a.nlat_out = pl->nlat_out; a.nlon_out = pl->nlon_out;
  a.K = pl->K; a.Kp = pl->Kp; a.pscale = pl->pscale;
  a.vec = aligned16(x) && pl->nlon_in % (dtype == B200SHT_F32 ? 4 : 8) == 0;
  a.rowptr = pl->d_fwd_rowptr; a.band = pl->d_fwd_band; a.pos = pl->d_fwd_pos; a.val = pl->d_fwd_val;
  for (int k0 = 0; k0 < pl->K; k0 += kDiscoMaxKC) {
    a.k0 = k0;
    a.KC = std::min(kDiscoMaxKC, pl->K - k0);
    int rc;
    switch (round_up(a.KC, 4)) {
      case 4: rc = launch_forward<4>(a, st); break;
      case 8: rc = launch_forward<8>(a, st); break;
      case 12: rc = launch_forward<12>(a, st); break;
      case 16: rc = launch_forward<16>(a, st); break;
      case 20: rc = launch_forward<20>(a, st); break;
      case 24: rc = launch_forward<24>(a, st); break;
      case 28: rc = launch_forward<28>(a, st); break;
      default: rc = launch_forward<32>(a, st); break;
    }
    if (rc) return rc;
  }
  return B200SHT_OK;
}

int disco_adjoint(const b200sht_disco_plan* pl, const float* dX, void* dx, int dtype, int B, int C, cudaStream_t st) {
  B200_REQUIRE(pl && dX && dx, "disco_adjoint: null argument");
  B200_REQUIRE(dtype == B200SHT_F32 || dtype == B200SHT_BF16, "disco_adjoint: dtype %d is neither fp32 nor bf16", dtype);
  B200_REQUIRE(B > 0 && C > 0, "disco_adjoint: bad batch %d / channels %d", B, C);
  DiscoAdjArgs a;
  a.dX = dX; a.dx = dx; a.dtype = dtype; a.BC = B * C;
  a.nlat_in = pl->nlat_in; a.nlon_in = pl->nlon_in; a.nlat_out = pl->nlat_out; a.nlon_out = pl->nlon_out;
  a.K = pl->K; a.Kp = pl->Kp; a.pscale = pl->pscale;
  a.vec = aligned16(dX) && pl->nlon_out % 4 == 0;
  a.rowptr = pl->d_adj_rowptr; a.band = pl->d_adj_band; a.pos = pl->d_adj_pos; a.val = pl->d_adj_val;
  a.TPJ = std::min(kDiscoThreads, round_up(ceil_div(a.nlon_in, kDiscoNJ), 32));
  a.R = std::max(1, std::min(kDiscoThreads / a.TPJ, a.BC));
  const int row_bytes = a.nlon_out * 4;
  while (a.R > 1 && (long long)a.R * row_bytes > kDiscoStageBytes) --a.R;
  a.KC = std::max(1, std::min({a.K, kDiscoMaxKC, kDiscoStageBytes / (a.R * row_bytes)}));
  a.ST = std::max(1, kDiscoStageBytes / (a.R * a.KC * row_bytes));
  const size_t smem = (size_t)kDiscoPC * kDiscoMaxKC * 4 + (size_t)kDiscoPC * sizeof(int4) + (size_t)a.R * a.KC * a.ST * row_bytes;
  B200_CHECK_CUDA((ensure_dynamic_smem<DiscoAdjTag>(disco_adjoint_kernel, smem)));
  B200_REQUIRE(ceil_div(a.BC, a.R) <= 65535, "disco_adjoint: B*C = %d rows is too many for one launch", a.BC);
  dim3 grid(a.nlat_in, ceil_div(a.BC, a.R), ceil_div(a.nlon_in, a.TPJ * kDiscoNJ));
  disco_adjoint_kernel<<<grid, a.R * a.TPJ, smem, st>>>(a);
  B200_CHECK_LAUNCH();
  return B200SHT_OK;
}

}  // namespace b200sht
