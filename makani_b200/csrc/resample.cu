// Bilinear resampling on the sphere (torch_harmonics.ResampleS2, mode "bilinear") and its exact adjoint.
//
//   forward  y[b,t,p] = lerp(lerp(X[b,a,l], X[b,a,r], wp), lerp(X[b,a+1,l], X[b,a+1,r], wp), wt)      a = lat_idx[t], wt = lat_w[t],
//                                                                                                 l, r, wp = lon_left[p], lon_right[p], lon_w[p]
//   adjoint  dx = R^T dy
//
// X is the input with the pole pseudo-rows when the plan expands the poles: expanded row 0 is the longitude mean of input row 0, expanded row
// nlat_in + 1 the mean of row nlat_in - 1, and expanded row e of the rest is input row e - 1.  Without expansion X is the input itself.
// Forward: one CTA per (output row t, chunk of PC planes).  A warp stages each of the <= 2 referenced input rows of a plane in shared memory
// with 16-byte loads (scalar head and tail where a row is not 16-byte aligned, i.e. nlon_in % 4 != 0) and reduces a pole row to its mean; then
// every thread evaluates 4 consecutive outputs from the longitude tables (read-only path) and writes them with one float4 store.
// Adjoint: one CTA per (input row i, chunk of planes).  The host builds two CSR lists: by expanded input row, the (t, weight) pairs of the output
// rows that reference it, and by input column, the (p, weight) pairs of the output columns that reference it.  The CTA sums the weighted dy rows
// of row i into shared memory z[p] (t ascending), then gathers dx[j] = sum over the column list of weight * z[p] (p ascending).  The CTAs of rows
// 0 and nlat_in - 1 of an expanded plan add the pole term uniformly: (1 / nlon_in) sum over the rows referencing the pseudo-row of w sum_p dy[t, p]
// (the longitude weights of every output column sum to 1).  Every element is summed by one thread or one warp in a fixed order: no atomics,
// and the results are bit-identical run to run.
#include "common.cuh"
#include <algorithm>
#include <cmath>
#include <type_traits>
#include <vector>

namespace b200sht {

struct ResamplePlan {
  int nlat_in, nlon_in, nlat_out, nlon_out, expand;
  int* d_lat_idx;      // [nlat_out] expanded row a of output row t
  float* d_lat_w;      // [nlat_out]
  int* d_lon_l;        // [nlon_out]
  int* d_lon_r;        // [nlon_out]
  float* d_lon_w;      // [nlon_out]
  int* d_row_ptr;      // [nexp + 1] CSR by expanded input row
  int* d_row_t;        // [2 nlat_out] output row
  float* d_row_w;      // [2 nlat_out] 1 - wt (row a) or wt (row a + 1)
  int* d_col_ptr;      // [nlon_in + 1] CSR by input column
  int* d_col_p;        // [2 nlon_out] output column
  float* d_col_w;      // [2 nlon_out] 1 - wp (column l) or wp (column r)
  size_t bytes;
};

}  // namespace b200sht

struct b200sht_resample_plan : public b200sht::ResamplePlan {};

namespace b200sht {

constexpr int kResThreads = 256;
constexpr int kResMaxPC = 8;                  // planes per CTA
constexpr int kResStageBytes = 64 * 1024;     // staged input rows (forward) or z rows (adjoint)

struct ResampleFwdArgs {
  const float* x; float* y; int planes, PC, vec;
  int nlat_in, nlon_in, nlat_out, nlon_out, expand;
  const int* lat_idx; const float* lat_w; const int* lon_l; const int* lon_r; const float* lon_w;
};

struct ResampleAdjArgs {
  const float* dy; float* dx; int planes, PC, vec_dy, vec_dx;
  int nlat_in, nlon_in, nlat_out, nlon_out, expand;
  const int* row_ptr; const int* row_t; const float* row_w; const int* col_ptr; const int* col_p; const float* col_w;
};

// torch.lerp's formulation: exact at w = 0 and w = 1, and lerp(a, a, w) = a
__device__ __forceinline__ float lerp_f(float a, float b, float w) {
  const float d = b - a;
  return w < 0.5f ? fmaf(w, d, a) : fmaf(-d, 1.f - w, b);
}

// one warp copies n floats from global to shared memory: 16-byte loads, scalar head and tail around the 16-byte aligned body
__device__ __forceinline__ void stage_row_warp(float* dst, const float* src, int n, int lane) {
  const int h = min(n, (int)(((16u - (unsigned)(reinterpret_cast<uintptr_t>(src) & 15u)) & 15u) >> 2));
  const int nb = (n - h) >> 2;
  if (lane < h) dst[lane] = __ldg(src + lane);
  const float4* s4 = reinterpret_cast<const float4*>(src + h);
  if ((reinterpret_cast<uintptr_t>(dst + h) & 15u) == 0) {
    float4* d4 = reinterpret_cast<float4*>(dst + h);
    for (int e = lane; e < nb; e += 32) d4[e] = __ldg(s4 + e);
  } else {
    for (int e = lane; e < nb; e += 32) {
      const float4 v = __ldg(s4 + e);
      float* d = dst + h + 4 * e;
      d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
    }
  }
  for (int e = h + 4 * nb + lane; e < n; e += 32) dst[e] = __ldg(src + e);
}

__device__ __forceinline__ float warp_sum(float s) {
#pragma unroll
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  return s;
}

__global__ void __launch_bounds__(kResThreads) resample_forward_kernel(ResampleFwdArgs a) {
  extern __shared__ __align__(16) unsigned char smem[];
  float* rows = reinterpret_cast<float*>(smem);              // [PC][2][nlon_in]
  float* pm = rows + (size_t)a.PC * 2 * a.nlon_in;          // [PC][2] mean of a staged pole row

  const int t = blockIdx.x;
  const int p0 = blockIdx.y * a.PC;
  const int np = min(a.PC, a.planes - p0);
  const int e0 = __ldg(a.lat_idx + t);
  const float wt = __ldg(a.lat_w + t);
  const bool pole0 = a.expand && e0 == 0, pole1 = a.expand && e0 + 1 == a.nlat_in + 1;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int k = warp; k < 2 * np; k += nw) {
    const int e = e0 + (k & 1);
    const int row = a.expand ? min(max(e - 1, 0), a.nlat_in - 1) : e;
    float* dst = rows + (size_t)k * a.nlon_in;
    stage_row_warp(dst, a.x + ((size_t)(p0 + (k >> 1)) * a.nlat_in + row) * a.nlon_in, a.nlon_in, lane);
    if ((k & 1) ? pole1 : pole0) {
      __syncwarp();
      float s = 0.f;
      for (int j = lane; j < a.nlon_in; j += 32) s += dst[j];
      s = warp_sum(s);
      if (lane == 0) pm[k] = s / (float)a.nlon_in;
    }
  }
  __syncthreads();

  auto value = [&](int pc, int l, int r, float wp) {
    const float* r0 = rows + (size_t)(2 * pc) * a.nlon_in;
    const float* r1 = r0 + a.nlon_in;
    const float v0 = pole0 ? pm[2 * pc] : lerp_f(r0[l], r0[r], wp);
    const float v1 = pole1 ? pm[2 * pc + 1] : lerp_f(r1[l], r1[r], wp);
    return lerp_f(v0, v1, wt);
  };
  if (a.vec) {
    const int nq = a.nlon_out >> 2;
    for (int e = threadIdx.x; e < np * nq; e += blockDim.x) {
      const int pc = e / nq, q = e - pc * nq;
      const int4 L = __ldg(reinterpret_cast<const int4*>(a.lon_l) + q);
      const int4 R = __ldg(reinterpret_cast<const int4*>(a.lon_r) + q);
      const float4 W = __ldg(reinterpret_cast<const float4*>(a.lon_w) + q);
      const float4 v = make_float4(value(pc, L.x, R.x, W.x), value(pc, L.y, R.y, W.y), value(pc, L.z, R.z, W.z), value(pc, L.w, R.w, W.w));
      reinterpret_cast<float4*>(a.y + ((size_t)(p0 + pc) * a.nlat_out + t) * a.nlon_out)[q] = v;
    }
  } else {
    for (int e = threadIdx.x; e < np * a.nlon_out; e += blockDim.x) {
      const int pc = e / a.nlon_out, p = e - pc * a.nlon_out;
      a.y[((size_t)(p0 + pc) * a.nlat_out + t) * a.nlon_out + p] = value(pc, __ldg(a.lon_l + p), __ldg(a.lon_r + p), __ldg(a.lon_w + p));
    }
  }
}

__global__ void __launch_bounds__(kResThreads, 4) resample_adjoint_kernel(ResampleAdjArgs a) {
  extern __shared__ __align__(16) unsigned char smem[];
  float* z = reinterpret_cast<float*>(smem);                 // [PC][nlon_out] weighted sum of the dy rows that reference row i
  float* pole = z + (size_t)a.PC * a.nlon_out;               // [PC] pole term of row i

  const int i = blockIdx.x;
  const int p0 = blockIdx.y * a.PC;
  const int np = min(a.PC, a.planes - p0);
  const int e = i + a.expand;
  const int ka = __ldg(a.row_ptr + e), kb = __ldg(a.row_ptr + e + 1);
  const size_t plane_out = (size_t)a.nlat_out * a.nlon_out;

  // z[pc][p] = sum_k w_k dy[pc, t_k, p], k ascending (t ascending)
  if (a.vec_dy) {
    const int nq = a.nlon_out >> 2;
    for (int n = threadIdx.x; n < np * nq; n += blockDim.x) {
      const int pc = n / nq, q = n - pc * nq;
      const float* d = a.dy + (size_t)(p0 + pc) * plane_out;
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int k = ka; k < kb; ++k) {
        const float w = __ldg(a.row_w + k);
        const float4 v = __ldg(reinterpret_cast<const float4*>(d + (size_t)__ldg(a.row_t + k) * a.nlon_out) + q);
        acc.x = fmaf(w, v.x, acc.x); acc.y = fmaf(w, v.y, acc.y); acc.z = fmaf(w, v.z, acc.z); acc.w = fmaf(w, v.w, acc.w);
      }
      reinterpret_cast<float4*>(z + (size_t)pc * a.nlon_out)[q] = acc;
    }
  } else {
    for (int n = threadIdx.x; n < np * a.nlon_out; n += blockDim.x) {
      const int pc = n / a.nlon_out, p = n - pc * a.nlon_out;
      const float* d = a.dy + (size_t)(p0 + pc) * plane_out + p;
      float acc = 0.f;
      for (int k = ka; k < kb; ++k) acc = fmaf(__ldg(a.row_w + k), __ldg(d + (size_t)__ldg(a.row_t + k) * a.nlon_out), acc);
      z[(size_t)pc * a.nlon_out + p] = acc;
    }
  }
  // pole term: one warp per plane, lanes over p, inner sum over the referencing rows, then a butterfly over the lanes
  const bool north = a.expand && i == 0, south = a.expand && i == a.nlat_in - 1;
  if (north || south) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    for (int pc = warp; pc < np; pc += nw) {
      const float* d = a.dy + (size_t)(p0 + pc) * plane_out;
      float s = 0.f;
      auto add_rows = [&](int ep) {
        const int qa = __ldg(a.row_ptr + ep), qb = __ldg(a.row_ptr + ep + 1);
        for (int p = lane; p < a.nlon_out; p += 32) {
          float c = 0.f;
          for (int k = qa; k < qb; ++k) c = fmaf(__ldg(a.row_w + k), __ldg(d + (size_t)__ldg(a.row_t + k) * a.nlon_out + p), c);
          s += c;
        }
      };
      if (north) add_rows(0);
      if (south) add_rows(a.nlat_in + 1);
      s = warp_sum(s);
      if (lane == 0) pole[pc] = s / (float)a.nlon_in;
    }
  } else if (threadIdx.x < np) {
    pole[threadIdx.x] = 0.f;
  }
  __syncthreads();

  // dx[pc][j] = sum over the column list of j of w * z[pc][p] (p ascending), + the pole term
  auto gather = [&](int pc, int j) {
    const float* zr = z + (size_t)pc * a.nlon_out;
    const int ca = __ldg(a.col_ptr + j), cb = __ldg(a.col_ptr + j + 1);
    float acc = 0.f;
    for (int k = ca; k < cb; ++k) acc = fmaf(__ldg(a.col_w + k), zr[__ldg(a.col_p + k)], acc);
    return acc + pole[pc];
  };
  if (a.vec_dx) {
    const int nq = a.nlon_in >> 2;
    for (int n = threadIdx.x; n < np * nq; n += blockDim.x) {
      const int pc = n / nq, q = n - pc * nq;
      const float4 v = make_float4(gather(pc, 4 * q), gather(pc, 4 * q + 1), gather(pc, 4 * q + 2), gather(pc, 4 * q + 3));
      reinterpret_cast<float4*>(a.dx + ((size_t)(p0 + pc) * a.nlat_in + i) * a.nlon_in)[q] = v;
    }
  } else {
    for (int n = threadIdx.x; n < np * a.nlon_in; n += blockDim.x) {
      const int pc = n / a.nlon_in, j = n - pc * a.nlon_in;
      a.dx[((size_t)(p0 + pc) * a.nlat_in + i) * a.nlon_in + j] = gather(pc, j);
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------------- plan
static void free_plan(ResamplePlan* pl) {
  cudaFree(pl->d_lat_idx); cudaFree(pl->d_lat_w); cudaFree(pl->d_lon_l); cudaFree(pl->d_lon_r); cudaFree(pl->d_lon_w);
  cudaFree(pl->d_row_ptr); cudaFree(pl->d_row_t); cudaFree(pl->d_row_w); cudaFree(pl->d_col_ptr); cudaFree(pl->d_col_p); cudaFree(pl->d_col_w);
}

// entries (key[n], val[n], w[n]) -> CSR over nkeys keys; the entries of a key keep their input order
static void build_csr(int nkeys, const std::vector<int>& key, const std::vector<int>& val, const std::vector<float>& w, std::vector<int>& ptr,
                      std::vector<int>& out_val, std::vector<float>& out_w) {
  ptr.assign(nkeys + 1, 0);
  for (int k : key) ++ptr[k + 1];
  for (int k = 0; k < nkeys; ++k) ptr[k + 1] += ptr[k];
  std::vector<int> fill(ptr.begin(), ptr.end() - 1);
  out_val.resize(key.size());
  out_w.resize(key.size());
  for (size_t n = 0; n < key.size(); ++n) {
    const int d = fill[key[n]]++;
    out_val[d] = val[n];
    out_w[d] = w[n];
  }
}

int resample_plan_create(b200sht_resample_plan** out, int nlat_in, int nlon_in, int nlat_out, int nlon_out, int expand_poles, const int* lat_idx,
                         const float* lat_w, const int* lon_left, const int* lon_right, const float* lon_w, cudaStream_t st) {
  B200_REQUIRE(out, "resample_plan_create: null plan pointer");
  *out = nullptr;
  B200_REQUIRE(nlat_in > 0 && nlon_in > 0 && nlat_out > 0 && nlon_out > 0, "resample_plan_create: bad sizes (nlat_in %d nlon_in %d nlat_out %d nlon_out %d)",
               nlat_in, nlon_in, nlat_out, nlon_out);
  B200_REQUIRE(lat_idx && lat_w && lon_left && lon_right && lon_w, "resample_plan_create: null table");
  if ((long long)nlon_in * 2 * 4 > kResStageBytes || (long long)nlon_out * 4 > kResStageBytes) {
    set_error("resample_plan_create: nlon_in %d / nlon_out %d exceed the staged row lengths (%d / %d floats)", nlon_in, nlon_out, kResStageBytes / 8,
              kResStageBytes / 4);
    return B200SHT_ERR_UNSUPPORTED;
  }
  const int expand = expand_poles ? 1 : 0;
  const int nexp = nlat_in + 2 * expand;
  for (int t = 0; t < nlat_out; ++t)
    B200_REQUIRE(lat_idx[t] >= 0 && lat_idx[t] + 1 < nexp && std::isfinite(lat_w[t]), "resample_plan_create: latitude entry %d (row %d, w %g) out of range",
                 t, lat_idx[t], (double)lat_w[t]);
  for (int p = 0; p < nlon_out; ++p)
    B200_REQUIRE(lon_left[p] >= 0 && lon_left[p] < nlon_in && lon_right[p] >= 0 && lon_right[p] < nlon_in && std::isfinite(lon_w[p]),
                 "resample_plan_create: longitude entry %d (%d, %d, w %g) out of range", p, lon_left[p], lon_right[p], (double)lon_w[p]);

  // the adjoint's lists: (1 - w) in fp64, rounded once
  std::vector<int> key, val, row_ptr, row_t, col_ptr, col_p;
  std::vector<float> w, row_w, col_w;
  for (int t = 0; t < nlat_out; ++t) {
    key.push_back(lat_idx[t]); val.push_back(t); w.push_back((float)(1.0 - (double)lat_w[t]));
    key.push_back(lat_idx[t] + 1); val.push_back(t); w.push_back(lat_w[t]);
  }
  build_csr(nexp, key, val, w, row_ptr, row_t, row_w);
  key.clear(); val.clear(); w.clear();
  for (int p = 0; p < nlon_out; ++p) {
    key.push_back(lon_left[p]); val.push_back(p); w.push_back((float)(1.0 - (double)lon_w[p]));
    key.push_back(lon_right[p]); val.push_back(p); w.push_back(lon_w[p]);
  }
  build_csr(nlon_in, key, val, w, col_ptr, col_p, col_w);

  b200sht_resample_plan* pl = new b200sht_resample_plan();
  memset(static_cast<ResamplePlan*>(pl), 0, sizeof(ResamplePlan));
  pl->nlat_in = nlat_in; pl->nlon_in = nlon_in; pl->nlat_out = nlat_out; pl->nlon_out = nlon_out; pl->expand = expand;
  cudaError_t err = cudaSuccess;
  auto upload = [&](auto** dst, const auto* src, size_t n) {
    using T = std::remove_cv_t<std::remove_reference_t<decltype(*src)>>;
    const size_t b = std::max<size_t>(n, 1) * sizeof(T);
    if (err == cudaSuccess) err = cudaMalloc(reinterpret_cast<void**>(dst), b);
    if (err == cudaSuccess && n) err = cudaMemcpyAsync(*dst, src, n * sizeof(T), cudaMemcpyHostToDevice, st);
    pl->bytes += b;
  };
  upload(&pl->d_lat_idx, lat_idx, nlat_out); upload(&pl->d_lat_w, lat_w, nlat_out);
  upload(&pl->d_lon_l, lon_left, nlon_out); upload(&pl->d_lon_r, lon_right, nlon_out); upload(&pl->d_lon_w, lon_w, nlon_out);
  upload(&pl->d_row_ptr, row_ptr.data(), row_ptr.size()); upload(&pl->d_row_t, row_t.data(), row_t.size());
  upload(&pl->d_row_w, row_w.data(), row_w.size());
  upload(&pl->d_col_ptr, col_ptr.data(), col_ptr.size()); upload(&pl->d_col_p, col_p.data(), col_p.size());
  upload(&pl->d_col_w, col_w.data(), col_w.size());
  if (err == cudaSuccess) err = cudaStreamSynchronize(st);   // the host tables and staging vectors go out of scope
  if (err != cudaSuccess) {
    set_error("resample_plan_create: %s", cudaGetErrorString(err));
    free_plan(pl);
    delete pl;
    return err == cudaErrorMemoryAllocation ? B200SHT_ERR_NOMEM : B200SHT_ERR_CUDA;
  }
  *out = pl;
  return B200SHT_OK;
}

int resample_plan_destroy(b200sht_resample_plan* pl) {
  if (!pl) return B200SHT_OK;
  free_plan(pl);
  delete pl;
  return B200SHT_OK;
}

long long resample_plan_query(const b200sht_resample_plan* pl, int what) {
  if (!pl) return -1;
  switch (what) {
    case 0: return pl->nlat_in;
    case 1: return pl->nlon_in;
    case 2: return pl->nlat_out;
    case 3: return pl->nlon_out;
    case 4: return pl->expand;
    case 5: return (long long)pl->bytes;
    default: return -1;
  }
}

// ------------------------------------------------------------------------------------------------------------------------- launches
struct ResampleFwdTag {};   // one cache of the shared-memory attribute per kernel
struct ResampleAdjTag {};

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

static int planes_per_cta(int planes, int row_bytes) { return std::max(1, std::min({kResMaxPC, planes, kResStageBytes / row_bytes})); }

int resample_forward(const b200sht_resample_plan* pl, const float* x, float* y, int planes, cudaStream_t st) {
  B200_REQUIRE(pl && x && y, "resample_forward: null argument");
  B200_REQUIRE(planes > 0, "resample_forward: bad plane count %d", planes);
  ResampleFwdArgs a;
  a.x = x; a.y = y; a.planes = planes;
  a.nlat_in = pl->nlat_in; a.nlon_in = pl->nlon_in; a.nlat_out = pl->nlat_out; a.nlon_out = pl->nlon_out; a.expand = pl->expand;
  a.lat_idx = pl->d_lat_idx; a.lat_w = pl->d_lat_w; a.lon_l = pl->d_lon_l; a.lon_r = pl->d_lon_r; a.lon_w = pl->d_lon_w;
  a.vec = aligned16(y) && pl->nlon_out % 4 == 0;
  a.PC = planes_per_cta(planes, 2 * pl->nlon_in * 4);
  B200_REQUIRE(ceil_div(planes, a.PC) <= 65535, "resample_forward: %d planes is too many for one launch", planes);
  const size_t smem = (size_t)a.PC * 2 * pl->nlon_in * 4 + (size_t)a.PC * 2 * 4;
  B200_CHECK_CUDA((ensure_dynamic_smem<ResampleFwdTag>(resample_forward_kernel, smem)));
  dim3 grid(pl->nlat_out, ceil_div(planes, a.PC));
  resample_forward_kernel<<<grid, kResThreads, smem, st>>>(a);
  B200_CHECK_LAUNCH();
  return B200SHT_OK;
}

int resample_adjoint(const b200sht_resample_plan* pl, const float* dy, float* dx, int planes, cudaStream_t st) {
  B200_REQUIRE(pl && dy && dx, "resample_adjoint: null argument");
  B200_REQUIRE(planes > 0, "resample_adjoint: bad plane count %d", planes);
  ResampleAdjArgs a;
  a.dy = dy; a.dx = dx; a.planes = planes;
  a.nlat_in = pl->nlat_in; a.nlon_in = pl->nlon_in; a.nlat_out = pl->nlat_out; a.nlon_out = pl->nlon_out; a.expand = pl->expand;
  a.row_ptr = pl->d_row_ptr; a.row_t = pl->d_row_t; a.row_w = pl->d_row_w; a.col_ptr = pl->d_col_ptr; a.col_p = pl->d_col_p; a.col_w = pl->d_col_w;
  a.vec_dy = aligned16(dy) && pl->nlon_out % 4 == 0;
  a.vec_dx = aligned16(dx) && pl->nlon_in % 4 == 0;
  a.PC = planes_per_cta(planes, pl->nlon_out * 4);
  B200_REQUIRE(ceil_div(planes, a.PC) <= 65535, "resample_adjoint: %d planes is too many for one launch", planes);
  const size_t smem = (size_t)a.PC * pl->nlon_out * 4 + (size_t)a.PC * 4;
  B200_CHECK_CUDA((ensure_dynamic_smem<ResampleAdjTag>(resample_adjoint_kernel, smem)));
  dim3 grid(pl->nlat_in, ceil_div(planes, a.PC));
  resample_adjoint_kernel<<<grid, kResThreads, smem, st>>>(a);
  B200_CHECK_LAUNCH();
  return B200SHT_OK;
}

}  // namespace b200sht
