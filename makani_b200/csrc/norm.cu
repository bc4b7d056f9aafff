// Pointwise tail of the SFNO block around the spectral filter (SURVEY row N2; reference: torch.nn.InstanceNorm2d(affine, eps 1e-6) + nn.GELU as
// built at makani/models/networks/sfnonet.py:618-620 and applied at :385-406, bias + GELU of the 1x1-convolution MLP / encoder / decoder,
// makani/models/common/layers.py:537-760).  At 721 x 1440 x 384 one activation is 0.8 GB in bf16: these layers are pure HBM traffic, and PyTorch's
// instance norm (batch-norm kernels with one block per channel) needs 15.6 ms of a 77 ms model step for them.
//
//   instance norm (+ GELU), rows = (b, c), n = H * W contiguous elements per row, every row split over `splits` CTAs:
//     forward : stats   (sum, sum of squares) of x - x[row start] per (row, pair of splits)     read x
//                       in fp64: x - pivot is exact, so a pivot far from the row mean (an outlier at x[row, 0]) costs no accuracy.  One CTA
//                       of 2 x 256 threads per pair of splits: its two fp64 sums, as (hi, lo) float pairs, fill the workspace slots of two
//                       splits; a row of one CTA writes its (mean, rstd) itself.
//               apply   y = [gelu]((x - mean) * rstd * gamma[c] + beta[c])                       read x, write y
//     backward: reduce  partial S1 = sum g, S2 = sum g * xhat   (g = dy, or dy * gelu'(z))      read x, dy
//               apply   dx = rstd * gamma[c] * (g - S1 / n - xhat * S2 / n)                      read x, dy, write dx
//     dgamma[c] = sum_b S2, dbeta[c] = sum_b S1 are formed by the caller from the per-row sums (tiny).
//   bias + GELU: y = gelu(x + bias[c]);  dx = dy * gelu'(x + bias[c]), per-(row, split) partial sums of dx for dbias.
// All other arithmetic in fp32, activations float or bf16, 16-byte vector accesses when the row length allows it.
#include <type_traits>

#include "common.cuh"

namespace b200sht {

constexpr int kNormThreads = 256;
constexpr int kNormMaxSplits = 64;

__device__ __forceinline__ float gelu_f(float z) { return 0.5f * z * (1.f + erff(z * 0.70710678118654752440f)); }
__device__ __forceinline__ float gelu_grad_f(float z) {
  return 0.5f * (1.f + erff(z * 0.70710678118654752440f)) + z * 0.39894228040143267794f * __expf(-0.5f * z * z);
}

template <typename T> __device__ __forceinline__ float ldf(const T* p, long long i);
template <> __device__ __forceinline__ float ldf<float>(const float* p, long long i) { return p[i]; }
template <> __device__ __forceinline__ float ldf<__nv_bfloat16>(const __nv_bfloat16* p, long long i) { return __bfloat162float(p[i]); }
template <typename T> __device__ __forceinline__ void stf(T* p, long long i, float v);
template <> __device__ __forceinline__ void stf<float>(float* p, long long i, float v) { p[i] = v; }
template <> __device__ __forceinline__ void stf<__nv_bfloat16>(__nv_bfloat16* p, long long i, float v) { p[i] = __float2bfloat16_rn(v); }

// 16-byte packets: 4 floats or 8 bf16
template <typename T> struct Pack;
template <> struct Pack<float> {
  static constexpr int kN = 4;
  float4 raw;
  __device__ __forceinline__ void load(const float* p) { raw = *reinterpret_cast<const float4*>(p); }
  __device__ __forceinline__ void store(float* p) const { *reinterpret_cast<float4*>(p) = raw; }
  __device__ __forceinline__ float get(int i) const { return i == 0 ? raw.x : i == 1 ? raw.y : i == 2 ? raw.z : raw.w; }
  __device__ __forceinline__ void set(int i, float v) { if (i == 0) raw.x = v; else if (i == 1) raw.y = v; else if (i == 2) raw.z = v; else raw.w = v; }
};
template <> struct Pack<__nv_bfloat16> {
  static constexpr int kN = 8;
  uint4 raw;
  __device__ __forceinline__ void load(const __nv_bfloat16* p) { raw = *reinterpret_cast<const uint4*>(p); }
  __device__ __forceinline__ void store(__nv_bfloat16* p) const { *reinterpret_cast<uint4*>(p) = raw; }
  __device__ __forceinline__ float get(int i) const {
    const uint32_t w = (i >> 1) == 0 ? raw.x : (i >> 1) == 1 ? raw.y : (i >> 1) == 2 ? raw.z : raw.w;
    return __uint_as_float((i & 1) ? (w & 0xffff0000u) : (w << 16));
  }
  __device__ __forceinline__ void set(int i, float v) {
    const uint32_t h = (uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(v));
    uint32_t* w = (i >> 1) == 0 ? &raw.x : (i >> 1) == 1 ? &raw.y : (i >> 1) == 2 ? &raw.z : &raw.w;
    *w = (i & 1) ? ((*w & 0x0000ffffu) | (h << 16)) : ((*w & 0xffff0000u) | h);
  }
};

struct NormArgs {
  const void* x;
  const void* dy;
  void* out;           // y (forward) / dx (backward)
  const float* gamma;  // [C] or null (1)
  const float* beta;   // [C] or null (0): instance-norm shift, or the bias of bias + GELU
  const float* stats;  // [rows][2] mean, rstd
  const float* sums;   // [rows][2] S1, S2 (backward apply)
  float* partial;      // [rows][splits][2]; forward statistics: [rows][splits][4], two fp64 sums each stored as a (hi, lo) float pair
  float* stats_out;    // forward statistics of a one-CTA row: [rows][2] mean, rstd
  long long n;         // elements per row
  long long chunk;     // elements per split (a multiple of 8); the last split runs to n
  int rows, C, splits, gelu;
  float eps;
};

// two block-wide sums (blockDim.x == NT); result valid in thread 0
template <int NT, typename A>
__device__ __forceinline__ void block_sum2(A& a, A& b) {
  __shared__ A sa[NT / 32], sb[NT / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { a += __shfl_xor_sync(0xffffffffu, a, o); b += __shfl_xor_sync(0xffffffffu, b, o); }
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) { sa[w] = a; sb[w] = b; }
  __syncthreads();
  if (w == 0) {
    a = l < NT / 32 ? sa[l] : A(0);
    b = l < NT / 32 ? sb[l] : A(0);
#pragma unroll
    for (int o = NT / 64; o > 0; o >>= 1) { a += __shfl_xor_sync(0xffffffffu, a, o); b += __shfl_xor_sync(0xffffffffu, b, o); }
  }
}

// (mean, rstd) of a row from the fp64 sums of x - pivot over its n elements
__device__ __forceinline__ void store_stats(float* out, double pivot, double s0, double s1, long long n, float eps) {
  const double md = s0 / (double)n;
  double var = s1 / (double)n - md * md;
  if (var < 0.0) var = 0.0;
  out[0] = (float)(pivot + md);
  out[1] = (float)(1.0 / sqrt(var + (double)eps));
}

// What a kernel does with one element.  MODE 0: forward statistics, 1: forward apply, 2: backward reduce, 3: backward apply,
// 4: bias + GELU forward, 5: bias + GELU backward (also accumulates sum dx).  NT threads per CTA.
template <typename T, int MODE, bool VEC, int NT>
__global__ void __launch_bounds__(NT) norm_kernel(const NormArgs a) {
  const int r = blockIdx.y, s = blockIdx.x;
  const long long beg = (long long)s * a.chunk, end = (s == a.splits - 1 || beg + a.chunk > a.n) ? a.n : beg + a.chunk;
  const T* x = static_cast<const T*>(a.x) + (size_t)r * a.n;
  const T* dy = static_cast<const T*>(a.dy) + (size_t)r * a.n;
  T* out = static_cast<T*>(a.out) + (size_t)r * a.n;
  const int c = r % a.C;
  const float gamma = a.gamma ? a.gamma[c] : 1.f, beta = a.beta ? a.beta[c] : 0.f;
  float mean = 0.f, rstd = 1.f, m1 = 0.f, m2 = 0.f;
  double pivot = 0.0;
  if (MODE == 0) pivot = (double)ldf<T>(x, 0);
  if (MODE == 1 || MODE == 2 || MODE == 3) { mean = a.stats[2 * r]; rstd = a.stats[2 * r + 1]; }
  if (MODE == 3) { m1 = a.sums[2 * r] / (float)a.n; m2 = a.sums[2 * r + 1] / (float)a.n; }
  const float gs = gamma * rstd;
  using Acc = typename std::conditional<MODE == 0, double, float>::type;
  Acc acc0 = 0, acc1 = 0, odd0 = 0, odd1 = 0;   // odd*: a second fp64 chain for the odd elements of a packet (half the dependent latency)

  auto element = [&](float xv, float dv, float& ov, int j) {
    if (MODE == 0) {
      const double d = (double)xv - pivot;
      if (j & 1) { odd0 += d; odd1 = fma(d, d, odd1); }
      else { acc0 += d; acc1 = fma(d, d, acc1); }
    } else if (MODE == 1) {
      const float z = fmaf((xv - mean) * rstd, gamma, beta);
      ov = a.gelu ? gelu_f(z) : z;
    } else if (MODE == 2 || MODE == 3) {
      const float xh = (xv - mean) * rstd;
      const float g = a.gelu ? dv * gelu_grad_f(fmaf(xh, gamma, beta)) : dv;
      if (MODE == 2) { acc0 += g; acc1 = fmaf(g, xh, acc1); }
      else ov = gs * (g - m1 - xh * m2);
    } else if (MODE == 4) {
      ov = gelu_f(xv + beta);
    } else {
      ov = dv * gelu_grad_f(xv + beta);
      acc0 += ov;
    }
  };
  constexpr bool kNeedDy = (MODE == 2 || MODE == 3 || MODE == 5), kWrites = (MODE == 1 || MODE == 3 || MODE == 4 || MODE == 5);
  if (VEC) {
    constexpr int kN = Pack<T>::kN;
    constexpr long long kStride = (long long)NT * kN;
    long long i = beg + (long long)threadIdx.x * kN;   // beg, n multiples of kN: whole packets
    // two packets per tensor in flight per thread (first measurement of the one-packet loop: 45-50 % of HBM, latency bound at 5 CTAs per SM)
    for (; i + kStride < end; i += 2 * kStride) {
      Pack<T> px0, px1, pd0, pd1, po0, po1;
      px0.load(x + i);
      px1.load(x + i + kStride);
      if (kNeedDy) { pd0.load(dy + i); pd1.load(dy + i + kStride); }
#pragma unroll
      for (int j = 0; j < kN; ++j) {
        float ov = 0.f;
        element(px0.get(j), kNeedDy ? pd0.get(j) : 0.f, ov, j);
        if (kWrites) po0.set(j, ov);
      }
#pragma unroll
      for (int j = 0; j < kN; ++j) {
        float ov = 0.f;
        element(px1.get(j), kNeedDy ? pd1.get(j) : 0.f, ov, j);
        if (kWrites) po1.set(j, ov);
      }
      if (kWrites) { po0.store(out + i); po1.store(out + i + kStride); }
    }
    for (; i < end; i += kStride) {
      Pack<T> px, pd, po;
      px.load(x + i);
      if (kNeedDy) pd.load(dy + i);
#pragma unroll
      for (int j = 0; j < kN; ++j) {
        float ov = 0.f;
        element(px.get(j), kNeedDy ? pd.get(j) : 0.f, ov, j);
        if (kWrites) po.set(j, ov);
      }
      if (kWrites) po.store(out + i);
    }
  } else {
    for (long long i = beg + threadIdx.x; i < end; i += NT) {
      float ov = 0.f;
      element(ldf<T>(x, i), kNeedDy ? ldf<T>(dy, i) : 0.f, ov, 0);
      if (kWrites) stf<T>(out, i, ov);
    }
  }
  if (MODE == 0 || MODE == 2 || MODE == 5) {
    acc0 += odd0; acc1 += odd1;
    block_sum2<NT>(acc0, acc1);
    if (threadIdx.x == 0) {
      if (MODE == 0 && a.splits == 1) {
        store_stats(a.stats_out + 2 * r, pivot, (double)acc0, (double)acc1, a.n, a.eps);
      } else if (MODE == 0) {
        float* p = a.partial + ((size_t)r * a.splits + s) * 4;
        p[0] = (float)acc0; p[1] = (float)(acc0 - (double)p[0]);
        p[2] = (float)acc1; p[3] = (float)(acc1 - (double)p[2]);
      } else {
        float* p = a.partial + ((size_t)r * a.splits + s) * 2;
        p[0] = (float)acc0; p[1] = (float)acc1;
      }
    }
  }
}

// per row: combine the split partials.  what 0: (sum d, sum d^2) about the pivot -> (mean, rstd); 1: plain sums (S1, S2)
template <typename T>
__global__ void norm_finalize_kernel(const float* __restrict__ partial, float* __restrict__ out, const void* x, int rows, int splits, long long n, float eps, int what) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  double s0 = 0.0, s1 = 0.0;
  if (what == 0) {
    for (int s = 0; s < splits; ++s) {
      const float* p = partial + ((size_t)r * splits + s) * 4;
      s0 += (double)p[0] + (double)p[1];
      s1 += (double)p[2] + (double)p[3];
    }
    store_stats(out + 2 * r, (double)ldf<T>(static_cast<const T*>(x) + (size_t)r * n, 0), s0, s1, n, eps);
  } else {
    for (int s = 0; s < splits; ++s) { s0 += partial[((size_t)r * splits + s) * 2]; s1 += partial[((size_t)r * splits + s) * 2 + 1]; }
    out[2 * r] = (float)s0;
    out[2 * r + 1] = (float)s1;
  }
}

// SMs of the current device (132 on an H100 SXM; also the value without a device, for the host-side workspace queries)
static int device_sms() {
  static int cached[64] = {0};
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (cached[dev] == 0) cached[dev] = (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0) ? n : 132;
  return cached[dev];
}

int norm_splits(int rows, long long n) {
  long long s = (8LL * device_sms() + rows - 1) / rows;   // >= 8 CTAs per SM's worth of blocks
  const long long by_len = n / 2048 > 0 ? n / 2048 : 1;  // but not less than 2048 elements per CTA
  if (s > by_len) s = by_len;
  if (s > kNormMaxSplits) s = kNormMaxSplits;
  return s < 1 ? 1 : (int)s;
}

template <typename T, int MODE>
static int launch_mode(const NormArgs& a, cudaStream_t st) {
  constexpr int NT = MODE == 0 ? 2 * kNormThreads : kNormThreads;
  const dim3 grid(a.splits, a.rows);
  const bool vec = (a.n % Pack<T>::kN == 0) && ((reinterpret_cast<uintptr_t>(a.x) & 15) == 0) && (a.dy == nullptr || (reinterpret_cast<uintptr_t>(a.dy) & 15) == 0) &&
                   (a.out == nullptr || (reinterpret_cast<uintptr_t>(a.out) & 15) == 0);
  if (vec) norm_kernel<T, MODE, true, NT><<<grid, NT, 0, st>>>(a);
  else norm_kernel<T, MODE, false, NT><<<grid, NT, 0, st>>>(a);
  B200_CHECK_LAUNCH();
  return 0;
}
template <int MODE>
static int launch_dtype(int dtype, const NormArgs& a, cudaStream_t st) {
  if (dtype == B200SHT_BF16) return launch_mode<__nv_bfloat16, MODE>(a, st);
  return launch_mode<float, MODE>(a, st);
}
static int finalize(int dtype, const float* partial, float* out, const void* x, int rows, int splits, long long n, float eps, int what, cudaStream_t st) {
  const int blocks = (rows + 127) / 128;
  if (dtype == B200SHT_BF16) norm_finalize_kernel<__nv_bfloat16><<<blocks, 128, 0, st>>>(partial, out, x, rows, splits, n, eps, what);
  else norm_finalize_kernel<float><<<blocks, 128, 0, st>>>(partial, out, x, rows, splits, n, eps, what);
  B200_CHECK_LAUNCH();
  return 0;
}

static int fill_args(NormArgs* a, int B, int C, long long hw) {
  B200_REQUIRE(B > 0 && C > 0 && hw > 0 && (long long)B * C <= 65535, "norm: bad shape (B %d, C %d, H*W %lld; B*C must be <= 65535)", B, C, hw);
  memset(a, 0, sizeof(*a));
  a->rows = B * C; a->C = C; a->n = hw;
  a->splits = norm_splits(a->rows, hw);
  long long chunk = (hw + a->splits - 1) / a->splits;
  a->chunk = (chunk + 7) / 8 * 8;
  return 0;
}

int instance_norm_forward(const void* x, void* y, const float* gamma, const float* beta, float* stats, float* ws, int dtype, int B, int C, long long hw, float eps,
                          int gelu, cudaStream_t st) {
  NormArgs a;
  int rc = fill_args(&a, B, C, hw);
  if (rc) return rc;
  a.x = x; a.partial = ws;
  NormArgs sa = a;   // statistics: one CTA of 2 x 256 threads per pair of splits, the last one also takes an odd split
  sa.splits = a.splits / 2 > 1 ? a.splits / 2 : 1;
  sa.chunk = 2 * a.chunk;
  sa.stats_out = stats; sa.eps = eps;
  rc = launch_dtype<0>(dtype, sa, st);
  if (!rc && sa.splits > 1) rc = finalize(dtype, ws, stats, x, a.rows, sa.splits, hw, eps, 0, st);
  a.out = y; a.gamma = gamma; a.beta = beta; a.stats = stats; a.gelu = gelu;
  if (!rc) rc = launch_dtype<1>(dtype, a, st);
  return rc;
}

int instance_norm_backward(const void* x, const void* dy, void* dx, const float* gamma, const float* beta, const float* stats, float* sums, float* ws, int dtype,
                           int B, int C, long long hw, int gelu, cudaStream_t st) {
  NormArgs a;
  int rc = fill_args(&a, B, C, hw);
  if (rc) return rc;
  a.x = x; a.dy = dy; a.gamma = gamma; a.beta = beta; a.stats = stats; a.partial = ws; a.gelu = gelu;
  rc = launch_dtype<2>(dtype, a, st);
  if (!rc) rc = finalize(dtype, ws, sums, x, a.rows, a.splits, hw, 0.f, 1, st);
  a.out = dx; a.sums = sums;
  if (!rc) rc = launch_dtype<3>(dtype, a, st);
  return rc;
}

int bias_gelu_forward(const void* x, const float* bias, void* y, int dtype, int B, int C, long long hw, cudaStream_t st) {
  NormArgs a;
  int rc = fill_args(&a, B, C, hw);
  if (rc) return rc;
  a.x = x; a.out = y; a.beta = bias;
  return launch_dtype<4>(dtype, a, st);
}

int bias_gelu_backward(const void* x, const float* bias, const void* dy, void* dx, float* row_sums, float* ws, int dtype, int B, int C, long long hw, cudaStream_t st) {
  NormArgs a;
  int rc = fill_args(&a, B, C, hw);
  if (rc) return rc;
  a.x = x; a.dy = dy; a.out = dx; a.beta = bias; a.partial = ws;
  rc = launch_dtype<5>(dtype, a, st);
  if (!rc && row_sums) rc = finalize(dtype, ws, row_sums, x, a.rows, a.splits, hw, 0.f, 1, st);
  return rc;
}

// ------------------------------------------------------------------------------------------------------------------------------------------------------
// Quadrature-weighted instance norm on the sphere (GeometricInstanceNormS2 / DistributedGeometricInstanceNormS2; reference:
// makani/models/common/layer_norm.py:30-152, makani/mpu/layer_norm.py:173-253, weights makani/utils/grids.py:97-191).  A row (b, c) is an H x W plane
// (the local shard on an h x w grid); q[i] is the weight of latitude row i, constant along longitude.  D is the normaliser (1 in the serial class,
// the total weight of the global crop in the distributed one), S the weight summed over every rank's shard.
//   partials : per row (sum q, mean, M2) in fp64, sums of q d, q d^2 about the pivot d = x - x[row, 0]                         read x
//   finalize : Chan / Welford combine of R ranks' triples in rank order -> (S, m, M2);  mu = S m / D,  var = (M2 + S (m - mu)^2) / D,
//              r = (var + eps)^-1/2,  corr = r mu (D - S) / D                                                                  (per row)
//   apply    : y = [gelu](gamma (x - mu) r + beta)                                                                             read x, write y
//   bwd sums : per row fp64 S1 = sum g, S2 = sum g xhat (unweighted; g = dy, or dy gelu'(z))                                   read x, dy
//   bwd apply: dx = gamma r (g - (q / D) (S1 + xhat S2 - corr S2)), S1 / S2 summed over R ranks in rank order                   read x, dy, write dx
//   dgamma[c] = sum_b S2, dbeta[c] = sum_b S1 of this shard's sums (the distributed class's partials, added up by the caller's gradient hooks)
// A 16-byte packet holds one latitude row's elements when W is a multiple of its width (then q is read once per packet); otherwise the scalar path.

struct GeoArgs {
  const void* x;
  const void* dy;
  void* out;            // y (apply) / dx (backward apply)
  const float* gamma;   // [C] or null (1)
  const float* beta;    // [C] or null (0)
  const float* q;       // [H] latitude weights (partials, backward apply)
  const float* stats;   // [rows][3] mu, r, corr
  const double* sums;   // [R][rows][2] S1, S2 (backward apply)
  double* part;         // per (row, split): partials [rows][splits][4] (sum q d, sum q d^2, sum q, pivot), bwd sums [rows][splits][2]
  double* row_out;      // one-split rows: the row's triple [rows][3] / sums [rows][2]
  long long n;          // H * W
  long long chunk;      // elements per split (a multiple of 8); the last split runs to n
  int rows, C, W, splits, gelu, R;
  float inv_d;          // 1 / D (backward apply)
};

// (sum q, mean, M2) of a row from its sums about the pivot; a row of zero weight has mean and M2 0 (the combine skips it)
__device__ __forceinline__ void geo_triple(double* out, double sq, double s1, double s2, double pivot) {
  if (sq > 0.0) {
    const double md = s1 / sq;
    const double m2 = s2 - s1 * md;
    out[0] = sq; out[1] = pivot + md; out[2] = m2 > 0.0 ? m2 : 0.0;
  } else {
    out[0] = 0.0; out[1] = 0.0; out[2] = 0.0;
  }
}

// sum of q over the elements [beg, end) of a row (q constant along each latitude row of W elements)
__device__ __forceinline__ double geo_weight_sum(const float* q, int W, long long beg, long long end) {
  double s = 0.0;
  for (long long lat = beg / W; lat * W < end; ++lat) {
    const long long a = lat * W > beg ? lat * W : beg, b = (lat + 1) * W < end ? (lat + 1) * W : end;
    s += (double)(b - a) * (double)q[lat];
  }
  return s;
}

// MODE 0: partials, 1: apply, 2: backward sums, 3: backward apply
template <typename T, int MODE, bool VEC, int NT>
__global__ void __launch_bounds__(NT) geo_norm_kernel(const GeoArgs a) {
  const int r = blockIdx.y, s = blockIdx.x;
  const long long beg = (long long)s * a.chunk, end = (s == a.splits - 1 || beg + a.chunk > a.n) ? a.n : beg + a.chunk;
  const T* x = static_cast<const T*>(a.x) + (size_t)r * a.n;
  const T* dy = static_cast<const T*>(a.dy) + (size_t)r * a.n;
  T* out = static_cast<T*>(a.out) + (size_t)r * a.n;
  const int c = r % a.C;
  const float gamma = a.gamma ? a.gamma[c] : 1.f, beta = a.beta ? a.beta[c] : 0.f;
  float mu = 0.f, rs = 1.f, k0 = 0.f, s2f = 0.f;
  double pivot = 0.0;
  if (MODE == 0) pivot = (double)ldf<T>(x, 0);
  if (MODE != 0) { mu = a.stats[3 * r]; rs = a.stats[3 * r + 1]; }
  if (MODE == 3) {
    double s1 = 0.0, s2 = 0.0;
    for (int k = 0; k < a.R; ++k) { s1 += a.sums[((size_t)k * a.rows + r) * 2]; s2 += a.sums[((size_t)k * a.rows + r) * 2 + 1]; }
    s2f = (float)s2;
    k0 = (float)(s1 - (double)a.stats[3 * r + 2] * s2);   // S1 - corr S2
  }
  const float gs = gamma * rs;
  // MODE 0: fp64 sums of q d and q d^2 (q applied per packet); MODE 2: fp64 sums of per-packet fp32 partials of g and g xhat
  double acc0 = 0.0, acc1 = 0.0;

  // one packet (or one element) of latitude weight qv; returns its unweighted partial sums through p0 / p1
  auto element = [&](float xv, float dv, float& ov, float qv, double& p0, double& p1, float& f0, float& f1) {
    if (MODE == 0) {
      const double d = (double)xv - pivot;
      p0 += d; p1 = fma(d, d, p1);
    } else if (MODE == 1) {
      const float z = fmaf((xv - mu) * rs, gamma, beta);
      ov = a.gelu ? gelu_f(z) : z;
    } else {
      const float xh = (xv - mu) * rs;
      const float g = a.gelu ? dv * gelu_grad_f(fmaf(xh, gamma, beta)) : dv;
      if (MODE == 2) { f0 += g; f1 = fmaf(g, xh, f1); }
      else ov = gs * (g - qv * fmaf(xh, s2f, k0));
    }
  };
  constexpr bool kNeedDy = (MODE == 2 || MODE == 3), kWrites = (MODE == 1 || MODE == 3), kNeedQ = (MODE == 0 || MODE == 3);
  auto row_weight = [&](long long i) -> float { return kNeedQ ? (MODE == 3 ? a.q[(int)(i / a.W)] * a.inv_d : a.q[(int)(i / a.W)]) : 0.f; };
  if (VEC) {
    constexpr int kN = Pack<T>::kN;
    constexpr long long kStride = (long long)NT * kN;
    // W a multiple of kN: a packet lies in one latitude row
    auto packet = [&](const Pack<T>& px, const Pack<T>& pd, long long i) {
      Pack<T> po;
      const float qv = row_weight(i);
      double p0 = 0.0, p1 = 0.0;
      float f0 = 0.f, f1 = 0.f;
#pragma unroll
      for (int j = 0; j < kN; ++j) {
        float ov = 0.f;
        element(px.get(j), kNeedDy ? pd.get(j) : 0.f, ov, qv, p0, p1, f0, f1);
        if (kWrites) po.set(j, ov);
      }
      if (kWrites) po.store(out + i);
      if (MODE == 0) { acc0 = fma((double)qv, p0, acc0); acc1 = fma((double)qv, p1, acc1); }
      if (MODE == 2) { acc0 += (double)f0; acc1 += (double)f1; }
    };
    long long i = beg + (long long)threadIdx.x * kN;
    for (; i + kStride < end; i += 2 * kStride) {   // two packets per tensor in flight per thread, as norm_kernel
      Pack<T> px0, px1, pd0, pd1;
      px0.load(x + i);
      px1.load(x + i + kStride);
      if (kNeedDy) { pd0.load(dy + i); pd1.load(dy + i + kStride); }
      packet(px0, pd0, i);
      packet(px1, pd1, i + kStride);
    }
    for (; i < end; i += kStride) {
      Pack<T> px, pd;
      px.load(x + i);
      if (kNeedDy) pd.load(dy + i);
      packet(px, pd, i);
    }
  } else {
    for (long long i = beg + threadIdx.x; i < end; i += NT) {
      const float qv = row_weight(i);
      double p0 = 0.0, p1 = 0.0;
      float f0 = 0.f, f1 = 0.f, ov = 0.f;
      element(ldf<T>(x, i), kNeedDy ? ldf<T>(dy, i) : 0.f, ov, qv, p0, p1, f0, f1);
      if (kWrites) stf<T>(out, i, ov);
      if (MODE == 0) { acc0 = fma((double)qv, p0, acc0); acc1 = fma((double)qv, p1, acc1); }
      if (MODE == 2) { acc0 += (double)f0; acc1 += (double)f1; }
    }
  }
  if (MODE == 0 || MODE == 2) {
    block_sum2<NT>(acc0, acc1);
    if (threadIdx.x == 0) {
      if (MODE == 0) {
        const double sq = geo_weight_sum(a.q, a.W, beg, end);
        if (a.splits == 1) geo_triple(a.row_out + 3 * (size_t)r, sq, acc0, acc1, pivot);
        else { double* p = a.part + ((size_t)r * a.splits + s) * 4; p[0] = acc0; p[1] = acc1; p[2] = sq; p[3] = pivot; }
      } else {
        double* p = a.splits == 1 ? a.row_out + 2 * (size_t)r : a.part + ((size_t)r * a.splits + s) * 2;
        p[0] = acc0; p[1] = acc1;
      }
    }
  }
}

// per row: add the split partials.  what 0: partials (sum q d, sum q d^2, sum q, pivot) -> (sum q, mean, M2);  1: backward sums (S1, S2)
__global__ void geo_split_combine_kernel(const double* __restrict__ part, double* __restrict__ out, int rows, int splits, int what) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  const int w = what == 0 ? 4 : 2;
  double s0 = 0.0, s1 = 0.0, s2 = 0.0;
  for (int s = 0; s < splits; ++s) {
    const double* p = part + ((size_t)r * splits + s) * w;
    s0 += p[0]; s1 += p[1];
    if (what == 0) s2 += p[2];
  }
  if (what == 0) geo_triple(out + 3 * (size_t)r, s2, s0, s1, part[(size_t)r * splits * 4 + 3]);
  else { out[2 * (size_t)r] = s0; out[2 * (size_t)r + 1] = s1; }
}

// per row: Chan / Welford combine of R ranks' (sum q, mean, M2) in rank order, then (mu, r, corr) for the normaliser D
__global__ void geo_finalize_kernel(const double* __restrict__ part, float* __restrict__ stats, int R, int rows, double D, float eps) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  double S = 0.0, m = 0.0, M2 = 0.0;
  for (int k = 0; k < R; ++k) {
    const double* p = part + ((size_t)k * rows + r) * 3;
    const double nb = p[0];
    if (!(nb > 0.0)) continue;
    const double n = S + nb, delta = p[1] - m;
    m += delta * (nb / n);
    M2 += p[2] + delta * delta * (S * nb / n);
    S = n;
  }
  const double mu = S * m / D;
  double var = (M2 + S * (m - mu) * (m - mu)) / D;
  if (var < 0.0) var = 0.0;
  const double rs = 1.0 / sqrt(var + (double)eps);
  stats[3 * (size_t)r] = (float)mu;
  stats[3 * (size_t)r + 1] = (float)rs;
  stats[3 * (size_t)r + 2] = (float)(rs * mu * (D - S) / D);
}

// per channel: dgamma[c] = sum_b S2, dbeta[c] = sum_b S1 of this shard's row sums (batch in order); either output may be null
__global__ void geo_param_grad_kernel(const double* __restrict__ sums, float* __restrict__ dgamma, float* __restrict__ dbeta, int B, int C) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double s1 = 0.0, s2 = 0.0;
  for (int b = 0; b < B; ++b) { s1 += sums[((size_t)b * C + c) * 2]; s2 += sums[((size_t)b * C + c) * 2 + 1]; }
  if (dgamma) dgamma[c] = (float)s2;
  if (dbeta) dbeta[c] = (float)s1;
}

template <typename T, int MODE>
static int geo_launch_mode(const GeoArgs& a, cudaStream_t st) {
  constexpr int NT = MODE == 0 ? 2 * kNormThreads : kNormThreads;
  const dim3 grid(a.splits, a.rows);
  const auto al = [](const void* p) { return p == nullptr || (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  const bool vec = (a.W % Pack<T>::kN == 0) && al(a.x) && al(a.dy) && al(a.out);
  if (vec) geo_norm_kernel<T, MODE, true, NT><<<grid, NT, 0, st>>>(a);
  else geo_norm_kernel<T, MODE, false, NT><<<grid, NT, 0, st>>>(a);
  B200_CHECK_LAUNCH();
  return 0;
}
template <int MODE>
static int geo_launch(int dtype, const GeoArgs& a, cudaStream_t st) {
  if (dtype == B200SHT_BF16) return geo_launch_mode<__nv_bfloat16, MODE>(a, st);
  return geo_launch_mode<float, MODE>(a, st);
}

// the split of a row for the statistics / backward-sum passes (`pair` 1: the 2 x 256-thread statistics CTA takes a pair of splits)
static int geo_fill(GeoArgs* a, int B, int C, int H, int W, bool pair) {
  B200_REQUIRE(B > 0 && C > 0 && H > 0 && W > 0 && (long long)B * C <= 65535 && (long long)H * W < (1LL << 31),
               "geometric_norm: bad shape (B %d, C %d, H %d, W %d; B*C must be <= 65535, H*W < 2^31)", B, C, H, W);
  memset(a, 0, sizeof(*a));
  a->rows = B * C; a->C = C; a->W = W; a->n = (long long)H * W; a->R = 1;
  a->splits = norm_splits(a->rows, a->n);
  long long chunk = (a->n + a->splits - 1) / a->splits;
  a->chunk = (chunk + 7) / 8 * 8;
  if (pair) {
    a->splits = a->splits / 2 > 1 ? a->splits / 2 : 1;
    a->chunk *= 2;
  }
  return 0;
}

long long geometric_norm_workspace_doubles(int B, int C, long long hw) { return (long long)B * C * norm_splits(B * C, hw) * 4; }

int geometric_norm_partials(const void* x, const float* q, double* partials, double* ws, int dtype, int B, int C, int H, int W, cudaStream_t st) {
  GeoArgs a;
  int rc = geo_fill(&a, B, C, H, W, true);
  if (rc) return rc;
  a.x = x; a.q = q; a.part = ws; a.row_out = partials;
  rc = geo_launch<0>(dtype, a, st);
  if (!rc && a.splits > 1) {
    geo_split_combine_kernel<<<(a.rows + 127) / 128, 128, 0, st>>>(ws, partials, a.rows, a.splits, 0);
    B200_CHECK_LAUNCH();
  }
  return rc;
}

int geometric_norm_finalize(const double* partials, int R, int rows, double D, float eps, float* stats, cudaStream_t st) {
  B200_REQUIRE(R > 0 && rows > 0 && D > 0.0, "geometric_norm_finalize: bad arguments (R %d, rows %d, D %g)", R, rows, D);
  geo_finalize_kernel<<<(rows + 127) / 128, 128, 0, st>>>(partials, stats, R, rows, D, eps);
  B200_CHECK_LAUNCH();
  return 0;
}

int geometric_norm_apply(const void* x, void* y, const float* gamma, const float* beta, const float* stats, int dtype, int B, int C, int H, int W, int gelu,
                         cudaStream_t st) {
  GeoArgs a;
  int rc = geo_fill(&a, B, C, H, W, false);
  if (rc) return rc;
  a.x = x; a.out = y; a.gamma = gamma; a.beta = beta; a.stats = stats; a.gelu = gelu;
  return geo_launch<1>(dtype, a, st);
}

int geometric_norm_backward_sums(const void* x, const void* dy, const float* gamma, const float* beta, const float* stats, double* sums, double* ws, int dtype,
                                 int B, int C, int H, int W, int gelu, cudaStream_t st) {
  GeoArgs a;
  int rc = geo_fill(&a, B, C, H, W, false);
  if (rc) return rc;
  a.x = x; a.dy = dy; a.gamma = gamma; a.beta = beta; a.stats = stats; a.gelu = gelu; a.part = ws; a.row_out = sums;
  rc = geo_launch<2>(dtype, a, st);
  if (!rc && a.splits > 1) {
    geo_split_combine_kernel<<<(a.rows + 127) / 128, 128, 0, st>>>(ws, sums, a.rows, a.splits, 1);
    B200_CHECK_LAUNCH();
  }
  return rc;
}

int geometric_norm_backward_apply(const void* x, const void* dy, void* dx, const float* gamma, const float* beta, const float* stats, const double* sums, int R,
                                  const float* q, double D, int dtype, int B, int C, int H, int W, int gelu, cudaStream_t st) {
  GeoArgs a;
  int rc = geo_fill(&a, B, C, H, W, false);
  if (rc) return rc;
  B200_REQUIRE(R > 0 && D > 0.0, "geometric_norm_backward_apply: bad arguments (R %d, D %g)", R, D);
  a.x = x; a.dy = dy; a.out = dx; a.gamma = gamma; a.beta = beta; a.stats = stats; a.sums = sums; a.R = R; a.q = q; a.gelu = gelu;
  a.inv_d = (float)(1.0 / D);
  return geo_launch<3>(dtype, a, st);
}

int geometric_norm_param_grads(const double* sums, float* dgamma, float* dbeta, int B, int C, cudaStream_t st) {
  B200_REQUIRE(B > 0 && C > 0, "geometric_norm_param_grads: bad shape (B %d, C %d)", B, C);
  geo_param_grad_kernel<<<(C + 127) / 128, 128, 0, st>>>(sums, dgamma, dbeta, B, C);
  B200_CHECK_LAUNCH();
  return 0;
}

}  // namespace b200sht

namespace b200sht {

// ------------------------------------------------------------------------------------------------------------------------------------------------------
// Channel layer norm (makani's DistributedLayerNorm, makani/mpu/layer_norm.py:256-290: nn.LayerNorm(C) over the channels of an NCHW activation, which
// makani runs as transpose -> layer_norm -> transpose -> .contiguous()).  Per grid point (b, p), p = i W + j, over the C values x[b, c, p] that lie
// hw elements apart:
//   forward : mu = mean_c x, var = mean_c (x - mu)^2, r = (var + eps)^-1/2, y = [gelu](gamma_c (x - mu) r + beta_c)                 read x, write y
//   backward: g = dy [gelu'(z)], dx = r (gamma g - mean_c(gamma g) - xhat mean_c(gamma g xhat))                            read x, dy, write dx
//             dgamma_c = sum g xhat, dbeta_c = sum g: per-CTA partials in fixed order, then a per-channel fp64 finalize (no atomics)
// A CTA takes a tile of 32 consecutive points (one warp wide, so every load of a channel row is 32 consecutive elements) and kLnMaxWarps warps
// split the channel loop.  The tile (x, and dy in the backward) is staged in shared memory on the first pass, so the second pass reads no HBM;
// a tile too large for shared memory is read twice from global memory instead (the second read mostly hits L2).  Statistics: fp32 Welford per
// thread about the point's channel-0 value, Chan-combined over the warps in warp order (an offset common to all channels does not cancel).  x / dx in T, y / dy in TO: (float, float),
// (bf16, bf16), and (bf16, float) for makani's layer under autocast, whose layer_norm returns fp32 for a bf16 input.
constexpr int kLnPoints = 32;
constexpr int kLnMaxWarps = 16;
constexpr int kLnUnroll = 4;
constexpr int kLnMaxStageBytes = 112 * 1024;   // at least two CTAs per SM

__device__ __forceinline__ float tof(float v) { return v; }
__device__ __forceinline__ float tof(__nv_bfloat16 v) { return __bfloat162float(v); }
template <typename T> __device__ __forceinline__ T fromf(float v);
template <> __device__ __forceinline__ float fromf<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 fromf<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

struct LnArgs {
  const void* x;
  const void* dy;
  void* out;            // y (forward) / dx (backward)
  const float* gamma;   // [C] or null (1)
  const float* beta;    // [C] or null (0)
  float* stats;         // [B * hw][2] mu, r
  float* partial;       // backward: [gridDim.x][C][2] sum g xhat, sum g
  long long hw, tiles_per_b, tiles;
  int C, gelu;
  float eps;
};

// the tile's first element of channel 0 and its lane's point
__device__ __forceinline__ long long ln_tile(const LnArgs& a, long long t, long long& p) {
  const long long b = t / a.tiles_per_b;
  p = (t - b * a.tiles_per_b) * kLnPoints + threadIdx.x;
  return b * a.C * a.hw;
}

template <typename T, typename TO, bool STAGE>
__global__ void __launch_bounds__(kLnPoints * kLnMaxWarps) ln_forward_kernel(const LnArgs a) {
  extern __shared__ __align__(16) unsigned char ln_smem[];
  __shared__ float red[2][kLnMaxWarps][kLnPoints];
  __shared__ float pt[2][kLnPoints];
  T* sx = reinterpret_cast<T*>(ln_smem);
  const int lane = threadIdx.x, wy = threadIdx.y, WY = blockDim.y, C = a.C;
  long long p;
  const long long base = ln_tile(a, blockIdx.x, p);
  const bool valid = p < a.hw;
  const T* x = static_cast<const T*>(a.x) + base + p;
  TO* y = static_cast<TO*>(a.out) + base + p;

  // Welford of d = x - x[channel 0]: for a point whose channels share a large offset, the d are exact (Sterbenz) and O(spread)
  const float pivot = valid ? tof(x[0]) : 0.f;
  float n = 0.f, mean = 0.f, m2 = 0.f;
  for (int c0 = wy; c0 < C; c0 += WY * kLnUnroll) {
    T v[kLnUnroll];
#pragma unroll
    for (int u = 0; u < kLnUnroll; ++u) {
      const int c = c0 + u * WY;
      v[u] = (valid && c < C) ? x[(long long)c * a.hw] : fromf<T>(0.f);
      if (STAGE && c < C) sx[c * kLnPoints + lane] = v[u];
    }
#pragma unroll
    for (int u = 0; u < kLnUnroll; ++u) {
      if (c0 + u * WY < C) {
        const float xv = tof(v[u]) - pivot;
        n += 1.f;
        const float d = xv - mean;
        mean += d / n;
        m2 = fmaf(d, xv - mean, m2);
      }
    }
  }
  red[0][wy][lane] = mean;
  red[1][wy][lane] = m2;
  __syncthreads();
  if (wy == 0) {
    float N = 0.f, M = 0.f, Q = 0.f;
    for (int k = 0; k < WY; ++k) {
      const float nb = (float)((C - k + WY - 1) / WY), nn = N + nb, d = red[0][k][lane] - M;
      M += d * (nb / nn);
      Q += red[1][k][lane] + d * d * (N * nb / nn);
      N = nn;
    }
    const float r = 1.f / sqrtf(Q / (float)C + a.eps);
    pt[0][lane] = pivot + M;
    pt[1][lane] = r;
    if (valid) { a.stats[2 * (base / C + p)] = pivot + M; a.stats[2 * (base / C + p) + 1] = r; }
  }
  __syncthreads();
  const float mu = pt[0][lane], r = pt[1][lane];
#pragma unroll kLnUnroll
  for (int c = wy; c < C; c += WY) {
    const float xv = tof(STAGE ? sx[c * kLnPoints + lane] : (valid ? x[(long long)c * a.hw] : fromf<T>(0.f)));
    const float z = fmaf((xv - mu) * r, a.gamma ? __ldg(a.gamma + c) : 1.f, a.beta ? __ldg(a.beta + c) : 0.f);
    if (valid) y[(long long)c * a.hw] = fromf<TO>(a.gelu ? gelu_f(z) : z);
  }
}

// persistent: CTA k takes tiles k, k + gridDim.x, ... and accumulates its parameter-gradient partials in shared memory, one warp per channel
template <typename T, typename TO, bool STAGE>
__global__ void __launch_bounds__(kLnPoints * kLnMaxWarps) ln_backward_kernel(const LnArgs a) {
  extern __shared__ __align__(16) unsigned char ln_smem[];
  __shared__ float red[2][kLnMaxWarps][kLnPoints];
  __shared__ float pt[2][kLnPoints];
  const int lane = threadIdx.x, wy = threadIdx.y, WY = blockDim.y, C = a.C;
  float* pacc = reinterpret_cast<float*>(ln_smem);                   // [C][2]
  T* sx = reinterpret_cast<T*>(ln_smem + ((size_t)C * 8 + 15) / 16 * 16);
  TO* sd = reinterpret_cast<TO*>(reinterpret_cast<unsigned char*>(sx) + ((size_t)C * kLnPoints * sizeof(T) + 15) / 16 * 16);
  for (int i = wy * kLnPoints + lane; i < 2 * C; i += WY * kLnPoints) pacc[i] = 0.f;
  __syncthreads();

  for (long long t = blockIdx.x; t < a.tiles; t += gridDim.x) {
    long long p;
    const long long base = ln_tile(a, t, p);
    const bool valid = p < a.hw;
    const T* x = static_cast<const T*>(a.x) + base + p;
    const TO* dy = static_cast<const TO*>(a.dy) + base + p;
    T* dx = static_cast<T*>(a.out) + base + p;
    const float mu = valid ? a.stats[2 * (base / C + p)] : 0.f, r = valid ? a.stats[2 * (base / C + p) + 1] : 0.f;

    float s1 = 0.f, s2 = 0.f;   // sum gamma g, sum gamma g xhat over this thread's channels
    for (int c0 = wy; c0 < C; c0 += WY * kLnUnroll) {
      T xr[kLnUnroll];
      TO dr[kLnUnroll];
#pragma unroll
      for (int u = 0; u < kLnUnroll; ++u) {
        const int c = c0 + u * WY;
        const bool in = valid && c < C;
        xr[u] = in ? x[(long long)c * a.hw] : fromf<T>(0.f);
        dr[u] = in ? dy[(long long)c * a.hw] : fromf<TO>(0.f);
        if (STAGE && c < C) { sx[c * kLnPoints + lane] = xr[u]; sd[c * kLnPoints + lane] = dr[u]; }
      }
#pragma unroll
      for (int u = 0; u < kLnUnroll; ++u) {
        const int c = c0 + u * WY;
        if (c < C) {
          const float gm = a.gamma ? __ldg(a.gamma + c) : 1.f;
          const float xh = (tof(xr[u]) - mu) * r;
          const float g = a.gelu ? tof(dr[u]) * gelu_grad_f(fmaf(xh, gm, a.beta ? __ldg(a.beta + c) : 0.f)) : tof(dr[u]);
          s1 = fmaf(gm, g, s1);
          s2 = fmaf(gm * g, xh, s2);
          float pg = g * xh, pb = g;
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) { pg += __shfl_xor_sync(0xffffffffu, pg, o); pb += __shfl_xor_sync(0xffffffffu, pb, o); }
          if (lane == 0) { pacc[2 * c] += pg; pacc[2 * c + 1] += pb; }
        }
      }
    }
    red[0][wy][lane] = s1;
    red[1][wy][lane] = s2;
    __syncthreads();
    if (wy == 0) {
      float t1 = 0.f, t2 = 0.f;
      for (int k = 0; k < WY; ++k) { t1 += red[0][k][lane]; t2 += red[1][k][lane]; }
      pt[0][lane] = t1 / (float)C;
      pt[1][lane] = t2 / (float)C;
    }
    __syncthreads();
    const float m1 = pt[0][lane], m2 = pt[1][lane];
#pragma unroll kLnUnroll
    for (int c = wy; c < C; c += WY) {
      const float xv = tof(STAGE ? sx[c * kLnPoints + lane] : (valid ? x[(long long)c * a.hw] : fromf<T>(0.f)));
      const float dv = tof(STAGE ? sd[c * kLnPoints + lane] : (valid ? dy[(long long)c * a.hw] : fromf<TO>(0.f)));
      const float gm = a.gamma ? __ldg(a.gamma + c) : 1.f;
      const float xh = (xv - mu) * r;
      const float g = a.gelu ? dv * gelu_grad_f(fmaf(xh, gm, a.beta ? __ldg(a.beta + c) : 0.f)) : dv;
      if (valid) dx[(long long)c * a.hw] = fromf<T>(r * (gm * g - m1 - xh * m2));
    }
    __syncthreads();   // the next tile overwrites the staged tile and red / pt
  }
  for (int i = wy * kLnPoints + lane; i < 2 * C; i += WY * kLnPoints) a.partial[(size_t)blockIdx.x * 2 * C + i] = pacc[i];
}

// per channel: the CTAs' partials added in CTA order in fp64; either output may be null
__global__ void ln_param_grad_kernel(const float* __restrict__ partial, float* __restrict__ dgamma, float* __restrict__ dbeta, int ctas, int C) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double sg = 0.0, sb = 0.0;
  for (int k = 0; k < ctas; ++k) { sg += partial[((size_t)k * C + c) * 2]; sb += partial[((size_t)k * C + c) * 2 + 1]; }
  if (dgamma) dgamma[c] = (float)sg;
  if (dbeta) dbeta[c] = (float)sb;
}

static int ln_fill(LnArgs* a, int B, int C, long long hw) {
  B200_REQUIRE(B > 0 && C > 0 && hw > 0, "layer_norm: bad shape (B %d, C %d, H*W %lld)", B, C, hw);
  memset(a, 0, sizeof(*a));
  a->C = C; a->hw = hw;
  a->tiles_per_b = (hw + kLnPoints - 1) / kLnPoints;
  a->tiles = a->tiles_per_b * B;
  B200_REQUIRE(a->tiles < (1LL << 31), "layer_norm: too many grid points (B %d, H*W %lld)", B, hw);
  return 0;
}

static int ln_warps(int C) { return C < kLnMaxWarps ? C : kLnMaxWarps; }
static size_t ln_fwd_stage_bytes(int C, size_t es) { return (size_t)C * kLnPoints * es; }
static size_t ln_bwd_stage_bytes(int C, size_t es, size_t eso) {
  return ((size_t)C * 8 + 15) / 16 * 16 + ((size_t)C * kLnPoints * es + 15) / 16 * 16 + (size_t)C * kLnPoints * eso;
}

// CTAs of the persistent backward: as many as fit on the device at once, at most one per tile
static int ln_bwd_ctas(long long tiles, int smem_bytes, const void* kernel, int threads) {
  int per_sm = 0;
  if (kernel == nullptr || cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, smem_bytes) != cudaSuccess || per_sm < 1) per_sm = 1;
  const long long n = (long long)per_sm * device_sms();
  return (int)(tiles < n ? tiles : n);
}

long long layer_norm_workspace_floats(int B, int C, long long hw) {
  const long long tiles = (long long)B * ((hw + kLnPoints - 1) / kLnPoints), cap = 32LL * device_sms();   // 32: most resident CTAs per SM
  return 2LL * C * (tiles < cap ? tiles : cap);
}

template <typename T, typename TO>
static int ln_forward_t(const LnArgs& a, cudaStream_t st) {
  const int wy = ln_warps(a.C);
  const size_t stage = ln_fwd_stage_bytes(a.C, sizeof(T));
  const dim3 block(kLnPoints, wy);
  if (stage <= (size_t)kLnMaxStageBytes) {
    B200_CHECK_CUDA(cudaFuncSetAttribute(ln_forward_kernel<T, TO, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)stage));
    ln_forward_kernel<T, TO, true><<<(unsigned)a.tiles, block, stage, st>>>(a);
  } else {
    ln_forward_kernel<T, TO, false><<<(unsigned)a.tiles, block, 0, st>>>(a);
  }
  B200_CHECK_LAUNCH();
  return 0;
}

template <typename T, typename TO>
static int ln_backward_t(LnArgs a, float* dgamma, float* dbeta, cudaStream_t st) {
  const int wy = ln_warps(a.C);
  const size_t stage = ln_bwd_stage_bytes(a.C, sizeof(T), sizeof(TO));
  const size_t pacc = ((size_t)a.C * 8 + 15) / 16 * 16;
  const bool staged = stage <= (size_t)kLnMaxStageBytes;
  const void* k = staged ? (const void*)ln_backward_kernel<T, TO, true> : (const void*)ln_backward_kernel<T, TO, false>;
  const int smem = (int)(staged ? stage : pacc);
  B200_REQUIRE(smem <= 200 * 1024, "layer_norm_backward: C %d too large", a.C);
  B200_CHECK_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  const int ctas = ln_bwd_ctas(a.tiles, smem, k, kLnPoints * wy);
  const dim3 block(kLnPoints, wy);
  if (staged) ln_backward_kernel<T, TO, true><<<ctas, block, smem, st>>>(a);
  else ln_backward_kernel<T, TO, false><<<ctas, block, smem, st>>>(a);
  B200_CHECK_LAUNCH();
  if (dgamma || dbeta) {
    ln_param_grad_kernel<<<(a.C + 127) / 128, 128, 0, st>>>(a.partial, dgamma, dbeta, ctas, a.C);
    B200_CHECK_LAUNCH();
  }
  return 0;
}

int layer_norm_forward(const void* x, void* y, const float* gamma, const float* beta, float* stats, int dtype, int out_dtype, int B, int C, long long hw,
                       float eps, int gelu, cudaStream_t st) {
  LnArgs a;
  int rc = ln_fill(&a, B, C, hw);
  if (rc) return rc;
  a.x = x; a.out = y; a.gamma = gamma; a.beta = beta; a.stats = stats; a.eps = eps; a.gelu = gelu;
  if (dtype == B200SHT_F32) return ln_forward_t<float, float>(a, st);
  if (out_dtype == B200SHT_BF16) return ln_forward_t<__nv_bfloat16, __nv_bfloat16>(a, st);
  return ln_forward_t<__nv_bfloat16, float>(a, st);
}

int layer_norm_backward(const void* x, const void* dy, void* dx, const float* gamma, const float* beta, const float* stats, float* dgamma, float* dbeta,
                        float* ws, int dtype, int out_dtype, int B, int C, long long hw, int gelu, cudaStream_t st) {
  LnArgs a;
  int rc = ln_fill(&a, B, C, hw);
  if (rc) return rc;
  a.x = x; a.dy = dy; a.out = dx; a.gamma = gamma; a.beta = beta; a.stats = const_cast<float*>(stats); a.partial = ws; a.gelu = gelu;
  if (dtype == B200SHT_F32) return ln_backward_t<float, float>(a, dgamma, dbeta, st);
  if (out_dtype == B200SHT_BF16) return ln_backward_t<__nv_bfloat16, __nv_bfloat16>(a, dgamma, dbeta, st);
  return ln_backward_t<__nv_bfloat16, float>(a, dgamma, dbeta, st);
}

}  // namespace b200sht
