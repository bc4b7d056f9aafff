// C ABI of the b200sht library (see include/b200sht.h for the contract and the reference interfaces replaced).
#include "common.cuh"
#include <cmath>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

namespace b200sht {
int& sm_reserve() { static thread_local int r = 0; return r; }

static thread_local std::string g_last_error;

void set_error(const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_last_error = buf;
}

// other translation units
bool make_fft_plan(int N, FftPlan* p);
int build_table(Plan* pl, const double* d_cost, cudaStream_t st);
int fft_analysis(const Plan* pl, const void* x, int dtype, int B, int C, float* X, int scale_mode, cudaStream_t st);
int fft_synthesis(const Plan* pl, const float* Z, void* y, int dtype, int B, int C, const float* bias, int scale_mode, cudaStream_t st);
int legendre_analysis_simt(const Plan* pl, const float* X, float* spec, int B, int C, cudaStream_t st);
int legendre_synthesis_simt(const Plan* pl, const float* spec, float* Z, int B, int C, cudaStream_t st);
int spec_unpack(const Plan* pl, const float* spec, void* coeffs, int B, int C, cudaStream_t st);
int spec_pack(const Plan* pl, const void* coeffs, float* spec, int B, int C, cudaStream_t st);
int bias_grad(const Plan* pl, const float* X, float* gbias, int B, int C, cudaStream_t st);
int mix_weight_relayout(int op, const void* w_native, float* w_packed, int L, int G, int Ci, int Co, int to_native, int round_tf32, cudaStream_t st);
int mix_forward_simt(const Plan* pl, int op, const float* x, const void* w, const void* cbias, float* y, int B, int G, int Ci, int Co, cudaStream_t st);
int mix_backward_simt(const Plan* pl, int op, const float* x, const void* w, const float* gy, float* gx, void* gw, void* gcbias, int B, int G,
                      int Ci, int Co, cudaStream_t st);
int complex_relu_fwd(const Plan* pl, int mode, const float* x, const float* bias, float slope, float* y, int B, int C, cudaStream_t st);
int complex_relu_bwd(const Plan* pl, int mode, const float* x, const float* bias, float slope, const float* gy, float* gx, float* gbias, int B,
                     int C, cudaStream_t st);
// tensor-core path (umma.cu)
int umma_plan_init(Plan* pl);
void umma_plan_destroy(Plan* pl);
int dft_plan_init(Plan* pl);
void dft_plan_destroy(Plan* pl);
int dft_host(int N, int mmax, int direction, int mode, const float* rowscale, const float* in, float* out);
int dft_profile_read(unsigned long long* out16);
int umma_profile_read(unsigned long long* out16);
int legendre_analysis_umma(const Plan* pl, const float* X, float* spec, int B, int C, cudaStream_t st, const float* X_lo = nullptr);
int legendre_synthesis_umma(const Plan* pl, const float* spec, float* Z, int B, int C, int tiled, cudaStream_t st, const float* spec_lo = nullptr);
int umma_plan_table_lo(const Plan* pl);
int tf32_residual(const float* src, float* dst, size_t n, cudaStream_t st);
bool dft_usable(const Plan* pl);
int mix_forward_umma(const Plan* pl, int op, const float* x, const void* w, const void* cbias, float* y, int B, int G, int Ci, int Co, cudaStream_t st);
int mix_backward_umma(const Plan* pl, int op, const float* x, const void* w, const float* gy, float* gx, void* gw, void* gcbias, int B, int G,
                      int Ci, int Co, cudaStream_t st);

// pointwise tail of the SFNO block (norm.cu)
int norm_splits(int rows, long long n);
int instance_norm_forward(const void* x, void* y, const float* gamma, const float* beta, float* stats, float* ws, int dtype, int B, int C, long long hw, float eps,
                          int gelu, cudaStream_t st);
int instance_norm_backward(const void* x, const void* dy, void* dx, const float* gamma, const float* beta, const float* stats, float* sums, float* ws, int dtype,
                           int B, int C, long long hw, int gelu, cudaStream_t st);
int bias_gelu_forward(const void* x, const float* bias, void* y, int dtype, int B, int C, long long hw, cudaStream_t st);
int bias_gelu_backward(const void* x, const float* bias, const void* dy, void* dx, float* row_sums, float* ws, int dtype, int B, int C, long long hw, cudaStream_t st);
long long geometric_norm_workspace_doubles(int B, int C, long long hw);
int geometric_norm_partials(const void* x, const float* q, double* partials, double* ws, int dtype, int B, int C, int H, int W, cudaStream_t st);
int geometric_norm_finalize(const double* partials, int R, int rows, double D, float eps, float* stats, cudaStream_t st);
int geometric_norm_apply(const void* x, void* y, const float* gamma, const float* beta, const float* stats, int dtype, int B, int C, int H, int W, int gelu,
                         cudaStream_t st);
int geometric_norm_backward_sums(const void* x, const void* dy, const float* gamma, const float* beta, const float* stats, double* sums, double* ws, int dtype,
                                 int B, int C, int H, int W, int gelu, cudaStream_t st);
int geometric_norm_backward_apply(const void* x, const void* dy, void* dx, const float* gamma, const float* beta, const float* stats, const double* sums, int R,
                                  const float* q, double D, int dtype, int B, int C, int H, int W, int gelu, cudaStream_t st);
int geometric_norm_param_grads(const double* sums, float* dgamma, float* dbeta, int B, int C, cudaStream_t st);

static inline cudaStream_t S(void* s) { return static_cast<cudaStream_t>(s); }
static inline int cp_of(int C) { return round_up(C, 4); }
// dims-only plan for the entry points that depend on (L, M) alone
static inline Plan lm_plan(int L, int M, int m0 = 0, int dense = 0) { Plan p; memset(&p, 0, sizeof(p)); p.lmax = L; p.mmax = M; p.m0 = m0; p.dense = dense; return p; }
int latspec_convert(const Plan* pl, float* lat, void* coeffs, int B, int C, int to_packed, cudaStream_t st);
int vector_spec_convert(const Plan* pl, float* spec, void* coeffs, int B, int C, int to_packed, int scaled, cudaStream_t st);
int umma_available();
int disco_plan_create(b200sht_disco_plan** out, int nlat_in, int nlon_in, int nlat_out, int nlon_out, int K, long long nnz, const int* ker,
                      const int* lat_out, const int* col_in, const double* vals, cudaStream_t st);
int disco_plan_destroy(b200sht_disco_plan* pl);
long long disco_plan_query(const b200sht_disco_plan* pl, int what);
int disco_forward(const b200sht_disco_plan* pl, const void* x, int dtype, int B, int C, float* X, cudaStream_t st);
int disco_adjoint(const b200sht_disco_plan* pl, const float* dX, void* dx, int dtype, int B, int C, cudaStream_t st);
int attention_forward(const b200sht_disco_plan* pl, const float* q, const float* k, const float* v, float* y, float* lse, int B, int H, int EK,
                      int EV, float scale, cudaStream_t st);
int attention_backward(const b200sht_disco_plan* pl, const float* q, const float* k, const float* v, const float* y, const float* lse,
                       const float* dy, float* dq, float* dk, float* dv, float* D, int B, int H, int EK, int EV, float scale, cudaStream_t st);
int resample_plan_create(b200sht_resample_plan** out, int nlat_in, int nlon_in, int nlat_out, int nlon_out, int expand_poles, const int* lat_idx,
                         const float* lat_w, const int* lon_left, const int* lon_right, const float* lon_w, cudaStream_t st);
int resample_plan_destroy(b200sht_resample_plan* pl);
long long resample_plan_query(const b200sht_resample_plan* pl, int what);
int resample_forward(const b200sht_resample_plan* pl, const float* x, float* y, int planes, cudaStream_t st);
int resample_adjoint(const b200sht_resample_plan* pl, const float* dy, float* dx, int planes, cudaStream_t st);

}  // namespace b200sht

using namespace b200sht;

extern "C" {

const char* b200sht_last_error(void) { return g_last_error.c_str(); }
int b200sht_version(void) { return 100; }

int b200sht_plan_create(b200sht_plan** out, int nlat, int nlon, int lmax, int mmax, const double* cost, const double* quad_w, int csphase,
                        void* stream) {
  return b200sht_plan_create_ex(out, nlat, nlon, lmax, mmax, 0, 0, cost, quad_w, csphase, stream);
}

int b200sht_plan_create_ex(b200sht_plan** out, int nlat, int nlon, int lmax, int mmax, int m_offset, int flags, const double* cost,
                           const double* quad_w, int csphase, void* stream) {
  B200_REQUIRE(out != nullptr && cost != nullptr && quad_w != nullptr, "plan_create: null argument");
  B200_REQUIRE(nlat >= 1 && nlon >= 2 && lmax >= 1 && mmax >= 1 && m_offset >= 0, "plan_create: bad sizes nlat=%d nlon=%d lmax=%d mmax=%d m_offset=%d", nlat,
               nlon, lmax, mmax, m_offset);
  B200_REQUIRE(m_offset + mmax <= nlon / 2 + 1, "plan_create: m_offset+mmax=%d exceeds nlon/2+1=%d", m_offset + mmax, nlon / 2 + 1);
  const int vector = (flags & B200SHT_PLAN_VECTOR) ? 1 : 0;
  B200_REQUIRE(!vector || !(flags & B200SHT_PLAN_FFT_ONLY), "plan_create: a vector plan holds tables (B200SHT_PLAN_VECTOR with B200SHT_PLAN_FFT_ONLY)");
  B200_REQUIRE(!vector || lmax <= (1 << 29), "plan_create: lmax=%d too large", lmax);
  b200sht_plan* pl = new b200sht_plan();
  memset(static_cast<Plan*>(pl), 0, sizeof(Plan));
  pl->nlat = nlat; pl->nlon = nlon; pl->lmax = vector ? 2 * lmax : lmax; pl->mmax = mmax; pl->kp = round_up(nlat, 8); pl->csphase = csphase;
  pl->m0 = m_offset; pl->no_table = (flags & B200SHT_PLAN_FFT_ONLY) ? 1 : 0; pl->vector = vector;
  if (!make_fft_plan(nlon, &pl->fft)) {
    set_error("plan_create: nlon=%d has a prime factor > 13 (unsupported FFT length)", nlon);
    delete pl;
    return B200SHT_ERR_UNSUPPORTED;
  }
  cudaStream_t st = S(stream);
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&pl->sm_count, cudaDevAttrMultiProcessorCount, dev);
  const size_t tbytes = pl->no_table ? 16 : sizeof(float) * (size_t)mmax * pl->lmax * pl->kp;
  double* d_cost = nullptr;
  if (e == cudaSuccess) e = cudaMalloc(&pl->d_table, tbytes);
  if (e == cudaSuccess) e = cudaMalloc(&pl->d_rowscale, sizeof(float) * pl->kp);
  if (e == cudaSuccess) e = cudaMalloc(&pl->d_twiddle, sizeof(float2) * nlon);
  if (e == cudaSuccess) e = cudaMalloc(&d_cost, sizeof(double) * nlat);
  if (e != cudaSuccess) {
    set_error("plan_create: allocation failed: %s", cudaGetErrorString(e));
    cudaFree(pl->d_table); cudaFree(pl->d_rowscale); cudaFree(pl->d_twiddle); cudaFree(d_cost);
    delete pl;
    return B200SHT_ERR_NOMEM;
  }
  std::vector<float> rs(pl->kp, 0.f);
  for (int k = 0; k < nlat; ++k) rs[k] = (float)(quad_w[k] * 2.0 * M_PI / (double)nlon);
  std::vector<float2> tw(nlon);
  for (int t = 0; t < nlon; ++t) {
    const double ang = -2.0 * M_PI * (double)t / (double)nlon;
    tw[t] = make_float2((float)cos(ang), (float)sin(ang));
  }
  int rc = 0;
  do {
    if ((e = cudaMemcpyAsync(pl->d_rowscale, rs.data(), sizeof(float) * pl->kp, cudaMemcpyHostToDevice, st)) != cudaSuccess) break;
    if ((e = cudaMemcpyAsync(pl->d_twiddle, tw.data(), sizeof(float2) * nlon, cudaMemcpyHostToDevice, st)) != cudaSuccess) break;
    if ((e = cudaMemcpyAsync(d_cost, cost, sizeof(double) * nlat, cudaMemcpyHostToDevice, st)) != cudaSuccess) break;
    if (!pl->no_table) rc = build_table(pl, d_cost, st);
    if (rc) break;
    // host staging vectors go out of scope: wait for the copies (plan creation is not on the hot path)
    e = cudaStreamSynchronize(st);
  } while (0);
  cudaFree(d_cost);
  if (e != cudaSuccess || rc != 0) {
    if (e != cudaSuccess) set_error("plan_create: %s", cudaGetErrorString(e));
    cudaFree(pl->d_table); cudaFree(pl->d_rowscale); cudaFree(pl->d_twiddle);
    delete pl;
    return rc ? rc : B200SHT_ERR_CUDA;
  }
  pl->umma_ok = (!pl->no_table && umma_plan_init(pl) == 0) ? 1 : 0;
  dft_plan_init(pl);   // optional: leaves dft_state null when the grid is outside the tensor-core DFT's range
  *out = pl;
  return 0;
}

int b200sht_plan_destroy(b200sht_plan* pl) {
  if (!pl) return 0;
  umma_plan_destroy(pl);
  dft_plan_destroy(pl);
  cudaFree(pl->d_table);
  cudaFree(pl->d_rowscale);
  cudaFree(pl->d_twiddle);
  delete pl;
  return 0;
}

int64_t b200sht_plan_query(const b200sht_plan* pl, int what) {
  if (!pl) return -1;
  switch (what) {
    case 0: return pl->nlat;
    case 1: return pl->nlon;
    case 2: return pl->vector ? pl->lmax / 2 : pl->lmax;
    case 3: return pl->mmax;
    case 4: return pl->kp;
    case 5: return (int64_t)sizeof(float) * pl->mmax * pl->lmax * pl->kp;
    case 6: return pl->umma_ok;
    case 7: return pl->m0;
    case 8: return (pl->umma_ok && dft_usable(pl)) ? 1 : 0;
    case 9: return pl->vector;
    default: return -1;
  }
}

const float* b200sht_plan_table(const b200sht_plan* pl) { return pl ? pl->d_table : nullptr; }
int b200sht_plan_copy_table(const b200sht_plan* pl, float* dst, void* stream) {
  B200_REQUIRE(pl && dst, "plan_copy_table: null argument");
  if (pl->vector) {   // D [mmax][lmax][kp], then Q: the two halves of each order's rows
    const size_t half = sizeof(float) * (size_t)(pl->lmax / 2) * pl->kp;
    for (int t = 0; t < 2; ++t)
      B200_CHECK_CUDA(cudaMemcpy2DAsync(reinterpret_cast<char*>(dst) + t * half * pl->mmax, half, reinterpret_cast<const char*>(pl->d_table) + t * half,
                                        2 * half, half, pl->mmax, cudaMemcpyDeviceToDevice, S(stream)));
    return 0;
  }
  B200_CHECK_CUDA(cudaMemcpyAsync(dst, pl->d_table, sizeof(float) * (size_t)pl->mmax * pl->lmax * pl->kp, cudaMemcpyDeviceToDevice, S(stream)));
  return 0;
}

// orders are padded to a multiple of 8: the tensor-core DFT reads the latspec planes in residue classes m = c + 8 * m2
int64_t b200sht_latspec_elems(const b200sht_plan* pl, int B, int C) { return (int64_t)round_up(pl->mmax, 8) * 2 * B * C * pl->kp; }
int64_t b200sht_spec_elems(const b200sht_plan* pl, int B, int C) { return (int64_t)pl->lmax * pl->mmax * 2 * B * cp_of(C); }
int64_t b200sht_spec_elems_lm(int L, int M, int B, int C) { return (int64_t)L * M * 2 * B * cp_of(C); }

// -------------------------------------------------------------------------------------------- stages
int b200sht_fft_analysis(const b200sht_plan* pl, const void* x, int dtype, int B, int C, float* latspec, int scale_mode, void* stream) {
  B200_REQUIRE(pl && x && latspec, "fft_analysis: null argument");
  B200_REQUIRE(scale_mode >= 0 && scale_mode <= 3, "fft_analysis: bad scale_mode %d", scale_mode);
  return fft_analysis(pl, x, dtype, B, C, latspec, scale_mode, S(stream));
}

int b200sht_fft_synthesis(const b200sht_plan* pl, const float* latspec, void* y, int dtype, int B, int C, const float* bias, int scale_mode,
                          void* stream) {
  B200_REQUIRE(pl && y && latspec, "fft_synthesis: null argument");
  B200_REQUIRE(scale_mode >= 0 && scale_mode <= 3, "fft_synthesis: bad scale_mode %d", scale_mode);
  return fft_synthesis(pl, latspec, y, dtype, B, C, bias, scale_mode, S(stream));
}

// ---------------------------------------------------------------------------------- fp32 operands on the tensor cores
// B200SHT_PREC_FP32X3: the Legendre stages run as 3 x TF32 (hi.hi + hi.lo + lo.hi with fp32 accumulation in registers) instead of the CUDA-core
// kernels.  The residual of the activation operand lives in a per-device scratch buffer that grows on demand: calls of this mode on one
// device must be issued from one stream at a time (they are stream-ordered through the same buffer).
static float* residual_scratch(size_t bytes) {
  struct Pool { float* p = nullptr; size_t n = 0; };
  static std::mutex mu;
  static Pool pools[64];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return nullptr;
  std::lock_guard<std::mutex> lock(mu);
  Pool& pool = pools[dev];
  if (pool.n < bytes) {
    if (pool.p) cudaFree(pool.p);   // synchronises the device: no kernel still reads the old buffer
    pool.p = nullptr; pool.n = 0;
    if (cudaMalloc(&pool.p, bytes) != cudaSuccess) { pool.p = nullptr; return nullptr; }
    pool.n = bytes;
  }
  return pool.p;
}

static int check_precision(int umma_ok, int precision, const char* who) {
  if (precision == B200SHT_PREC_FP32) return 0;
  if (precision == B200SHT_PREC_TF32 || precision == B200SHT_PREC_FP32X3) {
    if (!umma_ok) {
      set_error("%s: the tensor-core (TF32 / 3 x TF32) path is not available on this device/build (it needs sm_90); refusing to fall back silently", who);
      return B200SHT_ERR_UNSUPPORTED;
    }
    return 0;
  }
  set_error("%s: unknown precision %d", who, precision);
  return B200SHT_ERR_INVALID;
}

}  // extern "C"
// The Legendre stages on any plan with a table: the scalar entry points below serve scalar plans, the vector ones (b200sht_vector_*) run the
// same contractions on a vector plan's stacked D / Q table with the 2C component rows of C vector fields.
static int legendre_analysis_any(const b200sht_plan* pl, const float* latspec, float* spec, int B, int C, int precision, void* stream) {
  B200_REQUIRE(pl && latspec && spec && B > 0 && C > 0, "legendre_analysis: bad argument");
  B200_REQUIRE(!pl->no_table, "legendre_analysis: FFT-only plan");
  int rc = check_precision(pl->umma_ok, precision, "legendre_analysis");
  if (rc) return rc;
  if (precision == B200SHT_PREC_TF32) return legendre_analysis_umma(pl, latspec, spec, B, C, S(stream));
  if (precision == B200SHT_PREC_FP32X3) {
    const size_t n = (size_t)pl->mmax * 2 * B * C * pl->kp;
    float* lo = residual_scratch(n * sizeof(float));
    B200_REQUIRE(lo != nullptr, "legendre_analysis (3 x TF32): cannot allocate %zu bytes of scratch", n * sizeof(float));
    rc = umma_plan_table_lo(pl);
    if (!rc) rc = tf32_residual(latspec, lo, n, S(stream));
    if (!rc) rc = legendre_analysis_umma(pl, latspec, spec, B, C, S(stream), lo);
    return rc;
  }
  return legendre_analysis_simt(pl, latspec, spec, B, C, S(stream));
}

static int legendre_synthesis_any(const b200sht_plan* pl, const float* spec, float* latspec, int B, int C, int precision, void* stream) {
  B200_REQUIRE(pl && latspec && spec && B > 0 && C > 0, "legendre_synthesis: bad argument");
  B200_REQUIRE(!pl->no_table, "legendre_synthesis: FFT-only plan");
  int rc = check_precision(pl->umma_ok, precision, "legendre_synthesis");
  if (rc) return rc;
  if (precision == B200SHT_PREC_TF32) return legendre_synthesis_umma(pl, spec, latspec, B, C, 0, S(stream));
  if (precision == B200SHT_PREC_FP32X3) {
    const size_t n = (size_t)b200sht_spec_elems(pl, B, C);
    float* lo = residual_scratch(n * sizeof(float));
    B200_REQUIRE(lo != nullptr, "legendre_synthesis (3 x TF32): cannot allocate %zu bytes of scratch", n * sizeof(float));
    rc = umma_plan_table_lo(pl);
    if (!rc) rc = tf32_residual(spec, lo, n, S(stream));
    if (!rc) rc = legendre_synthesis_umma(pl, spec, latspec, B, C, 0, S(stream), lo);
    return rc;
  }
  return legendre_synthesis_simt(pl, spec, latspec, B, C, S(stream));
}

static int legendre_synthesis_tiled_any(const b200sht_plan* pl, const float* spec, float* latspec, int B, int C, void* stream) {
  B200_REQUIRE(pl && latspec && spec && B > 0 && C > 0, "legendre_synthesis_tiled: bad argument");
  B200_REQUIRE(!pl->no_table, "legendre_synthesis_tiled: FFT-only plan");
  B200_REQUIRE(pl->umma_ok && dft_usable(pl), "legendre_synthesis_tiled: the tensor-core DFT is not available for this plan (b200sht_plan_query(plan, 8) == 0)");
  return legendre_synthesis_umma(pl, spec, latspec, B, C, 1, S(stream));
}
extern "C" {

#define B200_SCALAR_PLAN(pl, who) B200_REQUIRE((pl) == nullptr || !(pl)->vector, who ": vector plan given to a scalar-transform entry point (use b200sht_vector_* / b200sht_vsht_*)")
#define B200_VECTOR_PLAN(pl, who) B200_REQUIRE((pl) != nullptr && (pl)->vector, who ": needs a vector plan (b200sht_plan_create_ex with B200SHT_PLAN_VECTOR)")

int b200sht_legendre_analysis(const b200sht_plan* pl, const float* latspec, float* spec, int B, int C, int precision, void* stream) {
  B200_SCALAR_PLAN(pl, "legendre_analysis");
  return legendre_analysis_any(pl, latspec, spec, B, C, precision, stream);
}
int b200sht_legendre_synthesis(const b200sht_plan* pl, const float* spec, float* latspec, int B, int C, int precision, void* stream) {
  B200_SCALAR_PLAN(pl, "legendre_synthesis");
  return legendre_synthesis_any(pl, spec, latspec, B, C, precision, stream);
}
int b200sht_legendre_synthesis_tiled(const b200sht_plan* pl, const float* spec, float* latspec, int B, int C, void* stream) {
  B200_SCALAR_PLAN(pl, "legendre_synthesis_tiled");
  return legendre_synthesis_tiled_any(pl, spec, latspec, B, C, stream);
}

// Legendre synthesis + longitude synthesis: through the tiled latspec layout and the tensor-core DFT when the plan supports it at TF32
static int synthesis_pair(const b200sht_plan* pl, const float* spec, float* lat, void* y, int dtype, int B, int C, const float* bias, int mode,
                          int precision, void* stream) {
  if (precision == B200SHT_PREC_TF32 && pl->umma_ok && dft_usable(pl)) {
    int rc = legendre_synthesis_tiled_any(pl, spec, lat, B, C, stream);
    if (!rc) rc = b200sht_fft_synthesis(pl, lat, y, dtype, B, C, bias, mode | 2, stream);
    return rc;
  }
  int rc = legendre_synthesis_any(pl, spec, lat, B, C, precision, stream);
  if (!rc) rc = b200sht_fft_synthesis(pl, lat, y, dtype, B, C, bias, mode, stream);
  return rc;
}

// Longitude analysis + Legendre analysis
static int analysis_pair(const b200sht_plan* pl, const void* x, int dtype, int B, int C, float* lat, float* spec, int mode, int precision, void* stream) {
  int rc = b200sht_fft_analysis(pl, x, dtype, B, C, lat, mode | (precision == B200SHT_PREC_TF32 ? 2 : 0), stream);
  if (!rc) rc = legendre_analysis_any(pl, lat, spec, B, C, precision, stream);
  return rc;
}

int b200sht_spec_unpack(int L, int M, const float* spec, void* coeffs, int B, int C, void* stream) {
  B200_REQUIRE(L > 0 && M > 0 && spec && coeffs, "spec_unpack: bad argument");
  Plan p = lm_plan(L, M);
  return spec_unpack(&p, spec, coeffs, B, C, S(stream));
}
int b200sht_spec_pack(int L, int M, const void* coeffs, float* spec, int B, int C, void* stream) {
  B200_REQUIRE(L > 0 && M > 0 && spec && coeffs, "spec_pack: bad argument");
  Plan p = lm_plan(L, M);
  return spec_pack(&p, coeffs, spec, B, C, S(stream));
}

int b200sht_spec_unpack_ex(int L, int M, int m_offset, int dense, const float* spec, void* coeffs, int B, int C, void* stream) {
  B200_REQUIRE(L > 0 && M > 0 && spec && coeffs, "spec_unpack: bad argument");
  Plan p = lm_plan(L, M, m_offset, dense);
  return spec_unpack(&p, spec, coeffs, B, C, S(stream));
}
int b200sht_spec_pack_ex(int L, int M, int m_offset, int dense, const void* coeffs, float* spec, int B, int C, void* stream) {
  B200_REQUIRE(L > 0 && M > 0 && spec && coeffs, "spec_pack: bad argument");
  Plan p = lm_plan(L, M, m_offset, dense);
  return spec_pack(&p, coeffs, spec, B, C, S(stream));
}
int b200sht_latspec_unpack(const b200sht_plan* pl, const float* latspec, void* coeffs, int B, int C, void* stream) {
  B200_REQUIRE(pl && latspec && coeffs, "latspec_unpack: null argument");
  return latspec_convert(pl, const_cast<float*>(latspec), coeffs, B, C, 0, S(stream));
}
int b200sht_latspec_pack(const b200sht_plan* pl, const void* coeffs, float* latspec, int B, int C, void* stream) {
  B200_REQUIRE(pl && latspec && coeffs, "latspec_pack: null argument");
  return latspec_convert(pl, latspec, const_cast<void*>(coeffs), B, C, 1, S(stream));
}

int b200sht_bias_grad(const b200sht_plan* pl, const float* latspec, float* gbias, int B, int C, void* stream) {
  B200_REQUIRE(pl && latspec && gbias, "bias_grad: null argument");
  return bias_grad(pl, latspec, gbias, B, C, S(stream));
}

// ------------------------------------------------------------------------- torch-harmonics boundary
static inline size_t align256(size_t b) { return (b + 255) / 256 * 256; }

int64_t b200sht_sht_workspace_bytes(const b200sht_plan* pl, int B, int C) {
  return (int64_t)(align256(sizeof(float) * b200sht_latspec_elems(pl, B, C)) + align256(sizeof(float) * b200sht_spec_elems(pl, B, C)));
}

static void split_ws(const b200sht_plan* pl, int B, int C, void* ws, float** latspec, float** spec) {
  *latspec = static_cast<float*>(ws);
  *spec = reinterpret_cast<float*>(static_cast<char*>(ws) + align256(sizeof(float) * b200sht_latspec_elems(pl, B, C)));
}

int b200sht_sht_forward(const b200sht_plan* pl, const void* x, int dtype, int B, int C, void* coeffs, void* ws, int precision, void* stream) {
  B200_REQUIRE(pl && x && coeffs && ws, "sht_forward: null argument");
  B200_SCALAR_PLAN(pl, "sht_forward");
  float *X, *sp;
  split_ws(pl, B, C, ws, &X, &sp);
  int rc = analysis_pair(pl, x, dtype, B, C, X, sp, 0, precision, stream);
  if (!rc) rc = b200sht_spec_unpack(pl->lmax, pl->mmax, sp, coeffs, B, C, stream);
  return rc;
}

int b200sht_sht_inverse(const b200sht_plan* pl, const void* coeffs, void* y, int dtype, int B, int C, void* ws, int precision, void* stream) {
  B200_REQUIRE(pl && y && coeffs && ws, "sht_inverse: null argument");
  B200_SCALAR_PLAN(pl, "sht_inverse");
  float *Z, *sp;
  split_ws(pl, B, C, ws, &Z, &sp);
  int rc = b200sht_spec_pack(pl->lmax, pl->mmax, coeffs, sp, B, C, stream);
  if (!rc) rc = synthesis_pair(pl, sp, Z, y, dtype, B, C, nullptr, 0, precision, stream);
  return rc;
}

int b200sht_sht_forward_adjoint(const b200sht_plan* pl, const void* gcoeffs, void* gx, int dtype, int B, int C, void* ws, int precision,
                                void* stream) {
  B200_REQUIRE(pl && gx && gcoeffs && ws, "sht_forward_adjoint: null argument");
  B200_SCALAR_PLAN(pl, "sht_forward_adjoint");
  float *Z, *sp;
  split_ws(pl, B, C, ws, &Z, &sp);
  int rc = b200sht_spec_pack(pl->lmax, pl->mmax, gcoeffs, sp, B, C, stream);
  if (!rc) rc = synthesis_pair(pl, sp, Z, gx, dtype, B, C, nullptr, 1, precision, stream);
  return rc;
}

int b200sht_sht_inverse_adjoint(const b200sht_plan* pl, const void* gy, int dtype, int B, int C, void* gcoeffs, void* ws, int precision,
                                void* stream) {
  B200_REQUIRE(pl && gy && gcoeffs && ws, "sht_inverse_adjoint: null argument");
  B200_SCALAR_PLAN(pl, "sht_inverse_adjoint");
  float *X, *sp;
  split_ws(pl, B, C, ws, &X, &sp);
  int rc = analysis_pair(pl, gy, dtype, B, C, X, sp, 1, precision, stream);
  if (!rc) rc = b200sht_spec_unpack(pl->lmax, pl->mmax, sp, gcoeffs, B, C, stream);
  return rc;
}

// ---------------------------------------------------------------------------------- vector SHT boundary
// Stage buffers of C vector fields are the scalar formats of their 2C component rows (b, c, component), with the vector plan's 2 lmax table rows.
static int vector_precision(int precision, const char* who) {
  if (precision == B200SHT_PREC_FP32X3) {
    set_error("%s: the vector transforms have no 3 x TF32 mode (use B200SHT_PREC_FP32 or B200SHT_PREC_TF32)", who);
    return B200SHT_ERR_UNSUPPORTED;
  }
  return 0;
}
#define B200_VECTOR_ARGS(pl, C, precision, who)                                                              \
  B200_VECTOR_PLAN(pl, who);                                                                                 \
  B200_REQUIRE((C) > 0 && (C) <= (1 << 28), who ": bad channel count %d", (C));                             \
  if (int _rc = vector_precision(precision, who)) return _rc
// the one-call entries and the tiled synthesis run the longitude stage (or the tensor-core DFT's tiled layout) over orders 0 .. mmax - 1: they
// need the plan of all orders, not an order shard of the distributed transforms
#define B200_VECTOR_ALL_ORDERS(pl, who) \
  B200_REQUIRE((pl)->m0 == 0, who ": vector plan with order offset %d (an order shard serves the stage entry points only)", (pl)->m0)

int b200sht_vector_legendre_analysis(const b200sht_plan* pl, const float* latspec, float* spec, int B, int C, int precision, void* stream) {
  B200_VECTOR_ARGS(pl, C, precision, "vector_legendre_analysis");
  return legendre_analysis_any(pl, latspec, spec, B, 2 * C, precision, stream);
}
int b200sht_vector_legendre_synthesis(const b200sht_plan* pl, const float* spec, float* latspec, int B, int C, int precision, void* stream) {
  B200_VECTOR_ARGS(pl, C, precision, "vector_legendre_synthesis");
  return legendre_synthesis_any(pl, spec, latspec, B, 2 * C, precision, stream);
}
int b200sht_vector_legendre_synthesis_tiled(const b200sht_plan* pl, const float* spec, float* latspec, int B, int C, void* stream) {
  B200_VECTOR_ARGS(pl, C, B200SHT_PREC_TF32, "vector_legendre_synthesis_tiled");
  B200_VECTOR_ALL_ORDERS(pl, "vector_legendre_synthesis_tiled");
  return legendre_synthesis_tiled_any(pl, spec, latspec, B, 2 * C, stream);
}
int b200sht_vector_spec_unpack(const b200sht_plan* pl, const float* spec, void* coeffs, int B, int C, int scaled, void* stream) {
  B200_VECTOR_ARGS(pl, C, B200SHT_PREC_FP32, "vector_spec_unpack");
  B200_REQUIRE(spec && coeffs && B > 0, "vector_spec_unpack: bad argument");
  return vector_spec_convert(pl, const_cast<float*>(spec), coeffs, B, C, 0, scaled ? 1 : 0, S(stream));
}
int b200sht_vector_spec_pack(const b200sht_plan* pl, const void* coeffs, float* spec, int B, int C, int scaled, void* stream) {
  B200_VECTOR_ARGS(pl, C, B200SHT_PREC_FP32, "vector_spec_pack");
  B200_REQUIRE(spec && coeffs && B > 0, "vector_spec_pack: bad argument");
  return vector_spec_convert(pl, spec, const_cast<void*>(coeffs), B, C, 1, scaled ? 1 : 0, S(stream));
}

int64_t b200sht_vsht_workspace_bytes(const b200sht_plan* pl, int B, int C) {
  if (!pl || !pl->vector || pl->m0 != 0 || B <= 0 || C <= 0 || C > (1 << 28)) return -1;
  return b200sht_sht_workspace_bytes(pl, B, 2 * C);
}

int b200sht_vsht_forward(const b200sht_plan* pl, const void* x, int dtype, int B, int C, void* coeffs, void* ws, int precision, void* stream) {
  B200_VECTOR_ARGS(pl, C, precision, "vsht_forward");
  B200_VECTOR_ALL_ORDERS(pl, "vsht_forward");
  B200_REQUIRE(x && coeffs && ws && B > 0, "vsht_forward: bad argument");
  float *X, *sp;
  split_ws(pl, B, 2 * C, ws, &X, &sp);
  int rc = analysis_pair(pl, x, dtype, B, 2 * C, X, sp, 0, precision, stream);
  if (!rc) rc = vector_spec_convert(pl, sp, coeffs, B, C, 0, 1, S(stream));
  return rc;
}

int b200sht_vsht_inverse(const b200sht_plan* pl, const void* coeffs, void* y, int dtype, int B, int C, void* ws, int precision, void* stream) {
  B200_VECTOR_ARGS(pl, C, precision, "vsht_inverse");
  B200_VECTOR_ALL_ORDERS(pl, "vsht_inverse");
  B200_REQUIRE(y && coeffs && ws && B > 0, "vsht_inverse: bad argument");
  float *Z, *sp;
  split_ws(pl, B, 2 * C, ws, &Z, &sp);
  int rc = vector_spec_convert(pl, sp, const_cast<void*>(coeffs), B, C, 1, 0, S(stream));
  if (!rc) rc = synthesis_pair(pl, sp, Z, y, dtype, B, 2 * C, nullptr, 0, precision, stream);
  return rc;
}

int b200sht_vsht_forward_adjoint(const b200sht_plan* pl, const void* gcoeffs, void* gx, int dtype, int B, int C, void* ws, int precision,
                                 void* stream) {
  B200_VECTOR_ARGS(pl, C, precision, "vsht_forward_adjoint");
  B200_VECTOR_ALL_ORDERS(pl, "vsht_forward_adjoint");
  B200_REQUIRE(gx && gcoeffs && ws && B > 0, "vsht_forward_adjoint: bad argument");
  float *Z, *sp;
  split_ws(pl, B, 2 * C, ws, &Z, &sp);
  int rc = vector_spec_convert(pl, sp, const_cast<void*>(gcoeffs), B, C, 1, 1, S(stream));
  if (!rc) rc = synthesis_pair(pl, sp, Z, gx, dtype, B, 2 * C, nullptr, 1, precision, stream);
  return rc;
}

int b200sht_vsht_inverse_adjoint(const b200sht_plan* pl, const void* gy, int dtype, int B, int C, void* gcoeffs, void* ws, int precision,
                                 void* stream) {
  B200_VECTOR_ARGS(pl, C, precision, "vsht_inverse_adjoint");
  B200_VECTOR_ALL_ORDERS(pl, "vsht_inverse_adjoint");
  B200_REQUIRE(gy && gcoeffs && ws && B > 0, "vsht_inverse_adjoint: bad argument");
  float *X, *sp;
  split_ws(pl, B, 2 * C, ws, &X, &sp);
  int rc = analysis_pair(pl, gy, dtype, B, 2 * C, X, sp, 1, precision, stream);
  if (!rc) rc = vector_spec_convert(pl, sp, gcoeffs, B, C, 0, 0, S(stream));
  return rc;
}

// --------------------------------------------------------------------------------------- channel mix
int64_t b200sht_mix_weight_elems(int op, int L, int M, int G, int Ci, int Co) {
  if (G <= 0 || Ci % G || Co % G) return -1;
  const int64_t Cig = Ci / G, Cog = Co / G, cop = round_up((int)Cog, 4);
  switch (op) {
    case B200SHT_OP_DHCONV: return (int64_t)L * G * Cig * cop * 2;
    case B200SHT_OP_LDEP: return (int64_t)L * Cig * cop * 2;
    case B200SHT_OP_SHARED: return Cig * cop * 2;
    case B200SHT_OP_DIAGONAL: return (int64_t)G * Cig * Cog * L * M * 2;
    case B200SHT_OP_SEP_DHCONV: return (int64_t)G * Cig * L * 2;
    case B200SHT_OP_SEP_DIAGONAL: return (int64_t)G * Cig * L * M * 2;
    default: return -1;
  }
}

int b200sht_mix_weight_pack(int op, const void* w_native, float* w_packed, int L, int G, int Ci, int Co, int precision, void* stream) {
  B200_REQUIRE(w_native && w_packed, "mix_weight_pack: null argument");
  return mix_weight_relayout(op, w_native, w_packed, L, G, Ci, Co, 0, precision == B200SHT_PREC_TF32, S(stream));
}
int b200sht_mix_weight_unpack(int op, const float* w_packed, void* w_native, int L, int G, int Ci, int Co, void* stream) {
  B200_REQUIRE(w_native && w_packed, "mix_weight_unpack: null argument");
  return mix_weight_relayout(op, w_native, const_cast<float*>(w_packed), L, G, Ci, Co, 1, 0, S(stream));
}

static bool dense_op(int op) { return op == B200SHT_OP_DHCONV || op == B200SHT_OP_SHARED || op == B200SHT_OP_LDEP; }
// The tensor-core mix addresses operands with TMA: group slices must start on 16-byte boundaries and the batch must divide 32.
// Other shapes (none of the shipped configs: G = 1, B = 1 per GPU) are served by the fp32 CUDA-core kernels.
static bool umma_mix_shape(int B, int G, int Ci, int Co) {
  return B >= 1 && 32 % B == 0 && (G == 1 || ((Ci / G) % 4 == 0 && (Co / G) % 4 == 0));
}

int b200sht_mix_uses_tensor_cores(int op, int B, int G, int Ci, int Co, int precision) {
  if (G <= 0 || Ci % G != 0 || Co % G != 0) return 0;
  return (precision == B200SHT_PREC_TF32 && dense_op(op & 0xff) && umma_mix_shape(B, G, Ci, Co)) ? 1 : 0;
}

int b200sht_mix_forward(int L, int M, int op, const float* x, const void* w, const void* cbias, float* y, int B, int G, int Ci, int Co,
                        int precision, void* stream) {
  B200_REQUIRE(L > 0 && M > 0 && x && w && y, "mix_forward: bad argument");
  int rc = check_precision(umma_available(), precision, "mix_forward");
  if (rc) return rc;
  Plan p = lm_plan(L, M, 0, (op & kDenseFlag) ? 1 : 0);
  op &= 0xff;
  const Plan* pl = &p;
  if (precision == B200SHT_PREC_TF32 && dense_op(op) && umma_mix_shape(B, G, Ci, Co)) return mix_forward_umma(pl, op, x, w, cbias, y, B, G, Ci, Co, S(stream));
  return mix_forward_simt(pl, op, x, w, cbias, y, B, G, Ci, Co, S(stream));  // per-mode operators are bandwidth bound: one path
}

int b200sht_mix_backward(int L, int M, int op, const float* x, const void* w, const float* gy, float* gx, void* gw, void* gcbias, int B,
                         int G, int Ci, int Co, int precision, void* stream) {
  B200_REQUIRE(L > 0 && M > 0 && w && gy, "mix_backward: bad argument");
  B200_REQUIRE(gw == nullptr || x != nullptr, "mix_backward: weight gradient needs x");
  int rc = check_precision(umma_available(), precision, "mix_backward");
  if (rc) return rc;
  Plan p = lm_plan(L, M, 0, (op & kDenseFlag) ? 1 : 0);
  op &= 0xff;
  const Plan* pl = &p;
  if (precision == B200SHT_PREC_TF32 && dense_op(op) && umma_mix_shape(B, G, Ci, Co)) return mix_backward_umma(pl, op, x, w, gy, gx, gw, gcbias, B, G, Ci, Co, S(stream));
  return mix_backward_simt(pl, op, x, w, gy, gx, gw, gcbias, B, G, Ci, Co, S(stream));
}

int b200sht_complex_relu_forward(int L, int M, int mode, const float* x, const float* bias, float slope, float* y, int B, int C,
                                 void* stream) {
  B200_REQUIRE(L > 0 && M > 0 && x && y, "complex_relu_forward: bad argument");
  Plan p = lm_plan(L, M, 0, (mode & kDenseFlag) ? 1 : 0);
  mode &= 0xff;
  return complex_relu_fwd(&p, mode, x, bias, slope, y, B, C, S(stream));
}
int b200sht_complex_relu_backward(int L, int M, int mode, const float* x, const float* bias, float slope, const float* gy, float* gx,
                                  float* gbias, int B, int C, void* stream) {
  B200_REQUIRE(L > 0 && M > 0 && x && gy && gx, "complex_relu_backward: bad argument");
  Plan p = lm_plan(L, M, 0, (mode & kDenseFlag) ? 1 : 0);
  mode &= 0xff;
  return complex_relu_bwd(&p, mode, x, bias, slope, gy, gx, gbias, B, C, S(stream));
}

// ---------------------------------------------------------------------------- SpectralConv, one call
struct ConvWs {
  float *lat_in, *spec_in, *spec_out, *lat_out;
  size_t total;
};

static ConvWs conv_ws(const b200sht_plan* f, const b200sht_plan* v, const b200sht_conv_desc* d, void* base) {
  ConvWs w;
  const int Cmax = d->Cin > d->Cout ? d->Cin : d->Cout;
  size_t off = 0;
  char* b = static_cast<char*>(base);
  w.lat_in = reinterpret_cast<float*>(b + off); off += align256(sizeof(float) * b200sht_latspec_elems(f, d->B, Cmax));
  w.spec_in = reinterpret_cast<float*>(b + off); off += align256(sizeof(float) * b200sht_spec_elems(f, d->B, Cmax));
  w.spec_out = reinterpret_cast<float*>(b + off); off += align256(sizeof(float) * b200sht_spec_elems(f, d->B, Cmax));
  w.lat_out = reinterpret_cast<float*>(b + off); off += align256(sizeof(float) * b200sht_latspec_elems(v, d->B, Cmax));
  w.total = off;
  return w;
}

static int check_conv(const b200sht_plan* f, const b200sht_plan* v, const b200sht_conv_desc* d) {
  B200_REQUIRE(f && v && d, "spectral_conv: null argument");
  B200_REQUIRE(!f->vector && !v->vector, "spectral_conv: vector plan given to a scalar-transform entry point");
  B200_REQUIRE(f->lmax == v->lmax && f->mmax == v->mmax, "spectral_conv: forward (%d,%d) and inverse (%d,%d) mode counts differ", f->lmax, f->mmax,
               v->lmax, v->mmax);
  B200_REQUIRE(d->B > 0 && d->G > 0 && d->Cin % d->G == 0 && d->Cout % d->G == 0, "spectral_conv: channels (%d,%d) not divisible by groups %d", d->Cin,
               d->Cout, d->G);
  return 0;
}

int64_t b200sht_spectral_conv_workspace_bytes(const b200sht_plan* f, const b200sht_plan* v, const b200sht_conv_desc* d) {
  if (check_conv(f, v, d)) return -1;
  return (int64_t)conv_ws(f, v, d, nullptr).total;
}

int b200sht_spectral_conv_forward(const b200sht_plan* f, const b200sht_plan* v, const b200sht_conv_desc* d, const void* x, const void* w,
                                  const float* bias, void* y, void* residual, float* spec_x_saved, void* workspace, void* stream) {
  int rc = check_conv(f, v, d);
  if (rc) return rc;
  B200_REQUIRE(x && w && y && workspace, "spectral_conv_forward: null argument");
  ConvWs ws = conv_ws(f, v, d, workspace);
  float* spec_x = spec_x_saved ? spec_x_saved : ws.spec_in;
  rc = analysis_pair(f, x, d->dtype, d->B, d->Cin, ws.lat_in, spec_x, 0, d->precision, stream);
  if (!rc && residual) {
    rc = synthesis_pair(v, spec_x, ws.lat_out, residual, d->dtype, d->B, d->Cin, nullptr, 0, d->precision, stream);
  }
  if (!rc) rc = b200sht_mix_forward(f->lmax, f->mmax, d->op, spec_x, w, nullptr, ws.spec_out, d->B, d->G, d->Cin, d->Cout, d->precision, stream);
  if (!rc) rc = synthesis_pair(v, ws.spec_out, ws.lat_out, y, d->dtype, d->B, d->Cout, bias, 0, d->precision, stream);
  return rc;
}

// elementwise accumulate of two packed spec tensors (residual-path gradient)
__global__ void axpy_kernel(float* __restrict__ a, const float* __restrict__ b, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) a[i] += b[i];
}

int b200sht_spectral_conv_backward(const b200sht_plan* f, const b200sht_plan* v, const b200sht_conv_desc* d, const void* gy, const void* gresidual,
                                   const float* spec_x_saved, const void* w, void* gx, void* gw, float* gbias, void* workspace, void* stream) {
  return b200sht_spectral_conv_backward_ex(f, v, d, gy, gresidual, spec_x_saved, w, gx, gw, gbias, workspace, nullptr, nullptr, stream);
}

int b200sht_spectral_conv_backward_ex(const b200sht_plan* f, const b200sht_plan* v, const b200sht_conv_desc* d, const void* gy, const void* gresidual,
                                      const float* spec_x_saved, const void* w, void* gx, void* gw, float* gbias, void* workspace,
                                      void* gw_native, void* wgrad_ready_event, void* stream) {
  int rc = check_conv(f, v, d);
  if (rc) return rc;
  B200_REQUIRE(gy && w && workspace, "spectral_conv_backward: null argument");
  B200_REQUIRE(gw == nullptr || spec_x_saved != nullptr, "spectral_conv_backward: weight gradient needs the saved spectrum");
  ConvWs ws = conv_ws(f, v, d, workspace);
  // dL/d(spec_out) = analysis_v(fft_v(gy, adjoint scaling))
  rc = analysis_pair(v, gy, d->dtype, d->B, d->Cout, ws.lat_out, ws.spec_out, 1, d->precision, stream);
  if (!rc && gbias) rc = b200sht_bias_grad(v, ws.lat_out, gbias, d->B, d->Cout, stream);   // the m = 0 plane of the complete latspec
  // with an event to signal, the weight gradient goes first and the input gradient of the mix joins the overlapped stages below
  const bool split_mix = wgrad_ready_event != nullptr && gw != nullptr && gx != nullptr;
  if (!rc) rc = b200sht_mix_backward(f->lmax, f->mmax, d->op, spec_x_saved, w, ws.spec_out, (gx && !split_mix) ? ws.spec_in : nullptr, gw, nullptr, d->B, d->G,
                                     d->Cin, d->Cout, d->precision, stream);
  // the weight gradient is final here: hand it to the caller (native layout + event) BEFORE the two input-gradient stages, so that a
  // data-parallel all-reduce on another stream overlaps legendre_synthesis + fft_synthesis instead of trailing the whole backward pass
  if (!rc && gw && gw_native) {
    const bool dense = (d->op == B200SHT_OP_DHCONV || d->op == B200SHT_OP_SHARED || d->op == B200SHT_OP_LDEP);
    B200_REQUIRE(dense, "spectral_conv_backward_ex: gw_native is for the packed (dense) operators; the others already return the native layout");
    rc = b200sht_mix_weight_unpack(d->op, static_cast<const float*>(gw), gw_native, f->lmax, d->G, d->Cin, d->Cout, stream);
  }
  if (!rc && wgrad_ready_event) B200_CHECK_CUDA(cudaEventRecord(static_cast<cudaEvent_t>(wgrad_ready_event), S(stream)));
  // the caller overlaps a collective with what follows: leave it a few SMs (B200SHT_OVERLAP_SMS, default 8; 0 = none)
  struct ReserveGuard {
    int saved;
    explicit ReserveGuard(bool on) : saved(sm_reserve()) {
      static const int n = [] { const char* e = getenv("B200SHT_OVERLAP_SMS"); return e ? atoi(e) : 8; }();
      if (on) sm_reserve() = n;
    }
    ~ReserveGuard() { sm_reserve() = saved; }
  } reserve_guard(wgrad_ready_event != nullptr);
  if (!rc && split_mix)
    rc = b200sht_mix_backward(f->lmax, f->mmax, d->op, spec_x_saved, w, ws.spec_out, ws.spec_in, nullptr, nullptr, d->B, d->G, d->Cin, d->Cout, d->precision, stream);
  if (!rc && gx) {
    if (gresidual) {
      rc = analysis_pair(v, gresidual, d->dtype, d->B, d->Cin, ws.lat_out, ws.spec_out, 1, d->precision, stream);
      if (!rc) {
        const long long n = b200sht_spec_elems(f, d->B, d->Cin);
        axpy_kernel<<<(unsigned)((n + 255) / 256), 256, 0, S(stream)>>>(ws.spec_in, ws.spec_out, n);
        B200_CHECK_LAUNCH();
      }
    }
    if (!rc) rc = synthesis_pair(f, ws.spec_in, ws.lat_in, gx, d->dtype, d->B, d->Cin, nullptr, 1, d->precision, stream);
  }
  return rc;
}

int b200sht_spectral_conv_forward_host(const b200sht_plan* f, const b200sht_plan* v, const b200sht_conv_desc* d, const void* x_host,
                                       const void* w_device, const float* bias_device, void* y_host, void* stream) {
  int rc = check_conv(f, v, d);
  if (rc) return rc;
  B200_REQUIRE(x_host && w_device && y_host, "spectral_conv_forward_host: null argument");
  const size_t esz = d->dtype == B200SHT_BF16 ? 2 : 4;
  const size_t xin = esz * (size_t)d->B * d->Cin * f->nlat * f->nlon, yout = esz * (size_t)d->B * d->Cout * v->nlat * v->nlon;
  const size_t wsb = conv_ws(f, v, d, nullptr).total;
  char* dev = nullptr;
  cudaStream_t st = S(stream);
  B200_CHECK_CUDA(cudaMallocAsync(&dev, align256(xin) + align256(yout) + wsb, st));
  void* dx = dev;
  void* dy = dev + align256(xin);
  void* dws = dev + align256(xin) + align256(yout);
  cudaError_t e = cudaMemcpyAsync(dx, x_host, xin, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) {
    rc = b200sht_spectral_conv_forward(f, v, d, dx, w_device, bias_device, dy, nullptr, nullptr, dws, stream);
    if (!rc) e = cudaMemcpyAsync(y_host, dy, yout, cudaMemcpyDeviceToHost, st);
  }
  cudaFreeAsync(dev, st);
  cudaError_t e2 = cudaStreamSynchronize(st);
  if (e != cudaSuccess || e2 != cudaSuccess) {
    set_error("spectral_conv_forward_host: %s", cudaGetErrorString(e != cudaSuccess ? e : e2));
    return B200SHT_ERR_CUDA;
  }
  return rc;
}

}  // extern "C"
namespace b200sht {
static int& pdl_flag() {
  static int on = [] { const char* e = getenv("B200SHT_PDL"); return e ? atoi(e) : 1; }();
  return on;
}
bool pdl_enabled() { return pdl_flag() != 0; }
}  // namespace b200sht
extern "C" {

// ------------------------------------------------------------------------------ pointwise tail of the SFNO block (row N2)
int64_t b200sht_pointwise_workspace_floats(int B, int C, int64_t hw) {
  if (B <= 0 || C <= 0 || hw <= 0) return -1;
  return (int64_t)B * C * norm_splits(B * C, hw) * 2;
}
static int check_pointwise(const void* a, const void* b, int dtype, const char* who) {
  B200_REQUIRE(a && b, "%s: null argument", who);
  B200_REQUIRE(dtype == B200SHT_F32 || dtype == B200SHT_BF16, "%s: unknown dtype %d", who, dtype);
  return 0;
}
int b200sht_instance_norm_forward(const void* x, void* y, const float* gamma, const float* beta, float* stats, float* workspace, int dtype, int B, int C,
                                  int64_t hw, float eps, int gelu, void* stream) {
  int rc = check_pointwise(x, y, dtype, "instance_norm_forward");
  if (rc) return rc;
  B200_REQUIRE(stats && workspace, "instance_norm_forward: null stats / workspace");
  return instance_norm_forward(x, y, gamma, beta, stats, workspace, dtype, B, C, hw, eps, gelu, S(stream));
}
int b200sht_instance_norm_backward(const void* x, const void* dy, void* dx, const float* gamma, const float* beta, const float* stats, float* sums,
                                   float* workspace, int dtype, int B, int C, int64_t hw, int gelu, void* stream) {
  int rc = check_pointwise(x, dy, dtype, "instance_norm_backward");
  if (rc) return rc;
  B200_REQUIRE(dx && stats && sums && workspace, "instance_norm_backward: null argument");
  return instance_norm_backward(x, dy, dx, gamma, beta, stats, sums, workspace, dtype, B, C, hw, gelu, S(stream));
}
int b200sht_bias_gelu_forward(const void* x, const float* bias, void* y, int dtype, int B, int C, int64_t hw, void* stream) {
  int rc = check_pointwise(x, y, dtype, "bias_gelu_forward");
  if (rc) return rc;
  return bias_gelu_forward(x, bias, y, dtype, B, C, hw, S(stream));
}
int b200sht_bias_gelu_backward(const void* x, const float* bias, const void* dy, void* dx, float* row_sums, float* workspace, int dtype, int B, int C, int64_t hw,
                               void* stream) {
  int rc = check_pointwise(x, dy, dtype, "bias_gelu_backward");
  if (rc) return rc;
  B200_REQUIRE(dx && workspace, "bias_gelu_backward: null argument");
  return bias_gelu_backward(x, bias, dy, dx, row_sums, workspace, dtype, B, C, hw, S(stream));
}

// ------------------------------------------------------------------------------ quadrature-weighted instance norm on the sphere
int64_t b200sht_geometric_norm_workspace_floats(int B, int C, int64_t hw) {
  if (B <= 0 || C <= 0 || hw <= 0) return -1;
  return 2 * (int64_t)geometric_norm_workspace_doubles(B, C, hw);
}
static int check_aligned8(const void* p, const char* who) {
  B200_REQUIRE(p && (reinterpret_cast<uintptr_t>(p) & 7) == 0, "%s: null or not 8-byte aligned fp64 buffer", who);
  return 0;
}
int b200sht_geometric_norm_partials(const void* x, const float* q, double* partials, float* workspace, int dtype, int B, int C, int H, int W, void* stream) {
  int rc = check_pointwise(x, q, dtype, "geometric_norm_partials");
  if (!rc) rc = check_aligned8(partials, "geometric_norm_partials");
  if (!rc) rc = check_aligned8(workspace, "geometric_norm_partials");
  if (rc) return rc;
  return geometric_norm_partials(x, q, partials, reinterpret_cast<double*>(workspace), dtype, B, C, H, W, S(stream));
}
int b200sht_geometric_norm_finalize(const double* partials, int R, int rows, double D, float eps, float* stats, void* stream) {
  int rc = check_aligned8(partials, "geometric_norm_finalize");
  if (rc) return rc;
  B200_REQUIRE(stats, "geometric_norm_finalize: null stats");
  return geometric_norm_finalize(partials, R, rows, D, eps, stats, S(stream));
}
int b200sht_geometric_norm_apply(const void* x, void* y, const float* gamma, const float* beta, const float* stats, int dtype, int B, int C, int H, int W,
                                 int gelu, void* stream) {
  int rc = check_pointwise(x, y, dtype, "geometric_norm_apply");
  if (rc) return rc;
  B200_REQUIRE(stats, "geometric_norm_apply: null stats");
  return geometric_norm_apply(x, y, gamma, beta, stats, dtype, B, C, H, W, gelu, S(stream));
}
int b200sht_geometric_norm_backward_sums(const void* x, const void* dy, const float* gamma, const float* beta, const float* stats, double* sums,
                                         float* workspace, int dtype, int B, int C, int H, int W, int gelu, void* stream) {
  int rc = check_pointwise(x, dy, dtype, "geometric_norm_backward_sums");
  if (!rc) rc = check_aligned8(sums, "geometric_norm_backward_sums");
  if (!rc) rc = check_aligned8(workspace, "geometric_norm_backward_sums");
  if (rc) return rc;
  B200_REQUIRE(stats, "geometric_norm_backward_sums: null stats");
  return geometric_norm_backward_sums(x, dy, gamma, beta, stats, sums, reinterpret_cast<double*>(workspace), dtype, B, C, H, W, gelu, S(stream));
}
int b200sht_geometric_norm_backward_apply(const void* x, const void* dy, void* dx, const float* gamma, const float* beta, const float* stats, const double* sums,
                                          int R, const float* q, double D, int dtype, int B, int C, int H, int W, int gelu, void* stream) {
  int rc = check_pointwise(x, dy, dtype, "geometric_norm_backward_apply");
  if (!rc) rc = check_aligned8(sums, "geometric_norm_backward_apply");
  if (rc) return rc;
  B200_REQUIRE(dx && stats && q, "geometric_norm_backward_apply: null argument");
  return geometric_norm_backward_apply(x, dy, dx, gamma, beta, stats, sums, R, q, D, dtype, B, C, H, W, gelu, S(stream));
}
int b200sht_geometric_norm_param_grads(const double* sums, float* dgamma, float* dbeta, int B, int C, void* stream) {
  int rc = check_aligned8(sums, "geometric_norm_param_grads");
  if (rc) return rc;
  return geometric_norm_param_grads(sums, dgamma, dbeta, B, C, S(stream));
}

int b200sht_debug_set_pdl(int on) {
  const int old = b200sht::pdl_flag();
  b200sht::pdl_flag() = on;
  return old;
}

int b200sht_debug_dft_profile(uint64_t* counters16) {
  B200_REQUIRE(counters16 != nullptr, "debug_dft_profile: null argument");
  return dft_profile_read(reinterpret_cast<unsigned long long*>(counters16));
}

int b200sht_debug_umma_profile(uint64_t* counters16) {
  B200_REQUIRE(counters16 != nullptr, "debug_umma_profile: null argument");
  return umma_profile_read(reinterpret_cast<unsigned long long*>(counters16));
}

int b200sht_debug_dft_host(int N, int mmax, int direction, int scale_mode, float row_scale, const float* in, float* out) {
  B200_REQUIRE(in && out && N > 0 && mmax > 0, "debug_dft_host: bad argument");
  return dft_host(N, mmax, direction, scale_mode & 1, &row_scale, in, out);
}

// ---- DISCO convolution (disco.cu)
int b200sht_disco_plan_create(b200sht_disco_plan** plan, int nlat_in, int nlon_in, int nlat_out, int nlon_out, int K, int64_t nnz, const int* ker,
                              const int* lat_out, const int* col_in, const double* vals, void* stream) {
  return disco_plan_create(plan, nlat_in, nlon_in, nlat_out, nlon_out, K, nnz, ker, lat_out, col_in, vals, S(stream));
}

int b200sht_disco_plan_destroy(b200sht_disco_plan* plan) { return disco_plan_destroy(plan); }

int64_t b200sht_disco_plan_query(const b200sht_disco_plan* plan, int what) { return disco_plan_query(plan, what); }

int b200sht_disco_forward(const b200sht_disco_plan* plan, const void* x, int dtype, int B, int C, float* X, void* stream) {
  return disco_forward(plan, x, dtype, B, C, X, S(stream));
}

int b200sht_disco_adjoint(const b200sht_disco_plan* plan, const float* dX, void* dx, int dtype, int B, int C, void* stream) {
  return disco_adjoint(plan, dX, dx, dtype, B, C, S(stream));
}

// ---- neighbourhood attention on the sphere (attention.cu)
int b200sht_attention_forward(const b200sht_disco_plan* plan, const float* q, const float* k, const float* v, float* y, float* lse, int B, int heads,
                              int ek, int ev, float scale, void* stream) {
  return attention_forward(plan, q, k, v, y, lse, B, heads, ek, ev, scale, S(stream));
}

int b200sht_attention_backward(const b200sht_disco_plan* plan, const float* q, const float* k, const float* v, const float* y, const float* lse,
                               const float* dy, float* dq, float* dk, float* dv, float* D, int B, int heads, int ek, int ev, float scale,
                               void* stream) {
  return attention_backward(plan, q, k, v, y, lse, dy, dq, dk, dv, D, B, heads, ek, ev, scale, S(stream));
}

// ---- bilinear resampling on the sphere (resample.cu)
int b200sht_resample_plan_create(b200sht_resample_plan** plan, int nlat_in, int nlon_in, int nlat_out, int nlon_out, int expand_poles, const int* lat_idx,
                                 const float* lat_w, const int* lon_left, const int* lon_right, const float* lon_w, void* stream) {
  return resample_plan_create(plan, nlat_in, nlon_in, nlat_out, nlon_out, expand_poles, lat_idx, lat_w, lon_left, lon_right, lon_w, S(stream));
}

int b200sht_resample_plan_destroy(b200sht_resample_plan* plan) { return resample_plan_destroy(plan); }

int64_t b200sht_resample_plan_query(const b200sht_resample_plan* plan, int what) { return resample_plan_query(plan, what); }

int b200sht_resample_forward(const b200sht_resample_plan* plan, const float* x, float* y, int planes, void* stream) {
  return resample_forward(plan, x, y, planes, S(stream));
}

int b200sht_resample_adjoint(const b200sht_resample_plan* plan, const float* dy, float* dx, int planes, void* stream) {
  return resample_adjoint(plan, dy, dx, planes, S(stream));
}

}  // extern "C"
