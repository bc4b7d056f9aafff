// Shared helpers for the b200sht library (error reporting, packed-format index math).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cstdint>
#include <cstdio>
#include <cstdarg>
#include <cstring>
#include "../../include/b200sht.h"

#define HD __host__ __device__ __forceinline__

namespace b200sht {

void set_error(const char* fmt, ...);

#define B200_CHECK_CUDA(expr)                                                                      \
  do {                                                                                             \
    cudaError_t _e = (expr);                                                                       \
    if (_e != cudaSuccess) {                                                                       \
      ::b200sht::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e));  \
      return B200SHT_ERR_CUDA;                                                                     \
    }                                                                                              \
  } while (0)

#define B200_CHECK_LAUNCH()  B200_CHECK_CUDA(cudaGetLastError())

#define B200_REQUIRE(cond, ...)                 \
  do {                                          \
    if (!(cond)) {                              \
      ::b200sht::set_error(__VA_ARGS__);        \
      return B200SHT_ERR_INVALID;               \
    }                                           \
  } while (0)

// round-to-nearest conversion to TF32 (10-bit mantissa), as cuBLAS applies to its TF32 GEMM inputs; the TF32 MMA itself
// truncates the low 13 mantissa bits of whatever it reads, so producers of tensor-core operands round first.
__device__ __forceinline__ float tf32_rn(float x) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
  return __uint_as_float(u);
}

HD int round_up(int a, int b) { return (a + b - 1) / b * b; }
HD int ceil_div(int a, int b) { return (a + b - 1) / b; }

// Block-triangular storage convention (DESIGN.md section 3): for order m only degrees l >= lstart(m) are
// stored/computed, for degree l only orders m < mend(l).  Entries with lstart(m) <= l < m hold exact zeros.
constexpr int kTriBlock = 32;
HD int lstart(int m) { return (m / kTriBlock) * kTriBlock; }
HD int mend(int l, int M) { int e = (l / kTriBlock + 1) * kTriBlock; return e < M ? e : M; }
// `dense` storage (used for the l/m-sharded spectra of the h x w model-parallel path): every (l, m) entry is stored
HD int mend_d(int l, int M, int dense) { return dense ? M : mend(l, M); }
constexpr int kDenseFlag = 0x100;  // or-ed into the `op` / `mode` argument of the mix / ComplexReLU entry points

struct FftPlan {
  int N;
  int nstages;
  int radix[20];
};

// The immutable plan object behind b200sht_plan.
struct Plan {
  int nlat, nlon, lmax, mmax, kp;   // lmax: table rows; a vector plan stacks D over Q, so there it is twice the caller's lmax
  int vector;           // vector-SHT plan: d_table[m] holds D (rows 0 .. lmax/2 - 1) then Q (rows lmax/2 .. lmax - 1), see legendre.cu
  int csphase;
  int m0;               // global order of local order 0 (m-sharded plans of the distributed SHT); 0 otherwise
  int no_table;         // FFT-only plan (latitude-sharded stage of the distributed SHT)
  int dense;            // dims-only plans: packed spec tensors store every (l, m) entry (no block triangle)
  float* d_table;       // [mmax][lmax][kp]
  float* d_table_tf32;  // same, rounded to nearest TF32 (operand of the tensor-core kernels); null when that path is unavailable
  float* d_table_lo;    // d_table - d_table_tf32 (second term of the 3 x TF32 strict-fp32 mode); allocated at its first use
  float* d_rowscale;    // [kp]  quad_w[k] * 2 pi / nlon (0 in the padding)
  float2* d_twiddle;    // [nlon] exp(-2 pi i t / nlon)
  FftPlan fft;
  int sm_count;
  int umma_ok;          // tensor-core path usable on this device (sm_90)
  void* umma_state;     // TMA descriptors etc. (owned by umma translation unit)
  void* dft_state;      // tensor-core DFT tables (dft.cu); null when the grid is outside its range or the tensor-core path is unavailable
};

// SMs left free by the persistent kernels launched from this thread (0 = use them all).  Set around the stages that are meant to run beside
// a collective on another stream (b200sht_spectral_conv_backward_ex): a persistent one-CTA-per-SM kernel leaves an NCCL kernel nowhere to
// run, the collective then lands between two kernels and the next one starts on fewer SMs with a static tile assignment -- slower than
// giving the SMs away up front.
int& sm_reserve();

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) once per (kernel, device) and size increase instead of before every launch: the call takes
// the context lock and was a measurable part of the host time per launch (13 launches per SpectralConv step).  One cache per kernel
// instantiation (the template parameter is the call site's tag type).
template <class Tag, class K>
inline cudaError_t ensure_dynamic_smem(K kernel, size_t bytes) {
  static int granted[64] = {0};
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  if (dev >= 0 && dev < 64 && (size_t)granted[dev] >= bytes) return cudaSuccess;
  e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  if (e == cudaSuccess && dev >= 0 && dev < 64) granted[dev] = (int)bytes;
  return e;
}
// ---- programmatic dependent launch (PDL) ------------------------------------------------------------------------------------------
// The hot kernels call pdl_trigger() first thing (their successor in the stream may be scheduled as soon as every CTA of this grid has done
// so or exited) and pdl_wait() after their prologue (barrier init, tensor-map prefetch, resident constant tables), i.e.
// before the first access to memory another kernel produces or still reads: the wait returns once all prerequisite grids have COMPLETED and
// their writes are visible.  A successor launched with launch_pdl() therefore overlaps its launch latency and prologue with the tail of this
// kernel; launched normally it serialises as always.  Both instructions are no-ops without a programmatic dependency.
// Rule for every kernel launched through launch_pdl(): no global load / store / TMA of non-constant data before pdl_wait().
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
bool pdl_enabled();   // B200SHT_PDL (default: see capi.cu)
template <class... KArgs, class... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  // not while SMs are reserved for a collective on another stream (b200sht_spectral_conv_backward_ex): an early-launched successor would park its
  // CTAs on exactly the SMs that were left free for the NCCL kernel
  attr[0].val.programmaticStreamSerializationAllowed = (pdl_enabled() && sm_reserve() == 0) ? 1 : 0;
  cfg.attrs = attr; cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

inline int usable_sms(int sms) { const int r = sm_reserve(); return (r > 0 && sms - r >= 1) ? sms - r : sms; }

}  // namespace b200sht

struct b200sht_plan : public b200sht::Plan {};
