// Longitude transform on the tensor cores (B200SHT_PREC_TF32): the truncated real DFT of every latitude row as
//   radix-8 butterflies + twiddles on the CUDA cores  x  one class-independent [M2 x N2/2] DFT matrix on the tensor cores (mma.sync TF32).
// Replaces the CUDA-core Stockham kernels of fft.cu for nlon = 8 * N2, N2 <= 190, mmax <= 256 (every shipped grid); see dft_math.cuh
// for the factorisation.  Reference semantics: 2 pi * torch.fft.rfft(x, norm="forward")[..., :mmax] and torch.fft.irfft(Z, n=nlon,
// norm="forward") inside torch_harmonics.RealSHT / InverseRealSHT (call sites makani/models/common/spectral_convolution.py:239,253).
//
// Why: the Stockham kernels are issue-bound on the CUDA cores: a 1440-point row is 34 kflop for 4.8 KB, far above the fp32 FMA rate over
// the HBM bandwidth of the GPU.  Here two of the three radix stages (the 31 x 180 sub-transform, 86 % of the flops) run on the tensor
// pipe at TF32 and only one radix-8 stage stays on the CUDA cores; no shared-memory exchange between stages is left.
//
// synthesis kernel (latspec -> rows):   D[j2][(class c, latitude k)] for the columns j2 <= N2/2 and an 8-row tile.  A = E^T resident in
//   shared memory (32 KB) in fragment order, B = the latspec tile [m2][(c, k)] streamed by TMA (16 KB per 8 rows) through an mbarrier ring
//   and rewritten in place into fragment order by the load warp, the cosine and sine sums of Zr and Zi in registers.  A task owns 8
//   columns j2; its m16n8 fragments give each thread the two latitudes 2 (lane % 4), + 1 of the column j2 = lane / 4 for all eight classes,
//   i.e. the inputs of its own butterflies:
//   S -> V(j2), V(N2-j2) -> twiddle -> radix-8 -> scale/bias -> bf16 into a shared-memory output tile, written out by TMA bulk stores.
// analysis kernel (rows -> latspec):    producer warps load the eight samples x[N2 j1 + j2] of a column (lanes = consecutive j2),
//   butterfly + twiddle them and write the even/odd combinations (Ye, Yo) as K-major TF32 operand tiles [(c, k)][j2] (128-byte
//   swizzle, conflict-free row stores); B = E resident (<= 24 KB); two warpgroups contract them with wgmma.m64n32k8 (one class per warp)
//   into D[(c,k)][m2] in registers over the K-blocks and write latspec straight from their fragments (32-byte runs along k).
#include "umma_common.cuh"
#include "wgmma_tf32.cuh"
#include "dft_math.cuh"
#include <cmath>
#include <cstdlib>
#include <vector>

namespace b200sht {

int umma_available();   // umma.cu

constexpr int kDftMaxHalf = 95;    // N2 / 2 <= 95: three 32-lane quadrants (synthesis) / three K-blocks (analysis)
constexpr int kDftSynWorkers = 10;   // MMA + epilogue warps of the synthesis kernel
constexpr int kDftSynThreads = 32 * (kDftSynWorkers + 2);   // + a TMA load warp and a TMA store warp: 3 warps per SM sub-partition, 168 registers
constexpr int kDftSynStages = 4;   // 16 KB each
// width of the output store box: the largest 8 d <= 256 (the TMA box limit) with d | N2, so that a row is a whole number of boxes
__host__ __device__ constexpr int dft_out_box(int N2) {
  int d = N2 < 32 ? N2 : 32;
  while (N2 % d != 0) --d;
  return 8 * d;
}

// n / d for 0 <= n < 2^31 by a multiply-high and a shift (d > 0 fixed per launch): the per-task index arithmetic of the synthesis workers
// without the ~25-instruction integer division
struct FastDiv {
  uint32_t m, s;
  int d;
  __device__ __forceinline__ int div(int n) const { return (int)((__umulhi((uint32_t)n, m) + (uint32_t)n) >> s); }
};
static FastDiv make_fastdiv(int d) {
  FastDiv f;
  f.d = d;
  f.s = 0;
  while ((1ll << f.s) < d) ++f.s;
  f.m = (uint32_t)((((1ull << 32) * ((1ull << f.s) - (unsigned long long)d)) / (unsigned long long)d) + 1);
  return f;
}

struct DftTables {
  float* et;      // synthesis A: [16 blocks of 8 j2][cos, sin][8 rows j2][32 m2], TF32-rounded; rows j2 > N2 / 2 are zero
  float* eb;      // analysis  B: [nkb][2][32 rows m2][32 j2 local]  (cos, sin), TF32-rounded
  float2* tw;     // [8][N2]  exp(+2 pi i c j2 / nlon)
  float* zeros;   // 8 * N2 floats of zeros: load target of the analysis lanes / rows that carry no sample (keeps the loads unconditional)
  int N2, half, M2, nkb;
};

bool dft_shape_ok(int nlon, int mmax) {
  if (nlon % 8 != 0) return false;
  const int N2 = nlon / 8;
  return N2 >= 2 && N2 / 2 <= kDftMaxHalf && (mmax + 7) / 8 <= 32 && mmax <= nlon / 2 + 1;
}

__global__ void dft_tables_kernel(float* et, float* eb, float2* tw, int N2, int half, int M2, int nkb, int nlon) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  // E^T tile: [16 blocks][cos, sin][8 rows j2][32 m2]
  if (i < 2 * 128 * 32) {
    const int m2 = i % 32, row = i / 32, p = (row >> 3) & 1, j2 = 8 * (row >> 4) + (row & 7);
    float v = 0.f;
    if (j2 <= half && m2 < M2) {
      const long long t = ((long long)m2 * j2) % N2;
      const double ang = 2.0 * M_PI * (double)t / (double)N2;
      v = tf32_rn((float)(p == 0 ? cos(ang) : sin(ang)));
    }
    et[i] = v;
  }
  if (i < nkb * 2 * 32 * 32) {
    const int jl = i % 32, m2 = (i / 32) % 32, p = (i / 1024) % 2, kb = i / 2048;
    const int j2 = kb * 32 + jl;
    float v = 0.f;
    if (j2 <= half && m2 < M2) {
      const long long t = ((long long)m2 * j2) % N2;
      const double ang = 2.0 * M_PI * (double)t / (double)N2;
      v = tf32_rn((float)(p == 0 ? cos(ang) : sin(ang)));
      if (2 * j2 == N2) v *= 0.5f;   // the column N2 / 2 is its own partner: the producers count it twice (no mask)
    }
    eb[i] = v;
  }
  if (i < 8 * N2) {
    const int j2 = i % N2, c = i / N2;
    const double ang = 2.0 * M_PI * (double)(c * j2) / (double)nlon;
    tw[i] = make_float2((float)cos(ang), (float)sin(ang));
  }
}

int dft_plan_init(Plan* pl) {
  pl->dft_state = nullptr;
  if (!umma_available()) return -1;
  if (!dft_shape_ok(pl->nlon, pl->mmax)) return -1;
  DftTables* t = new DftTables();
  t->N2 = pl->nlon / 8; t->half = t->N2 / 2; t->M2 = (pl->mmax + 7) / 8;
  t->nkb = (t->half + 1 + 31) / 32;   // 32-column K-blocks of j2 = 0 .. N2 / 2 (analysis)
  t->et = nullptr; t->eb = nullptr; t->tw = nullptr; t->zeros = nullptr;
  const size_t neb = (size_t)t->nkb * 2 * 32 * 32;
  cudaError_t e = cudaMalloc(&t->et, sizeof(float) * 2 * 128 * 32);
  if (e == cudaSuccess) e = cudaMalloc(&t->eb, sizeof(float) * neb);
  if (e == cudaSuccess) e = cudaMalloc(&t->tw, sizeof(float2) * 8 * t->N2);
  if (e == cudaSuccess) e = cudaMalloc(&t->zeros, sizeof(float) * 8 * t->N2);
  if (e == cudaSuccess) e = cudaMemset(t->zeros, 0, sizeof(float) * 8 * t->N2);
  if (e == cudaSuccess) {
    const int n = 8192 > 8 * t->N2 ? 8192 : 8 * t->N2;
    dft_tables_kernel<<<(n + 255) / 256, 256>>>(t->et, t->eb, t->tw, t->N2, t->half, t->M2, t->nkb, pl->nlon);
    e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaStreamSynchronize(0);
  }
  if (e != cudaSuccess) {
    cudaFree(t->et); cudaFree(t->eb); cudaFree(t->tw); cudaFree(t->zeros);
    delete t;
    return -1;
  }
  pl->dft_state = t;
  return 0;
}

void dft_plan_destroy(Plan* pl) {
  DftTables* t = static_cast<DftTables*>(pl->dft_state);
  if (!t) return;
  cudaFree(t->et); cudaFree(t->eb); cudaFree(t->tw); cudaFree(t->zeros);
  delete t;
  pl->dft_state = nullptr;
}

static bool dft_enabled() {
  static const int on = [] { const char* e = getenv("B200SHT_DFT"); return e ? atoi(e) : 1; }();
  return on != 0;
}
bool dft_usable(const Plan* pl) { return pl->dft_state != nullptr && dft_enabled(); }

// ----------------------------------------------------------------------------------------- wait-time profile
// B200SHT_DFT_PROF=1: every role accumulates the SM clocks it spends in its mbarrier waits (one atomic per wait, lane 0 of the warp) into 16
// counters, read back and cleared by b200sht_debug_dft_profile().  Slots -- analysis: 0 producers / raw samples, 1 producers / operand stage free,
// 2 loader / raw stage free, 3 MMA warps / operand stage full, 5 MMA-warp tiles, 6 CTA lifetime, 7 producer items; synthesis: 8 load warp /
// stage free, 9 workers / stage rewritten, 10 workers / output tile free, 11 store warp / output tile written, 12 CTA lifetime, 13 worker
// tasks, 14 load warp / tile landed.
static unsigned long long* g_dft_prof = nullptr;
static unsigned long long* dft_prof_buffer() {
  static const int on = [] { const char* e = getenv("B200SHT_DFT_PROF"); return e ? atoi(e) : 0; }();
  if (!on) return nullptr;
  if (!g_dft_prof) {
    if (cudaMalloc(&g_dft_prof, 16 * sizeof(unsigned long long)) != cudaSuccess) { g_dft_prof = nullptr; return nullptr; }
    cudaMemset(g_dft_prof, 0, 16 * sizeof(unsigned long long));
  }
  return g_dft_prof;
}
int dft_profile_read(unsigned long long* out16) {
  if (!g_dft_prof) { for (int i = 0; i < 16; ++i) out16[i] = 0; return 0; }
  B200_CHECK_CUDA(cudaDeviceSynchronize());
  B200_CHECK_CUDA(cudaMemcpy(out16, g_dft_prof, 16 * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
  B200_CHECK_CUDA(cudaMemset(g_dft_prof, 0, 16 * sizeof(unsigned long long)));
  return 0;
}
#ifdef B200SHT_DFT_PROFILE
constexpr bool kDftProfile = true;
#else
constexpr bool kDftProfile = false;   // the counters cost a few instructions per wait: compiled in only by `python -m makani_b200.build --profile`
#endif
__device__ __forceinline__ void prof_wait(unsigned long long* prof, int slot, uint64_t* bar, uint32_t parity, bool lead) {
  if (!kDftProfile || prof == nullptr) { mbar_wait(bar, parity); return; }
  const long long t0 = clock64();
  mbar_wait(bar, parity);
  if (lead) atomicAdd(prof + slot, (unsigned long long)(clock64() - t0));
}
// the same for the kernel that holds wgmma (the analysis): a lost arrival traps without the printf, whose call would make ptxas serialize
// every wgmma of the kernel; the counters are inline shared-memory atomics, so the profile build keeps the wgmma asynchronous too
__device__ __forceinline__ void prof_wait_nocall(unsigned long long* prof, int slot, uint64_t* bar, uint32_t parity, bool lead) {
  if (!kDftProfile || prof == nullptr) { mbar_wait_nocall(bar, parity); return; }
  const long long t0 = clock64();
  mbar_wait_nocall(bar, parity);
  if (lead) atomicAdd(prof + slot, (unsigned long long)(clock64() - t0));
}

// 3-D view (nlon, nlat, rows) of the synthesis output, box (ow, 8, 1), no swizzle
static int make_tmap_out(CUtensorMap* tm, void* base, bool bf16, int nlon, int nlat, long long rows, int ow) {
  TmapKey key;
  memset(&key, 0, sizeof(key));
  key.base = base; key.rank = 3; key.kind = bf16 ? 7 : 6;
  key.dims[0] = nlon; key.dims[1] = nlat; key.dims[2] = rows; key.box[0] = ow;
  int slot = 0;
  if (tmap_lookup(key, tm, &slot)) return 0;
  PFN_encodeTiled enc = get_encode();
  if (!enc) { set_error("cuTensorMapEncodeTiled is unavailable"); return B200SHT_ERR_UNSUPPORTED; }
  static thread_local bool ctx_bound = false;
  if (!ctx_bound) { cudaFree(nullptr); ctx_bound = true; }
  const int es = bf16 ? 2 : 4;
  cuuint64_t gd[3] = {(cuuint64_t)nlon, (cuuint64_t)nlat, (cuuint64_t)rows};
  cuuint64_t gst[2] = {(cuuint64_t)nlon * es, (cuuint64_t)nlon * nlat * es};
  cuuint32_t bx[3] = {(cuuint32_t)ow, 8, 1}, el[3] = {1, 1, 1};
  if (gst[0] % 16 != 0 || (reinterpret_cast<uintptr_t>(base) & 15) != 0 || (ow * es) % 16 != 0) {
    set_error("tensor map (output): base / row pitch / box row not 16-byte aligned");
    return B200SHT_ERR_INVALID;
  }
  CUresult r = enc(tm, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, base, gd, gst, bx, el,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled (output) failed (%d)", (int)r); return B200SHT_ERR_CUDA; }
  tmap_store(key, tm, slot);
  return 0;
}

// the two latitudes of a synthesis thread: a at p0, b at p1 (bf16: one conversion of the pair)
template <typename T> __device__ __forceinline__ void st_out2(uint8_t* p0, uint8_t* p1, float a, float b);
template <> __device__ __forceinline__ void st_out2<float>(uint8_t* p0, uint8_t* p1, float a, float b) {
  *reinterpret_cast<float*>(p0) = a;
  *reinterpret_cast<float*>(p1) = b;
}
template <> __device__ __forceinline__ void st_out2<__nv_bfloat16>(uint8_t* p0, uint8_t* p1, float a, float b) {
  const __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  *reinterpret_cast<__nv_bfloat16*>(p0) = v.x;
  *reinterpret_cast<__nv_bfloat16*>(p1) = v.y;
}
// raw sample bits of the next item (converted when consumed): float bits, or the bf16 pattern in the low half
template <typename T> __device__ __forceinline__ uint32_t ld_raw(const T* p);
template <> __device__ __forceinline__ uint32_t ld_raw<float>(const float* p) { return __float_as_uint(__ldg(p)); }
template <> __device__ __forceinline__ uint32_t ld_raw<__nv_bfloat16>(const __nv_bfloat16* p) { return (uint32_t)__ldg(reinterpret_cast<const unsigned short*>(p)); }

// How the CUDA-core producers turn an fp32 value into a TF32 operand (the MMA ignores the 13 low mantissa bits):
//   0  cvt.rna.tf32.f32                 3 instructions (FSETP + IADD + LOP3)
//   1  (bits + 0x1000) & ~0x1fff        2 instructions, same result for finite values
//   2  bias-compensated truncation      0 instructions: the value is pre-scaled by (1 + 2^-10 / 3) -- folded into the twiddle
//      factors -- so that the hardware truncation error x f - delta, delta ~ U[0, ulp), has zero mean over a binade; its rms is
//      0.304 ulp against 0.289 ulp for round-to-nearest, and TF32-exact inputs stay exact (x f < ulp / 3).
#ifndef B200_DFT_TF32_MODE
#define B200_DFT_TF32_MODE 2
#endif
constexpr float kTruncComp = 1.0f + 0.0009765625f / 3.0f;
__device__ __forceinline__ float tf32_operand(float v) {
#if B200_DFT_TF32_MODE == 0
  return tf32_rn(v);
#elif B200_DFT_TF32_MODE == 1
  return __uint_as_float((__float_as_uint(v) + 0x1000u) & 0xffffe000u);
#else
  return v;   // already scaled through the twiddles
#endif
}
__device__ __forceinline__ float tf32_operand_unscaled(float v) {   // class 0 carries no twiddle
#if B200_DFT_TF32_MODE == 2
  return v * kTruncComp;
#else
  return tf32_operand(v);
#endif
}

__device__ __forceinline__ pr pr_operand(pr v) { return make_pr(tf32_operand(v.v.x), tf32_operand(v.v.y)); }
__device__ __forceinline__ pr pr_operand_unscaled(pr v) {
#if B200_DFT_TF32_MODE == 2
  return rmul(v, kTruncComp);
#else
  return pr_operand(v);
#endif
}

template <typename T> __device__ __forceinline__ float ld_in(const T* p);
template <> __device__ __forceinline__ float ld_in<float>(const float* p) { return __ldg(p); }
template <> __device__ __forceinline__ float ld_in<__nv_bfloat16>(const __nv_bfloat16* p) {
  return __uint_as_float((uint32_t)__ldg(reinterpret_cast<const unsigned short*>(p)) << 16);
}

// ================================================================================================ synthesis
struct DftSynParams {
  alignas(64) CUtensorMap tmZ;   // tiled latspec as ((c % 4, k % 8), c / 4, m2, p, tile), box (32, 1, 32, 1, 1): MN-major B operand, N = (c, k)
  alignas(64) CUtensorMap tmY;   // the output as (nlon, nlat, R), box (ow, 8, 1), no swizzle: TMA clips the rows k >= nlat of an image's last tile
  const float* Z;
  const float* et;   // E^T tiles, [16 blocks][cos, sin][8 rows j2][32 m2]: read once per CTA into fragment order
  const float2* tw;
  const float* rowscale;
  const float* bias;
  unsigned long long* prof;
  FastDiv ktiles, C;   // 8-row tiles per image; channels (bias index r % C)
  int R, nlat, nlon, kp, mmax, N2, half, M2, mode, ntiles, has_nyq, ow;
};

// Order of the 32 orders m2 in the MMA K loop.  The sum over m2 may visit them in any order as long as A and B agree, and this one lets a
// thread load its B fragments of two k8 steps with one 16-byte load: the thread (g, q) of step s holds, in its K slots q and q + 4, the
// orders syn_kslot(s, q, 0 / 1) = 8 q + 4 (s / 2) + ((2 (s % 2) + 0 / 1 + q) % 4).  Over the four steps the slots of the lanes q hold
// 8 q .. 8 q + 7, rotated by q inside each group of four: the rotation keeps the load warp's rewrite of the stage free of bank conflicts.
__host__ __device__ constexpr int syn_kslot(int s, int q, int hi) { return 8 * q + 4 * (s >> 1) + ((2 * (s & 1) + hi + q) & 3); }
// 16-byte unit of the thread (g, q) in each 512-byte block of a rewritten stage: the eight threads of a quarter warp hit distinct bank
// groups both when the workers read (g = 2 t, 2 t + 1) and when the load warp writes (g = j, j + 4)
__device__ __forceinline__ uint32_t syn_unit(int g, int q) { return (uint32_t)(8 * (g >> 1) + 4 * ((g ^ (g >> 2)) & 1) + q); }

// shared memory: [A: 16 blocks x 4 k8 steps x 32 lanes x 16 B, 32 KB][B ring: kDftSynStages x 16 KB][output: 2 x 8 rows x nlon]
//                [tw table N2 x 8 float2][output offsets 8 x N2 int][barriers]
// warps 0 .. kDftSynWorkers - 1: MMA + epilogue; then the TMA load warp and the TMA store warp.
// B stage: TMA lands the tile as [plane][c / 4][32 rows m2][(c % 4, k)] (128-byte swizzle).  The load warp then rewrites each 4 KB block
// (plane, c / 4) in place as [c % 4][h][32 threads][4 orders]: the thread (g, q) finds the orders 8 q + 4 h + 0..3 (rotated by q, see
// syn_kslot) of the latitude g and the class c in one 16-byte unit, so a task loads its 64 B-fragment registers with 32 LDS.128 instead of
// 128 scalar loads, and the rewrite (32 LDS.128 + 32 STS.128 per lane and tile, conflict-free) is shared by all the tasks of the tile.
// The load warp runs one tile ahead with its TMA loads: before it rewrites tile n it issues the load of tile n + 1 as soon as the workers
// have released that stage (tile n - 3), so the workers find up to three tiles ready; it arrives on ready[s] when the rewrite is written.
// (Issuing further ahead without blocking was slower, 158 against 135 us: the warp then only looks for free stages once per landed tile.)
// The work of a tile is split into `nblk` tasks, one per 8 columns j2 <= N2 / 2, and the tasks (tile n, block b) of this CTA are dealt
// round-robin over `nwork` worker warps (task n * nblk + b), so each SM sub-partition holds several tasks in flight: the epilogue of one
// overlaps the MMAs of another.  nwork <= 2 nblk bounds the lead of a warp: consecutive tasks of a warp are at most two tiles apart, so when
// a warp reaches tile m, its previous task has seen tile m - 4 rewritten (ready) and stored (ofree).  Every mbarrier wait is then for the
// next phase of its barrier and never for one two phases away, which the parity test cannot tell apart.  All kDftSynWorkers warps work
// when nblk >= kDftSynWorkers / 2.  The A tile of block b stacks the cos and sin rows of its 8 columns, so the m16n8 accumulator fragment
// holds, per thread, S1 / S3 (B = Zr) and S4 / S2 (B = Zi) of the column j2 = 8 b + lane / 4 and the latitude pair 2 (lane % 4), + 1 for
// all eight classes: exactly the inputs of the radix-8 epilogue of j2 and N2 - j2, in 64 accumulator registers.
// Output: the epilogues write the finished values of tile n into the shared-memory tile n % 2, laid out as the TMA boxes of ow columns
// x 8 rows; when all nblk tasks of the tile have arrived on staged[n % 2], the store warp writes it with bulk tensor stores (whole 128-byte
// lines instead of 16-byte pieces of four rows per store instruction) and frees the buffer once the stores have read it.
// N2 is a run-time value here: the compile-time instantiations spilled at the 168-register cap, this one does not.
template <typename T>
__global__ void __launch_bounds__(kDftSynThreads, 1) dft_synthesis_kernel(const __grid_constant__ DftSynParams p) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ unsigned long long prof_s[16];   // wait-time profile (B200SHT_DFT_PROF): accumulated per CTA, flushed once at the end
  unsigned long long* const prof = (kDftProfile && p.prof) ? prof_s : nullptr;
  if (kDftProfile && threadIdx.x < 16) prof_s[threadIdx.x] = 0;
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* gbase = smem_raw + (base - raw);
  const int N2 = p.N2;
  const int nlon = 8 * N2;
  const int ow = p.ow;
  const uint32_t obytes = (8u * nlon * sizeof(T) + 1023u) & ~1023u;   // one output tile
  const uint32_t sB = base + 32768, sO = sB + kDftSynStages * 16384;
  T* const outS = reinterpret_cast<T*>(gbase + (sO - base));
  float4* tws = reinterpret_cast<float4*>(gbase + (sO - base) + 2 * obytes);   // [j2][c / 2]: the twiddles of the classes 2 i, 2 i + 1
  int* oofs = reinterpret_cast<int*>(reinterpret_cast<uint8_t*>(tws) + 8 * N2 * 8);
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(oofs) + 8 * N2 * 4);
  uint64_t* full = bars;                  // [stages] TMA landed
  uint64_t* ready = full + kDftSynStages;   // [stages] rewritten into fragment order
  uint64_t* empty = ready + kDftSynStages;  // [stages] read by all the tasks of its tile
  uint64_t* staged = empty + kDftSynStages;   // [2] output tile written by all its tasks
  uint64_t* ofree = staged + 2;    // [2] output tile read by its bulk stores

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;   // warp-uniform for the compiler
  pdl_trigger();
  const int nblk = (p.half + 8) / 8;          // 8-column blocks of j2 = 0 .. N2 / 2
  const int nwork = kDftSynWorkers < 2 * nblk ? kDftSynWorkers : 2 * nblk;   // see above
  const bool is_tma = (warp == kDftSynWorkers), is_store = (warp == kDftSynWorkers + 1);

  if (threadIdx.x == 0) {
    for (int s = 0; s < kDftSynStages; ++s) { mbar_init(&full[s], 1); mbar_init(&ready[s], 32); mbar_init(&empty[s], nblk); }
    for (int b = 0; b < 2; ++b) { mbar_init(&staged[b], 32 * nblk); mbar_init(&ofree[b], 1); }
    fence_barrier_init();
    prefetch_tmap(&p.tmZ);
    prefetch_tmap(&p.tmY);
  }
  {
    // A in fragment order: [block][k8 step s][lane (g, q)] = (cos, sin of the column 8 block + g) at the orders syn_kslot(s, q, 0), then (1).
    // All the 16-byte loads of a thread are issued before its stores: one memory latency for the prologue, not one per element.
    constexpr int kEt4 = 16 * 2 * 8 * 32 / 4, kPer = (kEt4 + kDftSynThreads - 1) / kDftSynThreads;
    float4 ev[kPer];
#pragma unroll
    for (int k = 0; k < kPer; ++k) {
      const int i = threadIdx.x + k * kDftSynThreads;
      if (i < kEt4) ev[k] = __ldg(reinterpret_cast<const float4*>(p.et) + i);
    }
#pragma unroll
    for (int k = 0; k < kPer; ++k) {
      const int i = threadIdx.x + k * kDftSynThreads;   // E^T float4: orders 4 (i % 8) .. + 3 of the row i / 8 = (block, cos / sin, g)
      if (i >= kEt4) continue;
      const int row = i >> 3, b = row >> 4, cs = (row >> 3) & 1, g = row & 7;
      const float v[4] = {ev[k].x, ev[k].y, ev[k].z, ev[k].w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {   // the inverse of syn_kslot: order m2 -> (step s, slot half hi) of the lanes q = m2 / 8
        const int m2 = 4 * (i & 7) + e, q = m2 >> 3, r = m2 & 7, u = ((r & 3) - q) & 3;
        const int s = 2 * (r >> 2) + (u >> 1), hi = u & 1;
        reinterpret_cast<float*>(gbase)[((b * 4 + s) * 32 + 4 * g + q) * 4 + 2 * hi + cs] = v[e];
      }
    }
  }
  for (int i = threadIdx.x; i < 4 * N2; i += blockDim.x) {
    const int j2 = i >> 2, c = 2 * (i & 3);
    tws[i] = make_float4(p.tw[c * N2 + j2].x, p.tw[c * N2 + j2].y, p.tw[(c + 1) * N2 + j2].x, p.tw[(c + 1) * N2 + j2].y);
  }
  for (int i = threadIdx.x; i < 8 * N2; i += blockDim.x) {   // output tile byte offset of the longitude N2 j1 + j2 (row 0) at [j2][j1]
    const int j = N2 * (i & 7) + (i >> 3);
    oofs[i] = ((j / ow) * 8 * ow + j % ow) * (int)sizeof(T);
  }
  __syncthreads();
  const long long t_cta0 = (kDftProfile && p.prof && threadIdx.x == 0) ? clock64() : 0;
  pdl_wait();   // the prologue read plan constants only (E^T, twiddles); the latspec tiles, bias and y belong to other kernels until here

  if (is_tma) {
    const int ntl = blockIdx.x < p.ntiles ? (p.ntiles - 1 - blockIdx.x) / gridDim.x + 1 : 0;   // tiles of this CTA
    auto load = [&](int n) {
      const int s = n % kDftSynStages, it = n / kDftSynStages;
      if (it > 0) prof_wait(prof, 8, &empty[s], (it - 1) & 1, true);
      mbar_expect_tx(&full[s], 16384);
      const uint32_t st = sB + s * 16384;
      const int ti = blockIdx.x + n * gridDim.x;
      tma_load_5d(st, &p.tmZ, &full[s], 0, 0, 0, 0, ti);           // re, classes 0..3
      tma_load_5d(st + 4096, &p.tmZ, &full[s], 0, 1, 0, 0, ti);    // re, classes 4..7
      tma_load_5d(st + 8192, &p.tmZ, &full[s], 0, 0, 0, 1, ti);    // im
      tma_load_5d(st + 12288, &p.tmZ, &full[s], 0, 1, 0, 1, ti);
    };
    // rewrite of a 4 KB block (plane, c / 4): the lane (q, b, t) reads the rows 8 q + 4 h + (i + q) % 4 (i = 0..3, h = b ^ pass) at the
    // latitudes 4 b .. 4 b + 3 of the class 4 (c / 4) + t, and writes the transposed 4 x 4 block as the units of the threads (4 b + j, q).
    // A quarter warp (one t) reads eight distinct rows modulo 8 -- eight distinct chunks under the swizzle -- and writes eight distinct
    // bank groups (syn_unit).
    const int q = lane & 3, b = (lane >> 2) & 1, t = lane >> 3;
    uint32_t src[2][4], dst[2][4];
#pragma unroll
    for (int pass = 0; pass < 2; ++pass) {
      const int h = b ^ pass;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        src[pass][i] = swz128((uint32_t)((8 * q + 4 * h + ((i + q) & 3)) * 128 + (2 * t + b) * 16));
        dst[pass][i] = (uint32_t)(t * 1024 + h * 512) + 16 * syn_unit(4 * b + i, q);
      }
    }
    if (lane == 0 && ntl > 0) load(0);
    for (int n = 0; n < ntl; ++n) {
      if (lane == 0 && n + 1 < ntl) load(n + 1);   // blocks until the workers have released tile n - 3
      const int s = n % kDftSynStages;
      prof_wait(prof, 14, &full[s], (n / kDftSynStages) & 1, lane == 0);
      uint8_t* const st = gbase + 32768 + s * 16384;
      // all 32 loads of the lane before its stores: one shared-memory round trip per tile (a tile of a short row has few tasks to hide it)
      float4 v[4][2][4];
#pragma unroll
      for (int blk4 = 0; blk4 < 4; ++blk4)   // (plane, c / 4): 4 KB apart
#pragma unroll
        for (int pass = 0; pass < 2; ++pass)
#pragma unroll
          for (int i = 0; i < 4; ++i) v[blk4][pass][i] = *reinterpret_cast<const float4*>(st + blk4 * 4096 + src[pass][i]);
      __syncwarp();   // every lane has read the stage before any lane overwrites it
#pragma unroll
      for (int blk4 = 0; blk4 < 4; ++blk4) {
        uint8_t* const sb = st + blk4 * 4096;
        const float4(&w)[2][4] = v[blk4];
#pragma unroll
        for (int pass = 0; pass < 2; ++pass) {
          *reinterpret_cast<float4*>(sb + dst[pass][0]) = make_float4(w[pass][0].x, w[pass][1].x, w[pass][2].x, w[pass][3].x);
          *reinterpret_cast<float4*>(sb + dst[pass][1]) = make_float4(w[pass][0].y, w[pass][1].y, w[pass][2].y, w[pass][3].y);
          *reinterpret_cast<float4*>(sb + dst[pass][2]) = make_float4(w[pass][0].z, w[pass][1].z, w[pass][2].z, w[pass][3].z);
          *reinterpret_cast<float4*>(sb + dst[pass][3]) = make_float4(w[pass][0].w, w[pass][1].w, w[pass][2].w, w[pass][3].w);
        }
      }
      fence_proxy_async();      // the next TMA load into the stage (async proxy) is ordered after these stores
      mbar_arrive(&ready[s]);   // every lane: its stores of the stage are released to the workers
    }
  } else if (is_store) {
    if (lane == 0) {
      int n = 0;
      for (int ti = blockIdx.x; ti < p.ntiles; ti += gridDim.x, ++n) {
        const int b = n & 1;
        prof_wait(prof, 11, &staged[b], (n >> 1) & 1, true);
        const int r = p.ktiles.div(ti), k0 = (ti - r * p.ktiles.d) * 8;
        if (k0 < p.nlat)   // tiles of the padding rows kp > nlat: nothing to store (rows k >= nlat of a partial tile are clipped by TMA)
          for (int bx = 0; bx * ow < nlon; ++bx) tma_store_3d(&p.tmY, sO + b * obytes + bx * 8 * ow * (uint32_t)sizeof(T), bx * ow, k0, r);
        bulk_commit();
        bulk_wait_read0();
        mbar_arrive(&ofree[b]);
      }
      bulk_wait0();
    }
    __syncwarp();
  } else {
    const int kpi = lane & 3;
    const bool n2odd = (N2 & 1) != 0;
    const float smul = p.mode == 0 ? 2.f : 1.f;
    const int nyq_m = nlon / 2;
    const uint8_t* const zl = gbase + 32768 + syn_unit(lane >> 2, kpi) * 16;   // this lane's unit in block 0 of stage 0
    const uint4* const al = reinterpret_cast<const uint4*>(gbase) + lane;
    int n = 0, blk = warp;   // task n * nblk + blk
    if (blk >= nblk) { blk -= nblk; ++n; }   // warp < nwork <= 2 nblk
    while (warp < nwork) {
      const int ti = blockIdx.x + n * gridDim.x;
      if (ti >= p.ntiles) break;
      const int r = p.ktiles.div(ti), k0 = (ti - r * p.ktiles.d) * 8;
      const int ka = k0 + 2 * kpi;
      const int s = n % kDftSynStages, it = n / kDftSynStages;
      // per-row output factors:  out = x * sc + off(parity of the longitude)
      float rsa = 1.f, rsb = 1.f, z0a = 0.f, z0b = 0.f, zna = 0.f, znb = 0.f;
      if (p.mode == 1) {
        const float2 rs = *reinterpret_cast<const float2*>(p.rowscale + ka);
        rsa = rs.x; rsb = rs.y;
      } else {
        // tiled latspec: element (m, plane, r, k) at ((tile * 2 + plane) * M2 + m / 8) * 64 + (m % 8) * 8 + k % 8, tile = r * ktiles + k / 8
        const float* zt = p.Z + (size_t)ti * 2 * p.M2 * 64 + 2 * kpi;
        const float2 z0 = *reinterpret_cast<const float2*>(zt);
        z0a = z0.x; z0b = z0.y;
        if (p.has_nyq) {
          const float2 zn = *reinterpret_cast<const float2*>(zt + (nyq_m >> 3) * 64 + (nyq_m & 7) * 8);
          zna = zn.x; znb = zn.y;
        }
      }
      const float bias = p.bias ? __ldg(p.bias + (r - p.C.div(r) * p.C.d)) : 0.f;
      const pr sc = make_pr(smul * rsa, smul * rsb);
      const pr off_e = make_pr(bias - rsa * (z0a + zna), bias - rsb * (z0b + znb));   // even longitude j
      const pr off_o = make_pr(bias - rsa * (z0a - zna), bias - rsb * (z0b - znb));   // odd longitude j
      prof_wait(prof, 9, &ready[s], it & 1, lane == 0);
      if (prof && lane == 0) atomicAdd(prof + 13, 1ull);
      // rows of the A tile blk: cos then sin of the columns j2 = 8 blk + lane / 4, so the accumulator elements 0, 1 / 2, 3 of
      // acc[0] are S1 = cos . Zr / S3 = sin . Zr, of acc[1] S4 = cos . Zi / S2 = sin . Zi (32 orders m2; columns (class c, latitude))
      float acc[2][8][4];
#pragma unroll
      for (int a = 0; a < 2; ++a)
#pragma unroll
        for (int c = 0; c < 8; ++c) acc[a][c][0] = acc[a][c][1] = acc[a][c][2] = acc[a][c][3] = 0.f;
      {
        const uint8_t* const zs = zl + s * 16384;
        const uint4* const ab = al + blk * 128;
#pragma unroll
        for (int h = 0; h < 2; ++h) {   // k8 steps 2 h, 2 h + 1: one 16-byte unit of B per class and plane
          const uint4 a0 = ab[64 * h], a1 = ab[64 * h + 32];
          const uint32_t fa0[4] = {a0.x, a0.y, a0.z, a0.w}, fa1[4] = {a1.x, a1.y, a1.z, a1.w};
#pragma unroll
          for (int c = 0; c < 8; ++c) {
            const uint4 zr = *reinterpret_cast<const uint4*>(zs + (c >> 2) * 4096 + (c & 3) * 1024 + h * 512);
            const uint4 zi = *reinterpret_cast<const uint4*>(zs + 8192 + (c >> 2) * 4096 + (c & 3) * 1024 + h * 512);
            const uint32_t zr0[2] = {zr.x, zr.y}, zr1[2] = {zr.z, zr.w}, zi0[2] = {zi.x, zi.y}, zi1[2] = {zi.z, zi.w};
            mma_tf32(acc[0][c], fa0, zr0);
            mma_tf32(acc[1][c], fa0, zi0);
            mma_tf32(acc[0][c], fa1, zr1);
            mma_tf32(acc[1][c], fa1, zi1);
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);   // this warp's reads of the stage are done
      {
        const int j2 = 8 * blk + (lane >> 2);
        const bool valid = j2 <= p.half;
        const bool paired = valid && j2 != 0 && 2 * j2 != N2;
        const int jp = N2 - j2;
        float2 tw[8], tp[8];
        {
          const float4* const tr = tws + 4 * (valid ? j2 : 0);   // class 0 of the table: 1
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float4 w = tr[i];
            tw[2 * i] = make_float2(w.x, w.y);
            tw[2 * i + 1] = make_float2(w.z, w.w);
          }
        }
        dft_partner_twiddles(tw, tp);
        // output tile element (row kr, longitude j) at ((j / ow) * 8 + kr) * ow + j % ow; rows 2 kpi and 2 kpi + 1 of this thread
        uint8_t* const ob0 = reinterpret_cast<uint8_t*>(outS) + (n & 1) * obytes + 2 * kpi * ow * (int)sizeof(T);
        uint8_t* const ob1 = ob0 + ow * (int)sizeof(T);
        if (n >= 2) prof_wait(prof, 10, &ofree[n & 1], ((n >> 1) - 1) & 1, lane == 0);
        {
          pr vr[8], vi[8], x[8];
#pragma unroll
          for (int c = 0; c < 8; ++c) {   // V(j2) = (S1 - S2, S3 + S4)
            vr[c] = make_pr(acc[0][c][0], acc[0][c][1]) - make_pr(acc[1][c][2], acc[1][c][3]);
            vi[c] = make_pr(acc[0][c][2], acc[0][c][3]) + make_pr(acc[1][c][0], acc[1][c][1]);
          }
          dft_syn_radix8<pr>(vr, vi, tw, x);
          const pr o0 = (j2 & 1) ? off_o : off_e, o1 = (j2 & 1) ? off_e : off_o;
          const int4* const op = reinterpret_cast<const int4*>(oofs + 8 * (valid ? j2 : 0));
          const int4 oa = op[0], ob4 = op[1];
          const int of[8] = {oa.x, oa.y, oa.z, oa.w, ob4.x, ob4.y, ob4.z, ob4.w};
#pragma unroll
          for (int j1 = 0; j1 < 8; ++j1) {   // longitude N2 j1 + j2
            const pr o = rfma(x[j1], sc, (n2odd && (j1 & 1)) ? o1 : o0);
            if (valid) st_out2<T>(ob0 + of[j1], ob1 + of[j1], o.v.x, o.v.y);
          }
        }
        {
          pr vr[8], vi[8], x[8];
#pragma unroll
          for (int c = 0; c < 8; ++c) {   // V(N2 - j2) = (S1 + S2, S4 - S3)
            vr[c] = make_pr(acc[0][c][0], acc[0][c][1]) + make_pr(acc[1][c][2], acc[1][c][3]);
            vi[c] = make_pr(acc[1][c][0], acc[1][c][1]) - make_pr(acc[0][c][2], acc[0][c][3]);
          }
          dft_syn_radix8<pr>(vr, vi, tp, x);
          const pr o0 = (jp & 1) ? off_o : off_e, o1 = (jp & 1) ? off_e : off_o;
          const int4* const op = reinterpret_cast<const int4*>(oofs + 8 * (paired ? jp : 0));
          const int4 oa = op[0], ob4 = op[1];
          const int of[8] = {oa.x, oa.y, oa.z, oa.w, ob4.x, ob4.y, ob4.z, ob4.w};
#pragma unroll
          for (int j1 = 0; j1 < 8; ++j1) {   // not for the unpaired columns 0 and N2 / 2
            const pr o = rfma(x[j1], sc, (n2odd && (j1 & 1)) ? o1 : o0);
            if (paired) st_out2<T>(ob0 + of[j1], ob1 + of[j1], o.v.x, o.v.y);
          }
        }
        fence_proxy_async();   // the bulk stores read the tile through the async proxy: every writing thread fences and arrives
        mbar_arrive(&staged[n & 1]);
      }
      blk += nwork;   // next task: nwork <= 2 nblk, so at most two wraps
      if (blk >= nblk) { blk -= nblk; ++n; }
      if (blk >= nblk) { blk -= nblk; ++n; }
    }
  }
  __syncthreads();
  if (kDftProfile && p.prof && threadIdx.x == 0) prof_s[12] = (unsigned long long)(clock64() - t_cta0);
  if (kDftProfile) __syncthreads();
  if (kDftProfile && p.prof && threadIdx.x < 16) atomicAdd(p.prof + threadIdx.x, prof_s[threadIdx.x]);
}

int dft_synthesis(const Plan* pl, const float* Z, void* y, int dtype, int B, int C, const float* bias, int mode, cudaStream_t st) {
  const DftTables* t = static_cast<const DftTables*>(pl->dft_state);
  B200_REQUIRE(t != nullptr, "dft_synthesis: plan has no DFT tables");
  const int R = B * C;
  DftSynParams p;
  memset(&p, 0, sizeof(p));
  p.Z = Z; p.et = t->et; p.tw = t->tw; p.rowscale = pl->d_rowscale; p.bias = bias; p.prof = dft_prof_buffer();
  p.R = R; p.C = make_fastdiv(C); p.nlat = pl->nlat; p.nlon = pl->nlon; p.kp = pl->kp; p.mmax = pl->mmax;
  p.N2 = t->N2; p.half = t->half; p.mode = mode;
  p.ktiles = make_fastdiv(pl->kp / 8); p.ntiles = R * (pl->kp / 8);
  p.has_nyq = (pl->mmax == pl->nlon / 2 + 1) ? 1 : 0;
  p.M2 = t->M2;
  {
    // tiled latspec (written by legendre_synthesis_umma(tiled = 1)): [tile = r * ktiles + k / 8][plane][m2][c = m % 8][k % 8]; a tile is 16 KB
    // contiguous, the 128-byte rows of the TMA box are (4 classes x 8 latitudes) of one m2: the MN-major B operand, N = (c, k)
    long long d[5] = {32, 2, t->M2, 2, (long long)R * (pl->kp / 8)}, s[5] = {1, 32, 64, (long long)t->M2 * 64, 2ll * t->M2 * 64};
    int bx[5] = {32, 1, 32, 1, 1};
    int rc = make_tmap(&p.tmZ, Z, 5, d, s, bx);
    if (rc) return rc;
  }
  const bool bf16 = (dtype == B200SHT_BF16);
  p.ow = dft_out_box(t->N2);
  {
    int rc = make_tmap_out(&p.tmY, y, bf16, pl->nlon, pl->nlat, R, p.ow);
    if (rc) return rc;
  }
  const size_t obytes = (8 * (size_t)pl->nlon * (bf16 ? 2 : 4) + 1023) & ~(size_t)1023;
  const size_t smem = 1024 + 32768 + (size_t)kDftSynStages * 16384 + 2 * obytes + 8 * (size_t)t->N2 * 8 + 8 * (size_t)t->N2 * 4 +
                      (3 * kDftSynStages + 4) * 8;
  const int sms = usable_sms(pl->sm_count > 0 ? pl->sm_count : 132);
  const int ctas = p.ntiles < sms ? p.ntiles : sms;
#define B200_LAUNCH_SYN(TT)                                                                                          \
  do {                                                                                                                \
    struct Tag {};                                                                                                    \
    B200_CHECK_CUDA((ensure_dynamic_smem<Tag>(dft_synthesis_kernel<TT>, smem)));                                     \
    B200_CHECK_CUDA(launch_pdl(dft_synthesis_kernel<TT>, dim3(ctas), dim3(kDftSynThreads), smem, st, p));            \
  } while (0)
  if (bf16) { B200_LAUNCH_SYN(__nv_bfloat16); } else { B200_LAUNCH_SYN(float); }
#undef B200_LAUNCH_SYN
  B200_CHECK_LAUNCH();
  return 0;
}

// ================================================================================================= analysis
__host__ __device__ constexpr int dft_box_group(int N2, int es) { return (N2 * es) % 16 == 0 ? 1 : (2 * N2 * es) % 16 == 0 ? 2 : (4 * N2 * es) % 16 == 0 ? 4 : 8; }

// 3-D view of the samples for the analysis loader: (column inside a group of gs row segments, group, row), box (box_cols, 8 / gs, 16), no swizzle
static int make_tmap_segments(CUtensorMap* tm, const void* base, bool bf16, int nlon, int gs, long long rows, int box_cols) {
  TmapKey key;
  memset(&key, 0, sizeof(key));
  key.base = base; key.rank = 3; key.kind = bf16 ? 5 : 4;
  key.dims[0] = nlon; key.dims[1] = gs; key.dims[2] = rows; key.box[0] = box_cols;
  int slot = 0;
  if (tmap_lookup(key, tm, &slot)) return 0;
  PFN_encodeTiled enc = get_encode();
  if (!enc) { set_error("cuTensorMapEncodeTiled is unavailable"); return B200SHT_ERR_UNSUPPORTED; }
  static thread_local bool ctx_bound = false;
  if (!ctx_bound) { cudaFree(nullptr); ctx_bound = true; }
  const int es = bf16 ? 2 : 4, N2 = nlon / 8;
  cuuint64_t gd[3] = {(cuuint64_t)gs * N2, (cuuint64_t)(8 / gs), (cuuint64_t)rows};
  cuuint64_t gst[2] = {(cuuint64_t)gs * N2 * es, (cuuint64_t)nlon * es};
  cuuint32_t bx[3] = {(cuuint32_t)box_cols, (cuuint32_t)(8 / gs), 16}, el[3] = {1, 1, 1};
  if (gst[0] % 16 != 0 || gst[1] % 16 != 0 || (reinterpret_cast<uintptr_t>(base) & 15) != 0 || (box_cols * es) % 16 != 0) {
    set_error("tensor map (segments): base / pitch / box row not 16-byte aligned");
    return B200SHT_ERR_INVALID;
  }
  CUresult r = enc(tm, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<void*>(base), gd, gst, bx, el,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled (segments) failed (%d)", (int)r); return B200SHT_ERR_CUDA; }
  tmap_store(key, tm, slot);
  return 0;
}

constexpr int kDftAnaStages = 2;   // operand ring: one stage = one K-block (32 columns) of a 16-row tile = 4 planes x 16 KB
constexpr int kDftAnaMma = 8, kDftAnaLoader = 8, kDftAnaProd0 = 9, kDftAnaThreads = 544;   // warp roles (below)

struct DftAnaParams {
  alignas(64) CUtensorMap tmB;   // E tiles (32 j2 local, nkb * 64 rows), box (32, 32): K-major B operand
  alignas(64) CUtensorMap tmXc;  // the input as [R * nlat rows][8 / gs groups][gs * N2], box (Wc columns, 8 / gs, 16 rows), no swizzle: columns j2
  alignas(64) CUtensorMap tmXp;  // same, box (Wp columns, 8 / gs, 16 rows): partner columns N2 - j2
  float* X;
  const float2* tw;
  const float* rowscale;
  unsigned long long* prof;
  int R, nlat, nlon, kp, mmax, N2, half, M2, nkb, mode, ntiles, ktiles, nraw, gs;   // ktiles: 16-row tiles per image
};

// warps: 0..7 MMA + epilogue, two warpgroups of wgmma (rows 16 w .. + 15 of the tile = class w), 8 loader (TMA: the resident B, then the
// samples), 9..16 producers.  On wgmma the MMA warps issue a few instructions per K-block and sleep in their waits, so the issue slots go to
// the producers: eight of them (one item of every K-block each) at 17 warps and 120 registers, no spills.
// shared memory: [B resident: nkb x (cos 4 KB | sin 4 KB)][A ring: 2 x 4 planes x 16 KB][raw ring: nraw x 16 boxes][twiddles][barriers]
//
// Data flow of one (tile, K-block): the loader thread brings the 8 + 8 sample boxes the K-block needs -- for each j1 the 32 columns
// j2 = 32 kb .. + 31 and their 32 partner columns N2 - j2, 16 rows each -- into a raw stage with 16 TMA boxes (deep asynchronous prefetch,
// no registers: the first version's LDG -> register path stalled 2.1 cycles per issued instruction on the loads, with the 96-register cap
// allowing only half an item of prefetch).  The producer warps (one row pair per item) read their samples with LDS, run the two radix-8
// butterflies + twiddles on the two rows of a pair, and write Ye / Yo of the 8 classes into the operand stage; then the MMA warps contract
// the stage with E.  N2T > 0: nlon / 8 as a compile-time constant.
template <typename T, int N2T>
__global__ void __launch_bounds__(kDftAnaThreads, 1) dft_analysis_kernel(const __grid_constant__ DftAnaParams p) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ unsigned long long prof_s[16];   // wait-time profile (B200SHT_DFT_PROF): accumulated per CTA, flushed once at the end
  unsigned long long* const prof = (kDftProfile && p.prof) ? prof_s : nullptr;
  if (kDftProfile && threadIdx.x < 16) prof_s[threadIdx.x] = 0;
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* gbase = smem_raw + (base - raw);
  // TMA needs 16-byte aligned box starts (found on the GPU: an unaligned inner coordinate is an illegal instruction): a box starts at the
  // column rounded down to kAl elements and is wide enough to still contain the 32 wanted ones.  fp32 column boxes are exact (N2 % 4 == 0 is
  // required by the host for fp32 input).
  constexpr int kAl = 16 / (int)sizeof(T);                       // 8 (bf16) / 4 (fp32)
  constexpr int kWc = (sizeof(T) == 2) ? 40 : 32, kWp = (sizeof(T) == 2) ? 40 : 36;
  constexpr uint32_t kColBytes = 16u * kWc * sizeof(T), kParBytes = 16u * kWp * sizeof(T);   // one box: 16 rows
  constexpr uint32_t kRawBytes = 8u * (kColBytes + kParBytes);
  const uint32_t oB = 0, oA = 3 * 8192, oR = oA + kDftAnaStages * 65536, oT = oR + (uint32_t)p.nraw * kRawBytes, oBar = oT + 3 * 7 * 32 * 8;
  const uint32_t sBm = base + oB, sAr = base + oA, sRaw = base + oR;
  uint8_t* gA = gbase + oA;
  const uint8_t* gR = gbase + oR;
  float2* twS = reinterpret_cast<float2*>(gbase + oT);   // [nkb][7][32] twiddles of the producer lanes
  uint64_t* full = reinterpret_cast<uint64_t*>(gbase + oBar);
  uint64_t* empty = full + kDftAnaStages;
  uint64_t* raw_full = empty + kDftAnaStages;
  uint64_t* raw_empty = raw_full + 4;
  uint64_t* b_full = raw_empty + 4;

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;   // warp-uniform for the compiler
  pdl_trigger();
  const int nkb = p.nkb;
  const int N2 = N2T > 0 ? N2T : p.N2;
  // row segments per sample box group: the smallest gs with (gs * N2 elements) a multiple of 16 bytes, so that the segments gm, gm + gs, ...
  // of all rows form one 3-D TMA box (2 gs boxes per K-block instead of 16)
  const int gs = N2T > 0 ? dft_box_group(N2T, (int)sizeof(T)) : p.gs;
  for (int i = threadIdx.x; i < nkb * 7 * 32; i += blockDim.x) {
    const int ln = i & 31, c = (i >> 5) % 7 + 1, kb = i / 224;
    const int j2 = 32 * kb + ln;
    float2 w = (j2 <= p.half) ? p.tw[c * N2 + j2] : make_float2(1.f, 0.f);
#if B200_DFT_TF32_MODE == 2
    w.x *= kTruncComp; w.y *= kTruncComp;
#endif
    twS[i] = w;
  }
  if (threadIdx.x == 0) {
    for (int s = 0; s < kDftAnaStages; ++s) { mbar_init(&full[s], 8 * 32); mbar_init(&empty[s], kDftAnaMma); }   // a K-block = 8 row pairs
    for (int s = 0; s < p.nraw; ++s) { mbar_init(&raw_full[s], 1); mbar_init(&raw_empty[s], 8); }
    mbar_init(b_full, 1);
    fence_barrier_init();
    prefetch_tmap(&p.tmB);
    prefetch_tmap(&p.tmXc);
    prefetch_tmap(&p.tmXp);
  }
  // imaginary parts of class 0 (rows 0..15 of the planes Ye_i, Yo_i of every operand stage): zero, never written again
  for (int i = threadIdx.x; i < kDftAnaStages * 2 * 512; i += blockDim.x) {
    const int st = i >> 10, pl = (i >> 9) & 1, off = i & 511;
    reinterpret_cast<float*>(gA + (size_t)st * 65536)[(pl ? 12288 : 4096) + off] = 0.f;
  }
  fence_proxy_async();   // wgmma reads them through the async proxy
  __syncthreads();
  const long long t_cta0 = (kDftProfile && p.prof && threadIdx.x == 0) ? clock64() : 0;
  pdl_wait();   // the prologue read plan constants only (twiddles); samples and latspec belong to other kernels until here

  if (warp == kDftAnaLoader) {
    // ------------------------------------------------------------------------------------- resident B, then the samples
    if (lane == 0) {
      mbar_expect_tx(b_full, (uint32_t)nkb * 8192);
      for (int kb = 0; kb < nkb; ++kb) {
        tma_load_2d(sBm + kb * 8192, &p.tmB, b_full, 0, kb * 64);
        tma_load_2d(sBm + kb * 8192 + 4096, &p.tmB, b_full, 0, kb * 64 + 32);
      }
      int n = 0;
      for (int ti = blockIdx.x; ti < p.ntiles; ti += gridDim.x, ++n) {
        const int r = ti / p.ktiles, row0 = r * p.nlat + (ti - r * p.ktiles) * 16;
        for (int kb = 0; kb < nkb; ++kb) {
          const int g = n * nkb + kb, rs = g % p.nraw, it = g / p.nraw;
          if (it > 0) prof_wait_nocall(prof, 2, &raw_empty[rs], (it - 1) & 1, true);
          mbar_expect_tx(&raw_full[rs], kRawBytes);
          const uint32_t dst = sRaw + rs * kRawBytes;
#pragma unroll
          for (int gm = 0; gm < 8; ++gm) {
            if (gm >= gs) break;
            // one box = the columns of the row segments j1 = gm, gm + gs, ...: (kW columns) x (8 / gs segments) x (16 rows)
            const int sc = N2 * gm + 32 * kb, sp = N2 * gm + N2 - 32 * kb - 31;   // first wanted column / partner column (sp < 0 only for N2 < 31)
            tma_load_3d(dst + gm * (8 / gs) * kColBytes, &p.tmXc, &raw_full[rs], (sc / kAl) * kAl, 0, row0);
            tma_load_3d(dst + 8 * kColBytes + gm * (8 / gs) * kParBytes, &p.tmXp, &raw_full[rs], sp < 0 ? 0 : (sp / kAl) * kAl, 0, row0);
          }
        }
      }
    }
    __syncwarp();
  } else if (warp < kDftAnaMma) {
    // ------------------------------------------------------------------------------------------- MMA + epilogue
    // D[(c, kr)][m2] = Xre: Ye_r cos + Yo_i sin,  Xim: Ye_i cos - Yo_r sin over the j2 of all K-blocks, on wgmma.m64n32k8: warpgroup wg
    // takes the rows 64 wg .. + 63 of the operand stage (classes 4 wg .. 4 wg + 3) against the 32 orders m2 of the resident E, four
    // products per k8 step, the negated one through the instruction's B scale.  Each warp's part of the m64n32 accumulator is the m16n8
    // fragment layout repeated: class c = warp, rows the latitudes kr = lane / 4 (+ 8), columns the orders m2 = 8 j + 2 (lane % 4) (+ 1).
    // One K-block's wgmma stay in flight: the stage before is released once wait_group 1 has retired its group.  No function call may
    // appear in this kernel (ptxas would serialize every wgmma): all its waits are the call-free ones.
    const size_t plane = (size_t)p.R * p.kp;
    const int c = warp, gq = lane >> 2, q = lane & 3;
    const uint32_t aw = sAr + (uint32_t)(warp >> 2) * 8192;   // this warpgroup's 64 rows of plane Ye_r of stage 0
    mbar_wait_nocall(b_full, 0);
    int n = 0;
    for (int ti = blockIdx.x; ti < p.ntiles; ti += gridDim.x, ++n) {
      const int r = ti / p.ktiles, k0 = (ti - r * p.ktiles) * 16;
      float acc[8][4];   // [0..3]: Xre, [4..7]: Xim, columns 8 j .. 8 j + 7
      int prev = 0;
      for (int kb = 0; kb < nkb; ++kb) {
        const int g = n * nkb + kb, s = g % kDftAnaStages, it = g / kDftAnaStages;
        prof_wait_nocall(prof, 3, &full[s], it & 1, lane == 0);
        const uint32_t a0 = aw + (uint32_t)s * 65536;   // planes Ye_r, Ye_i, Yo_r, Yo_i, 16 KB apart
        const uint64_t d_er = wgmma_desc_kmajor(a0), d_ei = wgmma_desc_kmajor(a0 + 16384);
        const uint64_t d_or = wgmma_desc_kmajor(a0 + 32768), d_oi = wgmma_desc_kmajor(a0 + 49152);
        const uint64_t d_c = wgmma_desc_kmajor(sBm + kb * 8192), d_s = wgmma_desc_kmajor(sBm + kb * 8192 + 4096);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int sd = (kb > 0 || k > 0) ? 1 : 0;   // the first product of a tile initializes the accumulators
          wgmma_tf32<32, 1, 8, 0>(acc, d_er + 2 * k, d_c + 2 * k, sd);    // Xre += Ye_r cos
          wgmma_tf32<32, 1, 8, 4>(acc, d_ei + 2 * k, d_c + 2 * k, sd);    // Xim += Ye_i cos
          wgmma_tf32<32, 1, 8, 0>(acc, d_oi + 2 * k, d_s + 2 * k, 1);     // Xre += Yo_i sin
          wgmma_tf32<32, -1, 8, 4>(acc, d_or + 2 * k, d_s + 2 * k, 1);    // Xim -= Yo_r sin
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (kb > 0 && lane == 0) mbar_arrive(&empty[prev]);   // this warp's wgmma of the K-block before have read its stage
        prev = s;
      }
      wgmma_wait<0>();
      wgmma_fence_operands(acc);
      if (lane == 0) mbar_arrive(&empty[prev]);
      if (prof && lane == 0) atomicAdd(prof + 5, 1ull);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int k = k0 + gq + 8 * h;
        if (k >= p.kp) continue;
        const float rs = (p.mode == 0) ? ((k < p.nlat) ? __ldg(p.rowscale + k) : 0.f) : 1.f;
        float* xb = p.X + (size_t)r * p.kp + k;
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int m = c + 8 * (8 * j + 2 * q + e);
            if (m >= p.mmax) continue;
            // The output is a TF32 value -- the bias-compensated truncation (see B200_DFT_TF32_MODE above) folded into the scale factor,
            // then the 13 low bits cleared (one LOP3 instead of the 3 instructions of cvt.rna).  The TF32 Legendre GEMM ignores those bits
            // anyway; readers of the fp32 value (the bias gradient, latspec_unpack) then see an unbiased TF32 value instead of one scaled
            // by 1 + 2^-10 / 3.
            const float sc = ((p.mode == 0) ? rs : ((m == 0 || 2 * m == p.nlon) ? 1.f : 2.f)) * kTruncComp;
            float* dst = xb + (size_t)m * 2 * plane;
            dst[0] = __uint_as_float(__float_as_uint(acc[j][2 * h + e] * sc) & 0xffffe000u);
            dst[plane] = __uint_as_float(__float_as_uint(acc[4 + j][2 * h + e] * sc) & 0xffffe000u);
          }
      }
    }
  } else {
    // ------------------------------------------------------------------------------------------- producers
    // Work item = (K-block kb, row pair q): rows 2q, 2q + 1 of the tile in the halves of register pairs (pr), lanes = the 32 columns of the
    // K-block.  Items are taken in K-block-major order (item = kb * 8 + q; warp w does w, w + nprod, ...): the MMAs of K-block kb run while
    // the warps work on kb + 1.  Each warp takes its items in increasing order, so every wait is on an earlier K-block: no cycle.  With
    // nprod <= 8 every warp has an item in every K-block (8 consecutive items cover all warps), so the raw_full and empty waits of a warp
    // are for consecutive uses of a stage and never alias a phase two uses old.
    const int pw = warp - kDftAnaProd0;
    constexpr int nprod = kDftAnaThreads / 32 - kDftAnaProd0;
    static_assert(nprod >= 1 && nprod <= 8, "every producer warp must take an item of every K-block (8 items each)");
    constexpr bool kBf16 = (sizeof(T) == 2);
    const T* const rawS = reinterpret_cast<const T*>(gR);
    int n = 0;
    for (int ti = blockIdx.x; ti < p.ntiles; ti += gridDim.x, ++n) {
      const int r = ti / p.ktiles, kt16 = (ti - r * p.ktiles) * 16;
      for (int item = pw; item < 8 * nkb; item += nprod) {
        const int kb = item >> 3, q = item & 7;
        const int k0 = kt16 + 2 * q;
        const int g = n * nkb + kb;
        const int j2 = 32 * kb + lane;
        const int rs = g % p.nraw;
        prof_wait_nocall(prof, 0, &raw_full[rs], (g / p.nraw) & 1, lane == 0);
        if (prof && lane == 0) atomicAdd(prof + 7, 1ull);
        const T* const rb = rawS + (size_t)rs * (kRawBytes / sizeof(T));
        pr xa[8], xb[8];
        // No per-lane masks on the samples: lanes beyond N2 / 2 feed rows of E that are zero, and the column N2 / 2 (its own partner) is
        // simply counted twice against a halved row of E; only column 0 (no partner) and rows beyond nlat are patched below, in branches
        // that are uniform (and rarely taken).
#pragma unroll
        for (int j1 = 0; j1 < 8; ++j1) {
          // column box gm: [16 rows][npb segments][kWc]; partner box: [16 rows][npb][kWp]; both start at the wanted column rounded down to kAl
          const int gm = j1 % gs, ga = j1 / gs, npb = 8 / gs;                  // box gm, segment ga of its npb segments
          const int sc = N2 * gm + 32 * kb, sp = N2 * gm + N2 - 32 * kb - 31;
          const int ic = sc - (sc / kAl) * kAl + lane;                          // column j2 = 32 kb + lane
          int ip = N2 * gm + N2 - j2 - (sp < 0 ? 0 : (sp / kAl) * kAl);          // column N2 - j2
          ip = ip < 0 ? 0 : (ip > kWp - 1 ? kWp - 1 : ip);                      // lanes without a partner read anything inside the box
          const T* b0 = rb + gm * (16 * npb * kWc) + (2 * q) * (npb * kWc) + ga * kWc;
          const T* b1 = rb + 8 * (16 * kWc) + gm * (16 * npb * kWp) + (2 * q) * (npb * kWp) + ga * kWp;
          const int rowc = npb * kWc, rowp = npb * kWp;                         // row pitch inside a box
          if constexpr (kBf16) {
            xa[j1] = make_pr(__uint_as_float((uint32_t)reinterpret_cast<const unsigned short*>(b0)[ic] << 16),
                             __uint_as_float((uint32_t)reinterpret_cast<const unsigned short*>(b0)[rowc + ic] << 16));
            xb[j1] = make_pr(__uint_as_float((uint32_t)reinterpret_cast<const unsigned short*>(b1)[ip] << 16),
                             __uint_as_float((uint32_t)reinterpret_cast<const unsigned short*>(b1)[rowp + ip] << 16));
          } else {
            xa[j1] = make_pr(reinterpret_cast<const float*>(b0)[ic], reinterpret_cast<const float*>(b0)[rowc + ic]);
            xb[j1] = make_pr(reinterpret_cast<const float*>(b1)[ip], reinterpret_cast<const float*>(b1)[rowp + ip]);
          }
        }
        if (kb == 0) {                                 // column 0 has no partner
#pragma unroll
          for (int j1 = 0; j1 < 8; ++j1) xb[j1] = (lane == 0) ? make_pr(0.f, 0.f) : xb[j1];
        }
        if (k0 + 1 >= p.nlat) {                        // rows beyond nlat belong to the next image (or are out of bounds): zeros
          const bool row0ok = k0 < p.nlat;
#pragma unroll
          for (int j1 = 0; j1 < 8; ++j1) {
            xa[j1] = make_pr(row0ok ? xa[j1].v.x : 0.f, 0.f);
            xb[j1] = make_pr(row0ok ? xb[j1].v.x : 0.f, 0.f);
          }
        }
        pr er[8], ei[8], br[8], bi[8];
        float2 tw[8], tp[8];
        tw[0] = make_float2(1.f, 0.f);
        const float2* const twl = twS + kb * 224 + lane;   // tw[c] = twl[(c - 1) * 32], already scaled for the truncation compensation
#pragma unroll
        for (int c = 1; c < 8; ++c) tw[c] = twl[(c - 1) * 32];
        dft_partner_twiddles(tw, tp);   // products of the tw components with constants of modulus 1: they carry the (1 + f) factor too
        dft_ana_radix8<pr>(xa, tw, er, ei);
        dft_ana_radix8<pr>(xb, tp, br, bi);
        // the raw stage may be refilled once every lane's shared-memory loads of it have completed: the butterflies have consumed them.  (An
        // arrival right after issuing the loads let the next TMA box overwrite samples that were still being read.)
        __syncwarp();
        if (lane == 0) mbar_arrive(&raw_empty[rs]);
        const int s = g % kDftAnaStages, it = g / kDftAnaStages;
        if (it > 0) prof_wait_nocall(prof, 1, &empty[s], (it - 1) & 1, lane == 0);
        float* const stg = reinterpret_cast<float*>(gA + (size_t)s * 65536);
        const int kr0 = 2 * q;
        // swizzled K-major position of (row c * 16 + kr, column lane): the XOR term depends on kr only (16 c is a multiple of 8)
        float* const d0 = stg + kr0 * 32 + ((((lane >> 2) ^ (kr0 & 7)) << 2) | (lane & 3));
        float* const d1 = stg + (kr0 + 1) * 32 + ((((lane >> 2) ^ ((kr0 + 1) & 7)) << 2) | (lane & 3));
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          pr ye_r = er[c] + br[c], yo_r = er[c] - br[c];
          if (c == 0) { ye_r = pr_operand_unscaled(ye_r); yo_r = pr_operand_unscaled(yo_r); }
          else { ye_r = pr_operand(ye_r); yo_r = pr_operand(yo_r); }
          d0[c * 512] = ye_r.v.x; d1[c * 512] = ye_r.v.y;
          d0[8192 + c * 512] = yo_r.v.x; d1[8192 + c * 512] = yo_r.v.y;
          if (c != 0) {   // the imaginary parts of class 0 are zero: those 16 rows of the two planes are cleared once at kernel start
            const pr ye_i = pr_operand(ei[c] + bi[c]), yo_i = pr_operand(ei[c] - bi[c]);
            d0[4096 + c * 512] = ye_i.v.x; d1[4096 + c * 512] = ye_i.v.y;
            d0[12288 + c * 512] = yo_i.v.x; d1[12288 + c * 512] = yo_i.v.y;
          }
        }
        fence_proxy_async();   // wgmma reads the stage through the async proxy: every writing thread fences and arrives
        mbar_arrive(&full[s]);
      }
    }
  }
  __syncthreads();
  if (kDftProfile && p.prof && threadIdx.x == 0) prof_s[6] = (unsigned long long)(clock64() - t_cta0);
  if (kDftProfile) __syncthreads();
  if (kDftProfile && p.prof && threadIdx.x < 16) atomicAdd(p.prof + threadIdx.x, prof_s[threadIdx.x]);
}

int dft_analysis(const Plan* pl, const void* x, int dtype, int B, int C, float* X, int mode, cudaStream_t st) {
  const DftTables* t = static_cast<const DftTables*>(pl->dft_state);
  B200_REQUIRE(t != nullptr, "dft_analysis: plan has no DFT tables");
  const int R = B * C;
  DftAnaParams p;
  memset(&p, 0, sizeof(p));
  p.X = X; p.tw = t->tw; p.rowscale = pl->d_rowscale; p.prof = dft_prof_buffer();
  p.R = R; p.nlat = pl->nlat; p.nlon = pl->nlon; p.kp = pl->kp; p.mmax = pl->mmax;
  p.N2 = t->N2; p.half = t->half; p.M2 = t->M2; p.nkb = t->nkb; p.mode = mode;
  p.ktiles = (pl->kp + 15) / 16; p.ntiles = R * p.ktiles;
  const bool bf16 = (dtype == B200SHT_BF16);
  p.nraw = bf16 ? 3 : 2;   // raw stages of 20 / 34 KB
  {
    long long d[2] = {32, (long long)t->nkb * 64}, s[2] = {1, 32};
    int bx[2] = {32, 32};
    int rc = make_tmap(&p.tmB, t->eb, 2, d, s, bx);
    if (rc) return rc;
  }
  B200_REQUIRE(bf16 || t->N2 % 4 == 0, "dft_analysis: fp32 input needs nlon %% 32 == 0 (16-byte aligned TMA boxes)");
  {
    p.gs = dft_box_group(t->N2, bf16 ? 2 : 4);
    int rc = make_tmap_segments(&p.tmXc, x, bf16, pl->nlon, p.gs, (long long)R * pl->nlat, bf16 ? 40 : 32);
    if (!rc) rc = make_tmap_segments(&p.tmXp, x, bf16, pl->nlon, p.gs, (long long)R * pl->nlat, bf16 ? 40 : 36);
    if (rc) return rc;
  }
  const size_t raw_bytes = bf16 ? (size_t)8 * 16 * (40 + 40) * 2 : (size_t)8 * 16 * (32 + 36) * 4;
  const size_t smem = 1024 + 3 * 8192 + (size_t)kDftAnaStages * 65536 + p.nraw * raw_bytes + 3 * 7 * 32 * 8 + 256;
  const int sms = usable_sms(pl->sm_count > 0 ? pl->sm_count : 132);
  const int ctas = p.ntiles < sms ? p.ntiles : sms;
  const int threads = kDftAnaThreads;
#define B200_LAUNCH_ANA(TT, NN)                                                                                                          \
  do {                                                                                                                                  \
    struct Tag {};                                                                                                                        \
    B200_CHECK_CUDA((ensure_dynamic_smem<Tag>(dft_analysis_kernel<TT, NN>, smem)));                                                      \
    B200_CHECK_CUDA(launch_pdl(dft_analysis_kernel<TT, NN>, dim3(ctas), dim3(threads), smem, st, p));                                                                         \
  } while (0)
#define B200_DISPATCH_ANA(TT)                                            \
  switch (t->N2) {                                                       \
    case 180: B200_LAUNCH_ANA(TT, 180); break; /* nlon 1440 */           \
    case 90: B200_LAUNCH_ANA(TT, 90); break;   /* nlon  720 */           \
    case 60: B200_LAUNCH_ANA(TT, 60); break;   /* nlon  480 */           \
    default: B200_LAUNCH_ANA(TT, 0); break;                              \
  }
  if (bf16) { B200_DISPATCH_ANA(__nv_bfloat16) } else { B200_DISPATCH_ANA(float) }
#undef B200_DISPATCH_ANA
#undef B200_LAUNCH_ANA
  B200_CHECK_LAUNCH();
  return 0;
}

// ============================================================================================ host emulation
// The same factorisation and the same __host__ __device__ radix-8 code as the kernels, with the tensor-core sums done in double
// precision on the host: unit-tests the index maps, twiddles and butterflies without a GPU (b200sht_debug_dft_host).
int dft_host(int N, int mmax, int direction, int mode, const float* rowscale, const float* in, float* out) {
  if (!dft_shape_ok(N, mmax)) { set_error("debug_dft_host: unsupported (nlon=%d, mmax=%d)", N, mmax); return B200SHT_ERR_UNSUPPORTED; }
  const int N2 = N / 8, half = N2 / 2, M2 = (mmax + 7) / 8;
  const float rs = rowscale ? rowscale[0] : 1.f;
  auto twid = [&](int j, float2* tw) {
    for (int c = 0; c < 8; ++c) {
      const double a = 2.0 * M_PI * (double)(c * j) / (double)N;
      tw[c] = make_float2((float)cos(a), (float)sin(a));
    }
  };
  if (direction == 1) {
    // in: float[2 * mmax] interleaved (re, im) -> out: float[N]
    std::vector<double> zr(8 * M2, 0.0), zi(8 * M2, 0.0);
    for (int m = 0; m < mmax; ++m) { zr[m] = in[2 * m]; zi[m] = in[2 * m + 1]; }
    const bool has_nyq = (mmax == N / 2 + 1);
    for (int j2 = 0; j2 <= half; ++j2) {
      float s1[8], s2[8], s3[8], s4[8];
      for (int c = 0; c < 8; ++c) {
        double a1 = 0, a2 = 0, a3 = 0, a4 = 0;
        for (int m2 = 0; m2 < M2; ++m2) {
          const double b = 2.0 * M_PI * (double)(((long long)m2 * j2) % N2) / (double)N2;
          a1 += cos(b) * zr[c + 8 * m2]; a2 += sin(b) * zi[c + 8 * m2]; a3 += sin(b) * zr[c + 8 * m2]; a4 += cos(b) * zi[c + 8 * m2];
        }
        s1[c] = (float)a1; s2[c] = (float)a2; s3[c] = (float)a3; s4[c] = (float)a4;
      }
      float2 tw[8], tp[8];
      twid(j2, tw);
      dft_partner_twiddles(tw, tp);
      for (int side = 0; side < 2; ++side) {
        if (side == 1 && (j2 == 0 || 2 * j2 == N2)) continue;
        const int jj = side ? N2 - j2 : j2;
        float vr[8], vi[8], x[8];
        for (int c = 0; c < 8; ++c) {
          vr[c] = side ? s1[c] + s2[c] : s1[c] - s2[c];
          vi[c] = side ? s4[c] - s3[c] : s3[c] + s4[c];
        }
        dft_syn_radix8<float>(vr, vi, side ? tp : tw, x);
        for (int j1 = 0; j1 < 8; ++j1) {
          const int j = N2 * j1 + jj;
          float v = x[j1];
          if (mode == 0) {
            v = 2.f * v - (float)zr[0];
            if (has_nyq) v -= (float)zr[N / 2] * ((j & 1) ? -1.f : 1.f);
          } else {
            v *= rs;
          }
          out[j] = v;
        }
      }
    }
    return 0;
  }
  // analysis: in float[N] -> out float[2 * mmax]
  std::vector<double> dre(8 * M2, 0.0), dim(8 * M2, 0.0);
  for (int j2 = 0; j2 <= half; ++j2) {
    float2 tw[8], tp[8];
    twid(j2, tw);
    dft_partner_twiddles(tw, tp);
    float xa[8], er[8], ei[8], orr[8], oi[8];
    for (int j1 = 0; j1 < 8; ++j1) xa[j1] = in[N2 * j1 + j2];
    dft_ana_radix8<float>(xa, tw, er, ei);
    const bool paired = (j2 != 0 && 2 * j2 != N2);
    if (paired) {
      float xb[8], br[8], bi[8];
      for (int j1 = 0; j1 < 8; ++j1) xb[j1] = in[N2 * j1 + N2 - j2];
      dft_ana_radix8<float>(xb, tp, br, bi);
      for (int c = 0; c < 8; ++c) { orr[c] = er[c] - br[c]; oi[c] = ei[c] - bi[c]; er[c] += br[c]; ei[c] += bi[c]; }
    } else {
      for (int c = 0; c < 8; ++c) { orr[c] = 0.f; oi[c] = 0.f; }
    }
    for (int c = 0; c < 8; ++c)
      for (int m2 = 0; m2 < M2; ++m2) {
        const double b = 2.0 * M_PI * (double)(((long long)m2 * j2) % N2) / (double)N2;
        dre[c + 8 * m2] += cos(b) * er[c] + sin(b) * oi[c];
        dim[c + 8 * m2] += cos(b) * ei[c] - sin(b) * orr[c];
      }
  }
  for (int m = 0; m < mmax; ++m) {
    const double sc = mode == 0 ? (double)rs : ((m == 0 || 2 * m == N) ? 1.0 : 2.0);
    out[2 * m] = (float)(dre[m] * sc);
    out[2 * m + 1] = (float)(dim[m] * sc);
  }
  return 0;
}

}  // namespace b200sht
