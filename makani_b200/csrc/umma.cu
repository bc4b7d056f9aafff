// Tensor-core path (B200SHT_PREC_TF32): the Legendre contractions and the dense channel mix as TMA-fed TF32 GEMMs with fp32
// accumulation.
//
//   one persistent engine (umma_kernel<Traits, NB, SPLIT>, one CTA per SM walking the tile list): warps 0..7 = consumers (two
//   warpgroups of 64 rows), warp 8 lane 0 = TMA producer; consumer warp w owns rows 16 w .. + 15 of the 128-row tile and stores its
//   accumulators itself (the TF32 synthesis stages them for bulk stores instead).  The tile width (NB fragments of 8 columns) and the
//   3 x TF32 mode are template parameters: the MMA loop is straight-line code without per-fragment predicates, and no instantiation spills
//   registers.  A ring of `stages` operand stages guarded by full/empty mbarriers runs continuously across tiles, so the producer
//   prefetches the next tile while the consumers finish the current one and write it out.
//
//   five Traits supply the per-operation pieces (tile coordinates, TMA boxes, MMA list, epilogue):
//     AnaTraits   spec[l][m][n]  = sum_k P[m][l][k] X[m][n][k]          A K-major,  B K-major     (RealSHT einsum "...km,mlk->...lm")
//     SynTraits   Z[m][n][k]     = sum_l P[m][l][k] spec[l][m][n]       A MN-major, B MN-major    (InverseRealSHT "...lm,mlk->...km")
//     MixFwd      y[row][o]      = sum_i x[row][i] w[i][o]   (complex)  A K-major,  B MN-major    (contractions.py:23 "bgixy,giox->bgoxy")
//     MixDgrad    gx[row][i]     = sum_o gy[row][o] conj(w[i][o])       A K-major,  B K-major
//     MixWgrad    gw[i][o]       = sum_row conj(x[row][i]) gy[row][o]   A MN-major, B MN-major
//   complex products use planar operands: 4 real MMAs into two accumulators (real, imaginary).
//
// Two MMA paths.  The TF32 GEMMs with two K-major operands (AnaTraits, MixDgradTraits; kKMajor) run on wgmma straight from the TMA
// ring: each warpgroup issues wgmma.m64nNk8 on its 64 rows against the whole tile width from shared-memory descriptors, keeps one
// stage's MMAs in flight and releases the stage before after wgmma.wait_group 1.  wgmma reads TF32 operands from shared memory only
// K-major, so synthesis (A and B), mix forward (B) and wgrad (A and B) stay on mma.m16n8k8 (TF32) fed by per-warp fragment loads, and so
// does the 3 x TF32 analysis (three products per fragment pair).  All shared-memory operand tiles use the 128-byte swizzle; every TMA box
// is [rows][32 floats] so it lands as rows of 128 B, the K-major layout of the wgmma descriptors.  The mma.sync fragments are read with
// 8- and 16-byte shared loads, conflict-free: within each 32-wide stage the K order, and for MN-major operands the row / column order, is
// permuted so that each thread's operands are contiguous (layouts KK / MM / KM below); the epilogues undo the permutation and store 8- or
// 16-byte vectors where the output is contiguous along the permuted index.  The H100 cost of this engine is recorded in DESIGN.md
// section 9.
#include "umma_common.cuh"
#include "wgmma_tf32.cuh"
#include <mutex>

namespace b200sht {

// ======================================================================================================= engine
constexpr int kConsumerWarps = 8;                         // 8 x 16 rows = the 128-row tile, two warpgroups of 64 rows
constexpr int kProducerWarp = kConsumerWarps;             // warps 0..7: MMA + epilogue, warp 8: TMA producer
constexpr int kUmmaThreads = 32 * (1 + kConsumerWarps);
constexpr int kMaxStages = 8;

struct EngineParams {
  int stages;
  uint32_t stage_bytes, tx_bytes;
  uint32_t out_bytes;      // output staging after the ring (bulk-store epilogue of SynTraits), 0 for the register epilogues
  int gx, gy, gz;          // logical tile grid (x fastest); CTAs walk it round-robin
  int split;               // 3 x TF32 (strict fp32 on the tensor cores): every stage also holds the residual tiles of both operands, `lo_off`
  uint32_t lo_off;         // bytes after the main tiles, and each MMA becomes hi.hi + hi.lo + lo.hi into the same accumulator
};

// ------------------------------------------------------------------------------------------- fragment layouts
// The engine is instantiated for a compile-time number NB of 8-column fragments per warp (the host pads N up to a built width; padded
// columns read zeros or stale shared memory and are never stored).  A warp's accumulator is float acc[NB][4] (real) or acc[2 NB][4]
// (complex: real part in 0 .. NB-1, imaginary part in NB .. 2 NB-1).  K is summed over, so the 32 K of a stage may be visited in any order
// that is the same for both operands, and the rows / columns of a fragment may be any rows / columns of the tile as long as the epilogue
// maps them back.  Three layouts, chosen per GEMM so that every fragment load is 8 or 16 bytes and bank-conflict-free under the 128-byte
// swizzle (g = lane / 4, q = lane % 4; the MMA's K positions q, q + 4 of k8 step s are called (s, q, h = 0 / 1)):
//   KK (both operands K-major: 3 x TF32 analysis) (s, q, h) -> K 8 q + 2 s + h: thread q owns K 8q .. 8q+7 of every row, two 16-byte loads
//        per row and stage (one per pair of k8 steps); rows / columns are the plain m16n8 ones.
//   MM (both operands MN-major: synthesis, wgrad) (s, q, h) -> K 8 s + 2 q + h.  A: the warp's rows g, g + 8 are adjacent physical rows
//        2g, 2g + 1 (one 8-byte load per K row); B: column g of fragments 4J .. 4J + 3 is physical column 32 J + 4 g .. + 3 (one 16-byte
//        load serves four fragments).
//   KM (A K-major, B MN-major: mix forward)        K as MM, B as MM; A: one 8-byte load per row and k8 step, rows g, g + 8 at physical
//        2 (g % 4) + g / 4 and that + 8, so that the eight rows of a load phase fall on distinct chunks after the swizzle.
enum class Lay { KK, MM, KM };

// tile row of accumulator element e (0..3) of this lane: rows of a fragment are g (e < 2) and g + 8 (e >= 2)
template <Lay L>
__device__ __forceinline__ int frag_row(int row0, int h) {
  const int g = (threadIdx.x & 31) >> 2;
  if (L == Lay::KK) return row0 + g + 8 * h;
  if (L == Lay::MM) return row0 + 2 * g + h;
  return row0 + 2 * (g & 3) + (g >> 2) + 8 * h;
}

// A fragments of one stage, KK: f[t] = k8 step 2 hh + t
__device__ __forceinline__ void lda_kk(const uint8_t* a, int row0, int hh, uint32_t (&f)[2][4]) {
  const int lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
  const uint32_t ko = (8 * q + 4 * hh) * 4;
  const uint4 x = lds128(a, (row0 + g) * 128 + ko), y = lds128(a, (row0 + g + 8) * 128 + ko);
  f[0][0] = x.x; f[0][1] = y.x; f[0][2] = x.y; f[0][3] = y.y;
  f[1][0] = x.z; f[1][1] = y.z; f[1][2] = x.w; f[1][3] = y.w;
}
// B fragment j, KK: f[t] = k8 step 2 hh + t
__device__ __forceinline__ void ldb_kk(const uint8_t* b, int j, int hh, uint32_t (&f)[2][2]) {
  const int lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
  const uint4 x = lds128(b, (8 * j + g) * 128 + (8 * q + 4 * hh) * 4);
  f[0][0] = x.x; f[0][1] = x.y; f[1][0] = x.z; f[1][1] = x.w;
}
// A fragment of k8 step s, MM (MN-major, [32 K][32 M] blocks of 4096 bytes)
__device__ __forceinline__ void lda_mm(const uint8_t* a, int row0, int s, uint32_t (&f)[4]) {
  const int lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
  const uint32_t o = (row0 >> 5) * 4096 + (8 * s + 2 * q) * 128 + ((row0 & 31) + 2 * g) * 4;
  const uint2 x = lds64(a, o), y = lds64(a, o + 128);
  f[0] = x.x; f[1] = x.y; f[2] = y.x; f[3] = y.y;
}
// A fragment of k8 step s, KM (K-major rows)
__device__ __forceinline__ void lda_km(const uint8_t* a, int row0, int s, uint32_t (&f)[4]) {
  const int lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
  const uint32_t o = (row0 + 2 * (g & 3) + (g >> 2)) * 128 + (8 * s + 2 * q) * 4;
  const uint2 x = lds64(a, o), y = lds64(a, o + 8 * 128);
  f[0] = x.x; f[1] = y.x; f[2] = x.y; f[3] = y.y;
}
// B fragments 4 J .. 4 J + 3 of k8 step s, MM / KM (MN-major)
__device__ __forceinline__ void ldb_mn(const uint8_t* b, int J, int s, uint32_t (&f)[4][2]) {
  const int lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
  const uint32_t o = J * 4096 + (8 * s + 2 * q) * 128 + g * 16;
  const uint4 x = lds128(b, o), y = lds128(b, o + 128);
  f[0][0] = x.x; f[0][1] = y.x; f[1][0] = x.y; f[1][1] = y.y;
  f[2][0] = x.z; f[2][1] = y.z; f[3][0] = x.w; f[3][1] = y.w;
}
template <int S>
__device__ __forceinline__ void sgn(const uint32_t (&a)[4], uint32_t (&o)[4]) {   // exact negation for S < 0: flip the sign bits
#pragma unroll
  for (int i = 0; i < 4; ++i) o[i] = S > 0 ? a[i] : a[i] ^ 0x80000000u;
}

// acc[j] += A(the warp's 16 rows) B(fragment j) over the 32 K of one stage.  SPLIT (3 x TF32): the residual tiles lie `lo` bytes after A and
// B, and every product becomes hi.hi + hi.lo + lo.hi, issued per fragment so that no operand is loaded twice.  KK serves the 3 x TF32
// analysis only: the plain TF32 K-major GEMMs run on wgmma (AnaTraits::wgmma, MixDgradTraits::wgmma).
template <Lay L, int NB, bool SPLIT>
__device__ __forceinline__ void gemm_real(const uint8_t* a, const uint8_t* b, uint32_t lo, int row0, float (&acc)[NB][4]) {
  if constexpr (L == Lay::KK) {
    static_assert(SPLIT, "KK on mma.sync: 3 x TF32 only");
#pragma unroll 2
    for (int hh = 0; hh < 2; ++hh) {
      uint32_t fa[2][4], la[2][4];
      lda_kk(a, row0, hh, fa);
      lda_kk(a + lo, row0, hh, la);
#pragma unroll
      for (int j = 0; j < NB; ++j) {
        uint32_t fb[2][2], lb[2][2];
        ldb_kk(b, j, hh, fb);
        ldb_kk(b + lo, j, hh, lb);
#pragma unroll
        for (int t = 0; t < 2; ++t) {
          mma_tf32(acc[j], fa[t], fb[t]);
          mma_tf32(acc[j], fa[t], lb[t]);
          mma_tf32(acc[j], la[t], fb[t]);
        }
      }
    }
  } else {
    static_assert(NB % 4 == 0, "MN-major B: NB must be a multiple of 4");
#pragma unroll
    for (int s = 0; s < 4; ++s) {
      uint32_t fa[4], la[4];
      if (L == Lay::MM) { lda_mm(a, row0, s, fa); if (SPLIT) lda_mm(a + lo, row0, s, la); }
      else { lda_km(a, row0, s, fa); if (SPLIT) lda_km(a + lo, row0, s, la); }
#pragma unroll
      for (int J = 0; J < NB / 4; ++J) {
        uint32_t fb[4][2], lb[4][2];
        ldb_mn(b, J, s, fb);
        if (SPLIT) ldb_mn(b + lo, J, s, lb);
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          mma_tf32(acc[4 * J + c], fa, fb[c]);
          if (SPLIT) { mma_tf32(acc[4 * J + c], fa, lb[c]); mma_tf32(acc[4 * J + c], la, fb[c]); }
        }
      }
    }
  }
}
// complex product of planar operands over one stage (S1..S3 = +-1):  re += ar br + S1 ai bi,  im += S2 ar bi + S3 ai br.  The signs go on
// the A fragments (MN-major B: a B load holds four fragments); the two B planes are consumed one after the other, so only one is held at
// a time.  MN-major B only (KM, MM): the K-major complex GEMM (dgrad) runs on wgmma.
template <Lay L, int NB, int S1, int S2, int S3>
__device__ __forceinline__ void gemm_cplx(const uint8_t* ar, const uint8_t* ai, const uint8_t* br, const uint8_t* bi, int row0, float (&acc)[2 * NB][4]) {
  static_assert(L != Lay::KK, "gemm_cplx: MN-major B only");
  static_assert(NB % 4 == 0, "MN-major B: NB must be a multiple of 4");
#pragma unroll 1   // one k8 step at a time: unrolled, the loads of the next steps are hoisted and the accumulators spill
  for (int s = 0; s < 4; ++s) {
    uint32_t fr[4], fi[4], x[4];
    if (L == Lay::MM) { lda_mm(ar, row0, s, fr); lda_mm(ai, row0, s, fi); }
    else { lda_km(ar, row0, s, fr); lda_km(ai, row0, s, fi); }
#pragma unroll
    for (int J = 0; J < NB / 4; ++J) {
      uint32_t g[4][2];
      ldb_mn(br, J, s, g);
      sgn<S3>(fi, x);
#pragma unroll
      for (int c = 0; c < 4; ++c) { mma_tf32(acc[4 * J + c], fr, g[c]); mma_tf32(acc[NB + 4 * J + c], x, g[c]); }
      ldb_mn(bi, J, s, g);
      uint32_t y[4];
      sgn<S1>(fi, x);
      sgn<S2>(fr, y);
#pragma unroll
      for (int c = 0; c < 4; ++c) { mma_tf32(acc[4 * J + c], x, g[c]); mma_tf32(acc[NB + 4 * J + c], y, g[c]); }
    }
  }
}

// f(h, col, re[V], im[V]) for every run of V contiguous tile columns this lane holds in tile row frag_row<L>(row0, h): V = 2 in KK (columns
// 8 j + 2 q, + 1), V = 4 in MM / KM (columns 32 J + 8 q + 4 e .. + 3 from fragments 4 J .. 4 J + 3).  im is the imaginary part of a
// complex accumulator (NA = 2 NB) and unused otherwise.
template <Lay L, int NB, int NA, class F>
__device__ __forceinline__ void for_each_run(const float (&acc)[NA][4], F f) {
  const int q = threadIdx.x & 3;
  constexpr int IM = NA == 2 * NB ? NB : 0;
  if constexpr (L == Lay::KK) {
#pragma unroll
    for (int j = 0; j < NB; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float re[2] = {acc[j][2 * h], acc[j][2 * h + 1]}, im[2] = {acc[IM + j][2 * h], acc[IM + j][2 * h + 1]};
        f(h, 8 * j + 2 * q, re, im);
      }
  } else {
#pragma unroll
    for (int J = 0; J < NB / 4; ++J)
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int x = 2 * h + e;
          const float re[4] = {acc[4 * J][x], acc[4 * J + 1][x], acc[4 * J + 2][x], acc[4 * J + 3][x]};
          const float im[4] = {acc[IM + 4 * J][x], acc[IM + 4 * J + 1][x], acc[IM + 4 * J + 2][x], acc[IM + 4 * J + 3][x]};
          f(h, 32 * J + 8 * q + 4 * e, re, im);
        }
  }
}

// ----------------------------------------------------------------------------------------- wait-time profile
// Built with -DB200SHT_UMMA_PROFILE (`python -m makani_b200.build --define B200SHT_UMMA_PROFILE --out libb200sht_umma_prof.so`, driven by
// scripts/umma_waitprof.py): every role sums the SM clocks it spends per state into g_umma_prof, read back and cleared by
// b200sht_debug_umma_profile().  Slots: 0 producer waits for a free stage (empty), 1 consumer warps wait for a loaded stage (full), 2 consumer
// warps in the MMA loop (without the full waits), 3 consumer warps in the epilogue, 4 consumer-warp lifetime, 5 producer lifetime,
// 6 tiles (consumer warps), 7 CTAs.  Consumer slots are sums over the 8 warps of every CTA.  On the wgmma path the MMA loop is the issue
// of the stage's wgmma and the wgmma.wait_group for the stage before.  The shipped build has none of it.
#ifdef B200SHT_UMMA_PROFILE
constexpr bool kUmmaProfile = true;
#else
constexpr bool kUmmaProfile = false;
#endif
__device__ unsigned long long g_umma_prof[16];
__device__ __forceinline__ long long prof_clock() { return kUmmaProfile ? clock64() : 0; }

__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, %0;" ::"n"(32 * kConsumerWarps) : "memory"); }   // warps 0..7 only

// Persistent engine: one CTA per SM loops over tiles.  The operand ring (full/empty) runs continuously across tiles, so the
// TMA producer prefetches the next tile while the consumer warps finish the current one.  NB: 8-column fragments per warp; SPLIT: 3 x TF32.
// Traits with kStaged (the synthesis, not in 3 x TF32) stage the finished tile in shared memory after the ring and bulk-store it from there.
// Traits with kKMajor (both operands K-major) run their TF32 instantiations on wgmma, one warpgroup per 64 rows.
template <class T, int NB, bool SPLIT>
__global__ void __launch_bounds__(kUmmaThreads, 1) umma_kernel(const __grid_constant__ typename T::Params p) {
  constexpr bool kStaged = T::kStaged && !SPLIT;
  constexpr bool kWgmma = T::kKMajor && !SPLIT;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* gbase = smem_raw + (base - raw);
  const int stages = p.stages;
  const uint32_t stage_bytes = p.stage_bytes;
  uint8_t* const out = gbase + (size_t)stages * stage_bytes;   // output staging (p.out_bytes, 1024-byte aligned)
  uint64_t* full = reinterpret_cast<uint64_t*>(out + p.out_bytes);
  uint64_t* empty = full + kMaxStages;
  const long long t_cta0 = prof_clock();

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;   // warp-uniform for the compiler
  pdl_trigger();   // the next kernel of the stream may be scheduled while this one runs (it waits for our completion before touching data)
  if (warp == kProducerWarp && lane == 0) {
    for (int s = 0; s < stages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], kConsumerWarps); }
    fence_barrier_init();
    T::prefetch(p);
  }
  __syncthreads();
  const int ntiles = p.gx * p.gy * p.gz;
  pdl_wait();      // prologue done (barriers, tensor-map prefetch): from here on this kernel reads what its predecessors wrote

  if (warp == kProducerWarp) {
    if (lane == 0) {
      unsigned long long w_empty = 0;
      int kbg = 0;   // k-block counter across tiles: position in the operand ring
      for (int ti = blockIdx.x; ti < ntiles; ti += gridDim.x) {
        typename T::Tile tile;
        if (!T::make_tile(p, tile, ti % p.gx, (ti / p.gx) % p.gy, ti / (p.gx * p.gy))) continue;
        const int nk = T::num_kblocks(p, tile);
        for (int kb = 0; kb < nk; ++kb, ++kbg) {
          const int s = kbg % stages, it = kbg / stages;
          if (it > 0) {
            const long long t0 = prof_clock();
            if constexpr (kWgmma) mbar_wait_nocall(&empty[s], (it - 1) & 1);   // no function call anywhere in a wgmma kernel
            else mbar_wait(&empty[s], (it - 1) & 1);
            if constexpr (kUmmaProfile) w_empty += clock64() - t0;
          }
          mbar_expect_tx(&full[s], p.tx_bytes);
          T::load(p, tile, kb, base + s * stage_bytes, &full[s]);
        }
      }
      if constexpr (kUmmaProfile) {
        atomicAdd(&g_umma_prof[0], w_empty);
        atomicAdd(&g_umma_prof[5], (unsigned long long)(clock64() - t_cta0));
        atomicAdd(&g_umma_prof[7], 1ull);
      }
    }
    __syncwarp();
  } else {
    const int row0 = 16 * warp;
    int kbg = 0;
    uint32_t piece = 0;   // staged epilogue: output pieces written so far (position in the double buffer)
    unsigned long long w_full = 0, t_loop = 0, t_epi = 0, n_tiles = 0;
    for (int ti = blockIdx.x; ti < ntiles; ti += gridDim.x) {
      typename T::Tile tile;
      if (!T::make_tile(p, tile, ti % p.gx, (ti / p.gx) % p.gy, ti / (p.gx * p.gy))) continue;
      const long long t0 = prof_clock();
      const int nk = T::num_kblocks(p, tile);   // >= 1 for the kKMajor Traits: their first wgmma (scale-d = 0) initializes acc
      float acc[NB * T::kPlanes][4];
      if constexpr (kWgmma) {
        // one stage's wgmma stay in flight: the stage before is released once wait_group 1 has retired its group
        int prev = 0;
        for (int kb = 0; kb < nk; ++kb, ++kbg) {
          const int s = kbg % stages, it = kbg / stages;
          const long long tw = prof_clock();
          mbar_wait_nocall(&full[s], it & 1);
          if constexpr (kUmmaProfile) w_full += clock64() - tw;
          wgmma_fence();
          T::template wgmma<NB>(p, base + s * stage_bytes, warp >> 2, kb > 0, acc);
          wgmma_commit();
          wgmma_wait<1>();
          if (kb > 0 && lane == 0) mbar_arrive(&empty[prev]);   // this warp's wgmma of the stage before have read it
          prev = s;
        }
        wgmma_wait<0>();
        wgmma_fence_operands(acc);
        if (lane == 0) mbar_arrive(&empty[prev]);
      } else {
#pragma unroll
        for (int j = 0; j < NB * T::kPlanes; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
        for (int kb = 0; kb < nk; ++kb, ++kbg) {
          const int s = kbg % stages, it = kbg / stages;
          const long long tw = prof_clock();
          mbar_wait(&full[s], it & 1);
          if constexpr (kUmmaProfile) w_full += clock64() - tw;
          T::template mma<NB, SPLIT>(p, gbase + (size_t)s * stage_bytes, row0, acc);
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty[s]);   // this warp's reads of the stage are done
        }
      }
      const long long t1 = prof_clock();
      if constexpr (kStaged) T::template epilogue_staged<NB>(p, tile, row0, acc, out, piece);
      else T::template epilogue<NB>(p, tile, row0, acc);
      if constexpr (kUmmaProfile) { t_loop += t1 - t0; t_epi += clock64() - t1; ++n_tiles; }
    }
    // the bulk stores must be complete (not only have read shared memory) before the CTA exits: a dependent kernel's griddepcontrol.wait
    // relies on grid completion for the visibility of this kernel's output
    if constexpr (kStaged) if (warp == 0) bulk_wait0();
    if constexpr (kUmmaProfile) if (lane == 0) {
      atomicAdd(&g_umma_prof[1], w_full);
      atomicAdd(&g_umma_prof[2], t_loop - w_full);
      atomicAdd(&g_umma_prof[3], t_epi);
      atomicAdd(&g_umma_prof[4], (unsigned long long)(clock64() - t_cta0));
      atomicAdd(&g_umma_prof[6], n_tiles);
    }
  }
}

// ================================================================================================ AnaTraits
struct AnaTraits {
  struct Params : EngineParams {
    alignas(64) CUtensorMap tmA;  // table  (k, l, m)       box (32, 128, 1)
    alignas(64) CUtensorMap tmB;  // X      (k, c, pb, m)   box (32, Cc, PBc, 1)
    alignas(64) CUtensorMap tmA_lo, tmB_lo;   // residuals of the table and of X (split mode)
    float* spec;
    int L, M, nlat, C, cp, PB, Cc, PBc, n_ct, N, m0;
    int nkb;             // 32-row K-blocks over the latitudes
  };
  static constexpr int kPlanes = 1;
  static constexpr bool kStaged = false;   // register epilogue
  static constexpr bool kKMajor = true;    // TF32 on wgmma
  struct Tile { int m, l0, c0, pb0; };
  __device__ static bool make_tile(const Params& p, Tile& t, int bx, int by, int bz) {
    t.m = bz;
    t.l0 = lstart(p.m0 + t.m) + 128 * bx;
    t.c0 = (by % p.n_ct) * p.Cc;
    t.pb0 = (by / p.n_ct) * p.PBc;
    return t.l0 < p.L;
  }
  __device__ static void prefetch(const Params& p) { prefetch_tmap(&p.tmA); prefetch_tmap(&p.tmB); }
  __device__ static int num_kblocks(const Params& p, const Tile&) { return p.nkb; }
  __device__ static void load(const Params& p, const Tile& t, int kb, uint32_t st, uint64_t* bar) {
    tma_load_3d(st, &p.tmA, bar, kb * 32, t.l0, t.m);
    tma_load_4d(st + 16384, &p.tmB, bar, kb * 32, t.c0, t.pb0, t.m);
    if (p.split) {
      tma_load_3d(st + p.lo_off, &p.tmA_lo, bar, kb * 32, t.l0, t.m);
      tma_load_4d(st + p.lo_off + 16384, &p.tmB_lo, bar, kb * 32, t.c0, t.pb0, t.m);
    }
  }
  template <int NB, bool SPLIT>   // 3 x TF32 only
  __device__ __forceinline__ static void mma(const Params& p, const uint8_t* st, int row0, float (&acc)[NB][4]) {
    gemm_real<Lay::KK, NB, SPLIT>(st, st + 16384, p.lo_off, row0, acc);
  }
  // warpgroup wg: rows 64 wg .. + 63 of the table tile (at st) against the N rows of X (at st + 16384); acc_on = 0: first stage of the tile
  template <int NB>
  __device__ __forceinline__ static void wgmma(const Params&, uint32_t st, int wg, bool acc_on, float (&acc)[NB][4]) {
    const uint64_t da = wgmma_desc_kmajor(st + 8192 * wg), db = wgmma_desc_kmajor(st + 16384);
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_tf32<8 * NB, 1, NB, 0>(acc, da + 2 * k, db + 2 * k, (k > 0 || acc_on) ? 1 : 0);
  }
  // column n = pbi * Cc + ci of the tile; Cc and cp are multiples of 4, so the column pair (n, n + 1) of a run is one float2 of spec
  template <int NB>
  __device__ __forceinline__ static void epilogue(const Params& p, const Tile& t, int row0, const float (&acc)[NB][4]) {
    const int ncols = p.Cc * p.PBc;
    const size_t JP = (size_t)p.PB * p.cp;
    const int l0 = t.l0 + frag_row<Lay::KK>(row0, 0);
    for_each_run<Lay::KK, NB>(acc, [&](int h, int n, const float (&v)[2], const float (&)[2]) {
      const int l = l0 + 8 * h;
      if (l >= p.L || n >= ncols) return;
      const int pbi = n / p.Cc, ci = n - pbi * p.Cc;
      const int pb = t.pb0 + pbi, c = t.c0 + ci;
      if (pb >= p.PB || c >= p.cp) return;
      float2* dst = reinterpret_cast<float2*>(p.spec + ((size_t)l * p.M + t.m) * JP + (size_t)pb * p.cp + c);
      float2 o = make_float2(v[0], v[1]);
      // strict fp32 (split) stays as accumulated; otherwise the consumers are TF32 MMAs: round to nearest here
      if (!p.split) { o.x = tf32_rn(o.x); o.y = tf32_rn(o.y); }
      *dst = o;
    });
  }
};

// ================================================================================================ SynTraits
struct SynTraits {
  struct Params : EngineParams {
    alignas(64) CUtensorMap tmA;  // table (k, l, m)   box (32, 32, 1)   MN-major A (M = k)
    alignas(64) CUtensorMap tmB;  // spec  (n, m, l)   box (32, 1, 32)   MN-major B (N = n)
    alignas(64) CUtensorMap tmA_lo, tmB_lo;   // residuals of the table and of spec (split mode)
    alignas(64) CUtensorMap tmZ;  // Z, bulk stores (k % 8, c, k / 8, pb, m) or tiled (k % 8, c, k / 8, plane 8 M2 + m, b)   box (8, 4, 16, 1, 1)
    float* Z;
    int L, M, nlat, kp, C, cp, PB, nblk, N, m0;
    int tiled, M2, KT, B;   // tiled output for the tensor-core DFT (dft.cu): Z[r][k / 8][p][m / 8][m % 8][k % 8], orders padded to 8 * M2
  };
  static constexpr int kPlanes = 1;
  // Bulk-store epilogue (TF32; the 3 x TF32 instantiations keep the register epilogue below: their doubled stages leave no room for it).
  // The output of a tile is staged as boxes of 4 columns x 128 latitudes, 2 KB each, laid out [k / 8][column][k % 8] -- the order of the
  // store map's box (8, 4, 16), which is the same in both layouts of Z.  Tiles of at most 20 fragments (160 columns) stage the whole
  // tile at once; wider ones stage 32 columns at a time in two alternating 16 KB buffers.
  static constexpr bool kStaged = true;
  static constexpr bool kKMajor = false;   // MN-major operands: mma.sync
  __host__ __device__ static constexpr uint32_t out_bytes(int nb) { return nb <= 20 ? 4096u * nb : 2u * 16384u; }
  struct Tile { int m, k0, n0, lbeg; };
  __device__ static bool make_tile(const Params& p, Tile& t, int bx, int by, int bz) {
    t.m = bz;
    t.k0 = 128 * bx;
    t.n0 = p.N * by;
    t.lbeg = lstart(p.m0 + t.m);
    return true;
  }
  __device__ static void prefetch(const Params& p) { prefetch_tmap(&p.tmA); prefetch_tmap(&p.tmB); }
  // orders m >= M exist only in the tiled layout (padding up to a multiple of 8): no degree contributes, the tile is written as zeros
  __device__ static int num_kblocks(const Params& p, const Tile& t) { return (t.m < p.M && t.lbeg < p.L) ? (p.L - t.lbeg + 31) / 32 : 0; }
  __device__ static void load(const Params& p, const Tile& t, int kb, uint32_t st, uint64_t* bar) {
    const int l = t.lbeg + kb * 32;
#pragma unroll
    for (int b = 0; b < 4; ++b) tma_load_3d(st + b * 4096, &p.tmA, bar, t.k0 + 32 * b, l, t.m);
    for (int b = 0; b < p.nblk; ++b) tma_load_3d(st + 16384 + b * 4096, &p.tmB, bar, t.n0 + 32 * b, t.m, l);
    if (p.split) {
#pragma unroll
      for (int b = 0; b < 4; ++b) tma_load_3d(st + p.lo_off + b * 4096, &p.tmA_lo, bar, t.k0 + 32 * b, l, t.m);
      for (int b = 0; b < p.nblk; ++b) tma_load_3d(st + p.lo_off + 16384 + b * 4096, &p.tmB_lo, bar, t.n0 + 32 * b, t.m, l);
    }
  }
  template <int NB, bool SPLIT>
  __device__ __forceinline__ static void mma(const Params& p, const uint8_t* st, int row0, float (&acc)[NB][4]) {
    gemm_real<Lay::MM, NB, SPLIT>(st, st + 16384, p.lo_off, row0, acc);
  }
  // column jp = pb * cp + c of the tile -> row (pb, c) of this order's slab of Z; orders without a contributing degree hold zero accumulators
  // In the MM layout a lane holds the latitude pair k, k + 1 (k even) of columns 32 J + 8 q + 4 e .. + 3: one 8-byte store per column in
  // both layouts of Z (k is the contiguous index of the standard layout and k % 8 that of the tiled one).  The column is decoded once per run.
  template <int NB>
  __device__ __forceinline__ static void epilogue(const Params& p, const Tile& t, int row0, const float (&acc)[NB][4]) {
    const int JP = p.PB * p.cp;
    const int k = t.k0 + frag_row<Lay::MM>(row0, 0);
    if (k >= p.kp) return;
    const bool pair = k + 1 < p.kp;
    const int q = threadIdx.x & 3;
#pragma unroll
    for (int J = 0; J < NB / 4; ++J)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int jp0 = t.n0 + 32 * J + 8 * q + 4 * e;
        int pb = jp0 / p.cp, c = jp0 - pb * p.cp;
#pragma unroll
        for (int i = 0; i < 4; ++i, ++c) {
          if (c == p.cp) { c = 0; ++pb; }
          if (jp0 + i >= JP) break;
          if (c >= p.C) continue;
          const float v0 = acc[4 * J + i][e], v1 = acc[4 * J + i][2 + e];
          float* dst;
          if (!p.tiled) {
            dst = p.Z + (size_t)t.m * p.PB * p.C * p.kp + (size_t)(pb * p.C + c) * p.kp + k;
          } else {   // pb = plane * B + b, image r = b * C + c:  Z[r][kt][plane][m2][c8][k8]
            const int pl = pb / p.B, b = pb - pl * p.B;
            const int o = (((b * p.C + c) * p.KT) * 2 + pl) * p.M2 * 64;
            dst = p.Z + (size_t)(k >> 3) * 2 * p.M2 * 64 + (t.m >> 3) * 64 + (t.m & 7) * 8 + (k & 7) + o;
          }
          if (pair) *reinterpret_cast<float2*>(dst) = make_float2(v0, v1);
          else *dst = v0;
        }
      }
  }

  // Columns 32 J .. + 31 of the warp's 16 rows into the 8 boxes at `buf`.  The lane holds latitudes k, k + 1 (k = row0 + 2 g) of columns
  // 32 J + 8 q + 4 e + c (c = 0..3): box 8 J + 2 q + e, column c, one 8-byte store at [k / 8][c][k % 8].  Lane q writes column c = i ^ q
  // in step i, so that the 16 lanes of a half-warp (g = 0..3 or 4..7: one k / 8) cover 16 different 8-byte bank slots.
  template <int NB>
  __device__ __forceinline__ static void stage_cols(const float (&acc)[NB][4], int J, int row0, uint8_t* buf) {
    const int lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
    const int k = row0 + 2 * g;
    uint8_t* const b0 = buf + (k >> 3) * 128 + (k & 7) * 4 + q * 4096;
#pragma unroll
    for (int e = 0; e < 2; ++e)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int c = i ^ q;
        const float v0 = c == 0 ? acc[4 * J][e] : c == 1 ? acc[4 * J + 1][e] : c == 2 ? acc[4 * J + 2][e] : acc[4 * J + 3][e];
        const float v1 = c == 0 ? acc[4 * J][2 + e] : c == 1 ? acc[4 * J + 1][2 + e] : c == 2 ? acc[4 * J + 2][2 + e] : acc[4 * J + 3][2 + e];
        *reinterpret_cast<float2*>(b0 + e * 2048 + c * 32) = make_float2(v0, v1);
      }
  }
  // Warp 0: bulk stores of the tile's boxes bt0 .. bt0 + nbx - 1 (staged 2 KB apart from `buf`), a few per lane, one bulk group per lane.
  // Boxes of columns past the tile's last one or of channel padding (c0 >= C) are skipped; the map's extents clip the rest: channels at C,
  // latitudes at kp.  Latitude padding rows (nlat <= k < kp) and orders without degrees hold zero accumulators and are stored as zeros.
  __device__ static void store_boxes(const Params& p, const Tile& t, int bt0, int nbx, uint32_t buf) {
    for (int b = threadIdx.x & 31; b < nbx; b += 32) {
      const int jp = t.n0 + 4 * (bt0 + b);
      const int pb = jp / p.cp, c0 = jp - pb * p.cp;
      if (pb >= p.PB || c0 >= p.C) continue;
      if (!p.tiled) {
        tma_store_5d(&p.tmZ, buf + b * 2048, 0, c0, t.k0 >> 3, pb, t.m);
      } else {   // pb = plane * B + b
        const int pl = pb / p.B;
        tma_store_5d(&p.tmZ, buf + b * 2048, 0, c0, t.k0 >> 3, pl * 8 * p.M2 + t.m, pb - pl * p.B);
      }
    }
    bulk_commit();
  }
  // All 8 consumer warps: wait until the buffer's previous stores have read it, stage, make the writes visible to the async proxy, and let
  // warp 0 issue the stores.  Nobody waits for the stores themselves: the consumers go on to the next tile's MMAs.
  template <int NB>
  __device__ __forceinline__ static void epilogue_staged(const Params& p, const Tile& t, int row0, const float (&acc)[NB][4], uint8_t* out,
                                                         uint32_t& piece) {
    const bool issuer = (threadIdx.x >> 5) == 0;
    if constexpr (NB <= 20) {
      if (issuer) bulk_wait_read<0>();
      consumer_sync();
#pragma unroll
      for (int J = 0; J < NB / 4; ++J) stage_cols<NB>(acc, J, row0, out + J * 16384);
      fence_proxy_async();
      consumer_sync();
      if (issuer) store_boxes(p, t, 0, 2 * NB, smem_u32(out));
    } else {
#pragma unroll
      for (int J = 0; J < NB / 4; ++J, ++piece) {
        uint8_t* const buf = out + (piece & 1) * 16384;
        if (issuer) bulk_wait_read<1>();   // the stores of the piece before last, which used this buffer
        consumer_sync();
        stage_cols<NB>(acc, J, row0, buf);
        fence_proxy_async();
        consumer_sync();
        if (issuer) store_boxes(p, t, 8 * J, 8, smem_u32(buf));
      }
    }
  }
};

// ====================================================================================================== mix
// spec tensor map: dims (c, b, p, m, l) with strides (1, cp, B*cp, 2*B*cp, M*2*B*cp) floats.
// weight tensor map (planar packed weight [Lw][G][Cig][2][cop]): dims (o, p, i, lg) strides (1, cop, 2*cop, Cig*2*cop).
struct MixParams : EngineParams {
  alignas(64) CUtensorMap tmX;   // operand read as rows (m, b)
  alignas(64) CUtensorMap tmX2;  // second spec operand (wgrad: gy)
  alignas(64) CUtensorMap tmW;
  float* out;              // spec (fwd / dgrad) or packed weight gradient (wgrad)
  const float2* cbias;
  int L, M, B, G, Cig, Cog, cpi, cpo, cop;
  int Mt;                  // m values per row tile (Mt * B <= 128 rows)
  int nblk, N;             // N = output columns per tile (<= 128); nblk = N / 32 (MN-major B operands)
  int n_nt;                // output tiles per group
  int shared_w;            // weight has no l dimension
  int dense;               // spec tensors store every (l, m) entry
  long long wl_stride;
  uint32_t offA_i, offB_r, offB_i;  // stage offsets of the imaginary A tile and the two B tiles (A_r at 0)
};

template <int V>
__device__ __forceinline__ void st_vec(float* dst, const float (&v)[V]) {   // dst 4 V-byte aligned
  if constexpr (V == 4) *reinterpret_cast<float4*>(dst) = make_float4(v[0], v[1], v[2], v[3]);
  else *reinterpret_cast<float2*>(dst) = make_float2(v[0], v[1]);
}

struct MixFwdTraits {
  using Params = MixParams;
  static constexpr int kPlanes = 2;
  static constexpr bool kStaged = false;   // register epilogue
  static constexpr bool kKMajor = false;   // MN-major B: mma.sync
  struct Tile { int l, m0, g, o0, lg; };
  __device__ static bool make_tile(const Params& p, Tile& t, int bx, int by, int bz) {
    t.l = bz;
    t.m0 = bx * p.Mt;
    t.g = by / p.n_nt;
    t.o0 = (by % p.n_nt) * p.N;
    t.lg = (p.shared_w ? 0 : t.l * p.G) + t.g;
    return t.m0 < mend_d(t.l, p.M, p.dense);
  }
  __device__ static void prefetch(const Params& p) { prefetch_tmap(&p.tmX); prefetch_tmap(&p.tmW); }
  __device__ static int num_kblocks(const Params& p, const Tile&) { return (p.Cig + 31) / 32; }
  __device__ static void load(const Params& p, const Tile& t, int kb, uint32_t st, uint64_t* bar) {
    const int c = t.g * p.Cig + kb * 32;
    tma_load_5d(st, &p.tmX, bar, c, 0, 0, t.m0, t.l);
    tma_load_5d(st + p.offA_i, &p.tmX, bar, c, 0, 1, t.m0, t.l);
    for (int b = 0; b < p.nblk; ++b) {
      tma_load_4d(st + p.offB_r + b * 4096, &p.tmW, bar, t.o0 + 32 * b, 0, kb * 32, t.lg);
      tma_load_4d(st + p.offB_i + b * 4096, &p.tmW, bar, t.o0 + 32 * b, 1, kb * 32, t.lg);
    }
  }
  // yr = xr wr - xi wi,  yi = xr wi + xi wr
  template <int NB, bool>
  __device__ __forceinline__ static void mma(const Params& p, const uint8_t* st, int row0, float (&acc)[2 * NB][4]) {
    gemm_cplx<Lay::KM, NB, -1, 1, 1>(st, st + p.offA_i, st + p.offB_r, st + p.offB_i, row0, acc);
  }
  // rows (mi, b) -> spec rows; columns -> output channels of group g; handles cbias and the zero channel padding.  A run of 2 or 4 columns
  // never straddles `limit` (cp_out, and NOg when G > 1, are multiples of 4; o0 of 16 or 32), so it is stored as one vector.
  template <Lay L, int NB>
  __device__ __forceinline__ static void store_rows(const Params& p, int l, int m0, int g, int o0, int NOg, int cp_out, int row0,
                                                    const float (&acc)[2 * NB][4], bool with_bias) {
    const int pad = cp_out - NOg * p.G;
    const int limit = NOg + ((g == p.G - 1) ? pad : 0);  // columns of this group incl. trailing zero padding
    const int mend = mend_d(l, p.M, p.dense);
    float* yrow[2];
    bool ok[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = frag_row<L>(row0, h), mi = r / p.B, b = r - mi * p.B, m = m0 + mi;
      ok[h] = r < p.Mt * p.B && m < mend;
      yrow[h] = p.out + ((size_t)l * p.M + m) * 2 * p.B * cp_out + (size_t)b * cp_out + g * NOg;
    }
    for_each_run<L, NB>(acc, [&](int h, int n, const auto& re, const auto& im) {
      constexpr int V = sizeof(re) / sizeof(float);
      const int o = o0 + n;
      if (!ok[h] || o >= limit) return;
      float a[V], c[V];
#pragma unroll
      for (int v = 0; v < V; ++v) {
        a[v] = re[v]; c[v] = im[v];
        if (o + v >= NOg) { a[v] = 0.f; c[v] = 0.f; }
        else if (with_bias) { const float2 cb = p.cbias[g * NOg + o + v]; a[v] += cb.x; c[v] += cb.y; }
        a[v] = tf32_rn(a[v]); c[v] = tf32_rn(c[v]);
      }
      st_vec<V>(yrow[h] + o, a);
      st_vec<V>(yrow[h] + o + (size_t)p.B * cp_out, c);
    });
  }
  template <int NB>
  __device__ __forceinline__ static void epilogue(const Params& p, const Tile& t, int row0, const float (&acc)[2 * NB][4]) {
    store_rows<Lay::KM, NB>(p, t.l, t.m0, t.g, t.o0, p.Cog, p.cpo, row0, acc, p.cbias != nullptr);
  }
};

struct MixDgradTraits {
  using Params = MixParams;   // tmX = gy (channels = Cout), out = gx; N tiles over i
  using Tile = MixFwdTraits::Tile;  // o0 is the first input channel i0 of the tile
  static constexpr int kPlanes = 2;
  static constexpr bool kStaged = false;   // register epilogue
  static constexpr bool kKMajor = true;    // wgmma
  __device__ static bool make_tile(const Params& p, Tile& t, int bx, int by, int bz) { return MixFwdTraits::make_tile(p, t, bx, by, bz); }
  __device__ static void prefetch(const Params& p) { prefetch_tmap(&p.tmX); prefetch_tmap(&p.tmW); }
  __device__ static int num_kblocks(const Params& p, const Tile&) { return (p.Cog + 31) / 32; }
  __device__ static void load(const Params& p, const Tile& t, int kb, uint32_t st, uint64_t* bar) {
    const int c = t.g * p.Cog + kb * 32;
    tma_load_5d(st, &p.tmX, bar, c, 0, 0, t.m0, t.l);
    tma_load_5d(st + p.offA_i, &p.tmX, bar, c, 0, 1, t.m0, t.l);
    tma_load_4d(st + p.offB_r, &p.tmW, bar, kb * 32, 0, t.o0, t.lg);   // box (32 o, 1, N i, 1): K-major rows i
    tma_load_4d(st + p.offB_i, &p.tmW, bar, kb * 32, 1, t.o0, t.lg);
  }
  // gxr = gr wr + gi wi,  gxi = gi wr - gr wi: four real wgmma per k8 step, the negated one through the instruction's B scale.  Warpgroup
  // wg: rows 64 wg .. + 63 of both gy planes; acc_on = 0: first stage of the tile
  template <int NB>
  __device__ __forceinline__ static void wgmma(const Params& p, uint32_t st, int wg, bool acc_on, float (&acc)[2 * NB][4]) {
    const uint64_t ar = wgmma_desc_kmajor(st + 8192 * wg), ai = wgmma_desc_kmajor(st + p.offA_i + 8192 * wg);
    const uint64_t br = wgmma_desc_kmajor(st + p.offB_r), bi = wgmma_desc_kmajor(st + p.offB_i);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int sd = (k > 0 || acc_on) ? 1 : 0;
      wgmma_tf32<8 * NB, 1, 2 * NB, 0>(acc, ar + 2 * k, br + 2 * k, sd);
      wgmma_tf32<8 * NB, 1, 2 * NB, NB>(acc, ai + 2 * k, br + 2 * k, sd);
      wgmma_tf32<8 * NB, 1, 2 * NB, 0>(acc, ai + 2 * k, bi + 2 * k, 1);
      wgmma_tf32<8 * NB, -1, 2 * NB, NB>(acc, ar + 2 * k, bi + 2 * k, 1);
    }
  }
  template <int NB>
  __device__ __forceinline__ static void epilogue(const Params& p, const Tile& t, int row0, const float (&acc)[2 * NB][4]) {
    MixFwdTraits::store_rows<Lay::KK, NB>(p, t.l, t.m0, t.g, t.o0, p.Cig, p.cpi, row0, acc, false);
  }
};

struct MixWgradTraits {
  using Params = MixParams;   // tmX = x (A, rows i), tmX2 = gy (B, cols o); K = spectral rows (m, b)
  static constexpr int kPlanes = 2;
  static constexpr bool kStaged = false;   // register epilogue
  static constexpr bool kKMajor = false;   // MN-major operands: mma.sync
  struct Tile { int lz, i0, g, o0; };
  __device__ static bool make_tile(const Params& p, Tile& t, int bx, int by, int bz) {
    t.lz = bz;
    t.i0 = bx * 128;
    t.g = by / p.n_nt;
    t.o0 = (by % p.n_nt) * p.N;
    return true;
  }
  __device__ static void prefetch(const Params& p) { prefetch_tmap(&p.tmX); prefetch_tmap(&p.tmX2); }
  __device__ static int kb_of_l(const Params& p, int l) { return (mend_d(l, p.M, p.dense) * p.B + 31) / 32; }
  __device__ static int num_kblocks(const Params& p, const Tile& t) {
    if (!p.shared_w) return kb_of_l(p, t.lz);
    int n = 0;
    for (int l = 0; l < p.L; ++l) n += kb_of_l(p, l);
    return n;
  }
  __device__ static void load(const Params& p, const Tile& t, int kb, uint32_t st, uint64_t* bar) {
    int l = t.lz;
    if (p.shared_w) {
      l = 0;
      int n = kb_of_l(p, 0);
      while (kb >= n) { kb -= n; ++l; n = kb_of_l(p, l); }
    }
    const int m = kb * (32 / p.B);
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      tma_load_5d(st + a * 4096, &p.tmX, bar, t.g * p.Cig + t.i0 + 32 * a, 0, 0, m, l);
      tma_load_5d(st + p.offA_i + a * 4096, &p.tmX, bar, t.g * p.Cig + t.i0 + 32 * a, 0, 1, m, l);
    }
    for (int b = 0; b < p.nblk; ++b) {
      tma_load_5d(st + p.offB_r + b * 4096, &p.tmX2, bar, t.g * p.Cog + t.o0 + 32 * b, 0, 0, m, l);
      tma_load_5d(st + p.offB_i + b * 4096, &p.tmX2, bar, t.g * p.Cog + t.o0 + 32 * b, 0, 1, m, l);
    }
  }
  // gwr = xr gr + xi gi,  gwi = xr gi - xi gr
  template <int NB, bool>
  __device__ __forceinline__ static void mma(const Params& p, const uint8_t* st, int row0, float (&acc)[2 * NB][4]) {
    gemm_cplx<Lay::MM, NB, 1, 1, -1>(st, st + p.offA_i, st + p.offB_r, st + p.offB_i, row0, acc);
  }
  // runs of 4 output channels (cop and o0 are multiples of 4): one float4 per run and plane
  template <int NB>
  __device__ __forceinline__ static void epilogue(const Params& p, const Tile& t, int row0, const float (&acc)[2 * NB][4]) {
    float* const out = p.out + (size_t)(p.shared_w ? 0 : t.lz) * p.wl_stride + (size_t)t.g * p.Cig * 2 * p.cop;
    for_each_run<Lay::MM, NB>(acc, [&](int h, int n, const float (&re)[4], const float (&im)[4]) {
      const int i = t.i0 + frag_row<Lay::MM>(row0, h), o = t.o0 + n;
      if (i >= p.Cig || o >= p.cop) return;
      float* row = out + (size_t)i * 2 * p.cop;
      float a[4], c[4];
#pragma unroll
      for (int v = 0; v < 4; ++v) { a[v] = (o + v < p.Cog) ? re[v] : 0.f; c[v] = (o + v < p.Cog) ? im[v] : 0.f; }
      st_vec<4>(row + o, a);
      st_vec<4>(row + p.cop + o, c);
    });
  }
};

// ================================================================================================== host side
// per device (a process may hold tensors on several GPUs): -1 unknown, 0 / 1
constexpr int kMaxDevices = 64;
static int g_umma_ok[kMaxDevices];
static int g_sm_count[kMaxDevices];
static std::once_flag g_dev_once;
static void init_dev_caches() { for (int i = 0; i < kMaxDevices; ++i) { g_umma_ok[i] = -1; g_sm_count[i] = 0; } }
int umma_available() {
  std::call_once(g_dev_once, init_dev_caches);
  int dev = 0, major = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 0;
  if (dev >= 0 && dev < kMaxDevices && g_umma_ok[dev] >= 0) return g_umma_ok[dev];
  if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess) return 0;
  const int ok = (major == 9 && get_encode() != nullptr) ? 1 : 0;   // the library is built for sm_90a only
  if (dev >= 0 && dev < kMaxDevices) g_umma_ok[dev] = ok;
  return ok;
}

int round_table_tf32(const float* src, float* dst, size_t n, cudaStream_t st);  // legendre.cu

int umma_plan_init(Plan* pl) {
  pl->umma_state = nullptr;
  pl->d_table_tf32 = nullptr;
  pl->d_table_lo = nullptr;
  if (!umma_available()) return -1;
  const size_t n = (size_t)pl->mmax * pl->lmax * pl->kp;
  if (cudaMalloc(&pl->d_table_tf32, n * sizeof(float)) != cudaSuccess) { pl->d_table_tf32 = nullptr; return -1; }
  if (round_table_tf32(pl->d_table, pl->d_table_tf32, n, 0) != 0 || cudaStreamSynchronize(0) != cudaSuccess) {
    cudaFree(pl->d_table_tf32);
    pl->d_table_tf32 = nullptr;
    return -1;
  }
  return 0;
}
void umma_plan_destroy(Plan* pl) {
  if (pl->d_table_tf32) cudaFree(pl->d_table_tf32);
  pl->d_table_tf32 = nullptr;
  if (pl->d_table_lo) cudaFree(pl->d_table_lo);
  pl->d_table_lo = nullptr;
}

int table_residual(const float* full, const float* hi, float* lo, size_t n, cudaStream_t st);  // legendre.cu
// residual table of the 3 x TF32 mode: built the first time a strict-fp32 Legendre stage runs on the tensor cores (most plans never need it)
int umma_plan_table_lo(const Plan* cpl) {
  static std::mutex mu;
  std::lock_guard<std::mutex> lock(mu);
  Plan* pl = const_cast<Plan*>(cpl);
  if (pl->d_table_lo) return 0;
  B200_REQUIRE(pl->d_table && pl->d_table_tf32, "3 x TF32: the plan has no Legendre table");
  const size_t n = (size_t)pl->mmax * pl->lmax * pl->kp;
  float* lo = nullptr;
  B200_CHECK_CUDA(cudaMalloc(&lo, n * sizeof(float)));
  int rc = table_residual(pl->d_table, pl->d_table_tf32, lo, n, 0);
  if (!rc && cudaStreamSynchronize(0) != cudaSuccess) rc = B200SHT_ERR_CUDA;
  if (rc) { cudaFree(lo); return rc; }
  pl->d_table_lo = lo;
  return 0;
}

constexpr size_t kSmemOptIn = 232448;                         // 227 KB: the most a CTA may use on an H100
constexpr size_t kSmemFixed = 1024 /*align*/ + 2 * kMaxStages * 8;
constexpr size_t kSmemMax = kSmemOptIn - 4096;  // ring-only kernels: 227 KB minus barriers / alignment slack

// out_bytes: output staging of the bulk-store epilogue; its ring gets exactly what is left of the 227 KB
static void pick_stages(EngineParams* e, uint32_t stage_bytes, int /*k-blocks per tile: the ring runs across tiles*/, uint32_t out_bytes = 0) {
  e->stage_bytes = stage_bytes;
  e->out_bytes = out_bytes;
  int s = (int)((out_bytes ? kSmemOptIn - kSmemFixed - out_bytes : kSmemMax) / stage_bytes);   // persistent: one CTA per SM owns it all
  if (s > kMaxStages) s = kMaxStages;
  if (s < 2) s = 2;
  e->stages = s;
}
static size_t smem_bytes(const EngineParams& e) { return (size_t)e.stages * e.stage_bytes + e.out_bytes + kSmemFixed; }

static int sm_count() {   // of the current device (the launch device: _lib.call makes the tensor's device current)
  std::call_once(g_dev_once, init_dev_caches);
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 132;
  if (dev >= 0 && dev < kMaxDevices && g_sm_count[dev] > 0) return g_sm_count[dev];
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
  if (dev >= 0 && dev < kMaxDevices) g_sm_count[dev] = n;
  return n;
}

template <class T, int NB, bool SPLIT>
struct KernelTag {};   // one shared-memory grant per instantiation
template <class T, int NB, bool SPLIT>
static int launch(typename T::Params& p, dim3 grid, cudaStream_t st) {
  p.gx = (int)grid.x; p.gy = (int)grid.y; p.gz = (int)grid.z;
  const long long ntiles = (long long)grid.x * grid.y * grid.z;
  if (ntiles <= 0) return 0;
  const size_t smem = smem_bytes(p);
  if (smem > 232448) { set_error("umma: %zu bytes of shared memory needed", smem); return B200SHT_ERR_UNSUPPORTED; }
  B200_CHECK_CUDA((ensure_dynamic_smem<KernelTag<T, NB, SPLIT>>(umma_kernel<T, NB, SPLIT>, smem)));
  // static round-robin over tiles: an odd CTA count not divisible by 3 keeps tile-grid periods (2 l- or m-tiles, 3 or 6 n/k-tiles)
  // from locking heavy tiles onto the same CTAs
  const int sms = usable_sms(sm_count());
  int ctas = (int)(ntiles < sms ? ntiles : sms);
  while (ctas > 1 && (ctas % 2 == 0 || ctas % 3 == 0)) --ctas;
  B200_CHECK_CUDA(launch_pdl(umma_kernel<T, NB, SPLIT>, dim3(ctas), dim3(kUmmaThreads), smem, st, p));
  B200_CHECK_LAUNCH();
  return 0;
}

// The tile widths (8-column fragments per warp) an engine is built for.  The host pads a tile's columns up to the next built width; the
// set is small because every width is a separate kernel (code size, build time).  Legendre: 20 fragments are the 152 + 8 columns of
// C = 73, B = 1, and 32 the 256 of C = 384; mix (complex, 2 NB accumulator fragments): up to 128 columns.
template <int... W>
struct Widths {
  static int pick(int nb) {
    for (int w : {W...})
      if (nb <= w) return w;
    return -1;
  }
  template <class T, bool SPLIT>
  static int launch_nb(typename T::Params& p, int nb, dim3 grid, cudaStream_t st) {
    int rc = B200SHT_ERR_UNSUPPORTED;
    const bool found = ((nb == W ? (rc = launch<T, W, SPLIT>(p, grid, st), true) : false) || ...);
    if (!found) set_error("umma: no engine built for %d fragments per warp", nb);
    return rc;
  }
};
using LegendreWidths = Widths<4, 8, 12, 16, 20, 24, 32>;
using SplitWidths = Widths<8, 16>;   // 3 x TF32 (precision fp32x3): residual fragments too, so tiles of at most 128 columns
using MixWidths = Widths<4, 8, 12>;  // complex: 2 x 96 accumulator columns

// ---------------------------------------------------------------------------------------------- Legendre
int legendre_analysis_umma(const Plan* pl, const float* X, float* spec, int B, int C, cudaStream_t st, const float* X_lo) {
  AnaTraits::Params p;
  memset(&p, 0, sizeof(p));
  p.nkb = ceil_div(pl->nlat, 32);
  const int cp = round_up(C, 4), PB = 2 * B;
  p.spec = spec; p.L = pl->lmax; p.M = pl->mmax; p.nlat = pl->nlat; p.C = C; p.cp = cp; p.PB = PB; p.m0 = pl->m0;
  const int maxc = X_lo ? 128 : 256;   // columns per tile (SplitWidths / LegendreWidths)
  if (cp <= 128) { p.Cc = cp; p.n_ct = 1; p.PBc = maxc / cp < PB ? maxc / cp : PB; }
  else { p.n_ct = ceil_div(cp, 128); p.Cc = round_up(ceil_div(cp, p.n_ct), 4); p.PBc = (2 * p.Cc <= maxc && PB >= 2) ? 2 : 1; }
  const int rows = p.Cc * p.PBc;
  const int nb = (X_lo ? SplitWidths::pick(ceil_div(rows, 8)) : LegendreWidths::pick(ceil_div(rows, 8)));
  B200_REQUIRE(nb > 0, "legendre_analysis: %d columns per tile", rows);
  p.N = 8 * nb;
  {
    long long d[3] = {pl->nlat, pl->lmax, pl->mmax}, s[3] = {1, pl->kp, (long long)pl->lmax * pl->kp};
    int bx[3] = {32, 128, 1};
    int rc = make_tmap(&p.tmA, pl->d_table_tf32, 3, d, s, bx);
    if (rc) return rc;
  }
  {
    long long d[4] = {pl->nlat, C, PB, pl->mmax}, s[4] = {1, pl->kp, (long long)C * pl->kp, (long long)PB * C * pl->kp};
    int bx[4] = {32, p.Cc, p.PBc, 1};
    int rc = make_tmap(&p.tmB, X, 4, d, s, bx);
    if (rc) return rc;
  }
  const uint32_t bbytes = (uint32_t)round_up(p.N * 128, 1024);
  p.split = X_lo != nullptr;
  if (p.split) {
    B200_REQUIRE(pl->d_table_lo != nullptr, "legendre_analysis (3 x TF32): the residual table is missing");
    long long d[3] = {pl->nlat, pl->lmax, pl->mmax}, s[3] = {1, pl->kp, (long long)pl->lmax * pl->kp};
    int bx[3] = {32, 128, 1};
    int rc = make_tmap(&p.tmA_lo, pl->d_table_lo, 3, d, s, bx);
    long long d4[4] = {pl->nlat, C, PB, pl->mmax}, s4[4] = {1, pl->kp, (long long)C * pl->kp, (long long)PB * C * pl->kp};
    int bx4[4] = {32, p.Cc, p.PBc, 1};
    if (!rc) rc = make_tmap(&p.tmB_lo, X_lo, 4, d4, s4, bx4);
    if (rc) return rc;
    p.lo_off = 16384 + bbytes;
  }
  pick_stages(&p, (16384 + bbytes) * (p.split ? 2 : 1), ceil_div(pl->nlat, 32));
  p.tx_bytes = (16384 + (uint32_t)rows * 128) * (p.split ? 2 : 1);
  dim3 grid(ceil_div(pl->lmax, 128), p.n_ct * ceil_div(PB, p.PBc), pl->mmax);
  return p.split ? SplitWidths::launch_nb<AnaTraits, true>(p, nb, grid, st) : LegendreWidths::launch_nb<AnaTraits, false>(p, nb, grid, st);
}

int legendre_synthesis_umma(const Plan* pl, const float* spec, float* Z, int B, int C, int tiled, cudaStream_t st, const float* spec_lo) {
  SynTraits::Params p;
  memset(&p, 0, sizeof(p));
  const int cp = round_up(C, 4), PB = 2 * B, JP = PB * cp;
  p.Z = Z; p.L = pl->lmax; p.M = pl->mmax; p.nlat = pl->nlat; p.kp = pl->kp; p.C = C; p.cp = cp; p.PB = PB; p.m0 = pl->m0;
  p.tiled = tiled; p.M2 = (pl->mmax + 7) / 8; p.KT = pl->kp / 8; p.B = B;
  B200_REQUIRE(!tiled || (long long)B * C * p.KT * 2 * p.M2 * 64 < (1ll << 31), "legendre_synthesis: tiled latspec of %d images exceeds 2^31 floats", B * C);
  const int maxblk = spec_lo ? 4 : 8;   // column blocks of 32 per tile (SplitWidths / LegendreWidths)
  const int nb = (spec_lo ? SplitWidths::pick : LegendreWidths::pick)(4 * (ceil_div(JP, 32) < maxblk ? ceil_div(JP, 32) : maxblk));
  p.nblk = nb / 4;   // column blocks of 32 loaded per stage; those past JP are zero-filled by TMA and not stored
  p.N = 8 * nb;
  {
    long long d[3] = {pl->nlat, pl->lmax, pl->mmax}, s[3] = {1, pl->kp, (long long)pl->lmax * pl->kp};
    int bx[3] = {32, 32, 1};
    int rc = make_tmap(&p.tmA, pl->d_table_tf32, 3, d, s, bx);
    if (rc) return rc;
  }
  {
    long long d[3] = {JP, pl->mmax, pl->lmax}, s[3] = {1, JP, (long long)pl->mmax * JP};
    int bx[3] = {32, 1, 32};
    int rc = make_tmap(&p.tmB, spec, 3, d, s, bx);
    if (rc) return rc;
  }
  p.split = spec_lo != nullptr;
  if (p.split) {
    B200_REQUIRE(pl->d_table_lo != nullptr, "legendre_synthesis (3 x TF32): the residual table is missing");
    long long d[3] = {pl->nlat, pl->lmax, pl->mmax}, s[3] = {1, pl->kp, (long long)pl->lmax * pl->kp};
    int bx[3] = {32, 32, 1};
    int rc = make_tmap(&p.tmA_lo, pl->d_table_lo, 3, d, s, bx);
    long long d2[3] = {JP, pl->mmax, pl->lmax}, s2[3] = {1, JP, (long long)pl->mmax * JP};
    int bx2[3] = {32, 1, 32};
    if (!rc) rc = make_tmap(&p.tmB_lo, spec_lo, 3, d2, s2, bx2);
    if (rc) return rc;
    p.lo_off = 16384 + 4096 * p.nblk;
  }
  uint32_t out_bytes = 0;
  if (!p.split) {   // store map of the bulk-store epilogue: boxes of 8 x 16 latitudes x 4 channels, clipped at channel C and latitude kp
    const long long kp = pl->kp, M2 = p.M2, KT = p.KT;
    long long d[5] = {8, C, KT, PB, pl->mmax}, s[5] = {1, kp, 8, C * kp, PB * C * kp};
    if (tiled) {
      const long long d2[5] = {8, C, KT, 16 * M2, B}, s2[5] = {1, KT * 128 * M2, 128 * M2, 8, C * KT * 128 * M2};
      memcpy(d, d2, sizeof(d)); memcpy(s, s2, sizeof(s));
    }
    int bx[5] = {8, 4, 16, 1, 1};
    int rc = make_tmap(&p.tmZ, Z, 5, d, s, bx, false);
    if (rc) return rc;
    out_bytes = SynTraits::out_bytes(nb);
  }
  pick_stages(&p, (16384 + 4096 * p.nblk) * (p.split ? 2 : 1), ceil_div(pl->lmax, 32), out_bytes);
  p.tx_bytes = (16384 + 4096 * p.nblk) * (p.split ? 2 : 1);
  dim3 grid(ceil_div(pl->kp, 128), ceil_div(JP, p.N), tiled ? 8 * p.M2 : pl->mmax);
  return p.split ? SplitWidths::launch_nb<SynTraits, true>(p, nb, grid, st) : LegendreWidths::launch_nb<SynTraits, false>(p, nb, grid, st);
}

// --------------------------------------------------------------------------------------------------- mix
static int spec_tmap(CUtensorMap* tm, const float* base, int L, int M, int B, int Ctot, int cp, int box_c, int box_b, int box_m) {
  long long d[5] = {Ctot, B, 2, M, L};
  long long s[5] = {1, cp, (long long)B * cp, 2ll * B * cp, (long long)M * 2 * B * cp};
  int bx[5] = {box_c, box_b, 1, box_m, 1};
  return make_tmap(tm, base, 5, d, s, bx);
}
static int weight_tmap(CUtensorMap* tm, const float* base, int Lw, int G, int Cig, int Cog, int cop, int box_o, int box_i) {
  long long d[4] = {Cog, 2, Cig, (long long)Lw * G};
  long long s[4] = {1, cop, 2ll * cop, (long long)Cig * 2 * cop};
  int bx[4] = {box_o, 1, box_i, 1};
  return make_tmap(tm, base, 4, d, s, bx);
}

static int fill_mix(const Plan* pl, int op, int B, int G, int Ci, int Co, MixParams* p) {
  B200_REQUIRE(B >= 1 && 32 % B == 0, "tensor-core mix: batch %d must divide 32 (use precision fp32 otherwise)", B);
  B200_REQUIRE(G == 1 || ((Ci / G) % 4 == 0 && (Co / G) % 4 == 0), "tensor-core mix: group slices (%d, %d channels) must be 16-byte aligned", Ci / G, Co / G);
  memset(p, 0, sizeof(*p));
  p->dense = pl->dense;
  p->L = pl->lmax; p->M = pl->mmax; p->B = B; p->G = G; p->Cig = Ci / G; p->Cog = Co / G;
  p->cpi = round_up(Ci, 4); p->cpo = round_up(Co, 4); p->cop = round_up(Co / G, 4);
  p->shared_w = (op == B200SHT_OP_SHARED);
  p->wl_stride = p->shared_w ? 0 : (long long)G * p->Cig * 2 * p->cop;
  p->Mt = 128 / B;
  return 0;
}

// Column tiling of a mix GEMM: equal tiles of at most 96 columns (no half-empty last tile: at C = 384 a 256 + 128 split wasted a quarter
// of the MMAs), so that the complex accumulator of a tile, 2 N columns, and the fragments of a stage fit the registers of the consumer
// warps without spilling (MixWidths).
static void split_cols(int cols, int gran, int* N, int* n_nt) {
  if (cols <= 96) { *n_nt = 1; *N = round_up(cols, gran); return; }
  *n_nt = ceil_div(cols, 96);
  *N = round_up(ceil_div(cols, *n_nt), 32);   // the epilogues drain 32 columns at a time: a tile must not end inside a chunk
}

int mix_forward_umma(const Plan* pl, int op, const float* x, const void* w, const void* cbias, float* y, int B, int G, int Ci, int Co, cudaStream_t st) {
  MixParams p;
  int rc = fill_mix(pl, op, B, G, Ci, Co, &p);
  if (rc) return rc;
  p.out = y; p.cbias = static_cast<const float2*>(cbias);
  const int cols = p.Cog + ((p.cpo - Co) > 0 ? (p.cpo - Co) : 0);   // last group's tile also writes the zero padding
  split_cols(cols, 32, &p.N, &p.n_nt);
  p.nblk = p.N / 32;
  p.offA_i = 16384; p.offB_r = 32768; p.offB_i = 32768 + 4096 * p.nblk;
  rc = spec_tmap(&p.tmX, x, p.L, p.M, B, Ci, p.cpi, 32, B, p.Mt);
  if (!rc) rc = weight_tmap(&p.tmW, static_cast<const float*>(w), p.shared_w ? 1 : p.L, G, p.Cig, p.Cog, p.cop, 32, 32);
  if (rc) return rc;
  pick_stages(&p, 32768 + 8192 * p.nblk, ceil_div(p.Cig, 32));
  p.tx_bytes = 2u * (uint32_t)(p.Mt * B) * 128 + 8192u * p.nblk;
  dim3 grid(ceil_div(p.M, p.Mt), p.n_nt * G, p.L);
  return MixWidths::launch_nb<MixFwdTraits, false>(p, p.N / 8, grid, st);
}

int mix_backward_umma(const Plan* pl, int op, const float* x, const void* w, const float* gy, float* gx, void* gw, void* gcbias, int B, int G,
                      int Ci, int Co, cudaStream_t st);

int mix_dgrad_umma(const Plan* pl, int op, const void* w, const float* gy, float* gx, int B, int G, int Ci, int Co, cudaStream_t st) {
  MixParams p;
  int rc = fill_mix(pl, op, B, G, Ci, Co, &p);
  if (rc) return rc;
  p.out = gx;
  const int cols = p.Cig + ((p.cpi - Ci) > 0 ? (p.cpi - Ci) : 0);
  split_cols(cols, 16, &p.N, &p.n_nt);
  p.N = 8 * MixWidths::pick(p.N / 8);   // one column tile when the width is padded (n_nt > 1 tiles are multiples of 32)
  const uint32_t bb = (uint32_t)round_up(p.N * 128, 1024);
  p.offA_i = 16384; p.offB_r = 32768; p.offB_i = 32768 + bb;
  rc = spec_tmap(&p.tmX, gy, p.L, p.M, B, Co, p.cpo, 32, B, p.Mt);
  if (!rc) rc = weight_tmap(&p.tmW, static_cast<const float*>(w), p.shared_w ? 1 : p.L, G, p.Cig, p.Cog, p.cop, 32, p.N);
  if (rc) return rc;
  pick_stages(&p, 32768 + 2 * bb, ceil_div(p.Cog, 32));
  p.tx_bytes = 2u * (uint32_t)(p.Mt * B) * 128 + 2u * (uint32_t)p.N * 128;
  dim3 grid(ceil_div(p.M, p.Mt), p.n_nt * G, p.L);
  return MixWidths::launch_nb<MixDgradTraits, false>(p, p.N / 8, grid, st);
}

int mix_wgrad_umma(const Plan* pl, int op, const float* x, const float* gy, float* gw, int B, int G, int Ci, int Co, cudaStream_t st) {
  MixParams p;
  int rc = fill_mix(pl, op, B, G, Ci, Co, &p);
  if (rc) return rc;
  p.out = gw;
  split_cols(p.cop, 32, &p.N, &p.n_nt);
  p.nblk = p.N / 32;
  p.offA_i = 16384; p.offB_r = 32768; p.offB_i = 32768 + 4096 * p.nblk;
  rc = spec_tmap(&p.tmX, x, p.L, p.M, B, Ci, p.cpi, 32, B, 32 / B);
  if (!rc) rc = spec_tmap(&p.tmX2, gy, p.L, p.M, B, Co, p.cpo, 32, B, 32 / B);
  if (rc) return rc;
  pick_stages(&p, 32768 + 8192 * p.nblk, 8);
  p.tx_bytes = 32768u + 8192u * p.nblk;
  dim3 grid(ceil_div(p.Cig, 128), p.n_nt * G, p.shared_w ? 1 : p.L);
  return MixWidths::launch_nb<MixWgradTraits, false>(p, p.N / 8, grid, st);
}

int umma_profile_read(unsigned long long* out16) {   // the wait-time counters of a B200SHT_UMMA_PROFILE build (zeros otherwise); clears them
  B200_CHECK_CUDA(cudaDeviceSynchronize());
  B200_CHECK_CUDA(cudaMemcpyFromSymbol(out16, g_umma_prof, 16 * sizeof(unsigned long long)));
  static const unsigned long long zeros[16] = {};
  B200_CHECK_CUDA(cudaMemcpyToSymbol(g_umma_prof, zeros, sizeof(zeros)));
  return 0;
}

int mix_cbias_grad(const float* gy, void* gcb, int L, int M, int B, int Co, int dense, cudaStream_t st);  // mix.cu

int mix_backward_umma(const Plan* pl, int op, const float* x, const void* w, const float* gy, float* gx, void* gw, void* gcbias, int B, int G,
                      int Ci, int Co, cudaStream_t st) {
  int rc = 0;
  if (gx) rc = mix_dgrad_umma(pl, op, w, gy, gx, B, G, Ci, Co, st);
  if (!rc && gw) rc = mix_wgrad_umma(pl, op, x, gy, static_cast<float*>(gw), B, G, Ci, Co, st);
  if (!rc && gcbias) rc = mix_cbias_grad(gy, gcbias, pl->lmax, pl->mmax, B, Co, pl->dense, st);
  return rc;
}

}  // namespace b200sht
