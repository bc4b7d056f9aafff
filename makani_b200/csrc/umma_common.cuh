// TMA / mbarrier PTX wrappers, TF32 MMA fragments and the tensor-map helper shared by umma.cu (Legendre + mix engine) and dft.cu
// (tensor-core longitude DFT).
#pragma once
#include "common.cuh"
#include <cuda.h>
#include <mutex>
#include <cstring>

namespace b200sht {

// =============================================================================================== PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ uint32_t mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t done;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(done)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return done;
}
// try_wait with a suspend-time hint: the warp sleeps in hardware (no issue slots) until the phase completes or ~`ns` elapse
__device__ __forceinline__ uint32_t mbar_try_wait_hint(uint64_t* bar, uint32_t parity, uint32_t ns) {
  uint32_t done;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(done)
      : "r"(smem_u32(bar)), "r"(parity), "r"(ns)
      : "memory");
  return done;
}
// bounded wait: a lost arrival traps (kernel error) instead of hanging the GPU.  The wall-clock check runs once per 256 wake-ups: the
// polling loop of the first version (clock64 + compare every iteration) cost the CUDA-core warps of dft.cu a third of their issue slots.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  uint32_t spins = 0;
  long long t0 = 0;
  while (!mbar_try_wait_hint(bar, parity, 20000u)) {
    if ((++spins & 255u) == 0) {
      const long long t = clock64();
      if (t0 == 0) t0 = t;
      else if (t - t0 > 4000000000LL) {
        printf("b200sht: mbarrier timeout block (%d,%d,%d) thread %d\n", blockIdx.x, blockIdx.y, blockIdx.z, threadIdx.x);
        __trap();
      }
    }
  }
}

// mbar_wait for a warp with wgmma in flight: a lost arrival traps without the printf, since a function call (vprintf) inside the wgmma
// pipeline makes ptxas serialize every wgmma of the kernel
__device__ __forceinline__ void mbar_wait_nocall(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  uint32_t spins = 0;
  long long t0 = 0;
  while (!mbar_try_wait_hint(bar, parity, 20000u)) {
    if ((++spins & 255u) == 0) {
      const long long t = clock64();
      if (t0 == 0) t0 = t;
      else if (t - t0 > 4000000000LL) __trap();
    }
  }
}

// wait of a warp that is not on the critical path (epilogue / MMA issuer of a CUDA-core-bound kernel): poll every `ns` nanoseconds
// instead of waking on every arrival, so that the waiting warps leave the issue slots to the working ones
__device__ __forceinline__ void mbar_wait_relaxed(uint64_t* bar, uint32_t parity, uint32_t ns) {
  if (mbar_try_wait(bar, parity)) return;
  uint32_t spins = 0;
  long long t0 = 0;
  for (;;) {
    __nanosleep(ns);
    if (mbar_try_wait(bar, parity)) return;
    if ((++spins & 255u) == 0) {
      const long long t = clock64();
      if (t0 == 0) t0 = t;
      else if (t - t0 > 4000000000LL) {
        printf("b200sht: mbarrier timeout block (%d,%d,%d) thread %d\n", blockIdx.x, blockIdx.y, blockIdx.z, threadIdx.x);
        __trap();
      }
    }
  }
}

__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* tm, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(dst),
               "l"(tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* tm, uint64_t* bar, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(dst),
               "l"(tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void tma_load_5d(uint32_t dst, const CUtensorMap* tm, uint64_t* bar, int c0, int c1, int c2, int c3, int c4) {
  asm volatile("cp.async.bulk.tensor.5d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];" ::"r"(dst),
               "l"(tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
               : "memory");
}
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* tm) { asm volatile("prefetch.tensormap [%0];" ::"l"(tm) : "memory"); }

// ------------------------------------------------------------------------------------------- warp-level TF32 MMA
// Operand tiles are written by TMA with the 128-byte swizzle (16-byte chunk c of a 128-byte row lands at c ^ (row % 8); stage bases are
// 1024-byte aligned).  Two layouts, both 32 floats wide:
//   K-major:  row r (an M or N index) holds 32 consecutive K values
//   MN-major: blocks of [32 K-rows][32 consecutive M / N values], 4096 bytes apart
// Hopper's wgmma reads TF32 operands from shared memory only K-major: umma.cu runs its GEMMs with two K-major operands on it (descriptors
// below), and so does the analysis of dft.cu; the others run on mma.m16n8k8.  The m16n8k8 fragments below (used by dft.cu) are loaded element by element, so both layouts feed the
// same instruction; the GEMM engine of umma.cu loads permuted fragments with 8- and 16-byte loads instead.
__device__ __forceinline__ uint32_t swz128(uint32_t off) { return off ^ ((off >> 3) & 0x70u); }
template <bool MN>
__device__ __forceinline__ uint32_t ld_op(const uint8_t* tile, int r, int k) {
  const uint32_t off = MN ? (uint32_t)((r >> 5) * 4096 + k * 128 + (r & 31) * 4) : (uint32_t)(r * 128 + k * 4);
  return *reinterpret_cast<const uint32_t*>(tile + swz128(off));
}
// 8 / 16 bytes at the unswizzled byte offset `off` of a swizzled tile (off a multiple of 8 / 16: the swizzle moves whole 16-byte chunks)
__device__ __forceinline__ uint2 lds64(const uint8_t* tile, uint32_t off) { return *reinterpret_cast<const uint2*>(tile + swz128(off)); }
__device__ __forceinline__ uint4 lds128(const uint8_t* tile, uint32_t off) { return *reinterpret_cast<const uint4*>(tile + swz128(off)); }
// A fragment of mma.m16n8k8 (rows r0 + g, r0 + g + 8; K columns k0 + q, k0 + q + 4; g = lane / 4, q = lane % 4)
template <bool MN>
__device__ __forceinline__ void frag_a(const uint8_t* tile, int r0, int k0, uint32_t (&a)[4]) {
  const int lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
  a[0] = ld_op<MN>(tile, r0 + g, k0 + q);
  a[1] = ld_op<MN>(tile, r0 + g + 8, k0 + q);
  a[2] = ld_op<MN>(tile, r0 + g, k0 + q + 4);
  a[3] = ld_op<MN>(tile, r0 + g + 8, k0 + q + 4);
}
// B fragment (column n0 + g; K rows k0 + q, k0 + q + 4)
template <bool MN>
__device__ __forceinline__ void frag_b(const uint8_t* tile, int n0, int k0, uint32_t (&b)[2]) {
  const int lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
  b[0] = ld_op<MN>(tile, n0 + g, k0 + q);
  b[1] = ld_op<MN>(tile, n0 + g, k0 + q + 4);
}
__device__ __forceinline__ void frag_neg(const uint32_t (&a)[4], uint32_t (&n)[4]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) n[i] = a[i] ^ 0x80000000u;   // exact negation: flip the sign bit
}
// d += a * b; the accumulator element e of the fragment is (row g + 8 (e / 2), column 2 q + e % 2).  The tensor core reads the TF32 part of
// each operand (the 13 low mantissa bits are ignored), so producers of operands round first.
__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// ------------------------------------------------------------------------------------------- warpgroup TF32 MMA (wgmma)
// Shared-memory descriptor of a K-major operand tile as TMA lands it: rows of 32 floats (128 B) with the 128-byte swizzle, 8-row groups
// 1024 B apart (stride byte offset), `saddr` in a 1024-byte-aligned swizzle pattern (base offset 0).  The leading byte offset is unused for
// swizzled K-major tiles of one swizzle atom's width.  The k8 step s of the 32 K starts 32 s bytes into the rows: desc + 2 s.
__device__ __forceinline__ uint64_t wgmma_desc_kmajor(uint32_t saddr) {
  return (uint64_t)((saddr & 0x3FFFFu) >> 4) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}
// orders the warpgroup's earlier register accesses of the accumulators before the wgmma that follow
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// wait until at most N of the warpgroup's committed wgmma groups are pending
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// pins accumulator registers after a wgmma_wait: their reads cannot be scheduled before it
template <int NA>
__device__ __forceinline__ void wgmma_fence_operands(float (&d)[NA][4]) {
#pragma unroll
  for (int j = 0; j < NA; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) asm volatile("" : "+f"(d[j][e])::"memory");
}

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* tm, uint64_t* bar, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(dst),
               "l"(tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
               : "memory");
}
// generic-proxy shared-memory writes -> visible to the async proxy (TMA)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// bulk tensor stores from shared memory.  Bulk async-groups are per thread: the thread that commits a group is the one that waits for it.
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* tm, uint32_t src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(tm), "r"(src), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void tma_store_5d(const CUtensorMap* tm, uint32_t src, int c0, int c1, int c2, int c3, int c4) {
  asm volatile("cp.async.bulk.tensor.5d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];" ::"l"(tm), "r"(src), "r"(c0), "r"(c1),
               "r"(c2), "r"(c3), "r"(c4)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// wait until at most N of this thread's groups still read shared memory (.read) / are still writing global memory
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void bulk_wait_read0() { bulk_wait_read<0>(); }
__device__ __forceinline__ void bulk_wait0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ================================================================================================== host side
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(ptr);
  });
  return fn;
}

// Encoded tensor maps are a pure function of (base, shape, strides, box, swizzle): in steady state the caching allocator hands the same
// buffers to every step, so the 2-3 driver encodes per launch are replaced by a lookup in a small per-thread direct-mapped cache.
struct TmapKey {
  const void* base;
  long long dims[5], strides[5];
  int box[5];
  int rank, kind;   // kind: 0 fp32 / 128-byte swizzle, 1 fp32 / no swizzle, 4 fp32 segments, 5 bf16 segments
};
struct TmapCache {
  static constexpr int kSlots = 128;
  CUtensorMap maps[kSlots];
  TmapKey keys[kSlots];
  bool used[kSlots];
};
inline TmapCache& tmap_cache() {
  static thread_local TmapCache* c = [] { TmapCache* p = new TmapCache(); memset(p->used, 0, sizeof(p->used)); return p; }();
  return *c;
}
inline int tmap_slot(const TmapKey& k) {
  const unsigned char* b = reinterpret_cast<const unsigned char*>(&k);
  uint64_t h = 1469598103934665603ull;
  for (size_t i = 0; i < sizeof(TmapKey); ++i) { h ^= b[i]; h *= 1099511628211ull; }
  return (int)(h % TmapCache::kSlots);
}
inline bool tmap_lookup(const TmapKey& k, CUtensorMap* tm, int* slot) {
  TmapCache& c = tmap_cache();
  *slot = tmap_slot(k);
  if (c.used[*slot] && memcmp(&c.keys[*slot], &k, sizeof(TmapKey)) == 0) { memcpy(tm, &c.maps[*slot], sizeof(CUtensorMap)); return true; }
  return false;
}
inline void tmap_store(const TmapKey& k, const CUtensorMap* tm, int slot) {
  TmapCache& c = tmap_cache();
  memcpy(&c.maps[slot], tm, sizeof(CUtensorMap));
  c.keys[slot] = k;
  c.used[slot] = true;
}

// fp32 tensor map, 128-byte swizzle (swizzle = false: none, box rows land densely).  dims[0] is the contiguous dimension; strides (in
// floats) for dims 1..rank-1, in any order.
inline int make_tmap(CUtensorMap* tm, const void* base, int rank, const long long* dims, const long long* strides, const int* box,
                     bool swizzle = true) {
  TmapKey key;
  memset(&key, 0, sizeof(key));
  key.base = base; key.rank = rank; key.kind = swizzle ? 0 : 1;
  for (int i = 0; i < rank; ++i) { key.dims[i] = dims[i]; key.strides[i] = i ? strides[i] : 1; key.box[i] = box[i]; }
  int slot = 0;
  if (tmap_lookup(key, tm, &slot)) return 0;
  PFN_encodeTiled enc = get_encode();
  if (!enc) { set_error("cuTensorMapEncodeTiled is unavailable"); return B200SHT_ERR_UNSUPPORTED; }
  // cuTensorMapEncodeTiled is a DRIVER call: it needs a current context.  A thread that has made no runtime call yet (PyTorch's autograd
  // thread entering a backward whose first action is this encode) has none -> CUDA_ERROR_INVALID_CONTEXT (201).  Bind the primary context once per thread.
  static thread_local bool ctx_bound = false;
  if (!ctx_bound) { cudaFree(nullptr); ctx_bound = true; }
  cuuint64_t gd[5], gs[4];
  cuuint32_t bx[5], es[5];
  for (int i = 0; i < rank; ++i) { gd[i] = (cuuint64_t)dims[i]; bx[i] = (cuuint32_t)box[i]; es[i] = 1; }
  for (int i = 1; i < rank; ++i) {
    gs[i - 1] = (cuuint64_t)strides[i] * 4;
    if (gs[i - 1] % 16 != 0) { set_error("tensor map stride %lld floats is not 16-byte aligned", strides[i]); return B200SHT_ERR_INVALID; }
  }
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) { set_error("tensor map base is not 16-byte aligned"); return B200SHT_ERR_INVALID; }
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, (cuuint32_t)rank, const_cast<void*>(base), gd, gs, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   swizzle ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed (%d), rank %d", (int)r, rank); return B200SHT_ERR_CUDA; }
  tmap_store(key, tm, slot);
  return 0;
}


// 2-D tensor map over a row-major matrix of fp32 or bf16 elements without swizzle: box rows land densely (box_cols * esize bytes apart)
inline int make_tmap_rows(CUtensorMap* tm, const void* base, bool bf16, long long cols, long long rows, int box_cols, int box_rows) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) { set_error("cuTensorMapEncodeTiled is unavailable"); return B200SHT_ERR_UNSUPPORTED; }
  static thread_local bool ctx_bound = false;
  if (!ctx_bound) { cudaFree(nullptr); ctx_bound = true; }
  const int es = bf16 ? 2 : 4;
  cuuint64_t gd[2] = {(cuuint64_t)cols, (cuuint64_t)rows}, gs[1] = {(cuuint64_t)cols * es};
  cuuint32_t bx[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows}, el[2] = {1, 1};
  if (gs[0] % 16 != 0 || (reinterpret_cast<uintptr_t>(base) & 15) != 0 || (box_cols * es) % 16 != 0) {
    set_error("tensor map (rows): base / row pitch / box row not 16-byte aligned");
    return B200SHT_ERR_INVALID;
  }
  CUresult r = enc(tm, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(base), gd, gs, bx, el,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled (rows) failed (%d)", (int)r); return B200SHT_ERR_CUDA; }
  return 0;
}

}  // namespace b200sht
