// Global attention on the sphere (torch_harmonics.AttentionS2): a quadrature-weighted flash attention on wgmma (DESIGN.md section 4.10).
// Per head (b, h), with the per-key bias b_j = log w_j (-inf for a zero quadrature weight):
//
//   y_i = sum_j exp(scale <q_i, k_j> + b_j) v_j / sum_j exp(scale <q_i, k_j> + b_j),   lse_i = log sum_j exp(scale <q_i, k_j> + b_j)
//
// Operands in global memory (fp32): q, o (BH, nq, dqk / dv), k (BH, nk, dqk), v (BH, dv, nk).  wgmma reads TF32 operands from shared memory
// K-major only, so every GEMM runs with both operands contracted along their contiguous axis:
//   forward   S = Q K^T (over d)   O += P V_j (over keys: v is (d, N), already K-major)
//   dK / dV   S^T = K Q^T, dP^T = V dO^T (over d; V as (N, d))   dV += P^T dO, dK += dS^T Q (over queries; dO^T, Q^T as (d, N))
//   dQ        S = Q K^T, dP = dO V^T (over d)   dQ += dS K (over keys; K^T as (d, N))
// A prep kernel writes each operand once into a workspace in the layout its GEMM reads, rounded to TF32 (round to nearest: the tensor core
// truncates); with 3 x TF32 (SPLIT) it also writes the residual lo = tf32(x - hi), and every product is a_lo b_hi + a_hi b_lo + a_hi b_hi.
//
// One CTA = one consumer warpgroup (warps 0-3, 64 resident rows: queries in the forward and dQ, keys in dK / dV) + one TMA producer warp.
// The resident tiles are loaded once; the streamed 32-row blocks come through an mbarrier ring of `stages` slots, each slot two tiles
// (hi and, with SPLIT, lo planes).  A head dim d is served in DC = ceil(d / 32) 32-float chunks (TMA fills the pad with zeros).  Softmax
// statistics are fp32 registers; the bias is added before the running max.  P and dS go through a 64 x 32 shared tile (written by the
// warpgroup, fence.proxy.async) into the second GEMM.  Every output element is summed by one warpgroup in a fixed order, with no atomics:
// results are bit-identical run to run.
#include "umma_common.cuh"
#include "wgmma_tf32.cuh"
#include <algorithm>
#include <cmath>

namespace b200sht {

constexpr int kAgThreads = 160;    // warps 0-3: consumer warpgroup; warp 4: TMA producer
constexpr int kAgBM = 64;          // resident rows per CTA
constexpr int kAgBN = 32;          // rows of a streamed block
constexpr int kAgMaxStages = 4;
constexpr int kAgMaxChunks = 4;    // head dims up to 128

enum AgKind { kAgFwd = 0, kAgDkv = 1, kAgDq = 2 };

struct AgParams {
  CUtensorMap res[2][2];       // [plane][resident operand], boxes of 64 rows
  CUtensorMap item[2][2][2];   // [plane][phase][tile], boxes of 32 rows (row tiles) or 32 columns (column tiles)
  const float* bias;           // (nk): log quadrature weight per key
  const float* lse;            // backward: (BH, nq)
  const float* D;              // backward: (BH, nq)
  float* out0;                 // fwd: o (BH, nq, dv); dkv: dk (BH, nk, dqk); dq: dq (BH, nq, dqk)
  float* out1;                 // fwd: lse (BH, nq); dkv: dv (BH, dv, nk)
  int nq, nk, dqk, dv, stages;
  float scale;
};

// resident operands and streamed tiles of each kernel: how many, and which tiles are column tiles ((d, N) layout, one TMA box)
template <int KIND> struct AgShape;
template <> struct AgShape<kAgFwd> {   // resident Q; per key block: K rows, V columns
  static constexpr int kRes = 1, kPhases = 1, kProd = 1;
  __device__ static constexpr bool cols(int, int t) { return t == 1; }
  __device__ static constexpr int ntiles(int) { return 2; }
};
template <> struct AgShape<kAgDkv> {   // resident K, V; per query block: (Q, dO) rows, then (Q^T, dO^T) columns
  static constexpr int kRes = 2, kPhases = 2, kProd = 2;
  __device__ static constexpr bool cols(int ph, int) { return ph == 1; }
  __device__ static constexpr int ntiles(int) { return 2; }
};
template <> struct AgShape<kAgDq> {    // resident Q, dO; per key block: (K, V) rows, then K^T columns
  static constexpr int kRes = 2, kPhases = 2, kProd = 1;
  __device__ static constexpr bool cols(int ph, int) { return ph == 1; }
  __device__ static constexpr int ntiles(int ph) { return ph == 0 ? 2 : 1; }
};

template <int DC> struct AgSizes {
  static constexpr uint32_t kRes = kAgBM * 32 * DC * 4;    // one resident tile
  static constexpr uint32_t kTile = kAgBN * 32 * DC * 4;   // one streamed tile (row or column)
  static constexpr uint32_t kProd = kAgBM * kAgBN * 4;     // one P / dS tile
};

__host__ __device__ constexpr uint32_t ag_fixed_bytes(int kind, int dc, bool split) {
  const int planes = split ? 2 : 1;
  const int nres = kind == kAgFwd ? 1 : 2, nprod = kind == kAgDkv ? 2 : 1;
  return (uint32_t)(planes * (nres * kAgBM * 32 * dc * 4 + nprod * kAgBM * kAgBN * 4));
}
__host__ __device__ constexpr uint32_t ag_slot_bytes(int dc, bool split) { return (uint32_t)((split ? 2 : 1) * 2 * kAgBN * 32 * dc * 4); }

__device__ __forceinline__ void ag_bar_sync() { asm volatile("bar.sync 1, 128;" ::: "memory"); }   // the consumer warpgroup

// ---------------------------------------------------------------------------------------------------------------------- MMA blocks
// acc (64 x 32) [+]= A B^T over DC chunks: A a resident row tile (chunks of 64 rows x 128 B), B a streamed row tile (chunks of 32 rows)
template <int DC, bool SPLIT>
__device__ __forceinline__ void ag_mma_rows(float (&acc)[4][4], uint32_t a, uint32_t a_lo, uint32_t b, uint32_t b_lo) {
#pragma unroll
  for (int c = 0; c < DC; ++c) {
    const uint64_t da = wgmma_desc_kmajor(a + c * AgSizes<1>::kRes), db = wgmma_desc_kmajor(b + c * AgSizes<1>::kTile);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int sd = (c > 0 || k > 0) ? 1 : 0;
      if constexpr (SPLIT) {
        const uint64_t dal = wgmma_desc_kmajor(a_lo + c * AgSizes<1>::kRes), dbl = wgmma_desc_kmajor(b_lo + c * AgSizes<1>::kTile);
        wgmma_tf32<32, 1, 4, 0>(acc, dal + 2 * k, db + 2 * k, sd);
        wgmma_tf32<32, 1, 4, 0>(acc, da + 2 * k, dbl + 2 * k, 1);
        wgmma_tf32<32, 1, 4, 0>(acc, da + 2 * k, db + 2 * k, 1);
      } else {
        wgmma_tf32<32, 1, 4, 0>(acc, da + 2 * k, db + 2 * k, sd);
      }
    }
  }
}

// acc (64 x 32 DC) = P B^T over the block's 32 rows: P a product tile (64 rows x 128 B), B a column tile (32 DC rows x 128 B).  The callers
// add the block's product to their running sums with fp32 FMAs.  Summed across blocks inside the tensor core's accumulator instead, the
// 3 x TF32 module missed fp32 accuracy over long sums (relative L2 3.2e-4 against fp64 at 65160 keys, 181 x 360 -> 361 x 720).
template <int DC, bool SPLIT>
__device__ __forceinline__ void ag_mma_cols(float (&acc)[4 * DC][4], uint32_t p, uint32_t p_lo, uint32_t b, uint32_t b_lo) {
  const uint64_t dp = wgmma_desc_kmajor(p), db = wgmma_desc_kmajor(b);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    if constexpr (SPLIT) {
      const uint64_t dpl = wgmma_desc_kmajor(p_lo), dbl = wgmma_desc_kmajor(b_lo);
      wgmma_tf32<32 * DC, 1, 4 * DC, 0>(acc, dpl + 2 * k, db + 2 * k, k > 0 ? 1 : 0);
      wgmma_tf32<32 * DC, 1, 4 * DC, 0>(acc, dp + 2 * k, dbl + 2 * k, 1);
      wgmma_tf32<32 * DC, 1, 4 * DC, 0>(acc, dp + 2 * k, db + 2 * k, 1);
    } else {
      wgmma_tf32<32 * DC, 1, 4 * DC, 0>(acc, dp + 2 * k, db + 2 * k, k > 0 ? 1 : 0);
    }
  }
}

// sum = sum * mul + blk, element by element
template <int N>
__device__ __forceinline__ void ag_accumulate(float (&sum)[N][4], const float (&blk)[N][4], const float (&mul)[2]) {
#pragma unroll
  for (int j = 0; j < N; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) sum[j][e] = fmaf(sum[j][e], mul[e >> 1], blk[j][e]);
}

// the 64 x 32 accumulator x into a product tile, rounded to TF32 (and its residual with SPLIT).  Element (j, e) of the fragment is row
// 16 warp + g + 8 (e / 2), column 8 j + 2 q + e % 2.
template <bool SPLIT>
__device__ __forceinline__ void ag_put_tile(uint8_t* t, uint8_t* t_lo, const float (&x)[4][4]) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, g = lane >> 2, q = lane & 3;
#pragma unroll
  for (int j = 0; j < 4; ++j)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const uint32_t off = swz128((uint32_t)((16 * w + g + 8 * h) * 128 + (8 * j + 2 * q) * 4));
      const float2 hi = make_float2(tf32_rn(x[j][2 * h]), tf32_rn(x[j][2 * h + 1]));
      *reinterpret_cast<float2*>(t + off) = hi;
      if constexpr (SPLIT)
        *reinterpret_cast<float2*>(t_lo + off) = make_float2(tf32_rn(x[j][2 * h] - hi.x), tf32_rn(x[j][2 * h + 1] - hi.y));
    }
}

template <int N>
__device__ __forceinline__ void ag_zero(float (&a)[N][4]) {
#pragma unroll
  for (int j = 0; j < N; ++j) a[j][0] = a[j][1] = a[j][2] = a[j][3] = 0.f;
}

// ---------------------------------------------------------------------------------------------------------------------- the kernel
template <int KIND, int DC, bool SPLIT>
__global__ void __launch_bounds__(kAgThreads, 1) attention_global_kernel(const __grid_constant__ AgParams p) {
  using Sh = AgShape<KIND>;
  using Sz = AgSizes<DC>;
  constexpr int kPlanes = SPLIT ? 2 : 1;
  constexpr uint32_t kSlot = 2 * Sz::kTile * kPlanes;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* gbase = smem_raw + (base - raw);
  const uint32_t res_s = base;                                              // [plane][operand]
  const uint32_t ring_s = res_s + kPlanes * Sh::kRes * Sz::kRes;            // [stage][plane][tile]
  const uint32_t prod_s = ring_s + p.stages * kSlot;                        // [plane][product]
  uint8_t* prod = gbase + (prod_s - base);
  uint64_t* bars = reinterpret_cast<uint64_t*>(prod + kPlanes * Sh::kProd * Sz::kProd);
  uint64_t* res_full = bars;
  uint64_t* full = bars + 1;
  uint64_t* empty = full + kAgMaxStages;

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  const int bh = blockIdx.y, row0 = blockIdx.x * kAgBM;
  const int nstream = KIND == kAgDkv ? p.nq : p.nk;   // rows of the streamed operands
  const int nblk = (nstream + kAgBN - 1) / kAgBN;
  const int nitems = nblk * Sh::kPhases;
  const int stages = p.stages;

  if (threadIdx.x == 128) {
    mbar_init(res_full, 1);
    for (int s = 0; s < stages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 4); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 4) {
    if (lane == 0) {
      mbar_expect_tx(res_full, kPlanes * Sh::kRes * Sz::kRes);
      for (int pl = 0; pl < kPlanes; ++pl)
        for (int r = 0; r < Sh::kRes; ++r)
          for (int c = 0; c < DC; ++c)
            tma_load_3d(res_s + (pl * Sh::kRes + r) * Sz::kRes + c * AgSizes<1>::kRes, &p.res[pl][r], res_full, 32 * c, row0, bh);
      for (int i = 0; i < nitems; ++i) {
        const int s = i % stages, it = i / stages, ph = i % Sh::kPhases, blk0 = (i / Sh::kPhases) * kAgBN;
        if (it > 0) mbar_wait_nocall(&empty[s], (it - 1) & 1);
        mbar_expect_tx(&full[s], kPlanes * Sh::ntiles(ph) * Sz::kTile);
        for (int pl = 0; pl < kPlanes; ++pl)
          for (int t = 0; t < Sh::ntiles(ph); ++t) {
            const uint32_t dst = ring_s + s * kSlot + (pl * 2 + t) * Sz::kTile;
            if (Sh::cols(ph, t)) tma_load_3d(dst, &p.item[pl][ph][t], &full[s], blk0, 0, bh);
            else
              for (int c = 0; c < DC; ++c) tma_load_3d(dst + c * AgSizes<1>::kTile, &p.item[pl][ph][t], &full[s], 32 * c, blk0, bh);
          }
      }
    }
    return;
  }

  const int g = lane >> 2, q = lane & 3;
  const uint32_t resA = res_s, resB = res_s + Sz::kRes;                       // hi planes of the resident operands
  const uint32_t resA_lo = resA + Sh::kRes * Sz::kRes, resB_lo = resB + Sh::kRes * Sz::kRes;
  auto tile = [&](int s, int pl, int t) { return ring_s + s * kSlot + (pl * 2 + t) * Sz::kTile; };
  uint8_t* prod0 = prod;
  uint8_t* prod1 = prod + Sz::kProd;                                          // dkv: dS^T
  uint8_t* prod0_lo = prod + Sh::kProd * Sz::kProd;
  uint8_t* prod1_lo = prod0_lo + Sz::kProd;
  const uint32_t prod0_s = prod_s, prod1_s = prod_s + Sz::kProd;
  const uint32_t prod0_lo_s = prod_s + Sh::kProd * Sz::kProd, prod1_lo_s = prod0_lo_s + Sz::kProd;
  mbar_wait_nocall(res_full, 0);

  if constexpr (KIND == kAgFwd) {
    float o[4 * DC][4];
    ag_zero(o);
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
    for (int i = 0; i < nitems; ++i) {
      const int s = i % stages, key0 = i * kAgBN;
      mbar_wait_nocall(&full[s], (i / stages) & 1);
      float sc[4][4];
      wgmma_fence();
      ag_mma_rows<DC, SPLIT>(sc, resA, resA_lo, tile(s, 0, 0), tile(s, 1, 0));
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_operands(sc);
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int key = key0 + 8 * j + 2 * q + (e & 1);
          const float b = key < p.nk ? __ldg(p.bias + key) : -INFINITY;
          sc[j][e] = fmaf(sc[j][e], p.scale, b);
          mx[e >> 1] = fmaxf(mx[e >> 1], sc[j][e]);
        }
      float alpha[2], rs[2] = {0.f, 0.f};
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
        mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
        const float mn = fmaxf(m[h], mx[h]);
        const float mu = mn == -INFINITY ? 0.f : mn;   // no finite logit yet: exp(-inf - 0) = 0 keeps l = 0, o = 0
        alpha[h] = expf(m[h] - mu);
        m[h] = mn;
        mx[h] = mu;
      }
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          sc[j][e] = expf(sc[j][e] - mx[e >> 1]);
          rs[e >> 1] += sc[j][e];
        }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        rs[h] += __shfl_xor_sync(0xffffffffu, rs[h], 1);
        rs[h] += __shfl_xor_sync(0xffffffffu, rs[h], 2);
        l[h] = fmaf(alpha[h], l[h], rs[h]);
      }
      ag_bar_sync();   // every warp's P V of the block before has read the product tile
      ag_put_tile<SPLIT>(prod0, prod0_lo, sc);
      fence_proxy_async();
      ag_bar_sync();
      float pv[4 * DC][4];
      wgmma_fence();
      ag_mma_cols<DC, SPLIT>(pv, prod0_s, prod0_lo_s, tile(s, 0, 1), tile(s, 1, 1));
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_operands(pv);
      if (lane == 0) mbar_arrive(&empty[s]);
      ag_accumulate(o, pv, alpha);
    }
    float* out = p.out0 + (size_t)bh * p.nq * p.dv;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = row0 + 16 * warp + g + 8 * h;
      if (row >= p.nq) continue;
      const float inv = 1.f / l[h];
#pragma unroll
      for (int j = 0; j < 4 * DC; ++j) {
        const int col = 8 * j + 2 * q;
        if (col < p.dv) *reinterpret_cast<float2*>(out + (size_t)row * p.dv + col) = make_float2(o[j][2 * h] * inv, o[j][2 * h + 1] * inv);
      }
      if (q == 0) p.out1[(size_t)bh * p.nq + row] = m[h] + logf(l[h]);
    }
  } else if constexpr (KIND == kAgDkv) {
    float dk[4 * DC][4], dv[4 * DC][4];
    ag_zero(dk);
    ag_zero(dv);
    const float one[2] = {1.f, 1.f};
    float kb[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int key = row0 + 16 * warp + g + 8 * h;
      kb[h] = key < p.nk ? __ldg(p.bias + key) : -INFINITY;
    }
    const float* lse = p.lse + (size_t)bh * p.nq;
    const float* Dq = p.D + (size_t)bh * p.nq;
    for (int b = 0; b < nblk; ++b) {
      const int q0 = b * kAgBN;
      int i = 2 * b, s = i % stages;
      mbar_wait_nocall(&full[s], (i / stages) & 1);
      float st[4][4], dpt[4][4];
      wgmma_fence();
      ag_mma_rows<DC, SPLIT>(st, resA, resA_lo, tile(s, 0, 0), tile(s, 1, 0));
      ag_mma_rows<DC, SPLIT>(dpt, resB, resB_lo, tile(s, 0, 1), tile(s, 1, 1));
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_operands(st);
      wgmma_fence_operands(dpt);
      if (lane == 0) mbar_arrive(&empty[s]);
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int qi = q0 + 8 * j + 2 * q + (e & 1);
          const float lq = qi < p.nq ? __ldg(lse + qi) : INFINITY, dq = qi < p.nq ? __ldg(Dq + qi) : 0.f;
          const float pr = expf(fmaf(st[j][e], p.scale, kb[e >> 1]) - lq);
          st[j][e] = pr;
          dpt[j][e] = pr * (dpt[j][e] - dq);
        }
      ag_bar_sync();
      ag_put_tile<SPLIT>(prod0, prod0_lo, st);
      ag_put_tile<SPLIT>(prod1, prod1_lo, dpt);
      fence_proxy_async();
      ag_bar_sync();
      i = 2 * b + 1;
      s = i % stages;
      mbar_wait_nocall(&full[s], (i / stages) & 1);
      float blk[4 * DC][4];
      wgmma_fence();
      ag_mma_cols<DC, SPLIT>(blk, prod0_s, prod0_lo_s, tile(s, 0, 1), tile(s, 1, 1));
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_operands(blk);
      ag_accumulate(dv, blk, one);
      wgmma_fence();
      ag_mma_cols<DC, SPLIT>(blk, prod1_s, prod1_lo_s, tile(s, 0, 0), tile(s, 1, 0));
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_operands(blk);
      if (lane == 0) mbar_arrive(&empty[s]);
      ag_accumulate(dk, blk, one);
    }
    float* odk = p.out0 + (size_t)bh * p.nk * p.dqk;
    float* odv = p.out1 + (size_t)bh * p.dv * p.nk;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int key = row0 + 16 * warp + g + 8 * h;
      if (key >= p.nk) continue;
#pragma unroll
      for (int j = 0; j < 4 * DC; ++j) {
        const int col = 8 * j + 2 * q;
        if (col < p.dqk)
          *reinterpret_cast<float2*>(odk + (size_t)key * p.dqk + col) = make_float2(dk[j][2 * h] * p.scale, dk[j][2 * h + 1] * p.scale);
        if (col < p.dv) {
          odv[(size_t)col * p.nk + key] = dv[j][2 * h];
          odv[(size_t)(col + 1) * p.nk + key] = dv[j][2 * h + 1];
        }
      }
    }
  } else {
    float dq[4 * DC][4];
    ag_zero(dq);
    const float one[2] = {1.f, 1.f};
    float lq[2], Dr[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = row0 + 16 * warp + g + 8 * h;
      lq[h] = row < p.nq ? __ldg(p.lse + (size_t)bh * p.nq + row) : INFINITY;
      Dr[h] = row < p.nq ? __ldg(p.D + (size_t)bh * p.nq + row) : 0.f;
    }
    for (int b = 0; b < nblk; ++b) {
      const int key0 = b * kAgBN;
      int i = 2 * b, s = i % stages;
      mbar_wait_nocall(&full[s], (i / stages) & 1);
      float sc[4][4], dp[4][4];
      wgmma_fence();
      ag_mma_rows<DC, SPLIT>(sc, resA, resA_lo, tile(s, 0, 0), tile(s, 1, 0));
      ag_mma_rows<DC, SPLIT>(dp, resB, resB_lo, tile(s, 0, 1), tile(s, 1, 1));
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_operands(sc);
      wgmma_fence_operands(dp);
      if (lane == 0) mbar_arrive(&empty[s]);
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int key = key0 + 8 * j + 2 * q + (e & 1);
          const float bk = key < p.nk ? __ldg(p.bias + key) : -INFINITY;
          const float pr = expf(fmaf(sc[j][e], p.scale, bk) - lq[e >> 1]);
          sc[j][e] = pr * (dp[j][e] - Dr[e >> 1]);
        }
      ag_bar_sync();
      ag_put_tile<SPLIT>(prod0, prod0_lo, sc);
      fence_proxy_async();
      ag_bar_sync();
      i = 2 * b + 1;
      s = i % stages;
      mbar_wait_nocall(&full[s], (i / stages) & 1);
      float blk[4 * DC][4];
      wgmma_fence();
      ag_mma_cols<DC, SPLIT>(blk, prod0_s, prod0_lo_s, tile(s, 0, 0), tile(s, 1, 0));
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_operands(blk);
      if (lane == 0) mbar_arrive(&empty[s]);
      ag_accumulate(dq, blk, one);
    }
    float* odq = p.out0 + (size_t)bh * p.nq * p.dqk;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = row0 + 16 * warp + g + 8 * h;
      if (row >= p.nq) continue;
#pragma unroll
      for (int j = 0; j < 4 * DC; ++j) {
        const int col = 8 * j + 2 * q;
        if (col < p.dqk)
          *reinterpret_cast<float2*>(odq + (size_t)row * p.dqk + col) = make_float2(dq[j][2 * h] * p.scale, dq[j][2 * h + 1] * p.scale);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------- prep kernels
// dst[bh] = src[bh] (rows x cols, contiguous) rounded to TF32, transposed when TRANS (dst row stride ld), residual into lo when lo != null
template <bool TRANS>
__global__ void __launch_bounds__(256) attention_global_prep_kernel(const float* __restrict__ src, int rows, int cols, float* __restrict__ hi,
                                                                    float* __restrict__ lo, int ld) {
  __shared__ float t[32][33];
  const size_t bh = blockIdx.z;
  const int r0 = blockIdx.y * 32, c0 = blockIdx.x * 32;
  const float* s = src + bh * rows * cols;
  const size_t dstride = (size_t)(TRANS ? cols : rows) * ld;
  for (int r = threadIdx.y; r < 32; r += 8) {
    const int rr = r0 + r, cc = c0 + threadIdx.x;
    t[r][threadIdx.x] = (rr < rows && cc < cols) ? s[(size_t)rr * cols + cc] : 0.f;
  }
  __syncthreads();
  for (int r = threadIdx.y; r < 32; r += 8) {
    int rr, cc;
    float x;
    if (TRANS) { rr = c0 + r; cc = r0 + threadIdx.x; x = t[threadIdx.x][r]; if (rr >= cols || cc >= rows) continue; }
    else { rr = r0 + r; cc = c0 + threadIdx.x; x = t[r][threadIdx.x]; if (rr >= rows || cc >= cols) continue; }
    const size_t o = bh * dstride + (size_t)rr * ld + cc;
    const float h = tf32_rn(x);
    hi[o] = h;
    if (lo) lo[o] = tf32_rn(x - h);
  }
}

// D[row] = sum_c do[row][c] o[row][c], in channel order
__global__ void attention_global_rowdot_kernel(const float* __restrict__ o, const float* __restrict__ dout, float* __restrict__ D, long long rows,
                                               int d) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  float acc = 0.f;
  for (int c = 0; c < d; ++c) acc = fmaf(dout[r * d + c], o[r * d + c], acc);
  D[r] = acc;
}

// ---------------------------------------------------------------------------------------------------------------------- host side
namespace {

struct AgWs {   // workspace buffers in floats, each 64-float aligned
  size_t off = 0;
  size_t take(size_t n) { const size_t o = off; off += (n + 63) / 64 * 64; return o; }
};

int ag_prep(const float* src, int BH, int rows, int cols, float* hi, float* lo, int ld, bool trans, cudaStream_t st) {
  const dim3 grid(ceil_div(cols, 32), ceil_div(rows, 32), BH), block(32, 8);
  if (trans) attention_global_prep_kernel<true><<<grid, block, 0, st>>>(src, rows, cols, hi, lo, ld);
  else attention_global_prep_kernel<false><<<grid, block, 0, st>>>(src, rows, cols, hi, lo, ld);
  B200_CHECK_LAUNCH();
  return 0;
}

// row tile map over (BH, n, dd) with row stride ld: boxes of 32 floats x box_rows rows
int ag_map_rows(CUtensorMap* tm, const float* x, int BH, int n, int dd, int box_rows) {
  const long long dims[3] = {dd, n, BH}, strides[3] = {1, dd, (long long)n * dd};
  const int box[3] = {32, box_rows, 1};
  return make_tmap(tm, x, 3, dims, strides, box);
}
// column tile map over (BH, dd, n) with row stride ld: boxes of 32 columns x 32 DC rows
int ag_map_cols(CUtensorMap* tm, const float* x, int BH, int n, int dd, int ld, int dc) {
  const long long dims[3] = {n, dd, BH}, strides[3] = {1, ld, (long long)dd * ld};
  const int box[3] = {32, 32 * dc, 1};
  return make_tmap(tm, x, 3, dims, strides, box);
}

template <int KIND, int DC, bool SPLIT>
int ag_launch_one(const AgParams& p, int grid_x, int BH, size_t smem, cudaStream_t st) {
  B200_CHECK_CUDA(cudaFuncSetAttribute(attention_global_kernel<KIND, DC, SPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  attention_global_kernel<KIND, DC, SPLIT><<<dim3(grid_x, BH), kAgThreads, smem, st>>>(p);
  B200_CHECK_LAUNCH();
  return 0;
}

template <int KIND, bool SPLIT>
int ag_dispatch(const AgParams& p, int dc, int grid_x, int BH, size_t smem, cudaStream_t st) {
  switch (dc) {
    case 1: return ag_launch_one<KIND, 1, SPLIT>(p, grid_x, BH, smem, st);
    case 2: return ag_launch_one<KIND, 2, SPLIT>(p, grid_x, BH, smem, st);
    case 3: return ag_launch_one<KIND, 3, SPLIT>(p, grid_x, BH, smem, st);
    default: return ag_launch_one<KIND, 4, SPLIT>(p, grid_x, BH, smem, st);
  }
}

// ring depth: up to 4 stages within half an SM's shared memory (two CTAs per SM), otherwise as many as one CTA can hold
int ag_launch(int kind, AgParams& p, int dc, bool split, int grid_x, int BH, cudaStream_t st) {
  const size_t fixed = 1024 + ag_fixed_bytes(kind, dc, split) + 8 * (1 + 2 * kAgMaxStages), slot = ag_slot_bytes(dc, split);
  const size_t half = 113 * 1024, full = 227 * 1024;
  int stages = fixed + 2 * slot <= half ? (int)std::min<size_t>(kAgMaxStages, (half - fixed) / slot)
                                        : (int)std::min<size_t>(kAgMaxStages, (full - fixed) / slot);
  B200_REQUIRE(stages >= 1, "attention_global: no ring fits in shared memory (kind %d, %d chunks)", kind, dc);
  p.stages = stages;
  const size_t smem = fixed + stages * slot;
  if (kind == kAgFwd) return split ? ag_dispatch<kAgFwd, true>(p, dc, grid_x, BH, smem, st) : ag_dispatch<kAgFwd, false>(p, dc, grid_x, BH, smem, st);
  if (kind == kAgDkv) return split ? ag_dispatch<kAgDkv, true>(p, dc, grid_x, BH, smem, st) : ag_dispatch<kAgDkv, false>(p, dc, grid_x, BH, smem, st);
  return split ? ag_dispatch<kAgDq, true>(p, dc, grid_x, BH, smem, st) : ag_dispatch<kAgDq, false>(p, dc, grid_x, BH, smem, st);
}

int ag_check(int BH, int nq, int nk, int dqk, int dv) {
  B200_REQUIRE(BH >= 1 && BH <= 65535 && nq >= 1 && nk >= 1, "attention_global: BH %d (1 .. 65535), nq %d, nk %d must be positive", BH, nq, nk);
  if (dqk < 8 || dv < 8 || dqk > 32 * kAgMaxChunks || dv > 32 * kAgMaxChunks || dqk % 8 || dv % 8) {
    set_error("attention_global: head dims %d, %d: multiples of 8 up to %d are served", dqk, dv, 32 * kAgMaxChunks);
    return B200SHT_ERR_UNSUPPORTED;
  }
  return 0;
}

// offsets (floats) of the backward's operands in the layouts its GEMMs read, and of D; the workspace query counts the same layout, so one
// backward workspace serves the full backward and either pass
struct AgBwdWs {
  size_t Q[2] = {}, Qt[2] = {}, K[2] = {}, Kt[2] = {}, Vn[2] = {}, dO[2] = {}, dOt[2] = {}, D = 0, total = 0;
};

AgBwdWs ag_bwd_ws(int BH, int nq, int nk, int dqk, int dv, int planes) {
  const size_t ldq = round_up(nq, 4), ldk = round_up(nk, 4);
  AgWs w;
  AgBwdWs l;
  for (int pl = 0; pl < planes; ++pl) {
    l.Q[pl] = w.take((size_t)BH * nq * dqk);
    l.Qt[pl] = w.take((size_t)BH * dqk * ldq);
    l.K[pl] = w.take((size_t)BH * nk * dqk);
    l.Kt[pl] = w.take((size_t)BH * dqk * ldk);
    l.Vn[pl] = w.take((size_t)BH * nk * dv);
    l.dO[pl] = w.take((size_t)BH * nq * dv);
    l.dOt[pl] = w.take((size_t)BH * dv * ldq);
  }
  l.D = w.take((size_t)BH * nq);
  l.total = w.off;
  return l;
}

enum { kAgPassKv = 1, kAgPassQ = 2 };

// the passes of the backward named in `passes`, given D: prepares each operand layout they read once, then dK / dV per key block (kv pass)
// and dQ per query block (q pass).  The full backward runs both on the same layouts; either pass alone reads only its own operands.
int ag_backward_passes(int passes, const float* q, const float* k, const float* v, const float* bias, const float* lse, const float* D,
                       const float* dout, float* dq, float* dk, float* dv_, int BH, int nq, int nk, int dqk, int dv, float scale, int split,
                       float* ws, cudaStream_t st) {
  const bool kv = passes & kAgPassKv, qp = passes & kAgPassQ;
  const int dc = ceil_div(std::max(dqk, dv), 32), ldq = round_up(nq, 4), ldk = round_up(nk, 4), planes = split ? 2 : 1;
  const AgBwdWs l = ag_bwd_ws(BH, nq, nk, dqk, dv, planes);
  float *Q[2] = {}, *Qt[2] = {}, *K[2] = {}, *Kt[2] = {}, *Vn[2] = {}, *dO[2] = {}, *dOt[2] = {};
  for (int pl = 0; pl < planes; ++pl) {
    Q[pl] = ws + l.Q[pl]; Qt[pl] = ws + l.Qt[pl]; K[pl] = ws + l.K[pl]; Kt[pl] = ws + l.Kt[pl];
    Vn[pl] = ws + l.Vn[pl]; dO[pl] = ws + l.dO[pl]; dOt[pl] = ws + l.dOt[pl];
  }
  if (int rc = ag_prep(q, BH, nq, dqk, Q[0], Q[1], dqk, false, st)) return rc;
  if (kv)
    if (int rc = ag_prep(q, BH, nq, dqk, Qt[0], Qt[1], ldq, true, st)) return rc;
  if (int rc = ag_prep(k, BH, nk, dqk, K[0], K[1], dqk, false, st)) return rc;
  if (qp)
    if (int rc = ag_prep(k, BH, nk, dqk, Kt[0], Kt[1], ldk, true, st)) return rc;
  if (int rc = ag_prep(v, BH, dv, nk, Vn[0], Vn[1], dv, true, st)) return rc;
  if (int rc = ag_prep(dout, BH, nq, dv, dO[0], dO[1], dv, false, st)) return rc;
  if (kv)
    if (int rc = ag_prep(dout, BH, nq, dv, dOt[0], dOt[1], ldq, true, st)) return rc;

  AgParams p;
  if (kv) {
    memset(&p, 0, sizeof(p));
    for (int pl = 0; pl < planes; ++pl) {   // dK / dV: resident K, V (key rows); per query block (Q, dO) rows, then (Q^T, dO^T) columns
      if (int rc = ag_map_rows(&p.res[pl][0], K[pl], BH, nk, dqk, kAgBM)) return rc;
      if (int rc = ag_map_rows(&p.res[pl][1], Vn[pl], BH, nk, dv, kAgBM)) return rc;
      if (int rc = ag_map_rows(&p.item[pl][0][0], Q[pl], BH, nq, dqk, kAgBN)) return rc;
      if (int rc = ag_map_rows(&p.item[pl][0][1], dO[pl], BH, nq, dv, kAgBN)) return rc;
      if (int rc = ag_map_cols(&p.item[pl][1][0], Qt[pl], BH, nq, dqk, ldq, dc)) return rc;
      if (int rc = ag_map_cols(&p.item[pl][1][1], dOt[pl], BH, nq, dv, ldq, dc)) return rc;
    }
    p.bias = bias; p.lse = lse; p.D = D; p.out0 = dk; p.out1 = dv_;
    p.nq = nq; p.nk = nk; p.dqk = dqk; p.dv = dv; p.scale = scale;
    if (int rc = ag_launch(kAgDkv, p, dc, split != 0, ceil_div(nk, kAgBM), BH, st)) return rc;
  }
  if (qp) {
    memset(&p, 0, sizeof(p));
    for (int pl = 0; pl < planes; ++pl) {   // dQ: resident Q, dO (query rows); per key block (K, V) rows, then K^T columns
      if (int rc = ag_map_rows(&p.res[pl][0], Q[pl], BH, nq, dqk, kAgBM)) return rc;
      if (int rc = ag_map_rows(&p.res[pl][1], dO[pl], BH, nq, dv, kAgBM)) return rc;
      if (int rc = ag_map_rows(&p.item[pl][0][0], K[pl], BH, nk, dqk, kAgBN)) return rc;
      if (int rc = ag_map_rows(&p.item[pl][0][1], Vn[pl], BH, nk, dv, kAgBN)) return rc;
      if (int rc = ag_map_cols(&p.item[pl][1][0], Kt[pl], BH, nk, dqk, ldk, dc)) return rc;
    }
    p.bias = bias; p.lse = lse; p.D = D; p.out0 = dq;
    p.nq = nq; p.nk = nk; p.dqk = dqk; p.dv = dv; p.scale = scale;
    if (int rc = ag_launch(kAgDq, p, dc, split != 0, ceil_div(nq, kAgBM), BH, st)) return rc;
  }
  return 0;
}

}  // namespace

long long attention_global_workspace_floats(int BH, int nq, int nk, int dqk, int dv, int split, int backward) {
  if (ag_check(BH, nq, nk, dqk, dv)) return -1;
  const size_t planes = split ? 2 : 1, ldk = round_up(nk, 4);
  if (backward) return (long long)ag_bwd_ws(BH, nq, nk, dqk, dv, (int)planes).total;
  AgWs w;
  for (size_t pl = 0; pl < planes; ++pl) { w.take((size_t)BH * nq * dqk); w.take((size_t)BH * nk * dqk); w.take((size_t)BH * dv * ldk); }
  return (long long)w.off;
}

int attention_global_forward(const float* q, const float* k, const float* v, const float* bias, float* o, float* lse, int BH, int nq, int nk,
                             int dqk, int dv, float scale, int split, float* ws, cudaStream_t st) {
  if (int rc = ag_check(BH, nq, nk, dqk, dv)) return rc;
  B200_REQUIRE(q && k && v && bias && o && lse && ws, "attention_global_forward: null pointer");
  const int dc = ceil_div(std::max(dqk, dv), 32), ldk = round_up(nk, 4), planes = split ? 2 : 1;
  AgWs w;
  float *Qh[2] = {}, *Kh[2] = {}, *Vt[2] = {};
  for (int pl = 0; pl < planes; ++pl) {
    Qh[pl] = ws + w.take((size_t)BH * nq * dqk);
    Kh[pl] = ws + w.take((size_t)BH * nk * dqk);
    Vt[pl] = ws + w.take((size_t)BH * dv * ldk);
  }
  if (int rc = ag_prep(q, BH, nq, dqk, Qh[0], Qh[1], dqk, false, st)) return rc;
  if (int rc = ag_prep(k, BH, nk, dqk, Kh[0], Kh[1], dqk, false, st)) return rc;
  if (int rc = ag_prep(v, BH, dv, nk, Vt[0], Vt[1], ldk, false, st)) return rc;
  AgParams p;
  memset(&p, 0, sizeof(p));
  for (int pl = 0; pl < planes; ++pl) {
    if (int rc = ag_map_rows(&p.res[pl][0], Qh[pl], BH, nq, dqk, kAgBM)) return rc;
    if (int rc = ag_map_rows(&p.item[pl][0][0], Kh[pl], BH, nk, dqk, kAgBN)) return rc;
    if (int rc = ag_map_cols(&p.item[pl][0][1], Vt[pl], BH, nk, dv, ldk, dc)) return rc;
  }
  p.bias = bias; p.out0 = o; p.out1 = lse;
  p.nq = nq; p.nk = nk; p.dqk = dqk; p.dv = dv; p.scale = scale;
  return ag_launch(kAgFwd, p, dc, split != 0, ceil_div(nq, kAgBM), BH, st);
}

int attention_global_rowdot(const float* o, const float* dout, float* D, long long rows, int dv, cudaStream_t st) {
  B200_REQUIRE(rows >= 1 && dv >= 1, "attention_global_rowdot: rows %lld and dv %d must be positive", rows, dv);
  B200_REQUIRE(o && dout && D, "attention_global_rowdot: null pointer");
  attention_global_rowdot_kernel<<<(unsigned)((rows + 255) / 256), 256, 0, st>>>(o, dout, D, rows, dv);
  B200_CHECK_LAUNCH();
  return 0;
}

int attention_global_backward_kv(const float* q, const float* k, const float* v, const float* bias, const float* lse, const float* D,
                                 const float* dout, float* dk, float* dv_, int BH, int nq, int nk, int dqk, int dv, float scale, int split,
                                 float* ws, cudaStream_t st) {
  if (int rc = ag_check(BH, nq, nk, dqk, dv)) return rc;
  B200_REQUIRE(q && k && v && bias && lse && D && dout && dk && dv_ && ws, "attention_global_backward_kv: null pointer");
  return ag_backward_passes(kAgPassKv, q, k, v, bias, lse, D, dout, nullptr, dk, dv_, BH, nq, nk, dqk, dv, scale, split, ws, st);
}

int attention_global_backward_q(const float* q, const float* k, const float* v, const float* bias, const float* lse, const float* D,
                                const float* dout, float* dq, int BH, int nq, int nk, int dqk, int dv, float scale, int split, float* ws,
                                cudaStream_t st) {
  if (int rc = ag_check(BH, nq, nk, dqk, dv)) return rc;
  B200_REQUIRE(q && k && v && bias && lse && D && dout && dq && ws, "attention_global_backward_q: null pointer");
  return ag_backward_passes(kAgPassQ, q, k, v, bias, lse, D, dout, dq, nullptr, nullptr, BH, nq, nk, dqk, dv, scale, split, ws, st);
}

// rowdot, then the kv and q passes on one set of prepared operands; D lives in the workspace
int attention_global_backward(const float* q, const float* k, const float* v, const float* bias, const float* o, const float* lse, const float* dout,
                              float* dq, float* dk, float* dv_, int BH, int nq, int nk, int dqk, int dv, float scale, int split, float* ws,
                              cudaStream_t st) {
  if (int rc = ag_check(BH, nq, nk, dqk, dv)) return rc;
  B200_REQUIRE(q && k && v && bias && o && lse && dout && dq && dk && dv_ && ws, "attention_global_backward: null pointer");
  float* D = ws + ag_bwd_ws(BH, nq, nk, dqk, dv, split ? 2 : 1).D;
  if (int rc = attention_global_rowdot(o, dout, D, (long long)BH * nq, dv, st)) return rc;
  return ag_backward_passes(kAgPassKv | kAgPassQ, q, k, v, bias, lse, D, dout, dq, dk, dv_, BH, nq, nk, dqk, dv, scale, split, ws, st);
}

}  // namespace b200sht
