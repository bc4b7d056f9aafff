// Longitude FFT stage of the SHT (replaces torch.fft.rfft / irfft inside torch_harmonics.RealSHT /
// InverseRealSHT; reference call sites /root/reference/makani/models/common/spectral_convolution.py:239,253 and
// the FFT twin /root/reference/makani/mpu/fft.py:62,109).
//
// A CTA transforms a tile of consecutive latitude rows of one (batch, channel) image with a mixed-radix Stockham FFT (radices up to
// 16 kept in registers, shared memory only for the exchange between stages), truncates to mmax, scales and writes the "latspec"
// layout [m][re/im][row r][k]: the results of one tile for one (m, re/im) are one contiguous 16- or 32-byte piece and the Legendre
// GEMM reads K-major operands straight from it.
//
// Two kernel families share the butterflies (fft_butterfly.cuh):
//   *_ct  : radix plan fixed at compile time (CT_PLANS): one half-length complex FFT per real row, two rows per 64-bit register
//           pair (pr: each operation on both rows), persistent CTAs with register prefetch of the next tile, first stage fused with the
//           global load, last stage of the inverse fused with the store, per-buffer conflict-free shared-memory layouts.
//   *_rt  : any length whose prime factors are <= 13 (runtime plan), two real rows packed into one complex sequence.
//
// The stage / butterfly code is __host__ __device__ so that the same arithmetic is unit-tested on the CPU
// (b200sht_debug_fft_host) without a GPU.
#include "common.cuh"
#include "fft_butterfly.cuh"
#include <cmath>
#include <cstdlib>
#include <vector>

namespace b200sht {

// ------------------------------------------------------------------------------------------------ plan
static const int kRadices[] = {16, 15, 13, 12, 11, 10, 9, 8, 7, 6, 5, 4, 3, 2};

static void plan_search(int n, int max_r, int* cur, int depth, int* best, int* best_len, int* best_sum) {
  if (n == 1) {
    int sum = 0;
    for (int i = 0; i < depth; ++i) sum += cur[i];
    if (depth < *best_len || (depth == *best_len && sum < *best_sum)) {
      *best_len = depth; *best_sum = sum;
      for (int i = 0; i < depth; ++i) best[i] = cur[i];
    }
    return;
  }
  if (depth >= 12 || depth + 1 > *best_len) return;
  for (int r : kRadices) {
    if (r > max_r || n % r) continue;
    cur[depth] = r;
    plan_search(n / r, r, cur, depth + 1, best, best_len, best_sum);
  }
}

// fewest stages, then smallest radix sum (balanced stages); radices in non-increasing order
bool make_fft_plan(int N, FftPlan* p) {
  p->N = N;
  p->nstages = 0;
  if (N < 2) return false;
  int n = N;
  for (int f : {2, 3, 5, 7, 11, 13})
    while (n % f == 0) n /= f;
  if (n != 1) return false;
  int cur[20], best[20], best_len = 13, best_sum = 1 << 30;
  plan_search(N, 16, cur, 0, best, &best_len, &best_sum);
  if (best_len > 12) return false;
  p->nstages = best_len;
  for (int i = 0; i < best_len; ++i) p->radix[i] = best[i];
  return true;
}

// butterflies: fft_butterfly.cuh (generic over one complex value / the packed values of two rows)

// One Stockham butterfly (index j of N/R) of a stage with sub-transform length Ns:  in -> out  (runtime plan / host)
template <int R>
HD void stage_butterfly(const float2* in, float2* out, const float2* tw, int N, int Ns, int j) {
  const int k = j % Ns;
  const int stride = N / R;
  const int tstep = k * (N / (Ns * R));
  float2 v[R];
#pragma unroll
  for (int r = 0; r < R; ++r) {
    float2 a = in[j + r * stride];
    if (r > 0 && k > 0) a = cmul(a, tw[r * tstep]);
    v[r] = a;
  }
  Butterfly<R>::run(v, tw, N);
  const int j0 = (j - k) * R + k;
#pragma unroll
  for (int r = 0; r < R; ++r) out[j0 + r * Ns] = v[r];
}

#define B200_RADIX_SWITCH(R, CALL)      \
  switch (R) {                          \
    case 2: { CALL(2); } break;         \
    case 3: { CALL(3); } break;         \
    case 4: { CALL(4); } break;         \
    case 5: { CALL(5); } break;         \
    case 6: { CALL(6); } break;         \
    case 7: { CALL(7); } break;         \
    case 8: { CALL(8); } break;         \
    case 9: { CALL(9); } break;         \
    case 10: { CALL(10); } break;       \
    case 11: { CALL(11); } break;       \
    case 12: { CALL(12); } break;       \
    case 13: { CALL(13); } break;       \
    case 15: { CALL(15); } break;       \
    default: { CALL(16); } break;       \
  }

// split the FFT of z = a + i b (a, b real rows) into the half spectra of a and b at mode m
HD void split_pair(float2 Z, float2 Zm /* = FFT(z)[(N-m)%N] */, float2& A, float2& Bq) {
  A = make_float2(0.5f * (Z.x + Zm.x), 0.5f * (Z.y - Zm.y));
  Bq = make_float2(0.5f * (Z.y + Zm.y), -0.5f * (Z.x - Zm.x));
}

struct FftParams {
  FftPlan fp;
  int nlat, nlon, mmax, kp;
  int R;            // B*C image rows
  int C;            // channels (bias index = r % C)
  int scale_mode;
  int round_tf32;   // analysis output feeds a TF32 tensor-core GEMM: round to nearest TF32 here
  const float2* twiddle;
  const float* rowscale;
  const float* bias;
};

__device__ __forceinline__ float ld_as_float(const float* p) { return __ldg(p); }
__device__ __forceinline__ float ld_as_float(const __nv_bfloat16* p) { return __bfloat162float(*p); }
__device__ __forceinline__ void st_from_float(float* p, float v) { *p = v; }
__device__ __forceinline__ void st_from_float(__nv_bfloat16* p, float v) { *p = __float2bfloat16_rn(v); }

__device__ __forceinline__ float finish_analysis(const FftParams& prm, float v) { return prm.round_tf32 ? tf32_rn(v) : v; }

__device__ __forceinline__ float mode_scale_analysis(const FftParams& prm, int m, int k) {
  if (k >= prm.nlat) return 0.f;  // rows in the k padding are written as exact zeros
  if (prm.scale_mode == 0) return prm.rowscale[k];
  return (m == 0 || 2 * m == prm.nlon) ? 1.f : 2.f;
}

// =========================================================================================== compile-time plans
// Real rows of even length N are transformed through ONE complex FFT of length H = N/2 each (z[n] = x[2n] + i x[2n+1], loaded
// as one 4- or 8-byte word), followed by the split  X[m] = E[m] + W_N^m O[m],  E = (Z[m] + conj Z[H-m])/2,
// O = (Z[m] - conj Z[H-m])/(2i).  A CTA owns ROWS consecutive latitude rows; the threads form GROUPS groups of TPG threads, a
// group owns RPT = ROWS/GROUPS rows.  One thread carries the same butterfly index of TWO adjacent rows in the two halves of 64-bit
// registers (value type cpair): every arithmetic operation acts on both rows, so the index computations
// and shared-memory addressing are shared by two rows.
//
// Exchange buffers (shared memory, Stockham: stage s reads one buffer and writes the other).  A buffer holds PROWS = ROWS/2 row
// pairs as two planes of 8-byte elements (real parts of both rows / imaginary parts of both rows), so every access is an 8-byte
// access by half warps and 16 lanes are conflict-free iff their slots are distinct modulo 16.  Element index -> slot:
//   LaySkew   slot = i + i/16.  For the buffer the first stage writes (lane j stores elements j*R0 + r: stride R0, a power of two
//             <= 16): 16 consecutive lanes land on 16 distinct slots mod 16, and runs of 16 consecutive elements that start at a
//             multiple of 16 stay contiguous.
//   LayBlock  slot = i + PAD * (i / BLK), BLK = R0*R1.  For the buffer the second stage writes (runs of Ns = R0 consecutive elements,
//             one run per BLK): PAD spreads the runs of one half warp over distinct slots mod 16; consecutive elements inside a
//             block stay contiguous (all loads of the following stage).
//   LayId     slot = i.  The last stage of the analysis writes runs of consecutive elements and the split pass reads runs (ascending
//             m, descending H-m): the memory of the first buffer is reused with the identity layout for them.
// (scripts/smem_sim.py models the wavefronts of every access of a plan; the former single skew i + i/R0 cost 1.77x the ideal
// wavefront count for the 1440-point plan, these two layouts 1.2x.)
struct LayId {
  __host__ __device__ static constexpr int at(int i) { return i; }
};
struct LaySkew {
  __host__ __device__ static constexpr int at(int i) { return i + (i >> 4); }
  __host__ __device__ static constexpr int size(int H) { return H + (H >> 4) + 1; }
};
template <int BLK, int PAD>
struct LayBlock {
  __host__ __device__ static constexpr int at(int i) { return i + PAD * (i / BLK); }
  __host__ __device__ static constexpr int size(int H) { return H + PAD * ((H + BLK - 1) / BLK); }
};
__host__ __device__ constexpr int ct_block_pad(int R0, int R1) {
  if (R0 >= 16) return 0;
  int p = 0;
  while ((R0 * R1 + p) % 16 != R0 % 16) ++p;
  return p;
}

// view of (some rows of) one exchange buffer
template <int PLANE, class LAY>
struct PairBuf {
  typedef LAY layout;
  pr* p;
  __device__ __forceinline__ PairBuf operator+(int i) const { return PairBuf{p + i}; }
  __device__ __forceinline__ cpair ld(int slot) const { cpair r; r.x = p[slot]; r.y = p[slot + PLANE]; return r; }
  __device__ __forceinline__ void st(int slot, const cpair& v) const { p[slot] = v.x; p[slot + PLANE] = v.y; }
};

// geometry shared by the kernels and the launcher
template <int ROWS, int R0, int R1, int R2>
struct CtGeom {
  static constexpr int H = R0 * R1 * R2, PROWS = ROWS / 2;
  typedef LaySkew LayS;
  typedef LayBlock<R0 * R1, ct_block_pad(R0, R1)> LayB;
  static constexpr int BSS = LayS::size(H), BSB = LayB::size(H);           // row-pair strides (8-byte elements)
  static constexpr int PLANE_S = PROWS * BSS, PLANE_B = PROWS * BSB;
  static constexpr int TW = (R1 * R0 + (R2 > 1 ? R2 * R0 * R1 : 0) + 1) & ~1;   // stage twiddles (float2), even count
  static constexpr size_t smem_fixed = 8 * ((size_t)TW + 2 * PLANE_S + 2 * PLANE_B);
  typedef PairBuf<PLANE_S, LayS> BufS;
  typedef PairBuf<PLANE_B, LayB> BufB;
  typedef PairBuf<PLANE_S, LayId> BufI;   // the memory of BufS under the identity layout
};

// stage of a compile-time plan: buffer `in` -> buffer `out`, row pairs row0 .. row0 + NPT - 1 of this thread's group
template <class PI, class PO, int H, int R, int Ns, int TPG, int NPT>
__device__ __forceinline__ void ct_stage(PI in, PO out, const float2* tws /* [R][Ns]: W^(r k H/(Ns R)) */, int in_stride, int out_stride, int t, int row0) {
  constexpr int NB = H / R;
  for (int j = t; j < NB; j += TPG) {
    const int k = j % Ns;
    const int j0 = (j - k) * R + k;
    float2 w[R];
    int si[R], di[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      si[r] = PI::layout::at(j + r * NB);
      di[r] = PO::layout::at(j0 + r * Ns);
      if (Ns > 1 && r > 0) w[r] = tws[r * Ns + k];   // consecutive threads -> consecutive k: conflict-free
    }
#pragma unroll
    for (int q = 0; q < NPT; ++q) {
      const PI src = in + (row0 + q) * in_stride;
      const PO dst = out + (row0 + q) * out_stride;
      cpair v[R];
#pragma unroll
      for (int r = 0; r < R; ++r) {
        cpair a = src.ld(si[r]);
        if (Ns > 1 && r > 0) a = cmulw(a, w[r]);
        v[r] = a;
      }
      Butterfly<R>::run(v, nullptr, H);
#pragma unroll
      for (int r = 0; r < R; ++r) dst.st(di[r], v[r]);
    }
  }
}

// per-stage twiddle tables in shared memory: tw1 [R1][R0] for the second stage (Ns = R0), tw2 [R2][R0*R1] for the third (Ns = R0*R1).
// W_H^e = W_N^(2e) comes from the plan's length-N table.
template <int R0, int R1, int R2>
__device__ __forceinline__ void ct_build_twiddles(float2* tw1, float2* tw2, const float2* __restrict__ twN, int nthreads) {
  constexpr int H = R0 * R1 * R2;
  for (int i = threadIdx.x; i < R1 * R0; i += nthreads) {
    const int r = i / R0, k = i - r * R0;
    tw1[i] = twN[2 * (r * k * (H / (R0 * R1)))];
  }
  if (R2 > 1)
    for (int i = threadIdx.x; i < R2 * R0 * R1; i += nthreads) {
      const int r = i / (R0 * R1), k = i - r * (R0 * R1);
      tw2[i] = twN[2 * (r * k)];
    }
}

__device__ __forceinline__ void st_pair(float* p, float a, float b) { *reinterpret_cast<float2*>(p) = make_float2(a, b); }
__device__ __forceinline__ void st_pair(__nv_bfloat16* p, float a, float b) {
  *reinterpret_cast<__nv_bfloat162*>(p) = __floats2bfloat162_rn(a, b);
}

// raw element pair as loaded from global memory (converted to float2 only when stage 0 consumes it)
template <typename T> struct RawPair;
template <> struct RawPair<float> {
  float2 v;
  __device__ __forceinline__ void load(const float* p) { v = __ldg(reinterpret_cast<const float2*>(p)); }
  __device__ __forceinline__ void zero() { v = make_float2(0.f, 0.f); }
  __device__ __forceinline__ float2 get() const { return v; }
};
template <> struct RawPair<__nv_bfloat16> {
  unsigned int v;
  __device__ __forceinline__ void load(const __nv_bfloat16* p) { v = __ldg(reinterpret_cast<const unsigned int*>(p)); }
  __device__ __forceinline__ void zero() { v = 0u; }
  __device__ __forceinline__ float2 get() const { return make_float2(__uint_as_float(v << 16), __uint_as_float(v & 0xffff0000u)); }
};

// barrier among the TPG threads of one row group (the stages between two block-wide passes touch only the group's own rows)
// (immediate barrier ids: with a register id ptxas reserves all 16 named barriers of the CTA, which caps the CTAs per SM)
template <int TPG, int GROUPS>
__device__ __forceinline__ void group_sync(int grp) {
  static_assert(GROUPS <= 4, "one named barrier per group");
  if (GROUPS == 1 || grp == 0) asm volatile("bar.sync 1, %0;" ::"n"(TPG) : "memory");
  else if (grp == 1) asm volatile("bar.sync 2, %0;" ::"n"(TPG) : "memory");
  else if (grp == 2) asm volatile("bar.sync 3, %0;" ::"n"(TPG) : "memory");
  else asm volatile("bar.sync 4, %0;" ::"n"(TPG) : "memory");
}

__device__ __forceinline__ cpair pack_rows(float2 a, float2 b) { return mk<cpair>(make_pr(a.x, b.x), make_pr(a.y, b.y)); }

// walk of the persistent CTA over the tiles (k tile, image r) without a division per tile
struct TileWalk {
  int kt, r, step_k, step_r, ntx;
  __device__ __forceinline__ TileWalk(int ntx_) : ntx(ntx_) {
    kt = blockIdx.x % ntx; r = blockIdx.x / ntx;
    step_k = gridDim.x % ntx; step_r = gridDim.x / ntx;
  }
  __device__ __forceinline__ void next() {
    kt += step_k; r += step_r;
    if (kt >= ntx) { kt -= ntx; ++r; }
  }
};

// x [R][nlat][nlon] -> latspec [mmax][2][R][kp]        plan (R0, R1, R2) for H = nlon / 2, R2 == 1 for two stages.
// Persistent CTAs walk the (row group, image) tiles; the stage-0 operands of the NEXT tile are loaded into registers right after
// stage 0 of the current one, so the HBM latency is hidden behind stages 1, 2 and the store pass.
template <typename T, int ROWS, int GROUPS, int TPG, int R0, int R1, int R2, int MINB>
__global__ void __launch_bounds__(GROUPS * TPG, MINB) fft_analysis_ct_kernel(const T* __restrict__ x, float* __restrict__ X, const FftParams prm) {
  typedef CtGeom<ROWS, R0, R1, R2> G;
  typedef typename G::BufS BufS;
  typedef typename G::BufB BufB;
  constexpr int H = G::H, N = 2 * H;
  constexpr int THREADS = GROUPS * TPG, RPT = ROWS / GROUPS, PPT = RPT / 2;
  constexpr int NB0 = H / R0;
  constexpr int QUADS = ROWS / 4;
  static_assert(ROWS % GROUPS == 0 && RPT % 2 == 0 && ROWS % 4 == 0, "row grouping");
  static_assert(NB0 <= TPG, "one stage-0 butterfly index per thread (register prefetch)");
  static_assert(THREADS % (16 * QUADS) == 0, "split pass: 16 consecutive orders of one quad per half warp");
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float2* tw1 = reinterpret_cast<float2*>(smem_raw);
  float2* tw2 = tw1 + R1 * R0;
  const BufS bS{reinterpret_cast<pr*>(tw1 + G::TW)};     // written by stage 0 (and stage 2)
  const BufB bB{bS.p + 2 * G::PLANE_S};                  // written by stage 1
  float2* twm = reinterpret_cast<float2*>(bB.p + 2 * G::PLANE_B);   // W_N^m, m < mmax (split pass)
  const int grp = threadIdx.x / TPG, t = threadIdx.x - grp * TPG;
  const int row0 = grp * RPT, prow0 = grp * PPT;
  const int ntx = (prm.kp + ROWS - 1) / ROWS;
  ct_build_twiddles<R0, R1, R2>(tw1, tw2, prm.twiddle, THREADS);
  for (int i = threadIdx.x; i < prm.mmax; i += THREADS) twm[i] = prm.twiddle[i];

  RawPair<T> raw[RPT][R0];
  auto load_tile = [&](int kt, int r) {
    const int k0 = kt * ROWS;
    const T* base = x + ((size_t)r * prm.nlat + k0) * N;
#pragma unroll
    for (int q = 0; q < RPT; ++q) {
      const int row = row0 + q;
      const bool valid = (t < NB0) && (k0 + row) < prm.nlat;
      const T* rp = base + (size_t)row * N + 2 * t;
#pragma unroll
      for (int rr = 0; rr < R0; ++rr) {
        if (valid) raw[q][rr].load(rp + 2 * rr * NB0);
        else raw[q][rr].zero();
      }
    }
  };
  TileWalk tw(ntx);
  if (tw.r < prm.R) load_tile(tw.kt, tw.r);
  __syncthreads();   // twiddle tables

  // split pass ownership: a half warp = 16 consecutive orders m of one quad of rows (conflict-free 8-byte shared loads)
  const int qd = (threadIdx.x / 16) % QUADS;
  const int m_first = (threadIdx.x % 16) + 16 * (threadIdx.x / (16 * QUADS));
  const size_t mstride = (size_t)2 * prm.R * prm.kp, pstride = (size_t)prm.R * prm.kp;
  const bool rnd = prm.round_tf32 != 0;

  while (tw.r < prm.R) {
    const int k0 = tw.kt * ROWS, r = tw.r;
    const int kq = k0 + qd * 4;
    // quadrature weights of this thread's quad of rows (consumed by the split pass at the end of the tile; zero in the padding)
    float4 rs4 = make_float4(0.f, 0.f, 0.f, 0.f);
    if (prm.scale_mode == 0 && kq < prm.kp) rs4 = __ldg(reinterpret_cast<const float4*>(prm.rowscale + kq));
    // ---- stage 0 from the prefetched registers
    if (t < NB0) {
      int di[R0];
#pragma unroll
      for (int rr = 0; rr < R0; ++rr) di[rr] = G::LayS::at(t * R0 + rr);
#pragma unroll
      for (int p = 0; p < PPT; ++p) {
        cpair v[R0];
#pragma unroll
        for (int rr = 0; rr < R0; ++rr) v[rr] = pack_rows(raw[2 * p][rr].get(), raw[2 * p + 1][rr].get());
        Butterfly<R0>::run(v, nullptr, H);
        const BufS dst = bS + (prow0 + p) * G::BSS;
#pragma unroll
        for (int rr = 0; rr < R0; ++rr) dst.st(di[rr], v[rr]);
      }
    }
    tw.next();
    if (tw.r < prm.R) load_tile(tw.kt, tw.r);   // in flight until the next iteration
    group_sync<TPG, GROUPS>(grp);
    ct_stage<BufS, BufB, H, R1, R0, TPG, PPT>(bS, bB, tw1, G::BSS, G::BSB, t, prow0);
    if (R2 > 1) {
      group_sync<TPG, GROUPS>(grp);
      ct_stage<BufB, typename G::BufI, H, (R2 > 1 ? R2 : 2), R0 * R1, TPG, PPT>(bB, typename G::BufI{bS.p}, tw2, G::BSB, G::BSS, t, prow0);
    }
    __syncthreads();   // the split pass reads the rows of every group
    // ---- split + truncate + scale + store: X[m] = (Z[m] + conj Z[H-m]) / 2 + W_N^m (Z[m] - conj Z[H-m]) / (2i), two 16-byte stores
    auto split = [&](auto res, int stride) {
      typedef typename decltype(res)::layout L;
      pr rsc[2];   // per-row factor / 2: quadrature weight (SHT forward) or 1 (adjoint of irfft), 0 in the latitude padding
      if (prm.scale_mode == 0) {
        rsc[0] = make_pr(0.5f * rs4.x, 0.5f * rs4.y);
        rsc[1] = make_pr(0.5f * rs4.z, 0.5f * rs4.w);
      } else {
        rsc[0] = make_pr(kq + 0 < prm.nlat ? 0.5f : 0.f, kq + 1 < prm.nlat ? 0.5f : 0.f);
        rsc[1] = make_pr(kq + 2 < prm.nlat ? 0.5f : 0.f, kq + 3 < prm.nlat ? 0.5f : 0.f);
      }
      const auto rb = res + (qd * 2) * stride;
      float* xbase = X + (size_t)r * prm.kp + kq;
      for (int m = m_first; m < prm.mmax; m += THREADS / QUADS) {
        const float2 wm = twm[m];                                 // W_N^m
        const int im = L::at(m == H ? 0 : m), ic = L::at((m == 0 || m == H) ? 0 : H - m);
        const float msc = (prm.scale_mode == 1 && !(m == 0 || 2 * m == N)) ? 2.f : 1.f;
        pr re[2], imv[2];
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const cpair Z = rb.ld(i * stride + im), Zc = rb.ld(i * stride + ic);
          const pr ex = Z.x + Zc.x, ey = Z.y - Zc.y;                            // 2 E
          const cpair od = mk<cpair>(Z.y + Zc.y, Zc.x - Z.x);                    // 2 O = (Z - conj Zc) / i
          const cpair wo = cmulw(od, wm);
          const pr sc = rmul(rsc[i], msc);
          re[i] = (ex + wo.x) * sc;
          imv[i] = (ey + wo.y) * sc;
        }
        float4 o_re = make_float4(re[0].v.x, re[0].v.y, re[1].v.x, re[1].v.y);
        float4 o_im = make_float4(imv[0].v.x, imv[0].v.y, imv[1].v.x, imv[1].v.y);
        if (rnd) {
          o_re = make_float4(tf32_rn(o_re.x), tf32_rn(o_re.y), tf32_rn(o_re.z), tf32_rn(o_re.w));
          o_im = make_float4(tf32_rn(o_im.x), tf32_rn(o_im.y), tf32_rn(o_im.z), tf32_rn(o_im.w));
        }
        if (kq < prm.kp) {
          float* dst = xbase + (size_t)m * mstride;
          *reinterpret_cast<float4*>(dst) = o_re;
          *reinterpret_cast<float4*>(dst + pstride) = o_im;
        }
      }
    };
    if constexpr (R2 > 1) split(typename G::BufI{bS.p}, G::BSS);
    else split(bB, G::BSB);
    __syncthreads();   // the buffers are reused by the next tile
  }
}

// latspec [mmax][2][R][kp] -> y [R][nlat][nlon]   (persistent, with register prefetch of the next tile's spectrum)
// TRUNC: 2 * mmax <= H, i.e. the partner X[H-q] of every retained order is beyond the truncation (zero): it is neither loaded nor multiplied.
template <typename T, int ROWS, int GROUPS, int TPG, int R0, int R1, int R2, int MINB, bool TRUNC>
__global__ void __launch_bounds__(GROUPS * TPG, MINB) fft_synthesis_ct_kernel(const float* __restrict__ Zs, T* __restrict__ y, const FftParams prm) {
  typedef CtGeom<ROWS, R0, R1, R2> G;
  typedef typename G::BufS BufS;
  typedef typename G::BufB BufB;
  constexpr int H = G::H, N = 2 * H;
  constexpr int THREADS = GROUPS * TPG, RPT = ROWS / GROUPS, PPT = RPT / 2;
  constexpr int RL = (R2 > 1) ? R2 : R1;       // radix of the last stage (fused with the store)
  constexpr int NsL = H / RL;
  constexpr int QUADS = ROWS / 4;
  constexpr int NQ16 = (H / 2 + 1 + 15) / 16;              // groups of 16 spectrum indices q in [0, H/2]
  constexpr int NITEMS = NQ16 * 16 * QUADS;                // item = (q, quad of 4 rows)
  constexpr int IPT = (NITEMS + THREADS - 1) / THREADS;    // spectrum-build items per thread
  static_assert(RPT % 2 == 0 && ROWS % 4 == 0, "row grouping");
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float2* tw1 = reinterpret_cast<float2*>(smem_raw);
  float2* tw2 = tw1 + R1 * R0;
  const BufS bS{reinterpret_cast<pr*>(tw1 + G::TW)};     // written by stage 0 (stride-R0 stores)
  const BufB bB{bS.p + 2 * G::PLANE_S};                  // written by the spectrum build and by stage 1
  float2* twm = reinterpret_cast<float2*>(bB.p + 2 * G::PLANE_B);   // W_N^q, q < mmax (spectrum build)
  const int grp = threadIdx.x / TPG, t = threadIdx.x - grp * TPG;
  const int row0 = grp * RPT, prow0 = grp * PPT;
  const int mmax = prm.mmax;
  const int ntx = (prm.kp + ROWS - 1) / ROWS;
  ct_build_twiddles<R0, R1, R2>(tw1, tw2, prm.twiddle, THREADS);
  for (int i = threadIdx.x; i < prm.mmax; i += THREADS) twm[i] = prm.twiddle[i];
  const float2* twL = (R2 > 1) ? tw2 : tw1;   // table of the last stage: [RL][NsL]

  // item e -> (q, quad): a half warp owns 16 consecutive q of one quad.  X[q] and X[H-q] of 4 rows (re, im) = four 16-byte loads
  float4 pa_r[IPT], pa_i[IPT], pb_r[IPT], pb_i[IPT];
  auto item_q = [](int e) { return (e % 16) + 16 * (e / (16 * QUADS)); };
  auto item_quad = [](int e) { return (e / 16) % QUADS; };
  auto load_tile = [&](int kt, int r) {
    const int k0 = kt * ROWS;
#pragma unroll
    for (int it = 0; it < IPT; ++it) {
      const int e = threadIdx.x + it * THREADS;
      const int qd = item_quad(e), q = item_q(e), q2 = H - q;
      const int k = k0 + qd * 4;
      const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
      pa_r[it] = z; pa_i[it] = z;
      if (!TRUNC) { pb_r[it] = z; pb_i[it] = z; }
      if (e < NITEMS && q <= H / 2 && k < prm.kp) {
        if (q < mmax) {
          const float* src = Zs + (((size_t)q * 2) * prm.R + r) * prm.kp + k;
          pa_r[it] = __ldg(reinterpret_cast<const float4*>(src));
          pa_i[it] = __ldg(reinterpret_cast<const float4*>(src + (size_t)prm.R * prm.kp));
        }
        if (!TRUNC && q2 < mmax) {
          const float* src = Zs + (((size_t)q2 * 2) * prm.R + r) * prm.kp + k;
          pb_r[it] = __ldg(reinterpret_cast<const float4*>(src));
          pb_i[it] = __ldg(reinterpret_cast<const float4*>(src + (size_t)prm.R * prm.kp));
        }
      }
    }
  };
  TileWalk tw(ntx);
  if (tw.r < prm.R) load_tile(tw.kt, tw.r);
  __syncthreads();

  while (tw.r < prm.R) {
    const int k0 = tw.kt * ROWS, r = tw.r;
    // per-row output factors of this thread's rows and the channel bias (consumed by the fused store at the end of the tile)
    float rsv[RPT];
#pragma unroll
    for (int i = 0; i < RPT; ++i) rsv[i] = (prm.scale_mode == 1 && k0 + row0 + i < prm.nlat) ? __ldg(prm.rowscale + k0 + row0 + i) : 1.f;
    const float bias = prm.bias ? __ldg(prm.bias + r % prm.C) : 0.f;
    // ---- build Z'[q] = (X[q] + conj X[H-q]) + i (X[q] - conj X[H-q]) W_N^-q for q in [0, H), stored swapped (im, re).
    //      With A = X[q], B = X[H-q]:  Z'[q] = s + i d conj(w),  Z'[H-q] = conj(s) + i conj(d) w  (W_N^(H-q) = -conj W_N^q).
    //      Rows beyond nlat carry whatever the padding holds; they are never stored.
#pragma unroll
    for (int it = 0; it < IPT; ++it) {
      const int e = threadIdx.x + it * THREADS;
      const int qd = item_quad(e), q = item_q(e);
      if (e >= NITEMS || q > H / 2) continue;
      const int q2 = H - q;                                    // partner index (q2 == H for q == 0)
      const int s1 = G::LayB::at(q), s2 = G::LayB::at(q2 == H ? 0 : q2);
      if (q >= mmax) {   // X[q] = X[H-q] = 0 (truncated spectrum): Z'[q] = Z'[H-q] = 0
        const cpair zero = mk<cpair>(make_pr(0.f, 0.f), make_pr(0.f, 0.f));
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const BufB rowp = bB + (qd * 2 + i) * G::BSB;
          rowp.st(s1, zero);
          if (q2 != q) rowp.st(s2, zero);
        }
        continue;
      }
      const bool a_self = (q == 0), b_self = (q2 == H);        // DC and Nyquist: imaginary part ignored, no halving
      const float ha = (prm.scale_mode == 1 && !a_self) ? 0.5f : 1.f;
      const float hb = (prm.scale_mode == 1 && !b_self) ? 0.5f : 1.f;
      const float2 wq = twm[q];                                 // W_N^q
      const float ar[4] = {pa_r[it].x, pa_r[it].y, pa_r[it].z, pa_r[it].w}, ai[4] = {pa_i[it].x, pa_i[it].y, pa_i[it].z, pa_i[it].w};
      if (TRUNC) {
        // B = 0:  Z'[q] = A + i A conj(w),  Z'[H-q] = conj(A) + i conj(A) w, stored (im, re):
        //   Z'[q]   = (Ai (1 + wy) + Ar wx,  Ar (1 + wy) - Ai wx)      Z'[H-q] = (Ar wx - Ai (1 - wy),  Ar (1 - wy) + Ai wx)
        const float wp = 1.f + wq.y, wn = 1.f - wq.y;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          pr Ar = make_pr(ar[2 * i], ar[2 * i + 1]), Ai = a_self ? make_pr(0.f, 0.f) : make_pr(ai[2 * i], ai[2 * i + 1]);
          if (prm.scale_mode == 1) { Ar = rmul(Ar, ha); Ai = rmul(Ai, ha); }
          const BufB rowp = bB + (qd * 2 + i) * G::BSB;
          rowp.st(s1, mk<cpair>(rfma(Ai, wp, rmul(Ar, wq.x)), rfma(Ai, -wq.x, rmul(Ar, wp))));
          if (q != 0 && q2 != q) rowp.st(s2, mk<cpair>(rfma(Ai, -wn, rmul(Ar, wq.x)), rfma(Ai, wq.x, rmul(Ar, wn))));
        }
        continue;
      }
      const float br[4] = {pb_r[it].x, pb_r[it].y, pb_r[it].z, pb_r[it].w}, bi[4] = {pb_i[it].x, pb_i[it].y, pb_i[it].z, pb_i[it].w};
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        pr Ar = make_pr(ar[2 * i], ar[2 * i + 1]), Ai = a_self ? make_pr(0.f, 0.f) : make_pr(ai[2 * i], ai[2 * i + 1]);
        pr Br = make_pr(br[2 * i], br[2 * i + 1]), Bi = b_self ? make_pr(0.f, 0.f) : make_pr(bi[2 * i], bi[2 * i + 1]);
        if (prm.scale_mode == 1) { Ar = rmul(Ar, ha); Ai = rmul(Ai, ha); Br = rmul(Br, hb); Bi = rmul(Bi, hb); }
        const pr sr = Ar + Br, si = Ai - Bi;              // s = A + conj B
        const pr dr = Ar - Br, di = Ai + Bi;              // d = A - conj B
        const BufB rowp = bB + (qd * 2 + i) * G::BSB;
        // t = d conj(w) = (dr wx + di wy, di wx - dr wy);  Z'[q] = (sr - t.y, si + t.x), stored (im, re)
        rowp.st(s1, mk<cpair>(rfma(di, wq.y, rfma(dr, wq.x, si)), rfma(dr, wq.y, rfma(di, -wq.x, sr))));
        if (q != 0 && q2 != q) {
          // conj(d) w = (dr wx + di wy, dr wy - di wx);  Z'[H-q] = (sr - (dr wy - di wx), -si + (dr wx + di wy)), stored (im, re)
          const pr nsi = Bi - Ai;
          rowp.st(s2, mk<cpair>(rfma(di, wq.y, rfma(dr, wq.x, nsi)), rfma(dr, -wq.y, rfma(di, wq.x, sr))));
        }
      }
    }
    tw.next();
    if (tw.r < prm.R) load_tile(tw.kt, tw.r);   // in flight until the next iteration
    __syncthreads();   // the spectrum build wrote the rows of every group
    ct_stage<BufB, BufS, H, R0, 1, TPG, PPT>(bB, bS, nullptr, G::BSB, G::BSS, t, prow0);
    group_sync<TPG, GROUPS>(grp);
    if (R2 > 1) {
      ct_stage<BufS, BufB, H, R1, R0, TPG, PPT>(bS, bB, tw1, G::BSS, G::BSB, t, prow0);
      group_sync<TPG, GROUPS>(grp);
    }
    // ---- last stage fused with the store: butterfly j yields z[e], e = j + rr * NsL, (x[2e], x[2e+1]) = (Im, Re) of the swapped result
    auto last = [&](auto src, int stride) {
      typedef typename decltype(src)::layout L;
      T* base = y + ((size_t)r * prm.nlat + k0) * N;
      const pr bias2 = make_pr(bias, bias);
      for (int j = t; j < NsL; j += TPG) {
        float2 w[RL];
        int si[RL];
#pragma unroll
        for (int rr = 0; rr < RL; ++rr) {
          si[rr] = L::at(j + rr * NsL);
          if (rr > 0) w[rr] = twL[rr * NsL + j];   // k = j
        }
#pragma unroll
        for (int p = 0; p < PPT; ++p) {
          const int rowa = row0 + 2 * p, rowb = rowa + 1;
          const auto sp = src + (prow0 + p) * stride;
          cpair v[RL];
#pragma unroll
          for (int rr = 0; rr < RL; ++rr) {
            cpair a = sp.ld(si[rr]);
            if (rr > 0) a = cmulw(a, w[rr]);
            v[rr] = a;
          }
          Butterfly<RL>::run(v, nullptr, H);
          const bool va = (k0 + rowa) < prm.nlat, vb = (k0 + rowb) < prm.nlat;
          const pr sc = make_pr(rsv[2 * p], rsv[2 * p + 1]);
          T* rpa = base + (size_t)rowa * N + 2 * j;
          T* rpb = rpa + N;
#pragma unroll
          for (int rr = 0; rr < RL; ++rr) {
            const pr o0 = rfma(v[rr].y, sc, bias2), o1 = rfma(v[rr].x, sc, bias2);
            if (va) st_pair(rpa + 2 * rr * NsL, o0.v.x, o1.v.x);
            if (vb) st_pair(rpb + 2 * rr * NsL, o0.v.y, o1.v.y);
          }
        }
      }
    };
    if constexpr (R2 > 1) last(bB, G::BSB);
    else last(bS, G::BSS);
    __syncthreads();   // the buffers are reused by the next tile
  }
}

// Hermitian-extend the truncated half spectra of rows a = k0+2q, b = a+1 into V = Za + i Zb, stored with real/imag swapped
// (inverse FFT == swap o forward FFT o swap); `IDX` maps a spectrum index to its (possibly skewed) buffer slot.
template <class IDX>
__device__ __forceinline__ void fill_spectrum(const float* __restrict__ Zs, float2* b0, int bufstride, int pairs, int nthreads, const FftParams& prm,
                                              int k0, int r, IDX idx) {
  const int N = prm.nlon, mmax = prm.mmax;
  {
    const int lo = mmax, span = N - 2 * mmax + 1;  // untouched middle of the spectrum: indices [mmax, N - mmax]
    if (span > 0)
      for (int e = threadIdx.x; e < pairs * span; e += nthreads) {
        const int q = e / span, i = e - q * span;
        b0[q * bufstride + idx(lo + i)] = make_float2(0.f, 0.f);
      }
  }
  for (int e = threadIdx.x; e < mmax * pairs; e += nthreads) {
    const int q = e % pairs, m = e / pairs;
    const int ka = k0 + 2 * q;
    float2 re2 = make_float2(0.f, 0.f), im2 = re2;
    if (ka < prm.kp) {  // kp is a multiple of 8 and ka is even: ka + 1 < kp as well
      re2 = *reinterpret_cast<const float2*>(Zs + (((size_t)m * 2 + 0) * prm.R + r) * prm.kp + ka);
      im2 = *reinterpret_cast<const float2*>(Zs + (((size_t)m * 2 + 1) * prm.R + r) * prm.kp + ka);
    }
    float ar = re2.x, br = re2.y, ai = im2.x, bi = im2.y;
    if (ka >= prm.nlat) { ar = 0.f; ai = 0.f; }
    if (ka + 1 >= prm.nlat) { br = 0.f; bi = 0.f; }
    const bool self_conj = (m == 0) || (2 * m == N);
    if (self_conj) { ai = 0.f; bi = 0.f; }
    if (prm.scale_mode == 1 && !self_conj) { ar *= 0.5f; ai *= 0.5f; br *= 0.5f; bi *= 0.5f; }
    // V[m] = (ar - bi) + i (ai + br);  V[N-m] = (ar + bi) + i (br - ai)   -- stored swapped (y, x)
    b0[q * bufstride + idx(m)] = make_float2(ai + br, ar - bi);
    if (!self_conj) b0[q * bufstride + idx(N - m)] = make_float2(br - ai, ar + bi);
  }
}

// ================================================================================================ runtime plans
constexpr int kFftThreads = 256;

template <int R>
__device__ __forceinline__ void run_stage(const float2* in, float2* out, const float2* tw, int N, int Ns, int pairs, int bufstride) {
  const int nb = N / R;
  for (int w = threadIdx.x; w < pairs * nb; w += kFftThreads) {
    const int q = w / nb, j = w - q * nb;
    stage_butterfly<R>(in + q * bufstride, out + q * bufstride, tw, N, Ns, j);
  }
}

// runs all stages; returns pointer to the buffer holding the result
__device__ __forceinline__ float2* run_fft(float2* b0, float2* b1, const float2* tw, const FftPlan& fp, int pairs, int bufstride) {
  float2* in = b0;
  float2* out = b1;
  int Ns = 1;
  const int N = fp.N;
  for (int s = 0; s < fp.nstages; ++s) {
    const int R = fp.radix[s];
#define CALL(RR) run_stage<RR>(in, out, tw, N, Ns, pairs, bufstride)
    B200_RADIX_SWITCH(R, CALL)
#undef CALL
    Ns *= R;
    __syncthreads();
    float2* t = in; in = out; out = t;
  }
  return in;
}

template <typename T, int PAIRS>
__global__ void __launch_bounds__(kFftThreads) fft_analysis_rt_kernel(const T* __restrict__ x, float* __restrict__ X, const FftParams prm) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int N = prm.nlon;
  const int NS = N + 1;  // padded per-pair stride (float2 units)
  float2* tw = reinterpret_cast<float2*>(smem_raw);
  float2* b0 = tw + N;
  float2* b1 = b0 + PAIRS * NS;
  constexpr int KC = 2 * PAIRS;
  const int k0 = blockIdx.x * KC;
  const int r = blockIdx.y;
  for (int t = threadIdx.x; t < N; t += kFftThreads) tw[t] = prm.twiddle[t];
  {
    float* bf = reinterpret_cast<float*>(b0);
    const T* base = x + ((size_t)r * prm.nlat + k0) * N;
    const int rows_valid = min(KC, prm.nlat - k0);
    for (int e = threadIdx.x; e < KC * N; e += kFftThreads) {
      const int kk = e / N, j = e - kk * N;
      const float v = (kk < rows_valid) ? ld_as_float(base + (size_t)kk * N + j) : 0.f;
      bf[((size_t)(kk >> 1) * NS + j) * 2 + (kk & 1)] = v;
    }
  }
  __syncthreads();
  float2* res = run_fft(b0, b1, tw, prm.fp, PAIRS, NS);
  const int total = prm.mmax * 2 * KC;
  for (int e = threadIdx.x; e < total; e += kFftThreads) {
    const int kk = e % KC;
    const int mp = e / KC;
    const int p = mp & 1, m = mp >> 1;
    const int q = kk >> 1;
    float2 A, Bq;
    split_pair(res[q * NS + m], res[q * NS + (m == 0 ? 0 : N - m)], A, Bq);
    const float2 val = (kk & 1) ? Bq : A;
    const int k = k0 + kk;
    X[(((size_t)m * 2 + p) * prm.R + r) * prm.kp + k] = finish_analysis(prm, (p ? val.y : val.x) * mode_scale_analysis(prm, m, k));
  }
}

template <typename T, int PAIRS>
__global__ void __launch_bounds__(kFftThreads) fft_synthesis_rt_kernel(const float* __restrict__ Zs, T* __restrict__ y, const FftParams prm) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int N = prm.nlon;
  const int NS = N + 1;
  float2* tw = reinterpret_cast<float2*>(smem_raw);
  float2* b0 = tw + N;
  float2* b1 = b0 + PAIRS * NS;
  constexpr int KC = 2 * PAIRS;
  const int k0 = blockIdx.x * KC;
  const int r = blockIdx.y;
  for (int t = threadIdx.x; t < N; t += kFftThreads) tw[t] = prm.twiddle[t];
  fill_spectrum(Zs, b0, NS, PAIRS, kFftThreads, prm, k0, r, [](int i) { return i; });
  __syncthreads();
  float2* res = run_fft(b0, b1, tw, prm.fp, PAIRS, NS);
  {
    const float* rf = reinterpret_cast<const float*>(res);
    T* base = y + ((size_t)r * prm.nlat + k0) * N;
    const int rows_valid = min(KC, prm.nlat - k0);
    const float bias = prm.bias ? prm.bias[r % prm.C] : 0.f;
    for (int e = threadIdx.x; e < rows_valid * N; e += kFftThreads) {
      const int kk = e / N, j = e - kk * N;
      const float sc = (prm.scale_mode == 1) ? prm.rowscale[k0 + kk] : 1.f;
      st_from_float(base + (size_t)kk * N + j, rf[((size_t)(kk >> 1) * NS + j) * 2 + (1 - (kk & 1))] * sc + bias);
    }
  }
}

// ===================================================================================================== dispatch
static size_t rt_smem_bytes(int N, int pairs) { return sizeof(float2) * ((size_t)N + 2 * (size_t)pairs * (N + 1)); }

static int rt_pick_pairs(int N) {
  if (rt_smem_bytes(N, 4) <= 110 * 1024) return 4;
  if (rt_smem_bytes(N, 2) <= 220 * 1024) return 2;
  if (rt_smem_bytes(N, 1) <= 220 * 1024) return 1;
  return 0;
}

static FftParams make_params(const Plan* pl, int B, int C, int scale_mode, const float* bias) {
  FftParams prm;
  prm.fp = pl->fft;
  prm.nlat = pl->nlat; prm.nlon = pl->nlon; prm.mmax = pl->mmax; prm.kp = pl->kp;
  prm.R = B * C; prm.C = C; prm.scale_mode = scale_mode & 1; prm.round_tf32 = (scale_mode >> 1) & 1;
  prm.twiddle = pl->d_twiddle; prm.rowscale = pl->d_rowscale; prm.bias = bias;
  return prm;
}

template <typename T, int ROWS, int GROUPS, int TPG, int R0, int R1, int R2, int MINB>
static int launch_ct(const Plan* pl, int dir, const void* in, void* out, const FftParams& prm, cudaStream_t st) {
  typedef CtGeom<ROWS, R0, R1, R2> G;
  static_assert(G::smem_fixed + 8 * (G::H + 2) <= 227 * 1024, "plan does not fit in shared memory");
  const size_t smem = G::smem_fixed + sizeof(float2) * (size_t)((pl->mmax + 1) & ~1);   // + W_N^m, m < mmax
  // persistent CTAs: as many as fit concurrently (by shared memory), each walks tiles blockIdx.x, + gridDim.x, ...
  const int ntiles = ceil_div(pl->kp, ROWS) * prm.R;
  int per_sm = (int)((227 * 1024) / (smem + 1024));
  if (per_sm < 1) per_sm = 1;
  if (per_sm > 4) per_sm = 4;
  const int sms = usable_sms(pl->sm_count > 0 ? pl->sm_count : 132);
  dim3 grid(ntiles < per_sm * sms ? ntiles : per_sm * sms);
  if (dir == 0) {
    auto k = fft_analysis_ct_kernel<T, ROWS, GROUPS, TPG, R0, R1, R2, MINB>;
    B200_CHECK_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k<<<grid, GROUPS * TPG, smem, st>>>(static_cast<const T*>(in), static_cast<float*>(out), prm);
  } else {
    auto k = (2 * pl->mmax <= G::H) ? fft_synthesis_ct_kernel<T, ROWS, GROUPS, TPG, R0, R1, R2, MINB, true>
                                    : fft_synthesis_ct_kernel<T, ROWS, GROUPS, TPG, R0, R1, R2, MINB, false>;
    B200_CHECK_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k<<<grid, GROUPS * TPG, smem, st>>>(static_cast<const float*>(in), static_cast<T*>(out), prm);
  }
  B200_CHECK_LAUNCH();
  return 0;
}

// lengths with a compile-time plan: (ROWS, GROUPS, TPG, R0, R1, R2, CTAs/SM) for H = nlon / 2 = R0*R1*R2.  R0 is a power of two <= 16
// (LaySkew); TPG >= H/R0, ~ max_s H/R_s.  Other lengths (odd, or not listed) run the runtime-plan kernels.
#define CT_PLANS(X)             \
  X(4, 2, 96, 8, 9, 10, 3)      /* nlon 1440: 4-row tiles, 2 groups x one row pair per thread, 3 CTAs/SM (measured: synthesis 149 us; 8-row tiles at 2 CTAs/SM 175 us,
                                   4 CTAs/SM at <= 80 registers 186 us);
                                   radix order 8-9-10: every exchange access conflict-free in scripts/smem_sim.py (8-10-9: 1.17x / 1.11x) */ \
  X(8, 4, 96, 8, 9, 5, 2)       /* nlon  720 */ \
  X(8, 4, 64, 8, 5, 6, 2)       /* nlon  480 */ \
  X(8, 4, 64, 4, 9, 5, 2)       /* nlon  360 */ \
  X(8, 4, 64, 8, 5, 3, 2)       /* nlon  240 */ \
  X(8, 4, 64, 2, 9, 5, 2)       /* nlon  180 */ \
  X(8, 4, 32, 8, 3, 3, 2)       /* nlon  144 */ \
  X(8, 4, 32, 4, 4, 4, 2)       /* nlon  128 */ \
  X(8, 4, 32, 4, 4, 3, 2)       /* nlon   96 */ \
  X(8, 4, 32, 4, 3, 3, 2)       /* nlon   72 */ \
  X(8, 4, 32, 4, 8, 1, 2)       /* nlon   64 */ \
  X(8, 4, 32, 8, 4, 4, 2)       /* nlon  256 */ \
  X(8, 4, 64, 8, 8, 4, 2)       /* nlon  512 */ \
  X(8, 4, 64, 8, 8, 8, 2)       /* nlon 1024 */ \
  X(8, 2, 160, 16, 10, 9, 1)    /* nlon 2880 */

template <typename T>
static int dispatch_ct(const Plan* pl, int dir, const void* in, void* out, const FftParams& prm, cudaStream_t st, bool* handled) {
  *handled = false;
  // the compile-time plans move element pairs / quads with vector loads: both tensors must be 16-byte aligned
  if (((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(out)) & 15) != 0) return 0;
  *handled = true;
  // A/B switch (B200SHT_FFT_VARIANT=1): 1440-point rows as 8-row tiles with 2 CTAs per SM instead of 4-row tiles with 3
  static const int variant = [] { const char* e = getenv("B200SHT_FFT_VARIANT"); return e ? atoi(e) : 0; }();
  if (variant == 1 && pl->nlon == 1440) return launch_ct<T, 8, 2, 96, 8, 9, 10, 2>(pl, dir, in, out, prm, st);
#define X(RW, G, TP, A, B_, C_, MB) \
  if (pl->nlon == 2 * (A) * (B_) * (C_)) return launch_ct<T, RW, G, TP, A, B_, C_, MB>(pl, dir, in, out, prm, st);
  CT_PLANS(X)
#undef X
  *handled = false;
  return 0;
}

// pairs per CTA for plan lookup by the grid computation (kp / (2 * pairs) must be integral: kp is a multiple of 8)
template <typename T>
static int launch_rt(const Plan* pl, int dir, const void* in, void* out, const FftParams& prm, cudaStream_t st) {
  const int pairs = rt_pick_pairs(pl->nlon);
  if (pairs == 0) { set_error("fft: nlon=%d too large for shared memory", pl->nlon); return B200SHT_ERR_UNSUPPORTED; }
  const size_t smem = rt_smem_bytes(pl->nlon, pairs);
  dim3 grid(pl->kp / (2 * pairs), prm.R);
#define LAUNCH(P)                                                                                                                          \
  if (dir == 0) {                                                                                                                          \
    B200_CHECK_CUDA(cudaFuncSetAttribute(fft_analysis_rt_kernel<T, P>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));            \
    fft_analysis_rt_kernel<T, P><<<grid, kFftThreads, smem, st>>>(static_cast<const T*>(in), static_cast<float*>(out), prm);                \
  } else {                                                                                                                                 \
    B200_CHECK_CUDA(cudaFuncSetAttribute(fft_synthesis_rt_kernel<T, P>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));           \
    fft_synthesis_rt_kernel<T, P><<<grid, kFftThreads, smem, st>>>(static_cast<const float*>(in), static_cast<T*>(out), prm);               \
  }
  if (pairs == 4) { LAUNCH(4) } else if (pairs == 2) { LAUNCH(2) } else { LAUNCH(1) }
#undef LAUNCH
  B200_CHECK_LAUNCH();
  return 0;
}

template <typename T>
static int run_fft_dir(const Plan* pl, int dir, const void* in, void* out, const FftParams& prm, cudaStream_t st) {
  bool handled = false;
  int rc = dispatch_ct<T>(pl, dir, in, out, prm, st, &handled);
  if (handled) return rc;
  return launch_rt<T>(pl, dir, in, out, prm, st);
}

// tensor-core DFT (dft.cu): used when the caller runs the TF32 precision (scale_mode bit 1) and the grid is in its range
bool dft_usable(const Plan* pl);
int dft_analysis(const Plan* pl, const void* x, int dtype, int B, int C, float* X, int mode, cudaStream_t st);
int dft_synthesis(const Plan* pl, const float* Z, void* y, int dtype, int B, int C, const float* bias, int mode, cudaStream_t st);

int fft_analysis(const Plan* pl, const void* x, int dtype, int B, int C, float* X, int scale_mode, cudaStream_t st) {
  B200_REQUIRE(B > 0 && C > 0 && (long long)B * C <= 65535, "fft_analysis: B*C=%lld out of range", (long long)B * C);
  B200_REQUIRE(dtype == B200SHT_F32 || dtype == B200SHT_BF16, "fft_analysis: unknown dtype %d", dtype);
  // tensor-core DFT: TMA reads the samples, so the input must be 16-byte aligned (and nlon % 32 == 0 for fp32 input); otherwise the CUDA-core FFT
  if ((scale_mode & 2) && dft_usable(pl) && (reinterpret_cast<uintptr_t>(x) & 15) == 0 && (dtype == B200SHT_BF16 || pl->nlon % 32 == 0))
    return dft_analysis(pl, x, dtype, B, C, X, scale_mode & 1, st);
  FftParams prm = make_params(pl, B, C, scale_mode, nullptr);
  if (dtype == B200SHT_F32) return run_fft_dir<float>(pl, 0, x, X, prm, st);
  if (dtype == B200SHT_BF16) return run_fft_dir<__nv_bfloat16>(pl, 0, x, X, prm, st);
  set_error("fft_analysis: unknown dtype %d", dtype);
  return B200SHT_ERR_INVALID;
}

int fft_synthesis(const Plan* pl, const float* Z, void* y, int dtype, int B, int C, const float* bias, int scale_mode, cudaStream_t st) {
  B200_REQUIRE(B > 0 && C > 0 && (long long)B * C <= 65535, "fft_synthesis: B*C=%lld out of range", (long long)B * C);
  B200_REQUIRE(dtype == B200SHT_F32 || dtype == B200SHT_BF16, "fft_synthesis: unknown dtype %d", dtype);
  if (scale_mode & 2) {   // the input is in the tiled layout of b200sht_legendre_synthesis_tiled: only the tensor-core DFT reads it
    B200_REQUIRE(dft_usable(pl), "fft_synthesis: scale_mode | 2 (tiled latspec, tensor-core DFT) is not available for this plan (b200sht_plan_query(plan, 8) == 0)");
    B200_REQUIRE((reinterpret_cast<uintptr_t>(Z) & 127) == 0, "fft_synthesis: the tiled latspec must be 128-byte aligned");
    return dft_synthesis(pl, Z, y, dtype, B, C, bias, scale_mode & 1, st);
  }
  // the run-time kernels read the latspec as float2 pairs of rows (fill_spectrum), the compile-time ones as float4 when it is 16-byte aligned
  B200_REQUIRE((reinterpret_cast<uintptr_t>(Z) & 7) == 0, "fft_synthesis: the latspec must be 8-byte aligned");
  FftParams prm = make_params(pl, B, C, scale_mode, bias);
  if (dtype == B200SHT_F32) return run_fft_dir<float>(pl, 1, Z, y, prm, st);
  if (dtype == B200SHT_BF16) return run_fft_dir<__nv_bfloat16>(pl, 1, Z, y, prm, st);
  set_error("fft_synthesis: unknown dtype %d", dtype);
  return B200SHT_ERR_INVALID;
}

// ---------------------------------------------------------------------------- host emulation (CPU tests)
static void host_fft(std::vector<float2>& a, const std::vector<float2>& tw, const FftPlan& fp) {
  const int N = fp.N;
  std::vector<float2> b(N);
  float2* in = a.data();
  float2* out = b.data();
  int Ns = 1;
  for (int s = 0; s < fp.nstages; ++s) {
    const int R = fp.radix[s];
    for (int j = 0; j < N / R; ++j) {
#define CALL(RR) stage_butterfly<RR>(in, out, tw.data(), N, Ns, j)
      B200_RADIX_SWITCH(R, CALL)
#undef CALL
    }
    Ns *= R;
    float2* t = in; in = out; out = t;
  }
  if (in != a.data()) for (int i = 0; i < N; ++i) a[i] = in[i];
}

void make_twiddles_host(int N, std::vector<float2>& tw) {
  tw.resize(N);
  for (int t = 0; t < N; ++t) {
    const double ang = -2.0 * M_PI * (double)t / (double)N;
    tw[t] = make_float2((float)cos(ang), (float)sin(ang));
  }
}

}  // namespace b200sht

using namespace b200sht;

// Debug entry points: run the *same* stage/butterfly/split code on the host (no GPU needed).
//   analysis : rows a, b (float[N]) -> Xa, Xb (float[2*mmax] interleaved), unscaled rfft
//   synthesis: Za, Zb (float[2*mmax]) -> rows a, b (float[N]) with irfft(norm="forward") semantics
extern "C" int b200sht_debug_fft_host(int N, int mmax, int direction, const float* in_a, const float* in_b, float* out_a, float* out_b) {
  FftPlan fp;
  if (!make_fft_plan(N, &fp)) { set_error("debug_fft_host: unsupported length %d", N); return B200SHT_ERR_UNSUPPORTED; }
  std::vector<float2> tw;
  make_twiddles_host(N, tw);
  std::vector<float2> buf(N);
  if (direction == 0) {
    for (int j = 0; j < N; ++j) buf[j] = make_float2(in_a[j], in_b[j]);
    host_fft(buf, tw, fp);
    for (int m = 0; m < mmax; ++m) {
      float2 A, Bq;
      split_pair(buf[m], buf[m == 0 ? 0 : N - m], A, Bq);
      out_a[2 * m] = A.x; out_a[2 * m + 1] = A.y;
      out_b[2 * m] = Bq.x; out_b[2 * m + 1] = Bq.y;
    }
  } else {
    for (int j = 0; j < N; ++j) buf[j] = make_float2(0.f, 0.f);
    for (int m = 0; m < mmax; ++m) {
      float ar = in_a[2 * m], ai = in_a[2 * m + 1], br = in_b[2 * m], bi = in_b[2 * m + 1];
      const bool self_conj = (m == 0) || (2 * m == N);
      if (self_conj) { ai = 0.f; bi = 0.f; }
      buf[m] = make_float2(ai + br, ar - bi);
      if (!self_conj) buf[N - m] = make_float2(br - ai, ar + bi);
    }
    host_fft(buf, tw, fp);
    for (int j = 0; j < N; ++j) { out_a[j] = buf[j].y; out_b[j] = buf[j].x; }
  }
  return 0;
}

extern "C" int b200sht_debug_fft_plan(int N, int* radices, int max_radices) {
  FftPlan fp;
  if (!make_fft_plan(N, &fp)) return B200SHT_ERR_UNSUPPORTED;
  for (int i = 0; i < fp.nstages && i < max_radices; ++i) radices[i] = fp.radix[i];
  return fp.nstages;
}
