// Per-mode complex channel mixing on packed spectral tensors (fp32 CUDA-core path) and weight re-layout.
//
// Replaces /root/reference/makani/models/common/contractions.py:
//   _contract_lwise  "bgixy,giox->bgoxy"  (:23)   -> OP_DHCONV      (dense kernels below)
//   _contract_lmwise "bgixy,gioxy->bgoxy" (:19)   -> OP_DIAGONAL    (per-mode kernels)
//   _contract_sep_lwise / _contract_sep_lmwise (:27,:31) -> OP_SEP_*
//   compl_mul2d_fwd "bixy,io->boxy" (:62), compl_exp_mul2d_fwd "bixy,xio->boxy" (:106) -> OP_SHARED / OP_LDEP
// and their autograd adjoints (PyTorch complex convention: grad_x = grad_y * conj(w), grad_w = conj(x) * grad_y).
#include "common.cuh"

namespace b200sht {

struct MixDims {
  int L, M, B, G, Cig, Cog;   // per-group channel counts
  int cpi, cpo;               // padded total channel counts of the in / out spec tensors
  int cop;                    // padded Cog in the packed weight (planar: float [L][G][Cig][2][cop])
  long long wl_stride;        // floats between consecutive l in the packed weight (0: shared)
  int dense;                  // spec tensors store every (l, m) entry (l/m-sharded spectra of the distributed path)
};

// ------------------------------------------------------------------------------------ weight re-layout
// native DHCONV complex [G][Cig][Cog][L]  <->  packed float [L][G][Cig][2][cop]  (real plane, imaginary plane per input row)
// A block moves a 128 (o) x 32 (l) tile through shared memory: 16 independent 8-byte loads per thread in flight (the 32 x 32 tiles of
// round 1 had 4 and ran at 1 TB/s, latency bound: 10 us per re-layout of the 10 MB weight, twice per training step).
constexpr int kWpO = 128, kWpL = 32;
__global__ void __launch_bounds__(256) weight_pack_dhconv_kernel(float2* __restrict__ wn, float* __restrict__ wp, int L, int GC /*G*Cig*/, int Cog,
                                                                 int cop, int to_native, int rnd) {
  __shared__ float2 tile[kWpO][kWpL + 1];
  pdl_trigger();
  pdl_wait();   // the weight (optimizer) and the packed buffer (the previous step's mix kernels may still read its memory) belong to earlier kernels
  const int gi = blockIdx.z;
  const int o0 = blockIdx.y * kWpO, l0 = blockIdx.x * kWpL;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  if (!to_native) {
    float2 v[kWpO / 8];
#pragma unroll
    for (int i = 0; i < kWpO / 8; ++i) {
      const int o = o0 + ty + 8 * i, l = l0 + tx;
      v[i] = (o < Cog && l < L) ? wn[((size_t)gi * Cog + o) * L + l] : make_float2(0.f, 0.f);
    }
#pragma unroll
    for (int i = 0; i < kWpO / 8; ++i) tile[ty + 8 * i][tx] = v[i];
    __syncthreads();
    for (int ll = ty; ll < kWpL; ll += 8) {
      const int l = l0 + ll;
      if (l >= L) continue;
      float* row = wp + ((size_t)l * GC + gi) * 2 * cop;
#pragma unroll
      for (int oo = 0; oo < kWpO; oo += 32) {
        const int o = o0 + oo + tx;
        if (o < cop) {
          const float2 t = tile[oo + tx][ll];
          row[o] = rnd ? tf32_rn(t.x) : t.x;
          row[cop + o] = rnd ? tf32_rn(t.y) : t.y;
        }
      }
    }
  } else {
    for (int ll = ty; ll < kWpL; ll += 8) {
      const int l = l0 + ll;
      const float* row = wp + ((size_t)(l < L ? l : 0) * GC + gi) * 2 * cop;
#pragma unroll
      for (int oo = 0; oo < kWpO; oo += 32) {
        const int o = o0 + oo + tx;
        tile[oo + tx][ll] = (l < L && o < cop) ? make_float2(row[o], row[cop + o]) : make_float2(0.f, 0.f);
      }
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < kWpO / 8; ++i) {
      const int o = o0 + ty + 8 * i, l = l0 + tx;
      if (o < Cog && l < L) wn[((size_t)gi * Cog + o) * L + l] = tile[ty + 8 * i][tx];
    }
  }
}

// native [rows][Co] complex <-> packed [rows][2][cop]   (OP_SHARED: rows = Ci, OP_LDEP: rows = L*Ci)
__global__ void weight_pad_kernel(float2* __restrict__ wn, float* __restrict__ wp, long long rows, int Co, int cop, int to_native, int rnd) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * cop) return;
  const long long row = idx / cop;
  const int o = (int)(idx - row * cop);
  float* prow = wp + row * 2 * cop;
  if (!to_native) {
    const float2 v = (o < Co) ? wn[row * Co + o] : make_float2(0.f, 0.f);
    prow[o] = rnd ? tf32_rn(v.x) : v.x;
    prow[cop + o] = rnd ? tf32_rn(v.y) : v.y;
  } else if (o < Co) {
    wn[row * Co + o] = make_float2(prow[o], prow[cop + o]);
  }
}

int mix_weight_relayout(int op, const void* w_native, float* w_packed, int L, int G, int Ci, int Co, int to_native, int round_tf32, cudaStream_t st) {
  B200_REQUIRE(G > 0 && Ci % G == 0 && Co % G == 0, "mix_weight: channels (%d,%d) not divisible by groups %d", Ci, Co, G);
  const int Cig = Ci / G, Cog = Co / G, cop = round_up(Cog, 4);
  if (op == B200SHT_OP_DHCONV) {
    dim3 grid(ceil_div(L, kWpL), ceil_div(cop, kWpO), G * Cig);
    B200_REQUIRE(grid.z <= 65535, "mix_weight: G*Cig=%u exceeds grid limit", grid.z);
    B200_CHECK_CUDA(launch_pdl(weight_pack_dhconv_kernel, grid, dim3(256), 0, st, static_cast<float2*>(const_cast<void*>(w_native)), w_packed, L, G * Cig, Cog, cop,
                               to_native, round_tf32));
  } else if (op == B200SHT_OP_SHARED || op == B200SHT_OP_LDEP) {
    B200_REQUIRE(G == 1, "mix_weight: OP_SHARED/OP_LDEP are ungrouped");
    const long long rows = (op == B200SHT_OP_SHARED) ? Ci : (long long)L * Ci;
    const long long total = rows * cop;
    weight_pad_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(static_cast<float2*>(const_cast<void*>(w_native)), w_packed, rows, Co, cop, to_native, round_tf32);
  } else {
    set_error("mix_weight: operator %d has no packed weight", op);
    return B200SHT_ERR_INVALID;
  }
  B200_CHECK_LAUNCH();
  return 0;
}

// ------------------------------------------------------------------------------- dense forward / dgrad
// MODE 0: y[row, o] = sum_i x[row, i] * w[i][o] (+ cbias[o])       K = Cig, outputs Cog
// MODE 1: gx[row, i] = sum_o gy[row, o] * conj(w[i][o])            K = Cog, outputs Cig
// rows = (m, b), m < mend(l).  grid: (row tiles, out tiles * G, L)
template <int MODE>
__global__ void __launch_bounds__(256) mix_dense_kernel(const float* __restrict__ xin, const float* __restrict__ w, const float2* __restrict__ cbias,
                                                        float* __restrict__ yout, const MixDims d) {
  __shared__ float Xr[16][33], Xi[16][33], Wr[16][33], Wi[16][33];
  const int l = blockIdx.z;
  const int nrows = mend_d(l, d.M, d.dense) * d.B;
  const int row0 = blockIdx.x * 32;
  if (row0 >= nrows) return;
  const int K = MODE == 0 ? d.Cig : d.Cog;          // contraction length
  const int NO = MODE == 0 ? d.Cog : d.Cig;         // outputs per group
  const int cp_in = MODE == 0 ? d.cpi : d.cpo;      // padded channels of the tensor we read
  const int cp_out = MODE == 0 ? d.cpo : d.cpi;
  const int ntile = ceil_div(NO + 3, 32);           // +3: room for the zero padding after the last group
  const int g = blockIdx.y / ntile, ot = blockIdx.y % ntile;
  const int o0 = ot * 32;
  const int pad_out = cp_out - NO * d.G;
  const int out_limit = NO + ((g == d.G - 1) ? pad_out : 0);
  if (o0 >= out_limit) return;
  const int t = threadIdx.x;
  const int ty = t >> 4, tx = t & 15;
  const float* wl = w + (size_t)l * d.wl_stride;

  // loader coordinates
  const int xrow = t >> 3, xk = (t & 7) * 2;
  const int grow = row0 + xrow;
  const float* xbase = nullptr;
  if (grow < nrows) {
    const int m = grow / d.B, b = grow % d.B;
    xbase = xin + ((size_t)l * d.M + m) * 2 * d.B * cp_in + (size_t)b * cp_in + g * K;
  }
  const size_t xplane = (size_t)d.B * cp_in;

  float ar[2][2] = {{0.f, 0.f}, {0.f, 0.f}}, ai[2][2] = {{0.f, 0.f}, {0.f, 0.f}};

  for (int k0 = 0; k0 < K; k0 += 16) {
    float x0r = 0.f, x1r = 0.f, x0i = 0.f, x1i = 0.f;
    if (xbase) {
      if (k0 + xk < K) { x0r = xbase[k0 + xk]; x0i = xbase[xplane + k0 + xk]; }
      if (k0 + xk + 1 < K) { x1r = xbase[k0 + xk + 1]; x1i = xbase[xplane + k0 + xk + 1]; }
    }
    float w0r = 0.f, w0i = 0.f, w1r = 0.f, w1i = 0.f;
    int wkk, woo;
    if (MODE == 0) {  // tile [kk = i][oo = o]: thread -> kk = t/16, oo = (t%16)*2, +1
      wkk = t >> 4; woo = (t & 15) * 2;
      const int i = k0 + wkk, o = o0 + woo;
      if (i < K) {
        const float* p = wl + (size_t)(g * d.Cig + i) * 2 * d.cop + o;
        if (o < d.Cog) { w0r = p[0]; w0i = p[d.cop]; }
        if (o + 1 < d.Cog) { w1r = p[1]; w1i = p[d.cop + 1]; }
      }
    } else {          // tile [kk = o][oo = i]: thread -> ii = t/8, kq = (t%8)*2
      woo = t >> 3; wkk = (t & 7) * 2;
      const int i = o0 + woo, o = k0 + wkk;
      if (i < d.Cig) {
        const float* p = wl + (size_t)(g * d.Cig + i) * 2 * d.cop + o;
        if (o < K) { w0r = p[0]; w0i = p[d.cop]; }
        if (o + 1 < K) { w1r = p[1]; w1i = p[d.cop + 1]; }
      }
    }
    __syncthreads();
    Xr[xk][xrow] = x0r; Xi[xk][xrow] = x0i; Xr[xk + 1][xrow] = x1r; Xi[xk + 1][xrow] = x1i;
    if (MODE == 0) { Wr[wkk][woo] = w0r; Wi[wkk][woo] = w0i; Wr[wkk][woo + 1] = w1r; Wi[wkk][woo + 1] = w1i; }
    else { Wr[wkk][woo] = w0r; Wi[wkk][woo] = w0i; Wr[wkk + 1][woo] = w1r; Wi[wkk + 1][woo] = w1i; }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      float xr[2] = {Xr[kk][ty * 2], Xr[kk][ty * 2 + 1]}, xi[2] = {Xi[kk][ty * 2], Xi[kk][ty * 2 + 1]};
      float wr[2] = {Wr[kk][tx * 2], Wr[kk][tx * 2 + 1]}, wi[2] = {Wi[kk][tx * 2], Wi[kk][tx * 2 + 1]};
#pragma unroll
      for (int a = 0; a < 2; ++a)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          if (MODE == 0) {
            ar[a][c] = fmaf(xr[a], wr[c], fmaf(-xi[a], wi[c], ar[a][c]));
            ai[a][c] = fmaf(xr[a], wi[c], fmaf(xi[a], wr[c], ai[a][c]));
          } else {
            ar[a][c] = fmaf(xr[a], wr[c], fmaf(xi[a], wi[c], ar[a][c]));
            ai[a][c] = fmaf(xi[a], wr[c], fmaf(-xr[a], wi[c], ai[a][c]));
          }
        }
    }
  }
#pragma unroll
  for (int a = 0; a < 2; ++a) {
    const int row = row0 + ty * 2 + a;
    if (row >= nrows) continue;
    const int m = row / d.B, b = row % d.B;
    float* ybase = yout + ((size_t)l * d.M + m) * 2 * d.B * cp_out + (size_t)b * cp_out + g * NO;
    const size_t yplane = (size_t)d.B * cp_out;
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const int o = o0 + tx * 2 + c;
      if (o >= out_limit) continue;
      float vr = ar[a][c], vi = ai[a][c];
      if (MODE == 0 && cbias != nullptr && o < NO) { const float2 cb = cbias[g * NO + o]; vr += cb.x; vi += cb.y; }
      ybase[o] = vr;
      ybase[yplane + o] = vi;
    }
  }
}

// ----------------------------------------------------------------------------------------- dense wgrad
// gw[l][g][i][o] = sum_rows conj(x[row, i]) * gy[row, o]; for a shared weight (wl_stride == 0) the sum also runs over l.
// grid: (i tiles, o tiles * G, Lw)
__global__ void __launch_bounds__(256) mix_wgrad_kernel(const float* __restrict__ xin, const float* __restrict__ gy, float* __restrict__ gw,
                                                        const MixDims d, int shared_w) {
  __shared__ float Xr[16][33], Xi[16][33], Gr[16][33], Gi[16][33];
  const int ntile_o = ceil_div(d.cop, 32);
  const int g = blockIdx.y / ntile_o, ot = blockIdx.y % ntile_o;
  const int i0 = blockIdx.x * 32, o0 = ot * 32;
  const int t = threadIdx.x;
  const int ty = t >> 4, tx = t & 15;
  const int lrow = t >> 4, cq = (t & 15) * 2;   // loader: 16 rows x 32 channels (2 per thread)
  float ar[2][2] = {{0.f, 0.f}, {0.f, 0.f}}, ai[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
  const int lbeg = shared_w ? 0 : blockIdx.z, lend = shared_w ? d.L : blockIdx.z + 1;
  for (int l = lbeg; l < lend; ++l) {
    const int nrows = mend_d(l, d.M, d.dense) * d.B;
    for (int r0 = 0; r0 < nrows; r0 += 16) {
      const int row = r0 + lrow;
      float x0r = 0.f, x0i = 0.f, x1r = 0.f, x1i = 0.f, g0r = 0.f, g0i = 0.f, g1r = 0.f, g1i = 0.f;
      if (row < nrows) {
        const int m = row / d.B, b = row % d.B;
        const float* xb = xin + ((size_t)l * d.M + m) * 2 * d.B * d.cpi + (size_t)b * d.cpi + g * d.Cig;
        const float* gb = gy + ((size_t)l * d.M + m) * 2 * d.B * d.cpo + (size_t)b * d.cpo + g * d.Cog;
        const size_t xp = (size_t)d.B * d.cpi, gp = (size_t)d.B * d.cpo;
        const int i = i0 + cq, o = o0 + cq;
        if (i < d.Cig) { x0r = xb[i]; x0i = xb[xp + i]; }
        if (i + 1 < d.Cig) { x1r = xb[i + 1]; x1i = xb[xp + i + 1]; }
        if (o < d.Cog) { g0r = gb[o]; g0i = gb[gp + o]; }
        if (o + 1 < d.Cog) { g1r = gb[o + 1]; g1i = gb[gp + o + 1]; }
      }
      __syncthreads();
      Xr[lrow][cq] = x0r; Xi[lrow][cq] = x0i; Xr[lrow][cq + 1] = x1r; Xi[lrow][cq + 1] = x1i;
      Gr[lrow][cq] = g0r; Gi[lrow][cq] = g0i; Gr[lrow][cq + 1] = g1r; Gi[lrow][cq + 1] = g1i;
      __syncthreads();
#pragma unroll
      for (int kk = 0; kk < 16; ++kk) {
        float xr[2] = {Xr[kk][ty * 2], Xr[kk][ty * 2 + 1]}, xi[2] = {Xi[kk][ty * 2], Xi[kk][ty * 2 + 1]};
        float gr[2] = {Gr[kk][tx * 2], Gr[kk][tx * 2 + 1]}, gi[2] = {Gi[kk][tx * 2], Gi[kk][tx * 2 + 1]};
#pragma unroll
        for (int a = 0; a < 2; ++a)
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            ar[a][c] = fmaf(xr[a], gr[c], fmaf(xi[a], gi[c], ar[a][c]));
            ai[a][c] = fmaf(xr[a], gi[c], fmaf(-xi[a], gr[c], ai[a][c]));
          }
      }
    }
  }
  float* gwl = gw + (size_t)(shared_w ? 0 : blockIdx.z) * d.wl_stride;
#pragma unroll
  for (int a = 0; a < 2; ++a) {
    const int i = i0 + ty * 2 + a;
    if (i >= d.Cig) continue;
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const int o = o0 + tx * 2 + c;
      if (o >= d.cop) continue;
      float* p = gwl + (size_t)(g * d.Cig + i) * 2 * d.cop + o;
      p[0] = (o < d.Cog) ? ar[a][c] : 0.f;
      p[d.cop] = (o < d.Cog) ? ai[a][c] : 0.f;
    }
  }
}

// complex bias gradient (OP_SHARED / OP_LDEP): gcb[o] = sum over the stored triangle and batch of gy[.., o]
__global__ void mix_cbias_grad_kernel(const float* __restrict__ gy, float2* __restrict__ gcb, int L, int M, int B, int cpo, int dense) {
  const int o = blockIdx.x;
  float sr = 0.f, si = 0.f;
  for (int l = 0; l < L; ++l) {
    const int nrows = mend_d(l, M, dense) * B;
    for (int row = threadIdx.x; row < nrows; row += blockDim.x) {
      const int m = row / B, b = row % B;
      const float* base = gy + ((size_t)l * M + m) * 2 * B * cpo + (size_t)b * cpo + o;
      sr += base[0];
      si += base[(size_t)B * cpo];
    }
  }
  __shared__ float rr[32], ri[32];
  for (int s = 16; s > 0; s >>= 1) { sr += __shfl_xor_sync(0xffffffffu, sr, s); si += __shfl_xor_sync(0xffffffffu, si, s); }
  if ((threadIdx.x & 31) == 0) { rr[threadIdx.x >> 5] = sr; ri[threadIdx.x >> 5] = si; }
  __syncthreads();
  if (threadIdx.x < 32) {
    float a = threadIdx.x < (blockDim.x >> 5) ? rr[threadIdx.x] : 0.f, b2 = threadIdx.x < (blockDim.x >> 5) ? ri[threadIdx.x] : 0.f;
    for (int s = 16; s > 0; s >>= 1) { a += __shfl_xor_sync(0xffffffffu, a, s); b2 += __shfl_xor_sync(0xffffffffu, b2, s); }
    if (threadIdx.x == 0) gcb[o] = make_float2(a, b2);
  }
}

int mix_cbias_grad(const float* gy, void* gcb, int L, int M, int B, int Co, int dense, cudaStream_t st) {
  mix_cbias_grad_kernel<<<Co, 256, 0, st>>>(gy, static_cast<float2*>(gcb), L, M, B, round_up(Co, 4), dense);
  B200_CHECK_LAUNCH();
  return 0;
}

// ------------------------------------------------------------------------- per-mode (non-dense) operators
// OP_DIAGONAL      w native complex [G][Cig][Cog][L][M]
// OP_SEP_DHCONV    w native complex [G][Cig][L]         (Co == Ci)
// OP_SEP_DIAGONAL  w native complex [G][Cig][L][M]
// one thread per (l, m, b, padded out channel); purely bandwidth bound (each weight is used once per batch element).  The threads of the
// channel padding [NOut, cp_out) write its exact zeros, as every other producer of a packed spectrum does.
template <int OP, int MODE>  // MODE 0 forward, 1 dgrad
__global__ void mix_permode_kernel(const float* __restrict__ xin, const float2* __restrict__ w, float* __restrict__ yout, const MixDims d) {
  const int NOut = MODE == 0 ? d.Cog * d.G : d.Cig * d.G;
  const int cp_in = MODE == 0 ? d.cpi : d.cpo, cp_out = MODE == 0 ? d.cpo : d.cpi;
  const long long total = (long long)d.L * d.M * d.B * cp_out;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int m = (int)(idx % d.M);
  long long rest = idx / d.M;
  const int l = (int)(rest % d.L); rest /= d.L;
  const int oc = (int)(rest % cp_out);
  const int b = (int)(rest / cp_out);
  if (m >= mend_d(l, d.M, d.dense)) return;
  float* yb = yout + ((size_t)l * d.M + m) * 2 * d.B * cp_out + (size_t)b * cp_out;
  if (oc >= NOut) {
    yb[oc] = 0.f;
    yb[(size_t)d.B * cp_out + oc] = 0.f;
    return;
  }
  const float* xb = xin + ((size_t)l * d.M + m) * 2 * d.B * cp_in + (size_t)b * cp_in;
  const size_t xp = (size_t)d.B * cp_in;
  float vr = 0.f, vi = 0.f;
  if (OP == B200SHT_OP_DIAGONAL) {
    const int K = MODE == 0 ? d.Cig : d.Cog;
    const int NOg = MODE == 0 ? d.Cog : d.Cig;
    const int g = oc / NOg, oo = oc % NOg;
    for (int kk = 0; kk < K; ++kk) {
      const int i = MODE == 0 ? kk : oo, o = MODE == 0 ? oo : kk;
      const float2 ww = w[((((size_t)g * d.Cig + i) * d.Cog + o) * d.L + l) * d.M + m];
      const float xr = xb[g * K + kk], xi = xb[xp + g * K + kk];
      if (MODE == 0) { vr += xr * ww.x - xi * ww.y; vi += xr * ww.y + xi * ww.x; }
      else { vr += xr * ww.x + xi * ww.y; vi += xi * ww.x - xr * ww.y; }
    }
  } else {
    const float2 ww = (OP == B200SHT_OP_SEP_DHCONV) ? w[(size_t)oc * d.L + l] : w[((size_t)oc * d.L + l) * d.M + m];
    const float xr = xb[oc], xi = xb[xp + oc];
    if (MODE == 0) { vr = xr * ww.x - xi * ww.y; vi = xr * ww.y + xi * ww.x; }
    else { vr = xr * ww.x + xi * ww.y; vi = xi * ww.x - xr * ww.y; }
  }
  yb[oc] = vr;
  yb[(size_t)d.B * cp_out + oc] = vi;
}

// wgrad for per-mode operators: one thread per weight element, reduction over batch (and m for SEP_DHCONV)
template <int OP>
__global__ void mix_permode_wgrad_kernel(const float* __restrict__ xin, const float* __restrict__ gy, float2* __restrict__ gw, const MixDims d) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long total;
  if (OP == B200SHT_OP_DIAGONAL) total = (long long)d.G * d.Cig * d.Cog * d.L * d.M;
  else if (OP == B200SHT_OP_SEP_DHCONV) total = (long long)d.G * d.Cig * d.L;
  else total = (long long)d.G * d.Cig * d.L * d.M;
  if (idx >= total) return;
  float sr = 0.f, si = 0.f;
  const size_t xp = (size_t)d.B * d.cpi, gp = (size_t)d.B * d.cpo;
  if (OP == B200SHT_OP_SEP_DHCONV) {
    const int l = (int)(idx % d.L);
    const int c = (int)(idx / d.L);
    const int me = mend_d(l, d.M, d.dense);
    for (int m = 0; m < me; ++m)
      for (int b = 0; b < d.B; ++b) {
        const float* xb = xin + ((size_t)l * d.M + m) * 2 * d.B * d.cpi + (size_t)b * d.cpi + c;
        const float* gb = gy + ((size_t)l * d.M + m) * 2 * d.B * d.cpo + (size_t)b * d.cpo + c;
        const float xr = xb[0], xi = xb[xp], gr = gb[0], gi = gb[gp];
        sr += xr * gr + xi * gi; si += xr * gi - xi * gr;
      }
  } else {
    const int m = (int)(idx % d.M);
    long long rest = idx / d.M;
    const int l = (int)(rest % d.L); rest /= d.L;
    int ci, co;
    if (OP == B200SHT_OP_DIAGONAL) {
      const int o = (int)(rest % d.Cog); rest /= d.Cog;
      const int i = (int)(rest % d.Cig);
      const int g = (int)(rest / d.Cig);
      ci = g * d.Cig + i; co = g * d.Cog + o;
    } else { ci = co = (int)rest; }
    if (m < mend_d(l, d.M, d.dense))
      for (int b = 0; b < d.B; ++b) {
        const float* xb = xin + ((size_t)l * d.M + m) * 2 * d.B * d.cpi + (size_t)b * d.cpi + ci;
        const float* gb = gy + ((size_t)l * d.M + m) * 2 * d.B * d.cpo + (size_t)b * d.cpo + co;
        const float xr = xb[0], xi = xb[xp], gr = gb[0], gi = gb[gp];
        sr += xr * gr + xi * gi; si += xr * gi - xi * gr;
      }
  }
  gw[idx] = make_float2(sr, si);
}

// ------------------------------------------------------------------------------------------ host side
static int make_dims(const Plan* pl, int op, int B, int G, int Ci, int Co, MixDims* d) {
  B200_REQUIRE(B > 0 && G > 0 && Ci > 0 && Co > 0 && Ci % G == 0 && Co % G == 0, "mix: bad dims B=%d G=%d Ci=%d Co=%d", B, G, Ci, Co);
  if (op == B200SHT_OP_SEP_DHCONV || op == B200SHT_OP_SEP_DIAGONAL) B200_REQUIRE(Ci == Co, "mix: separable operator needs Ci == Co");
  if (op == B200SHT_OP_SHARED || op == B200SHT_OP_LDEP) B200_REQUIRE(G == 1, "mix: OP_SHARED/OP_LDEP are ungrouped");
  d->dense = pl->dense;
  d->L = pl->lmax; d->M = pl->mmax; d->B = B; d->G = G; d->Cig = Ci / G; d->Cog = Co / G;
  d->cpi = round_up(Ci, 4); d->cpo = round_up(Co, 4); d->cop = round_up(Co / G, 4);
  d->wl_stride = (op == B200SHT_OP_SHARED) ? 0 : (long long)G * (Ci / G) * d->cop * 2;
  return 0;
}

static bool is_dense(int op) { return op == B200SHT_OP_DHCONV || op == B200SHT_OP_SHARED || op == B200SHT_OP_LDEP; }

int mix_forward_simt(const Plan* pl, int op, const float* x, const void* w, const void* cbias, float* y, int B, int G, int Ci, int Co,
                     cudaStream_t st) {
  MixDims d;
  int rc = make_dims(pl, op, B, G, Ci, Co, &d);
  if (rc) return rc;
  if (is_dense(op)) {
    const int ntile = ceil_div(d.Cog + 3, 32);
    dim3 grid(ceil_div(d.M * B, 32), ntile * G, d.L);
    B200_REQUIRE(grid.y <= 65535 && grid.z <= 65535, "mix_forward: grid too large");
    mix_dense_kernel<0><<<grid, 256, 0, st>>>(x, static_cast<const float*>(w), static_cast<const float2*>(cbias), y, d);
  } else {
    const long long total = (long long)d.L * d.M * B * d.cpo;
    const unsigned nb = (unsigned)((total + 255) / 256);
    const float2* wn = static_cast<const float2*>(w);
    if (op == B200SHT_OP_DIAGONAL) mix_permode_kernel<B200SHT_OP_DIAGONAL, 0><<<nb, 256, 0, st>>>(x, wn, y, d);
    else if (op == B200SHT_OP_SEP_DHCONV) mix_permode_kernel<B200SHT_OP_SEP_DHCONV, 0><<<nb, 256, 0, st>>>(x, wn, y, d);
    else if (op == B200SHT_OP_SEP_DIAGONAL) mix_permode_kernel<B200SHT_OP_SEP_DIAGONAL, 0><<<nb, 256, 0, st>>>(x, wn, y, d);
    else { set_error("mix_forward: unknown operator %d", op); return B200SHT_ERR_INVALID; }
  }
  B200_CHECK_LAUNCH();
  return 0;
}

int mix_backward_simt(const Plan* pl, int op, const float* x, const void* w, const float* gy, float* gx, void* gw, void* gcbias, int B, int G,
                      int Ci, int Co, cudaStream_t st) {
  MixDims d;
  int rc = make_dims(pl, op, B, G, Ci, Co, &d);
  if (rc) return rc;
  if (is_dense(op)) {
    if (gx) {
      const int ntile = ceil_div(d.Cig + 3, 32);
      dim3 grid(ceil_div(d.M * B, 32), ntile * G, d.L);
      B200_REQUIRE(grid.y <= 65535 && grid.z <= 65535, "mix_backward: grid too large");
      mix_dense_kernel<1><<<grid, 256, 0, st>>>(gy, static_cast<const float*>(w), nullptr, gx, d);
      B200_CHECK_LAUNCH();
    }
    if (gw) {
      const int shared_w = (op == B200SHT_OP_SHARED);
      dim3 grid(ceil_div(d.Cig, 32), ceil_div(d.cop, 32) * G, shared_w ? 1 : d.L);
      mix_wgrad_kernel<<<grid, 256, 0, st>>>(x, gy, static_cast<float*>(gw), d, shared_w);
      B200_CHECK_LAUNCH();
    }
    if (gcbias) {
      mix_cbias_grad_kernel<<<Co, 256, 0, st>>>(gy, static_cast<float2*>(gcbias), d.L, d.M, B, d.cpo, d.dense);
      B200_CHECK_LAUNCH();
    }
  } else {
    const float2* wn = static_cast<const float2*>(w);
    if (gx) {
      const long long total = (long long)d.L * d.M * B * d.cpi;
      const unsigned nb = (unsigned)((total + 255) / 256);
      if (op == B200SHT_OP_DIAGONAL) mix_permode_kernel<B200SHT_OP_DIAGONAL, 1><<<nb, 256, 0, st>>>(gy, wn, gx, d);
      else if (op == B200SHT_OP_SEP_DHCONV) mix_permode_kernel<B200SHT_OP_SEP_DHCONV, 1><<<nb, 256, 0, st>>>(gy, wn, gx, d);
      else if (op == B200SHT_OP_SEP_DIAGONAL) mix_permode_kernel<B200SHT_OP_SEP_DIAGONAL, 1><<<nb, 256, 0, st>>>(gy, wn, gx, d);
      else { set_error("mix_backward: unknown operator %d", op); return B200SHT_ERR_INVALID; }
      B200_CHECK_LAUNCH();
    }
    if (gw) {
      float2* g2 = static_cast<float2*>(gw);
      long long total;
      if (op == B200SHT_OP_DIAGONAL) {
        total = (long long)G * d.Cig * d.Cog * d.L * d.M;
        mix_permode_wgrad_kernel<B200SHT_OP_DIAGONAL><<<(unsigned)((total + 255) / 256), 256, 0, st>>>(x, gy, g2, d);
      } else if (op == B200SHT_OP_SEP_DHCONV) {
        total = (long long)G * d.Cig * d.L;
        mix_permode_wgrad_kernel<B200SHT_OP_SEP_DHCONV><<<(unsigned)((total + 255) / 256), 256, 0, st>>>(x, gy, g2, d);
      } else {
        total = (long long)G * d.Cig * d.L * d.M;
        mix_permode_wgrad_kernel<B200SHT_OP_SEP_DIAGONAL><<<(unsigned)((total + 255) / 256), 256, 0, st>>>(x, gy, g2, d);
      }
      B200_CHECK_LAUNCH();
    }
  }
  return 0;
}

}  // namespace b200sht
