// Spherical noise (makani's IsotropicGaussianRandomFieldS2 / DiffusionNoiseS2, DESIGN.md section 4.12): the state update from host-drawn
// standard normals, the state -> synthesis-input conversion and the weight gradient of a learnable per-(l, m) sigma.
//
// state: fp32 [B][T][C][L][M][2] (makani's layout; read as complex [B][T*C][L][M]).  The AR step and the memoryless update round exactly as
// torch's elementwise sequence in makani/models/noise.py does (separate multiplies and adds, IEEE sqrt and division), so they are compared
// bit for bit; the T x T discount of the stationary redraw is an fp32 FMA sum.
#include "common.cuh"

namespace b200sht {

// one thread per (b, c, l, m) column: it owns all T steps of that column, so the history shifts in place without a race
__global__ void __launch_bounds__(256) noise_update_kernel(float2* __restrict__ state, const float2* __restrict__ xi, const float* __restrict__ sigma,
                                                           const float* __restrict__ phi, const float* __restrict__ discount, int B, int T, int C,
                                                           int L, int M, int mode, int reflect) {
  const long long LM = (long long)L * M, CLM = C * LM;
  const long long n = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= B * CLM) return;
  const int b = (int)(n / CLM);
  const long long rem = n - b * CLM;
  const int c = (int)(rem / LM);
  const long long lm = rem - c * LM;
  const int l = (int)(lm / M);
  auto at = [&](int t) { return ((long long)b * T + t) * CLM + c * LM + lm; };
  auto flip = [&](float v) { return reflect ? -v : v; };

  if (mode == B200SHT_NOISE_BASE) {  // state = r xi
    for (int t = 0; t < T; ++t) {
      const float2 x = xi[at(t)];
      state[at(t)] = make_float2(flip(x.x), flip(x.y));
    }
    return;
  }
  const float s = sigma[(long long)c * L + l];
  const float p = phi[c];
  if (mode == B200SHT_NOISE_AR) {  // new step = phi state[T-1] + r sigma xi; older steps move down by one
    const float2 x = xi[(long long)b * CLM + c * LM + lm];
    const float2 last = state[at(T - 1)];
    for (int t = 0; t + 1 < T; ++t) state[at(t)] = state[at(t + 1)];
    state[at(T - 1)] = make_float2(__fadd_rn(__fmul_rn(p, last.x), flip(__fmul_rn(s, x.x))),
                                   __fadd_rn(__fmul_rn(p, last.y), flip(__fmul_rn(s, x.y))));
    return;
  }
  // stationary redraw: w = r sigma xi, w[0] /= sqrt(1 - phi^2), then state[t] = sum_{q <= t} discount[c][t][q] w[q]
  const float d = __fsqrt_rn(__fsub_rn(1.f, __fmul_rn(p, p)));
  for (int t = 0; t < T; ++t) {
    const float2 x = xi[at(t)];
    float2 w = make_float2(flip(__fmul_rn(s, x.x)), flip(__fmul_rn(s, x.y)));
    if (t == 0) w = make_float2(__fdiv_rn(w.x, d), __fdiv_rn(w.y, d));
    state[at(t)] = w;
  }
  if (T > 1) {
    const float* D = discount + (long long)c * T * T;
    for (int t = T - 1; t >= 0; --t) {  // downwards: row t reads w[0 .. t], which rows above it have not overwritten
      float2 acc = make_float2(0.f, 0.f);
      for (int q = 0; q <= t; ++q) {
        const float2 w = state[at(q)];
        acc.x = fmaf(D[t * T + q], w.x, acc.x);
        acc.y = fmaf(D[t * T + q], w.y, acc.y);
      }
      state[at(t)] = acc;
    }
  }
}

// torch computes `state / math.sqrt(2)` on CUDA as a multiply by the fp32 reciprocal of the fp32 divisor
static float inv_sqrt2() { return 1.0f / (float)1.4142135623730951; }

// (a + i b) sigma as torch multiplies a complex64 by a real tensor promoted to complex (sigma + 0 i): (a sigma - b 0) + i (a 0 + b sigma).
// The zero products only decide the sign of a zero result (where sigma = 0, m > l), and keep it torch's bit for bit.
__device__ __forceinline__ float2 noise_coeff(float2 v, const float* sigma, long long lm, float inv) {
  if (!sigma) return v;
  const float s = sigma[lm];
  const float a = __fmul_rn(v.x, inv), b = __fmul_rn(v.y, inv);
  return make_float2(__fsub_rn(__fmul_rn(a, s), __fmul_rn(b, 0.f)), __fadd_rn(__fmul_rn(a, 0.f), __fmul_rn(b, s)));
}

// packed spec [L][M][2][B][cp] of the complex [B][TC][L][M] state, as b200sht_spec_pack writes it: block per (l, b), a 32 m x 32 c tile
__global__ void __launch_bounds__(256) noise_spectrum_packed_kernel(const float2* __restrict__ state, const float* __restrict__ sigma,
                                                                    float* __restrict__ spec, int L, int M, int B, int TC, int cp, float inv) {
  __shared__ float tile[2][32][33];
  const int l = blockIdx.z / B, b = blockIdx.z % B;
  const int m0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  if (l < lstart(m0)) return;  // the whole tile lies below the block triangle (lstart is constant over 32 aligned orders)
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int JP = 2 * B * cp;
  for (int cc = ty; cc < 32; cc += 8) {
    const int c = c0 + cc, m = m0 + tx;
    float2 v = make_float2(0.f, 0.f);
    if (c < TC && m < M) v = noise_coeff(state[((long long)(b * TC + c) * L + l) * M + m], sigma, (long long)l * M + m, inv);
    tile[0][tx][cc] = v.x;
    tile[1][tx][cc] = v.y;
  }
  __syncthreads();
  for (int mm = ty; mm < 32; mm += 8) {
    const int m = m0 + mm, c = c0 + tx;
    if (m < M && c < cp) {
      float* row = spec + ((long long)l * M + m) * JP;
      row[(0 * B + b) * cp + c] = tile[0][mm][tx];
      row[(1 * B + b) * cp + c] = tile[1][mm][tx];
    }
  }
}

__global__ void __launch_bounds__(256) noise_spectrum_complex_kernel(const float2* __restrict__ state, const float* __restrict__ sigma,
                                                                     float2* __restrict__ out, long long n, long long LM, float inv) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = noise_coeff(state[i], sigma, i % LM, inv);
}

// dsigma[l][m] = sum_b sum_c Re(conj(g) state / sqrt 2): one fp32 FMA chain per (l, m), b outer, c inner, re before im.  Both kernels below
// sum in this order, so the result does not depend on the gradient's layout and is bit-identical run to run.
__device__ __forceinline__ float sigma_grad_step(float acc, float gr, float gi, float2 z, float inv) {
  acc = fmaf(gr, __fmul_rn(z.x, inv), acc);
  return fmaf(gi, __fmul_rn(z.y, inv), acc);
}

// complex gradient [B][TC][L][M]: one thread per (l, m); consecutive threads read consecutive (l, m) of g and of the state
__global__ void __launch_bounds__(256) noise_sigma_grad_complex_kernel(const float2* __restrict__ state, const float2* __restrict__ grad,
                                                                       float* __restrict__ dsigma, int B, int TC, long long LM, float inv) {
  const long long lm = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (lm >= LM) return;
  float acc = 0.f;
  for (int b = 0; b < B; ++b)
    for (int c = 0; c < TC; ++c) {
      const long long i = (long long)(b * TC + c) * LM + lm;
      acc = sigma_grad_step(acc, grad[i].x, grad[i].y, state[i], inv);
    }
  dsigma[lm] = acc;
}

// packed gradient [L][M][2][B][cp]: block per (l, 32 orders); per (b, 32 channels) the g tile is read along c (a packed row) and the state tile
// along m, both coalesced, through shared memory; warp 0 then runs the 32 chains of the tile.  Entries l < m get 0 (l < lstart(m) is not
// stored; lstart(m) <= l < m holds zeros).
__global__ void __launch_bounds__(256) noise_sigma_grad_packed_kernel(const float2* __restrict__ state, const float* __restrict__ grad,
                                                                      float* __restrict__ dsigma, int B, int TC, int L, int M, float inv) {
  __shared__ float g_tile[2][32][33];  // [re/im][m][c]
  __shared__ float z_tile[2][32][33];  // [re/im][c][m]
  const int l = blockIdx.y, m0 = blockIdx.x * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int m = m0 + tx;
  float acc = 0.f;
  if (l >= lstart(m0)) {  // uniform over the block
    const int cp = round_up(TC, 4);
    const long long JP = 2LL * B * cp;
    for (int b = 0; b < B; ++b) {
      for (int c0 = 0; c0 < TC; c0 += 32) {
        for (int r = ty; r < 32; r += 8) {
          const int mr = m0 + r, c = c0 + tx;   // g: row (l, mr), channels along the warp
          const bool in_g = mr < M && c < TC;
          const float* row = grad + ((long long)l * M + mr) * JP;
          g_tile[0][r][tx] = in_g ? row[(0 * B + b) * cp + c] : 0.f;
          g_tile[1][r][tx] = in_g ? row[(1 * B + b) * cp + c] : 0.f;
          const int cz = c0 + r;               // state: channel cz, orders along the warp
          const float2 z = (m < M && cz < TC) ? state[((long long)(b * TC + cz) * L + l) * M + m] : make_float2(0.f, 0.f);
          z_tile[0][r][tx] = z.x;
          z_tile[1][r][tx] = z.y;
        }
        __syncthreads();
        if (ty == 0) {
          const int n = min(32, TC - c0);
          for (int cc = 0; cc < n; ++cc)
            acc = sigma_grad_step(acc, g_tile[0][tx][cc], g_tile[1][tx][cc], make_float2(z_tile[0][cc][tx], z_tile[1][cc][tx]), inv);
        }
        __syncthreads();
      }
    }
  }
  if (ty == 0 && m < M) dsigma[(long long)l * M + m] = (l >= m) ? acc : 0.f;
}

int noise_update(float* state, const float* xi, const float* sigma, const float* phi, const float* discount, int B, int T, int C, int L, int M,
                 int mode, int reflect, cudaStream_t st) {
  B200_REQUIRE(state && xi && B > 0 && T > 0 && C > 0 && L > 0 && M > 0, "noise_update: bad argument");
  B200_REQUIRE(mode == B200SHT_NOISE_AR || mode == B200SHT_NOISE_STATIONARY || mode == B200SHT_NOISE_BASE, "noise_update: unknown mode %d", mode);
  B200_REQUIRE(mode == B200SHT_NOISE_BASE || (sigma && phi), "noise_update: the AR step and the stationary redraw need sigma and phi");
  B200_REQUIRE(!(mode == B200SHT_NOISE_STATIONARY && T > 1 && !discount), "noise_update: the stationary redraw of T > 1 steps needs the discount");
  const long long cols = (long long)B * C * L * M;
  const long long blocks = (cols + 255) / 256;
  B200_REQUIRE(blocks <= 0x7fffffffLL, "noise_update: %lld columns exceed the grid limit", cols);
  noise_update_kernel<<<(unsigned)blocks, 256, 0, st>>>(reinterpret_cast<float2*>(state), reinterpret_cast<const float2*>(xi), sigma, phi, discount,
                                                       B, T, C, L, M, mode, reflect);
  B200_CHECK_LAUNCH();
  return 0;
}

int noise_spectrum(const float* state, const float* sigma, float* out, int B, int TC, int L, int M, int packed, cudaStream_t st) {
  B200_REQUIRE(state && out && B > 0 && TC > 0 && L > 0 && M > 0, "noise_spectrum: bad argument");
  const float2* s2 = reinterpret_cast<const float2*>(state);
  if (packed) {
    const int cp = round_up(TC, 4);
    dim3 grid(ceil_div(M, 32), ceil_div(cp, 32), L * B);
    B200_REQUIRE(grid.z <= 65535 && grid.y <= 65535, "noise_spectrum: lmax*B=%u or channels exceed the grid limit", grid.z);
    noise_spectrum_packed_kernel<<<grid, 256, 0, st>>>(s2, sigma, out, L, M, B, TC, cp, inv_sqrt2());
  } else {
    const long long n = (long long)B * TC * L * M;
    const long long blocks = (n + 255) / 256;
    B200_REQUIRE(blocks <= 0x7fffffffLL, "noise_spectrum: %lld coefficients exceed the grid limit", n);
    noise_spectrum_complex_kernel<<<(unsigned)blocks, 256, 0, st>>>(s2, sigma, reinterpret_cast<float2*>(out), n, (long long)L * M, inv_sqrt2());
  }
  B200_CHECK_LAUNCH();
  return 0;
}

int noise_sigma_grad(const float* state, const float* grad, float* dsigma, int B, int TC, int L, int M, int packed, cudaStream_t st) {
  B200_REQUIRE(state && grad && dsigma && B > 0 && TC > 0 && L > 0 && M > 0, "noise_sigma_grad: bad argument");
  const long long LM = (long long)L * M;
  const float2* s2 = reinterpret_cast<const float2*>(state);
  if (packed) {
    noise_sigma_grad_packed_kernel<<<dim3(ceil_div(M, 32), L), 256, 0, st>>>(s2, grad, dsigma, B, TC, L, M, inv_sqrt2());
  } else {
    noise_sigma_grad_complex_kernel<<<(unsigned)((LM + 255) / 256), 256, 0, st>>>(s2, reinterpret_cast<const float2*>(grad), dsigma, B, TC, LM,
                                                                                  inv_sqrt2());
  }
  B200_CHECK_LAUNCH();
  return 0;
}

}  // namespace b200sht
