// ComplexReLU on packed spectral tensors (replaces /root/reference/makani/models/common/activations.py:88-127).
// Elementwise over the stored block-triangle; bias is per channel ([C]) or null (= 0).
#include "common.cuh"

namespace b200sht {

__device__ __forceinline__ float leaky(float x, float s) { return x > 0.f ? x : s * x; }
__device__ __forceinline__ float dleaky(float x, float s) { return x > 0.f ? 1.f : s; }

template <bool BWD>
__global__ void complex_relu_kernel(int mode, const float* __restrict__ x, const float* __restrict__ bias, float slope, const float* __restrict__ gy,
                                    float* __restrict__ out, int L, int M, int B, int C, int cp, int dense) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)L * M * B * cp;
  if (idx >= total) return;
  const int c = (int)(idx % cp);
  long long rest = idx / cp;
  const int b = (int)(rest % B); rest /= B;
  const int m = (int)(rest % M);
  const int l = (int)(rest / M);
  if (m >= mend_d(l, M, dense)) return;
  const size_t base = ((size_t)l * M + m) * 2 * B * cp + (size_t)b * cp + c;
  const size_t plane = (size_t)B * cp;
  if (c >= C) {  // keep the channel padding at zero
    out[base] = 0.f; out[base + plane] = 0.f;
    return;
  }
  const float xr = x[base], xi = x[base + plane];
  const float bb = bias ? bias[c] : 0.f;
  float o_r, o_i;
  if (!BWD) {
    if (mode == 0) { o_r = leaky(xr, slope); o_i = xi; }
    else if (mode == 1) { o_r = leaky(xr, slope); o_i = leaky(xi, slope); }
    else if (mode == 2) {
      const float za = sqrtf(xr * xr + xi * xi);
      if (za > 0.f && za + bb > 0.f) { const float s = (za + bb) / za; o_r = s * xr; o_i = s * xi; }
      else { o_r = 0.f; o_i = 0.f; }
    } else {
      const float ang = atan2f(xi, xr) - bb;
      const bool cond = (ang >= 0.f) && (ang < 1.57079632679489661923f);
      o_r = cond ? xr : slope * xr; o_i = cond ? xi : slope * xi;
    }
  } else {
    const float gr = gy[base], gi = gy[base + plane];
    if (mode == 0) { o_r = gr * dleaky(xr, slope); o_i = gi; }
    else if (mode == 1) { o_r = gr * dleaky(xr, slope); o_i = gi * dleaky(xi, slope); }
    else if (mode == 2) {
      const float za = sqrtf(xr * xr + xi * xi);
      if (za > 0.f && za + bb > 0.f) {
        const float iz3 = bb / (za * za * za);
        const float drr = 1.f + iz3 * xi * xi, dri = -iz3 * xr * xi, dii = 1.f + iz3 * xr * xr;
        o_r = gr * drr + gi * dri;
        o_i = gr * dri + gi * dii;
      } else { o_r = 0.f; o_i = 0.f; }
    } else {
      const float ang = atan2f(xi, xr) - bb;
      const bool cond = (ang >= 0.f) && (ang < 1.57079632679489661923f);
      o_r = cond ? gr : slope * gr; o_i = cond ? gi : slope * gi;
    }
  }
  out[base] = o_r;
  out[base + plane] = o_i;
}

// modulus bias gradient: gbias[c] = sum over the stored triangle and batch of (gr xr + gi xi) / |z| where |z| > 0 and |z| + bias[c] > 0.
// One block per channel in a fixed order (per-thread strided sums, then a fixed tree): the same bits on every run.
__global__ void complex_relu_bias_grad_kernel(const float* __restrict__ x, const float* __restrict__ bias, const float* __restrict__ gy,
                                              float* __restrict__ gbias, int L, int M, int B, int cp, int dense) {
  const int c = blockIdx.x;
  const float bb = bias ? bias[c] : 0.f;
  const size_t plane = (size_t)B * cp;
  float s = 0.f;
  for (int l = 0; l < L; ++l) {
    const int nrows = mend_d(l, M, dense) * B;
    for (int row = threadIdx.x; row < nrows; row += blockDim.x) {
      const int m = row / B, b = row % B;
      const size_t base = ((size_t)l * M + m) * 2 * plane + (size_t)b * cp + c;
      const float xr = x[base], xi = x[base + plane];
      const float za = sqrtf(xr * xr + xi * xi);
      if (za > 0.f && za + bb > 0.f) s += (gy[base] * xr + gy[base + plane] * xi) / za;
    }
  }
  __shared__ float part[32];
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    float a = threadIdx.x < (blockDim.x >> 5) ? part[threadIdx.x] : 0.f;
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    if (threadIdx.x == 0) gbias[c] = a;
  }
}

int complex_relu_fwd(const Plan* pl, int mode, const float* x, const float* bias, float slope, float* y, int B, int C, cudaStream_t st) {
  B200_REQUIRE(mode >= 0 && mode <= 3, "complex_relu: unknown mode %d", mode);
  const int cp = round_up(C, 4);
  const long long total = (long long)pl->lmax * pl->mmax * B * cp;
  complex_relu_kernel<false><<<(unsigned)((total + 255) / 256), 256, 0, st>>>(mode, x, bias, slope, nullptr, y, pl->lmax, pl->mmax, B, C, cp, pl->dense);
  B200_CHECK_LAUNCH();
  return 0;
}

int complex_relu_bwd(const Plan* pl, int mode, const float* x, const float* bias, float slope, const float* gy, float* gx, float* gbias, int B,
                     int C, cudaStream_t st) {
  B200_REQUIRE(mode >= 0 && mode <= 3, "complex_relu: unknown mode %d", mode);
  const int cp = round_up(C, 4);
  const long long total = (long long)pl->lmax * pl->mmax * B * cp;
  if (gbias && mode == 2) {  // before gx is written: gx may alias gy or x
    complex_relu_bias_grad_kernel<<<C, 256, 0, st>>>(x, bias, gy, gbias, pl->lmax, pl->mmax, B, cp, pl->dense);
    B200_CHECK_LAUNCH();
  } else if (gbias) {
    B200_CHECK_CUDA(cudaMemsetAsync(gbias, 0, sizeof(float) * C, st));
  }
  complex_relu_kernel<true><<<(unsigned)((total + 255) / 256), 256, 0, st>>>(mode, x, bias, slope, gy, gx, pl->lmax, pl->mmax, B, C, cp, pl->dense);
  B200_CHECK_LAUNCH();
  return 0;
}

}  // namespace b200sht
