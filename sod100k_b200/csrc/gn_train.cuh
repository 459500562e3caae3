// gn_train.cuh — GroupNorm(groups, C) + PReLU for training (csnet_train_gn_*): F.prelu(F.group_norm(z, groups, gamma, beta, eps), a).
//
// A group of image n is the contiguous span of (C / groups) planes starting at channel g C / groups, L = (C / groups) HW values.
//   stats   one block per (image, group): one pass of shifted sums of (z - K) and (z - K)^2 in fp32 per thread, K the mean of 32
//           samples spread over the span, merged in double by a fixed tree; mean = K + S1 / L, var = (S2 - S1^2 / L) / L
//   fwd     one block per (channel, image): u = gamma (z - mean) r + beta, r = rsqrtf(var + eps); y = u > 0 ? u : a u
//   bwd     gn_bwd_reduce_kernel: per (image, channel) S_du = sum du, S_dux = sum du xhat, S_a = sum dy u [u <= 0]
//           (du = dy prelu'(u), xhat = (z - mean) r) by a fixed tree;
//           gn_bwd_dz_kernel: per (image, group) G1 = sum_c gamma_c S_du, G2 = sum_c gamma_c S_dux in channel order (double), then
//           dz = r (gamma du - G1 / L - xhat G2 / L); the image-0 blocks also write dgamma = sum_n S_dux, dbeta = sum_n S_du,
//           dslope = sum_n S_a with the images in order.
// No atomics: every sum has one order, so the results are the same bits on every run.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace csnet {
namespace gn {

constexpr int kStatThreads = 512;
constexpr int kThreads = 256;

template <int T>
__device__ __forceinline__ double block_sum_d(double v, double* sh) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) sh[w] = v;
  __syncthreads();
  double r = 0.0;
  if (threadIdx.x == 0)
    for (int i = 0; i < T / 32; ++i) r += sh[i];
  return r;                                                     // valid in thread 0
}

template <int T>
__device__ __forceinline__ float block_sum_f(float v, float* sh) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) sh[w] = v;
  __syncthreads();
  float r = 0.f;
  if (threadIdx.x == 0)
    for (int i = 0; i < T / 32; ++i) r += sh[i];
  return r;
}

__global__ void __launch_bounds__(kStatThreads) gn_stats_kernel(const float* __restrict__ z, int C, int HW, int groups, float* mean,
                                                                float* var) {
  __shared__ double sh[kStatThreads / 32];
  __shared__ float Ks;
  const int ng = blockIdx.x, n = ng / groups, g = ng - n * groups, cg = C / groups;
  const int64_t L = (int64_t)cg * HW;
  const float* p = z + ((int64_t)n * C + (int64_t)g * cg) * HW;
  if (threadIdx.x < 32) {
    float v = __ldg(p + ((int64_t)threadIdx.x * L) / 32);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (threadIdx.x == 0) Ks = v * (1.f / 32.f);
  }
  __syncthreads();
  const float K = Ks;
  float s = 0.f, q = 0.f;
  for (int64_t i = threadIdx.x; i < L; i += kStatThreads) {
    const float d = __ldg(p + i) - K;
    s += d;
    q = fmaf(d, d, q);
  }
  const double S1 = block_sum_d<kStatThreads>((double)s, sh);
  const double S2 = block_sum_d<kStatThreads>((double)q, sh);
  if (threadIdx.x == 0) {
    const double m1 = S1 / (double)L, vv = (S2 - S1 * m1) / (double)L;
    mean[ng] = (float)((double)K + m1);
    var[ng] = (float)(vv > 0.0 ? vv : 0.0);
  }
}

__global__ void __launch_bounds__(kThreads) gn_prelu_fwd_kernel(const float* __restrict__ z, float* __restrict__ y, int C, int HW,
                                                                int groups, const float* mean, const float* var, const float* gamma,
                                                                const float* beta, const float* slope, float eps) {
  const int c = blockIdx.x, n = blockIdx.y, ng = n * groups + c / (C / groups);
  const float m = mean[ng], r = rsqrtf(var[ng] + eps), gm = gamma[c], bt = beta[c], a = slope[c];
  const float* p = z + ((int64_t)n * C + c) * HW;
  float* o = y + ((int64_t)n * C + c) * HW;
  for (int i = threadIdx.x; i < HW; i += kThreads) {
    const float u = fmaf(gm, (p[i] - m) * r, bt);
    o[i] = u > 0.f ? u : a * u;
  }
}

__global__ void __launch_bounds__(kThreads) gn_bwd_reduce_kernel(const float* __restrict__ z, const float* __restrict__ dy, int C, int HW,
                                                                 int groups, const float* mean, const float* var, const float* gamma,
                                                                 const float* beta, const float* slope, float eps, float* ws) {
  __shared__ float sh[kThreads / 32];
  const int c = blockIdx.x, n = blockIdx.y, ng = n * groups + c / (C / groups);
  const float m = mean[ng], r = rsqrtf(var[ng] + eps), gm = gamma[c], bt = beta[c], a = slope[c];
  const float* p = z + ((int64_t)n * C + c) * HW;
  const float* d = dy + ((int64_t)n * C + c) * HW;
  float s_du = 0.f, s_dux = 0.f, s_a = 0.f;
  for (int i = threadIdx.x; i < HW; i += kThreads) {
    const float xh = (p[i] - m) * r, u = fmaf(gm, xh, bt), g = d[i];
    const float du = u > 0.f ? g : a * g;
    s_du += du;
    s_dux = fmaf(du, xh, s_dux);
    if (!(u > 0.f)) s_a = fmaf(g, u, s_a);
  }
  s_du = block_sum_f<kThreads>(s_du, sh);
  s_dux = block_sum_f<kThreads>(s_dux, sh);
  s_a = block_sum_f<kThreads>(s_a, sh);
  if (threadIdx.x == 0) {
    float* w = ws + ((int64_t)n * C + c) * 3;
    w[0] = s_du; w[1] = s_dux; w[2] = s_a;
  }
}

__global__ void __launch_bounds__(kThreads) gn_bwd_dz_kernel(const float* __restrict__ z, const float* __restrict__ dy, float* __restrict__ dz,
                                                             int N, int C, int HW, int groups, const float* mean, const float* var,
                                                             const float* gamma, const float* beta, const float* slope, float eps,
                                                             const float* ws, float* dgamma, float* dbeta, float* dslope) {
  __shared__ float G[2];
  const int c = blockIdx.x, n = blockIdx.y, cg = C / groups, g0 = (c / cg) * cg, ng = n * groups + c / cg;
  if (threadIdx.x == 0) {
    double g1 = 0.0, g2 = 0.0;
    for (int k = 0; k < cg; ++k) {
      const float* w = ws + ((int64_t)n * C + g0 + k) * 3;
      g1 += (double)gamma[g0 + k] * (double)w[0];
      g2 += (double)gamma[g0 + k] * (double)w[1];
    }
    const double L = (double)cg * (double)HW;
    G[0] = (float)(g1 / L);
    G[1] = (float)(g2 / L);
    if (n == 0) {
      float sg = 0.f, sb = 0.f, sa = 0.f;
      for (int i = 0; i < N; ++i) {
        const float* w = ws + ((int64_t)i * C + c) * 3;
        sb += w[0]; sg += w[1]; sa += w[2];
      }
      dgamma[c] = sg; dbeta[c] = sb; dslope[c] = sa;
    }
  }
  __syncthreads();
  const float m = mean[ng], r = rsqrtf(var[ng] + eps), gm = gamma[c], bt = beta[c], a = slope[c], m1 = G[0], m2 = G[1];
  const float* p = z + ((int64_t)n * C + c) * HW;
  const float* d = dy + ((int64_t)n * C + c) * HW;
  float* o = dz + ((int64_t)n * C + c) * HW;
  for (int i = threadIdx.x; i < HW; i += kThreads) {
    const float xh = (p[i] - m) * r, u = fmaf(gm, xh, bt), g = d[i];
    const float du = u > 0.f ? g : a * g;
    o[i] = r * (gm * du - m1 - xh * m2);
  }
}

}  // namespace gn
}  // namespace csnet
