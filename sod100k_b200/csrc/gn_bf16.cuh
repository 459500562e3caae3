// gn_bf16.cuh — GroupNorm(groups, C) + PReLU for training with bf16 activation storage (csnet_train_gn_*_bf16): gn_train.cuh's
// kernels on bf16 z / y / dy / dz.  Each load is widened to fp32 exactly and each store rounded once to nearest-even bf16; the
// statistics, the sums and their fixed order are gn_train.cuh's, so the results are the same bits on every run.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "gn_train.cuh"

namespace csnet {
namespace gn {

using bf16 = __nv_bfloat16;
__device__ __forceinline__ float ldf(const bf16* p) { return __bfloat162float(*p); }

__global__ void __launch_bounds__(kStatThreads) gn_stats_bf16_kernel(const bf16* __restrict__ z, int C, int HW, int groups, float* mean,
                                                                     float* var) {
  __shared__ double sh[kStatThreads / 32];
  __shared__ float Ks;
  const int ng = blockIdx.x, n = ng / groups, g = ng - n * groups, cg = C / groups;
  const int64_t L = (int64_t)cg * HW;
  const bf16* p = z + ((int64_t)n * C + (int64_t)g * cg) * HW;
  if (threadIdx.x < 32) {
    float v = ldf(p + ((int64_t)threadIdx.x * L) / 32);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (threadIdx.x == 0) Ks = v * (1.f / 32.f);
  }
  __syncthreads();
  const float K = Ks;
  float s = 0.f, q = 0.f;
  for (int64_t i = threadIdx.x; i < L; i += kStatThreads) {
    const float d = ldf(p + i) - K;
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

__global__ void __launch_bounds__(kThreads) gn_prelu_fwd_bf16_kernel(const bf16* __restrict__ z, bf16* __restrict__ y, int C, int HW,
                                                                     int groups, const float* mean, const float* var, const float* gamma,
                                                                     const float* beta, const float* slope, float eps) {
  const int c = blockIdx.x, n = blockIdx.y, ng = n * groups + c / (C / groups);
  const float m = mean[ng], r = rsqrtf(var[ng] + eps), gm = gamma[c], bt = beta[c], a = slope[c];
  const bf16* p = z + ((int64_t)n * C + c) * HW;
  bf16* o = y + ((int64_t)n * C + c) * HW;
  for (int i = threadIdx.x; i < HW; i += kThreads) {
    const float u = fmaf(gm, (ldf(p + i) - m) * r, bt);
    o[i] = __float2bfloat16_rn(u > 0.f ? u : a * u);
  }
}

__global__ void __launch_bounds__(kThreads) gn_bwd_reduce_bf16_kernel(const bf16* __restrict__ z, const bf16* __restrict__ dy, int C,
                                                                      int HW, int groups, const float* mean, const float* var,
                                                                      const float* gamma, const float* beta, const float* slope,
                                                                      float eps, float* ws) {
  __shared__ float sh[kThreads / 32];
  const int c = blockIdx.x, n = blockIdx.y, ng = n * groups + c / (C / groups);
  const float m = mean[ng], r = rsqrtf(var[ng] + eps), gm = gamma[c], bt = beta[c], a = slope[c];
  const bf16* p = z + ((int64_t)n * C + c) * HW;
  const bf16* d = dy + ((int64_t)n * C + c) * HW;
  float s_du = 0.f, s_dux = 0.f, s_a = 0.f;
  for (int i = threadIdx.x; i < HW; i += kThreads) {
    const float xh = (ldf(p + i) - m) * r, u = fmaf(gm, xh, bt), g = ldf(d + i);
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

__global__ void __launch_bounds__(kThreads) gn_bwd_dz_bf16_kernel(const bf16* __restrict__ z, const bf16* __restrict__ dy,
                                                                  bf16* __restrict__ dz, int N, int C, int HW, int groups,
                                                                  const float* mean, const float* var, const float* gamma,
                                                                  const float* beta, const float* slope, float eps, const float* ws,
                                                                  float* dgamma, float* dbeta, float* dslope) {
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
  const bf16* p = z + ((int64_t)n * C + c) * HW;
  const bf16* d = dy + ((int64_t)n * C + c) * HW;
  bf16* o = dz + ((int64_t)n * C + c) * HW;
  for (int i = threadIdx.x; i < HW; i += kThreads) {
    const float xh = (ldf(p + i) - m) * r, u = fmaf(gm, xh, bt), g = ldf(d + i);
    const float du = u > 0.f ? g : a * g;
    o[i] = __float2bfloat16_rn(r * (gm * du - m1 - xh * m2));
  }
}

}  // namespace gn
}  // namespace csnet
