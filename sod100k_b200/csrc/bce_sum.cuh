// bce_sum.cuh — F.binary_cross_entropy_with_logits(reduction='sum') / divisor (CSF+Res2Net/solver.py:101-102), deterministic.
//
// bce_sum_kernel: block b sums the terms max(z, 0) - z t + log1p(exp(-|z|)) of its grid-stride elements in a fixed order, reduces
// them over the block in a fixed tree and stores part[b]; it also writes dz = (sigmoid(z) - t) * inv_d, inv_d = f32(1 / divisor),
// autograd's gradient through the division.  bce_sum_merge_kernel adds the parts in block order and divides by (float)divisor.  The
// block count is a function of n alone, so a loss has the same bits on every run and every GPU; no floating-point atomics.
// csnet_train_bce_sum (train_ops.cu) is the entry point; tests/test_gpu_csf_train_data.py checks both kernels against float64.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

namespace csnet {
namespace bce {

constexpr int kThreads = 256;
constexpr int kPerThread = 8;
constexpr int kMaxBlocks = 1024;

// Sum over the block in a fixed order: shuffle tree within each warp, then the warps' sums in warp order by warp 0.  Valid in thread 0.
__device__ __forceinline__ float block_sum(float v) {
  __shared__ float part[kThreads / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x < 32) {
    v = threadIdx.x < kThreads / 32 ? part[threadIdx.x] : 0.f;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  }
  return v;
}

__global__ void __launch_bounds__(kThreads) bce_sum_kernel(const float* __restrict__ z, const float* __restrict__ t, float* __restrict__ dz,
                                                           float* __restrict__ part, int64_t n, float inv_d) {
  float s = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
    const float v = z[i], y = t[i];
    s += fmaxf(v, 0.f) - v * y + log1pf(expf(-fabsf(v)));
    if (dz) dz[i] = (1.f / (1.f + expf(-v)) - y) * inv_d;
  }
  s = block_sum(s);
  if (threadIdx.x == 0) part[blockIdx.x] = s;
}

__global__ void __launch_bounds__(kThreads) bce_sum_merge_kernel(const float* __restrict__ part, int parts, float divisor,
                                                                 float* __restrict__ loss) {
  float s = 0.f;
  for (int p = threadIdx.x; p < parts; p += kThreads) s += part[p];
  s = block_sum(s);
  if (threadIdx.x == 0) loss[0] = s / divisor;
}

// Blocks of the first kernel, i.e. floats of `part` the caller provides.
inline int blocks(int64_t n) {
  const int64_t want = (n + kThreads * kPerThread - 1) / (kThreads * kPerThread);
  return (int)(want < kMaxBlocks ? want : kMaxBlocks);
}

inline void launch(const float* z, const float* t, float* dz, float* part, float* loss, int64_t n, int divisor, cudaStream_t stream) {
  const int b = blocks(n);
  bce_sum_kernel<<<b, kThreads, 0, stream>>>(z, t, dz, part, n, (float)(1.0 / (double)divisor));
  bce_sum_merge_kernel<<<1, kThreads, 0, stream>>>(part, b, (float)divisor, loss);
}

}  // namespace bce
}  // namespace csnet
