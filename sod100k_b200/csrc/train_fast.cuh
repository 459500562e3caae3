// train_fast.cuh — the fp32 __global__s of the register-tiled training kernels (CSNet_training/train.py:203-216: F.conv2d forward, its data
// and weight gradients as autograd computes them; model/csnet.py:664-726 for the paths of a gOctaveConv).
//
// Everything here is DENSE: stride 1, same spatial size in and out, zero padding pad = dil * (k / 2).  The down-sampling a path
// may carry (2x2 average of a stride-2 conv, max-pool of a high -> low path) is materialised once by pool_fwd_kernel (with the
// arg-max, so the backward routes exactly like max_pool2d: first maximum in row-major order), so the three convolution kernels
// never see it.  The per-thread bodies live in train_body.cuh, templated on the activation type; these are their fp32 instances
// (train_bf16.cu holds the bf16-storage ones).  fp32 storage and fp32 FMA (the parity configuration: gradients within 1e-3 of autograd); the FP32 pipe is the
// roofline of these kernels, so each thread owns a 4 px x 16 channel (forward / dgrad) or 4 x 4 (x 3 taps) (wgrad) register tile
// and reads its operands from shared memory as 16-byte vectors.
//
//   conv1x1_kernel<PX, VEC> / conv1x1_narrow_kernel   every 1x1 mix and its data gradient: inputs global -> registers (each input element is
//                         needed by exactly one thread), weights in shared memory, several channels of loads issued ahead of their FMAs.
//   conv_fwd_kernel<KS>   3x3 (KS = 3, dil 1) and dilated (KS = 0) mixes: dst = sum over conv paths (K-concatenated in the loop) + bilinear
//                         resample-add paths; with `transposed` the data gradient of one path (weights read as [co][flipped tap][ci]
//                         while staging); input tile with halo staged by cp.async.
//   conv_wgrad_kernel<KS> dw[ci][tap][co] = sum_{n,y,x} in[n][ci][y+ky-1][x+kx-1] * ddst[n][co][y][x]: per-block partials over a
//                         share of the (image, row band) units, two cp.async stages in flight, interleaved 4 x 4 thread tiles on a
//                         bank-conflict-free channel pitch, merged IN ORDER by reduce_partials_kernel (no atomics).
//   dw3_kernel / dw3_bwd_kernel (dw3_wgrad_kernel)   depthwise 3x3 (Conv2dX100 groups=C): a 4-pixel column strip per thread sliding down
//                         the rows; the backward produces dx and the dw partials in one pass over dy.
//   pool_fwd / pool2_fwd / pool_bwd(4), resample_bwd_kernel<UP>   the pooling a path carries (with arg-max) and the bilinear adjoint.
#pragma once
#include "train_body.cuh"

namespace csnet {
namespace tf {

template <int KS>
__global__ void __launch_bounds__(kT, 2) conv_fwd_kernel(const __grid_constant__ ConvArgs A) {
  extern __shared__ __align__(16) float smem[];
  conv_fwd_body<KS, float, float>(A, smem);
}

template <int PX, bool VEC>
__global__ void __launch_bounds__(kT, 2) conv1x1_kernel(const __grid_constant__ C1Args A) {
  extern __shared__ __align__(16) float wsm[];                          // [wrows][Cpad]: every path's weights, zero outside its slice
  conv1x1_body<PX, VEC, float, float>(A, wsm);
}

__global__ void __launch_bounds__(kT, 3) conv1x1_narrow_kernel(const __grid_constant__ C1Args A) {
  extern __shared__ __align__(16) float wsm[];
  conv1x1_narrow_body<float, float>(A, wsm);
}

template <int KS>
__global__ void __launch_bounds__(kT, 2) conv_wgrad_kernel(const __grid_constant__ WgradArgs A) {
  extern __shared__ __align__(16) float smem[];
  conv_wgrad_body<KS, float, float>(A, smem);
}

// out[e] = scale * sum over parts (in part order) of part[p][e]
__global__ void __launch_bounds__(kT) reduce_partials_kernel(const float* __restrict__ part, int parts, int n, float scale, float* __restrict__ out) {
  const int e = blockIdx.x * kT + threadIdx.x;
  if (e >= n) return;
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
  int p = 0;
  for (; p + 4 <= parts; p += 4) {
    s0 += part[(size_t)p * n + e]; s1 += part[(size_t)(p + 1) * n + e]; s2 += part[(size_t)(p + 2) * n + e]; s3 += part[(size_t)(p + 3) * n + e];
  }
  for (; p < parts; ++p) s0 += part[(size_t)p * n + e];
  out[e] = ((s0 + s1) + (s2 + s3)) * scale;
}

__global__ void __launch_bounds__(kT) pool_fwd_kernel(const float* __restrict__ src, int N, int Cs, int c0, int cin, int Hs, int Ws, int pre_avg,
                                                      int pool, float* __restrict__ dst, uint8_t* __restrict__ idx) {
  pool_fwd_body(src, N, Cs, c0, cin, Hs, Ws, pre_avg, pool, dst, idx);
}

__global__ void __launch_bounds__(kT) pool2_fwd_kernel(const float* __restrict__ src, int N, int Cs, int c0, int cin, int Hs, int Ws,
                                                       float* __restrict__ dst, uint8_t* __restrict__ idx) {
  pool2_fwd_body(src, N, Cs, c0, cin, Hs, Ws, dst, idx);
}

__global__ void __launch_bounds__(kT) pool_bwd_kernel(const float* __restrict__ dpool, const uint8_t* __restrict__ idx, int N, int cin, int Hs, int Ws,
                                                      int pre_avg, int pool, float* __restrict__ dsrc) {
  pool_bwd_body(dpool, idx, N, cin, Hs, Ws, pre_avg, pool, dsrc);
}

__global__ void __launch_bounds__(kT) pool_bwd4_kernel(const float* __restrict__ dpool, const uint8_t* __restrict__ idx, int N, int cin, int Hs, int Ws,
                                                       int pre_avg, int pool, float* __restrict__ dsrc) {
  pool_bwd4_body(dpool, idx, N, cin, Hs, Ws, pre_avg, pool, dsrc);
}

template <int UP>
__global__ void __launch_bounds__(kT) resample_bwd_kernel(const float* __restrict__ ddst, int N, int C, int H, int W, int cout0, int cin, int Hs, int Ws,
                                                          float* __restrict__ dsrc) {
  resample_bwd_body<UP>(ddst, N, C, H, W, cout0, cin, Hs, Ws, dsrc);
}

__global__ void __launch_bounds__(kT) dw3_kernel(const float* __restrict__ x, const float* __restrict__ w, float* __restrict__ y, int N, int C, int H,
                                                 int W, float scale, int flip, int quads, int rows) {
  dw3_body(x, w, y, N, C, H, W, scale, flip, quads, rows);
}

__global__ void __launch_bounds__(kT) dw3_wgrad_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ part, int N, int C,
                                                       int H, int W, int quads, int rows) {
  dw3_wgrad_body(x, dy, part, N, C, H, W, quads, rows);
}

__global__ void __launch_bounds__(kT) dw3_bwd_kernel(const float* __restrict__ x, const float* __restrict__ dy, const float* __restrict__ w,
                                                     float* __restrict__ dx, float* __restrict__ part, int N, int C, int H, int W, float scale,
                                                     int quads, int rows) {
  dw3_bwd_body(x, dy, w, dx, part, N, C, H, W, scale, quads, rows);
}

}  // namespace tf
}  // namespace csnet
