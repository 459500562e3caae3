// gemm_f32.cuh — stride-1 convolutions (1x1, and 3x3 with dilation d and zero padding d) as an fp32 FMA implicit GEMM, in the three
// forms training needs (include/csnet_b200.h, csnet_train_conv_*).  Per image, NCHW:
//
//   fwd    C[co][p]      = sum over segments, (ci, t)  of  w_s[co][ci][t] * x_s[ci][p + off_t]          M = cout, N = HW
//   dgrad  C[ci][p]      = sum over segments, (co, t)  of  w_s[co][ci][t] * dy_s[co][p - off_t]         M = cin,  N = HW
//   wgrad  C[co][ci, t]  = sum over images, pixels p   of  dy[co][p] * x[ci][p + off_t]                 M = cout, N = cin k^2
//
// off_t is the tap's (ky - 1, kx - 1) * dil for 3x3 and 0 for 1x1; out-of-plane taps read zero.  A block computes a BM x BN tile of C
// with 256 threads, each a TM x TN register tile, over BK-deep k tiles staged in shared memory by 4-byte cp.async with zero fill
// (so padding, plane edges and the ragged ends of M, N and K cost no branches in the inner loop), STAGES deep.  A k tile never crosses
// a segment (or, for wgrad, an image): a segment's last tile is zero-filled past its end.
//
// Split-K: when the M x N tiles cannot fill the GPU, split z of S takes the k tiles [z T / S, (z + 1) T / S) and writes its tile to
// the workspace; merge_kernel adds the S partials in split order, then the bias, then (accumulate) the old value.  Without a split the
// GEMM kernel applies the same epilogue itself.  Every sum has a fixed order: the result is the same bits on every run.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/csnet_b200.h"

namespace csnet {
namespace g32 {

enum Form { kFwd = CSNET_CONV_FWD, kDgrad = CSNET_CONV_DGRAD, kWgrad = CSNET_CONV_WGRAD };
constexpr int kThreads = 256;
constexpr int kMaxSegs = 8;
constexpr int kStages = 4;

struct Seg {
  const float* src;
  const float* w;
  int C, c0, cin, cout0, cout, dil, ldw;
  int tile0;                 // first global k tile of the segment (fwd / dgrad)
  int K;                     // k extent: fwd cin k^2, dgrad cout k^2
};

struct Args {
  Seg seg[kMaxSegs];
  int nseg;
  float* dst;                // fwd / dgrad: [N][Cd][HW] at channel d0; wgrad: dw with row stride ldd
  const float* bias;         // fwd: [M] or null
  const float* dy;           // wgrad: the output gradient [N][Cy][HW], channels from y0
  int Cd, d0, ldd;
  int Cy, y0;
  int N, H, W, HW;
  int M, Ncol;               // GEMM extents of one image (wgrad: of the whole call)
  int ktiles, kt_img;        // k tiles of the call; wgrad: k tiles per image
  int splits, accumulate;
  float* ws;                 // splits > 1: partials [splits][images][M][Ncol]
};

__device__ __forceinline__ void cp4(float* smem, const float* g, bool valid) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;\n" ::"r"(s), "l"(g), "r"(valid ? 4 : 0));
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N> __device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

template <int BM, int BN, int BK, int TM, int TN>
struct Tile {
  static_assert((BM / TM) * (BN / TN) == kThreads, "256 threads per block");
  static_assert(BM * BK == 4 * kThreads && BK * BN == 4 * kThreads, "four staged elements of A and of B per thread");
  static constexpr int LA = (BM * BK) / kThreads;     // A elements a thread stages per k tile
  static constexpr int LB = (BK * BN) / kThreads;
  static constexpr int PM = BM + 4, PN = BN + 4;      // padded shared rows (16-byte aligned)
  static constexpr int kSmemFloats = kStages * BK * (PM + PN);
};

// Row (column) i of a thread's register tile: TM / 4 4-wide groups spaced BM * 4 / TM apart, so one warp's float4 reads of a
// k row cover distinct banks.
template <int B, int T> __device__ __forceinline__ int tile_idx(int t, int i) { return (i / 4) * (B * 4 / T) + t * 4 + (i & 3); }

template <int BM, int BN, int BK, int TM, int TN, int KS, int FORM>
__global__ void __launch_bounds__(kThreads) gemm_f32_kernel(const __grid_constant__ Args A) {
  using TL = Tile<BM, BN, BK, TM, TN>;
  constexpr int KK = KS * KS;
  extern __shared__ __align__(16) float smem[];
  float* As = smem;                                   // [stage][BK][PM]
  float* Bs = smem + kStages * BK * TL::PM;           // [stage][BK][PN]
  const int tid = threadIdx.x, tx = tid % (BN / TN), ty = tid / (BN / TN);
  const int n0 = blockIdx.x * BN, m0 = blockIdx.y * BM;
  const int img = FORM == kWgrad ? 0 : (int)blockIdx.z / A.splits;
  const int split = (int)blockIdx.z % A.splits;
  const int t_begin = (int)(((int64_t)split * A.ktiles) / A.splits), t_end = (int)(((int64_t)(split + 1) * A.ktiles) / A.splits);
  const int nt = t_end - t_begin;

  // fwd / dgrad: a thread's B column (pixel) is the same in every k tile (LB elements k = tid / BN + i * (256 / BN))
  int py = 0, px = 0;
  const int bn_col = tid % BN;
  if (FORM != kWgrad) { const int p = n0 + bn_col; py = p / A.W; px = p - py * A.W; }

  auto load = [&](int g, int stage) {
    float* as = As + stage * BK * TL::PM;
    float* bs = Bs + stage * BK * TL::PN;
    if (FORM == kWgrad) {
      const int im = g / A.kt_img, p0 = (g - im * A.kt_img) * BK;
      const Seg& S = A.seg[0];
      // A[m = co][k = p] = dy[im][cout0 + co][p0 + k]; consecutive threads take consecutive k
#pragma unroll
      for (int i = 0; i < TL::LA; ++i) {
        const int e = tid + i * kThreads, m = e / BK, k = e % BK, p = p0 + k, co = m0 + m;
        const bool v = co < A.M && p < A.HW;
        cp4(as + k * TL::PM + m, A.dy + (v ? ((int64_t)im * A.Cy + A.y0 + co) * A.HW + p : 0), v);
      }
      // B[k = p][n = (ci, t)] = x[im][c0 + ci][p + off_t]; a thread's k (pixel) is fixed: one divide per tile
      const int k = tid % BK, p = p0 + k;
      const int y = p / A.W, x = p - y * A.W;
#pragma unroll
      for (int i = 0; i < TL::LB; ++i) {
        const int n = tid / BK + i * (kThreads / BK), col = n0 + n;
        const int ci = col / KK, t = col - ci * KK;
        const int yy = y + (KS == 3 ? (t / 3 - 1) * S.dil : 0), xx = x + (KS == 3 ? (t % 3 - 1) * S.dil : 0);
        const bool v = col < A.Ncol && p < A.HW && yy >= 0 && yy < A.H && xx >= 0 && xx < A.W;
        const float* src = S.src + (v ? ((int64_t)im * S.C + S.c0 + ci) * A.HW + (int64_t)yy * A.W + xx : 0);
        cp4(bs + k * TL::PN + n, src, v);
      }
      return;
    }
    int s = 0;
    while (s + 1 < A.nseg && g >= A.seg[s + 1].tile0) ++s;
    const Seg& S = A.seg[s];
    const int k0 = (g - S.tile0) * BK;
    if (FORM == kFwd) {
      // A[m = co][k = (ci, t)] = w[co * ldw + k]: contiguous in k
#pragma unroll
      for (int i = 0; i < TL::LA; ++i) {
        const int e = tid + i * kThreads, m = e / BK, k = e % BK, co = m0 + m, kk = k0 + k;
        const bool v = co < A.M && kk < S.K;
        cp4(as + k * TL::PM + m, S.w + (v ? (int64_t)co * S.ldw + kk : 0), v);
      }
    } else {
      // A[m = ci][k = (co, t)] = w[co * ldw + ci k^2 + t]: consecutive threads take consecutive ci
#pragma unroll
      for (int i = 0; i < TL::LA; ++i) {
        const int e = tid + i * kThreads, k = e / BM, m = e % BM, ci = m0 + m, kk = k0 + k;
        const int co = kk / KK, t = kk - co * KK;
        const bool v = ci < A.M && kk < S.K;
        cp4(as + k * TL::PM + m, S.w + (v ? (int64_t)co * S.ldw + ci * KK + t : 0), v);
      }
    }
    // B[k][n = p]: fwd x[img][c0 + ci][p + off_t], dgrad dy[img][cout0 + co][p - off_t]
#pragma unroll
    for (int i = 0; i < TL::LB; ++i) {
      const int k = tid / BN + i * (kThreads / BN), kk = k0 + k;
      const int c = kk / KK, t = kk - c * KK;
      const int sy = FORM == kFwd ? 1 : -1;
      const int yy = py + (KS == 3 ? sy * (t / 3 - 1) * S.dil : 0), xx = px + (KS == 3 ? sy * (t % 3 - 1) * S.dil : 0);
      const int ch = FORM == kFwd ? S.c0 + c : S.cout0 + c;
      const bool v = kk < S.K && n0 + bn_col < A.HW && yy >= 0 && yy < A.H && xx >= 0 && xx < A.W;
      cp4(bs + k * TL::PN + bn_col, S.src + (v ? ((int64_t)img * S.C + ch) * A.HW + (int64_t)yy * A.W + xx : 0), v);
    }
  };

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

#pragma unroll
  for (int s = 0; s < kStages - 1; ++s) {
    if (s < nt) load(t_begin + s, s);
    cp_commit();
  }
  for (int it = 0; it < nt; ++it) {
    cp_wait<kStages - 2>();
    __syncthreads();                                   // tile it is visible; tile it - 1's buffer is free
    if (it + kStages - 1 < nt) load(t_begin + it + kStages - 1, (it + kStages - 1) % kStages);
    cp_commit();
    const float* as = As + (it % kStages) * BK * TL::PM;
    const float* bs = Bs + (it % kStages) * BK * TL::PN;
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float a[TM], b[TN];
#pragma unroll
      for (int i = 0; i < TM; i += 4) {
        const float4 v = *reinterpret_cast<const float4*>(as + k * TL::PM + tile_idx<BM, TM>(ty, i));
        a[i] = v.x; a[i + 1] = v.y; a[i + 2] = v.z; a[i + 3] = v.w;
      }
#pragma unroll
      for (int j = 0; j < TN; j += 4) {
        const float4 v = *reinterpret_cast<const float4*>(bs + k * TL::PN + tile_idx<BN, TN>(tx, j));
        b[j] = v.x; b[j + 1] = v.y; b[j + 2] = v.z; b[j + 3] = v.w;
      }
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
  }
  cp_wait<0>();

  // epilogue: the partial of this split, or the finished value
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int m = m0 + tile_idx<BM, TM>(ty, i);
    if (m >= A.M) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      const int n = n0 + tile_idx<BN, TN>(tx, j);
      if (n >= A.Ncol) continue;
      if (A.splits > 1) {
        const int images = (int)gridDim.z / A.splits;
        A.ws[(((int64_t)split * images + img) * A.M + m) * A.Ncol + n] = acc[i][j];
      } else {
        float v = acc[i][j];
        if (FORM == kFwd && A.bias) v += A.bias[m];
        float* o = FORM == kWgrad ? A.dst + (int64_t)m * A.ldd + n : A.dst + (((int64_t)img * A.Cd + A.d0 + m) * A.HW + n);
        *o = A.accumulate ? *o + v : v;
      }
    }
  }
}

// dst = (accumulate ? old : 0) + (bias + sum of the splits' partials in split order)
template <int FORM>
__global__ void __launch_bounds__(kThreads) gemm_merge_kernel(const __grid_constant__ Args A, int images) {
  const int64_t per = (int64_t)A.M * A.Ncol, total = per * images;
  for (int64_t e = blockIdx.x * (int64_t)kThreads + threadIdx.x; e < total; e += (int64_t)gridDim.x * kThreads) {
    const int img = (int)(e / per);
    const int64_t r = e - img * per;
    const int m = (int)(r / A.Ncol), n = (int)(r - (int64_t)m * A.Ncol);
    float v = A.ws[e];
    for (int s = 1; s < A.splits; ++s) v += A.ws[(int64_t)s * total + e];
    if (FORM == kFwd && A.bias) v += A.bias[m];
    float* o = FORM == kWgrad ? A.dst + (int64_t)m * A.ldd + n : A.dst + (((int64_t)img * A.Cd + A.d0 + m) * A.HW + n);
    *o = A.accumulate ? *o + v : v;
  }
}

}  // namespace g32
}  // namespace csnet
