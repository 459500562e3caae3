// gemm_bf16.cuh — the three convolution forms of gemm_f32.cuh (forward, data gradient, weight gradient; 1x1, and 3x3 with dilation
// d and zero padding d; up to 8 K segments; weight slices through ldw; bias; accumulate) as a tensor-core implicit GEMM: bf16
// operands, fp32 accumulation (include/csnet_b200.h, csnet_train_conv_*_bf16).  Per image, NCHW, the same sums as gemm_f32:
//
//   fwd    C[co][p]      = sum over segments, (ci, t)  of  w_s[co][ci][t] * x_s[ci][p + off_t]          M = cout, N = HW
//   dgrad  C[ci][p]      = sum over segments, (co, t)  of  w_s[co][ci][t] * dy_s[co][p - off_t]         M = cin,  N = HW
//   wgrad  C[co][ci, t]  = sum over images, pixels p   of  dy[co][p] * x[ci][p + off_t]                 M = cout, N = cin k^2
//
// A block of 256 threads (8 warps, 2 x 4) computes a 128 x 128 tile of C; each warp a 64 x 32 tile as 4 x 4 mma.sync.m16n8k16
// (bf16 x bf16 -> fp32).  k tiles are 32 deep.  The operands are gathers (taps, padding, channel slices, planes whose rows are not
// 16-byte multiples), so each thread loads its 16 A and 16 B elements of the next k tile with 2-byte loads into registers while the
// warps run the current tile's MMAs, and stores them to the other of two shared-memory buffers: [row][k] with a 40-element pitch,
// which ldmatrix reads without bank conflicts.  Out-of-range elements (padding, plane edges, ragged M, N, K) load as zero.  A k tile
// never crosses a segment (or, for wgrad, an image).
//
// Split-K: as gemm_f32, split z of S takes k tiles [z T / S, (z + 1) T / S), writes an fp32 partial to the workspace, and
// gemm_bf16_merge_kernel adds the partials in split order, then the bias, then (accumulate) the old value, and rounds once to the
// destination's type.  Without a split the GEMM kernel applies that epilogue itself.  mma.sync's sums have a fixed order, and there
// are no atomics: the result is the same bits on every run.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/csnet_b200.h"

namespace csnet {
namespace gbf {

enum Form { kFwd = CSNET_CONV_FWD, kDgrad = CSNET_CONV_DGRAD, kWgrad = CSNET_CONV_WGRAD };
constexpr int kThreads = 256;
constexpr int kMaxSegs = 8;
constexpr int BM = 128, BN = 128, BK = 32;
constexpr int kPitch = BK + 8;                      // shared row pitch in bf16: 80 bytes, ldmatrix's 8 rows hit distinct banks
constexpr int kLA = BM * BK / kThreads, kLB = BN * BK / kThreads;   // 16 elements of A and of B per thread and k tile
constexpr int kSmemBytes = 2 * (BM + BN) * kPitch * 2;

struct Seg {
  const __nv_bfloat16* src;
  const __nv_bfloat16* w;
  int C, c0, cin, cout0, cout, dil, ldw;
  int tile0;                 // first global k tile of the segment (fwd / dgrad)
  int K;                     // k extent: fwd cin k^2, dgrad cout k^2
};

struct Args {
  Seg seg[kMaxSegs];
  int nseg;
  void* dst;                 // fwd / dgrad: [N][Cd][HW] at channel d0, bf16 or fp32; wgrad: fp32 dw with row stride ldd
  const float* bias;         // fwd: [M] or null
  const __nv_bfloat16* dy;   // wgrad: the output gradient [N][Cy][HW], channels from y0
  int Cd, d0, ldd;
  int Cy, y0;
  int N, H, W, HW;
  int M, Ncol;               // GEMM extents of one image (wgrad: of the whole call)
  int ktiles, kt_img;        // k tiles of the call; wgrad: k tiles per image
  int splits, accumulate;
  float* ws;                 // splits > 1: partials [splits][images][M][Ncol]
};

__device__ __forceinline__ float to_f(float v) { return v; }
__device__ __forceinline__ float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }
template <typename T> __device__ __forceinline__ T from_f(float v);
template <> __device__ __forceinline__ float from_f<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

__device__ __forceinline__ unsigned short ld_bf16(const __nv_bfloat16* p, bool valid) {
  return valid ? __ldg(reinterpret_cast<const unsigned short*>(p)) : (unsigned short)0;
}

__device__ __forceinline__ void ldsm_x4(unsigned& r0, unsigned& r1, unsigned& r2, unsigned& r3, const void* p) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(p);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];\n"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(s));
}

__device__ __forceinline__ void mma_bf16(float* c, const unsigned* a, unsigned b0, unsigned b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
               "{%0, %1, %2, %3};\n"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// dst element (m, n) of image img: the finished value v (bias added), plus the old value when accumulating, rounded once.
template <int FORM, typename TD>
__device__ __forceinline__ void store_out(const Args& A, int img, int m, int n, float v) {
  if (FORM == kFwd && A.bias) v += A.bias[m];
  TD* o = FORM == kWgrad ? reinterpret_cast<TD*>(A.dst) + (int64_t)m * A.ldd + n
                         : reinterpret_cast<TD*>(A.dst) + (((int64_t)img * A.Cd + A.d0 + m) * A.HW + n);
  *o = from_f<TD>(A.accumulate ? to_f(*o) + v : v);
}

template <int KS, int FORM, typename TD>
__global__ void __launch_bounds__(kThreads) gemm_bf16_kernel(const __grid_constant__ Args A) {
  constexpr int KK = KS * KS;
  __shared__ __align__(16) __nv_bfloat16 As[2][BM * kPitch];   // [m][k]
  __shared__ __align__(16) __nv_bfloat16 Bs[2][BN * kPitch];   // [n][k]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm0 = (warp >> 2) * 64, wn0 = (warp & 3) * 32;
  const int n0 = blockIdx.x * BN, m0 = blockIdx.y * BM;
  const int img = FORM == kWgrad ? 0 : (int)blockIdx.z / A.splits;
  const int split = (int)blockIdx.z % A.splits;
  const int t_begin = (int)(((int64_t)split * A.ktiles) / A.splits), t_end = (int)(((int64_t)(split + 1) * A.ktiles) / A.splits);
  const int nt = t_end - t_begin;

  // fwd / dgrad: a thread's B column (pixel) is the same in every k tile (k = tid / BN + 2 i)
  int py = 0, px = 0;
  const int bn_col = tid % BN;
  if (FORM != kWgrad) { const int p = n0 + bn_col; py = p / A.W; px = p - py * A.W; }

  unsigned short ra[kLA], rb[kLB];
  // the (row, k) of staged element i: k fastest where the source is contiguous in k, else the row fastest
  const bool a_kfast = FORM != kDgrad;
  auto a_pos = [&](int i, int& m, int& k) {
    const int e = tid + i * kThreads;
    if (a_kfast) { m = e / BK; k = e % BK; } else { k = e / BM; m = e % BM; }
  };
  auto b_pos = [&](int i, int& n, int& k) {
    const int e = tid + i * kThreads;
    if (FORM == kWgrad) { n = e / BK; k = e % BK; } else { k = e / BN; n = e % BN; }
  };

  auto load = [&](int g) {
    if (FORM == kWgrad) {
      const int im = g / A.kt_img, p0 = (g - im * A.kt_img) * BK;
      const Seg& S = A.seg[0];
#pragma unroll
      for (int i = 0; i < kLA; ++i) {                 // A[m = co][k = p] = dy[im][y0 + co][p0 + k]
        int m, k;
        a_pos(i, m, k);
        const int co = m0 + m, p = p0 + k;
        const bool v = co < A.M && p < A.HW;
        ra[i] = ld_bf16(A.dy + (v ? ((int64_t)im * A.Cy + A.y0 + co) * A.HW + p : 0), v);
      }
      const int k = tid % BK, p = p0 + k;             // B[k = p][n = (ci, t)] = x[im][c0 + ci][p + off_t]: k fixed per thread
      const int y = p / A.W, x = p - y * A.W;
#pragma unroll
      for (int i = 0; i < kLB; ++i) {
        const int col = n0 + tid / BK + i * (kThreads / BK);
        const int ci = col / KK, t = col - ci * KK;
        const int yy = y + (KS == 3 ? (t / 3 - 1) * S.dil : 0), xx = x + (KS == 3 ? (t % 3 - 1) * S.dil : 0);
        const bool v = col < A.Ncol && p < A.HW && yy >= 0 && yy < A.H && xx >= 0 && xx < A.W;
        rb[i] = ld_bf16(S.src + (v ? ((int64_t)im * S.C + S.c0 + ci) * A.HW + (int64_t)yy * A.W + xx : 0), v);
      }
      return;
    }
    int s = 0;
    while (s + 1 < A.nseg && g >= A.seg[s + 1].tile0) ++s;
    const Seg& S = A.seg[s];
    const int k0 = (g - S.tile0) * BK;
#pragma unroll
    for (int i = 0; i < kLA; ++i) {
      int m, k;
      a_pos(i, m, k);
      const int r = m0 + m, kk = k0 + k;
      const bool v = r < A.M && kk < S.K;
      int64_t off = 0;
      if (v) {
        if (FORM == kFwd) off = (int64_t)r * S.ldw + kk;                         // A[co][(ci, t)] = w[co ldw + k]
        else { const int co = kk / KK, t = kk - co * KK; off = (int64_t)co * S.ldw + r * KK + t; }   // A[ci][(co, t)]
      }
      ra[i] = ld_bf16(S.w + off, v);
    }
#pragma unroll
    for (int i = 0; i < kLB; ++i) {                   // B[k][n = p]: fwd x[img][c0 + ci][p + off_t], dgrad dy[img][cout0 + co][p - off_t]
      const int k = tid / BN + i * (kThreads / BN), kk = k0 + k;
      const int c = kk / KK, t = kk - c * KK;
      const int sy = FORM == kFwd ? 1 : -1;
      const int yy = py + (KS == 3 ? sy * (t / 3 - 1) * S.dil : 0), xx = px + (KS == 3 ? sy * (t % 3 - 1) * S.dil : 0);
      const int ch = FORM == kFwd ? S.c0 + c : S.cout0 + c;
      const bool v = kk < S.K && n0 + bn_col < A.HW && yy >= 0 && yy < A.H && xx >= 0 && xx < A.W;
      rb[i] = ld_bf16(S.src + (v ? ((int64_t)img * S.C + ch) * A.HW + (int64_t)yy * A.W + xx : 0), v);
    }
  };
  auto stash = [&](int buf) {
    unsigned short* as = reinterpret_cast<unsigned short*>(As[buf]);
    unsigned short* bs = reinterpret_cast<unsigned short*>(Bs[buf]);
#pragma unroll
    for (int i = 0; i < kLA; ++i) { int m, k; a_pos(i, m, k); as[m * kPitch + k] = ra[i]; }
#pragma unroll
    for (int i = 0; i < kLB; ++i) { int n, k; b_pos(i, n, k); bs[n * kPitch + k] = rb[i]; }
  };

  float acc[4][4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int r = 0; r < 4; ++r) acc[i][j][r] = 0.f;

  // ldmatrix row addresses: A x4 covers (rows 0-15) x (k 0-7, 8-15); B x4 covers (n 0-7, 8-15) x (k 0-7, 8-15)
  const int a_row = lane & 15, a_col = (lane >> 4) * 8;
  const int b_row = (lane & 7) + (lane >> 4) * 8, b_col = ((lane >> 3) & 1) * 8;

  if (nt > 0) { load(t_begin); stash(0); }
  __syncthreads();
  for (int it = 0; it < nt; ++it) {
    const int buf = it & 1;
    if (it + 1 < nt) load(t_begin + it + 1);         // next tile's global loads under this tile's MMAs
    const __nv_bfloat16* as = As[buf];
    const __nv_bfloat16* bs = Bs[buf];
#pragma unroll
    for (int ks = 0; ks < BK; ks += 16) {
      unsigned a[4][4], b[4][2];
#pragma unroll
      for (int mi = 0; mi < 4; ++mi)
        ldsm_x4(a[mi][0], a[mi][1], a[mi][2], a[mi][3], as + (wm0 + mi * 16 + a_row) * kPitch + ks + a_col);
#pragma unroll
      for (int nj = 0; nj < 2; ++nj)
        ldsm_x4(b[2 * nj][0], b[2 * nj][1], b[2 * nj + 1][0], b[2 * nj + 1][1], bs + (wn0 + nj * 16 + b_row) * kPitch + ks + b_col);
#pragma unroll
      for (int mi = 0; mi < 4; ++mi)
#pragma unroll
        for (int ni = 0; ni < 4; ++ni) mma_bf16(acc[mi][ni], a[mi], b[ni][0], b[ni][1]);
    }
    if (it + 1 < nt) stash(buf ^ 1);                 // the other buffer was last read in iteration it - 1, before its barrier
    __syncthreads();
  }

  // epilogue: c[r] of an m16n8 tile is row lane / 4 (+ 8 for r >= 2), column 2 (lane % 4) + (r & 1)
#pragma unroll
  for (int mi = 0; mi < 4; ++mi)
#pragma unroll
    for (int ni = 0; ni < 4; ++ni)
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int m = m0 + wm0 + mi * 16 + (lane >> 2) + (r >= 2 ? 8 : 0);
        const int n = n0 + wn0 + ni * 8 + (lane & 3) * 2 + (r & 1);
        if (m >= A.M || n >= A.Ncol) continue;
        if (A.splits > 1) {
          const int images = (int)gridDim.z / A.splits;
          A.ws[(((int64_t)split * images + img) * A.M + m) * A.Ncol + n] = acc[mi][ni][r];
        } else {
          store_out<FORM, TD>(A, img, m, n, acc[mi][ni][r]);
        }
      }
}

// dst = rn((accumulate ? old : 0) + (bias + sum of the splits' partials in split order))
template <int FORM, typename TD>
__global__ void __launch_bounds__(kThreads) gemm_bf16_merge_kernel(const __grid_constant__ Args A, int images) {
  const int64_t per = (int64_t)A.M * A.Ncol, total = per * images;
  for (int64_t e = blockIdx.x * (int64_t)kThreads + threadIdx.x; e < total; e += (int64_t)gridDim.x * kThreads) {
    const int img = (int)(e / per);
    const int64_t r = e - img * per;
    const int m = (int)(r / A.Ncol), n = (int)(r - (int64_t)m * A.Ncol);
    float v = A.ws[e];
    for (int s = 1; s < A.splits; ++s) v += A.ws[(int64_t)s * total + e];
    store_out<FORM, TD>(A, img, m, n, v);
  }
}

}  // namespace gbf
}  // namespace csnet
