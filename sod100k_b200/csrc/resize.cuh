// resize.cuh — CSNET_OP_RESIZE: bilinear resize of a channel slice to the destination's size at any ratio (include/csnet_b200.h).
//
// F.interpolate(size=(H, W), mode='bilinear', align_corners=False) as ATen computes it in fp32: per axis the taps of mae_tap
// (image_io.cuh), the four samples combined as ATen's CPU kernel does (the two taps along a row, then the two rows), optionally
// added to the destination once in fp32 and rounded once to its dtype.  The CSF+Res2Net head uses it where a gOctConv resizes
// between stages whose sizes are not exact multiples (gOctConv.py:99,102) and for the final resize to the image (csf_res2net.py:258).
// resize_value is plain host/device code so tests/emu compiles the same source for the CPU.
#pragma once
#include <stdint.h>

#include "image_io.cuh"

#ifndef CSNET_HOST_EMU
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#endif

namespace csnet {

CSNET_IO_HD float rz_f32(float v) { return v; }
#ifndef CSNET_HOST_EMU
CSNET_IO_HD float rz_f32(__half v) { return __half2float(v); }
CSNET_IO_HD float rz_f32(__nv_bfloat16 v) { return __bfloat162float(v); }
#endif

// Scale of an axis of n_in -> n_out samples (ATen's area_pixel_compute_scale with size= given).
CSNET_IO_HD float resize_scale(int n_in, int n_out) { return (float)n_in / (float)n_out; }

// One output value: plane = the source channel [Hs][Ws] (row stride ws), ty / tx = mae_tap of the output row / column.  With
// `accumulate` the destination's old value `old` is added once.
template <typename TS>
CSNET_IO_HD float resize_value(const TS* plane, int ws, MaeTap ty, MaeTap tx, bool accumulate, float old) {
  const TS* r0 = plane + (int64_t)ty.i0 * ws;
  const TS* r1 = plane + (int64_t)ty.i1 * ws;
  const float t0 = rz_f32(r0[tx.i0]) * tx.l0 + rz_f32(r0[tx.i1]) * tx.l1;
  const float t1 = rz_f32(r1[tx.i0]) * tx.l0 + rz_f32(r1[tx.i1]) * tx.l1;
  const float v = t0 * ty.l0 + t1 * ty.l1;
  return accumulate ? old + v : v;
}

#ifndef CSNET_HOST_EMU
constexpr int kRzThreads = 256;
constexpr int kRzRows = 4;                // output rows per block
constexpr int kRzChans = 8;               // channels per block
constexpr int kRzCols = 512;              // column taps staged per slice

struct RzArgs {
  const void* src;
  void* dst;
  int32_t Cs, Hs, Ws, c0;                 // source tensor, first channel read
  int32_t Cd, Hd, Wd, cout0;              // destination tensor, first channel written
  int32_t C;                              // channels resized
  int32_t accumulate;
  float sy, sx;                           // resize_scale of each axis
};

template <typename T> __device__ __forceinline__ T rz_cvt(float v);
template <> __device__ __forceinline__ float rz_cvt<float>(float v) { return v; }
template <> __device__ __forceinline__ __half rz_cvt<__half>(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ __nv_bfloat16 rz_cvt<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

// Grid: (output-row tiles of kRzRows, channel groups of kRzChans, image).  The block computes the column taps of a slice once into
// shared memory and the row taps of its rows once; consecutive threads take consecutive output columns of one (channel, row) line,
// so loads of the two source rows and the stores are coalesced.  A 16-bit destination is stored in aligned pairs: unit u of a line
// covers columns 2u - lead and 2u - lead + 1, lead being the parity of the line's first element.
template <typename TS, typename TD>
__global__ void __launch_bounds__(kRzThreads) resize_kernel(const __grid_constant__ RzArgs A) {
  __shared__ MaeTap col[kRzCols];
  __shared__ MaeTap row[kRzRows];
  constexpr bool kPair = sizeof(TD) == 2;
  const int oy0 = blockIdx.x * kRzRows, rows = A.Hd - oy0 < kRzRows ? A.Hd - oy0 : kRzRows;
  const int cb = blockIdx.y * kRzChans, chans = A.C - cb < kRzChans ? A.C - cb : kRzChans;
  const int n = blockIdx.z, lines = rows * chans;
  if ((int)threadIdx.x < rows) row[threadIdx.x] = mae_tap(oy0 + threadIdx.x, A.Hs, A.sy);
  const TS* src = reinterpret_cast<const TS*>(A.src);
  TD* dst = reinterpret_cast<TD*>(A.dst);
  for (int cx0 = 0; cx0 < A.Wd; cx0 += kRzCols) {
    const int cw = A.Wd - cx0 < kRzCols ? A.Wd - cx0 : kRzCols;
    __syncthreads();                                            // the previous slice's taps are consumed
    for (int i = threadIdx.x; i < cw; i += kRzThreads) col[i] = mae_tap(cx0 + i, A.Ws, A.sx);
    __syncthreads();
    const int units = kPair ? (cw + 2) / 2 : cw;                // 16-bit: one more unit covers a leading odd column
    for (int t = threadIdx.x; t < lines * units; t += kRzThreads) {
      const int line = t / units, u = t - line * units;
      const int c = cb + line / rows, r = line - (line / rows) * rows;
      const MaeTap ty = row[r];
      const TS* plane = src + ((int64_t)n * A.Cs + A.c0 + c) * A.Hs * A.Ws;
      const int64_t e0 = (((int64_t)n * A.Cd + A.cout0 + c) * A.Hd + oy0 + r) * A.Wd + cx0;
      if (kPair) {
        const int lead = (int)(e0 & 1), x0 = 2 * u - lead, x1 = x0 + 1;
        const bool v0 = x0 >= 0 && x0 < cw, v1 = x1 < cw;
        if (v0 && v1) {                                         // e0 + x0 is even: one 32-bit access
          float o0 = 0.f, o1 = 0.f;
          if (A.accumulate) { o0 = rz_f32(dst[e0 + x0]); o1 = rz_f32(dst[e0 + x1]); }
          struct alignas(4) Pair { TD a, b; } p;
          p.a = rz_cvt<TD>(resize_value(plane, A.Ws, ty, col[x0], A.accumulate != 0, o0));
          p.b = rz_cvt<TD>(resize_value(plane, A.Ws, ty, col[x1], A.accumulate != 0, o1));
          *reinterpret_cast<Pair*>(dst + e0 + x0) = p;
        } else {
          const int x = v0 ? x0 : x1;
          if (x < 0 || x >= cw) continue;
          const float o = A.accumulate ? rz_f32(dst[e0 + x]) : 0.f;
          dst[e0 + x] = rz_cvt<TD>(resize_value(plane, A.Ws, ty, col[x], A.accumulate != 0, o));
        }
      } else {
        const float o = A.accumulate ? rz_f32(dst[e0 + u]) : 0.f;
        dst[e0 + u] = rz_cvt<TD>(resize_value(plane, A.Ws, ty, col[u], A.accumulate != 0, o));
      }
    }
  }
}

template <typename TS>
inline void launch_resize_to(const RzArgs& A, int dst_dtype, dim3 grid, cudaStream_t stream) {
  if (dst_dtype == CSNET_F16) resize_kernel<TS, __half><<<grid, kRzThreads, 0, stream>>>(A);
  else if (dst_dtype == CSNET_BF16) resize_kernel<TS, __nv_bfloat16><<<grid, kRzThreads, 0, stream>>>(A);
  else resize_kernel<TS, float><<<grid, kRzThreads, 0, stream>>>(A);
}

inline void launch_resize(const RzArgs& A, int src_dtype, int dst_dtype, int N, cudaStream_t stream) {
  const dim3 grid((unsigned)((A.Hd + kRzRows - 1) / kRzRows), (unsigned)((A.C + kRzChans - 1) / kRzChans), (unsigned)N);
  if (src_dtype == CSNET_F16) launch_resize_to<__half>(A, dst_dtype, grid, stream);
  else if (src_dtype == CSNET_BF16) launch_resize_to<__nv_bfloat16>(A, dst_dtype, grid, stream);
  else launch_resize_to<float>(A, dst_dtype, grid, stream);
}
#endif

}  // namespace csnet
