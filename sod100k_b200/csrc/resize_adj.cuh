// resize_adj.cuh — the adjoint of CSNET_OP_RESIZE's bilinear resize (resize.cuh), for training: the gradient of
// F.interpolate(src, size=(Hd, Wd), mode='bilinear', align_corners=False) with respect to src.
//
// The forward gives output o of an axis the taps mae_tap(o) = (i0, i1, l0, l1).  Along an axis source s receives
//   w(o, s) = [i0(o) == s] l0(o) + [i1(o) == s] l1(o)
// from every output o whose taps touch it, and the 2-D weight is wy * wx.  Gather form: one thread per source pixel adds
//   dsrc[sy][sx] = sum over oy of wy(oy, sy) * (sum over ox of wx(ox, sx) * ddst[oy][ox])
// with oy and ox ascending over the ranges rz_src_range returns, so no atomics are needed and the order is fixed.
// rz_src_range inverts the taps by binary search over mae_tap itself (i0 and i1 never decrease with o), so it agrees with the
// forward's taps bit for bit.  It is plain host/device code: tests/emu compiles it for the CPU.
#pragma once
#include <stdint.h>

#include "image_io.cuh"
#include "resize.cuh"

namespace csnet {

struct RzRange {
  int lo, hi;               // outputs lo..hi (inclusive) touch the source sample; empty when lo > hi
};

CSNET_IO_HD RzRange rz_src_range(int s, int n_in, int n_out, float scale) {
  int a = 0, b = n_out;                                         // first o with i1(o) >= s
  while (a < b) {
    const int m = (a + b) / 2;
    if (mae_tap(m, n_in, scale).i1 >= s) b = m; else a = m + 1;
  }
  RzRange r;
  r.lo = a;
  a = 0; b = n_out;                                             // first o with i0(o) > s
  while (a < b) {
    const int m = (a + b) / 2;
    if (mae_tap(m, n_in, scale).i0 > s) b = m; else a = m + 1;
  }
  r.hi = a - 1;
  return r;
}

// Weight output o gives source s along one axis.
CSNET_IO_HD float rz_adj_weight(MaeTap t, int s) { return (t.i0 == s ? t.l0 : 0.f) + (t.i1 == s ? t.l1 : 0.f); }

// One source value of the adjoint: g = the output-gradient channel [Hd][Wd] (fp32, or bf16 widened exactly; the sums are fp32).
template <typename T>
CSNET_IO_HD float resize_adj_value(const T* g, int Hs, int Ws, int Hd, int Wd, float sy, float sx, int ys, int xs) {
  const RzRange ry = rz_src_range(ys, Hs, Hd, sy), rx = rz_src_range(xs, Ws, Wd, sx);
  float acc = 0.f;
  for (int oy = ry.lo; oy <= ry.hi; ++oy) {
    const float wy = rz_adj_weight(mae_tap(oy, Hs, sy), ys);
    const T* row = g + (int64_t)oy * Wd;
    float r = 0.f;
    for (int ox = rx.lo; ox <= rx.hi; ++ox) r += rz_adj_weight(mae_tap(ox, Ws, sx), xs) * rz_f32(row[ox]);
    acc += wy * r;
  }
  return acc;
}

#ifndef CSNET_HOST_EMU
constexpr int kRzAdjThreads = 256;

// Grid: (source-pixel blocks, channels, images); a thread per source pixel.
__global__ void __launch_bounds__(kRzAdjThreads) resize_bwd_kernel(const float* __restrict__ ddst, float* __restrict__ dsrc, int C,
                                                                   int Hs, int Ws, int Hd, int Wd, float sy, float sx) {
  const int p = blockIdx.x * kRzAdjThreads + threadIdx.x;
  if (p >= Hs * Ws) return;
  const int c = blockIdx.y, n = blockIdx.z, ys = p / Ws, xs = p - ys * Ws;
  const float* g = ddst + ((int64_t)n * C + c) * Hd * Wd;
  dsrc[((int64_t)n * C + c) * Hs * Ws + p] = resize_adj_value(g, Hs, Ws, Hd, Wd, sy, sx, ys, xs);
}
#endif

}  // namespace csnet
