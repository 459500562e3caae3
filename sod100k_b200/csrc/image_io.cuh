// image_io.cuh — images of any size in, saliency maps at each image's own size out (CSNet/test.py:71-98, both skimage resizes).
//
// The reference resizes every image to the network size with skimage `resize(img, (H, W), mode='reflect', anti_aliasing=False)`
// and resizes the sigmoid map back to the image's (h, w) the same way.  For skimage >= 0.19 and order 1 (the default for float
// input) that is scipy.ndimage.zoom(order=1, mode='mirror', grid_mode=True), the channel axis untouched: separable bilinear
// interpolation at source coordinate c = (o + 0.5) * n_in / n_out - 0.5, mirrored about the edge samples.  The per-pixel
// functions below are plain host/device code so tests/emu compiles the same source for the CPU.
//
//   in:  taps x / 255 (img_as_float), bilinear in double, (v - mean[c]) / std[c] in double, rounded once to fp32, planar NCHW
//   out: s = sigmoid(logit) in fp32 (post_u8_kernel's expression), bilinear in double rounded to fp32 (zoom of a float32 map
//        returns float32), s * 255.f truncated to uint8
// Where the coordinate lands on a sample (t == 0, every pixel at identity size) the lerps return that sample exactly, so a batch
// already at the network size gives the bytes of csnet_plan_run_host_u8.
#pragma once
#include <math.h>
#include <stdint.h>

#include "../../include/csnet_b200.h"

#ifdef CSNET_HOST_EMU
#define CSNET_IO_HD inline
#else
#define CSNET_IO_HD __host__ __device__ __forceinline__
#endif

namespace csnet {

constexpr int kMaxImageSide = 32767;      // csnet_plan_run_host_images_u8 rejects larger images

// One output index along an axis of n_in -> n_out samples: value = (1 - t) * in[i0] + t * in[i1].
struct ImgTap {
  int i0, i1;
  double t;
};

CSNET_IO_HD ImgTap img_tap(int o, int n_in, int n_out) {
  ImgTap r{0, 0, 0.0};
  if (n_in == 1) return r;                                      // a one-sample axis is constant
  double c = ((double)o + 0.5) * ((double)n_in / (double)n_out) - 0.5;
  const double last = (double)(n_in - 1);
  if (c < 0.0) c = -c;                                          // mirror about the edge samples
  if (c > last) c = 2.0 * last - c;
  int i0 = (int)floor(c);
  i0 = i0 < 0 ? 0 : (i0 > n_in - 2 ? n_in - 2 : i0);
  r.i0 = i0;
  r.i1 = i0 + 1;
  r.t = c - (double)i0;
  return r;
}

// Exact at t == 0 and t == 1, with or without FMA contraction.
CSNET_IO_HD double img_lerp(double a, double b, double t) { return (1.0 - t) * a + t * b; }

// Network input, channel c, at the output pixel (ty, tx) of one packed HWC uint8 image of width w.  tab[x] = x / 255.0.
CSNET_IO_HD float img_in_value(const uint8_t* img, int w, const double* tab, ImgTap ty, ImgTap tx, int c, double mean, double stdv) {
  const uint8_t* r0 = img + (int64_t)ty.i0 * w * 3 + c;
  const uint8_t* r1 = img + (int64_t)ty.i1 * w * 3 + c;
  const double top = img_lerp(tab[r0[tx.i0 * 3]], tab[r0[tx.i1 * 3]], tx.t);
  const double bot = img_lerp(tab[r1[tx.i0 * 3]], tab[r1[tx.i1 * 3]], tx.t);
  return (float)((img_lerp(top, bot, ty.t) - mean) / stdv);
}

CSNET_IO_HD float img_sigmoid(float z) { return 1.f / (1.f + expf(-z)); }

// Saliency map byte at the output pixel (ty, tx) of one image's logits plane z [H][W] (row stride W).
CSNET_IO_HD uint8_t img_out_value(const float* z, int W, ImgTap ty, ImgTap tx) {
  const float* r0 = z + (int64_t)ty.i0 * W;
  const float* r1 = z + (int64_t)ty.i1 * W;
  const double top = img_lerp((double)img_sigmoid(r0[tx.i0]), (double)img_sigmoid(r0[tx.i1]), tx.t);
  const double bot = img_lerp((double)img_sigmoid(r1[tx.i0]), (double)img_sigmoid(r1[tx.i1]), tx.t);
  const float s = (float)img_lerp(top, bot, ty.t);
  return (uint8_t)(s * 255.f);
}

#ifndef CSNET_HOST_EMU
constexpr int kImgThreads = 256;          // also the x / 255 table's length
constexpr int kImgRows = 4;               // output rows per block of resize_in_u8_kernel

struct ImgNorm {
  double mean[3], std[3];
};

// Ragged uint8 HWC images -> fp32 [N,3,H,W].  Grid: (output-row tiles, image).  The block computes its column taps once per
// 256-column slice, then every thread takes (row, column) pixels of the tile.
__global__ void __launch_bounds__(kImgThreads) resize_in_u8_kernel(const uint8_t* __restrict__ x, const csnet_image_geom* __restrict__ geom,
                                                                  int H, int W, const __grid_constant__ ImgNorm A, float* __restrict__ y) {
  __shared__ double tab[256];
  __shared__ double col_t[kImgThreads];
  __shared__ int col_i0[kImgThreads], col_i1[kImgThreads];
  const int n = blockIdx.y, oy0 = blockIdx.x * kImgRows, rows = H - oy0 < kImgRows ? H - oy0 : kImgRows;
  const csnet_image_geom g = geom[n];
  const uint8_t* img = x + g.src_off;
  tab[threadIdx.x] = (double)threadIdx.x / 255.0;
  for (int cx0 = 0; cx0 < W; cx0 += kImgThreads) {
    const int cw = W - cx0 < kImgThreads ? W - cx0 : kImgThreads;
    __syncthreads();                                            // the previous slice's taps are consumed
    if ((int)threadIdx.x < cw) {
      const ImgTap t = img_tap(cx0 + threadIdx.x, g.w, W);
      col_i0[threadIdx.x] = t.i0;
      col_i1[threadIdx.x] = t.i1;
      col_t[threadIdx.x] = t.t;
    }
    __syncthreads();
    for (int p = threadIdx.x; p < rows * cw; p += kImgThreads) {
      const int r = p / cw, cx = p - r * cw, oy = oy0 + r;
      const ImgTap ty = img_tap(oy, g.h, H), tx{col_i0[cx], col_i1[cx], col_t[cx]};
#pragma unroll
      for (int c = 0; c < 3; ++c)
        y[(((int64_t)n * 3 + c) * H + oy) * W + cx0 + cx] = img_in_value(img, g.w, tab, ty, tx, c, A.mean[c], A.std[c]);
    }
  }
}

// fp32 logits [N,1,H,W] -> each image's uint8 map [h][w] at its dst_off.  Grid: (blocks per image, image); each block
// grid-strides over its image's pixels.
__global__ void __launch_bounds__(kImgThreads) resize_out_u8_kernel(const float* __restrict__ z, int H, int W,
                                                                   const csnet_image_geom* __restrict__ geom, uint8_t* __restrict__ y) {
  const int n = blockIdx.y;
  const csnet_image_geom g = geom[n];
  const float* zn = z + (int64_t)n * H * W;
  uint8_t* out = y + g.dst_off;
  const int64_t hw = (int64_t)g.h * g.w;
  for (int64_t p = (int64_t)blockIdx.x * kImgThreads + threadIdx.x; p < hw; p += (int64_t)gridDim.x * kImgThreads) {
    const int oy = (int)p / g.w, ox = (int)p - oy * g.w;     // h * w < 2^31
    out[p] = img_out_value(zn, W, img_tap(oy, H, g.h), img_tap(ox, W, g.w));
  }
}

inline ImgNorm img_norm(const float* mean, const float* stdv) {
  ImgNorm A{};
  for (int c = 0; c < 3; ++c) { A.mean[c] = (double)mean[c]; A.std[c] = (double)stdv[c]; }
  return A;
}

inline void launch_resize_in(const uint8_t* x, const csnet_image_geom* geom, int N, int H, int W, const ImgNorm& A, float* y,
                             cudaStream_t stream) {
  resize_in_u8_kernel<<<dim3((unsigned)((H + kImgRows - 1) / kImgRows), (unsigned)N), kImgThreads, 0, stream>>>(x, geom, H, W, A, y);
}

// The map sizes live on the device, so the grid is sized from the batch alone: about 32 blocks per SM in all, which keeps the
// SMs busy to the end of a batch whose images differ in size; blocks past a small image's end exit at once.
inline void launch_resize_out(const float* z, int N, int H, int W, const csnet_image_geom* geom, uint8_t* y, int num_sms,
                              cudaStream_t stream) {
  const int bx = (32 * num_sms + N - 1) / N;
  resize_out_u8_kernel<<<dim3((unsigned)bx, (unsigned)N), kImgThreads, 0, stream>>>(z, H, W, geom, y);
}
#endif

}  // namespace csnet
