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
//   eval: the `out` bytes counted against each image's GT into SalMetric's histograms (sal_metric.cpp:86-120), the map optional
//
// Training (CSNet_training/utils/prepare_data.py:109-139, train.py:250-293) reuses the same resize:
//   train: a crop window and a flip per sample remap the taps of the cropped, flipped array into the stored image; image as `in`,
//          mask m / 255 bilinear in double rounded once to fp32
//   val:   the per-image MAE of train.py's loop, whose resize back to the GT's size is F.interpolate (ATen's fp32 bilinear), not skimage
//
// CSF+Res2Net's test (CSF+Res2Net/solver.py:62-78, dataset.py:83-96) runs each image at its own size, so neither side resizes:
//   csf in:  img_csf_in_value, numpy's three fp32 roundings of load_image_test
//   csf out: img_csf_out_value, cv2.imwrite of the fp32 array 255 * sigmoid: rounded half to even and saturated, not truncated
//   csf train: `csf in` and img_csf_label_value (m / 255 in fp32), both flipped along W (img_csf_src_col); solver.py:81-127
// The map and SalMetric kernels are templates on the per-pixel map function (CsnetMap, CsfMap), so both networks share one counter.
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

// A tap of the cropped, flipped axis the reference resizes (n samples, cut at `off` of the stored axis), read from the stored
// image: sample i of the crop is stored at off + i, or at off + n - 1 - i when the axis is flipped.
CSNET_IO_HD ImgTap img_tap_crop(ImgTap t, int off, int n, bool flip) {
  t.i0 = flip ? off + n - 1 - t.i0 : off + t.i0;
  t.i1 = flip ? off + n - 1 - t.i1 : off + t.i1;
  return t;
}

// Training target at the output pixel (ty, tx) of one packed uint8 mask [h][w] of width w: m / 255 interpolated in double, rounded
// once to fp32 (SalData's resize of img_as_float(gt), then train.py's .float()).
CSNET_IO_HD float img_mask_value(const uint8_t* m, int w, const double* tab, ImgTap ty, ImgTap tx) {
  const uint8_t* r0 = m + (int64_t)ty.i0 * w;
  const uint8_t* r1 = m + (int64_t)ty.i1 * w;
  const double top = img_lerp(tab[r0[tx.i0]], tab[r0[tx.i1]], tx.t);
  const double bot = img_lerp(tab[r1[tx.i0]], tab[r1[tx.i1]], tx.t);
  return (float)img_lerp(top, bot, ty.t);
}

CSNET_IO_HD float img_sigmoid(float z) { return 1.f / (1.f + expf(-z)); }

// One output index of F.interpolate(mode='bilinear', align_corners=False) as ATen computes it in fp32: scale = (float)n_in / n_out,
// source = max(scale * (d + 0.5) - 0.5, 0), the upper sample clamped to the last one.  Not the skimage resize of img_tap.
struct MaeTap {
  int i0, i1;
  float l0, l1;
};

CSNET_IO_HD MaeTap mae_tap(int d, int n_in, float scale) {
  float src = scale * ((float)d + 0.5f) - 0.5f;
  src = src < 0.f ? 0.f : src;
  MaeTap r;
  r.i0 = (int)src;
  r.i1 = r.i0 < n_in - 1 ? r.i0 + 1 : r.i0;
  r.l1 = src - (float)r.i0;
  r.l0 = 1.f - r.l1;
  return r;
}

// One pixel of train.py's validation MAE (CSNet_training/train.py:273-278): s = sigmoid(z) resized to the GT's size, q = (int)(s * 255)
// truncated, |q / 255 - g / 255| in fp32, the GT side being float64 g / 255 rounded to fp32 (img_as_float, then .float()).
CSNET_IO_HD float img_mae_term(const float* z, int W, MaeTap ty, MaeTap tx, uint8_t g) {
  const float* r0 = z + (int64_t)ty.i0 * W;
  const float* r1 = z + (int64_t)ty.i1 * W;
  const float v = ty.l0 * (tx.l0 * img_sigmoid(r0[tx.i0]) + tx.l1 * img_sigmoid(r0[tx.i1])) +
                  ty.l1 * (tx.l0 * img_sigmoid(r1[tx.i0]) + tx.l1 * img_sigmoid(r1[tx.i1]));
  const int q = (int)(v * 255.f);
  return fabsf((float)q / 255.f - (float)((double)g / 255.0));
}

// Saliency map byte at the output pixel (ty, tx) of one image's logits plane z [H][W] (row stride W).
CSNET_IO_HD uint8_t img_out_value(const float* z, int W, ImgTap ty, ImgTap tx) {
  const float* r0 = z + (int64_t)ty.i0 * W;
  const float* r1 = z + (int64_t)ty.i1 * W;
  const double top = img_lerp((double)img_sigmoid(r0[tx.i0]), (double)img_sigmoid(r0[tx.i1]), tx.t);
  const double bot = img_lerp((double)img_sigmoid(r1[tx.i0]), (double)img_sigmoid(r1[tx.i1]), tx.t);
  const float s = (float)img_lerp(top, bot, ty.t);
  return (uint8_t)(s * 255.f);
}

// CSF+Res2Net's test path (CSF+Res2Net/dataset/dataset.py:83-96 load_image_test, solver.py:62-78 test): no resize on either side.
// Input channel c of a uint8 value u: numpy's three roundings, `in_ = f32(im) / 255` in fp32, then `in_ -= mean` and `in_ /= std`
// with float64 mean / std, each computed in float64 and stored back into the fp32 array.
CSNET_IO_HD float img_csf_in_value(uint8_t u, double mean, double stdv) {
  const float a = (float)u / 255.f;
  const float b = (float)((double)a - mean);
  return (float)((double)b / stdv);
}

// Map byte of a sigmoid value s: `255 * pred` in fp32, then cv2.imwrite's convertTo(CV_8U), i.e. saturate(round half to even).
// A NaN gives 0, as cvRound's INT_MIN saturates.
CSNET_IO_HD uint8_t img_csf_out_byte(float s) {
  const float r = rintf(255.f * s);
  return r >= 255.f ? (uint8_t)255 : (r > 0.f ? (uint8_t)r : (uint8_t)0);
}

CSNET_IO_HD uint8_t img_csf_out_value(float z) { return img_csf_out_byte(img_sigmoid(z)); }

// CSF+Res2Net's training sample (dataset.py:23-33 ImageDataTrain.__getitem__, load_image, load_sal_label, cv_random_flip): the image
// as img_csf_in_value (load_image rounds as load_image_test does), the label `np.array(Image.open(gt), float32) / 255.`, which numpy
// divides in fp32, and both flipped along W when randint(0, 1) gave 1.  No crop, no resize.
CSNET_IO_HD float img_csf_label_value(uint8_t u) { return (float)u / 255.f; }

// Stored column of output column x of a w-wide row, flipped (img[:, :, ::-1]) when flip is 1.
CSNET_IO_HD int img_csf_src_col(int x, int w, int flip) { return flip == 1 ? w - 1 - x : x; }

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

// Map byte at pixel (oy, ox) of an h x w map from one image's logits plane zn [H][W]: the two per-pixel map functions the map and
// SalMetric kernels are instantiated with.
struct CsnetMap {            // CSNet/test.py: sigmoid, skimage resize back to (h, w), truncation
  __device__ __forceinline__ uint8_t operator()(const float* zn, int H, int W, int h, int w, int oy, int ox) const {
    return img_out_value(zn, W, img_tap(oy, H, h), img_tap(ox, W, w));
  }
};

struct CsfMap {              // CSF+Res2Net solver.test: the logits are at the image's size (h, w == H, W), sigmoid, round to even
  __device__ __forceinline__ uint8_t operator()(const float* zn, int, int W, int, int, int oy, int ox) const {
    return img_csf_out_value(zn[(int64_t)oy * W + ox]);
  }
};

// fp32 logits [N,1,H,W] -> each image's uint8 map [h][w] at its dst_off.  Grid: (blocks per image, image); each block
// grid-strides over its image's pixels.
template <class Map>
__global__ void __launch_bounds__(kImgThreads) resize_out_u8_kernel(const float* __restrict__ z, int H, int W,
                                                                   const csnet_image_geom* __restrict__ geom, uint8_t* __restrict__ y) {
  const int n = blockIdx.y;
  const csnet_image_geom g = geom[n];
  const float* zn = z + (int64_t)n * H * W;
  uint8_t* out = y + g.dst_off;
  const int64_t hw = (int64_t)g.h * g.w;
  for (int64_t p = (int64_t)blockIdx.x * kImgThreads + threadIdx.x; p < hw; p += (int64_t)gridDim.x * kImgThreads) {
    const int oy = (int)p / g.w, ox = (int)p - oy * g.w;     // h * w < 2^31
    out[p] = Map()(zn, H, W, g.h, g.w, oy, ox);
  }
}

// SalMetric counts (sal_metric.cpp:86-120) of each image's map as resize_out_u8_kernel<Map> computes it, against the image's uint8 GT
// [h][w] at m + dst_off; the map is stored at y + dst_off only when y is non-null.  Grid as resize_out_u8_kernel.  Each warp counts
// into its own shared histograms (a saliency map piles most pixels into a few bins), the block adds them to image n's global ones
// with integer atomics: the counts are exact and do not depend on the grid or the batch.  hist_all / hist_pos / abs_sum start at 0.
template <class Map>
__global__ void __launch_bounds__(kImgThreads) salmetric_images_u8_kernel(const float* __restrict__ z, int H, int W,
                                                                         const csnet_image_geom* __restrict__ geom,
                                                                         const uint8_t* __restrict__ m, uint8_t* __restrict__ y,
                                                                         uint32_t* __restrict__ hist_all, uint32_t* __restrict__ hist_pos,
                                                                         unsigned long long* __restrict__ abs_sum) {
  constexpr int kWarps = kImgThreads / 32;
  __shared__ uint32_t ha[kWarps][256], hp[kWarps][256];
  __shared__ unsigned long long sd;
  const int n = blockIdx.y;
  const csnet_image_geom g = geom[n];
  const int64_t hw = (int64_t)g.h * g.w;
  if ((int64_t)blockIdx.x * kImgThreads >= hw) return;         // the whole block lies past a small image's end
  for (int i = threadIdx.x; i < kWarps * 256; i += kImgThreads) { (&ha[0][0])[i] = 0u; (&hp[0][0])[i] = 0u; }
  if (threadIdx.x == 0) sd = 0ull;
  __syncthreads();
  const float* zn = z + (int64_t)n * H * W;
  const uint8_t* gt = m + g.dst_off;
  uint32_t* wa = ha[threadIdx.x >> 5];
  uint32_t* wp = hp[threadIdx.x >> 5];
  unsigned long long d = 0;
  for (int64_t p = (int64_t)blockIdx.x * kImgThreads + threadIdx.x; p < hw; p += (int64_t)gridDim.x * kImgThreads) {
    const int oy = (int)p / g.w, ox = (int)p - oy * g.w;     // h * w < 2^31
    const uint8_t q = Map()(zn, H, W, g.h, g.w, oy, ox);
    if (y) y[g.dst_off + p] = q;
    const int t = gt[p];
    atomicAdd(&wa[q], 1u);
    if (t > 128) atomicAdd(&wp[q], 1u);
    d += (unsigned)(q > t ? q - t : t - q);
  }
  atomicAdd(&sd, d);
  __syncthreads();
  uint32_t sa = 0, sp = 0;                                      // kImgThreads == 256: one bin per thread
#pragma unroll
  for (int w = 0; w < kWarps; ++w) { sa += ha[w][threadIdx.x]; sp += hp[w][threadIdx.x]; }
  if (sa) atomicAdd(hist_all + (int64_t)n * 256 + threadIdx.x, sa);
  if (sp) atomicAdd(hist_pos + (int64_t)n * 256 + threadIdx.x, sp);
  if (threadIdx.x == 0 && sd) atomicAdd(abs_sum + n, sd);
}

// Training batch from a packed uint8 dataset (SalData.__getitem__ in train mode, CSNet_training/utils/prepare_data.py:109-139):
// sample n crops its image and mask to (h, w) at (y0, x0), flips them (1 'lr', 2 'ud') and resizes both to (H, W).  The crop and
// flip only move the taps (img_tap_crop).  Grid and column taps as resize_in_u8_kernel; y fp32 [N,3,H,W], target fp32 [N,1,H,W].
__global__ void __launch_bounds__(kImgThreads) train_batch_u8_kernel(const uint8_t* __restrict__ x, const uint8_t* __restrict__ m,
                                                                    const csnet_image_geom* __restrict__ geom,
                                                                    const csnet_train_sample* __restrict__ samples, int H, int W,
                                                                    const __grid_constant__ ImgNorm A, float* __restrict__ y,
                                                                    float* __restrict__ target) {
  __shared__ double tab[256];
  __shared__ double col_t[kImgThreads];
  __shared__ int col_i0[kImgThreads], col_i1[kImgThreads];
  const int n = blockIdx.y, oy0 = blockIdx.x * kImgRows, rows = H - oy0 < kImgRows ? H - oy0 : kImgRows;
  const csnet_train_sample s = samples[n];
  const csnet_image_geom g = geom[s.image];
  const uint8_t* img = x + g.src_off;
  const uint8_t* msk = m + g.dst_off;
  tab[threadIdx.x] = (double)threadIdx.x / 255.0;
  for (int cx0 = 0; cx0 < W; cx0 += kImgThreads) {
    const int sw = W - cx0 < kImgThreads ? W - cx0 : kImgThreads;
    __syncthreads();                                            // the previous slice's taps are consumed
    if ((int)threadIdx.x < sw) {
      const ImgTap t = img_tap_crop(img_tap(cx0 + threadIdx.x, s.w, W), s.x0, s.w, s.flip == 1);
      col_i0[threadIdx.x] = t.i0;
      col_i1[threadIdx.x] = t.i1;
      col_t[threadIdx.x] = t.t;
    }
    __syncthreads();
    for (int p = threadIdx.x; p < rows * sw; p += kImgThreads) {
      const int r = p / sw, cx = p - r * sw, oy = oy0 + r;
      const ImgTap ty = img_tap_crop(img_tap(oy, s.h, H), s.y0, s.h, s.flip == 2), tx{col_i0[cx], col_i1[cx], col_t[cx]};
#pragma unroll
      for (int c = 0; c < 3; ++c)
        y[(((int64_t)n * 3 + c) * H + oy) * W + cx0 + cx] = img_in_value(img, g.w, tab, ty, tx, c, A.mean[c], A.std[c]);
      target[((int64_t)n * H + oy) * W + cx0 + cx] = img_mask_value(msk, g.w, tab, ty, tx);
    }
  }
}

// CSF+Res2Net network input: N images of one size H x W, each packed uint8 HWC at its src_off -> fp32 [N,3,H,W]
// (img_csf_in_value).  Grid: (pixel blocks, image); a thread reads one pixel's 3 bytes and writes it to the 3 planes.
__global__ void __launch_bounds__(kImgThreads) csf_input_u8_kernel(const uint8_t* __restrict__ x, const csnet_image_geom* __restrict__ geom,
                                                                  int H, int W, const __grid_constant__ ImgNorm A, float* __restrict__ y) {
  const int n = blockIdx.y;
  const int64_t hw = (int64_t)H * W, p = (int64_t)blockIdx.x * kImgThreads + threadIdx.x;
  if (p >= hw) return;
  const uint8_t* px = x + geom[n].src_off + 3 * p;
  float* yn = y + (int64_t)n * 3 * hw + p;
#pragma unroll
  for (int c = 0; c < 3; ++c) yn[c * hw] = img_csf_in_value(px[c], A.mean[c], A.std[c]);
}

// CSF+Res2Net training batch: sample n is image samples[n].image of the packed set (H x W, as every sample of the call), flipped along
// W when its flip is 1 -> x fp32 [N,3,H,W] (img_csf_in_value) and target fp32 [N,1,H,W] (img_csf_label_value).  Grid as
// csf_input_u8_kernel: a thread reads one pixel's 3 image bytes and its mask byte.
__global__ void __launch_bounds__(kImgThreads) csf_train_batch_u8_kernel(const uint8_t* __restrict__ x, const uint8_t* __restrict__ m,
                                                                        const csnet_image_geom* __restrict__ geom,
                                                                        const csnet_train_sample* __restrict__ samples, int H, int W,
                                                                        const __grid_constant__ ImgNorm A, float* __restrict__ y,
                                                                        float* __restrict__ target) {
  const int n = blockIdx.y;
  const int64_t hw = (int64_t)H * W, p = (int64_t)blockIdx.x * kImgThreads + threadIdx.x;
  if (p >= hw) return;
  const csnet_train_sample s = samples[n];
  const csnet_image_geom g = geom[s.image];
  const int oy = (int)(p / W), ox = (int)(p - (int64_t)oy * W);
  const int64_t q = (int64_t)oy * W + img_csf_src_col(ox, W, s.flip);
  const uint8_t* px = x + g.src_off + 3 * q;
  float* yn = y + (int64_t)n * 3 * hw + p;
#pragma unroll
  for (int c = 0; c < 3; ++c) yn[c * hw] = img_csf_in_value(px[c], A.mean[c], A.std[c]);
  target[(int64_t)n * hw + p] = img_csf_label_value(m[g.dst_off + q]);
}

constexpr int kMaeThreads = 512;

// Validation MAE per image (train.py:262-279) from fp32 logits [N,1,H,W] and each image's uint8 GT [h][w] at its dst_off.  One block
// per image: every thread sums its pixels in double in a fixed order and the block adds the partial sums in a fixed tree, so an
// image's MAE has the same bits in any batch.
__global__ void __launch_bounds__(kMaeThreads) val_mae_u8_kernel(const float* __restrict__ z, int H, int W, const uint8_t* __restrict__ m,
                                                                const csnet_image_geom* __restrict__ geom, double* __restrict__ mae) {
  __shared__ double part[kMaeThreads / 32];
  const int n = blockIdx.x;
  const csnet_image_geom g = geom[n];
  const float* zn = z + (int64_t)n * H * W;
  const uint8_t* gt = m + g.dst_off;
  const float sy = (float)H / (float)g.h, sx = (float)W / (float)g.w;
  const int hw = g.h * g.w;                                     // h, w <= 32767
  double sum = 0.0;
  for (int p = threadIdx.x; p < hw; p += kMaeThreads) {
    const int oy = p / g.w, ox = p - oy * g.w;
    sum += (double)img_mae_term(zn, W, mae_tap(oy, H, sy), mae_tap(ox, W, sx), gt[p]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_down_sync(0xffffffffu, sum, o);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = sum;
  __syncthreads();
  if (threadIdx.x < 32) {
    sum = threadIdx.x < kMaeThreads / 32 ? part[threadIdx.x] : 0.0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_down_sync(0xffffffffu, sum, o);
    if (threadIdx.x == 0) mae[n] = sum / ((double)g.h * (double)g.w);
  }
}

inline ImgNorm img_norm(const float* mean, const float* stdv) {
  ImgNorm A{};
  for (int c = 0; c < 3; ++c) { A.mean[c] = (double)mean[c]; A.std[c] = (double)stdv[c]; }
  return A;
}

inline ImgNorm img_norm(const double* mean, const double* stdv) {
  ImgNorm A{};
  for (int c = 0; c < 3; ++c) { A.mean[c] = mean[c]; A.std[c] = stdv[c]; }
  return A;
}

inline void launch_resize_in(const uint8_t* x, const csnet_image_geom* geom, int N, int H, int W, const ImgNorm& A, float* y,
                             cudaStream_t stream) {
  resize_in_u8_kernel<<<dim3((unsigned)((H + kImgRows - 1) / kImgRows), (unsigned)N), kImgThreads, 0, stream>>>(x, geom, H, W, A, y);
}

// The map sizes live on the device, so the grid is sized from the batch alone: about 32 blocks per SM in all, which keeps the
// SMs busy to the end of a batch whose images differ in size; blocks past a small image's end exit at once.
template <class Map = CsnetMap>
inline void launch_resize_out(const float* z, int N, int H, int W, const csnet_image_geom* geom, uint8_t* y, int num_sms,
                              cudaStream_t stream) {
  const int bx = (32 * num_sms + N - 1) / N;
  resize_out_u8_kernel<Map><<<dim3((unsigned)bx, (unsigned)N), kImgThreads, 0, stream>>>(z, H, W, geom, y);
}

template <class Map = CsnetMap>
inline void launch_salmetric_images(const float* z, int N, int H, int W, const csnet_image_geom* geom, const uint8_t* m, uint8_t* y,
                                    uint32_t* hist_all, uint32_t* hist_pos, unsigned long long* abs_sum, int num_sms, cudaStream_t stream) {
  static_assert(kImgThreads == 256, "one histogram bin per thread");
  const int bx = (32 * num_sms + N - 1) / N;
  salmetric_images_u8_kernel<Map><<<dim3((unsigned)bx, (unsigned)N), kImgThreads, 0, stream>>>(z, H, W, geom, m, y, hist_all, hist_pos,
                                                                                               abs_sum);
}

inline void launch_csf_input(const uint8_t* x, const csnet_image_geom* geom, int N, int H, int W, const ImgNorm& A, float* y,
                             cudaStream_t stream) {
  const int64_t bx = ((int64_t)H * W + kImgThreads - 1) / kImgThreads;
  csf_input_u8_kernel<<<dim3((unsigned)bx, (unsigned)N), kImgThreads, 0, stream>>>(x, geom, H, W, A, y);
}

inline void launch_csf_train_batch(const uint8_t* x, const uint8_t* m, const csnet_image_geom* geom, const csnet_train_sample* samples,
                                   int N, int H, int W, const ImgNorm& A, float* y, float* target, cudaStream_t stream) {
  const int64_t bx = ((int64_t)H * W + kImgThreads - 1) / kImgThreads;
  csf_train_batch_u8_kernel<<<dim3((unsigned)bx, (unsigned)N), kImgThreads, 0, stream>>>(x, m, geom, samples, H, W, A, y, target);
}

inline void launch_train_batch(const uint8_t* x, const uint8_t* m, const csnet_image_geom* geom, const csnet_train_sample* samples, int N,
                               int H, int W, const ImgNorm& A, float* y, float* target, cudaStream_t stream) {
  train_batch_u8_kernel<<<dim3((unsigned)((H + kImgRows - 1) / kImgRows), (unsigned)N), kImgThreads, 0, stream>>>(x, m, geom, samples, H,
                                                                                                                    W, A, y, target);
}

inline void launch_val_mae(const float* z, int N, int H, int W, const uint8_t* m, const csnet_image_geom* geom, double* mae,
                           cudaStream_t stream) {
  val_mae_u8_kernel<<<(unsigned)N, kMaeThreads, 0, stream>>>(z, H, W, m, geom, mae);
}
#endif

}  // namespace csnet
