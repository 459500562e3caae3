/*
 * csnet_b200.h — C ABI of libcsnet_b200.so, the H100 (sm_90a) CSNet forward/backward engine.
 *
 * The reference (ShangHua-Gao/SOD100K) has no FFI of its own: its hot path is Python calling
 * torch.nn.functional (ATen/cuDNN).  This header is the boundary a maintainer would bind instead of
 * those library calls; every entry point names the reference call site it replaces.  All arguments
 * are plain pointers and sizes; device pointers are raw CUdeviceptr-compatible addresses; `stream`
 * is a cudaStream_t passed as void*.  No torch types cross this boundary.
 *
 * Execution model: the host side (sod100k_b200/compiler.py, mirroring the reference's module tree
 * CSNet/model/csnet.py) lowers a CSNet `layer_config` + `state_dict` into a flat PROGRAM: a tensor
 * table, a list of fused ops and one fp32 parameter blob.  A plan owns the blob copy and the
 * activation arena on one device and replays the program for a batch.
 *
 * Data layout in HBM: activations are planar NCHW (batch stride C*H*W, plane stride H*W, row
 * stride W, all dense), element type per tensor (fp32 / fp16 / bf16).  Channel counts are never
 * padded (CSNet widths are 8..79 and differ per layer), so algorithmic bytes == allocated bytes.
 *
 * Errors: every function returns 0 on success or a negative CSNET_E_* code; csnet_last_error()
 * returns a thread-local message.  The reference's own convention is Python exceptions
 * (CSNet/test.py:24 `assert`); the Python wrapper turns non-zero codes into RuntimeError.
 * Threading: a plan is used by one host thread / one stream at a time; no global mutable state.
 * Ownership: the caller owns inputs, outputs and parameters; the plan owns its blob copy + arena.
 */
#ifndef CSNET_B200_H
#define CSNET_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CSNET_ABI_VERSION 14

enum { CSNET_F32 = 0, CSNET_F16 = 1, CSNET_BF16 = 2 };

enum {
  CSNET_OK = 0,
  CSNET_E_INVALID = -1,   /* malformed program / argument */
  CSNET_E_CUDA = -2,      /* CUDA runtime error (message holds cudaGetErrorString) */
  CSNET_E_NOMEM = -3,
  CSNET_E_UNSUPPORTED = -4
};

#define CSNET_MAX_PATHS 8
#define CSNET_MAX_EXT 24

/* One activation tensor of the program (per image: [C,H,W]; a run adds the batch dimension). */
typedef struct {
  int32_t C, H, W;
  int32_t dtype;          /* CSNET_F32 / F16 / BF16 */
  int32_t external;       /* >= 0: bound at run time to ext_ptrs[external]; -1: lives in the arena */
  int32_t _pad;
  int64_t arena_offset;   /* bytes PER IMAGE from the arena base (multiple of 256); the run address is
                             base + N * arena_offset, so tensors of a smaller batch stay disjoint */
} csnet_tensor_desc;

/*
 * One accumulation path of a MIX op.  out[cout0 : cout0+cout] += path(src[c0 : c0+cin]).
 *
 * ksize > 0 — convolution path, replaces the F.conv2d calls of gOctaveConv.forward
 *   (CSNet/model/csnet.py:702-717), Conv2dX100.forward (CSNet/model/conv2d.py:104) and
 *   MSBlock.forward (csnet.py:141-146), with the resampling the reference does around them folded
 *   into the read: pre_avg=f (1 means 2) down-samples by f first — avg_pool2d(2,2) for f=2 (csnet.py:679-680) and
 *   F.interpolate(bilinear) to 1/f size for f=2,4,8 (CSF+Res2Net/networks/gOctConv.py:101-102) —, pool=k applies
 *   max_pool2d(k,k) next (csnet.py:709-712); the convolution (cross-correlation, zero padding `pad`,
 *   dilation `dil`, stride `stride`) then runs on that pooled grid.
 *   A plain 1x1 conv path may carry up > 1: the source is bilinearly up-sampled FIRST (same linear map as the
 *   reference's conv-then-interpolate; used by 16-bit programs when cin <= cout).
 * ksize == 0 — resample-add path: channel c of src is bilinearly up-sampled by the integer factor
 *   `up` (align_corners=False, source index (dst+0.5)/up-0.5 clamped at 0 — F.interpolate at
 *   csnet.py:705-707 and :382-385) and added to out[cout0+c]; cin == cout.
 */
typedef struct {
  int32_t src;            /* tensor id */
  int32_t c0, cin;
  int32_t pre_avg, pool;
  int32_t ksize, dil, stride, pad;
  int32_t up;
  int32_t cout0, cout;
  int64_t w_off;          /* blob offset (floats) of weights laid out [cin][ksize*ksize][cout] (cout innermost,
                             the compiler transposes the reference's [cout][cin][k][k]); -1 if ksize==0 */
} csnet_path_desc;

enum {
  CSNET_OP_MIX = 1,       /* dst = prelu(sum_paths + bias)   — gOctaveCBR / MSBlock / cls_layer */
  CSNET_OP_DW = 2,        /* dst = prelu(dw3x3(src) + bias)  — SimplifiedGOctConvBR branch */
  CSNET_OP_GN = 4,        /* dst = prelu(GroupNorm(src)): per-image statistics over (C/groups, H, W), eps 1e-5 — the CSF+Res2Net
                             head (CSF+Res2Net/networks/gOctConv.py:133, csf_res2net.py:220).  paths[0].src = input,
                             paths[0].up = groups, ext_off[0] / ext_off[1] = gamma / beta, slope_off = PReLU slope. */
  CSNET_OP_ILBLOCK = 3,   /* whole ILBlock of the 1x1 kind in one kernel (ILBlock.forward, csnet.py:72-76):
                             paths[0].src / paths[1].src = high / low resolution inputs (cin = channels),
                             dst / dst2 = high / low resolution outputs (dst2 = -1 for a 2->1 block);
                             16-bit activations only.  ext_off[] (blob offsets, floats):
                               0 WH  packed 16-bit [ru16(Cho)][K8], K8 = ru8(Chi+Cli): columns [W_hh | W_lh]
                                     (the kernel up-samples x_l before the conv: same linear map), BN scale folded
                               1 WL  packed 16-bit [ru16(Clo)][K8]: columns [W_ll | W_hl] (x_l, then max-pooled x_h)
                               2,3   conv bias / PReLU slope of the hi branch      4,5  of the lo branch
                               6-8   conv3x3_1 hi: weights [C][9], bias, slope     9-11 conv3x3_1 lo
                               12-14 conv3x3_2 hi                                  15-17 conv3x3_2 lo
                             Stem form (the first block, `first=True`, csnet.py:60-71): paths[0] and paths[1] both name
                             the fp32 input image (cin <= 3) with ksize = 3, pad = 1, paths[1].pool = 2; both branches are
                             3x3 convs of it (lo: of its 2x2 max-pool).  WH / WL are then [ru16(C)][32] with column
                             k = ci*9 + ky*3 + kx; the kernel builds the im2col planes in shared memory. */
  CSNET_OP_MIXPROJ = 5,    /* a MIX op whose Cmid-channel result is never stored: a 1x1 projection to the single dst channel
                             runs in the epilogue, dst = proj_b + sum_c proj_w[c] * prelu(mix[c] + bias[c])  (CSNet.forward,
                             csnet.py:383-384: fuse1x1 -> cls_layer).  paths / bias_off / slope_off describe the Cmid-channel
                             MIX; ext_off[0] = proj_w offset (Cmid floats), ext_off[1] = proj_b offset or -1,
                             ext_off[2] = Cmid (<= 80).  Tensor-core kernel only: 16-bit sources, stride-1 conv paths. */
  CSNET_OP_RESIZE = 6      /* bilinear resize to the destination's size, any ratio (F.interpolate(size=dst (H, W), mode='bilinear',
                             align_corners=False): CSF+Res2Net/networks/gOctConv.py:99,102 and csf_res2net.py:258):
                               dst[:, cout0 + c] = (accumulate ? dst[:, cout0 + c] : 0) + bilinear(src[:, c0 + c]),  c < cout.
                             Per axis scale = (float)in / out, source index max(scale * (d + 0.5) - 0.5, 0), the upper tap clamped
                             at the border; the four taps are combined in fp32 in ATen's order, an accumulate adds once in fp32
                             and rounds once to dst's dtype.  Any sizes >= 1 on either side; src / dst fp32, fp16 or bf16 each.
                             paths[0]: src, c0, cin, cout0, cout with cin == cout and ksize == 0; pre_avg, pool, dil, stride,
                             pad and up are unused and must be 0 or 1, w_off -1.  n_paths == 1, src != dst, dst2 == -1,
                             bias_off == slope_off == -1.  ext_off[0] = accumulate flag (0 or 1), ext_off[1..23] == -1.
                             An accumulate reads its destination: a plan with exactly two externals runs small batches through
                             staging buffers (csnet_plan_run) that do not hold external 1's old values. */
};

/*
 * One fused op.  Epilogue (both kinds): y = acc + bias[c] (bias_off >= 0), then PReLU with
 * per-channel slope (slope_off >= 0): y > 0 ? y : slope[c]*y  (F.batch_norm + F.prelu,
 * csnet.py:786,791,846-847,148; eval-mode BN scale is folded into the weights by the compiler).
 * CSNET_OP_DW uses paths[0] with ksize=3, dil=1, pad=1, cin==cout, weights [C][9]
 * (Conv2dX100 groups=C, csnet.py:817-824).
 */
typedef struct {
  int32_t kind;
  int32_t dst;            /* tensor id */
  int32_t n_paths;
  int32_t dst2;           /* second destination (CSNET_OP_ILBLOCK) or -1 */
  int64_t bias_off;       /* blob offset of bias[dst.C] or -1 */
  int64_t slope_off;      /* blob offset of PReLU slope[dst.C] or -1 */
  csnet_path_desc paths[CSNET_MAX_PATHS];
  int64_t ext_off[CSNET_MAX_EXT];   /* kind-specific blob offsets, -1 when unused.  CSNET_OP_MIX: ext_off[23] == 1
                                       forbids the tensor-core kernel (weights do not fit the 16-bit operand type) */
} csnet_op_desc;

typedef struct csnet_plan csnet_plan;

/* ABI version of the loaded library (== CSNET_ABI_VERSION of the header it was built from). */
int csnet_abi_version(void);

/* Thread-local description of the last error returned on this thread ("" if none). */
const char* csnet_last_error(void);

/* Number of CUDA devices visible; < 0 on error.  Used by the wrapper to fail loudly without a GPU. */
int csnet_device_count(void);

/*
 * Build a plan on `device` for batches up to `max_batch`.  Validates the program (shapes of every
 * path against its destination, blob bounds) and allocates blob + arena.
 * Replaces: model construction + `.cuda()` (CSNet/test.py:39-40, CSNet_training/train.py:77-92).
 */
int csnet_plan_create(csnet_plan** out, const csnet_tensor_desc* tensors, int32_t n_tensors,
                      const csnet_op_desc* ops, int32_t n_ops, int64_t blob_floats,
                      int32_t max_batch, int32_t device);

/* Upload the fp32 parameter blob (host pointer, `n` floats == blob_floats) on `stream`.
 * Replaces: load_state_dict + per-call `100.0 * weight` / BN arithmetic (conv2d.py:104, csnet.py:786). */
int csnet_plan_set_blob(csnet_plan* plan, const float* host_blob, int64_t n, void* stream);

/*
 * Run the program for a batch of N images.  ext_ptrs[i] is the DEVICE address bound to tensors with
 * external == i (network input fp32 NCHW, logits fp32 NCHW, ...).  Asynchronous on `stream`.
 * Replaces: CSNet.forward (CSNet/model/csnet.py:365-387) == `model(input_var)` at CSNet/test.py:90.
 */
int csnet_plan_run(csnet_plan* plan, int32_t N, const void* const* ext_ptrs, int32_t n_ext, void* stream);

/*
 * Same as csnet_plan_run, but records a CUDA event on `stream` around every op and writes each op's device
 * time in milliseconds to ms_per_op[n_ops] (synchronises the stream).  Measurement aid for bench.py's roofline.
 */
int csnet_plan_profile(csnet_plan* plan, int32_t N, const void* const* ext_ptrs, int32_t n_ext, void* stream,
                       float* ms_per_op, int32_t n_ops);

/* Device address of an arena tensor for a batch of N (for tests / taps); NULL if external/invalid. */
void* csnet_plan_tensor_ptr(csnet_plan* plan, int32_t tensor, int32_t N);

/* Copy an arena tensor of the last run of batch N into caller-owned DEVICE memory (same dtype, dense). */
int csnet_plan_read_tensor(csnet_plan* plan, int32_t tensor, int32_t N, void* dst_device, void* stream);

/* Name of the kernel (family) csnet_plan_run launches for op `op_index` of this plan — measurement aid: bench.py groups the per-op
 * times of csnet_plan_profile by kernel to find the dominant one.  "" for an invalid index. */
const char* csnet_plan_op_kernel(const csnet_plan* plan, int32_t op_index);

/* Number of kernel launches one csnet_plan_run issues (bench.py reports it as gpu_launches). */
int32_t csnet_plan_launches(const csnet_plan* plan);

/* Bytes of arena the plan holds. */
int64_t csnet_plan_arena_bytes(const csnet_plan* plan);

void csnet_plan_destroy(csnet_plan* plan);

/*
 * Convenience for hosts that keep their data in pageable/pinned HOST memory (the e2e path of
 * bench.py and of CSNet/test.py:86-93): copies x (fp32 NCHW, N*3*H*W floats) to the device, runs,
 * copies the logits (N*H*W floats) back and returns when y_host is complete.  Batches of 64 or more are cut into
 * three chunks (N/8, the rest, N/8) that pipeline H2D copy / kernels / D2H copy on separate streams (use pinned host memory).
 * Smaller batches, and every batch of csnet_plan_run_host_u8, run as one chunk (csnet_plan_run_host_images_u8 cuts like this call).
 * The plan must bind external 0 = input, external 1 = logits.
 */
int csnet_plan_run_host(csnet_plan* plan, int32_t N, const float* x_host, float* y_host, void* stream);

/*
 * Same pipeline with the reference's pre- and post-processing moved onto the device (CSNet/test.py:68-69,86-96; SURVEY §8 f3):
 * x_hwc = uint8 [N][H][W][3] images as io.imread returns them (already at the network size), y_u8 = uint8 [N][H][W] saliency maps
 * = (sigmoid(logits) * 255) truncated, exactly what test.py writes to png.  The input becomes (x / 255 - mean[c]) / std[c]
 * (evaluated in float64, rounded to fp32, like the host code).  4x fewer bytes over PCIe in both directions.
 */
int csnet_plan_run_host_u8(csnet_plan* plan, int32_t N, const uint8_t* x_hwc, uint8_t* y_u8, const float* mean, const float* std,
                           void* stream);

/*
 * Images of any size (CSNet/test.py:71-98 with both of its skimage resizes, SURVEY §8 f3).  A ragged batch is packed: image i is
 * uint8 [h][w][3] at byte src_off of the input, and its saliency map is uint8 [h][w] at byte dst_off of the output.
 *   in:  resize(img_as_float(img), (H, W), mode='reflect', anti_aliasing=False), then (v - mean[c]) / std[c], all in float64,
 *        rounded once to the fp32 NCHW network input [N,3,H,W];
 *   out: sigmoid(logit) in fp32, resize back to (h, w) the same way (float64, rounded to fp32), * 255 truncated to uint8.
 * The resize is skimage >= 0.19's: scipy.ndimage.zoom(order=1, mode='mirror', grid_mode=True).  At h, w == H, W both sides give
 * exactly the bytes of csnet_plan_run_host_u8.
 */
typedef struct {
  int64_t src_off;        /* byte offset of the image in the packed input */
  int64_t dst_off;        /* byte offset of its map in the packed output */
  int32_t h, w;
} csnet_image_geom;       /* 24 bytes */

/* Device to device, asynchronous on `stream` (current device): x_packed / geom (DEVICE, N entries) -> x_nchw fp32 [N,3,H,W].
 * mean / std are host float[3].  The caller guarantees that every image lies inside x_packed (geometry on the device is not checked). */
int csnet_resize_u8_to_input(const uint8_t* x_packed, const csnet_image_geom* geom, int32_t N, int32_t H, int32_t W, const float* mean,
                             const float* std, float* x_nchw, void* stream);

/* Device to device, asynchronous on `stream`: logits fp32 [N,1,H,W] -> each image's map at y_packed + dst_off (geometry on the
 * DEVICE; the maps must not overlap). */
int csnet_resize_logits_to_u8(const float* logits, int32_t N, int32_t H, int32_t W, const csnet_image_geom* geom, uint8_t* y_packed,
                              void* stream);

/* SalMetric on the maps csnet_resize_logits_to_u8 would write, without the png round trip (CSNet/eval.py, sal_metric.cpp:86-120).
 * Device to device, asynchronous on `stream` (current device): logits fp32 [N,1,H,W], geometry on the DEVICE, image n's GT uint8 [h][w]
 * at m_packed + dst_off (the masks of a SalImages set).  Each map byte q is computed as csnet_resize_logits_to_u8 computes it; per
 * image n: hist_all[n][q]++, hist_pos[n][q]++ where gt > 128, abs_sum[n] += |q - gt| (DEVICE uint32 [N][256], [N][256], uint64 [N],
 * zeroed by the call).  The counts are exact and the same for an image in any batch.  y_packed may be NULL: with it the maps are
 * also stored at y_packed + dst_off, without it no map is written. */
int csnet_salmetric_images_u8(const float* logits, int32_t N, int32_t H, int32_t W, const csnet_image_geom* geom, const uint8_t* m_packed,
                              uint8_t* y_packed, uint32_t* hist_all, uint32_t* hist_pos, unsigned long long* abs_sum, void* stream);

/*
 * Host to host, synchronised like csnet_plan_run_host: x_packed (x_bytes bytes) and the HOST geometry geom[N] in, the maps out to
 * y_packed (y_bytes bytes), through the plan's network size H x W.  Every entry is checked before any copy or launch: 1 <= h, w <=
 * 32767, every image inside x_bytes, every map inside y_bytes, and the maps back to back in input order (each map's dst_off is
 * where the previous one ends).  Anything else returns CSNET_E_INVALID.  Same pipeline as csnet_plan_run_host (pinned memory for
 * overlap); the plan's input must have 3 channels.
 */
int csnet_plan_run_host_images_u8(csnet_plan* plan, int32_t N, const uint8_t* x_packed, int64_t x_bytes, const csnet_image_geom* geom,
                                  uint8_t* y_packed, int64_t y_bytes, const float* mean, const float* std, void* stream);

/*
 * Training data on the device (CSNet_training/utils/prepare_data.py:109-139 SalData.__getitem__, train.py:250-293 val).  A dataset
 * is packed once: image i is uint8 [h][w][3] at byte src_off of x_packed, its mask uint8 [h][w] at byte dst_off of m_packed
 * (csnet_image_geom as above).  Geometry and samples live on the DEVICE and are not checked there; the caller guarantees every
 * index, window and offset.  Bad scalar arguments return CSNET_E_INVALID.  Asynchronous on `stream` (current device).
 */
typedef struct {
  int32_t image;          /* index into geom */
  int32_t y0, x0, h, w;   /* crop window img[y0:y0+h, x0:x0+w] */
  int32_t flip;           /* 0 none, 1 'lr' (np.fliplr), 2 'ud' (np.flipud), applied after the crop */
} csnet_train_sample;     /* 24 bytes */

/* N training samples: x_nchw fp32 [N,3,H,W] = ((resize(crop/flip(x / 255)) - mean[c]) / std[c]) and target fp32 [N,1,H,W] =
 * resize(crop/flip(m / 255)), evaluated in float64 and rounded once, the resize being csnet_resize_u8_to_input's.  mean / std are
 * host float[3]; samples DEVICE [N]. */
int csnet_train_batch_u8(const uint8_t* x_packed, const uint8_t* m_packed, const csnet_image_geom* geom, const csnet_train_sample* samples,
                         int32_t N, int32_t H, int32_t W, const float* mean, const float* std, float* x_nchw, float* target, void* stream);

/* Validation MAE per image (train.py:262-279): logits fp32 [N,1,H,W], image n's GT uint8 [h][w] at m_packed + geom[n].dst_off
 * (geom DEVICE [N]).  mae DEVICE float64 [N] = mean |(int)(interp(sigmoid(z)) * 255) / 255 - g / 255|, interp being
 * F.interpolate(size=(h, w), mode='bilinear', align_corners=False) in fp32.  Deterministic: no atomics, the same bits for an image
 * in any batch. */
int csnet_val_mae_u8(const float* logits, int32_t N, int32_t H, int32_t W, const uint8_t* m_packed, const csnet_image_geom* geom,
                     double* mae, void* stream);

/*
 * CSF+Res2Net's test path (CSF+Res2Net/solver.py:62-78 with dataset.py:83-96 load_image_test): every image runs at its own size, so
 * a call takes N images that are all H x W (each geom entry's h, w equal H, W) and nothing is resized.  Packed sets, geometry on the
 * DEVICE (not checked there), CSNET_E_INVALID for a null pointer or N outside [1, 65535] or H, W outside [1, 32767], asynchronous on
 * `stream` (current device), as the calls above.
 */
/* x_nchw fp32 [N,3,H,W] from the uint8 HWC images at src_off, with numpy's three roundings:
 * x = f32(f64(f32(f64(f32(u) / 255.f) - mean[c])) / std[c]).  mean / std are host double[3]. */
int csnet_csf_input_u8(const uint8_t* x_packed, const csnet_image_geom* geom, int32_t N, int32_t H, int32_t W, const double* mean,
                       const double* std, float* x_nchw, void* stream);

/* Training samples (CSF+Res2Net/solver.py:81-127 with dataset.py:23-33, 69-114): sample n is image samples[n].image of the packed set,
 * flipped along W when samples[n].flip is 1 (cv_random_flip), never cropped or resized.  x_nchw fp32 [N,3,H,W] as csnet_csf_input_u8
 * computes it; target fp32 [N,1,H,W] = f32(m) / 255.f from the mask at m_packed + dst_off (load_sal_label).  samples DEVICE [N] with
 * y0 = x0 = 0, h = H, w = W, flip 0 or 1; mean / std host double[3]. */
int csnet_csf_train_batch_u8(const uint8_t* x_packed, const uint8_t* m_packed, const csnet_image_geom* geom, const csnet_train_sample* samples,
                             int32_t N, int32_t H, int32_t W, const double* mean, const double* std, float* x_nchw, float* target,
                             void* stream);

/* Logits fp32 [N,1,H,W] -> each image's map at y_packed + dst_off, q = saturate(rint(255.f * sigmoid(z))) with round half to even
 * (cv2.imwrite of solver.test's fp32 array) and sigmoid = 1.f / (1.f + expf(-z)) as torch's CUDA kernel computes it. */
int csnet_csf_maps_u8(const float* logits, int32_t N, int32_t H, int32_t W, const csnet_image_geom* geom, uint8_t* y_packed, void* stream);

/* csnet_salmetric_images_u8 for the maps csnet_csf_maps_u8 writes: the same outputs, zeroed by the call, exact and the same for an
 * image in any batch; y_packed may be NULL. */
int csnet_salmetric_csf_u8(const float* logits, int32_t N, int32_t H, int32_t W, const csnet_image_geom* geom, const uint8_t* m_packed,
                           uint8_t* y_packed, uint32_t* hist_all, uint32_t* hist_pos, unsigned long long* abs_sum, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Training primitives (fp32 planar NCHW device tensors; the _bf16 calls below store activations in bf16).  The reference trains through torch autograd
 * (CSNet_training/train.py:203-216); train-mode BatchNorm makes the reference MODULE the closed unit, so the
 * boundary is one call per module piece.  sod100k_b200/train_ops.py wraps them in torch.autograd.Function s.
 * All return 0 / CSNET_E_*; csnet_train_last_error() holds the message.
 * ------------------------------------------------------------------------------------------------------------ */

/* One path of a raw (pre-BN) conv mix, device pointers resolved.  Same semantics as csnet_path_desc; `w` is the
 * path's weight in kernel layout [cin][ksize*ksize][cout] (fp32), NULL for resample-add paths (ksize == 0). */
typedef struct {
  const void* src;        /* [N, C, H, W]: fp32 for the calls above, the call's source dtype for the _bf16 calls */
  const float* w;
  int32_t C, H, W;
  int32_t c0, cin;
  int32_t pre_avg, pool;
  int32_t ksize, dil, stride, pad;
  int32_t up;
  int32_t cout0, cout;
} csnet_train_path;

const char* csnet_train_last_error(void);

/* F.batch_norm(training=True) statistics: per-channel mean and BIASED variance over (N, H*W)  (csnet.py:786,846). */
int csnet_train_bn_stats(const float* z, int32_t N, int32_t C, int32_t HW, float* mean, float* var, void* stream);
/* y = PReLU(gamma*(z-mean)/sqrt(var+eps)+beta); gap (optional, [N*C]) = per-image channel means of y, the quantity
 * Oct_bn_hook pools (csnet.py:403-404). */
int csnet_train_bn_prelu_fwd(const float* z, float* y, int32_t N, int32_t C, int32_t HW, const float* mean, const float* var,
                             const float* gamma, const float* beta, const float* slope, float eps, float* gap, void* stream);
/* autograd of the above: dz plus dgamma / dbeta / dslope ([C] each).  frozen=1: mean / var were constants (eval-mode
 * BatchNorm inside a training graph, as CSF+Res2Net/solver.py keeps its net), so the batch-statistic terms vanish. */
int csnet_train_bn_prelu_bwd(const float* z, const float* dy, float* dz, int32_t N, int32_t C, int32_t HW, const float* mean,
                             const float* var, const float* gamma, const float* beta, const float* slope, float eps,
                             float* dgamma, float* dbeta, float* dslope, int32_t frozen, void* stream);
/* Depthwise 3x3 pad 1 with effective weight scale*w (Conv2dX100, conv2d.py:104); transposed=1 gives the data gradient. */
int csnet_train_dw_conv(const float* x, const float* w, float* y, int32_t N, int32_t C, int32_t H, int32_t W, float scale,
                        int32_t transposed, void* stream);
int csnet_train_dw_wgrad(const float* x, const float* dy, float* dw, int32_t N, int32_t C, int32_t H, int32_t W, float scale,
                         void* stream);
/* Both gradients of the depthwise conv in one pass over dy (autograd of F.conv2d(x, 100 * w, groups=C), conv2d.py:104): dx [N,C,H,W], dw [C][9]. */
int csnet_train_dw_bwd(const float* x, const float* dy, const float* w, float* dx, float* dw, int32_t N, int32_t C, int32_t H, int32_t W,
                       float scale, void* stream);
/* Raw conv mix (gOctaveConv.forward csnet.py:664-726 for one output branch; MSBlock :141-146): dst = sum of paths. */
int csnet_train_mix_fwd(float* dst, int32_t N, int32_t C, int32_t H, int32_t W, const csnet_train_path* paths, int32_t n_paths,
                        void* stream);
/* Gradient of one path w.r.t. its source slice: dsrc is [N, cin, path.H, path.W] (through max/avg pooling, the conv,
 * or the bilinear up-sample for resample paths). */
int csnet_train_mix_dgrad(const float* ddst, int32_t N, int32_t C, int32_t H, int32_t W, const csnet_train_path* path, float* dsrc,
                          void* stream);
/* Gradient of one conv path w.r.t. its weight, kernel layout [cin][k*k][cout]. */
int csnet_train_mix_wgrad(const float* ddst, int32_t N, int32_t C, int32_t H, int32_t W, const csnet_train_path* path, float* dw,
                          void* stream);
/* The down-sampling a path carries, materialised once (F.avg_pool2d(2) of a stride-2 gOctaveConv, csnet.py:683-686, then F.max_pool2d(pool)
 * of a high -> low path, :692-698): dst [N, cin, Hs/f, Ws/f] from channels [c0, c0+cin) of src [N, Cs, Hs, Ws], f = (pre_avg ? 2 : 1) * pool;
 * idx (uint8, same shape, required when pool > 1) = position of the first maximum in the window.  _bwd routes the gradient of dst back to
 * dsrc [N, cin, Hs, Ws] the way autograd does (max: to the recorded position; average: a quarter to each). */
int csnet_train_pool_fwd(const float* src, int32_t N, int32_t Cs, int32_t c0, int32_t cin, int32_t Hs, int32_t Ws, int32_t pre_avg, int32_t pool,
                         float* dst, uint8_t* idx, void* stream);
int csnet_train_pool_bwd(const float* dpool, const uint8_t* idx, int32_t N, int32_t cin, int32_t Hs, int32_t Ws, int32_t pre_avg, int32_t pool,
                         float* dsrc, void* stream);
/* Channel slimming on the device (SURVEY 8 f4; build_model_with_weight and its loaders, CSNet_training/model/csnet.py:571-818):
 * dst[i][j][:] = src[out_idx[i]][in_idx[j]][:] for i < n_out, j < n_in; src is [Co][Ci][kk] fp32, dst [dCo][dCi][kk] (the caller zeroes it:
 * the reference fills torch.zeros), the index lists are device int64 (torch.nonzero of the BatchNorm-gamma masks). */
int csnet_slim_gather(const float* src, int32_t Co, int32_t Ci, int32_t kk, const int64_t* out_idx, int32_t n_out, const int64_t* in_idx, int32_t n_in,
                      float* dst, int32_t dCo, int32_t dCi, void* stream);
/* F.binary_cross_entropy_with_logits (mean) and its gradient * grad_scale (train.py:209). */
int csnet_train_bce(const float* logits, const float* target, float* dlogits, float* loss, int64_t n, float grad_scale, void* stream);
/* F.binary_cross_entropy_with_logits(reduction='sum') / divisor (CSF+Res2Net/solver.py:101-102): loss[0] = fp32 sum of the n terms
 * divided by (float)divisor, dlogits (may be NULL) = (sigmoid(z) - t) * f32(1 / divisor).  Deterministic: per-block partials merged
 * in a fixed order, no floating-point atomics, the block count a function of n alone.  n >= 1, divisor >= 1. */
int csnet_train_bce_sum(const float* logits, const float* target, float* dlogits, float* loss, int64_t n, int32_t divisor, void* stream);
/* torch.optim.Adam step (train.py:108-123) over many tensors: `chunk_table_device` = n_chunks records
 * {float* p; const float* g; float* m; float* v; int32 n; float weight_decay} (40 bytes each). */
int csnet_train_adam(const void* chunk_table_device, int32_t n_chunks, float lr, float beta1, float beta2, float eps, int32_t step,
                     float grad_scale, void* stream);

/* ---- bf16 activation storage (sod100k_b200/train_ops.py picks these when the step stores bf16) ---------------------------------
 * The same operations as the fp32 calls above, on bf16 planar NCHW activations and activation gradients (pointers are void*).
 * Weights, weight gradients, BatchNorm mean / var / gamma / beta / slope and their gradients, and the per-image channel means stay
 * fp32; every kernel accumulates in fp32 and rounds each bf16 store to nearest even; reductions keep the fp32 calls' order (no
 * floating-point atomics: the same bits on every run).  Where a call can mix types, a dtype argument (CSNET_BF16 or CSNET_F32)
 * names each side, and at least one side is bf16: the stem reads the fp32 network input, cls_layer writes fp32 logits.
 * A shape the register-tiled kernels do not take (a stride-2 or pooled conv path not materialised by _pool_fwd_bf16, rows wider
 * than 1024 pixels, mixed kernel sizes in one mix, a 1x1 mix with over 96 KiB of weights) returns CSNET_E_UNSUPPORTED; nothing is
 * computed in fp32 behind the caller. */
int csnet_train_bn_stats_bf16(const void* z, int32_t N, int32_t C, int32_t HW, float* mean, float* var, void* stream);
int csnet_train_bn_prelu_fwd_bf16(const void* z, void* y, int32_t N, int32_t C, int32_t HW, const float* mean, const float* var,
                                  const float* gamma, const float* beta, const float* slope, float eps, float* gap, void* stream);
int csnet_train_bn_prelu_bwd_bf16(const void* z, const void* dy, void* dz, int32_t N, int32_t C, int32_t HW, const float* mean,
                                  const float* var, const float* gamma, const float* beta, const float* slope, float eps,
                                  float* dgamma, float* dbeta, float* dslope, int32_t frozen, void* stream);
int csnet_train_dw_conv_bf16(const void* x, const float* w, void* y, int32_t N, int32_t C, int32_t H, int32_t W, float scale,
                             int32_t transposed, void* stream);
int csnet_train_dw_wgrad_bf16(const void* x, const void* dy, float* dw, int32_t N, int32_t C, int32_t H, int32_t W, float scale,
                              void* stream);
int csnet_train_dw_bwd_bf16(const void* x, const void* dy, const float* w, void* dx, float* dw, int32_t N, int32_t C, int32_t H,
                            int32_t W, float scale, void* stream);
/* every path's src has src_dtype; dst has dst_dtype */
int csnet_train_mix_fwd_bf16(void* dst, int32_t dst_dtype, int32_t N, int32_t C, int32_t H, int32_t W, const csnet_train_path* paths,
                             int32_t n_paths, int32_t src_dtype, void* stream);
/* conv paths: ddst / dsrc of the given dtypes; resample paths: both bf16 */
int csnet_train_mix_dgrad_bf16(const void* ddst, int32_t ddst_dtype, int32_t N, int32_t C, int32_t H, int32_t W,
                               const csnet_train_path* path, void* dsrc, int32_t dsrc_dtype, void* stream);
/* path.src has src_dtype, ddst has ddst_dtype; dw is fp32 */
int csnet_train_mix_wgrad_bf16(const void* ddst, int32_t ddst_dtype, int32_t N, int32_t C, int32_t H, int32_t W,
                               const csnet_train_path* path, float* dw, int32_t src_dtype, void* stream);
/* the pooled copy of a bf16 source is bf16 */
int csnet_train_pool_fwd_bf16(const void* src, int32_t N, int32_t Cs, int32_t c0, int32_t cin, int32_t Hs, int32_t Ws, int32_t pre_avg,
                              int32_t pool, void* dst, uint8_t* idx, void* stream);
int csnet_train_pool_bwd_bf16(const void* dpool, const uint8_t* idx, int32_t N, int32_t cin, int32_t Hs, int32_t Ws, int32_t pre_avg,
                              int32_t pool, void* dsrc, void* stream);

/* ---- synchronized BatchNorm + PReLU (nn.SyncBatchNorm over G ranks; csrc/bn_sync.cu) -------------------------------------------
 * Each direction is two calls around one all-reduce(SUM) the caller issues on a zeroed float64 row buffer in which rank `rank`
 * fills only its own row, so the sum is an exact gather and every rank merges the same rows in rank order.  z / dy / dz hold
 * `dtype` (CSNET_F32 or CSNET_BF16); the forward between the two halves is csnet_train_bn_prelu_fwd[_bf16] with the merged
 * statistics.  No floating-point atomics: the same bits on every run. */
/* row `rank` of rows [G][C][3] = (count, mean, M2 = sum (z - mean)^2) of each channel over this rank's z [N][C][HW] */
int csnet_train_bn_sync_partial(const void* z, int32_t dtype, int32_t N, int32_t C, int32_t HW, int32_t rank, double* rows,
                                void* stream);
/* rows 0..G-1 merged in rank order (Chan's pairwise update, float64): mean / biased var [C] of the global batch; count[0]: its size */
int csnet_train_bn_sync_merge(const double* rows, int32_t G, int32_t C, float* mean, float* var, double* count, void* stream);
/* mean / var: the merged statistics.  dgamma / dbeta / dslope [C]: this rank's parameter gradients; row `rank` of rows [G][C][2] =
 * (sum du, sum du * xhat) over this rank's batch */
int csnet_train_bn_sync_bwd_reduce(const void* z, const void* dy, int32_t dtype, int32_t N, int32_t C, int32_t HW, const float* mean,
                                   const float* var, const float* gamma, const float* beta, const float* slope, float eps, float* dgamma,
                                   float* dbeta, float* dslope, int32_t rank, double* rows, void* stream);
/* dz = gamma r (du - S1 / M - xhat S2 / M), S1 / S2 the rows of all G ranks summed in rank order, M = count[0] (global) */
int csnet_train_bn_sync_bwd_apply(const void* z, const void* dy, void* dz, int32_t dtype, int32_t N, int32_t C, int32_t HW, const float* mean,
                                  const float* var, const float* gamma, const float* beta, const float* slope, float eps, const double* rows,
                                  int32_t G, const double* count, void* stream);

/* ---- CSF+Res2Net head training (fp32; sod100k_b200/modular_r.py wraps them) ---------------------------------------------------
 * Convolutions as an fp32 FMA implicit GEMM (csrc/gemm_f32.cuh).  One segment is one stride-1 convolution of a channel slice of
 * `src` with a weight slice: element (co, ci, ky, kx) of the weight is w[co * ldw + ci * ksize * ksize + ky * ksize + kx]
 * (a slice [co0:, ci0:] of an OIHW parameter is w = param + (co0 * Cin + ci0) * k * k, ldw = Cin * k * k).  ksize is 1, or 3
 * with dilation `dil` and zero padding `dil`; every tensor has the destination's H x W.  All segments of one call share ksize.
 * Split-K partials go to the caller's workspace `ws` and are merged in split order: no floating-point atomics, the same bits on
 * every run.  splits = 0 / tile = 0 let the library choose; tile 1 is the 64x64 block tile, 2 the 128x128 one. */
typedef struct {
  const float* src;       /* fp32 [N, C, H, W]: fwd / wgrad the conv's input, dgrad the gradient of the conv's output tensor */
  const float* w;         /* weight slice (unused by wgrad, which writes the gradient at the same layout) */
  int32_t C, c0, cin;     /* channels of src; the conv reads input channels [c0, c0 + cin) (dgrad: c0 unused) */
  int32_t cout0, cout;    /* the conv's output channels [cout0, cout0 + cout): fwd writes them, dgrad / wgrad read their gradient */
  int32_t ksize, dil, ldw;
} csnet_conv_seg;         /* 48 bytes */

enum { CSNET_CONV_FWD = 0, CSNET_CONV_DGRAD = 1, CSNET_CONV_WGRAD = 2 };

/* The launch a conv call makes: splits, the longest chain of fp32 additions one output element passes through before the split
 * merge (chain), and the workspace bytes it needs.  Arguments as the call's. */
int csnet_train_conv_plan(int32_t form, int32_t N, int32_t H, int32_t W, const csnet_conv_seg* segs, int32_t n_segs, int32_t splits,
                          int32_t tile, int32_t* splits_out, int32_t* chain_out, int64_t* ws_bytes);
/* dst[:, cout0:cout0+cout] (+)= bias + sum over segments of conv(src[:, c0:c0+cin], w): segments share cout0 / cout (and cin may
 * differ); dst is fp32 [N, C, H, W]; bias [cout] or NULL; accumulate adds the old value once. */
int csnet_train_conv_fwd(float* dst, int32_t N, int32_t C, int32_t H, int32_t W, const csnet_conv_seg* segs, int32_t n_segs,
                         const float* bias, int32_t accumulate, int32_t splits, int32_t tile, float* ws, int64_t ws_bytes, void* stream);
/* Data gradient: dsrc[:, c0:c0+cin] (+)= sum over segments of the transposed conv of src_s[:, cout0_s:cout0_s+cout_s] (each
 * segment's src is the gradient of an output the source fed); every segment has cin = the slice width; dsrc is [N, C, H, W]. */
int csnet_train_conv_dgrad(float* dsrc, int32_t N, int32_t C, int32_t H, int32_t W, int32_t c0, int32_t cin, const csnet_conv_seg* segs,
                           int32_t n_segs, int32_t accumulate, int32_t splits, int32_t tile, float* ws, int64_t ws_bytes, void* stream);
/* Weight gradient of one segment: dw[co * ldw + ci * k * k + t] (+)= sum over images and pixels of ddst[n, cout0 + co] times the
 * input tap t of src[n, c0 + ci]; ddst is fp32 [N, Cd, H, W]. */
int csnet_train_conv_wgrad(const float* ddst, int32_t N, int32_t Cd, int32_t H, int32_t W, const csnet_conv_seg* seg, float* dw,
                           int32_t accumulate, int32_t splits, int32_t tile, float* ws, int64_t ws_bytes, void* stream);
/* Bias gradient: db[c] = sum over images and pixels of ddst[n, c0 + c], images in order. */
int csnet_train_bias_grad(const float* ddst, int32_t N, int32_t C, int32_t HW, int32_t c0, int32_t cout, float* db, void* stream);
/* F.group_norm(z, groups, eps) statistics per (image, group) over (C / groups) * HW values: mean and biased variance [N * groups]. */
int csnet_train_gn_stats(const float* z, int32_t N, int32_t C, int32_t HW, int32_t groups, float* mean, float* var, void* stream);
/* y = PReLU(gamma[c] * (z - mean) * rsqrt(var + eps) + beta[c], slope[c]) with the (image, group) statistics above. */
int csnet_train_gn_prelu_fwd(const float* z, float* y, int32_t N, int32_t C, int32_t HW, int32_t groups, const float* mean,
                             const float* var, const float* gamma, const float* beta, const float* slope, float eps, void* stream);
/* Autograd of the above (statistics depend on z): dz, and dgamma / dbeta / dslope [C] summed over images in order.  ws: 3 N C floats. */
int csnet_train_gn_prelu_bwd(const float* z, const float* dy, float* dz, int32_t N, int32_t C, int32_t HW, int32_t groups,
                             const float* mean, const float* var, const float* gamma, const float* beta, const float* slope, float eps,
                             float* dgamma, float* dbeta, float* dslope, float* ws, void* stream);
/* dst (+)= F.interpolate(src, size=(Hd, Wd), mode='bilinear', align_corners=False), fp32 [N, C, Hs, Ws] -> [N, C, Hd, Wd]: the
 * CSNET_OP_RESIZE kernel.  _bwd is its exact adjoint: dsrc = the transposed tap matrix applied to ddst, gathered per source pixel. */
int csnet_train_resize_fwd(const float* src, int32_t N, int32_t C, int32_t Hs, int32_t Ws, float* dst, int32_t Hd, int32_t Wd,
                           int32_t accumulate, void* stream);
int csnet_train_resize_bwd(const float* ddst, int32_t N, int32_t C, int32_t Hd, int32_t Wd, float* dsrc, int32_t Hs, int32_t Ws,
                           void* stream);

/* ---- CSF+Res2Net head training with bf16 activation storage (sod100k_b200/modular_r.py picks these when net.train_storage is
 * "bf16") ----------------------------------------------------------------------------------------------------------------------
 * The calls above on bf16 planar NCHW activations and activation gradients (pointers are void*).  Convolutions run on a tensor-core
 * implicit GEMM (csrc/gemm_bf16.cuh: mma.sync bf16 x bf16 -> fp32, 128 x 128 x 32 block tiles): operands bf16, accumulation fp32,
 * the weights the fp32 parameters rounded to nearest-even bf16 (csnet_train_cast_bf16).  Forward and data-gradient destinations are
 * bf16 or fp32 (dst_dtype / dsrc_dtype: CSNET_BF16 or CSNET_F32); weight gradients, bias, GroupNorm statistics, gamma / beta / slope and
 * their gradients stay fp32.  Every bf16 store is rounded once to nearest even; split-K partials are merged in split order and
 * reductions keep the fp32 calls' order (no floating-point atomics: the same bits on every run).  Segments, splits and workspace
 * are as for csnet_train_conv_*; there is one block tile, so no tile argument. */
typedef struct {
  const void* src;        /* bf16 [N, C, H, W]: fwd / wgrad the conv's input, dgrad the gradient of the conv's output tensor */
  const void* w;          /* bf16 weight slice (unused by wgrad, which writes the fp32 gradient at the same layout) */
  int32_t C, c0, cin;
  int32_t cout0, cout;
  int32_t ksize, dil, ldw;
} csnet_conv_seg_bf16;    /* 48 bytes, csnet_conv_seg's layout */

/* dst[i] = bf16 nearest-even rounding of src[i], i < n (the weights of a step, rounded once) */
int csnet_train_cast_bf16(const float* src, void* dst, int64_t n, void* stream);
/* splits, the k extent of one split (chain) and the workspace bytes of a conv call, arguments as the call's */
int csnet_train_conv_plan_bf16(int32_t form, int32_t N, int32_t H, int32_t W, const csnet_conv_seg_bf16* segs, int32_t n_segs,
                               int32_t splits, int32_t* splits_out, int32_t* chain_out, int64_t* ws_bytes);
int csnet_train_conv_fwd_bf16(void* dst, int32_t dst_dtype, int32_t N, int32_t C, int32_t H, int32_t W, const csnet_conv_seg_bf16* segs,
                              int32_t n_segs, const float* bias, int32_t accumulate, int32_t splits, float* ws, int64_t ws_bytes,
                              void* stream);
int csnet_train_conv_dgrad_bf16(void* dsrc, int32_t dsrc_dtype, int32_t N, int32_t C, int32_t H, int32_t W, int32_t c0, int32_t cin,
                                const csnet_conv_seg_bf16* segs, int32_t n_segs, int32_t accumulate, int32_t splits, float* ws,
                                int64_t ws_bytes, void* stream);
/* ddst bf16; dw fp32 */
int csnet_train_conv_wgrad_bf16(const void* ddst, int32_t N, int32_t Cd, int32_t H, int32_t W, const csnet_conv_seg_bf16* seg, float* dw,
                                int32_t accumulate, int32_t splits, float* ws, int64_t ws_bytes, void* stream);
/* z, y, dy, dz bf16; mean / var / ws and the parameter gradients fp32 */
int csnet_train_gn_stats_bf16(const void* z, int32_t N, int32_t C, int32_t HW, int32_t groups, float* mean, float* var, void* stream);
int csnet_train_gn_prelu_fwd_bf16(const void* z, void* y, int32_t N, int32_t C, int32_t HW, int32_t groups, const float* mean,
                                  const float* var, const float* gamma, const float* beta, const float* slope, float eps, void* stream);
int csnet_train_gn_prelu_bwd_bf16(const void* z, const void* dy, void* dz, int32_t N, int32_t C, int32_t HW, int32_t groups,
                                  const float* mean, const float* var, const float* gamma, const float* beta, const float* slope, float eps,
                                  float* dgamma, float* dbeta, float* dslope, float* ws, void* stream);
/* bf16 on both sides; the adjoint sums in fp32 over the same taps as csnet_train_resize_bwd */
int csnet_train_resize_fwd_bf16(const void* src, int32_t N, int32_t C, int32_t Hs, int32_t Ws, void* dst, int32_t Hd, int32_t Wd,
                                int32_t accumulate, void* stream);
int csnet_train_resize_bwd_bf16(const void* ddst, int32_t N, int32_t C, int32_t Hd, int32_t Wd, void* dsrc, int32_t Hs, int32_t Ws,
                                void* stream);

/* ---- evaluation: the counting part of SalMetric on the device (CSNet_training/SalMetric/src/sal_metric.cpp:86-120) ----
 * prob: device float32 [N][HW] saliency in [0,1] (after sigmoid); gt: device uint8 [N][HW] ground truth.  Per image:
 * q = (uint8)(prob * 255) (CSNet/test.py:94-96), hist_all[q]++, hist_pos[q]++ where gt > 128, abs_sum += |q - gt|.
 * hist_all / hist_pos: device uint32 [N][256], abs_sum: device uint64 [N]; all three are zeroed by the call.  The caller
 * turns them into precision / recall per threshold (suffix sums), F-measure and MAE (sod100k_b200/salmetric.py). */
int csnet_salmetric_hist(const float* prob, const uint8_t* gt, int32_t N, int64_t HW, uint32_t* hist_all, uint32_t* hist_pos,
                         unsigned long long* abs_sum, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* CSNET_B200_H */
