// train_bf16.cu — bf16 activation storage for the CSNet training step, C ABI `csnet_train_*_bf16`.
//
// The same kernels as the fp32 step (train_body.cuh's bodies, so the same reduction orders), instantiated with bf16 activations:
// conv outputs, BN + PReLU outputs, depthwise outputs, pooled copies and all their gradients are read and written as bf16 by the
// kernels themselves.  Weights, weight gradients, BatchNorm statistics, the per-image channel means and every accumulator stay fp32;
// every store to bf16 rounds to nearest even.  Two boundaries of the network mix types: the stem reads the fp32 input (and its
// weight gradient reads fp32 sources against a bf16 gradient), and cls_layer writes fp32 logits (its data gradient reads an fp32
// gradient).  The mix entry points therefore take the element type of each side.
//
// There is no generic fallback here: a shape the register-tiled kernels do not take returns CSNET_E_UNSUPPORTED.
#include <cuda_runtime.h>

#include <string>

#include "../../include/csnet_b200.h"
#include "train_body.cuh"
#include "train_host.h"

namespace csnet {
namespace bf {

using tf::bf16;
using tf::kT;

template <int KS, class TI, class TO>
__global__ void __launch_bounds__(kT, 2) conv_fwd_bf16_kernel(const __grid_constant__ tf::ConvArgs A) {
  extern __shared__ __align__(16) float smem[];
  tf::conv_fwd_body<KS, TI, TO>(A, smem);
}

// the scalar-load form (odd widths) keeps 3 channels of loads in flight: 4 or more spill past 128 registers
template <int PX, bool VEC, class TI, class TO>
__global__ void __launch_bounds__(kT, 2) conv1x1_bf16_kernel(const __grid_constant__ tf::C1Args A) {
  extern __shared__ __align__(16) float wsm[];
  tf::conv1x1_body<PX, VEC, TI, TO, VEC ? 6 : 3>(A, wsm);
}

// 6 channels of bf16 loads in flight (8 spill past the 80 registers of three CTAs per SM); 8 of fp32 loads, as the fp32 kernel
template <class TI, class TO>
__global__ void __launch_bounds__(kT, 3) conv1x1_narrow_bf16_kernel(const __grid_constant__ tf::C1Args A) {
  extern __shared__ __align__(16) float wsm[];
  tf::conv1x1_narrow_body<TI, TO, sizeof(TI) == 2 ? 6 : 8>(A, wsm);
}

template <int KS, class TI, class TD>
__global__ void __launch_bounds__(kT, 2) conv_wgrad_bf16_kernel(const __grid_constant__ tf::WgradArgs A) {
  extern __shared__ __align__(16) float smem[];
  tf::conv_wgrad_body<KS, TI, TD>(A, smem);
}

__global__ void __launch_bounds__(kT) pool_fwd_bf16_kernel(const bf16* __restrict__ src, int N, int Cs, int c0, int cin, int Hs, int Ws, int pre_avg,
                                                           int pool, bf16* __restrict__ dst, uint8_t* __restrict__ idx) {
  tf::pool_fwd_body(src, N, Cs, c0, cin, Hs, Ws, pre_avg, pool, dst, idx);
}

__global__ void __launch_bounds__(kT) pool2_fwd_bf16_kernel(const bf16* __restrict__ src, int N, int Cs, int c0, int cin, int Hs, int Ws,
                                                            bf16* __restrict__ dst, uint8_t* __restrict__ idx) {
  tf::pool2_fwd_body(src, N, Cs, c0, cin, Hs, Ws, dst, idx);
}

__global__ void __launch_bounds__(kT) pool_bwd_bf16_kernel(const bf16* __restrict__ dpool, const uint8_t* __restrict__ idx, int N, int cin, int Hs,
                                                           int Ws, int pre_avg, int pool, bf16* __restrict__ dsrc) {
  tf::pool_bwd_body(dpool, idx, N, cin, Hs, Ws, pre_avg, pool, dsrc);
}

__global__ void __launch_bounds__(kT) pool_bwd4_bf16_kernel(const bf16* __restrict__ dpool, const uint8_t* __restrict__ idx, int N, int cin, int Hs,
                                                            int Ws, int pre_avg, int pool, bf16* __restrict__ dsrc) {
  tf::pool_bwd4_body(dpool, idx, N, cin, Hs, Ws, pre_avg, pool, dsrc);
}

template <int UP>
__global__ void __launch_bounds__(kT) resample_bwd_bf16_kernel(const bf16* __restrict__ ddst, int N, int C, int H, int W, int cout0, int cin, int Hs,
                                                               int Ws, bf16* __restrict__ dsrc) {
  tf::resample_bwd_body<UP>(ddst, N, C, H, W, cout0, cin, Hs, Ws, dsrc);
}

__global__ void __launch_bounds__(kT) dw3_bf16_kernel(const bf16* __restrict__ x, const float* __restrict__ w, bf16* __restrict__ y, int N, int C,
                                                      int H, int W, float scale, int flip, int quads, int rows) {
  tf::dw3_body(x, w, y, N, C, H, W, scale, flip, quads, rows);
}

__global__ void __launch_bounds__(kT) dw3_wgrad_bf16_kernel(const bf16* __restrict__ x, const bf16* __restrict__ dy, float* __restrict__ part, int N,
                                                            int C, int H, int W, int quads, int rows) {
  tf::dw3_wgrad_body(x, dy, part, N, C, H, W, quads, rows);
}

__global__ void __launch_bounds__(kT) dw3_bwd_bf16_kernel(const bf16* __restrict__ x, const bf16* __restrict__ dy, const float* __restrict__ w,
                                                          bf16* __restrict__ dx, float* __restrict__ part, int N, int C, int H, int W, float scale,
                                                          int quads, int rows) {
  tf::dw3_bwd_body(x, dy, w, dx, part, N, C, H, W, scale, quads, rows);
}

__global__ void __launch_bounds__(kT) bn_stats_bf16_kernel(const bf16* __restrict__ z, int N, int C, int HW, int S, float* mean, float* var,
                                                           float* ws, unsigned* cnt) {
  tf::bn_stats_body(z, N, C, HW, S, mean, var, ws, cnt);
}

__global__ void __launch_bounds__(kT) bn_prelu_fwd_bf16_kernel(const bf16* __restrict__ z, bf16* __restrict__ y, int C, int HW, const float* mean,
                                                               const float* var, const float* gamma, const float* beta, const float* slope,
                                                               float eps, float* gap) {
  tf::bn_prelu_fwd_body(z, y, C, HW, mean, var, gamma, beta, slope, eps, gap);
}

__global__ void __launch_bounds__(kT) bn_prelu_bwd_reduce_bf16_kernel(const bf16* __restrict__ z, const bf16* __restrict__ dy, int N, int C, int HW,
                                                                      int S, const float* mean, const float* var, const float* gamma,
                                                                      const float* beta, const float* slope, float eps, float* dgamma,
                                                                      float* dbeta, float* dslope, float* ws, unsigned* cnt) {
  tf::bn_prelu_bwd_reduce_body(z, dy, N, C, HW, S, mean, var, gamma, beta, slope, eps, dgamma, dbeta, dslope, ws, cnt);
}

__global__ void __launch_bounds__(kT) bn_prelu_bwd_apply_bf16_kernel(const bf16* __restrict__ z, const bf16* __restrict__ dy, bf16* __restrict__ dz,
                                                                     int N, int C, int HW, const float* mean, const float* var,
                                                                     const float* gamma, const float* beta, const float* slope, float eps,
                                                                     const float* dgamma, const float* dbeta, int frozen) {
  tf::bn_prelu_bwd_apply_body(z, dy, dz, N, C, HW, mean, var, gamma, beta, slope, eps, dgamma, dbeta, frozen);
}

// ---- host ------------------------------------------------------------------------------------------------------------------------
using namespace csnet::tr;

int fail(int code, const std::string& msg) {
  train_set_error(msg.c_str());
  return code;
}

#define BF_CHECK(expr)                                                                              \
  do {                                                                                              \
    cudaError_t e_ = (expr);                                                                        \
    if (e_ != cudaSuccess) return fail(CSNET_E_CUDA, std::string(#expr) + ": " + cudaGetErrorString(e_)); \
  } while (0)

// The element types of a call's two sides: both bf16, or one side fp32 (the stem's input, cls_layer's logits and their gradients).
enum Io { kBB, kFB, kBF, kBad };
Io io_of(int32_t in, int32_t out) {
  if (in == CSNET_BF16 && out == CSNET_BF16) return kBB;
  if (in == CSNET_F32 && out == CSNET_BF16) return kFB;
  if (in == CSNET_BF16 && out == CSNET_F32) return kBF;
  return kBad;
}
int esize(int32_t dtype) { return dtype == CSNET_F32 ? 4 : 2; }

template <class TI, class TO>
int launch_conv1x1(const tf::ConvArgs& F, cudaStream_t st, const char* who) {
  tf::C1Args A{};
  const int px = (F.W % 4 != 0 && F.W % 2 == 0) ? 2 : 4;
  A.dst = F.dst; A.N = F.N; A.C = F.C; A.H = F.H; A.W = F.W; A.quads = (F.W + px - 1) / px; A.vec = (F.W % px) == 0; A.transposed = F.transposed;
  A.n_conv = F.n_conv; A.n_rs = F.n_rs; A.Cpad = (F.C + 31) / 32 * 32;
  int rows = 0;
  for (int i = 0; i < F.n_conv; ++i) {
    const tf::ConvPath& P = F.p[i];
    tf::C1Path& Q = A.p[i];
    Q.src = P.src; Q.w = P.w; Q.Cs = P.Cs; Q.c0 = P.c0; Q.cin = P.cin; Q.cout0 = P.cout0; Q.cout = P.cout; Q.woff = rows;
    rows += P.cin;
  }
  for (int i = 0; i < F.n_rs; ++i) A.rs[i] = F.rs[i];
  A.wrows = rows;
  const size_t smem = (size_t)rows * A.Cpad * sizeof(float);
  if (smem > 96 * 1024) return fail(CSNET_E_UNSUPPORTED, std::string(who) + ": the 1x1 weights exceed 96 KiB of shared memory");
  static bool attr_dev[kMaxDevices] = {false};
  bool& attr = attr_dev[current_device()];
  if (!attr) {
    cudaFuncSetAttribute(conv1x1_bf16_kernel<2, true, TI, TO>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
    cudaFuncSetAttribute(conv1x1_bf16_kernel<4, true, TI, TO>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
    cudaFuncSetAttribute(conv1x1_bf16_kernel<4, false, TI, TO>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
    cudaFuncSetAttribute(conv1x1_narrow_bf16_kernel<TI, TO>, cudaFuncAttributeMaxDynamicSharedMemorySize, 72 * 1024);
    attr = true;
  }
  const size_t tasks = (size_t)A.N * A.H * A.quads;
  const unsigned blocks = (unsigned)((tasks + kT - 1) / kT);
  const bool narrow = A.C <= 24;                             // the fp32 dispatch's choice, for the same reasons
  if (narrow && px == 4 && A.vec && smem <= 72 * 1024) conv1x1_narrow_bf16_kernel<TI, TO><<<blocks, kT, smem, st>>>(A);
  else if (px == 2) conv1x1_bf16_kernel<2, true, TI, TO><<<blocks, kT, smem, st>>>(A);
  else if (A.vec) conv1x1_bf16_kernel<4, true, TI, TO><<<blocks, kT, smem, st>>>(A);
  else conv1x1_bf16_kernel<4, false, TI, TO><<<blocks, kT, smem, st>>>(A);
  BF_CHECK(cudaGetLastError());
  return CSNET_OK;
}

template <class TI, class TO>
int launch_conv(tf::ConvArgs& A, cudaStream_t st, const char* who) {
  if (A.n_conv == 0 || A.ksize == 1) return launch_conv1x1<TI, TO>(A, st, who);
  const int kk = A.ksize * A.ksize;
  size_t tile = 0, wsm = 0;
  bool dil1 = true;
  for (int i = 0; i < A.n_conv; ++i) {
    const tf::ConvPath& P = A.p[i];
    const size_t t = (size_t)P.chunk * A.ipb * P.rows * P.Wp, w = (size_t)P.chunk * kk * tf::kCoT;
    tile = t > tile ? t : tile; wsm = w > wsm ? w : wsm;
    dil1 = dil1 && P.dil == 1;
  }
  A.tile_floats = (int)((tile * sizeof(TI) + 15) / 16 * 4);   // the weights start 16-byte aligned after the tile
  const size_t smem = A.tile_floats * sizeof(float) + wsm * sizeof(float);
  const int bands = (A.H + A.R - 1) / A.R;
  const unsigned grid = (unsigned)(((A.N + A.ipb - 1) / A.ipb) * bands);
  static bool attr_dev[kMaxDevices] = {false};
  bool& attr = attr_dev[current_device()];
  if (!attr) {
    cudaFuncSetAttribute(conv_fwd_bf16_kernel<0, TI, TO>, cudaFuncAttributeMaxDynamicSharedMemorySize, kFastSmemMax);
    cudaFuncSetAttribute(conv_fwd_bf16_kernel<3, TI, TO>, cudaFuncAttributeMaxDynamicSharedMemorySize, kFastSmemMax);
    attr = true;
  }
  if (A.ksize == 3 && dil1) conv_fwd_bf16_kernel<3, TI, TO><<<grid, kT, smem, st>>>(A);
  else conv_fwd_bf16_kernel<0, TI, TO><<<grid, kT, smem, st>>>(A);
  BF_CHECK(cudaGetLastError());
  return CSNET_OK;
}

// An fp32 destination (cls_layer's logits) is taken for 1x1 mixes only.
int launch_conv_io(Io io, tf::ConvArgs& A, cudaStream_t st, const char* who) {
  if (io == kBB) return launch_conv<bf16, bf16>(A, st, who);
  if (io == kFB) return launch_conv<float, bf16>(A, st, who);
  if (A.n_conv > 0 && A.ksize != 1) return fail(CSNET_E_UNSUPPORTED, std::string(who) + ": an fp32 destination takes 1x1 mixes only");
  return launch_conv1x1<bf16, float>(A, st, who);
}

template <class TI, class TD>
int launch_wgrad(const WgradPlan& G, cudaStream_t st) {
  static bool attr_dev[kMaxDevices] = {false};
  bool& attr = attr_dev[current_device()];
  if (!attr) {
    cudaFuncSetAttribute(conv_wgrad_bf16_kernel<0, TI, TD>, cudaFuncAttributeMaxDynamicSharedMemorySize, kFastSmemMax);
    cudaFuncSetAttribute(conv_wgrad_bf16_kernel<1, TI, TD>, cudaFuncAttributeMaxDynamicSharedMemorySize, kFastSmemMax);
    cudaFuncSetAttribute(conv_wgrad_bf16_kernel<3, TI, TD>, cudaFuncAttributeMaxDynamicSharedMemorySize, kFastSmemMax);
    attr = true;
  }
  const dim3 grid(G.gx, G.groups);
  if (G.form == 1) conv_wgrad_bf16_kernel<1, TI, TD><<<grid, kT, G.smem, st>>>(G.A);
  else if (G.form == 3) conv_wgrad_bf16_kernel<3, TI, TD><<<grid, kT, G.smem, st>>>(G.A);
  else conv_wgrad_bf16_kernel<0, TI, TD><<<grid, kT, G.smem, st>>>(G.A);
  BF_CHECK(cudaGetLastError());
  return CSNET_OK;
}

// depthwise launch geometry (as the fp32 entry points): 4-pixel strips of up to 8 rows; backward grids capped per channel
struct DwGeom { int quads, rows, bands; };
DwGeom dw_geom(int H, int W) { const int q = (W + 3) / 4, r = H < 8 ? H : 8; return {q, r, (H + r - 1) / r}; }
int dw_blocks(int N, const DwGeom& g, int C, int per_sm) {
  const size_t tasks = (size_t)N * g.bands * g.quads;
  int bx = (int)((tasks + kT - 1) / kT), cap = per_sm * num_sms() / C;
  cap = cap < 1 ? 1 : cap;
  return bx > cap ? cap : bx;
}

}  // namespace bf
}  // namespace csnet

using namespace csnet::bf;
using csnet::tf::bf16;

extern "C" {

int csnet_train_bn_stats_bf16(const void* z, int32_t N, int32_t C, int32_t HW, float* mean, float* var, void* stream) {
  if (!z || !mean || !var || N < 1 || C < 1 || HW < 1) return fail(CSNET_E_INVALID, "csnet_train_bn_stats_bf16: bad arguments");
  const int S = reduce_segments(N, C, HW);
  float* ws = nullptr;
  unsigned* cnt = nullptr;
  if (int rc = reduce_workspace(C, N * S, (cudaStream_t)stream, &ws, &cnt)) return rc;
  bn_stats_bf16_kernel<<<dim3(C, N * S), kT, 0, (cudaStream_t)stream>>>(static_cast<const bf16*>(z), N, C, HW, S, mean, var, ws, cnt);
  BF_CHECK(cudaGetLastError());
  return CSNET_OK;
}

int csnet_train_bn_prelu_fwd_bf16(const void* z, void* y, int32_t N, int32_t C, int32_t HW, const float* mean, const float* var, const float* gamma,
                                  const float* beta, const float* slope, float eps, float* gap, void* stream) {
  if (!z || !y || N < 1 || C < 1 || HW < 1) return fail(CSNET_E_INVALID, "csnet_train_bn_prelu_fwd_bf16: bad arguments");
  bn_prelu_fwd_bf16_kernel<<<dim3(C, N), kT, 0, (cudaStream_t)stream>>>(static_cast<const bf16*>(z), static_cast<bf16*>(y), C, HW, mean, var, gamma,
                                                                        beta, slope, eps, gap);
  BF_CHECK(cudaGetLastError());
  return CSNET_OK;
}

int csnet_train_bn_prelu_bwd_bf16(const void* z, const void* dy, void* dz, int32_t N, int32_t C, int32_t HW, const float* mean, const float* var,
                                  const float* gamma, const float* beta, const float* slope, float eps, float* dgamma, float* dbeta, float* dslope,
                                  int32_t frozen, void* stream) {
  if (!z || !dy || !dz || N < 1 || C < 1 || HW < 1) return fail(CSNET_E_INVALID, "csnet_train_bn_prelu_bwd_bf16: bad arguments");
  const int S = reduce_segments(N, C, HW);
  float* ws = nullptr;
  unsigned* cnt = nullptr;
  if (int rc = reduce_workspace(C, N * S, (cudaStream_t)stream, &ws, &cnt)) return rc;
  const bf16* zb = static_cast<const bf16*>(z);
  const bf16* dyb = static_cast<const bf16*>(dy);
  bn_prelu_bwd_reduce_bf16_kernel<<<dim3(C, N * S), kT, 0, (cudaStream_t)stream>>>(zb, dyb, N, C, HW, S, mean, var, gamma, beta, slope, eps, dgamma,
                                                                                  dbeta, dslope, ws, cnt);
  BF_CHECK(cudaGetLastError());
  bn_prelu_bwd_apply_bf16_kernel<<<dim3(C, N), kT, 0, (cudaStream_t)stream>>>(zb, dyb, static_cast<bf16*>(dz), N, C, HW, mean, var, gamma, beta,
                                                                              slope, eps, dgamma, dbeta, frozen);
  BF_CHECK(cudaGetLastError());
  return CSNET_OK;
}

int csnet_train_dw_conv_bf16(const void* x, const float* w, void* y, int32_t N, int32_t C, int32_t H, int32_t W, float scale, int32_t transposed,
                             void* stream) {
  if (!x || !w || !y || N < 1 || C < 1 || H < 1 || W < 1) return fail(CSNET_E_INVALID, "csnet_train_dw_conv_bf16: bad arguments");
  const DwGeom g = dw_geom(H, W);
  const size_t tasks = (size_t)N * C * g.bands * g.quads;
  dw3_bf16_kernel<<<(unsigned)((tasks + kT - 1) / kT), kT, 0, (cudaStream_t)stream>>>(static_cast<const bf16*>(x), w, static_cast<bf16*>(y), N, C, H,
                                                                                       W, scale, transposed, g.quads, g.rows);
  BF_CHECK(cudaGetLastError());
  return CSNET_OK;
}

int csnet_train_dw_wgrad_bf16(const void* x, const void* dy, float* dw, int32_t N, int32_t C, int32_t H, int32_t W, float scale, void* stream) {
  if (!x || !dy || !dw || N < 1 || C < 1 || H < 1 || W < 1) return fail(CSNET_E_INVALID, "csnet_train_dw_wgrad_bf16: bad arguments");
  const DwGeom g = dw_geom(H, W);
  const int bx = dw_blocks(N, g, C, 4);
  float* part = nullptr;
  if (int rc = partial_workspace((size_t)bx * C * 9, (cudaStream_t)stream, &part)) return rc;
  dw3_wgrad_bf16_kernel<<<dim3(bx, C), kT, 0, (cudaStream_t)stream>>>(static_cast<const bf16*>(x), static_cast<const bf16*>(dy), part, N, C, H, W,
                                                                      g.quads, g.rows);
  BF_CHECK(cudaGetLastError());
  return reduce_partials(part, bx, C * 9, scale, dw, (cudaStream_t)stream);
}

int csnet_train_dw_bwd_bf16(const void* x, const void* dy, const float* w, void* dx, float* dw, int32_t N, int32_t C, int32_t H, int32_t W,
                            float scale, void* stream) {
  if (!x || !dy || !w || !dx || !dw || N < 1 || C < 1 || H < 1 || W < 1) return fail(CSNET_E_INVALID, "csnet_train_dw_bwd_bf16: bad arguments");
  const DwGeom g = dw_geom(H, W);
  const int bx = dw_blocks(N, g, C, 8);
  float* part = nullptr;
  if (int rc = partial_workspace((size_t)bx * C * 9, (cudaStream_t)stream, &part)) return rc;
  dw3_bwd_bf16_kernel<<<dim3(bx, C), kT, 0, (cudaStream_t)stream>>>(static_cast<const bf16*>(x), static_cast<const bf16*>(dy), w,
                                                                    static_cast<bf16*>(dx), part, N, C, H, W, scale, g.quads, g.rows);
  BF_CHECK(cudaGetLastError());
  return reduce_partials(part, bx, C * 9, scale, dw, (cudaStream_t)stream);
}

int csnet_train_mix_fwd_bf16(void* dst, int32_t dst_dtype, int32_t N, int32_t C, int32_t H, int32_t W, const csnet_train_path* paths, int32_t n_paths,
                             int32_t src_dtype, void* stream) {
  const char* who = "csnet_train_mix_fwd_bf16";
  const Io io = io_of(src_dtype, dst_dtype);
  if (io == kBad) return fail(CSNET_E_INVALID, std::string(who) + ": dtypes must be bf16, or fp32 on one side (the fp32 step has csnet_train_mix_fwd)");
  if (!dst || !paths || n_paths < 1 || n_paths > CSNET_MAX_PATHS) return fail(CSNET_E_INVALID, std::string(who) + ": bad arguments");
  tf::ConvArgs F{};
  F.dst = dst; F.N = N; F.C = C; F.H = H; F.W = W; F.ksize = 1;
  if (!conv_tile_geometry(F)) return fail(CSNET_E_UNSUPPORTED, std::string(who) + ": rows wider than 1024 pixels");
  int ks = 0;
  for (int p = 0; p < n_paths; ++p) {
    const csnet::MixPath P = to_path(paths[p]);
    if (P.ksize == 0) {
      if (F.n_rs >= tf::kMaxRs || P.up < 2 || P.pre_avg || P.pool != 1 || P.H * P.up != H || P.W * P.up != W)
        return fail(CSNET_E_UNSUPPORTED, std::string(who) + ": resample-add path " + std::to_string(p) + " is not a x2^k up-sample of the output plane");
      tf::RsPath& Q = F.rs[F.n_rs++];
      Q.src = P.src; Q.Cs = P.C; Q.c0 = P.c0; Q.Hs = P.H; Q.Ws = P.W; Q.up = P.up; Q.cout0 = P.cout0; Q.cout = P.cout;
    } else {
      if (F.n_conv >= tf::kMaxConv || !dense_conv_path(P, H, W) || (ks && ks != P.ksize))
        return fail(CSNET_E_UNSUPPORTED, std::string(who) + ": conv path " + std::to_string(p) +
                                             " is not dense (stride 1, same plane, pad = dil * (k / 2), no pooling; pool it first) or mixes kernel sizes");
      ks = P.ksize;
      tf::ConvPath& Q = F.p[F.n_conv++];
      Q.src = P.src; Q.w = P.w; Q.Cs = P.C; Q.c0 = P.c0; Q.cin = P.cin; Q.cout0 = P.cout0; Q.cout = P.cout; Q.dil = P.dil;
    }
  }
  F.ksize = ks ? ks : 1;
  for (int i = 0; i < F.n_conv; ++i)
    if (!conv_path_geometry(F.p[i], F, esize(src_dtype))) return fail(CSNET_E_UNSUPPORTED, std::string(who) + ": the input tile does not fit shared memory");
  return launch_conv_io(io, F, (cudaStream_t)stream, who);
}

int csnet_train_mix_dgrad_bf16(const void* ddst, int32_t ddst_dtype, int32_t N, int32_t C, int32_t H, int32_t W, const csnet_train_path* path,
                               void* dsrc, int32_t dsrc_dtype, void* stream) {
  const char* who = "csnet_train_mix_dgrad_bf16";
  const Io io = io_of(ddst_dtype, dsrc_dtype);
  if (io == kBad) return fail(CSNET_E_INVALID, std::string(who) + ": dtypes must be bf16, or fp32 on one side (the fp32 step has csnet_train_mix_dgrad)");
  if (!ddst || !path || !dsrc) return fail(CSNET_E_INVALID, std::string(who) + ": bad arguments");
  const csnet::MixPath P = to_path(*path);
  if (P.ksize == 0) {
    if (io != kBB || (P.up != 2 && P.up != 4) || P.pre_avg || P.pool != 1 || P.H * P.up != H || P.W * P.up != W ||
        (size_t)N * P.cin * P.H * P.W >= (1ull << 32))
      return fail(CSNET_E_UNSUPPORTED, std::string(who) + ": resample paths take bf16 on both sides and a x2 / x4 up-sample of the output plane");
    const size_t total = (size_t)N * P.cin * P.H * P.W;
    const unsigned blocks = (unsigned)((total + kT - 1) / kT);
    const bf16* d = static_cast<const bf16*>(ddst);
    bf16* s = static_cast<bf16*>(dsrc);
    if (P.up == 2) resample_bwd_bf16_kernel<2><<<blocks, kT, 0, (cudaStream_t)stream>>>(d, N, C, H, W, P.cout0, P.cin, P.H, P.W, s);
    else resample_bwd_bf16_kernel<4><<<blocks, kT, 0, (cudaStream_t)stream>>>(d, N, C, H, W, P.cout0, P.cin, P.H, P.W, s);
    BF_CHECK(cudaGetLastError());
    return CSNET_OK;
  }
  if (!dense_conv_path(P, H, W))
    return fail(CSNET_E_UNSUPPORTED, std::string(who) + ": the path is not dense (stride 1, same plane, pad = dil * (k / 2), no pooling)");
  tf::ConvArgs F{};
  F.dst = dsrc; F.N = N; F.C = P.cin; F.H = H; F.W = W; F.ksize = P.ksize; F.transposed = 1; F.n_conv = 1;
  tf::ConvPath& Q = F.p[0];
  Q.src = ddst; Q.w = P.w; Q.Cs = C; Q.c0 = P.cout0; Q.cin = P.cout; Q.cout0 = 0; Q.cout = P.cin; Q.dil = P.dil;
  if (!conv_tile_geometry(F) || !conv_path_geometry(Q, F, esize(ddst_dtype)))
    return fail(CSNET_E_UNSUPPORTED, std::string(who) + ": the plane does not fit the tiled kernel");
  return launch_conv_io(io, F, (cudaStream_t)stream, who);
}

int csnet_train_mix_wgrad_bf16(const void* ddst, int32_t ddst_dtype, int32_t N, int32_t C, int32_t H, int32_t W, const csnet_train_path* path, float* dw,
                               int32_t src_dtype, void* stream) {
  const char* who = "csnet_train_mix_wgrad_bf16";
  const Io io = io_of(src_dtype, ddst_dtype);
  if (io == kBad) return fail(CSNET_E_INVALID, std::string(who) + ": dtypes must be bf16, or fp32 on one side (the fp32 step has csnet_train_mix_wgrad)");
  if (!ddst || !path || !dw) return fail(CSNET_E_INVALID, std::string(who) + ": bad arguments");
  const csnet::MixPath P = to_path(*path);
  if (P.ksize == 0) return fail(CSNET_E_INVALID, std::string(who) + ": resample paths have no weights");
  WgradPlan G;
  if (!wgrad_plan(P, ddst, N, C, H, W, esize(src_dtype), esize(ddst_dtype), G))
    return fail(CSNET_E_UNSUPPORTED, std::string(who) + ": only dense 3x3 paths (any dilation) and 1x1 paths at dilation 1 are taken");
  float* part = nullptr;
  if (int rc = partial_workspace((size_t)G.gx * G.nel, (cudaStream_t)stream, &part)) return rc;
  G.A.part = part;
  int rc;
  if (io == kBB) rc = launch_wgrad<bf16, bf16>(G, (cudaStream_t)stream);
  else if (io == kFB) rc = launch_wgrad<float, bf16>(G, (cudaStream_t)stream);
  else rc = launch_wgrad<bf16, float>(G, (cudaStream_t)stream);
  if (rc) return rc;
  return reduce_partials(part, G.gx, G.nel, 1.f, dw, (cudaStream_t)stream);
}

int csnet_train_pool_fwd_bf16(const void* src, int32_t N, int32_t Cs, int32_t c0, int32_t cin, int32_t Hs, int32_t Ws, int32_t pre_avg, int32_t pool,
                              void* dst, uint8_t* idx, void* stream) {
  if (!src || !dst || pre_avg < 0 || pre_avg > 1 || pool < 1 || pool > 8 || (pool > 1 && !idx)) return fail(CSNET_E_INVALID, "csnet_train_pool_fwd_bf16: bad arguments");
  const int f = (pre_avg ? 2 : 1) * pool;
  const size_t total = (size_t)N * cin * (Hs / f) * (Ws / f);
  if (total == 0) return CSNET_OK;
  const bf16* s = static_cast<const bf16*>(src);
  bf16* d = static_cast<bf16*>(dst);
  if (!pre_avg && pool == 2 && Ws % 4 == 0 && Hs % 2 == 0 && total < (1ull << 31))
    pool2_fwd_bf16_kernel<<<(unsigned)((total / 2 + kT - 1) / kT), kT, 0, (cudaStream_t)stream>>>(s, N, Cs, c0, cin, Hs, Ws, d, idx);
  else
    pool_fwd_bf16_kernel<<<(unsigned)((total + kT - 1) / kT), kT, 0, (cudaStream_t)stream>>>(s, N, Cs, c0, cin, Hs, Ws, pre_avg, pool, d, idx);
  BF_CHECK(cudaGetLastError());
  return CSNET_OK;
}

int csnet_train_pool_bwd_bf16(const void* dpool, const uint8_t* idx, int32_t N, int32_t cin, int32_t Hs, int32_t Ws, int32_t pre_avg, int32_t pool,
                              void* dsrc, void* stream) {
  if (!dpool || !dsrc || pre_avg < 0 || pre_avg > 1 || pool < 1 || pool > 8 || (pool > 1 && !idx)) return fail(CSNET_E_INVALID, "csnet_train_pool_bwd_bf16: bad arguments");
  const size_t total = (size_t)N * cin * Hs * Ws;
  if (total == 0) return CSNET_OK;
  const bf16* d = static_cast<const bf16*>(dpool);
  bf16* s = static_cast<bf16*>(dsrc);
  if (Ws % 4 == 0 && total < (1ull << 32))
    pool_bwd4_bf16_kernel<<<(unsigned)((total / 4 + kT - 1) / kT), kT, 0, (cudaStream_t)stream>>>(d, idx, N, cin, Hs, Ws, pre_avg, pool, s);
  else
    pool_bwd_bf16_kernel<<<(unsigned)((total + kT - 1) / kT), kT, 0, (cudaStream_t)stream>>>(d, idx, N, cin, Hs, Ws, pre_avg, pool, s);
  BF_CHECK(cudaGetLastError());
  return CSNET_OK;
}

}  // extern "C"
