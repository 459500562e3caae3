// train_csf.cu — training kernels of the CSF+Res2Net head (fp32), C ABI csnet_train_conv_* / _bias_grad / _gn_* (include/csnet_b200.h), and the
// bf16-storage twins of the _gn_* calls (the bf16 convolutions are in train_csf_bf16.cu).
//
// The head (fuse, ms, fuse1x1, cls_layer: networks/gOctConv.py, csf_res2net.py) is 1x1 and dilated 3x3 convolutions with K = 128..3840
// and N = 128..1408 channels, GroupNorm(32) + PReLU, and bilinear resizes between the Res2Net stages.  The convolutions run on the fp32
// implicit GEMM of gemm_f32.cuh, GroupNorm on gn_train.cuh; the resize pair sits in plan.cu beside the RESIZE op's launch.
#include <cuda_runtime.h>

#include <cstdint>
#include <string>

#include "../../include/csnet_b200.h"
#include "gemm_f32.cuh"
#include "gn_bf16.cuh"
#include "gn_train.cuh"

namespace csnet {
void train_set_error(const char* msg);     // train_ops.cu: the message csnet_train_last_error returns
}

namespace {

int cfail(int code, const std::string& what) {
  csnet::train_set_error(what.c_str());
  return code;
}

#define CF_CHECK(expr)                                                                           \
  do {                                                                                           \
    cudaError_t e_ = (expr);                                                                     \
    if (e_ != cudaSuccess) return cfail(CSNET_E_CUDA, std::string(#expr) + ": " + cudaGetErrorString(e_)); \
  } while (0)

int num_sms() {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 132;
  }
  return sms;
}

using csnet::g32::Args;
namespace g32 = csnet::g32;

struct Geo {
  int bm, bn, bk;
};
constexpr Geo kSmall{64, 64, 16}, kBig{128, 128, 8};

// What a call does: the tile, the GEMM extents, the k tiles and the split.  Fills everything in `A` but the pointers.
int conv_setup(int form, int N, int H, int W, const csnet_conv_seg* segs, int n_segs, int splits, int tile, Args& A, Geo& geo) {
  if (form < 0 || form > 2 || N < 1 || H < 1 || W < 1 || !segs || n_segs < 1 || n_segs > g32::kMaxSegs)
    return cfail(CSNET_E_INVALID, "conv: bad form, shape or segment count");
  if ((int64_t)H * W > (1 << 30)) return cfail(CSNET_E_INVALID, "conv: plane too large");
  if (form == CSNET_CONV_WGRAD && n_segs != 1) return cfail(CSNET_E_INVALID, "conv wgrad: one segment per call");
  if (splits < 0 || tile < 0 || tile > 2) return cfail(CSNET_E_INVALID, "conv: bad splits / tile");
  const int ks = segs[0].ksize;
  A = Args{};
  A.nseg = n_segs;
  A.N = N; A.H = H; A.W = W; A.HW = H * W;
  for (int s = 0; s < n_segs; ++s) {
    const csnet_conv_seg& q = segs[s];
    if (q.ksize != ks || (ks != 1 && ks != 3) || q.dil < 1 || q.cin < 1 || q.cout < 1 || q.C < 1 || q.ldw < q.cin * ks * ks)
      return cfail(CSNET_E_INVALID, "conv: bad segment (ksize 1 or 3 shared by all, dil >= 1, ldw >= cin k^2)");
    if (form != CSNET_CONV_DGRAD && (q.c0 < 0 || q.c0 + q.cin > q.C)) return cfail(CSNET_E_INVALID, "conv: input slice outside src");
    if (form == CSNET_CONV_DGRAD && (q.cout0 < 0 || q.cout0 + q.cout > q.C)) return cfail(CSNET_E_INVALID, "conv dgrad: gradient slice outside src");
    if (form == CSNET_CONV_WGRAD && q.cout0 < 0) return cfail(CSNET_E_INVALID, "conv wgrad: gradient slice outside ddst");
    if (form == CSNET_CONV_FWD && (q.cout != segs[0].cout || q.cout0 != segs[0].cout0)) return cfail(CSNET_E_INVALID, "conv fwd: segments write one slice");
    if (form == CSNET_CONV_DGRAD && q.cin != segs[0].cin) return cfail(CSNET_E_INVALID, "conv dgrad: segments feed one slice");
    g32::Seg& S = A.seg[s];
    S.src = (const float*)q.src; S.w = q.w;
    S.C = q.C; S.c0 = q.c0; S.cin = q.cin; S.cout0 = q.cout0; S.cout = q.cout; S.dil = q.dil; S.ldw = q.ldw;
    S.K = form == CSNET_CONV_FWD ? q.cin * ks * ks : q.cout * ks * ks;
  }
  if (form == CSNET_CONV_FWD) { A.M = segs[0].cout; A.Ncol = A.HW; }
  else if (form == CSNET_CONV_DGRAD) { A.M = segs[0].cin; A.Ncol = A.HW; }
  else { A.M = segs[0].cout; A.Ncol = segs[0].cin * ks * ks; }
  const bool big = tile == 2 || (tile == 0 && A.M >= 128 && A.Ncol >= 128);
  geo = big ? kBig : kSmall;
  int t = 0;
  if (form == CSNET_CONV_WGRAD) {
    A.kt_img = (A.HW + geo.bk - 1) / geo.bk;
    t = A.kt_img * N;
  } else {
    for (int s = 0; s < n_segs; ++s) { A.seg[s].tile0 = t; t += (A.seg[s].K + geo.bk - 1) / geo.bk; }
  }
  A.ktiles = t;
  const int images = form == CSNET_CONV_WGRAD ? 1 : N;
  const int64_t blocks = (int64_t)((A.M + geo.bm - 1) / geo.bm) * ((A.Ncol + geo.bn - 1) / geo.bn) * images;
  if (splits == 0) {                                            // fill two waves; keep >= 4 k tiles per split
    const int64_t want = blocks >= 2 * num_sms() ? 1 : (2 * num_sms() + blocks - 1) / blocks;
    int64_t cap = t / 4 < 64 ? t / 4 : 64;
    splits = (int)(want < cap ? want : cap);
    if (splits < 1) splits = 1;
  }
  if (splits > t) splits = t > 0 ? t : 1;
  if (blocks * splits > 0x7fffffffLL || (int64_t)images * splits > 65535)
    return cfail(CSNET_E_INVALID, "conv: grid too large");
  A.splits = splits;
  return 0;
}

int64_t ws_need(const Args& A, int form) {
  const int images = form == CSNET_CONV_WGRAD ? 1 : A.N;
  return A.splits > 1 ? (int64_t)A.splits * images * A.M * A.Ncol * 4 : 0;
}

int chain(const Args& A, const Geo& g) { return ((A.ktiles + A.splits - 1) / A.splits) * g.bk; }

template <int BM, int BN, int BK, int TM, int TN, int KS, int FORM>
int launch_t(const Args& A, cudaStream_t st) {
  auto k = g32::gemm_f32_kernel<BM, BN, BK, TM, TN, KS, FORM>;
  const int smem = g32::Tile<BM, BN, BK, TM, TN>::kSmemFloats * 4;
  const int images = FORM == g32::kWgrad ? 1 : A.N;
  const dim3 grid((unsigned)((A.Ncol + BN - 1) / BN), (unsigned)((A.M + BM - 1) / BM), (unsigned)(images * A.splits));
  k<<<grid, g32::kThreads, smem, st>>>(A);
  CF_CHECK(cudaGetLastError());
  if (A.splits > 1) {
    const int64_t total = (int64_t)images * A.M * A.Ncol;
    int64_t blocks = (total + g32::kThreads - 1) / g32::kThreads;
    if (blocks > 8 * num_sms()) blocks = 8 * num_sms();
    g32::gemm_merge_kernel<FORM><<<(unsigned)blocks, g32::kThreads, 0, st>>>(A, images);
    CF_CHECK(cudaGetLastError());
  }
  return 0;
}

template <int FORM>
int launch_form(const Args& A, const Geo& g, int ks, cudaStream_t st) {
  const bool big = g.bm == 128;
  if (ks == 1) return big ? launch_t<128, 128, 8, 8, 8, 1, FORM>(A, st) : launch_t<64, 64, 16, 4, 4, 1, FORM>(A, st);
  return big ? launch_t<128, 128, 8, 8, 8, 3, FORM>(A, st) : launch_t<64, 64, 16, 4, 4, 3, FORM>(A, st);
}

int conv_run(int form, Args& A, const Geo& g, int ks, float* ws, int64_t ws_bytes, void* stream) {
  const int64_t need = ws_need(A, form);
  if (need > 0 && (!ws || ws_bytes < need)) return cfail(CSNET_E_INVALID, "conv: workspace too small for the split (csnet_train_conv_plan)");
  A.ws = ws;
  cudaStream_t st = (cudaStream_t)stream;
  if (form == CSNET_CONV_FWD) return launch_form<g32::kFwd>(A, g, ks, st);
  if (form == CSNET_CONV_DGRAD) return launch_form<g32::kDgrad>(A, g, ks, st);
  return launch_form<g32::kWgrad>(A, g, ks, st);
}

__global__ void __launch_bounds__(256) bias_grad_kernel(const float* __restrict__ dy, int N, int C, int HW, int c0, float* db) {
  __shared__ float sh[8];
  const int c = blockIdx.x;
  float s = 0.f;
  for (int n = 0; n < N; ++n) {
    const float* p = dy + ((int64_t)n * C + c0 + c) * HW;
    float t = 0.f;
    for (int i = threadIdx.x; i < HW; i += 256) t += p[i];
    s += csnet::gn::block_sum_f<256>(t, sh);                   // image sums added in image order (thread 0)
  }
  if (threadIdx.x == 0) db[c] = s;
}

}  // namespace

extern "C" {

int csnet_train_conv_plan(int32_t form, int32_t N, int32_t H, int32_t W, const csnet_conv_seg* segs, int32_t n_segs, int32_t splits,
                          int32_t tile, int32_t* splits_out, int32_t* chain_out, int64_t* ws_bytes) {
  Args A;
  Geo g;
  if (int rc = conv_setup(form, N, H, W, segs, n_segs, splits, tile, A, g)) return rc;
  if (splits_out) *splits_out = A.splits;
  if (chain_out) *chain_out = chain(A, g);
  if (ws_bytes) *ws_bytes = ws_need(A, form);
  return 0;
}

int csnet_train_conv_fwd(float* dst, int32_t N, int32_t C, int32_t H, int32_t W, const csnet_conv_seg* segs, int32_t n_segs,
                         const float* bias, int32_t accumulate, int32_t splits, int32_t tile, float* ws, int64_t ws_bytes, void* stream) {
  Args A;
  Geo g;
  if (int rc = conv_setup(CSNET_CONV_FWD, N, H, W, segs, n_segs, splits, tile, A, g)) return rc;
  if (!dst || segs[0].cout0 < 0 || segs[0].cout0 + segs[0].cout > C) return cfail(CSNET_E_INVALID, "conv fwd: output slice outside dst");
  A.dst = dst; A.Cd = C; A.d0 = segs[0].cout0; A.bias = bias; A.accumulate = accumulate != 0;
  return conv_run(CSNET_CONV_FWD, A, g, segs[0].ksize, ws, ws_bytes, stream);
}

int csnet_train_conv_dgrad(float* dsrc, int32_t N, int32_t C, int32_t H, int32_t W, int32_t c0, int32_t cin, const csnet_conv_seg* segs,
                           int32_t n_segs, int32_t accumulate, int32_t splits, int32_t tile, float* ws, int64_t ws_bytes, void* stream) {
  Args A;
  Geo g;
  if (int rc = conv_setup(CSNET_CONV_DGRAD, N, H, W, segs, n_segs, splits, tile, A, g)) return rc;
  if (!dsrc || c0 < 0 || cin != segs[0].cin || c0 + cin > C) return cfail(CSNET_E_INVALID, "conv dgrad: gradient slice outside dsrc");
  A.dst = dsrc; A.Cd = C; A.d0 = c0; A.accumulate = accumulate != 0;
  return conv_run(CSNET_CONV_DGRAD, A, g, segs[0].ksize, ws, ws_bytes, stream);
}

int csnet_train_conv_wgrad(const float* ddst, int32_t N, int32_t Cd, int32_t H, int32_t W, const csnet_conv_seg* seg, float* dw,
                           int32_t accumulate, int32_t splits, int32_t tile, float* ws, int64_t ws_bytes, void* stream) {
  Args A;
  Geo g;
  if (int rc = conv_setup(CSNET_CONV_WGRAD, N, H, W, seg, 1, splits, tile, A, g)) return rc;
  if (!ddst || !dw || seg->cout0 + seg->cout > Cd) return cfail(CSNET_E_INVALID, "conv wgrad: gradient slice outside ddst");
  A.dy = ddst; A.Cy = Cd; A.y0 = seg->cout0; A.dst = dw; A.ldd = seg->ldw; A.accumulate = accumulate != 0;
  return conv_run(CSNET_CONV_WGRAD, A, g, seg->ksize, ws, ws_bytes, stream);
}

int csnet_train_bias_grad(const float* ddst, int32_t N, int32_t C, int32_t HW, int32_t c0, int32_t cout, float* db, void* stream) {
  if (!ddst || !db || N < 1 || HW < 1 || cout < 1 || c0 < 0 || c0 + cout > C) return cfail(CSNET_E_INVALID, "bias_grad: bad arguments");
  bias_grad_kernel<<<cout, 256, 0, (cudaStream_t)stream>>>(ddst, N, C, HW, c0, db);
  CF_CHECK(cudaGetLastError());
  return 0;
}

static int gn_args_ok(int N, int C, int HW, int groups) { return N >= 1 && HW >= 1 && groups >= 1 && C >= groups && C % groups == 0 && N <= 65535; }

int csnet_train_gn_stats(const float* z, int32_t N, int32_t C, int32_t HW, int32_t groups, float* mean, float* var, void* stream) {
  if (!z || !mean || !var || !gn_args_ok(N, C, HW, groups)) return cfail(CSNET_E_INVALID, "gn_stats: bad arguments");
  csnet::gn::gn_stats_kernel<<<N * groups, csnet::gn::kStatThreads, 0, (cudaStream_t)stream>>>(z, C, HW, groups, mean, var);
  CF_CHECK(cudaGetLastError());
  return 0;
}

int csnet_train_gn_prelu_fwd(const float* z, float* y, int32_t N, int32_t C, int32_t HW, int32_t groups, const float* mean,
                             const float* var, const float* gamma, const float* beta, const float* slope, float eps, void* stream) {
  if (!z || !y || !mean || !var || !gamma || !beta || !slope || !gn_args_ok(N, C, HW, groups))
    return cfail(CSNET_E_INVALID, "gn_prelu_fwd: bad arguments");
  csnet::gn::gn_prelu_fwd_kernel<<<dim3(C, N), csnet::gn::kThreads, 0, (cudaStream_t)stream>>>(z, y, C, HW, groups, mean, var, gamma,
                                                                                            beta, slope, eps);
  CF_CHECK(cudaGetLastError());
  return 0;
}

int csnet_train_gn_prelu_bwd(const float* z, const float* dy, float* dz, int32_t N, int32_t C, int32_t HW, int32_t groups,
                             const float* mean, const float* var, const float* gamma, const float* beta, const float* slope, float eps,
                             float* dgamma, float* dbeta, float* dslope, float* ws, void* stream) {
  if (!z || !dy || !dz || !mean || !var || !gamma || !beta || !slope || !dgamma || !dbeta || !dslope || !ws ||
      !gn_args_ok(N, C, HW, groups))
    return cfail(CSNET_E_INVALID, "gn_prelu_bwd: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  csnet::gn::gn_bwd_reduce_kernel<<<dim3(C, N), csnet::gn::kThreads, 0, st>>>(z, dy, C, HW, groups, mean, var, gamma, beta, slope, eps, ws);
  CF_CHECK(cudaGetLastError());
  csnet::gn::gn_bwd_dz_kernel<<<dim3(C, N), csnet::gn::kThreads, 0, st>>>(z, dy, dz, N, C, HW, groups, mean, var, gamma, beta, slope, eps,
                                                                         ws, dgamma, dbeta, dslope);
  CF_CHECK(cudaGetLastError());
  return 0;
}

// The same calls on bf16 z / y / dy / dz (CSF+Res2Net training with bf16 storage).
int csnet_train_gn_stats_bf16(const void* z, int32_t N, int32_t C, int32_t HW, int32_t groups, float* mean, float* var, void* stream) {
  if (!z || !mean || !var || !gn_args_ok(N, C, HW, groups)) return cfail(CSNET_E_INVALID, "gn_stats_bf16: bad arguments");
  csnet::gn::gn_stats_bf16_kernel<<<N * groups, csnet::gn::kStatThreads, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)z, C, HW, groups, mean, var);
  CF_CHECK(cudaGetLastError());
  return 0;
}

int csnet_train_gn_prelu_fwd_bf16(const void* z, void* y, int32_t N, int32_t C, int32_t HW, int32_t groups, const float* mean,
                                  const float* var, const float* gamma, const float* beta, const float* slope, float eps, void* stream) {
  if (!z || !y || !mean || !var || !gamma || !beta || !slope || !gn_args_ok(N, C, HW, groups))
    return cfail(CSNET_E_INVALID, "gn_prelu_fwd_bf16: bad arguments");
  csnet::gn::gn_prelu_fwd_bf16_kernel<<<dim3(C, N), csnet::gn::kThreads, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)z, (__nv_bfloat16*)y, C, HW, groups, mean, var, gamma,
                                                                              beta, slope, eps);
  CF_CHECK(cudaGetLastError());
  return 0;
}

int csnet_train_gn_prelu_bwd_bf16(const void* z, const void* dy, void* dz, int32_t N, int32_t C, int32_t HW, int32_t groups,
                                  const float* mean, const float* var, const float* gamma, const float* beta, const float* slope, float eps,
                                  float* dgamma, float* dbeta, float* dslope, float* ws, void* stream) {
  if (!z || !dy || !dz || !mean || !var || !gamma || !beta || !slope || !dgamma || !dbeta || !dslope || !ws ||
      !gn_args_ok(N, C, HW, groups))
    return cfail(CSNET_E_INVALID, "gn_prelu_bwd_bf16: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  csnet::gn::gn_bwd_reduce_bf16_kernel<<<dim3(C, N), csnet::gn::kThreads, 0, st>>>((const __nv_bfloat16*)z, (const __nv_bfloat16*)dy, C, HW, groups, mean, var, gamma, beta,
                                                             slope, eps, ws);
  CF_CHECK(cudaGetLastError());
  csnet::gn::gn_bwd_dz_bf16_kernel<<<dim3(C, N), csnet::gn::kThreads, 0, st>>>((const __nv_bfloat16*)z, (const __nv_bfloat16*)dy, (__nv_bfloat16*)dz, N, C, HW, groups, mean, var, gamma,
                                                         beta, slope, eps, ws, dgamma, dbeta, dslope);
  CF_CHECK(cudaGetLastError());
  return 0;
}

}  // extern "C"
