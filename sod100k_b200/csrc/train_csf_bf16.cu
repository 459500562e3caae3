// train_csf_bf16.cu — the CSF+Res2Net head's convolutions with bf16 activation storage (include/csnet_b200.h, csnet_train_conv_*_bf16
// and csnet_train_cast_bf16).
//
// Convolutions run on the tensor-core implicit GEMM of gemm_bf16.cuh (bf16 operands, fp32 accumulation); the weights are the fp32
// parameters rounded once to nearest-even bf16 by csnet_train_cast_bf16.  The bf16 GroupNorm and resize calls sit beside their fp32
// twins (train_csf.cu, plan.cu).
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <cstdint>
#include <string>

#include "../../include/csnet_b200.h"
#include "gemm_bf16.cuh"

namespace csnet {
void train_set_error(const char* msg);     // train_ops.cu: the message csnet_train_last_error returns
}

namespace {

using bf16 = __nv_bfloat16;
namespace gbf = csnet::gbf;
using gbf::Args;

int cfail(int code, const std::string& what) {
  csnet::train_set_error(what.c_str());
  return code;
}

#define CB_CHECK(expr)                                                                           \
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

// What a call does: the GEMM extents, the k tiles and the split (conv_setup of train_csf.cu with the one 128 x 128 x 32 tile).
int conv_setup(int form, int N, int H, int W, const csnet_conv_seg_bf16* segs, int n_segs, int splits, Args& A) {
  if (form < 0 || form > 2 || N < 1 || H < 1 || W < 1 || !segs || n_segs < 1 || n_segs > gbf::kMaxSegs)
    return cfail(CSNET_E_INVALID, "conv_bf16: bad form, shape or segment count");
  if ((int64_t)H * W > (1 << 30)) return cfail(CSNET_E_INVALID, "conv_bf16: plane too large");
  if (form == CSNET_CONV_WGRAD && n_segs != 1) return cfail(CSNET_E_INVALID, "conv_bf16 wgrad: one segment per call");
  if (splits < 0) return cfail(CSNET_E_INVALID, "conv_bf16: bad splits");
  const int ks = segs[0].ksize;
  A = Args{};
  A.nseg = n_segs;
  A.N = N; A.H = H; A.W = W; A.HW = H * W;
  for (int s = 0; s < n_segs; ++s) {
    const csnet_conv_seg_bf16& q = segs[s];
    if (q.ksize != ks || (ks != 1 && ks != 3) || q.dil < 1 || q.cin < 1 || q.cout < 1 || q.C < 1 || q.ldw < q.cin * ks * ks || !q.src)
      return cfail(CSNET_E_INVALID, "conv_bf16: bad segment (ksize 1 or 3 shared by all, dil >= 1, ldw >= cin k^2, src set)");
    if (form != CSNET_CONV_WGRAD && !q.w) return cfail(CSNET_E_INVALID, "conv_bf16: null weight");
    if (form != CSNET_CONV_DGRAD && (q.c0 < 0 || q.c0 + q.cin > q.C)) return cfail(CSNET_E_INVALID, "conv_bf16: input slice outside src");
    if (form == CSNET_CONV_DGRAD && (q.cout0 < 0 || q.cout0 + q.cout > q.C)) return cfail(CSNET_E_INVALID, "conv_bf16 dgrad: gradient slice outside src");
    if (form == CSNET_CONV_WGRAD && q.cout0 < 0) return cfail(CSNET_E_INVALID, "conv_bf16 wgrad: gradient slice outside ddst");
    if (form == CSNET_CONV_FWD && (q.cout != segs[0].cout || q.cout0 != segs[0].cout0)) return cfail(CSNET_E_INVALID, "conv_bf16 fwd: segments write one slice");
    if (form == CSNET_CONV_DGRAD && q.cin != segs[0].cin) return cfail(CSNET_E_INVALID, "conv_bf16 dgrad: segments feed one slice");
    gbf::Seg& S = A.seg[s];
    S.src = (const bf16*)q.src; S.w = (const bf16*)q.w;
    S.C = q.C; S.c0 = q.c0; S.cin = q.cin; S.cout0 = q.cout0; S.cout = q.cout; S.dil = q.dil; S.ldw = q.ldw;
    S.K = form == CSNET_CONV_FWD ? q.cin * ks * ks : q.cout * ks * ks;
  }
  if (form == CSNET_CONV_FWD) { A.M = segs[0].cout; A.Ncol = A.HW; }
  else if (form == CSNET_CONV_DGRAD) { A.M = segs[0].cin; A.Ncol = A.HW; }
  else { A.M = segs[0].cout; A.Ncol = segs[0].cin * ks * ks; }
  int t = 0;
  if (form == CSNET_CONV_WGRAD) {
    A.kt_img = (A.HW + gbf::BK - 1) / gbf::BK;
    t = A.kt_img * N;
  } else {
    for (int s = 0; s < n_segs; ++s) { A.seg[s].tile0 = t; t += (A.seg[s].K + gbf::BK - 1) / gbf::BK; }
  }
  A.ktiles = t;
  const int images = form == CSNET_CONV_WGRAD ? 1 : N;
  const int64_t blocks = (int64_t)((A.M + gbf::BM - 1) / gbf::BM) * ((A.Ncol + gbf::BN - 1) / gbf::BN) * images;
  if (splits == 0) {                                            // fill two waves; keep >= 4 k tiles per split
    const int64_t want = blocks >= 2 * num_sms() ? 1 : (2 * num_sms() + blocks - 1) / blocks;
    int64_t cap = t / 4 < 64 ? t / 4 : 64;
    splits = (int)(want < cap ? want : cap);
    if (splits < 1) splits = 1;
  }
  if (splits > t) splits = t > 0 ? t : 1;
  if (blocks * splits > 0x7fffffffLL || (int64_t)images * splits > 65535)
    return cfail(CSNET_E_INVALID, "conv_bf16: grid too large");
  A.splits = splits;
  return 0;
}

int64_t ws_need(const Args& A, int form) {
  const int images = form == CSNET_CONV_WGRAD ? 1 : A.N;
  return A.splits > 1 ? (int64_t)A.splits * images * A.M * A.Ncol * 4 : 0;
}

int chain(const Args& A) { return ((A.ktiles + A.splits - 1) / A.splits) * gbf::BK; }

template <int KS, int FORM, typename TD>
int launch_t(const Args& A, cudaStream_t st) {
  const int images = FORM == gbf::kWgrad ? 1 : A.N;
  const dim3 grid((unsigned)((A.Ncol + gbf::BN - 1) / gbf::BN), (unsigned)((A.M + gbf::BM - 1) / gbf::BM), (unsigned)(images * A.splits));
  gbf::gemm_bf16_kernel<KS, FORM, TD><<<grid, gbf::kThreads, 0, st>>>(A);
  CB_CHECK(cudaGetLastError());
  if (A.splits > 1) {
    const int64_t total = (int64_t)images * A.M * A.Ncol;
    int64_t blocks = (total + gbf::kThreads - 1) / gbf::kThreads;
    if (blocks > 8 * num_sms()) blocks = 8 * num_sms();
    gbf::gemm_bf16_merge_kernel<FORM, TD><<<(unsigned)blocks, gbf::kThreads, 0, st>>>(A, images);
    CB_CHECK(cudaGetLastError());
  }
  return 0;
}

template <int FORM, typename TD>
int launch_form(const Args& A, int ks, cudaStream_t st) {
  return ks == 1 ? launch_t<1, FORM, TD>(A, st) : launch_t<3, FORM, TD>(A, st);
}

int conv_run(int form, int dst_dtype, Args& A, int ks, float* ws, int64_t ws_bytes, void* stream) {
  const int64_t need = ws_need(A, form);
  if (need > 0 && (!ws || ws_bytes < need)) return cfail(CSNET_E_INVALID, "conv_bf16: workspace too small for the split (csnet_train_conv_plan_bf16)");
  A.ws = ws;
  cudaStream_t st = (cudaStream_t)stream;
  const bool f32 = dst_dtype == CSNET_F32;
  if (form == CSNET_CONV_FWD) return f32 ? launch_form<gbf::kFwd, float>(A, ks, st) : launch_form<gbf::kFwd, bf16>(A, ks, st);
  if (form == CSNET_CONV_DGRAD) return f32 ? launch_form<gbf::kDgrad, float>(A, ks, st) : launch_form<gbf::kDgrad, bf16>(A, ks, st);
  return launch_form<gbf::kWgrad, float>(A, ks, st);
}

__global__ void __launch_bounds__(256) cast_bf16_kernel(const float* __restrict__ src, bf16* __restrict__ dst, int64_t n) {
  for (int64_t i = blockIdx.x * 256ll + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256) dst[i] = __float2bfloat16_rn(src[i]);
}

}  // namespace

extern "C" {

int csnet_train_conv_plan_bf16(int32_t form, int32_t N, int32_t H, int32_t W, const csnet_conv_seg_bf16* segs, int32_t n_segs,
                               int32_t splits, int32_t* splits_out, int32_t* chain_out, int64_t* ws_bytes) {
  Args A;
  if (int rc = conv_setup(form, N, H, W, segs, n_segs, splits, A)) return rc;
  if (splits_out) *splits_out = A.splits;
  if (chain_out) *chain_out = chain(A);
  if (ws_bytes) *ws_bytes = ws_need(A, form);
  return 0;
}

int csnet_train_conv_fwd_bf16(void* dst, int32_t dst_dtype, int32_t N, int32_t C, int32_t H, int32_t W, const csnet_conv_seg_bf16* segs,
                              int32_t n_segs, const float* bias, int32_t accumulate, int32_t splits, float* ws, int64_t ws_bytes,
                              void* stream) {
  Args A;
  if (int rc = conv_setup(CSNET_CONV_FWD, N, H, W, segs, n_segs, splits, A)) return rc;
  if (dst_dtype != CSNET_F32 && dst_dtype != CSNET_BF16) return cfail(CSNET_E_INVALID, "conv_fwd_bf16: dst_dtype must be CSNET_F32 or CSNET_BF16");
  if (!dst || segs[0].cout0 < 0 || segs[0].cout0 + segs[0].cout > C) return cfail(CSNET_E_INVALID, "conv_fwd_bf16: output slice outside dst");
  A.dst = dst; A.Cd = C; A.d0 = segs[0].cout0; A.bias = bias; A.accumulate = accumulate != 0;
  return conv_run(CSNET_CONV_FWD, dst_dtype, A, segs[0].ksize, ws, ws_bytes, stream);
}

int csnet_train_conv_dgrad_bf16(void* dsrc, int32_t dsrc_dtype, int32_t N, int32_t C, int32_t H, int32_t W, int32_t c0, int32_t cin,
                                const csnet_conv_seg_bf16* segs, int32_t n_segs, int32_t accumulate, int32_t splits, float* ws,
                                int64_t ws_bytes, void* stream) {
  Args A;
  if (int rc = conv_setup(CSNET_CONV_DGRAD, N, H, W, segs, n_segs, splits, A)) return rc;
  if (dsrc_dtype != CSNET_F32 && dsrc_dtype != CSNET_BF16) return cfail(CSNET_E_INVALID, "conv_dgrad_bf16: dsrc_dtype must be CSNET_F32 or CSNET_BF16");
  if (!dsrc || c0 < 0 || cin != segs[0].cin || c0 + cin > C) return cfail(CSNET_E_INVALID, "conv_dgrad_bf16: gradient slice outside dsrc");
  A.dst = dsrc; A.Cd = C; A.d0 = c0; A.accumulate = accumulate != 0;
  return conv_run(CSNET_CONV_DGRAD, dsrc_dtype, A, segs[0].ksize, ws, ws_bytes, stream);
}

int csnet_train_conv_wgrad_bf16(const void* ddst, int32_t N, int32_t Cd, int32_t H, int32_t W, const csnet_conv_seg_bf16* seg, float* dw,
                                int32_t accumulate, int32_t splits, float* ws, int64_t ws_bytes, void* stream) {
  Args A;
  if (int rc = conv_setup(CSNET_CONV_WGRAD, N, H, W, seg, 1, splits, A)) return rc;
  if (!ddst || !dw || seg->cout0 + seg->cout > Cd) return cfail(CSNET_E_INVALID, "conv_wgrad_bf16: gradient slice outside ddst");
  A.dy = (const bf16*)ddst; A.Cy = Cd; A.y0 = seg->cout0; A.dst = dw; A.ldd = seg->ldw; A.accumulate = accumulate != 0;
  return conv_run(CSNET_CONV_WGRAD, CSNET_F32, A, seg->ksize, ws, ws_bytes, stream);
}

int csnet_train_cast_bf16(const float* src, void* dst, int64_t n, void* stream) {
  if (!src || !dst || n < 1) return cfail(CSNET_E_INVALID, "cast_bf16: bad arguments");
  int64_t blocks = (n + 255) / 256;
  if (blocks > 8 * num_sms()) blocks = 8 * num_sms();
  cast_bf16_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(src, (bf16*)dst, n);
  CB_CHECK(cudaGetLastError());
  return 0;
}

}  // extern "C"
