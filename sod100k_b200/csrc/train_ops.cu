// train_ops.cu — module-granular training primitives (fp32 activations), C ABI `csnet_train_*`.
//
// The reference trains with torch autograd over F.conv2d / F.batch_norm / F.prelu / pooling / F.interpolate
// (CSNet_training/train.py:203-216).  Train-mode BatchNorm puts a batch-wide reduction between every conv and its
// PReLU, so the closed unit here is the reference MODULE: raw conv mix -> batch statistics -> normalise + PReLU,
// and the matching backward pieces.  These kernels are generic (any shape) and correctness-first; they reuse the
// per-thread bodies of generic_ops.cuh for the forward mix.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdint>
#include <string>

#include "../../include/csnet_b200.h"
#include "bce_sum.cuh"
#include "generic_ops.cuh"
#include "train_fast.cuh"
#include "train_host.h"

namespace {

int tfail(int code, const char* what, cudaError_t e);
#define TR_CHECK(expr)                                              \
  do {                                                              \
    cudaError_t e_ = (expr);                                        \
    if (e_ != cudaSuccess) return tfail(CSNET_E_CUDA, #expr, e_);   \
  } while (0)

constexpr int kT = 256;

using csnet::tf::block_sum3;
using csnet::tf::warp_sum;

// ---- BatchNorm (train) + PReLU: the fp32 instances of train_body.cuh's bodies ------------------------------------------------
__global__ void __launch_bounds__(kT) bn_stats_kernel(const float* __restrict__ z, int N, int C, int HW, int S, float* mean,
                                                      float* var, float* ws, unsigned* cnt) {
  csnet::tf::bn_stats_body(z, N, C, HW, S, mean, var, ws, cnt);
}

__global__ void __launch_bounds__(kT) bn_prelu_fwd_kernel(const float* __restrict__ z, float* __restrict__ y, int C, int HW,
                                                          const float* mean, const float* var, const float* gamma,
                                                          const float* beta, const float* slope, float eps, float* gap) {
  csnet::tf::bn_prelu_fwd_body(z, y, C, HW, mean, var, gamma, beta, slope, eps, gap);
}

__global__ void __launch_bounds__(kT) bn_prelu_bwd_reduce_kernel(const float* __restrict__ z, const float* __restrict__ dy, int N,
                                                                 int C, int HW, int S, const float* mean, const float* var,
                                                                 const float* gamma, const float* beta, const float* slope,
                                                                 float eps, float* dgamma, float* dbeta, float* dslope, float* ws,
                                                                 unsigned* cnt) {
  csnet::tf::bn_prelu_bwd_reduce_body(z, dy, N, C, HW, S, mean, var, gamma, beta, slope, eps, dgamma, dbeta, dslope, ws, cnt);
}

__global__ void __launch_bounds__(kT) bn_prelu_bwd_apply_kernel(const float* __restrict__ z, const float* __restrict__ dy,
                                                                float* __restrict__ dz, int N, int C, int HW, const float* mean,
                                                                const float* var, const float* gamma, const float* beta,
                                                                const float* slope, float eps, const float* dgamma,
                                                                const float* dbeta, int frozen) {
  csnet::tf::bn_prelu_bwd_apply_body(z, dy, dz, N, C, HW, mean, var, gamma, beta, slope, eps, dgamma, dbeta, frozen);
}

// ---- MIX forward (raw: no bias / slope) -----------------------------------------------------------------------
__global__ void __launch_bounds__(kT, 2) tr_mix_fwd_kernel(const __grid_constant__ csnet::MixArgs A) {
  __shared__ float ws[csnet::kMixStageFloats];
  const int co_base = blockIdx.y * csnet::kMixCT, n = blockIdx.z;
  const int pix = blockIdx.x * kT + threadIdx.x;
  const bool live = pix < A.H * A.W;
  const int oy = live ? pix / A.W : 0, ox = live ? pix % A.W : 0;
  float acc[csnet::kMixCT];
#pragma unroll
  for (int t = 0; t < csnet::kMixCT; ++t) acc[t] = 0.f;
  for (int p = 0; p < A.n_paths; ++p) {
    const csnet::MixPath& P = A.p[p];
    if (P.ksize == 0 || !csnet::mix_path_live(P, co_base)) continue;      // block-uniform
    const int chunk = csnet::mix_chunk_channels(P.ksize);
    for (int ci0 = 0; ci0 < P.cin; ci0 += chunk) {
      const int ci1 = ci0 + chunk < P.cin ? ci0 + chunk : P.cin;
      __syncthreads();
      csnet::mix_stage_chunk(P, co_base, ci0, ci1, ws, threadIdx.x, kT);
      __syncthreads();
      if (live) csnet::mix_acc_chunk(P, ws, ci0, ci1, n, oy, ox, acc);
    }
  }
  if (live) csnet::mix_finish(A, n, oy, ox, co_base, acc);
}

// ---- MIX backward: data gradient of ONE path, gather over source elements -------------------------------------
// dsrc[n][ci][ys][xs] for the source slice [c0, c0+cin) (dsrc holds exactly cin channels).
__global__ void __launch_bounds__(kT) tr_mix_dgrad_kernel(const float* __restrict__ ddst, int C, int H, int W, const csnet::MixPath P,
                                                          float* __restrict__ dsrc) {
  const int ci = blockIdx.y, n = blockIdx.z;
  const int pix = blockIdx.x * kT + threadIdx.x;
  if (pix >= P.H * P.W) return;
  const int ys = pix / P.W, xs = pix % P.W;
  const size_t dplane = (size_t)H * W;
  const float* dd = ddst + ((size_t)n * C + P.cout0) * dplane;
  float g = 0.f;
  if (P.ksize == 0) {
    // adjoint of the bilinear up-sample by `up` (align_corners=False, source index clamped at 0)
    const int up = P.up;
    const float inv = 1.f / (float)up;
    const float* d = dd + (size_t)ci * dplane;                 // resample paths map channel c -> cout0 + c
    const int y_lo = ys * up - up < 0 ? 0 : ys * up - up, y_hi = (ys * up + 2 * up) > H ? H : ys * up + 2 * up;
    const int x_lo = xs * up - up < 0 ? 0 : xs * up - up, x_hi = (xs * up + 2 * up) > W ? W : xs * up + 2 * up;
    for (int oy = y_lo; oy < y_hi; ++oy) {
      float sy = ((float)oy + 0.5f) * inv - 0.5f;
      sy = sy < 0.f ? 0.f : sy;
      const int y0 = (int)sy, y1 = y0 + (y0 < P.H - 1 ? 1 : 0);
      const float ly = sy - (float)y0, wy = (y0 == ys ? 1.f - ly : 0.f) + (y1 == ys ? ly : 0.f);
      if (wy == 0.f) continue;
      for (int ox = x_lo; ox < x_hi; ++ox) {
        float sx = ((float)ox + 0.5f) * inv - 0.5f;
        sx = sx < 0.f ? 0.f : sx;
        const int x0 = (int)sx, x1 = x0 + (x0 < P.W - 1 ? 1 : 0);
        const float lx = sx - (float)x0, wx = (x0 == xs ? 1.f - lx : 0.f) + (x1 == xs ? lx : 0.f);
        if (wx != 0.f) g += wy * wx * d[(size_t)oy * W + ox];
      }
    }
    dsrc[((size_t)n * P.cin + ci) * P.H * P.W + pix] = g;
    return;
  }
  // conv path: which conv-grid cell does this source element feed, and with which factor?
  int yc = ys, xc = xs;
  float factor = 1.f;
  const int64_t plane = ((int64_t)n * P.C + P.c0 + ci) * (int64_t)P.H * P.W;
  if (P.pre_avg) { yc >>= 1; xc >>= 1; factor = 0.25f; }
  if (P.pool > 1) {
    // max_pool2d backward routes the gradient to the FIRST maximum of the window (row-major scan, strict >)
    const int ym = yc / P.pool, xm = xc / P.pool;
    float best = -INFINITY;
    int by = -1, bx = -1;
    for (int py = 0; py < P.pool; ++py)
      for (int px = 0; px < P.pool; ++px) {
        const int ya = ym * P.pool + py, xa = xm * P.pool + px;
        float v;
        if (P.pre_avg) {
          const int64_t b = plane + (int64_t)(2 * ya) * P.W + 2 * xa;
          const float* s = reinterpret_cast<const float*>(P.src);
          v = (((s[b] + s[b + 1]) + s[b + P.W]) + s[b + P.W + 1]) * 0.25f;
        } else {
          v = reinterpret_cast<const float*>(P.src)[plane + (int64_t)ya * P.W + xa];
        }
        if (v > best) { best = v; by = ya; bx = xa; }
      }
    if (by != yc || bx != xc) { dsrc[((size_t)n * P.cin + ci) * P.H * P.W + pix] = 0.f; return; }
    yc = ym; xc = xm;
  }
  const int kk = P.ksize * P.ksize;
  for (int ky = 0; ky < P.ksize; ++ky) {
    const int ty = yc + P.pad - ky * P.dil;
    if (ty < 0 || ty % P.stride) continue;
    const int oy = ty / P.stride;
    if (oy >= H) continue;
    for (int kx = 0; kx < P.ksize; ++kx) {
      const int tx = xc + P.pad - kx * P.dil;
      if (tx < 0 || tx % P.stride) continue;
      const int ox = tx / P.stride;
      if (ox >= W) continue;
      const float* wr = P.w + ((size_t)ci * kk + ky * P.ksize + kx) * P.cout;
      const float* d = dd + (size_t)oy * W + ox;
      for (int co = 0; co < P.cout; ++co) g += wr[co] * d[(size_t)co * dplane];
    }
  }
  dsrc[((size_t)n * P.cin + ci) * P.H * P.W + pix] = g * factor;
}

// ---- MIX backward: weight gradient of ONE conv path: dw[ci][tap][co] (kernel layout), batch split over grid.z ----
__global__ void __launch_bounds__(kT) tr_mix_wgrad_kernel(const float* __restrict__ ddst, int N, int C, int H, int W,
                                                          const csnet::MixPath P, float* dw) {
  constexpr int COT = 8;
  const int ci = blockIdx.x, kk = P.ksize * P.ksize, tap = blockIdx.y % kk, cot = blockIdx.y / kk;
  const int ky = tap / P.ksize, kx = tap % P.ksize, co0 = cot * COT;
  const int div = (P.pre_avg ? 2 : 1) * P.pool, Hc = P.H / div, Wc = P.W / div;
  float acc[COT];
#pragma unroll
  for (int t = 0; t < COT; ++t) acc[t] = 0.f;
  const size_t dplane = (size_t)H * W;
  for (int n = blockIdx.z; n < N; n += gridDim.z) {
    const int64_t plane = ((int64_t)n * P.C + P.c0 + ci) * (int64_t)P.H * P.W;
    const float* dd = ddst + ((size_t)n * C + P.cout0 + co0) * dplane;
    for (int i = threadIdx.x; i < H * W; i += kT) {
      const int oy = i / W, ox = i % W;
      const int y = oy * P.stride - P.pad + ky * P.dil, x = ox * P.stride - P.pad + kx * P.dil;
      if (y < 0 || y >= Hc || x < 0 || x >= Wc) continue;
      const float v = csnet::fetch_pooled(P, plane, y, x);
#pragma unroll
      for (int t = 0; t < COT; ++t)
        if (co0 + t < P.cout) acc[t] += v * dd[(size_t)t * dplane + i];
    }
  }
#pragma unroll
  for (int t = 0; t < COT; t += 3) {
    float a = acc[t], b = t + 1 < COT ? acc[t + 1] : 0.f, c = t + 2 < COT ? acc[t + 2] : 0.f;
    block_sum3(a, b, c);
    if (threadIdx.x == 0) {
      float* o = dw + ((size_t)ci * kk + tap) * P.cout + co0;
      if (co0 + t < P.cout) atomicAdd(o + t, a);
      if (t + 1 < COT && co0 + t + 1 < P.cout) atomicAdd(o + t + 1, b);
      if (t + 2 < COT && co0 + t + 2 < P.cout) atomicAdd(o + t + 2, c);
    }
  }
}

// ---- loss, optimiser ---------------------------------------------------------------------------------------
// F.binary_cross_entropy_with_logits(mean): loss = mean(max(z,0) - z*t + log1p(exp(-|z|))), dz = (sigmoid(z) - t) / n
__global__ void __launch_bounds__(kT) bce_kernel(const float* __restrict__ z, const float* __restrict__ t, float* dz, float* loss,
                                                 int64_t n, float inv_n, float grad_scale) {
  float s = 0.f, d0 = 0.f, d1 = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * kT + threadIdx.x; i < n; i += (int64_t)gridDim.x * kT) {
    const float v = z[i], y = t[i];
    s += fmaxf(v, 0.f) - v * y + log1pf(expf(-fabsf(v)));
    if (dz) dz[i] = (1.f / (1.f + expf(-v)) - y) * inv_n * grad_scale;
  }
  block_sum3(s, d0, d1);
  if (threadIdx.x == 0) atomicAdd(loss, s * inv_n);
}

// torch.optim.Adam (L2 weight decay folded into the gradient), many tensors per launch via a chunk table
struct AdamChunk { float* p; const float* g; float* m; float* v; int32_t n; float wd; };
__global__ void __launch_bounds__(kT) adam_kernel(const AdamChunk* chunks, float lr, float b1, float b2, float eps, float bc1,
                                                  float bc2_sqrt, float grad_scale) {
  const AdamChunk ch = chunks[blockIdx.x];
  for (int i = threadIdx.x; i < ch.n; i += kT) {
    const float p = ch.p[i];
    const float g = ch.g[i] * grad_scale + ch.wd * p;
    const float m = b1 * ch.m[i] + (1.f - b1) * g, v = b2 * ch.v[i] + (1.f - b2) * g * g;
    ch.m[i] = m; ch.v[i] = v;
    ch.p[i] = p - (lr / bc1) * (m / (sqrtf(v) / bc2_sqrt + eps));
  }
}

// Channel slimming (CSNet_training/model/csnet.py:571-760): dst[i][j][:] = src[out_idx[i]][in_idx[j]][:] for the surviving channels,
// dst [dCo][dCi][kk] (zero elsewhere, set by the caller), src [Co][Ci][kk]; indices outside the source are skipped.
__global__ void __launch_bounds__(kT) slim_gather_kernel(const float* __restrict__ src, int Co, int Ci, int kk, const long long* __restrict__ oi, int no,
                                                         const long long* __restrict__ ii, int ni, float* __restrict__ dst, int dCi) {
  const long long e = (long long)blockIdx.x * kT + threadIdx.x, total = (long long)no * ni * kk;
  if (e >= total) return;
  const int t = (int)(e % kk), j = (int)((e / kk) % ni), i = (int)(e / ((long long)kk * ni));
  const long long so = oi[i], si = ii[j];
  if (so < 0 || so >= Co || si < 0 || si >= Ci) return;
  dst[((long long)i * dCi + j) * kk + t] = src[(so * Ci + si) * kk + t];
}

thread_local std::string t_err;
int tfail(int code, const char* what, cudaError_t e) {
  t_err = std::string(what) + ": " + cudaGetErrorString(e);
  return code;
}

// ---- SalMetric counting (sal_metric.cpp:86-120): per-image 256-bin histograms of the quantised saliency ----------------
__global__ void __launch_bounds__(kT) salmetric_hist_kernel(const float* __restrict__ prob, const uint8_t* __restrict__ gt, int64_t HW,
                                                            uint32_t* hist_all, uint32_t* hist_pos, unsigned long long* abs_sum) {
  __shared__ uint32_t ha[256], hp[256];
  __shared__ unsigned long long sd;
  const int n = blockIdx.y;
  ha[threadIdx.x] = 0u; hp[threadIdx.x] = 0u;              // kT == 256
  if (threadIdx.x == 0) sd = 0ull;
  __syncthreads();
  unsigned int d = 0;
  for (int64_t i = (int64_t)blockIdx.x * kT + threadIdx.x; i < HW; i += (int64_t)gridDim.x * kT) {
    const double v = (double)prob[n * HW + i] * 255.0;     // the reference multiplies a float64 array (skimage resize output)
    const int q = v <= 0.0 ? 0 : (v >= 255.0 ? 255 : (int)v);
    const int g = gt[n * HW + i];
    atomicAdd(&ha[q], 1u);
    if (g > 128) atomicAdd(&hp[q], 1u);
    d += (unsigned)(q > g ? q - g : g - q);
  }
  atomicAdd(&sd, (unsigned long long)d);
  __syncthreads();
  if (ha[threadIdx.x]) atomicAdd(hist_all + (size_t)n * 256 + threadIdx.x, ha[threadIdx.x]);
  if (hp[threadIdx.x]) atomicAdd(hist_pos + (size_t)n * 256 + threadIdx.x, hp[threadIdx.x]);
  if (threadIdx.x == 0) atomicAdd(abs_sum + n, sd);
}

}  // namespace

namespace csnet {
// The other training sources (train_csf.cu, train_bf16.cu, plan.cu's resize pair) report through csnet_train_last_error too.
void train_set_error(const char* msg) { t_err = msg; }

namespace tr {

MixPath to_path(const csnet_train_path& q) {
  csnet::MixPath m{};
  m.src = q.src; m.w = q.w; m.dtype = CSNET_F32; m.C = q.C; m.H = q.H; m.W = q.W; m.c0 = q.c0; m.cin = q.cin;
  m.pre_avg = q.pre_avg; m.pool = q.pool; m.ksize = q.ksize; m.dil = q.dil; m.stride = q.stride; m.pad = q.pad; m.up = q.up;
  m.cout0 = q.cout0; m.cout = q.cout;
  return m;
}

// Workspace of the channel reductions: partials [C][parts][3] + one ticket counter per channel.  One set PER DEVICE (indexed by
// the current device, i.e. the device of the tensors the caller's torch stream belongs to), grown on demand; the training entry
// points of one device are meant to be issued on ONE stream (calls serialise there, so sharing within a device is safe).
struct RedWs { float* ws = nullptr; unsigned* cnt = nullptr; size_t ws_cap = 0, cnt_cap = 0; float* part = nullptr; size_t part_cap = 0; };
static RedWs g_red[kMaxDevices];

int reduce_workspace(int C, int parts, cudaStream_t st, float** ws, unsigned** cnt) {
  int dev = 0;
  TR_CHECK(cudaGetDevice(&dev));
  if (dev < 0 || dev >= kMaxDevices) { t_err = "device index out of range"; return CSNET_E_INVALID; }
  RedWs& R = g_red[dev];
  const size_t need = (size_t)C * parts * 3;
  if (need > R.ws_cap) {
    TR_CHECK(cudaStreamSynchronize(st));
    if (R.ws) cudaFree(R.ws);
    R.ws = nullptr; R.ws_cap = 0;
    TR_CHECK(cudaMalloc(&R.ws, need * 2 * sizeof(float)));
    R.ws_cap = need * 2;
  }
  if ((size_t)C > R.cnt_cap) {
    TR_CHECK(cudaStreamSynchronize(st));
    if (R.cnt) cudaFree(R.cnt);
    R.cnt = nullptr; R.cnt_cap = 0;
    const size_t cap = (size_t)C * 2 < 1024 ? 1024 : (size_t)C * 2;
    TR_CHECK(cudaMalloc(&R.cnt, cap * sizeof(unsigned)));
    TR_CHECK(cudaMemset(R.cnt, 0, cap * sizeof(unsigned)));
    R.cnt_cap = cap;
  }
  *ws = R.ws;
  *cnt = R.cnt;
  return CSNET_OK;
}

// Block partials of the weight-gradient kernels ([blocks][elements] floats), one buffer per device, grown on demand.
int partial_workspace(size_t floats, cudaStream_t st, float** out) {
  int dev = 0;
  TR_CHECK(cudaGetDevice(&dev));
  if (dev < 0 || dev >= kMaxDevices) { t_err = "device index out of range"; return CSNET_E_INVALID; }
  RedWs& R = g_red[dev];
  if (floats > R.part_cap) {
    TR_CHECK(cudaStreamSynchronize(st));
    if (R.part) cudaFree(R.part);
    R.part = nullptr; R.part_cap = 0;
    const size_t cap = floats * 2 < (1u << 20) ? (1u << 20) : floats * 2;
    TR_CHECK(cudaMalloc(&R.part, cap * sizeof(float)));
    R.part_cap = cap;
  }
  *out = R.part;
  return CSNET_OK;
}

// ---- fast (register-tiled) dispatch: train_fast.cuh ------------------------------------------------------------------------------

int current_device() {
  int dev = 0;
  cudaGetDevice(&dev);
  return dev < 0 || dev >= kMaxDevices ? 0 : dev;
}

int num_sms() {
  static int sms[kMaxDevices] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= kMaxDevices) return 132;
  if (!sms[dev]) cudaDeviceGetAttribute(&sms[dev], cudaDevAttrMultiProcessorCount, dev);
  return sms[dev] > 0 ? sms[dev] : 132;
}

bool conv_tile_geometry(tf::ConvArgs& A) {
  A.quads = (A.W + 3) / 4;
  A.vec = (A.W % 4) == 0;
  if (A.quads > tf::kT) return false;
  if (A.H * A.quads * 2 <= tf::kT) { A.R = A.H; A.ipb = tf::kT / (A.H * A.quads); }
  else { A.ipb = 1; A.R = tf::kT / A.quads; if (A.R > A.H) A.R = A.H; }
  if (A.ipb > A.N) A.ipb = A.N;
  return true;
}

bool conv_path_geometry(tf::ConvPath& P, const tf::ConvArgs& A, int esize) {
  const int kk = A.ksize * A.ksize;
  P.halo = P.dil * (A.ksize / 2);
  P.hp = (P.halo + 3) / 4 * 4;
  P.Wp = (A.W + 2 * P.hp + 3) / 4 * 4;
  P.rows = A.R + 2 * P.halo;
  const size_t per_ci = (size_t)A.ipb * P.rows * P.Wp * esize, per_w = (size_t)kk * tf::kCoT * sizeof(float);
  size_t chunk = kFastSmem / per_ci;
  if (chunk > kFastWsm / per_w) chunk = kFastWsm / per_w;
  if (chunk < 1) return false;
  P.chunk = chunk < (size_t)P.cin ? (int)chunk : P.cin;
  return true;
}

bool dense_conv_path(const csnet::MixPath& P, int H, int W) {
  return P.ksize >= 1 && (P.ksize & 1) && P.stride == 1 && P.pre_avg == 0 && P.pool == 1 && P.up == 1 && P.H == H && P.W == W &&
         P.pad == P.dil * (P.ksize / 2) && P.dil >= 1;
}

// segments per image plane: enough parts to fill the GPU for narrow layers and small batches, at most 64 per plane
int reduce_segments(int N, int C, int HW) {
  int S = 1;
  while ((long)N * C * S < 1184 && S < 64 && HW / (S * 2) >= 2048) S *= 2;
  return S;
}

// Geometry of the register-tiled weight gradient of one dense path (3x3 at any dilation, or 1x1 at dilation 1); false: the
// shape is not taken.  esize_in / esize_dd: bytes per element of the source and of the destination gradient.
bool wgrad_plan(const MixPath& P, const void* ddst, int N, int C, int H, int W, int esize_in, int esize_dd, WgradPlan& out) {
  if (!(dense_conv_path(P, H, W) && (P.ksize == 3 || (P.ksize == 1 && P.dil == 1)))) return false;
  const int kk = P.ksize * P.ksize;
  const int form = P.ksize == 1 ? 1 : (P.dil == 1 ? 3 : 0);    // template argument of conv_wgrad_kernel
  tf::WgradArgs G{};
  G.in = P.src; G.dd = ddst; G.N = N; G.Cs = P.C; G.c0 = P.c0; G.cin = P.cin; G.Cd = C; G.cout0 = P.cout0;
  G.cout = P.cout; G.H = H; G.W = W; G.dil = P.dil;
  G.cin4 = (P.cin + 3) / 4 * 4; G.cout4 = (P.cout + 3) / 4 * 4;
  G.hp = form == 0 ? (P.dil + 3) / 4 * 4 : 4;
  G.Wp = (W + 2 * G.hp + 3) / 4 * 4; G.quads = (W + 3) / 4; G.vec = (W % 4) == 0;
  auto rows_in = [&](int r) { return form == 0 ? 3 * r : r + (form == 3 ? 2 : 0); };
  auto pitch = [](int elems) { return elems + ((4 - elems % 32) + 32) % 32; };          // == 4 (mod 32); elems is a multiple of 4
  auto stage_bytes = [&](int r) {
    return (size_t)G.cin4 * pitch(rows_in(r) * G.Wp) * esize_in + (size_t)G.cout4 * pitch(r * G.Wp) * esize_dd;
  };
  int R = 0;                                               // the largest row band whose operands fit
  for (int r = 1; r <= H && r <= 16; ++r)
    if (stage_bytes(r) <= kFastSmemMax / 2) R = r;        // two stages in flight
  if (R < 1) return false;
  G.R = R;
  G.cpi = pitch(rows_in(R) * G.Wp); G.cpd = pitch(R * G.Wp);
  const int bands = (H + R - 1) / R;
  G.units = N * bands;
  G.mt = G.cin4 / 4 * (form == 1 ? 1 : 3); G.nt = G.cout4 / 4; G.tiles = G.mt * G.nt;
  int groups = 1;
  if (G.tiles <= tf::kT) {
    if (G.tiles >= 32) G.tpad = (G.tiles + 31) / 32 * 32;
    else { G.tpad = 1; while (G.tpad < G.tiles) G.tpad *= 2; }
    G.splits = tf::kT / G.tpad;
  } else {
    G.tpad = tf::kT; G.splits = 1; groups = (G.tiles + tf::kT - 1) / tf::kT;
  }
  const size_t stage = stage_bytes(R),
               red = (size_t)G.splits * G.tpad * (form == 1 ? 16 : 48) * sizeof(float);
  int gx = 2 * num_sms() / groups;
  gx = gx < 1 ? 1 : gx;
  gx = gx > G.units ? G.units : gx;
  out.A = G;
  out.form = form; out.gx = gx; out.groups = groups; out.nel = P.cin * kk * P.cout;
  out.smem = 2 * stage > red ? 2 * stage : red;
  return true;
}

int reduce_partials(const float* part, int parts, int n, float scale, float* out, cudaStream_t st) {
  tf::reduce_partials_kernel<<<(n + tf::kT - 1) / tf::kT, tf::kT, 0, st>>>(part, parts, n, scale, out);
  TR_CHECK(cudaGetLastError());
  return CSNET_OK;
}

}  // namespace tr
}  // namespace csnet

using namespace csnet::tr;

// 1x1 mixes (and mixes of resample-add paths only): the direct kernel
static int launch_conv1x1(const tf::ConvArgs& F, cudaStream_t st) {
  tf::C1Args A{};
  // 4 px x 16 channels per pass; rows that are only 8-byte multiples (14 wide) take 2 px x 32 channels with 8-byte loads.  (2 px x 32
  // measured SLOWER on the wide planes — 18 -> 18 @224^2: 1.12 ms vs 0.79 ms — twice the load instructions for the same bytes.)
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
  if (smem > 96 * 1024) return kNotHandled;                // (not a CSNet shape) -> the generic kernel
  static bool attr_dev[kMaxDevices] = {false};                // function attributes are per device
  bool& attr = attr_dev[current_device()];
  if (!attr) {
    cudaFuncSetAttribute(tf::conv1x1_kernel<2, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
    cudaFuncSetAttribute(tf::conv1x1_kernel<4, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
    cudaFuncSetAttribute(tf::conv1x1_kernel<4, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
    attr = true;
  }
  const size_t tasks = (size_t)A.N * A.H * A.quads;
  const unsigned blocks = (unsigned)((tasks + tf::kT - 1) / tf::kT);
  // <= 24 output channels: the narrow form (8 channels per pass, three CTAs per SM) hides the load latency a little better
  // (18 -> 18 @224^2 0.494 -> 0.472 ms, 13 -> 18 0.415 -> 0.357 ms; 34 -> 31 @112^2 is 8 % slower with it).
  const bool narrow = A.C <= 24;
  static bool attr_n_dev[kMaxDevices] = {false};
  bool& attr_n = attr_n_dev[current_device()];
  if (narrow && !attr_n) { cudaFuncSetAttribute(tf::conv1x1_narrow_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 72 * 1024); attr_n = true; }
  if (narrow && px == 4 && A.vec && smem <= 72 * 1024) tf::conv1x1_narrow_kernel<<<blocks, tf::kT, smem, st>>>(A);
  else if (px == 2) tf::conv1x1_kernel<2, true><<<blocks, tf::kT, smem, st>>>(A);
  else if (A.vec) tf::conv1x1_kernel<4, true><<<blocks, tf::kT, smem, st>>>(A);
  else tf::conv1x1_kernel<4, false><<<blocks, tf::kT, smem, st>>>(A);
  TR_CHECK(cudaGetLastError());
  return CSNET_OK;
}

static int launch_conv(tf::ConvArgs& A, cudaStream_t st) {
  if (A.n_conv == 0 || A.ksize == 1) {
    return launch_conv1x1(A, st);
  }
  const int kk = A.ksize * A.ksize;
  size_t tile = 0, wsm = 0;
  bool dil1 = true;
  for (int i = 0; i < A.n_conv; ++i) {
    const tf::ConvPath& P = A.p[i];
    const size_t t = (size_t)P.chunk * A.ipb * P.rows * P.Wp, w = (size_t)P.chunk * kk * tf::kCoT;
    tile = t > tile ? t : tile; wsm = w > wsm ? w : wsm;
    dil1 = dil1 && P.dil == 1;
  }
  A.tile_floats = (int)tile;
  const size_t smem = (tile + wsm) * sizeof(float);
  const int bands = (A.H + A.R - 1) / A.R;
  const unsigned grid = (unsigned)(((A.N + A.ipb - 1) / A.ipb) * bands);
  static bool attr_dev[kMaxDevices] = {false};
  bool& attr = attr_dev[current_device()];
  if (!attr) {
    cudaFuncSetAttribute(tf::conv_fwd_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, kFastSmemMax);
    cudaFuncSetAttribute(tf::conv_wgrad_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, kFastSmemMax);
    cudaFuncSetAttribute(tf::conv_fwd_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, kFastSmemMax);
    cudaFuncSetAttribute(tf::conv_wgrad_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, kFastSmemMax);
    cudaFuncSetAttribute(tf::conv_wgrad_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, kFastSmemMax);
    attr = true;
  }
  if (A.ksize == 3 && dil1) tf::conv_fwd_kernel<3><<<grid, tf::kT, smem, st>>>(A);
  else tf::conv_fwd_kernel<0><<<grid, tf::kT, smem, st>>>(A);
  TR_CHECK(cudaGetLastError());
  return CSNET_OK;
}

static thread_local float* g_red_ws = nullptr;          // the current call's workspace (set by reduce_workspace)
static thread_local unsigned* g_red_cnt = nullptr;
static int reduce_workspace(int C, int parts, cudaStream_t st) { return csnet::tr::reduce_workspace(C, parts, st, &g_red_ws, &g_red_cnt); }

extern "C" {

const char* csnet_train_last_error(void) { return t_err.c_str(); }

int csnet_train_bn_stats(const float* z, int32_t N, int32_t C, int32_t HW, float* mean, float* var, void* stream) {
  const int S = reduce_segments(N, C, HW);
  if (int rc = reduce_workspace(C, N * S, (cudaStream_t)stream)) return rc;
  bn_stats_kernel<<<dim3(C, N * S), kT, 0, (cudaStream_t)stream>>>(z, N, C, HW, S, mean, var, g_red_ws, g_red_cnt);
  TR_CHECK(cudaGetLastError());
  return CSNET_OK;
}

int csnet_train_bn_prelu_fwd(const float* z, float* y, int32_t N, int32_t C, int32_t HW, const float* mean, const float* var,
                             const float* gamma, const float* beta, const float* slope, float eps, float* gap, void* stream) {
  bn_prelu_fwd_kernel<<<dim3(C, N), kT, 0, (cudaStream_t)stream>>>(z, y, C, HW, mean, var, gamma, beta, slope, eps, gap);
  TR_CHECK(cudaGetLastError());
  return CSNET_OK;
}

int csnet_train_bn_prelu_bwd(const float* z, const float* dy, float* dz, int32_t N, int32_t C, int32_t HW, const float* mean,
                             const float* var, const float* gamma, const float* beta, const float* slope, float eps,
                             float* dgamma, float* dbeta, float* dslope, int32_t frozen, void* stream) {
  const int S = reduce_segments(N, C, HW);
  if (int rc = reduce_workspace(C, N * S, (cudaStream_t)stream)) return rc;
  bn_prelu_bwd_reduce_kernel<<<dim3(C, N * S), kT, 0, (cudaStream_t)stream>>>(z, dy, N, C, HW, S, mean, var, gamma, beta, slope, eps,
                                                                            dgamma, dbeta, dslope, g_red_ws, g_red_cnt);
  TR_CHECK(cudaGetLastError());
  bn_prelu_bwd_apply_kernel<<<dim3(C, N), kT, 0, (cudaStream_t)stream>>>(z, dy, dz, N, C, HW, mean, var, gamma, beta, slope, eps, dgamma, dbeta, frozen);
  TR_CHECK(cudaGetLastError());
  return CSNET_OK;
}

int csnet_train_dw_conv(const float* x, const float* w, float* y, int32_t N, int32_t C, int32_t H, int32_t W, float scale,
                        int32_t transposed, void* stream) {
  const int quads = (W + 3) / 4, rows = H < 8 ? H : 8, bands = (H + rows - 1) / rows;
  const size_t tasks = (size_t)N * C * bands * quads;
  tf::dw3_kernel<<<(unsigned)((tasks + tf::kT - 1) / tf::kT), tf::kT, 0, (cudaStream_t)stream>>>(x, w, y, N, C, H, W, scale, transposed, quads, rows);
  TR_CHECK(cudaGetLastError());
  return CSNET_OK;
}

int csnet_train_dw_wgrad(const float* x, const float* dy, float* dw, int32_t N, int32_t C, int32_t H, int32_t W, float scale, void* stream) {
  const int quads = (W + 3) / 4, rows = H < 8 ? H : 8, bands = (H + rows - 1) / rows;
  const size_t tasks = (size_t)N * bands * quads;
  int bx = (int)((tasks + tf::kT - 1) / tf::kT), cap = 4 * num_sms() / C;
  cap = cap < 1 ? 1 : cap;
  bx = bx > cap ? cap : bx;
  float* part = nullptr;
  if (int rc = partial_workspace((size_t)bx * C * 9, (cudaStream_t)stream, &part)) return rc;
  tf::dw3_wgrad_kernel<<<dim3(bx, C), tf::kT, 0, (cudaStream_t)stream>>>(x, dy, part, N, C, H, W, quads, rows);
  TR_CHECK(cudaGetLastError());
  tf::reduce_partials_kernel<<<(C * 9 + tf::kT - 1) / tf::kT, tf::kT, 0, (cudaStream_t)stream>>>(part, bx, C * 9, scale, dw);
  TR_CHECK(cudaGetLastError());
  return CSNET_OK;
}

int csnet_train_dw_bwd(const float* x, const float* dy, const float* w, float* dx, float* dw, int32_t N, int32_t C, int32_t H, int32_t W, float scale,
                       void* stream) {
  if (!x || !dy || !w || !dx || !dw) { t_err = "csnet_train_dw_bwd: null argument"; return CSNET_E_INVALID; }
  const int quads = (W + 3) / 4, rows = H < 8 ? H : 8, bands = (H + rows - 1) / rows;
  const size_t tasks = (size_t)N * bands * quads;
  int bx = (int)((tasks + tf::kT - 1) / tf::kT), cap = 8 * num_sms() / C;
  cap = cap < 1 ? 1 : cap;
  bx = bx > cap ? cap : bx;
  float* part = nullptr;
  if (int rc = partial_workspace((size_t)bx * C * 9, (cudaStream_t)stream, &part)) return rc;
  tf::dw3_bwd_kernel<<<dim3(bx, C), tf::kT, 0, (cudaStream_t)stream>>>(x, dy, w, dx, part, N, C, H, W, scale, quads, rows);
  TR_CHECK(cudaGetLastError());
  tf::reduce_partials_kernel<<<(C * 9 + tf::kT - 1) / tf::kT, tf::kT, 0, (cudaStream_t)stream>>>(part, bx, C * 9, scale, dw);
  TR_CHECK(cudaGetLastError());
  return CSNET_OK;
}

int csnet_train_mix_fwd(float* dst, int32_t N, int32_t C, int32_t H, int32_t W, const csnet_train_path* paths, int32_t n_paths, void* stream) {
  if (n_paths < 1 || n_paths > CSNET_MAX_PATHS) { t_err = "csnet_train_mix_fwd: n_paths"; return CSNET_E_INVALID; }
  csnet::MixArgs A{};
  A.dst = dst; A.bias = nullptr; A.slope = nullptr; A.dtype = CSNET_F32; A.C = C; A.H = H; A.W = W; A.n_paths = n_paths;
  for (int p = 0; p < n_paths; ++p) A.p[p] = to_path(paths[p]);
  // every conv path dense with one kernel size, every other path a bilinear resample-add: the register-tiled kernel
  tf::ConvArgs F{};
  F.dst = dst; F.N = N; F.C = C; F.H = H; F.W = W; F.ksize = 1;
  bool ok = conv_tile_geometry(F);
  int ks = 0;
  for (int p = 0; p < n_paths && ok; ++p) {
    const csnet::MixPath& P = A.p[p];
    if (P.ksize == 0) {
      if (F.n_rs >= tf::kMaxRs || P.up < 2 || P.pre_avg || P.pool != 1 || P.H * P.up != H || P.W * P.up != W) { ok = false; break; }
      tf::RsPath& Q = F.rs[F.n_rs++];
      Q.src = reinterpret_cast<const float*>(P.src); Q.Cs = P.C; Q.c0 = P.c0; Q.Hs = P.H; Q.Ws = P.W; Q.up = P.up; Q.cout0 = P.cout0; Q.cout = P.cout;
    } else {
      if (F.n_conv >= tf::kMaxConv || !dense_conv_path(P, H, W) || (ks && ks != P.ksize)) { ok = false; break; }
      ks = P.ksize;
      tf::ConvPath& Q = F.p[F.n_conv++];
      Q.src = reinterpret_cast<const float*>(P.src); Q.w = P.w; Q.Cs = P.C; Q.c0 = P.c0; Q.cin = P.cin; Q.cout0 = P.cout0; Q.cout = P.cout; Q.dil = P.dil;
    }
  }
  if (ok) {
    F.ksize = ks ? ks : 1;
    for (int i = 0; i < F.n_conv && ok; ++i) ok = conv_path_geometry(F.p[i], F, sizeof(float));
  }
  if (ok) {
    const int rc = launch_conv(F, (cudaStream_t)stream);
    if (rc != kNotHandled) return rc;
  }
  tr_mix_fwd_kernel<<<dim3((H * W + kT - 1) / kT, (C + csnet::kMixCT - 1) / csnet::kMixCT, N), kT, 0, (cudaStream_t)stream>>>(A);
  TR_CHECK(cudaGetLastError());
  return CSNET_OK;
}

int csnet_train_mix_dgrad(const float* ddst, int32_t N, int32_t C, int32_t H, int32_t W, const csnet_train_path* path, float* dsrc, void* stream) {
  const csnet::MixPath P = to_path(*path);
  if (P.pre_avg > 2 || P.up > 1 && P.ksize > 0) { t_err = "csnet_train_mix_dgrad: down-sample factors > 2 / input-side up-sampling are inference-only"; return CSNET_E_UNSUPPORTED; }
  if ((size_t)N * P.cin * P.H * P.W < (1ull << 32) && P.ksize == 0 && (P.up == 2 || P.up == 4) && !P.pre_avg && P.pool == 1 && P.H * P.up == H && P.W * P.up == W) {
    const size_t total = (size_t)N * P.cin * P.H * P.W;
    const unsigned blocks = (unsigned)((total + tf::kT - 1) / tf::kT);
    if (P.up == 2) tf::resample_bwd_kernel<2><<<blocks, tf::kT, 0, (cudaStream_t)stream>>>(ddst, N, C, H, W, P.cout0, P.cin, P.H, P.W, dsrc);
    else tf::resample_bwd_kernel<4><<<blocks, tf::kT, 0, (cudaStream_t)stream>>>(ddst, N, C, H, W, P.cout0, P.cin, P.H, P.W, dsrc);
    TR_CHECK(cudaGetLastError());
    return CSNET_OK;
  }
  if (dense_conv_path(P, H, W)) {
    tf::ConvArgs F{};
    F.dst = dsrc; F.N = N; F.C = P.cin; F.H = H; F.W = W; F.ksize = P.ksize; F.transposed = 1; F.n_conv = 1;
    tf::ConvPath& Q = F.p[0];
    Q.src = ddst; Q.w = P.w; Q.Cs = C; Q.c0 = P.cout0; Q.cin = P.cout; Q.cout0 = 0; Q.cout = P.cin; Q.dil = P.dil;
    if (conv_tile_geometry(F) && conv_path_geometry(Q, F, sizeof(float))) {
      const int rc = launch_conv(F, (cudaStream_t)stream);
      if (rc != kNotHandled) return rc;
    }
  }
  tr_mix_dgrad_kernel<<<dim3((P.H * P.W + kT - 1) / kT, P.cin, N), kT, 0, (cudaStream_t)stream>>>(ddst, C, H, W, P, dsrc);
  TR_CHECK(cudaGetLastError());
  return CSNET_OK;
}

int csnet_train_mix_wgrad(const float* ddst, int32_t N, int32_t C, int32_t H, int32_t W, const csnet_train_path* path, float* dw, void* stream) {
  const csnet::MixPath P = to_path(*path);
  if (P.ksize == 0) { t_err = "csnet_train_mix_wgrad: resample paths have no weights"; return CSNET_E_INVALID; }
  if (P.pre_avg > 2 || P.up > 1) { t_err = "csnet_train_mix_wgrad: down-sample factors > 2 / input-side up-sampling are inference-only"; return CSNET_E_UNSUPPORTED; }
  const int kk = P.ksize * P.ksize;
  WgradPlan G;
  if (wgrad_plan(P, ddst, N, C, H, W, sizeof(float), sizeof(float), G)) {
    float* part = nullptr;
    if (int rc = partial_workspace((size_t)G.gx * G.nel, (cudaStream_t)stream, &part)) return rc;
    G.A.part = part;
    static bool attr_dev[kMaxDevices] = {false};
    bool& attr = attr_dev[current_device()];
    if (!attr) {
      cudaFuncSetAttribute(tf::conv_wgrad_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, kFastSmemMax);
      cudaFuncSetAttribute(tf::conv_wgrad_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, kFastSmemMax);
      cudaFuncSetAttribute(tf::conv_wgrad_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, kFastSmemMax);
      attr = true;
    }
    const dim3 grid(G.gx, G.groups);
    if (G.form == 1) tf::conv_wgrad_kernel<1><<<grid, tf::kT, G.smem, (cudaStream_t)stream>>>(G.A);
    else if (G.form == 3) tf::conv_wgrad_kernel<3><<<grid, tf::kT, G.smem, (cudaStream_t)stream>>>(G.A);
    else tf::conv_wgrad_kernel<0><<<grid, tf::kT, G.smem, (cudaStream_t)stream>>>(G.A);
    TR_CHECK(cudaGetLastError());
    return reduce_partials(part, G.gx, G.nel, 1.f, dw, (cudaStream_t)stream);
  }
  TR_CHECK(cudaMemsetAsync(dw, 0, (size_t)P.cin * kk * P.cout * sizeof(float), (cudaStream_t)stream));
  const int split = N < 32 ? N : 32;
  tr_mix_wgrad_kernel<<<dim3(P.cin, kk * ((P.cout + 7) / 8), split), kT, 0, (cudaStream_t)stream>>>(ddst, N, C, H, W, P, dw);
  TR_CHECK(cudaGetLastError());
  return CSNET_OK;
}

int csnet_train_pool_fwd(const float* src, int32_t N, int32_t Cs, int32_t c0, int32_t cin, int32_t Hs, int32_t Ws, int32_t pre_avg, int32_t pool,
                         float* dst, uint8_t* idx, void* stream) {
  if (!src || !dst || pre_avg < 0 || pre_avg > 1 || pool < 1 || pool > 8 || (pool > 1 && !idx)) { t_err = "csnet_train_pool_fwd: bad arguments"; return CSNET_E_INVALID; }
  const int f = (pre_avg ? 2 : 1) * pool;
  const size_t total = (size_t)N * cin * (Hs / f) * (Ws / f);
  if (total == 0) return CSNET_OK;
  if (!pre_avg && pool == 2 && Ws % 4 == 0 && Hs % 2 == 0 && total < (1ull << 31))
    tf::pool2_fwd_kernel<<<(unsigned)((total / 2 + tf::kT - 1) / tf::kT), tf::kT, 0, (cudaStream_t)stream>>>(src, N, Cs, c0, cin, Hs, Ws, dst, idx);
  else
    tf::pool_fwd_kernel<<<(unsigned)((total + tf::kT - 1) / tf::kT), tf::kT, 0, (cudaStream_t)stream>>>(src, N, Cs, c0, cin, Hs, Ws, pre_avg, pool, dst, idx);
  TR_CHECK(cudaGetLastError());
  return CSNET_OK;
}

int csnet_train_pool_bwd(const float* dpool, const uint8_t* idx, int32_t N, int32_t cin, int32_t Hs, int32_t Ws, int32_t pre_avg, int32_t pool,
                         float* dsrc, void* stream) {
  if (!dpool || !dsrc || pre_avg < 0 || pre_avg > 1 || pool < 1 || pool > 8 || (pool > 1 && !idx)) { t_err = "csnet_train_pool_bwd: bad arguments"; return CSNET_E_INVALID; }
  const size_t total = (size_t)N * cin * Hs * Ws;
  if (total == 0) return CSNET_OK;
  if (Ws % 4 == 0 && total < (1ull << 32)) tf::pool_bwd4_kernel<<<(unsigned)((total / 4 + tf::kT - 1) / tf::kT), tf::kT, 0, (cudaStream_t)stream>>>(dpool, idx, N, cin, Hs, Ws, pre_avg, pool, dsrc);
  else tf::pool_bwd_kernel<<<(unsigned)((total + tf::kT - 1) / tf::kT), tf::kT, 0, (cudaStream_t)stream>>>(dpool, idx, N, cin, Hs, Ws, pre_avg, pool, dsrc);
  TR_CHECK(cudaGetLastError());
  return CSNET_OK;
}

int csnet_slim_gather(const float* src, int32_t Co, int32_t Ci, int32_t kk, const int64_t* out_idx, int32_t n_out, const int64_t* in_idx, int32_t n_in,
                      float* dst, int32_t dCo, int32_t dCi, void* stream) {
  if (!src || !dst || Co <= 0 || Ci <= 0 || kk <= 0 || n_out < 0 || n_in < 0 || n_out > dCo || n_in > dCi || (n_out > 0 && !out_idx) || (n_in > 0 && !in_idx)) {
    t_err = "csnet_slim_gather: bad arguments";
    return CSNET_E_INVALID;
  }
  const long long total = (long long)n_out * n_in * kk;
  if (total == 0) return CSNET_OK;
  slim_gather_kernel<<<(unsigned)((total + kT - 1) / kT), kT, 0, (cudaStream_t)stream>>>(src, Co, Ci, kk, reinterpret_cast<const long long*>(out_idx), n_out,
                                                                                      reinterpret_cast<const long long*>(in_idx), n_in, dst, dCi);
  TR_CHECK(cudaGetLastError());
  return CSNET_OK;
}

int csnet_train_bce(const float* logits, const float* target, float* dlogits, float* loss, int64_t n, float grad_scale, void* stream) {
  TR_CHECK(cudaMemsetAsync(loss, 0, sizeof(float), (cudaStream_t)stream));
  const int blocks = (int)((n + kT * 8 - 1) / (kT * 8) < 1184 ? (n + kT * 8 - 1) / (kT * 8) : 1184);
  bce_kernel<<<blocks < 1 ? 1 : blocks, kT, 0, (cudaStream_t)stream>>>(logits, target, dlogits, loss, n, 1.f / (float)n, grad_scale);
  TR_CHECK(cudaGetLastError());
  return CSNET_OK;
}

int csnet_train_bce_sum(const float* logits, const float* target, float* dlogits, float* loss, int64_t n, int32_t divisor, void* stream) {
  if (!logits || !target || !loss || n < 1 || divisor < 1) { t_err = "csnet_train_bce_sum: bad arguments"; return CSNET_E_INVALID; }
  float* part = nullptr;
  if (int rc = partial_workspace((size_t)csnet::bce::blocks(n), (cudaStream_t)stream, &part)) return rc;
  csnet::bce::launch(logits, target, dlogits, part, loss, n, divisor, (cudaStream_t)stream);
  TR_CHECK(cudaGetLastError());
  return CSNET_OK;
}

int csnet_train_adam(const void* chunk_table_device, int32_t n_chunks, float lr, float beta1, float beta2, float eps, int32_t step,
                     float grad_scale, void* stream) {
  const float bc1 = 1.f - powf(beta1, (float)step), bc2 = 1.f - powf(beta2, (float)step);
  adam_kernel<<<n_chunks, kT, 0, (cudaStream_t)stream>>>(reinterpret_cast<const AdamChunk*>(chunk_table_device), lr, beta1, beta2,
                                                        eps, bc1, sqrtf(bc2), grad_scale);
  TR_CHECK(cudaGetLastError());
  return CSNET_OK;
}

int csnet_salmetric_hist(const float* prob, const uint8_t* gt, int32_t N, int64_t HW, uint32_t* hist_all, uint32_t* hist_pos,
                         unsigned long long* abs_sum, void* stream) {
  if (!prob || !gt || !hist_all || !hist_pos || !abs_sum || N <= 0 || HW <= 0) { t_err = "csnet_salmetric_hist: bad arguments"; return CSNET_E_INVALID; }
  static_assert(kT == 256, "one histogram bin per thread");
  cudaStream_t st = (cudaStream_t)stream;
  TR_CHECK(cudaMemsetAsync(hist_all, 0, (size_t)N * 256 * sizeof(uint32_t), st));
  TR_CHECK(cudaMemsetAsync(hist_pos, 0, (size_t)N * 256 * sizeof(uint32_t), st));
  TR_CHECK(cudaMemsetAsync(abs_sum, 0, (size_t)N * sizeof(unsigned long long), st));
  const int64_t want = (HW + kT * 16 - 1) / (kT * 16);
  const int bx = (int)(want < 1 ? 1 : (want > 64 ? 64 : want));
  salmetric_hist_kernel<<<dim3(bx, N), kT, 0, st>>>(prob, gt, HW, hist_all, hist_pos, abs_sum);
  TR_CHECK(cudaGetLastError());
  return CSNET_OK;
}

}  // extern "C"
