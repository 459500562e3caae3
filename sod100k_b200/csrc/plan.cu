// plan.cu — C ABI (include/csnet_b200.h) and the program executor of libcsnet_b200.so.
//
// A plan holds: the validated program, the device copy of the parameter blob, and one activation arena.
// csnet_plan_run() walks the op list and launches one fused kernel per op on the caller's stream.
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cstdint>
#include <new>
#include <string>
#include <vector>

#include "../../include/csnet_b200.h"
#include "generic_ops.cuh"
#include "il_block.cuh"
#include "il_stream.cuh"
#include "mix_stream.cuh"
#include "ms_direct.cuh"
#include "mix_tc.cuh"
#include "dw_fast.cuh"
#include "image_io.cuh"
#include "resize.cuh"
#include "resize_adj.cuh"

namespace {

thread_local std::string g_err;

int fail(int code, const std::string& msg) {
  g_err = msg;
  return code;
}

#define CU_CHECK(expr)                                                                         \
  do {                                                                                         \
    cudaError_t e_ = (expr);                                                                   \
    if (e_ != cudaSuccess)                                                                     \
      return fail(CSNET_E_CUDA, std::string(#expr) + ": " + cudaGetErrorString(e_));           \
  } while (0)

size_t dtype_size(int dt) { return dt == CSNET_F32 ? 4 : 2; }

// The entry points select the plan's device for their CUDA calls and put the caller's current device back on return:
// torch (the host side's plumbing) keeps its own notion of the current device.
struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(int dev) {
    if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
    if (prev != dev) cudaSetDevice(dev);
    else prev = -1;
  }
  ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

// ------------------------------------------------------------------------------------------------
// kernels
// ------------------------------------------------------------------------------------------------
constexpr int kThreads = 256;

__global__ void __launch_bounds__(kThreads, 2) mix_generic_kernel(const __grid_constant__ csnet::MixArgs A) {
  __shared__ float ws[csnet::kMixStageFloats];
  const int co_base = blockIdx.y * csnet::kMixCT, n = blockIdx.z;
  const int pix = blockIdx.x * kThreads + threadIdx.x;
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
      csnet::mix_stage_chunk(P, co_base, ci0, ci1, ws, threadIdx.x, kThreads);
      __syncthreads();
      if (live) csnet::mix_acc_chunk(P, ws, ci0, ci1, n, oy, ox, acc);
    }
  }
  if (live) csnet::mix_finish(A, n, oy, ox, co_base, acc);
}

__global__ void __launch_bounds__(kThreads) dw_generic_kernel(const __grid_constant__ csnet::DwArgs A) {
  const int item = blockIdx.x * kThreads + threadIdx.x;
  const int strips = (A.H + csnet::kDwRows - 1) / csnet::kDwRows;
  if (item >= strips * A.W) return;
  csnet::dw_thread(A, blockIdx.z, blockIdx.y, (item / A.W) * csnet::kDwRows, item % A.W);
}

// GroupNorm statistics: one CTA per (group, image)
__global__ void __launch_bounds__(kThreads) gn_stats_kernel(const __grid_constant__ csnet::GnArgs A) {
  const int g = blockIdx.x, n = blockIdx.y, cpg = A.C / A.groups;
  const int64_t base = ((int64_t)n * A.C + (int64_t)g * cpg) * A.HW, cnt = (int64_t)cpg * A.HW;
  __shared__ float sh[2][kThreads / 32];
  __shared__ float mu_s;
  float s = 0.f;
  for (int64_t i = threadIdx.x; i < cnt; i += kThreads) s += csnet::ld_elem(A.src, A.src_dtype, base + i);
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) sh[0][threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < kThreads / 32; ++i) t += sh[0][i];
    mu_s = t / (float)cnt;
  }
  __syncthreads();
  const float mu = mu_s;
  float q = 0.f;
  for (int64_t i = threadIdx.x; i < cnt; i += kThreads) {
    const float d = csnet::ld_elem(A.src, A.src_dtype, base + i) - mu;
    q += d * d;
  }
  for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  if ((threadIdx.x & 31) == 0) sh[1][threadIdx.x >> 5] = q;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < kThreads / 32; ++i) t += sh[1][i];
    A.stats[((int64_t)n * A.groups + g) * 2] = mu;
    A.stats[((int64_t)n * A.groups + g) * 2 + 1] = rsqrtf(t / (float)cnt + 1e-5f);
  }
}

__global__ void __launch_bounds__(kThreads) gn_apply_kernel(const __grid_constant__ csnet::GnArgs A) {
  const int c = blockIdx.y, n = blockIdx.z, g = c / (A.C / A.groups);
  const float mu = A.stats[((int64_t)n * A.groups + g) * 2], r = A.stats[((int64_t)n * A.groups + g) * 2 + 1];
  const float ga = A.gamma[c] * r, be = A.beta[c] - mu * ga;
  const bool has_slope = A.slope != nullptr;
  const float sl = has_slope ? A.slope[c] : 1.f;
  const int64_t base = ((int64_t)n * A.C + c) * A.HW;
  for (int i = blockIdx.x * kThreads + threadIdx.x; i < A.HW; i += gridDim.x * kThreads) {
    float v = csnet::ld_elem(A.src, A.src_dtype, base + i) * ga + be;
    if (has_slope) v = v > 0.f ? v : sl * v;
    csnet::st_elem(A.dst, A.dst_dtype, base + i, v);
  }
}

// Device-side pre / post-processing of CSNet/test.py:68-69,86-96 (SURVEY §8 f3): uint8 HWC image -> (x / 255 - mean) / std as the
// fp32 NCHW network input (the reference computes it in float64 on the host and rounds to fp32: same here), and
// sigmoid(logit) * 255 -> uint8 (astype truncation) of the saliency map.
struct PreArgs { double mean[3], std[3]; };
__global__ void __launch_bounds__(kThreads) pre_u8_kernel(const uint8_t* __restrict__ x, float* __restrict__ y, int64_t npix, int64_t hw, const __grid_constant__ PreArgs A) {
  const int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x;          // pixel over (n, h, w)
  if (i >= npix) return;
  const int64_t n = i / hw, p = i - n * hw;
#pragma unroll
  for (int c = 0; c < 3; ++c) y[(n * 3 + c) * hw + p] = (float)(((double)x[i * 3 + c] / 255.0 - A.mean[c]) / A.std[c]);
}
__global__ void __launch_bounds__(kThreads) post_u8_kernel(const float* __restrict__ z, uint8_t* __restrict__ y, int64_t n) {
  const int64_t i = ((int64_t)blockIdx.x * kThreads + threadIdx.x) * 4;
  if (i >= n) return;
  uchar4 o;
  const float4 v = *reinterpret_cast<const float4*>(z + i);                // n % 4 == 0 (W % 16 == 0)
  o.x = (unsigned char)((1.f / (1.f + expf(-v.x))) * 255.f); o.y = (unsigned char)((1.f / (1.f + expf(-v.y))) * 255.f);
  o.z = (unsigned char)((1.f / (1.f + expf(-v.z))) * 255.f); o.w = (unsigned char)((1.f / (1.f + expf(-v.w))) * 255.f);
  *reinterpret_cast<uchar4*>(y + i) = o;
}

}  // namespace

// ------------------------------------------------------------------------------------------------
// plan
// ------------------------------------------------------------------------------------------------
struct TcChoice {
  int mt = 0;            // 0: generic kernel; else number of m16 tiles of the tensor-core kernel
  int dtype = 0;         // CSNET_F16 / CSNET_BF16 operand type
  int xs_halves = 0;
  int rows = 1;          // output rows per warp of mix_tc (tile height 8 * rows)
  int kc = 8;            // input channels per staged chunk
  int kk = 1;            // largest tap count among the conv paths
};

// The kernel (family) launch_op() runs for an op, chosen once per op when the plan is created (choose_kernel).
enum class Kern : uint8_t { Msd, MixStream, MixTc, Pool2, Upsample, Resample, MixGeneric, Gn, IlStream, IlBlock, DwFast, DwGeneric, Resize };

// Small batches of a two-external plan up to this size replay a captured graph (csnet_plan_run).
constexpr int kGraphMaxN = 8;

size_t tc_smem_bytes(const TcChoice& c) {
  return ((size_t)c.kc * c.xs_halves + (size_t)c.kk * c.mt * 16 * (c.kc + 8)) * 2;
}

using IlKernel = void (*)(csnet::IlArgs);
using TcKernel = void (*)(csnet::MixArgs, csnet::TcGeom);

// How launch_op() runs one op: the kernel chosen for it and every kernel argument that does not depend on the call, planned
// when the plan is created (the epilogue tables when the blob is set).  launch_op() binds the activation addresses, the batch
// and the tensor maps.  A streaming record stays zero when its kernel cannot take the op.
struct OpLaunch {
  Kern kern = Kern::MixGeneric;
  TcChoice tc;                                    // MIX ops: mt > 0 if the tensor-core kernel can take the op
  csnet::MsArgs ms{};                             // MIX ops: the streaming kernel's arguments (n_in > 0 if it can take the op)
  csnet::IlArgs il{};                             // ILBLOCK ops: the tiled kernel's arguments with the tile chosen
  csnet::IlsArgs ils{};                           // ILBLOCK ops: the streaming kernel's arguments (ns > 0 if it can take the op)
  size_t smem = 0;                                // MixTc / IlBlock: dynamic shared memory of a launch
  TcKernel tc_fn = nullptr;                       // MixTc: the mix_tc_kernel instantiation
  IlKernel il_fn = nullptr;                       // IlBlock: the il_block_kernel instantiation
  uint16_t* w16[CSNET_MAX_PATHS] = {};            // MixTc: per path, packed 16-bit weights (device)
};

struct csnet_plan {
  int device = 0;
  int max_batch = 0;
  std::vector<csnet_tensor_desc> tensors;
  std::vector<csnet_op_desc> ops;
  int64_t blob_floats = 0;
  float* blob = nullptr;
  char* arena = nullptr;
  int64_t arena_per_image = 0;   // bytes
  int n_ext = 0;
  std::vector<OpLaunch> launch;                   // per op
  // small-batch replay: the whole op list captured once per batch size into a CUDA graph over plan-owned input / output staging
  // (CSNet/test.py calls the model one image at a time: ~80 launches per forward are launch-bound there)
  struct GraphSlot { cudaGraphExec_t exec = nullptr; void* in = nullptr; void* out = nullptr; size_t in_bytes = 0, out_bytes = 0; };
  std::vector<GraphSlot> graphs;                  // index = batch size
  cudaStream_t cap_stream = nullptr;
  bool ms_enabled = true;                         // CSNET_MS=0 at plan creation: mix_tc / generic kernels only
  int num_sms = 132;
  int ils_force_ns = 0;                           // CSNET_ILS_NS=k: force k column strips (0: automatic)
  bool ils_enabled = true;                        // CSNET_ILS=0 at plan creation: tiled kernel only
  int ils_min_chunks = 592;                       // batches with fewer 4-row chunks per ILBlock run the tiled kernel
  // host-buffer pipeline (csnet_plan_run_host): copy streams, ping-pong staging, ordering events
  cudaStream_t s_h2d = nullptr, s_d2h = nullptr;
  void* h_in8[2] = {nullptr, nullptr};             // uint8 staging of csnet_plan_run_host_u8 / _images_u8
  void* h_out8[2] = {nullptr, nullptr};
  size_t h_in8_bytes = 0, h_out8_bytes = 0;
  csnet_image_geom* h_geom = nullptr;              // csnet_plan_run_host_images_u8: the batch's geometry, rebased per chunk
  int32_t h_geom_n = 0;
  void* h_in[2] = {nullptr, nullptr};
  void* h_out[2] = {nullptr, nullptr};
  size_t h_in_bytes = 0, h_out_bytes = 0;
  cudaEvent_t ev_h2d[2] = {nullptr, nullptr}, ev_comp[2] = {nullptr, nullptr}, ev_d2h[2] = {nullptr, nullptr};
  float* gn_stats = nullptr;      // [max_batch][max groups][2] scratch of the GroupNorm ops
  int gn_groups_max = 0;

  void* tensor_ptr(int t, int N, const void* const* ext) const {
    const csnet_tensor_desc& d = tensors[t];
    if (d.external >= 0) return ext ? const_cast<void*>(ext[d.external]) : nullptr;
    return arena + (int64_t)N * d.arena_offset;
  }
};

namespace {

// Channels of a MIX-kind op's result: the destination's, or ext_off[2] when a projection consumes it in the epilogue.
static inline int mix_channels(const csnet_plan& P, const csnet_op_desc& op) {
  return op.kind == CSNET_OP_MIXPROJ ? (int)op.ext_off[2] : P.tensors[op.dst].C;
}

int validate(const csnet_plan& P) {
  const int nt = (int)P.tensors.size();
  char buf[256];
  for (int t = 0; t < nt; ++t) {
    const csnet_tensor_desc& d = P.tensors[t];
    if (d.C <= 0 || d.H <= 0 || d.W <= 0 || d.dtype < 0 || d.dtype > 2) {
      snprintf(buf, sizeof buf, "tensor %d: bad dims/dtype", t);
      return fail(CSNET_E_INVALID, buf);
    }
    if (d.external < 0 && (d.arena_offset < 0 || d.arena_offset % 256 != 0)) {
      snprintf(buf, sizeof buf, "tensor %d: arena offset must be a non-negative multiple of 256", t);
      return fail(CSNET_E_INVALID, buf);
    }
  }
  for (size_t i = 0; i < P.ops.size(); ++i) {
    const csnet_op_desc& op = P.ops[i];
    auto bad = [&](const char* why) {
      snprintf(buf, sizeof buf, "op %zu: %s", i, why);
      return fail(CSNET_E_INVALID, buf);
    };
    if (op.kind != CSNET_OP_MIX && op.kind != CSNET_OP_DW && op.kind != CSNET_OP_ILBLOCK && op.kind != CSNET_OP_GN &&
        op.kind != CSNET_OP_MIXPROJ && op.kind != CSNET_OP_RESIZE)
      return bad("unknown kind");
    if (op.dst < 0 || op.dst >= nt) return bad("dst out of range");
    if (op.kind == CSNET_OP_RESIZE) {
      if (op.n_paths != 1) return bad("RESIZE takes one path");
      if (op.dst2 != -1 || op.bias_off != -1 || op.slope_off != -1) return bad("RESIZE has no second destination, bias or slope");
      if (op.ext_off[0] != 0 && op.ext_off[0] != 1) return bad("RESIZE accumulate flag (ext_off[0]) must be 0 or 1");
      for (int e = 1; e < CSNET_MAX_EXT; ++e)
        if (op.ext_off[e] != -1) return bad("RESIZE uses ext_off[0] only");
      const csnet_path_desc& q = op.paths[0];
      if (q.src < 0 || q.src >= nt) return bad("path src out of range");
      if (q.src == op.dst) return bad("in-place op");
      const csnet_tensor_desc &S = P.tensors[q.src], &D = P.tensors[op.dst];
      if (q.ksize != 0 || q.cin != q.cout) return bad("RESIZE path: ksize 0, cin == cout");
      if (q.c0 < 0 || q.cin <= 0 || q.c0 + q.cin > S.C) return bad("path input channel slice");
      if (q.cout0 < 0 || q.cout0 + q.cout > D.C) return bad("path output channel slice");
      for (int v : {q.pre_avg, q.pool, q.dil, q.stride, q.pad, q.up})
        if (v != 0 && v != 1) return bad("RESIZE path: pre_avg, pool, dil, stride, pad and up must be 0 or 1");
      if (q.w_off != -1) return bad("RESIZE path has no weights (w_off -1)");
      continue;
    }
    if (op.kind == CSNET_OP_GN) {
      if (op.n_paths != 1) return bad("GN takes one input");
      const int a = op.paths[0].src, groups = op.paths[0].up;
      if (a < 0 || a >= nt || a == op.dst) return bad("GN input");
      const csnet_tensor_desc &X = P.tensors[a], &Y = P.tensors[op.dst];
      if (X.C != Y.C || X.H != Y.H || X.W != Y.W) return bad("GN shape");
      if (groups < 1 || X.C % groups) return bad("GN groups must divide the channels");
      if (op.ext_off[0] < 0 || op.ext_off[0] + X.C > P.blob_floats || op.ext_off[1] < 0 || op.ext_off[1] + X.C > P.blob_floats)
        return bad("GN gamma/beta outside blob");
      if (op.slope_off >= 0 && op.slope_off + X.C > P.blob_floats) return bad("slope outside blob");
      continue;
    }
    if (op.kind == CSNET_OP_ILBLOCK) {
      if (op.n_paths != 2) return bad("ILBLOCK takes two inputs");
      if (op.dst2 >= nt) return bad("dst2 out of range");
      const csnet_tensor_desc& Yh = P.tensors[op.dst];
      const int a = op.paths[0].src, b = op.paths[1].src;
      if (a < 0 || a >= nt || b < 0 || b >= nt) return bad("ILBLOCK input out of range");
      const csnet_tensor_desc &Xh = P.tensors[a], &Xl = P.tensors[b];
      if (a == op.dst || b == op.dst || a == op.dst2 || b == op.dst2) return bad("in-place op");
      const bool stem = op.paths[0].ksize == 3;          // stem form: both branches are 3x3 convs of one fp32 image
      if (Yh.dtype == CSNET_F32) return bad("ILBLOCK needs a 16-bit destination");
      if (Yh.W % 8 || Yh.H % 2) return bad("ILBLOCK needs W % 8 == 0 and H % 2 == 0");
      if (stem) {
        if (a != b || Xh.dtype != CSNET_F32 || Xh.C * 9 > 32) return bad("ILBLOCK stem form takes one fp32 image of at most 3 channels");
        if (Xh.H != Yh.H || Xh.W != Yh.W) return bad("ILBLOCK input/output resolutions");
        if (op.paths[1].ksize != 3 || op.paths[1].pool != 2) return bad("ILBLOCK stem form: lo path is a 3x3 conv of the 2x2 max-pool");
      } else {
        if (Xh.dtype != Yh.dtype || Xl.dtype != Yh.dtype) return bad("ILBLOCK needs one 16-bit dtype");
        if (Xh.H != Yh.H || Xh.W != Yh.W || Xl.H * 2 != Xh.H || Xl.W * 2 != Xh.W) return bad("ILBLOCK input/output resolutions");
      }
      if (op.paths[0].cin != Xh.C || op.paths[1].cin != Xl.C) return bad("ILBLOCK consumes whole input tensors");
      int Clo = 0;
      if (op.dst2 >= 0) {
        const csnet_tensor_desc& Yl = P.tensors[op.dst2];
        if (Yl.dtype != Yh.dtype || Yl.H * 2 != Yh.H || Yl.W * 2 != Yh.W) return bad("ILBLOCK lo output shape");
        Clo = Yl.C;
      }
      const int nreq = Clo > 0 ? 18 : 15;
      for (int e = 0; e < nreq; ++e) {
        if (Clo == 0 && (e == 4 || e == 5 || (e >= 9 && e <= 11))) continue;
        if (op.ext_off[e] < 0 || op.ext_off[e] >= P.blob_floats) return bad("ILBLOCK parameter offset outside blob");
      }
      continue;
    }
    if (op.n_paths < 1 || op.n_paths > CSNET_MAX_PATHS) return bad("n_paths out of range");
    const csnet_tensor_desc& D = P.tensors[op.dst];
    const int Cm = mix_channels(P, op);               // channels of the MIX result (== D.C unless projected away)
    if (op.kind == CSNET_OP_MIXPROJ) {
      if (D.C != 1 || Cm < 1 || Cm > 80) return bad("MIXPROJ projects 1..80 channels onto one");
      if (op.ext_off[0] < 0 || op.ext_off[0] + Cm > P.blob_floats) return bad("projection weights outside blob");
      if (op.ext_off[1] >= P.blob_floats) return bad("projection bias outside blob");
    }
    if (op.bias_off >= 0 && op.bias_off + Cm > P.blob_floats) return bad("bias outside blob");
    if (op.slope_off >= 0 && op.slope_off + Cm > P.blob_floats) return bad("slope outside blob");
    if (op.kind == CSNET_OP_DW && op.n_paths != 1) return bad("DW takes one path");
    for (int p = 0; p < op.n_paths; ++p) {
      const csnet_path_desc& q = op.paths[p];
      if (q.src < 0 || q.src >= nt) return bad("path src out of range");
      if (q.src == op.dst) return bad("in-place op");
      const csnet_tensor_desc& S = P.tensors[q.src];
      if (q.c0 < 0 || q.cin <= 0 || q.c0 + q.cin > S.C) return bad("path input channel slice");
      if (q.cout0 < 0 || q.cout <= 0 || q.cout0 + q.cout > Cm) return bad("path output channel slice");
      if (op.kind == CSNET_OP_DW) {
        if (q.ksize != 3 || q.dil != 1 || q.pad != 1 || q.stride != 1 || q.pre_avg || q.pool != 1 || q.up != 1)
          return bad("DW must be 3x3 pad 1");
        if (q.cin != D.C || q.cout != D.C || q.c0 != 0 || q.cout0 != 0 || S.C != D.C || S.H != D.H || S.W != D.W)
          return bad("DW shape");
        if (q.w_off < 0 || q.w_off + (int64_t)D.C * 9 > P.blob_floats) return bad("DW weights outside blob");
        continue;
      }
      if (q.ksize == 0) {
        if (q.up < 1 || q.cin != q.cout || q.pool < 1) return bad("resample path");
        if (q.pre_avg != 0 && q.pre_avg != 1 && q.pre_avg != 2 && q.pre_avg != 4 && q.pre_avg != 8) return bad("pre_avg must be 0, 1, 2, 4 or 8");
        const int div = csnet::pre_factor(q.pre_avg) * q.pool;
        if (div > 1 && q.up != 1) return bad("a resample path either up-samples or down-samples");
        if (S.H % div || S.W % div) return bad("pooling does not divide the source");
        if (S.H / div * q.up != D.H || S.W / div * q.up != D.W) return bad("resample path size");
      } else {
        if (q.ksize != 1 && q.ksize != 3) return bad("ksize must be 1 or 3");
        if (q.up < 1) return bad("conv path up < 1");
        if (q.up > 1 && (q.ksize != 1 || q.pool != 1 || q.pre_avg || q.stride != 1 || q.pad != 0))
          return bad("input-side up-sampling is only defined for plain 1x1 conv paths");
        if (q.pool < 1 || q.stride < 1 || q.dil < 1 || q.pad < 0) return bad("conv path params");
        if (q.pre_avg != 0 && q.pre_avg != 1 && q.pre_avg != 2 && q.pre_avg != 4 && q.pre_avg != 8) return bad("pre_avg must be 0, 1, 2, 4 or 8");
        const int div = csnet::pre_factor(q.pre_avg) * q.pool;
        if (S.H % div || S.W % div) return bad("pooling does not divide the source");
        const int Hc = q.up > 1 ? S.H * q.up : S.H / div, Wc = q.up > 1 ? S.W * q.up : S.W / div;
        const int Ho = (Hc + 2 * q.pad - q.dil * (q.ksize - 1) - 1) / q.stride + 1;
        const int Wo = (Wc + 2 * q.pad - q.dil * (q.ksize - 1) - 1) / q.stride + 1;
        if (Ho != D.H || Wo != D.W) return bad("conv path output size != dst");
        const int64_t nw = (int64_t)q.cout * q.cin * q.ksize * q.ksize;
        if (q.w_off < 0 || q.w_off + nw > P.blob_floats) return bad("weights outside blob");
      }
    }
  }
  return CSNET_OK;
}

csnet::MixArgs make_mix(const csnet_plan& P, const csnet_op_desc& op, int N, const void* const* ext) {
  csnet::MixArgs A{};
  const csnet_tensor_desc& D = P.tensors[op.dst];
  A.dst = P.tensor_ptr(op.dst, N, ext);
  A.bias = op.bias_off >= 0 ? P.blob + op.bias_off : nullptr;
  A.slope = op.slope_off >= 0 ? P.blob + op.slope_off : nullptr;
  A.dtype = D.dtype; A.C = mix_channels(P, op); A.H = D.H; A.W = D.W;
  A.n_paths = op.n_paths;
  if (op.kind == CSNET_OP_MIXPROJ) {
    A.proj_w = P.blob + op.ext_off[0];
    A.proj_b = op.ext_off[1] >= 0 ? P.blob + op.ext_off[1] : nullptr;
  }
  for (int p = 0; p < op.n_paths; ++p) {
    const csnet_path_desc& q = op.paths[p];
    const csnet_tensor_desc& S = P.tensors[q.src];
    csnet::MixPath& m = A.p[p];
    m.src = P.tensor_ptr(q.src, N, ext);
    m.w = q.ksize > 0 ? P.blob + q.w_off : nullptr;
    m.dtype = S.dtype; m.C = S.C; m.H = S.H; m.W = S.W;
    m.c0 = q.c0; m.cin = q.cin; m.pre_avg = q.pre_avg; m.pool = q.pool;
    m.ksize = q.ksize; m.dil = q.dil; m.stride = q.stride; m.pad = q.pad; m.up = q.up;
    m.cout0 = q.cout0; m.cout = q.cout;
  }
  return A;
}

int round_up(int v, int m) { return (v + m - 1) / m * m; }

int padded_region(int n) {
  int np = round_up(n, 8);
  if (((np >> 3) & 1) == 0) np += 8;      // NP/8 odd: the 8 rows of an ldmatrix hit 8 distinct 16-byte bank groups
  return np;
}

// cuTensorMapEncodeTiled comes from the driver; resolve it through the runtime so the library links against
// cudart only.
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn encode_tiled_fn() {
  static EncodeTiledFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      p = nullptr;
    return reinterpret_cast<EncodeTiledFn>(p);
  }();
  return fn;
}

// Kernel arguments of a fused ILBlock op on the tiled kernel, but for the activation addresses (bound at launch), and its
// tile; false if no tile fits shared memory.
bool plan_il(const csnet_plan& P, const csnet_op_desc& op, csnet::IlArgs* out) {
  csnet::IlArgs A{};
  const csnet_tensor_desc &Xh = P.tensors[op.paths[0].src], &Xl = P.tensors[op.paths[1].src], &Yh = P.tensors[op.dst];
  A.H = Yh.H; A.W = Yh.W;
  A.Chi = Xh.C; A.Cli = Xl.C; A.Cho = Yh.C; A.Clo = op.dst2 >= 0 ? P.tensors[op.dst2].C : 0;
  A.first = op.paths[0].ksize == 3;
  if (A.first) { A.Chi = Xh.C * 9; A.Cli = 0; }   // im2col rows of the image; no lo input tensor
  auto f = [&](int e) { return op.ext_off[e] >= 0 ? P.blob + op.ext_off[e] : nullptr; };
  A.wh = reinterpret_cast<const uint32_t*>(f(0));
  A.wl = reinterpret_cast<const uint32_t*>(f(1));
  A.bias_h = f(2); A.slope_h = f(3); A.bias_l = f(4); A.slope_l = f(5);
  A.dw1h = {f(6), f(7), f(8)};   A.dw1l = {f(9), f(10), f(11)};
  A.dw2h = {f(12), f(13), f(14)}; A.dw2l = {f(15), f(16), f(17)};
  A.K8 = round_up(A.Chi + A.Cli, 8);
  if (A.K8 > 8 * csnet::kIlMaxK8) return false;
  A.MH16 = round_up(A.Cho, 16);
  A.ML16 = A.Clo > 0 ? round_up(A.Clo, 16) : 0;
  A.rowsAh = A.K8 > A.Cho ? A.K8 : A.Cho;
  A.rowsAl = A.Clo > 0 ? (A.K8 > A.Clo ? A.K8 : A.Clo) : A.Cli;
  static const int cand[][2] = {{32, 32}, {28, 32}, {16, 64}, {16, 32}, {8, 16}};   // the instantiated tile geometries
  double best = -1;
  for (int chunked = 0; chunked < 2; ++chunked) {
    for (auto& c : cand) {
      csnet::IlArgs T = A;
      T.TH = c[0]; T.TW = c[1];
      T.t2h = chunked ? 8 : A.Cho;                       // chunked: the depthwise tail runs 8 hi channels at a time
      if (chunked && A.Cho <= 8) continue;
      const int NPH = ((T.TH + 8) | 1) * (T.TW + 8), NPL = ((T.TH / 2 + 4) | 1) * (T.TW / 2 + 8);
      if (csnet::il_smem_bytes(T, NPH, NPL) > 227 * 1024) continue;
      // stem form: the fp32 image tile is staged in the T2 buffers before they are needed
      if (A.first && (size_t)Xh.C * (T.TH + 12) * (T.TW + 24) * 4 > ((size_t)T.t2h * NPH + (size_t)A.Clo * NPL) * 2) continue;
      const int ty = (A.H + T.TH - 1) / T.TH, tx = (A.W + T.TW - 1) / T.TW;
      const double cost = (double)ty * tx * NPH * (chunked ? 1.15 : 1.0);   // halo work, small penalty for the extra barriers
      if (best < 0 || cost < best) { best = cost; T.tiles_x = tx; *out = T; }
    }
  }
  return best >= 0;
}

size_t il_smem_of(const csnet::IlArgs& A) {
  return csnet::il_smem_bytes(A, ((A.TH + 8) | 1) * (A.TW + 8), ((A.TH / 2 + 4) | 1) * (A.TW / 2 + 8));
}

// 5-D map over a planar [N][C][H][W] 16-bit tensor with W split into (W/8, 8): dims (8 px, C, W/8, H, N).  A box
// (8, slots, groups, rows, 1) lands in shared memory as [row][group][slot][8 px] — the tensor-core operand layout of
// il_stream.cuh; slots past C are zero-filled.
bool encode_group_map(CUtensorMap* tm, const void* base, int N, int C, int H, int W, int slots, int groups, int rows) {
  EncodeTiledFn fn = encode_tiled_fn();
  if (!fn) return false;
  const cuuint64_t dims[5] = {8, (cuuint64_t)C, (cuuint64_t)(W / 8), (cuuint64_t)H, (cuuint64_t)N};
  const cuuint64_t strides[4] = {(cuuint64_t)H * W * 2, 16, (cuuint64_t)W * 2, (cuuint64_t)C * H * W * 2};
  const cuuint32_t box[5] = {8, (cuuint32_t)slots, (cuuint32_t)groups, (cuuint32_t)rows, 1};
  const cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  return fn(tm, CU_TENSOR_MAP_DATA_TYPE_UINT16, 5, const_cast<void*>(base), dims, strides, box, estr,
            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// 4-D map over a planar fp32 tensor [N][C][H][W]: box (bw floats, rows, bc channels, 1) -> [c][row][bw] in shared memory,
// zeros outside.
bool encode_image_map(CUtensorMap* tm, const void* base, int N, int C, int H, int W, int bw, int rows, int bc) {
  EncodeTiledFn fn = encode_tiled_fn();
  if (!fn) return false;
  const cuuint64_t dims[4] = {(cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)C, (cuuint64_t)N};
  const cuuint64_t strides[3] = {(cuuint64_t)W * 4, (cuuint64_t)H * W * 4, (cuuint64_t)C * H * W * 4};
  const cuuint32_t box[4] = {(cuuint32_t)bw, (cuuint32_t)rows, (cuuint32_t)bc, 1};
  const cuuint32_t estr[4] = {1, 1, 1, 1};
  return fn(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<void*>(base), dims, strides, box, estr,
            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// Kernel arguments of an ILBlock op on the streaming kernel, but for the outputs, the batch and the epilogue tables; false if
// the op does not qualify (the tiled kernel runs it).  The parameter pointers are the tiled kernel's (`il`).
// Picks the column-strip split: the fewest strips that fit the thread / shared-memory limits.
bool plan_ils(const csnet_plan& P, const csnet_op_desc& op, const csnet::IlArgs& il, csnet::IlsArgs* out) {
  if (!P.ils_enabled || encode_tiled_fn() == nullptr) return false;
  const csnet_tensor_desc &Xh = P.tensors[op.paths[0].src], &Xl = P.tensors[op.paths[1].src], &Yh = P.tensors[op.dst];
  if (Yh.dtype != CSNET_F16) return false;
  const bool stem = op.paths[0].ksize == 3;                              // stem form: 3x3 convs of the fp32 image (im2col K = 9 Ci)
  csnet::IlsArgs A{};
  A.H = Yh.H; A.W = Yh.W;
  A.Chi = stem ? Xh.C * 9 : Xh.C; A.Cli = stem ? 0 : Xl.C; A.Cho = Yh.C; A.Clo = op.dst2 >= 0 ? P.tensors[op.dst2].C : 0;
  A.Ci = stem ? Xh.C : 0;
  if (stem && (Xh.dtype != CSNET_F32 || A.Chi > 32 || A.W % 4)) return false;
  if (A.W % 16 || A.H % 4 || A.Cho > csnet::kIlsMaxC || A.Clo > csnet::kIlsMaxC || A.Chi + A.Cli > 64) return false;
  A.K8 = stem ? 32 : round_up(A.Chi + A.Cli, 8);                      // the compiler packs the stem's weights as [M16][32]
  A.K16 = round_up(A.Chi + A.Cli, 16);
  A.NH = round_up(A.Cho, 16);
  A.NL = A.Clo > 0 ? round_up(A.Clo, 16) : 0;
  A.GH = A.W / 8; A.GL = A.W / 16;
  A.SH = (A.K16 > A.NH ? A.K16 : A.NH) + 1;            // odd: consecutive pixel groups start in different bank groups
  A.SL = A.Clo > 0 ? A.K16 + 1 : (A.Cli | 1);
  A.ST = A.NL + 1;
  A.cpi = A.H / 4;
  auto r128 = [](int v) { return (v + 127) / 128 * 128; };
  bool found = false;
  csnet::IlsArgs best{};
  for (int ns = 1; ns <= 16; ++ns) {
    if (P.ils_force_ns > 0 && ns != P.ils_force_ns) continue;
    if (A.GH % ns || (A.GH / ns) % 2) continue;
    csnet::IlsArgs T = A;
    T.ns = ns; T.gsn = A.GH / ns; T.hl = ns > 1 ? 1 : 0;
    T.GR = T.gsn + 2 * T.hl; T.GLR = T.gsn / 2 + 2 * T.hl;
    // tail tasks (a channel, two 8-pixel groups of a strip row) are packed: hi ones, then lo ones
    T.dw_warps = (T.Cho * (T.gsn / 2) + T.Clo * ((T.gsn / 2 + 1) / 2) + 31) / 32;
    if (T.dw_warps < 4) T.dw_warps = 4;                                   // the GEMM needs one warpgroup
    const int warps = T.dw_warps;
    if (warps * 32 > csnet::kIlsMaxThreads || T.SH > 256 || T.SL > 256 || T.GR > 256) continue;
    const int nbh = (4 * T.GR + 7) / 8, nbl = T.Clo > 0 ? (2 * T.GLR + 7) / 8 : 0;     // 64-pixel GEMM blocks of a chunk
    T.BW = 8 * T.GR + 8;                                                  // stem: image block row = the tile's pixels + 4 on each side
    if (stem && T.BW > 256) continue;
    T.lo_stage_bytes = stem ? r128(T.BW * 4 * T.Ci * 4) : r128(2 * T.GLR * T.SL * 16);
    T.hi_stage_bytes = r128(4 * T.GR * T.SH * 16);
    T.off_xl = 0;
    T.off_xh = csnet::kIlsLoStages * T.lo_stage_bytes;
    T.off_t1l = T.off_xh + csnet::kIlsHiStages * T.hi_stage_bytes;
    T.off_wbh = T.off_t1l + r128(2 * T.GLR * T.ST * 16);
    T.off_wbl = T.off_wbh + r128(T.NH * T.K16 * 2);
    T.off_bar = T.off_wbl + r128(T.NL * T.K16 * 2);
    T.off_zero = T.off_bar + 256;
    T.off_epi = T.off_zero + 128;                          // 4 tables of 64 floats + 512 bytes of scratch rows
    T.off_dwp = T.off_epi + 1536;                          // depthwise-tail parameter records, one per hi / lo channel
    T.off_xlo = T.off_dwp + r128((T.Cho + T.Clo) * csnet::kIlsDwpBytes);   // stem: GEMM operand of the lo chunk (the ring holds image blocks)
    int end = T.off_xlo + (stem ? r128(2 * T.GLR * T.SL * 16) : 0);
    // the last GEMM block of a chunk reads (never uses) up to 7 pixel groups past the chunk: keep them inside
    const int over_h = T.off_xh + T.hi_stage_bytes + nbh * 8 * T.SH * 16,
              over_l = (stem ? T.off_xlo : T.off_xl + 2 * T.lo_stage_bytes) + nbl * 8 * T.SL * 16;
    end = over_h > end ? over_h : end;
    end = over_l > end ? over_l : end;
    T.smem_bytes = end + 128;
    if (T.smem_bytes > 227 * 1024) continue;
    // the depthwise tail's work does not depend on the strips, everything else scales with the tile's groups per strip
    // group, GR / gsn = 1 + 2 hl / gsn, which only grows with ns: the first split that fits is the cheapest
    best = T;
    found = true;
    break;
  }
  if (!found) return false;
  best.wh = il.wh; best.wl = il.wl;
  best.dw1h = il.dw1h; best.dw1l = il.dw1l; best.dw2h = il.dw2h; best.dw2l = il.dw2l;
  *out = best;
  return true;
}

// MSBlock form of a MIX op: every path a dilated 3x3 (pad == dil in {1, 2, 4, 8, 16}, stride 1) of the SAME whole fp16 tensor,
// at most 8 output channels per path (the concat = disjoint cout slices), fp16 destination of the same size.
bool is_msd(const csnet_plan& P, const csnet_op_desc& op) {
  if (op.kind != CSNET_OP_MIX || op.ext_off[23] == 1 || op.n_paths < 1) return false;
  const csnet_tensor_desc& D = P.tensors[op.dst];
  if (D.dtype != CSNET_F16 || D.W % 8) return false;
  for (int p = 0; p < op.n_paths; ++p) {
    const csnet_path_desc& q = op.paths[p];
    const csnet_tensor_desc& S = P.tensors[q.src];
    if (q.ksize != 3 || q.src != op.paths[0].src || q.c0 != 0 || q.cin != S.C || q.stride != 1 || q.pad != q.dil || q.pool != 1 || q.pre_avg ||
        q.up != 1 || S.dtype != CSNET_F16 || S.H != D.H || S.W != D.W || q.cout > 8 || q.cin > 128)
      return false;
    if (q.dil != 1 && q.dil != 2 && q.dil != 4 && q.dil != 8 && q.dil != 16) return false;
  }
  return true;
}

// Kernel arguments of a MIX op on the streaming 1x1 MIX kernel, but for the activation addresses, the batch and the epilogue
// tables; false if the op does not qualify.
bool plan_ms(const csnet_plan& P, const csnet_op_desc& op, csnet::MsArgs* out) {
  if (!P.ms_enabled || encode_tiled_fn() == nullptr) return false;
  if (op.kind == CSNET_OP_MIX && op.ext_off[23] == 1) return false;      // the compiler's veto of 16-bit weights
  const csnet_tensor_desc& D = P.tensors[op.dst];
  csnet::MsArgs A{};
  A.C = mix_channels(P, op);
  A.has_proj = op.kind == CSNET_OP_MIXPROJ;
  if (A.C > csnet::kMsMaxC || D.W % 8 || D.H % csnet::kMsRows) return false;
  if (A.has_proj ? D.dtype != CSNET_F32 : D.dtype == CSNET_BF16) return false;
  A.dst_f32 = D.dtype == CSNET_F32;
  A.H = D.H; A.W = D.W; A.G = D.W / 8; A.NN = round_up(A.C, 16);
  int off = 0;
  auto r128 = [](int v) { return (v + 127) / 128 * 128; };
  for (int p = 0; p < op.n_paths; ++p) {
    const csnet_path_desc& q = op.paths[p];
    const csnet_tensor_desc& S = P.tensors[q.src];
    if (q.ksize == 0) {
      if (A.n_rs >= csnet::kMsMaxRs || q.up < 2 || q.pool != 1 || q.pre_avg || S.H * q.up != D.H || S.W * q.up != D.W || S.dtype != CSNET_F32 || q.cout0 != 0) return false;
      if (S.W % 4 || S.W > 256 || q.cout > 256) return false;                 // a TMA box row: a multiple of 16 bytes, <= 256 elements
      const int j = A.n_rs++;
      A.r_dtype[j] = S.dtype; A.r_up[j] = q.up; A.r_H[j] = S.H; A.r_W[j] = S.W; A.r_C[j] = S.C; A.r_c0[j] = q.c0; A.r_cout0[j] = q.cout0; A.r_n[j] = q.cout;
      continue;
    }
    const bool k3 = q.ksize == 3 && q.pad == 1 && q.dil == 1, k1 = q.ksize == 1 && q.pad == 0;
    if (A.n_in >= csnet::kMsMaxIn || !(k1 || k3) || (A.n_in > 0 && (int)k3 != A.k3) || q.stride != 1 || q.up != 1 || q.pool != 1 || q.pre_avg ||
        S.dtype != CSNET_F16 || S.H != D.H || S.W != D.W || q.cin > 64)
      return false;
    A.k3 = k3;
    const int i = A.n_in++;
    A.w[i] = P.blob + q.w_off;
    A.cin[i] = q.cin; A.cout0[i] = q.cout0; A.cout[i] = q.cout;
    A.K16[i] = round_up(q.cin, 16); A.S[i] = A.K16[i] + 1;
    if (q.c0 != 0) return false;                                           // (a channel-sliced source would need a c0 coordinate)
  }
  if (A.n_in == 0) return false;
  const int taps = A.k3 ? 9 : 1;
  int wb = 0, smax = 0;
  for (int i = 0; i < A.n_in; ++i) { wb += r128(taps * A.NN * A.K16[i] * 2); smax = A.S[i] > smax ? A.S[i] : smax; }
  // the stage layout of a chunk height: per input its tile (3x3: and the two shifted copies), then per resample path the
  // fp32 box [r_n][r_rows][r_W] of the low-resolution rows that a chunk's taps reach
  auto shape = [&](int rows) {
    csnet::MsArgs T = A;
    T.rows = rows;
    T.nb = (rows * T.G + 7) / 8;
    T.cpi = D.H / rows;
    int off = 0;
    T.tx_bytes = 0;
    for (int i = 0; i < T.n_in; ++i) {
      const int trows = rows + (T.k3 ? 2 : 0);
      T.in_off[i] = off;
      T.copy_bytes[i] = r128(trows * T.G * T.S[i] * 16);
      off += (T.k3 ? 3 : 1) * T.copy_bytes[i];
      T.tx_bytes += trows * T.G * T.S[i] * 16;
    }
    for (int j = 0; j < T.n_rs; ++j) {
      T.r_rows[j] = 0;
      for (int c = 0; c < T.cpi; ++c) {
        const int last = csnet::ms_tap(T.r_H[j], T.r_W[j], T.r_up[j], c * rows + rows - 1, 0).o10 / T.r_W[j];
        const int n = last - csnet::ms_row0(T.r_H[j], T.r_W[j], T.r_up[j], c * rows) + 1;
        T.r_rows[j] = n > T.r_rows[j] ? n : T.r_rows[j];
      }
      T.r_off[j] = off;
      off += r128(T.r_n[j] * T.r_rows[j] * T.r_W[j] * 4);
      T.tx_bytes += T.r_n[j] * T.r_rows[j] * T.r_W[j] * 4;
    }
    T.stage_bytes = off;
    // the last block of a chunk reads past the chunk's groups (rows it does not store): slack after the ring keeps that in bounds
    const int slack = (T.nb * 8 - rows * T.G) * smax * 16;
    T.n_stages = (227 * 1024 - (wb + slack + 512 + 1280 + 128)) / T.stage_bytes;   // weights, slack, barriers, tables, alignment
    T.n_stages = T.n_stages > 6 ? 6 : T.n_stages;
    T.off_stage = 0;
    int o = T.n_stages * T.stage_bytes + slack;
    for (int i = 0; i < T.n_in; ++i) { T.off_wb[i] = o; o += r128(taps * T.NN * T.K16[i] * 2); }
    T.off_bar = o; o += 512;
    T.off_tab = o; o += 1280;
    T.smem_bytes = o + 128;
    return T;
  };
  // chunk height: the smallest that divides H, gives every consumer warpgroup a 64-pixel block per chunk and leaves 3 ring
  // stages; otherwise kMsRows, or 1 row when kMsRows leaves fewer than 2 stages
  bool found = false;
  for (int rows = 1; rows <= 16 && !found; ++rows) {
    if (D.H % rows) continue;
    const csnet::MsArgs T = shape(rows);
    if (T.nb >= csnet::kMsGroups && T.n_stages >= 3) { A = T; found = true; }
  }
  if (!found) {
    A = shape(csnet::kMsRows);
    if (A.n_stages < 2) A = shape(1);
    if (A.n_stages < 2) return false;
  }
  A.has_slope = op.slope_off >= 0;
  *out = A;
  return true;
}

// The il_block_kernel instantiation of a tile (plan_il's candidates).
template <typename T>
IlKernel il_kernel(const csnet::IlArgs& A) {
  if (A.TH == 32) return csnet::il_block_kernel<T, 32, 32>;
  if (A.TH == 28) return csnet::il_block_kernel<T, 28, 32>;
  if (A.TH == 16) return A.TW == 64 ? csnet::il_block_kernel<T, 16, 64> : csnet::il_block_kernel<T, 16, 32>;
  return csnet::il_block_kernel<T, 8, 16>;
}

// Can this MIX op run on the tensor-core kernel (mix_tc.cuh)?  Needs 16-bit operands somewhere, stride-1 conv
// paths and at most 80 output channels; ext_off[23] == 1 is the compiler's veto (weights overflow 16 bits).
TcChoice choose_tc(const csnet_plan& P, const csnet_op_desc& op) {
  TcChoice c;
  if (op.kind == CSNET_OP_MIXPROJ) { /* no other kernel implements it */ }
  else if (op.kind != CSNET_OP_MIX || op.ext_off[23] == 1) return c;
  const csnet_tensor_desc& D = P.tensors[op.dst];
  const int Cm = mix_channels(P, op);
  int dt = D.dtype != CSNET_F32 ? D.dtype : -1, pad = 0, nconv = 0, kk = 1, cin_max = 0;
  for (int p = 0; p < op.n_paths; ++p) {
    const csnet_path_desc& q = op.paths[p];
    if (q.ksize == 0 && (q.pre_avg || q.pool > 1)) return c;     // down-sampling resample paths: generic kernels only
    if (q.ksize == 0) continue;
    ++nconv;
    if (q.stride != 1) return c;
    if (dt < 0 && P.tensors[q.src].dtype != CSNET_F32) dt = P.tensors[q.src].dtype;
    pad = q.pad > pad ? q.pad : pad;
    kk = q.ksize * q.ksize > kk ? q.ksize * q.ksize : kk;
    cin_max = q.cin > cin_max ? q.cin : cin_max;
  }
  if (dt < 0 || nconv == 0 || pad > csnet::kTcMaxPad) return c;
  c.mt = Cm > 80 ? 5 : (Cm + 15) / 16;               // more than 80 output channels: 80-channel slices over grid.y
  c.dtype = dt;
  // wide halos (dilated MS convs): taller tiles while the accumulators fit (MT * rows <= 4)
  c.rows = pad >= 4 ? (c.mt == 1 ? 4 : (c.mt == 2 ? 2 : 1)) : 1;
  c.xs_halves = csnet::tc_plane_halves(pad, c.rows);
  c.kk = kk;
  c.kc = 8;
  for (int kc : {32, 16}) {                       // the largest chunk that keeps two CTAs per SM resident
    TcChoice t = c;
    t.kc = kc;
    if (kc <= ((cin_max + 7) & ~7) && tc_smem_bytes(t) <= 100 * 1024) { c.kc = kc; break; }
  }
  return c;
}

// The kernel that runs an op; the first one in this order that takes the op wins.  Every input is fixed when the plan is
// created (the op, its tensors, its planned record R, max_batch, the SM count, the switches), never by the batch of a call:
// every sub-batch of a plan runs the same kernels, bit for bit.
Kern choose_kernel(const csnet_plan& P, const csnet_op_desc& op, const OpLaunch& R) {
  const csnet_tensor_desc& D = P.tensors[op.dst];
  if (op.kind == CSNET_OP_RESIZE) return Kern::Resize;
  if (is_msd(P, op)) return Kern::Msd;
  if (R.ms.n_in > 0 && (int64_t)P.max_batch * (D.H / csnet::kMsRows) >= (int64_t)2 * P.num_sms) return Kern::MixStream;
  if ((op.kind == CSNET_OP_MIX || op.kind == CSNET_OP_MIXPROJ) && R.tc.mt > 0) return Kern::MixTc;
  if (op.kind == CSNET_OP_MIX && op.n_paths == 1 && op.paths[0].ksize == 0 && op.paths[0].cout0 == 0 && op.paths[0].cout == D.C) {
    const csnet_path_desc& q = op.paths[0];                    // a pure resample
    const csnet_tensor_desc& Sq = P.tensors[q.src];
    const bool avg2 = q.pre_avg == 1 && q.pool == 1, max2 = q.pre_avg == 0 && q.pool == 2;
    const bool fast = Sq.dtype == D.dtype && D.dtype != CSNET_F32 && D.W % 4 == 0 && op.bias_off < 0 && op.slope_off < 0;
    if (fast && (avg2 || max2) && q.up == 1 && q.c0 == 0) return Kern::Pool2;
    if (fast && q.up > 1 && !q.pre_avg && q.pool == 1) return Kern::Upsample;
    return Kern::Resample;
  }
  if (op.kind == CSNET_OP_MIX) return Kern::MixGeneric;
  if (op.kind == CSNET_OP_GN) return Kern::Gn;
  if (op.kind == CSNET_OP_ILBLOCK)
    return R.ils.ns > 0 && (int64_t)P.max_batch * (D.H / 4) >= (int64_t)P.ils_min_chunks ? Kern::IlStream : Kern::IlBlock;
  const csnet_tensor_desc& Sd = P.tensors[op.paths[0].src];
  return op.ext_off[23] != 1 && Sd.dtype == D.dtype && D.dtype != CSNET_F32 && D.W % 4 == 0 ? Kern::DwFast : Kern::DwGeneric;
}

// The mix_tc_kernel instantiation of a choice (choose_tc gives rows 4 only with mt 1, rows 2 only with mt 2).
template <typename T>
TcKernel tc_kernel(const TcChoice& c) {
  if (c.rows == 4) return csnet::mix_tc_kernel<T, 1, 4>;
  if (c.rows == 2) return csnet::mix_tc_kernel<T, 2, 2>;
  switch (c.mt) {
    case 1: return csnet::mix_tc_kernel<T, 1>;
    case 2: return csnet::mix_tc_kernel<T, 2>;
    case 3: return csnet::mix_tc_kernel<T, 3>;
    case 4: return csnet::mix_tc_kernel<T, 4>;
    default: return csnet::mix_tc_kernel<T, 5>;
  }
}

// The dynamic shared memory a kernel may opt into on sm_90 (227 KB less its static shared memory; these kernels have none).
// Each kernel is given all of it, not what one plan needs: the attribute belongs to the kernel, so a plan created later must
// not lower the limit an existing plan relies on.
constexpr int kSmemOptIn = 227 * 1024;

const char* const kKernNames[] = {
    "msd_kernel (ms_direct.cuh, FP32 pipe)", "mix_stream_kernel (TMA + wgmma)", "mix_tc_kernel (mma.sync)",
    "pool2 / upsample / resample kernels", "pool2 / upsample / resample kernels", "pool2 / upsample / resample kernels",
    "mix_generic_kernel", "gn kernels", "il_stream_kernel (TMA + wgmma)", "il_block_kernel (mma.sync, tiled)", "dw kernels", "dw kernels",
    "resize_kernel"};
static_assert(sizeof kKernNames / sizeof kKernNames[0] == (size_t)Kern::Resize + 1, "one name per Kern");

// Plan op i: choose its kernel and fill its launch record (kernel, static arguments, packed-weight buffers), and let the
// kernel use the shared memory it needs.
int plan_op(csnet_plan& P, size_t i) {
  const csnet_op_desc& op = P.ops[i];
  OpLaunch& R = P.launch[i];
  if (op.kind == CSNET_OP_MIX || op.kind == CSNET_OP_MIXPROJ) {
    R.tc = choose_tc(P, op);
    if (tc_smem_bytes(R.tc) > 200 * 1024) R.tc = TcChoice();
    if (op.kind == CSNET_OP_MIXPROJ && R.tc.mt == 0)
      return fail(CSNET_E_UNSUPPORTED, "MIXPROJ op does not qualify for the tensor-core kernel (16-bit sources, stride 1, pad <= limit)");
    plan_ms(P, op, &R.ms);
  } else if (op.kind == CSNET_OP_ILBLOCK) {
    if (!plan_il(P, op, &R.il)) return fail(CSNET_E_UNSUPPORTED, "ILBLOCK op does not fit shared memory");
    plan_ils(P, op, R.il, &R.ils);
  }
  R.kern = choose_kernel(P, op, R);
  cudaError_t e = cudaSuccess;
  switch (R.kern) {
    case Kern::MixStream:
      e = R.ms.has_proj && R.ms.n_rs > 0
              ? cudaFuncSetAttribute(csnet::mix_stream_kernel<__half, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemOptIn)
              : cudaFuncSetAttribute(csnet::mix_stream_kernel<__half>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemOptIn);
      break;
    case Kern::MixTc: {
      const int C = mix_channels(P, op), slice = R.tc.mt * 16, m16t = (C + slice - 1) / slice * slice, WR = R.tc.kc + 8;
      for (int p = 0; p < op.n_paths; ++p) {
        const csnet_path_desc& q = op.paths[p];
        if (q.ksize == 0) continue;
        const size_t halves = (size_t)((q.cin + R.tc.kc - 1) / R.tc.kc) * q.ksize * q.ksize * m16t * WR;
        e = cudaMalloc(&R.w16[p], halves * 2);
        if (e != cudaSuccess) return fail(CSNET_E_NOMEM, std::string("cudaMalloc(packed weights): ") + cudaGetErrorString(e));
      }
      R.smem = tc_smem_bytes(R.tc);
      R.tc_fn = R.tc.dtype == CSNET_F16 ? tc_kernel<__half>(R.tc) : tc_kernel<__nv_bfloat16>(R.tc);
      e = cudaFuncSetAttribute(R.tc_fn, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemOptIn);
      break;
    }
    case Kern::IlStream: {
      const bool stem = R.ils.Ci > 0;
      e = cudaFuncSetAttribute(stem ? csnet::il_stream_kernel<__half, true> : csnet::il_stream_kernel<__half, false>,
                               cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemOptIn);
      // two CTAs of <= 113 KB share an SM only with the full shared-memory carve-out
      if (e == cudaSuccess && !stem)
        e = cudaFuncSetAttribute(csnet::il_stream_kernel<__half, false>, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
      break;
    }
    case Kern::IlBlock:
      R.smem = il_smem_of(R.il);
      R.il_fn = P.tensors[op.dst].dtype == CSNET_F16 ? il_kernel<__half>(R.il) : il_kernel<__nv_bfloat16>(R.il);
      e = cudaFuncSetAttribute(R.il_fn, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemOptIn);
      break;
    default:
      break;
  }
  if (e != cudaSuccess)
    return fail(CSNET_E_CUDA, std::string("cudaFuncSetAttribute(") + kKernNames[(int)R.kern] + "): " + cudaGetErrorString(e));
  return CSNET_OK;
}

}  // namespace

namespace csnet {
void train_set_error(const char* msg);     // train_ops.cu: the message csnet_train_last_error returns
}

extern "C" {

int csnet_abi_version(void) { return CSNET_ABI_VERSION; }

const char* csnet_last_error(void) { return g_err.c_str(); }

int csnet_device_count(void) {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return fail(CSNET_E_CUDA, std::string("cudaGetDeviceCount: ") + cudaGetErrorString(e));
  }
  return n;
}

int csnet_plan_create(csnet_plan** out, const csnet_tensor_desc* tensors, int32_t n_tensors,
                      const csnet_op_desc* ops, int32_t n_ops, int64_t blob_floats, int32_t max_batch,
                      int32_t device) {
  if (!out || !tensors || !ops || n_tensors <= 0 || n_ops <= 0 || blob_floats <= 0 || max_batch <= 0)
    return fail(CSNET_E_INVALID, "csnet_plan_create: null/empty argument");
  csnet_plan* P = new (std::nothrow) csnet_plan();
  if (!P) return fail(CSNET_E_NOMEM, "host allocation failed");
  P->device = device;
  P->max_batch = max_batch;
  P->tensors.assign(tensors, tensors + n_tensors);
  P->ops.assign(ops, ops + n_ops);
  P->blob_floats = blob_floats;
  int rc = validate(*P);
  if (rc != CSNET_OK) { delete P; return rc; }
  for (const auto& d : P->tensors) {
    if (d.external >= 0) { P->n_ext = d.external + 1 > P->n_ext ? d.external + 1 : P->n_ext; continue; }
    const int64_t end = d.arena_offset + (int64_t)d.C * d.H * d.W * (int64_t)dtype_size(d.dtype);
    P->arena_per_image = end > P->arena_per_image ? end : P->arena_per_image;
  }
  P->arena_per_image = (P->arena_per_image + 255) / 256 * 256;
  auto cleanup = [&](int code, const std::string& m) { csnet_plan_destroy(P); return fail(code, m); };
  DeviceGuard guard_(device);
  cudaError_t e = cudaSuccess;
  {
    int cur = -1;
    if (cudaGetDevice(&cur) != cudaSuccess || cur != device) return cleanup(CSNET_E_CUDA, "cudaSetDevice failed");
  }
  e = cudaMalloc(&P->blob, (size_t)blob_floats * sizeof(float));
  if (e != cudaSuccess) return cleanup(CSNET_E_NOMEM, std::string("cudaMalloc(blob): ") + cudaGetErrorString(e));
  const size_t arena_bytes = (size_t)P->arena_per_image * (size_t)max_batch + 256;
  e = cudaMalloc(&P->arena, arena_bytes);
  if (e != cudaSuccess) return cleanup(CSNET_E_NOMEM, std::string("cudaMalloc(arena): ") + cudaGetErrorString(e));
  for (const auto& op : P->ops)
    if (op.kind == CSNET_OP_GN && op.paths[0].up > P->gn_groups_max) P->gn_groups_max = op.paths[0].up;
  if (P->gn_groups_max > 0) {
    e = cudaMalloc(&P->gn_stats, (size_t)max_batch * P->gn_groups_max * 2 * sizeof(float));
    if (e != cudaSuccess) return cleanup(CSNET_E_NOMEM, std::string("cudaMalloc(gn stats): ") + cudaGetErrorString(e));
  }
  {
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) == cudaSuccess && prop.multiProcessorCount > 0) P->num_sms = prop.multiProcessorCount;
  }
  // the kernel switches, read when the plan is created: CSNET_MS=0 keeps 1x1 MIX ops off mix_stream, CSNET_ILS=0 keeps
  // ILBLOCK ops off il_stream, CSNET_ILS_NS forces its column strips and CSNET_ILS_MIN_CHUNKS its batch threshold
  if (const char* s = getenv("CSNET_MS")) P->ms_enabled = s[0] != '0';
  if (const char* s = getenv("CSNET_ILS")) P->ils_enabled = s[0] != '0';
  if (const char* s = getenv("CSNET_ILS_NS")) P->ils_force_ns = atoi(s);
  P->ils_min_chunks = 4 * P->num_sms;
  if (const char* s = getenv("CSNET_ILS_MIN_CHUNKS")) P->ils_min_chunks = atoi(s);
  P->launch.resize(P->ops.size());
  for (size_t i = 0; i < P->ops.size(); ++i) {
    rc = plan_op(*P, i);
    if (rc != CSNET_OK) { csnet_plan_destroy(P); return rc; }
  }
  *out = P;
  return CSNET_OK;
}

static void drop_graphs(csnet_plan* P);

int csnet_plan_set_blob(csnet_plan* P, const float* host_blob, int64_t n, void* stream) {
  if (!P || !host_blob || n != P->blob_floats) return fail(CSNET_E_INVALID, "csnet_plan_set_blob: size mismatch");
  DeviceGuard guard_(P->device);
  CU_CHECK(cudaMemcpyAsync(P->blob, host_blob, (size_t)n * sizeof(float), cudaMemcpyHostToDevice, (cudaStream_t)stream));
  drop_graphs(P);                                   // captured launches carry parameter tables of the old blob
  // the streaming kernels take their bias / PReLU / projection epilogue tables in the kernel arguments
  for (size_t i = 0; i < P->ops.size(); ++i) {
    const csnet_op_desc& op = P->ops[i];
    OpLaunch& R = P->launch[i];
    if (R.kern == Kern::IlStream) {
      csnet::IlsArgs& A = R.ils;
      for (int c = 0; c < A.Cho; ++c) { A.bias_h[c] = host_blob[op.ext_off[2] + c]; A.sm1_h[c] = host_blob[op.ext_off[3] + c] - 1.f; }
      for (int c = 0; c < A.Clo; ++c) { A.bias_l[c] = host_blob[op.ext_off[4] + c]; A.sm1_l[c] = host_blob[op.ext_off[5] + c] - 1.f; }
    }
    if (R.kern == Kern::MixStream) {
      csnet::MsArgs& A = R.ms;
      for (int c = 0; c < A.C; ++c) {
        A.bias[c] = op.bias_off >= 0 ? host_blob[op.bias_off + c] : 0.f;
        A.sm1[c] = op.slope_off >= 0 ? host_blob[op.slope_off + c] - 1.f : 0.f;
        A.proj[c] = A.has_proj ? host_blob[op.ext_off[0] + c] : 0.f;
      }
      A.proj_b = A.has_proj && op.ext_off[1] >= 0 ? host_blob[op.ext_off[1]] : 0.f;
    }
  }
  // tensor-core MIX ops read their weights as 16-bit [chunk][tap][m16_total][kc + 8] blocks: pack them here, once per
  // weight update, so the kernels stage them with plain 16-byte copies
  std::vector<std::vector<uint16_t>> keep;
  for (size_t i = 0; i < P->ops.size(); ++i) {
    const OpLaunch& R = P->launch[i];
    if (R.kern != Kern::MixTc) continue;
    const TcChoice& tc = R.tc;
    const csnet_op_desc& op = P->ops[i];
    const int C = mix_channels(*P, op), slice = tc.mt * 16, m16t = (C + slice - 1) / slice * slice, WR = tc.kc + 8;
    for (int p = 0; p < op.n_paths; ++p) {
      const csnet_path_desc& q = op.paths[p];
      if (q.ksize == 0) continue;
      const int kk = q.ksize * q.ksize, nchunks = (q.cin + tc.kc - 1) / tc.kc;
      std::vector<uint16_t> h((size_t)nchunks * kk * m16t * WR, 0);
      const float* w = host_blob + q.w_off;                         // [cin][kk][cout]
      for (int ci = 0; ci < q.cin; ++ci)
        for (int tap = 0; tap < kk; ++tap)
          for (int co = 0; co < q.cout; ++co) {
            const float v = w[((size_t)ci * kk + tap) * q.cout + co];
            uint16_t bits;
            if (tc.dtype == CSNET_F16) { __half hv = __float2half_rn(v); memcpy(&bits, &hv, 2); }
            else { __nv_bfloat16 hv = __float2bfloat16_rn(v); memcpy(&bits, &hv, 2); }
            h[(((size_t)(ci / tc.kc) * kk + tap) * m16t + q.cout0 + co) * WR + ci % tc.kc] = bits;
          }
      CU_CHECK(cudaMemcpyAsync(R.w16[p], h.data(), h.size() * 2, cudaMemcpyHostToDevice, (cudaStream_t)stream));
      keep.push_back(std::move(h));
    }
  }
  CU_CHECK(cudaStreamSynchronize((cudaStream_t)stream));
  return CSNET_OK;
}

static int check_run_args(csnet_plan* P, int32_t N, const void* const* ext_ptrs, int32_t n_ext) {
  if (!P) return fail(CSNET_E_INVALID, "null plan");
  if (N <= 0 || N > P->max_batch) return fail(CSNET_E_INVALID, "batch size outside [1, max_batch]");
  if (n_ext < P->n_ext || (P->n_ext > 0 && !ext_ptrs)) return fail(CSNET_E_INVALID, "missing external tensor pointers");
  for (int i = 0; i < P->n_ext; ++i)
    if (!ext_ptrs[i]) return fail(CSNET_E_INVALID, "null external tensor pointer");
  return CSNET_OK;
}

static int launch_op(csnet_plan* P, size_t i, int32_t N, const void* const* ext_ptrs, cudaStream_t stream) {
  const csnet_op_desc& op = P->ops[i];
  const csnet_tensor_desc& D = P->tensors[op.dst];
  const OpLaunch& R = P->launch[i];
  switch (R.kern) {
    case Kern::Msd:
      // MSBlock: one launch per dilated path on the FP32 pipe (ms_direct.cuh)
      for (int p = 0; p < op.n_paths; ++p) {
        const csnet_path_desc& q = op.paths[p];
        csnet::MsdArgs A{};
        A.src = reinterpret_cast<const uint16_t*>(P->tensor_ptr(q.src, N, ext_ptrs));
        A.dst = reinterpret_cast<uint16_t*>(P->tensor_ptr(op.dst, N, ext_ptrs));
        A.w = P->blob + q.w_off;
        A.bias = op.bias_off >= 0 ? P->blob + op.bias_off : nullptr;
        A.slope = op.slope_off >= 0 ? P->blob + op.slope_off : nullptr;
        A.N = N; A.Cin = q.cin; A.H = D.H; A.W = D.W; A.Ctot = D.C; A.cout0 = q.cout0; A.cout = q.cout;
        csnet::msd_launch<__half>(q.dil, A, stream);
      }
      break;
    case Kern::MixStream: {
      // streaming 1x1 MIX kernel (mix_stream.cuh): TMA operand tiles -> wgmma -> epilogue (resample-adds, PReLU, projection)
      csnet::MsArgs A = R.ms;
      A.N = N;
      A.total_chunks = N * A.cpi;
      A.dst = P->tensor_ptr(op.dst, N, ext_ptrs);
      CUtensorMap maps[csnet::kMsMaxIn], rmaps[csnet::kMsMaxRs];
      memset(maps, 0, sizeof maps);
      for (int p = 0, in = 0, rs = 0; p < op.n_paths; ++p) {         // numbered as plan_ms does: each kind in path order
        const csnet_path_desc& q = op.paths[p];
        const csnet_tensor_desc& S = P->tensors[q.src];
        if (q.ksize == 0) {
          if (!encode_image_map(&rmaps[rs], P->tensor_ptr(q.src, N, ext_ptrs), N, S.C, S.H, S.W, S.W, A.r_rows[rs], A.r_n[rs]))
            return fail(CSNET_E_CUDA, "cuTensorMapEncodeTiled failed (streaming MIX)");
          ++rs;
          continue;
        }
        if (!encode_group_map(&maps[in], P->tensor_ptr(q.src, N, ext_ptrs), N, S.C, S.H, S.W, A.S[in], A.G, A.rows + (A.k3 ? 2 : 0)))
          return fail(CSNET_E_CUDA, "cuTensorMapEncodeTiled failed (streaming MIX)");
        ++in;
      }
      for (int k = A.n_in; k < csnet::kMsMaxIn; ++k) maps[k] = maps[0];
      for (int k = A.n_rs; k < csnet::kMsMaxRs; ++k) rmaps[k] = maps[0];
      int grid = A.total_chunks / 2;
      grid = grid < 1 ? 1 : (grid > P->num_sms ? P->num_sms : grid);
      if (A.has_proj && A.n_rs > 0)
        csnet::mix_stream_kernel<__half, true><<<grid, csnet::kMsThreads, A.smem_bytes, stream>>>(A, maps[0], maps[1], maps[2], rmaps[0], rmaps[1]);
      else
        csnet::mix_stream_kernel<__half><<<grid, csnet::kMsThreads, A.smem_bytes, stream>>>(A, maps[0], maps[1], maps[2], rmaps[0], rmaps[1]);
      break;
    }
    case Kern::MixTc: {
      csnet::MixArgs A = make_mix(*P, op, N, ext_ptrs);
      const TcChoice& tc = R.tc;
      const int Cm = A.C;
      csnet::TcGeom G{};
      G.tiles_x = (D.W + csnet::kTcTW - 1) / csnet::kTcTW; G.xs_halves = tc.xs_halves; G.kc = tc.kc; G.rows = tc.rows;
      const int th = csnet::kTcTH * tc.rows;
      G.m16_total = (Cm + tc.mt * 16 - 1) / (tc.mt * 16) * (tc.mt * 16);
      for (int p = 0; p < op.n_paths; ++p) G.w16[p] = R.w16[p];
      dim3 grid(G.tiles_x * ((D.H + th - 1) / th), (Cm + tc.mt * 16 - 1) / (tc.mt * 16), N);
      R.tc_fn<<<grid, csnet::kTcThreads, R.smem, stream>>>(A, G);
      break;
    }
    case Kern::Pool2: {
      csnet::MixArgs A = make_mix(*P, op, N, ext_ptrs);
      const bool max2 = op.paths[0].pool == 2;
      const dim3 grid((D.H * (D.W / 4) + 255) / 256, D.C, N);    // avg_pool2d(2, 2) / max_pool2d(2, 2) of a 16-bit tensor
      if (D.dtype == CSNET_F16) csnet::pool2_fast_kernel<__half><<<grid, 256, 0, stream>>>(A, max2);
      else csnet::pool2_fast_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>(A, max2);
      break;
    }
    case Kern::Upsample: {
      csnet::MixArgs A = make_mix(*P, op, N, ext_ptrs);
      const dim3 grid((D.H * (D.W / 4) + 255) / 256, D.C, N);    // bilinear up-sampling, 16-bit to 16-bit
      if (D.dtype == CSNET_F16) csnet::upsample_fast_kernel<__half><<<grid, 256, 0, stream>>>(A);
      else csnet::upsample_fast_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>(A);
      break;
    }
    case Kern::Resample:
      csnet::resample_fast_kernel<<<dim3((D.H * D.W + 255) / 256, D.C, N), 256, 0, stream>>>(make_mix(*P, op, N, ext_ptrs));
      break;
    case Kern::MixGeneric: {
      dim3 grid((D.H * D.W + kThreads - 1) / kThreads, (D.C + csnet::kMixCT - 1) / csnet::kMixCT, N);
      mix_generic_kernel<<<grid, kThreads, 0, stream>>>(make_mix(*P, op, N, ext_ptrs));
      break;
    }
    case Kern::Gn: {
      const csnet_tensor_desc& S = P->tensors[op.paths[0].src];
      csnet::GnArgs A{};
      A.src = P->tensor_ptr(op.paths[0].src, N, ext_ptrs);
      A.dst = P->tensor_ptr(op.dst, N, ext_ptrs);
      A.gamma = P->blob + op.ext_off[0];
      A.beta = P->blob + op.ext_off[1];
      A.slope = op.slope_off >= 0 ? P->blob + op.slope_off : nullptr;
      A.stats = P->gn_stats;
      A.src_dtype = S.dtype; A.dst_dtype = D.dtype; A.C = D.C; A.HW = D.H * D.W; A.groups = op.paths[0].up;
      gn_stats_kernel<<<dim3(A.groups, N), kThreads, 0, stream>>>(A);
      const int bx = (A.HW + kThreads * 4 - 1) / (kThreads * 4);
      gn_apply_kernel<<<dim3(bx < 1 ? 1 : bx, D.C, N), kThreads, 0, stream>>>(A);
      break;
    }
    case Kern::IlStream: {
      // streaming kernel (il_stream.cuh): TMA operand tiles, wgmma GEMM, register-resident depthwise tail
      csnet::IlsArgs A = R.ils;
      A.yh = P->tensor_ptr(op.dst, N, ext_ptrs);
      A.yl = op.dst2 >= 0 ? P->tensor_ptr(op.dst2, N, ext_ptrs) : nullptr;
      A.N = N;
      A.total_chunks = N * A.ns * A.cpi;
      CUtensorMap tmH, tmL;
      const bool stem = A.Ci > 0;
      if (stem) {
        if (!encode_image_map(&tmL, P->tensor_ptr(op.paths[0].src, N, ext_ptrs), N, A.Ci, A.H, A.W, A.BW, 4, A.Ci))
          return fail(CSNET_E_CUDA, "cuTensorMapEncodeTiled failed (streaming ILBlock, image)");
        tmH = tmL;
      } else if (!encode_group_map(&tmH, P->tensor_ptr(op.paths[0].src, N, ext_ptrs), N, A.Chi, A.H, A.W, A.SH, A.GR, 4) ||
                 !encode_group_map(&tmL, P->tensor_ptr(op.paths[1].src, N, ext_ptrs), N, A.Cli, A.H / 2, A.W / 2, A.SL, A.GLR, 2))
        return fail(CSNET_E_CUDA, "cuTensorMapEncodeTiled failed (streaming ILBlock)");
      int grid = A.total_chunks / 4;
      grid = grid < 1 ? 1 : (grid > P->num_sms ? P->num_sms : grid);     // persistent: one CTA per SM
      if (stem) csnet::il_stream_kernel<__half, true><<<grid, A.dw_warps * 32, A.smem_bytes, stream>>>(A, tmH, tmL);
      else csnet::il_stream_kernel<__half, false><<<grid, A.dw_warps * 32, A.smem_bytes, stream>>>(A, tmH, tmL);
      break;
    }
    case Kern::IlBlock: {
      csnet::IlArgs A = R.il;
      A.xh = P->tensor_ptr(op.paths[0].src, N, ext_ptrs);
      if (!A.first) A.xl = P->tensor_ptr(op.paths[1].src, N, ext_ptrs);   // (the stem form has no lo input tensor)
      A.yh = P->tensor_ptr(op.dst, N, ext_ptrs);
      if (op.dst2 >= 0) A.yl = P->tensor_ptr(op.dst2, N, ext_ptrs);
      const int tiles_y = (A.H + A.TH - 1) / A.TH;
      dim3 grid(A.tiles_x * tiles_y, 1, N);
      R.il_fn<<<grid, csnet::kIlThreads, R.smem, stream>>>(A);
      break;
    }
    case Kern::DwFast:
    case Kern::DwGeneric: {
      const csnet_path_desc& q = op.paths[0];
      const csnet_tensor_desc& S = P->tensors[q.src];
      csnet::DwArgs A{};
      A.src = P->tensor_ptr(q.src, N, ext_ptrs);
      A.dst = P->tensor_ptr(op.dst, N, ext_ptrs);
      A.w = P->blob + q.w_off;
      A.bias = op.bias_off >= 0 ? P->blob + op.bias_off : nullptr;
      A.slope = op.slope_off >= 0 ? P->blob + op.slope_off : nullptr;
      A.src_dtype = S.dtype; A.dst_dtype = D.dtype; A.C = D.C; A.H = D.H; A.W = D.W;
      if (R.kern == Kern::DwFast) {
        const int tasks = (D.W / 4) * ((D.H + csnet::kDwfRun - 1) / csnet::kDwfRun);
        dim3 grid((tasks + csnet::kDwfThreads - 1) / csnet::kDwfThreads, D.C, N);
        if (D.dtype == CSNET_F16) csnet::dw_fast_kernel<__half><<<grid, csnet::kDwfThreads, 0, stream>>>(A);
        else csnet::dw_fast_kernel<__nv_bfloat16><<<grid, csnet::kDwfThreads, 0, stream>>>(A);
      } else {
        const int strips = (D.H + csnet::kDwRows - 1) / csnet::kDwRows;
        dim3 grid((strips * D.W + kThreads - 1) / kThreads, D.C, N);
        dw_generic_kernel<<<grid, kThreads, 0, stream>>>(A);
      }
      break;
    }
    case Kern::Resize: {
      // bilinear resize at any ratio (resize.cuh)
      const csnet_path_desc& q = op.paths[0];
      const csnet_tensor_desc& S = P->tensors[q.src];
      csnet::RzArgs A{};
      A.src = P->tensor_ptr(q.src, N, ext_ptrs);
      A.dst = P->tensor_ptr(op.dst, N, ext_ptrs);
      A.Cs = S.C; A.Hs = S.H; A.Ws = S.W; A.c0 = q.c0;
      A.Cd = D.C; A.Hd = D.H; A.Wd = D.W; A.cout0 = q.cout0;
      A.C = q.cout; A.accumulate = (int)op.ext_off[0];
      A.sy = csnet::resize_scale(S.H, D.H); A.sx = csnet::resize_scale(S.W, D.W);
      csnet::launch_resize(A, S.dtype, D.dtype, N, stream);
      break;
    }
  }
  CU_CHECK(cudaGetLastError());
  return CSNET_OK;
}

static int run_ops(csnet_plan* P, int32_t N, const void* const* ext_ptrs, cudaStream_t stream) {
  for (size_t i = 0; i < P->ops.size(); ++i) {
    const int rc = launch_op(P, i, N, ext_ptrs, stream);
    if (rc != CSNET_OK) return rc;
  }
  return CSNET_OK;
}

static void drop_graphs(csnet_plan* P) {
  for (auto& g : P->graphs) {
    if (g.exec) cudaGraphExecDestroy(g.exec);
    if (g.in) cudaFree(g.in);
    if (g.out) cudaFree(g.out);
    g = csnet_plan::GraphSlot();
  }
}

// Small batches of a two-external plan (input, logits): copy the input into the plan's staging buffer, replay the captured
// graph, copy the logits out — three stream operations instead of one launch per op.
static int run_graph(csnet_plan* P, int32_t N, const void* const* ext_ptrs, cudaStream_t stream) {
  if ((int)P->graphs.size() <= N) P->graphs.resize((size_t)N + 1);
  csnet_plan::GraphSlot& G = P->graphs[N];
  const csnet_tensor_desc *in = nullptr, *out = nullptr;
  for (const auto& d : P->tensors) {
    if (d.external == 0) in = &d;
    if (d.external == 1) out = &d;
  }
  if (!G.exec) {
    G.in_bytes = (size_t)N * in->C * in->H * in->W * dtype_size(in->dtype);
    G.out_bytes = (size_t)N * out->C * out->H * out->W * dtype_size(out->dtype);
    CU_CHECK(cudaMalloc(&G.in, G.in_bytes));
    CU_CHECK(cudaMalloc(&G.out, G.out_bytes));
    const void* ext[2] = {G.in, G.out};
    cudaGraph_t graph = nullptr;
    // capture on a stream of our own: the caller's may be the legacy default stream, which cannot be captured
    if (!P->cap_stream) CU_CHECK(cudaStreamCreateWithFlags(&P->cap_stream, cudaStreamNonBlocking));
    CU_CHECK(cudaStreamBeginCapture(P->cap_stream, cudaStreamCaptureModeThreadLocal));
    const int rc = run_ops(P, N, ext, P->cap_stream);
    const cudaError_t e = cudaStreamEndCapture(P->cap_stream, &graph);
    if (rc != CSNET_OK || e != cudaSuccess || !graph) {
      if (graph) cudaGraphDestroy(graph);
      cudaGetLastError();
      return rc != CSNET_OK ? rc : fail(CSNET_E_CUDA, std::string("graph capture: ") + cudaGetErrorString(e));
    }
    const cudaError_t e2 = cudaGraphInstantiate(&G.exec, graph, 0);
    cudaGraphDestroy(graph);
    if (e2 != cudaSuccess) { G.exec = nullptr; return fail(CSNET_E_CUDA, std::string("cudaGraphInstantiate: ") + cudaGetErrorString(e2)); }
  }
  CU_CHECK(cudaMemcpyAsync(G.in, ext_ptrs[0], G.in_bytes, cudaMemcpyDeviceToDevice, stream));
  CU_CHECK(cudaGraphLaunch(G.exec, stream));
  CU_CHECK(cudaMemcpyAsync(const_cast<void*>(ext_ptrs[1]), G.out, G.out_bytes, cudaMemcpyDeviceToDevice, stream));
  return CSNET_OK;
}

int csnet_plan_run(csnet_plan* P, int32_t N, const void* const* ext_ptrs, int32_t n_ext, void* stream_) {
  int rc = check_run_args(P, N, ext_ptrs, n_ext);
  if (rc != CSNET_OK) return rc;
  cudaStream_t stream = (cudaStream_t)stream_;
  DeviceGuard guard_(P->device);
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  if (N <= kGraphMaxN && P->n_ext == 2 && cudaStreamIsCapturing(stream, &cap) == cudaSuccess && cap == cudaStreamCaptureStatusNone)
    return run_graph(P, N, ext_ptrs, stream);
  return run_ops(P, N, ext_ptrs, stream);
}

int csnet_plan_profile(csnet_plan* P, int32_t N, const void* const* ext_ptrs, int32_t n_ext, void* stream_,
                       float* ms_per_op, int32_t n_ops) {
  int rc = check_run_args(P, N, ext_ptrs, n_ext);
  if (rc != CSNET_OK) return rc;
  if (!ms_per_op || n_ops != (int32_t)P->ops.size()) return fail(CSNET_E_INVALID, "csnet_plan_profile: n_ops mismatch");
  cudaStream_t stream = (cudaStream_t)stream_;
  DeviceGuard guard_(P->device);
  std::vector<cudaEvent_t> ev(P->ops.size() + 1);
  for (auto& e : ev) CU_CHECK(cudaEventCreate(&e));
  CU_CHECK(cudaEventRecord(ev[0], stream));
  for (size_t i = 0; i < P->ops.size() && rc == CSNET_OK; ++i) {
    rc = launch_op(P, i, N, ext_ptrs, stream);
    if (rc == CSNET_OK && cudaEventRecord(ev[i + 1], stream) != cudaSuccess) rc = fail(CSNET_E_CUDA, "cudaEventRecord");
  }
  cudaError_t e = cudaStreamSynchronize(stream);
  if (rc == CSNET_OK && e != cudaSuccess) rc = fail(CSNET_E_CUDA, std::string("sync: ") + cudaGetErrorString(e));
  if (rc == CSNET_OK)
    for (size_t i = 0; i < P->ops.size(); ++i) cudaEventElapsedTime(&ms_per_op[i], ev[i], ev[i + 1]);
  for (auto& e2 : ev) cudaEventDestroy(e2);
  return rc;
}

void* csnet_plan_tensor_ptr(csnet_plan* P, int32_t tensor, int32_t N) {
  if (!P || tensor < 0 || tensor >= (int)P->tensors.size() || N <= 0 || N > P->max_batch) return nullptr;
  if (P->tensors[tensor].external >= 0) return nullptr;
  return P->tensor_ptr(tensor, N, nullptr);
}

int csnet_plan_read_tensor(csnet_plan* P, int32_t tensor, int32_t N, void* dst, void* stream) {
  void* src = csnet_plan_tensor_ptr(P, tensor, N);
  if (!src || !dst) return fail(CSNET_E_INVALID, "csnet_plan_read_tensor: bad tensor / batch / destination");
  const csnet_tensor_desc& d = P->tensors[tensor];
  DeviceGuard guard_(P->device);
  CU_CHECK(cudaMemcpyAsync(dst, src, (size_t)N * d.C * d.H * d.W * dtype_size(d.dtype), cudaMemcpyDeviceToDevice,
                           (cudaStream_t)stream));
  return CSNET_OK;
}

// Which kernel launch_op() runs for op i, by name (bench.py groups per-op times by kernel).
const char* csnet_plan_op_kernel(const csnet_plan* P, int32_t i) {
  if (!P || i < 0 || i >= (int32_t)P->ops.size()) return "";
  return kKernNames[(int)P->launch[i].kern];
}

int32_t csnet_plan_launches(const csnet_plan* P) {
  if (!P) return 0;
  int32_t n = 0;
  for (size_t i = 0; i < P->ops.size(); ++i)
    n += P->launch[i].kern == Kern::Gn ? 2 : (P->launch[i].kern == Kern::Msd ? P->ops[i].n_paths : 1);
  return n;
}

int64_t csnet_plan_arena_bytes(const csnet_plan* P) { return P ? P->arena_per_image * (int64_t)P->max_batch : 0; }

void csnet_plan_destroy(csnet_plan* P) {
  if (!P) return;
  drop_graphs(P);
  if (P->cap_stream) cudaStreamDestroy(P->cap_stream);
  DeviceGuard guard_(P->device);
  if (P->blob) cudaFree(P->blob);
  if (P->arena) cudaFree(P->arena);
  if (P->gn_stats) cudaFree(P->gn_stats);
  for (const OpLaunch& R : P->launch)
    for (uint16_t* q : R.w16)
      if (q) cudaFree(q);
  for (int b = 0; b < 2; ++b) {
    if (P->h_in[b]) cudaFree(P->h_in[b]);
    if (P->h_out[b]) cudaFree(P->h_out[b]);
    if (P->h_in8[b]) cudaFree(P->h_in8[b]);
    if (P->h_out8[b]) cudaFree(P->h_out8[b]);
    if (P->ev_h2d[b]) cudaEventDestroy(P->ev_h2d[b]);
    if (P->ev_comp[b]) cudaEventDestroy(P->ev_comp[b]);
    if (P->ev_d2h[b]) cudaEventDestroy(P->ev_d2h[b]);
  }
  if (P->h_geom) cudaFree(P->h_geom);
  if (P->s_h2d) cudaStreamDestroy(P->s_h2d);
  if (P->s_d2h) cudaStreamDestroy(P->s_d2h);
  delete P;
}

// What the host buffers of a csnet_plan_run_host* call hold: fp32 tensors, uint8 images at the network size, or packed uint8
// images of any size with their geometry.
enum class HostIo { F32, U8, Images };
struct HostImages {
  const csnet_image_geom* geom;
  int64_t x_bytes, y_bytes;
};

static int run_host_impl(csnet_plan* P, int32_t N, const void* x_host, void* y_host, void* stream_, HostIo io, const float* mean,
                         const float* stdv, const HostImages* im = nullptr);

int csnet_plan_run_host(csnet_plan* P, int32_t N, const float* x_host, float* y_host, void* stream_) {
  return run_host_impl(P, N, x_host, y_host, stream_, HostIo::F32, nullptr, nullptr);
}

int csnet_plan_run_host_u8(csnet_plan* P, int32_t N, const uint8_t* x_hwc, uint8_t* y_u8, const float* mean, const float* stdv, void* stream_) {
  if (!mean || !stdv) return fail(CSNET_E_INVALID, "null mean / std");
  return run_host_impl(P, N, x_hwc, y_u8, stream_, HostIo::U8, mean, stdv);
}

int csnet_plan_run_host_images_u8(csnet_plan* P, int32_t N, const uint8_t* x_packed, int64_t x_bytes, const csnet_image_geom* geom,
                                  uint8_t* y_packed, int64_t y_bytes, const float* mean, const float* stdv, void* stream_) {
  if (!geom || !mean || !stdv) return fail(CSNET_E_INVALID, "null geometry / mean / std");
  const HostImages im{geom, x_bytes, y_bytes};
  return run_host_impl(P, N, x_packed, y_packed, stream_, HostIo::Images, mean, stdv, &im);
}

int csnet_resize_u8_to_input(const uint8_t* x_packed, const csnet_image_geom* geom, int32_t N, int32_t H, int32_t W, const float* mean,
                             const float* stdv, float* x_nchw, void* stream) {
  if (!x_packed || !geom || !mean || !stdv || !x_nchw) return fail(CSNET_E_INVALID, "csnet_resize_u8_to_input: null argument");
  if (N <= 0 || N > 65535 || H <= 0 || W <= 0) return fail(CSNET_E_INVALID, "csnet_resize_u8_to_input: N outside [1, 65535] or empty H x W");
  csnet::launch_resize_in(x_packed, geom, N, H, W, csnet::img_norm(mean, stdv), x_nchw, (cudaStream_t)stream);
  CU_CHECK(cudaGetLastError());
  return CSNET_OK;
}

int csnet_resize_logits_to_u8(const float* logits, int32_t N, int32_t H, int32_t W, const csnet_image_geom* geom, uint8_t* y_packed,
                              void* stream) {
  if (!logits || !geom || !y_packed) return fail(CSNET_E_INVALID, "csnet_resize_logits_to_u8: null argument");
  if (N <= 0 || N > 65535 || H <= 0 || W <= 0) return fail(CSNET_E_INVALID, "csnet_resize_logits_to_u8: N outside [1, 65535] or empty H x W");
  int dev = 0, sms = 0;
  CU_CHECK(cudaGetDevice(&dev));
  CU_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  csnet::launch_resize_out(logits, N, H, W, geom, y_packed, sms, (cudaStream_t)stream);
  CU_CHECK(cudaGetLastError());
  return CSNET_OK;
}

// Training pair of the RESIZE op (fp32): the forward is launch_resize itself, the backward its adjoint (resize_adj.cuh).
int csnet_train_resize_fwd(const float* src, int32_t N, int32_t C, int32_t Hs, int32_t Ws, float* dst, int32_t Hd, int32_t Wd,
                           int32_t accumulate, void* stream) {
  if (!src || !dst || N < 1 || N > 65535 || C < 1 || C > 8 * 65535 || Hs < 1 || Ws < 1 || Hd < 1 || Wd < 1) {
    csnet::train_set_error("csnet_train_resize_fwd: bad arguments");
    return CSNET_E_INVALID;
  }
  csnet::RzArgs A{};
  A.src = src; A.dst = dst;
  A.Cs = C; A.Hs = Hs; A.Ws = Ws; A.c0 = 0;
  A.Cd = C; A.Hd = Hd; A.Wd = Wd; A.cout0 = 0;
  A.C = C; A.accumulate = accumulate != 0;
  A.sy = csnet::resize_scale(Hs, Hd); A.sx = csnet::resize_scale(Ws, Wd);
  csnet::launch_resize(A, CSNET_F32, CSNET_F32, N, (cudaStream_t)stream);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { csnet::train_set_error(cudaGetErrorString(e)); return CSNET_E_CUDA; }
  return CSNET_OK;
}

int csnet_train_resize_bwd(const float* ddst, int32_t N, int32_t C, int32_t Hd, int32_t Wd, float* dsrc, int32_t Hs, int32_t Ws,
                           void* stream) {
  if (!ddst || !dsrc || N < 1 || N > 65535 || C < 1 || C > 65535 || Hs < 1 || Ws < 1 || Hd < 1 || Wd < 1 || (int64_t)Hs * Ws > (1 << 30)) {
    csnet::train_set_error("csnet_train_resize_bwd: bad arguments");
    return CSNET_E_INVALID;
  }
  const dim3 grid((unsigned)((Hs * Ws + csnet::kRzAdjThreads - 1) / csnet::kRzAdjThreads), (unsigned)C, (unsigned)N);
  csnet::resize_bwd_kernel<<<grid, csnet::kRzAdjThreads, 0, (cudaStream_t)stream>>>(ddst, dsrc, C, Hs, Ws, Hd, Wd,
                                                                                   csnet::resize_scale(Hs, Hd), csnet::resize_scale(Ws, Wd));
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { csnet::train_set_error(cudaGetErrorString(e)); return CSNET_E_CUDA; }
  return CSNET_OK;
}

int csnet_salmetric_images_u8(const float* logits, int32_t N, int32_t H, int32_t W, const csnet_image_geom* geom, const uint8_t* m_packed,
                              uint8_t* y_packed, uint32_t* hist_all, uint32_t* hist_pos, unsigned long long* abs_sum, void* stream) {
  if (!logits || !geom || !m_packed || !hist_all || !hist_pos || !abs_sum)
    return fail(CSNET_E_INVALID, "csnet_salmetric_images_u8: null argument");
  if (N <= 0 || N > 65535 || H <= 0 || W <= 0 || H > csnet::kMaxImageSide || W > csnet::kMaxImageSide)
    return fail(CSNET_E_INVALID, "csnet_salmetric_images_u8: N outside [1, 65535] or H, W outside [1, 32767]");
  cudaStream_t st = (cudaStream_t)stream;
  int dev = 0, sms = 0;
  CU_CHECK(cudaGetDevice(&dev));
  CU_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  CU_CHECK(cudaMemsetAsync(hist_all, 0, (size_t)N * 256 * sizeof(uint32_t), st));
  CU_CHECK(cudaMemsetAsync(hist_pos, 0, (size_t)N * 256 * sizeof(uint32_t), st));
  CU_CHECK(cudaMemsetAsync(abs_sum, 0, (size_t)N * sizeof(unsigned long long), st));
  csnet::launch_salmetric_images(logits, N, H, W, geom, m_packed, y_packed, hist_all, hist_pos, abs_sum, sms, st);
  CU_CHECK(cudaGetLastError());
  return CSNET_OK;
}

int csnet_csf_input_u8(const uint8_t* x_packed, const csnet_image_geom* geom, int32_t N, int32_t H, int32_t W, const double* mean,
                       const double* stdv, float* x_nchw, void* stream) {
  if (!x_packed || !geom || !mean || !stdv || !x_nchw) return fail(CSNET_E_INVALID, "csnet_csf_input_u8: null argument");
  if (N <= 0 || N > 65535 || H <= 0 || W <= 0 || H > csnet::kMaxImageSide || W > csnet::kMaxImageSide)
    return fail(CSNET_E_INVALID, "csnet_csf_input_u8: N outside [1, 65535] or H, W outside [1, 32767]");
  csnet::launch_csf_input(x_packed, geom, N, H, W, csnet::img_norm(mean, stdv), x_nchw, (cudaStream_t)stream);
  CU_CHECK(cudaGetLastError());
  return CSNET_OK;
}

int csnet_csf_train_batch_u8(const uint8_t* x_packed, const uint8_t* m_packed, const csnet_image_geom* geom, const csnet_train_sample* samples,
                             int32_t N, int32_t H, int32_t W, const double* mean, const double* stdv, float* x_nchw, float* target,
                             void* stream) {
  if (!x_packed || !m_packed || !geom || !samples || !mean || !stdv || !x_nchw || !target)
    return fail(CSNET_E_INVALID, "csnet_csf_train_batch_u8: null argument");
  if (N <= 0 || N > 65535 || H <= 0 || W <= 0 || H > csnet::kMaxImageSide || W > csnet::kMaxImageSide)
    return fail(CSNET_E_INVALID, "csnet_csf_train_batch_u8: N outside [1, 65535] or H, W outside [1, 32767]");
  csnet::launch_csf_train_batch(x_packed, m_packed, geom, samples, N, H, W, csnet::img_norm(mean, stdv), x_nchw, target,
                                (cudaStream_t)stream);
  CU_CHECK(cudaGetLastError());
  return CSNET_OK;
}

int csnet_csf_maps_u8(const float* logits, int32_t N, int32_t H, int32_t W, const csnet_image_geom* geom, uint8_t* y_packed, void* stream) {
  if (!logits || !geom || !y_packed) return fail(CSNET_E_INVALID, "csnet_csf_maps_u8: null argument");
  if (N <= 0 || N > 65535 || H <= 0 || W <= 0 || H > csnet::kMaxImageSide || W > csnet::kMaxImageSide)
    return fail(CSNET_E_INVALID, "csnet_csf_maps_u8: N outside [1, 65535] or H, W outside [1, 32767]");
  int dev = 0, sms = 0;
  CU_CHECK(cudaGetDevice(&dev));
  CU_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  csnet::launch_resize_out<csnet::CsfMap>(logits, N, H, W, geom, y_packed, sms, (cudaStream_t)stream);
  CU_CHECK(cudaGetLastError());
  return CSNET_OK;
}

int csnet_salmetric_csf_u8(const float* logits, int32_t N, int32_t H, int32_t W, const csnet_image_geom* geom, const uint8_t* m_packed,
                           uint8_t* y_packed, uint32_t* hist_all, uint32_t* hist_pos, unsigned long long* abs_sum, void* stream) {
  if (!logits || !geom || !m_packed || !hist_all || !hist_pos || !abs_sum)
    return fail(CSNET_E_INVALID, "csnet_salmetric_csf_u8: null argument");
  if (N <= 0 || N > 65535 || H <= 0 || W <= 0 || H > csnet::kMaxImageSide || W > csnet::kMaxImageSide)
    return fail(CSNET_E_INVALID, "csnet_salmetric_csf_u8: N outside [1, 65535] or H, W outside [1, 32767]");
  cudaStream_t st = (cudaStream_t)stream;
  int dev = 0, sms = 0;
  CU_CHECK(cudaGetDevice(&dev));
  CU_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  CU_CHECK(cudaMemsetAsync(hist_all, 0, (size_t)N * 256 * sizeof(uint32_t), st));
  CU_CHECK(cudaMemsetAsync(hist_pos, 0, (size_t)N * 256 * sizeof(uint32_t), st));
  CU_CHECK(cudaMemsetAsync(abs_sum, 0, (size_t)N * sizeof(unsigned long long), st));
  csnet::launch_salmetric_images<csnet::CsfMap>(logits, N, H, W, geom, m_packed, y_packed, hist_all, hist_pos, abs_sum, sms, st);
  CU_CHECK(cudaGetLastError());
  return CSNET_OK;
}

int csnet_train_batch_u8(const uint8_t* x_packed, const uint8_t* m_packed, const csnet_image_geom* geom, const csnet_train_sample* samples,
                         int32_t N, int32_t H, int32_t W, const float* mean, const float* stdv, float* x_nchw, float* target, void* stream) {
  if (!x_packed || !m_packed || !geom || !samples || !mean || !stdv || !x_nchw || !target)
    return fail(CSNET_E_INVALID, "csnet_train_batch_u8: null argument");
  if (N <= 0 || N > 65535 || H <= 0 || W <= 0 || H > csnet::kMaxImageSide || W > csnet::kMaxImageSide)
    return fail(CSNET_E_INVALID, "csnet_train_batch_u8: N outside [1, 65535] or H, W outside [1, 32767]");
  csnet::launch_train_batch(x_packed, m_packed, geom, samples, N, H, W, csnet::img_norm(mean, stdv), x_nchw, target, (cudaStream_t)stream);
  CU_CHECK(cudaGetLastError());
  return CSNET_OK;
}

int csnet_val_mae_u8(const float* logits, int32_t N, int32_t H, int32_t W, const uint8_t* m_packed, const csnet_image_geom* geom,
                     double* mae, void* stream) {
  if (!logits || !m_packed || !geom || !mae) return fail(CSNET_E_INVALID, "csnet_val_mae_u8: null argument");
  if (N <= 0 || N > 65535 || H <= 0 || W <= 0 || H > csnet::kMaxImageSide || W > csnet::kMaxImageSide)
    return fail(CSNET_E_INVALID, "csnet_val_mae_u8: N outside [1, 65535] or H, W outside [1, 32767]");
  csnet::launch_val_mae(logits, N, H, W, m_packed, geom, mae, (cudaStream_t)stream);
  CU_CHECK(cudaGetLastError());
  return CSNET_OK;
}

// csnet_plan_run_host_images_u8's geometry, checked before anything is copied or launched.
static int check_images(const csnet_image_geom* g, int32_t N, int64_t x_bytes, int64_t y_bytes) {
  for (int32_t i = 0; i < N; ++i) {
    auto bad = [&](const char* why) { return fail(CSNET_E_INVALID, "run_host_images_u8: image " + std::to_string(i) + why); };
    if (g[i].h < 1 || g[i].w < 1 || g[i].h > csnet::kMaxImageSide || g[i].w > csnet::kMaxImageSide) return bad(": h or w outside [1, 32767]");
    const int64_t hw = (int64_t)g[i].h * g[i].w;
    if (g[i].src_off < 0 || g[i].src_off > x_bytes - 3 * hw) return bad(" lies outside the input buffer");
    if (g[i].dst_off < 0 || g[i].dst_off > y_bytes - hw) return bad(": its map lies outside the output buffer");
    if (i > 0 && g[i].dst_off != g[i - 1].dst_off + (int64_t)g[i - 1].h * g[i - 1].w)
      return bad(": its map does not start where the previous one ends");
  }
  return CSNET_OK;
}

// Ping-pong staging pair that only ever grows.
static cudaError_t grow_staging(void* (&buf)[2], size_t& bytes, size_t need) {
  if (need <= bytes) return cudaSuccess;
  bytes = 0;
  for (int b = 0; b < 2; ++b) {
    if (buf[b]) cudaFree(buf[b]);
    buf[b] = nullptr;
    const cudaError_t e = cudaMalloc(&buf[b], need);
    if (e != cudaSuccess) return e;
  }
  bytes = need;
  return cudaSuccess;
}

static int run_host_impl(csnet_plan* P, int32_t N, const void* x_host, void* y_host, void* stream_, HostIo io, const float* mean,
                         const float* stdv, const HostImages* im) {
  if (!P || !x_host || !y_host) return fail(CSNET_E_INVALID, "null argument");
  if (N <= 0 || N > P->max_batch) return fail(CSNET_E_INVALID, "batch size outside [1, max_batch]");
  if (P->n_ext != 2) return fail(CSNET_E_INVALID, "run_host needs a plan with externals {0: input, 1: logits}");
  const csnet_tensor_desc *in = nullptr, *lo = nullptr;
  for (const auto& d : P->tensors) {
    if (d.external == 0) in = &d;
    if (d.external == 1) lo = &d;
  }
  if (!in || !lo || in->dtype != CSNET_F32 || lo->dtype != CSNET_F32)
    return fail(CSNET_E_INVALID, "run_host: externals must be fp32");
  if (io != HostIo::F32 && in->C != 3) return fail(CSNET_E_INVALID, "run_host_u8: the network input must have 3 channels");
  if (io == HostIo::Images) {
    if (lo->C != 1) return fail(CSNET_E_INVALID, "run_host_images_u8: the logits must have 1 channel");
    if (N > 65535) return fail(CSNET_E_INVALID, "run_host_images_u8: more than 65535 images");
    const int rc = check_images(im->geom, N, im->x_bytes, im->y_bytes);
    if (rc != CSNET_OK) return rc;
  }
  cudaStream_t stream = (cudaStream_t)stream_;
  DeviceGuard guard_(P->device);
  // The batch is cut into chunks that flow through a three-stage pipeline: H2D copy (own stream) -> program
  // (caller's stream) -> D2H copy (own stream), with ping-pong device staging, so the PCIe copies of chunk i+1 / i-1
  // overlap the kernels of chunk i.  Pinned host memory is needed for the copies to be truly asynchronous.
  // Schedule: batches under 64 images run as one chunk.  Larger fp32 batches run a small first and last chunk (N/8 images)
  // that keep the exposed copies short — the first H2D and the last D2H are the only ones nothing overlaps — and one large
  // middle chunk that keeps the kernels at large-batch efficiency.  The uint8 form's copies are 4x smaller: one chunk.
  // Measured at bs 256: fp32 32 / 192 / 32 16.5 ms (4 equal chunks 25.2 ms, 2 equal 24.5 ms, ramps of 4-6 chunks 17.3-20.0 ms);
  // uint8 one chunk 14.7 ms (32 / 192 / 32 16.1 ms).
  // Ragged images run the fp32 schedule: their copies scale with the images, not with the network size.  Measured at bs 256,
  // h, w in [180, 520] (91 MB in, 30 MB out), fp16 csnet-L-x2 at 224x224 on an H100 80GB HBM3 at 700 W: 32 / 192 / 32 19.60 /
  // 19.47 ms, one chunk 19.79 / 18.91 ms; the same within the spread, and the edge chunks bound the exposed copies for larger images.
  const int edge = N < 64 || io == HostIo::U8 ? 0 : N * 32 / 256;
  int sizes[3], n_sizes = 0;
  if (edge > 0) sizes[n_sizes++] = edge;
  sizes[n_sizes++] = N - 2 * edge;
  if (edge > 0) sizes[n_sizes++] = edge;
  int chunk = 0;
  for (int i = 0; i < n_sizes; ++i) chunk = sizes[i] > chunk ? sizes[i] : chunk;
  const size_t xin = (size_t)in->C * in->H * in->W * sizeof(float), yout = (size_t)lo->C * lo->H * lo->W * sizeof(float);
  if (!P->s_h2d) {
    CU_CHECK(cudaStreamCreateWithFlags(&P->s_h2d, cudaStreamNonBlocking));
    CU_CHECK(cudaStreamCreateWithFlags(&P->s_d2h, cudaStreamNonBlocking));
    for (int b = 0; b < 2; ++b) {
      CU_CHECK(cudaEventCreateWithFlags(&P->ev_h2d[b], cudaEventDisableTiming));
      CU_CHECK(cudaEventCreateWithFlags(&P->ev_comp[b], cudaEventDisableTiming));
      CU_CHECK(cudaEventCreateWithFlags(&P->ev_d2h[b], cudaEventDisableTiming));
    }
  }
  if (P->h_in_bytes < (size_t)chunk * xin) {
    for (int b = 0; b < 2; ++b) {
      if (P->h_in[b]) cudaFree(P->h_in[b]);
      if (P->h_out[b]) cudaFree(P->h_out[b]);
      CU_CHECK(cudaMalloc(&P->h_in[b], (size_t)chunk * xin));
      CU_CHECK(cudaMalloc(&P->h_out[b], (size_t)chunk * yout));
    }
    P->h_in_bytes = (size_t)chunk * xin;
    P->h_out_bytes = (size_t)chunk * yout;
  }
  const size_t xin8 = xin / sizeof(float), yout8 = yout / sizeof(float);      // bytes per image of the uint8 forms
  // uint8 staging: the largest chunk's bytes.  Ragged images: the largest byte range that one chunk's images (maps) cover in the
  // packed input (output); each chunk copies its range, and its geometry is rebased to the staging buffers.
  size_t in8 = io == HostIo::U8 ? (size_t)chunk * xin8 : 0, out8 = io == HostIo::U8 ? (size_t)chunk * yout8 : 0;
  int64_t x_lo[3] = {}, x_len[3] = {}, y_lo[3] = {}, y_len[3] = {};
  std::vector<csnet_image_geom> geom;
  if (io == HostIo::Images) {
    geom.assign(im->geom, im->geom + N);
    for (int it = 0, n0 = 0; it < n_sizes; n0 += sizes[it], ++it) {
      const int n1 = n0 + sizes[it];
      int64_t a = INT64_MAX, z = 0;
      for (int n = n0; n < n1; ++n) {
        const int64_t s = geom[n].src_off, e = s + 3 * (int64_t)geom[n].h * geom[n].w;
        a = s < a ? s : a;
        z = e > z ? e : z;
      }
      x_lo[it] = a;
      x_len[it] = z - a;
      y_lo[it] = geom[n0].dst_off;
      y_len[it] = geom[n1 - 1].dst_off + (int64_t)geom[n1 - 1].h * geom[n1 - 1].w - y_lo[it];
      for (int n = n0; n < n1; ++n) { geom[n].src_off -= x_lo[it]; geom[n].dst_off -= y_lo[it]; }
      in8 = (size_t)x_len[it] > in8 ? (size_t)x_len[it] : in8;
      out8 = (size_t)y_len[it] > out8 ? (size_t)y_len[it] : out8;
    }
  }
  CU_CHECK(grow_staging(P->h_in8, P->h_in8_bytes, in8));
  CU_CHECK(grow_staging(P->h_out8, P->h_out8_bytes, out8));
  if (io == HostIo::Images) {
    if (P->h_geom_n < N) {
      if (P->h_geom) cudaFree(P->h_geom);
      P->h_geom = nullptr;
      P->h_geom_n = 0;
      CU_CHECK(cudaMalloc(&P->h_geom, (size_t)N * sizeof(csnet_image_geom)));
      P->h_geom_n = N;
    }
    // every chunk's rebased geometry in one upload, ahead of the first chunk's images on the same stream
    CU_CHECK(cudaMemcpyAsync(P->h_geom, geom.data(), (size_t)N * sizeof(csnet_image_geom), cudaMemcpyHostToDevice, P->s_h2d));
  }
  PreArgs PA{};
  if (io == HostIo::U8) for (int c = 0; c < 3; ++c) { PA.mean[c] = (double)mean[c]; PA.std[c] = (double)stdv[c]; }
  const csnet::ImgNorm IA = io == HostIo::Images ? csnet::img_norm(mean, stdv) : csnet::ImgNorm{};
  int rc = CSNET_OK;
  for (int it = 0, n0 = 0; it < n_sizes && rc == CSNET_OK; n0 += sizes[it], ++it) {
    const int b = it & 1, nb = sizes[it];
    if (it >= 2) CU_CHECK(cudaStreamWaitEvent(P->s_h2d, P->ev_comp[b], 0));     // staging input b was consumed
    if (io == HostIo::U8) CU_CHECK(cudaMemcpyAsync(P->h_in8[b], (const uint8_t*)x_host + (size_t)n0 * xin8, (size_t)nb * xin8, cudaMemcpyHostToDevice, P->s_h2d));
    else if (io == HostIo::Images) CU_CHECK(cudaMemcpyAsync(P->h_in8[b], (const uint8_t*)x_host + x_lo[it], (size_t)x_len[it], cudaMemcpyHostToDevice, P->s_h2d));
    else CU_CHECK(cudaMemcpyAsync(P->h_in[b], (const float*)x_host + (size_t)n0 * (xin / sizeof(float)), (size_t)nb * xin, cudaMemcpyHostToDevice, P->s_h2d));
    CU_CHECK(cudaEventRecord(P->ev_h2d[b], P->s_h2d));
    CU_CHECK(cudaStreamWaitEvent(stream, P->ev_h2d[b], 0));
    if (it >= 2) CU_CHECK(cudaStreamWaitEvent(stream, P->ev_d2h[b], 0));         // staging output b was drained
    if (io == HostIo::U8) {
      const int64_t npix = (int64_t)nb * in->H * in->W;
      pre_u8_kernel<<<(unsigned)((npix + kThreads - 1) / kThreads), kThreads, 0, stream>>>((const uint8_t*)P->h_in8[b], (float*)P->h_in[b], npix, (int64_t)in->H * in->W, PA);
    }
    if (io == HostIo::Images) {
      csnet::launch_resize_in((const uint8_t*)P->h_in8[b], P->h_geom + n0, nb, in->H, in->W, IA, (float*)P->h_in[b], stream);
      CU_CHECK(cudaGetLastError());
    }
    const void* ext[2] = {P->h_in[b], P->h_out[b]};
    rc = run_ops(P, nb, ext, stream);               // (its own staging: no graph path)
    if (rc != CSNET_OK) break;
    if (io == HostIo::U8) {
      const int64_t nel = (int64_t)nb * lo->C * lo->H * lo->W;
      post_u8_kernel<<<(unsigned)((nel / 4 + kThreads - 1) / kThreads), kThreads, 0, stream>>>((const float*)P->h_out[b], (uint8_t*)P->h_out8[b], nel);
    }
    if (io == HostIo::Images) {
      csnet::launch_resize_out((const float*)P->h_out[b], nb, lo->H, lo->W, P->h_geom + n0, (uint8_t*)P->h_out8[b], P->num_sms, stream);
      CU_CHECK(cudaGetLastError());
    }
    CU_CHECK(cudaEventRecord(P->ev_comp[b], stream));
    CU_CHECK(cudaStreamWaitEvent(P->s_d2h, P->ev_comp[b], 0));
    if (io == HostIo::U8) CU_CHECK(cudaMemcpyAsync((uint8_t*)y_host + (size_t)n0 * yout8, P->h_out8[b], (size_t)nb * yout8, cudaMemcpyDeviceToHost, P->s_d2h));
    else if (io == HostIo::Images) CU_CHECK(cudaMemcpyAsync((uint8_t*)y_host + y_lo[it], P->h_out8[b], (size_t)y_len[it], cudaMemcpyDeviceToHost, P->s_d2h));
    else CU_CHECK(cudaMemcpyAsync((float*)y_host + (size_t)n0 * (yout / sizeof(float)), P->h_out[b], (size_t)nb * yout, cudaMemcpyDeviceToHost, P->s_d2h));
    CU_CHECK(cudaEventRecord(P->ev_d2h[b], P->s_d2h));
  }
  cudaError_t e1 = cudaStreamSynchronize(P->s_d2h), e2 = cudaStreamSynchronize(stream), e3 = cudaStreamSynchronize(P->s_h2d);
  if (rc == CSNET_OK && (e1 != cudaSuccess || e2 != cudaSuccess || e3 != cudaSuccess))
    rc = fail(CSNET_E_CUDA, std::string("run_host sync: ") + cudaGetErrorString(e1 != cudaSuccess ? e1 : (e2 != cudaSuccess ? e2 : e3)));
  return rc;
}

}  // extern "C"
