// train_host.h — host-side helpers of the CSNet training entry points, shared by train_ops.cu (fp32 storage) and train_bf16.cu
// (bf16 storage): per-device workspaces, launch geometry of the register-tiled kernels, the ordered merge of weight-gradient partials.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>

#include "../../include/csnet_b200.h"
#include "generic_ops.cuh"
#include "train_body.cuh"

namespace csnet {

void train_set_error(const char* msg);

namespace tr {

namespace tf = csnet::tf;

constexpr int kMaxDevices = 16;
constexpr int kNotHandled = 1;                            // the shape does not fit the fast kernel: the caller runs the generic one
constexpr size_t kFastSmem = 92 * 1024;                   // operand tiles; + kFastWsm of weights: two blocks per SM
constexpr size_t kFastWsm = 16 * 1024;
constexpr int kFastSmemMax = (int)(kFastSmem + kFastWsm);

// The channel-reduction workspace (partials [C][parts][3], one ticket counter per channel) and the weight-gradient partials
// ([blocks][elements] floats) of the current device, grown on demand.
int reduce_workspace(int C, int parts, cudaStream_t st, float** ws, unsigned** cnt);
int partial_workspace(size_t floats, cudaStream_t st, float** out);
int current_device();
int num_sms();
// segments per image plane of the BatchNorm reductions
int reduce_segments(int N, int C, int HW);

MixPath to_path(const csnet_train_path& q);
bool dense_conv_path(const MixPath& P, int H, int W);
bool conv_tile_geometry(tf::ConvArgs& A);
// esize: bytes per element of the staged source tile
bool conv_path_geometry(tf::ConvPath& P, const tf::ConvArgs& A, int esize);

struct WgradPlan {
  tf::WgradArgs A;
  int form, gx, groups, nel;      // form: conv_wgrad template argument (1, 3, 0); grid (gx, groups); nel: weight-gradient elements
  size_t smem;
};
bool wgrad_plan(const MixPath& P, const void* ddst, int N, int C, int H, int W, int esize_in, int esize_dd, WgradPlan& out);
// out[e] = scale * sum over parts, in part order, of part[p][e]
int reduce_partials(const float* part, int parts, int n, float scale, float* out, cudaStream_t st);

}  // namespace tr
}  // namespace csnet
