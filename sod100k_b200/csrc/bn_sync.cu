// bn_sync.cu — synchronized train-mode BatchNorm + PReLU (nn.SyncBatchNorm) for the CSNet training step, C ABI `csnet_train_bn_sync_*`.
//
// With G ranks each holding a shard of the global batch, the statistics and the backward sums are those of the whole batch.
// Each direction is two entry points around one collective the caller issues: dist.all_reduce(SUM) on a zeroed float64 row
// buffer [G][C][k] in which rank r fills only row r.  Every element has one nonzero term, so the sum is an exact gather
// (x + 0 == x) whatever order the collective adds in, and every rank then merges the same numbers in rank order: the ranks
// hold bit-identical statistics, and shards may have any sizes.
//
//   forward   _partial   (count, mean_r, M2_r) of this rank's shard, float64, into row `rank` of [G][C][3]: the grid, shift K and
//                        ordered last-block merge of bn_stats_body; M2_r = S2 - S1^2 / M over the shifted sums
//             _merge     one thread per channel merges rows 0..G-1 in rank order with Chan's pairwise update in double and writes
//                        the fp32 mean and biased variance csnet_train_bn_prelu_fwd[_bf16] takes, and the global count
//   backward  _bwd_reduce  the grid and ordered merge of bn_prelu_bwd_reduce_body: local dbeta / dgamma / dslope (parameter
//                        gradients: the caller's gradient all-reduce sums them) and (S1, S2) in float64 into row `rank` of [G][C][2]
//             _bwd_apply dz = gamma r (du - sum S1 / M - xhat sum S2 / M), the rows summed in rank order, M the global count
//
// No floating-point atomics: the same bits on every run.  Activations are fp32 or bf16 (`dtype`); statistics, sums and
// gradients of the parameters are fp32 / float64 either way.
#include <cuda_runtime.h>

#include <string>

#include "../../include/csnet_b200.h"
#include "train_body.cuh"
#include "train_host.h"

namespace csnet {
namespace bs {

using tf::bf16;
using tf::f32;
using tf::kT;
using tf::ldg1;

// row[3c..3c+2] = (M, K + S1 / M, S2 - S1^2 / M) of channel c over this shard
template <class T>
__device__ __forceinline__ void partial_body(const T* __restrict__ z, int N, int C, int HW, int S, double* row, float* ws, unsigned* cnt) {
  const int c = blockIdx.x, part = blockIdx.y, parts = gridDim.y, n = part / S, sg = part - n * S;
  const int seg = (HW + S - 1) / S, i0 = sg * seg, i1 = (i0 + seg) < HW ? (i0 + seg) : HW;
  const T* p = z + ((size_t)n * C + c) * HW;
  __shared__ float Ks;
  if (threadIdx.x < 32) {
    const int l = threadIdx.x, img = l % N, off = (int)(((long long)l * HW) / 32 + 17) % HW;
    const float v = tf::warp_sum(ldg1(z + ((size_t)img * C + c) * HW + off)) * (1.f / 32.f);
    if (l == 0) Ks = v;
  }
  __syncthreads();
  const float K = Ks;
  float s = 0.f, q = 0.f, d1 = 0.f;
  if (((HW | i0) & 3) == 0 && ((i1 - i0) & 3) == 0) {
    const typename tf::Vec4<T>::type* p4 = reinterpret_cast<const typename tf::Vec4<T>::type*>(p + i0);
    for (int i = threadIdx.x; i < (i1 - i0) / 4; i += kT) {
      const float4 v = tf::to_f4(__ldg(p4 + i));
      const float a = v.x - K, b = v.y - K, cc = v.z - K, d = v.w - K;
      s += (a + b) + (cc + d);
      q += (a * a + b * b) + (cc * cc + d * d);
    }
  } else {
    for (int i = i0 + threadIdx.x; i < i1; i += kT) { const float d = f32(p[i]) - K; s += d; q += d * d; }
  }
  tf::block_sum3(s, q, d1);
  float* w = ws + ((size_t)c * parts + part) * 3;
  if (threadIdx.x == 0) { w[0] = s; w[1] = q; w[2] = (float)(i1 > i0 ? i1 - i0 : 0); }
  if (!tf::last_block_of(cnt + c, parts)) return;
  if (threadIdx.x == 0) {
    __threadfence();
    const volatile float* v = ws + (size_t)c * parts * 3;
    double S1 = 0.0, S2 = 0.0, M = 0.0;
    for (int k = 0; k < parts; ++k) { S1 += (double)v[3 * k]; S2 += (double)v[3 * k + 1]; M += (double)v[3 * k + 2]; }
    const double m1 = S1 / M, m2 = S2 - S1 * m1;
    row[3 * c] = M; row[3 * c + 1] = (double)K + m1; row[3 * c + 2] = m2 > 0.0 ? m2 : 0.0;
    cnt[c] = 0u;
  }
}

// row[2c], row[2c+1] = S1 = sum du, S2 = sum du * xhat over this shard (mean / var: the global statistics)
template <class T>
__device__ __forceinline__ void bwd_reduce_body(const T* __restrict__ z, const T* __restrict__ dy, int N, int C, int HW, int S, const float* mean,
                                                const float* var, const float* gamma, const float* beta, const float* slope, float eps,
                                                float* dgamma, float* dbeta, float* dslope, double* row, float* ws, unsigned* cnt) {
  const int c = blockIdx.x, part = blockIdx.y, parts = gridDim.y, n = part / S, sg = part - n * S;
  const int seg = (HW + S - 1) / S, i0 = sg * seg, i1 = (i0 + seg) < HW ? (i0 + seg) : HW;
  const float mu = mean[c], r = rsqrtf(var[c] + eps), g = gamma[c], b = beta[c], a = slope[c];
  float s1 = 0.f, s2 = 0.f, s3 = 0.f;
  const T* p = z + ((size_t)n * C + c) * HW;
  const T* q = dy + ((size_t)n * C + c) * HW;
  for (int i = i0 + threadIdx.x; i < i1; i += kT) {
    const float xh = (f32(p[i]) - mu) * r, u = g * xh + b, d = f32(q[i]);
    const float du = u > 0.f ? d : a * d;
    s1 += du; s2 += du * xh;
    if (!(u > 0.f)) s3 += d * u;
  }
  tf::block_sum3(s1, s2, s3);
  float* w = ws + ((size_t)c * parts + part) * 3;
  if (threadIdx.x == 0) { w[0] = s1; w[1] = s2; w[2] = s3; }
  if (!tf::last_block_of(cnt + c, parts)) return;
  if (threadIdx.x == 0) {
    __threadfence();
    const volatile float* v = ws + (size_t)c * parts * 3;
    double t1 = 0.0, t2 = 0.0, t3 = 0.0;
    for (int k = 0; k < parts; ++k) { t1 += (double)v[3 * k]; t2 += (double)v[3 * k + 1]; t3 += (double)v[3 * k + 2]; }
    dbeta[c] = (float)t1; dgamma[c] = (float)t2; dslope[c] = (float)t3;
    row[2 * c] = t1; row[2 * c + 1] = t2;
    cnt[c] = 0u;
  }
}

template <class T>
__device__ __forceinline__ void bwd_apply_body(const T* __restrict__ z, const T* __restrict__ dy, T* __restrict__ dz, int C, int HW, const float* mean,
                                               const float* var, const float* gamma, const float* beta, const float* slope, float eps,
                                               const double* rows, int G, const double* count) {
  const int c = blockIdx.x, n = blockIdx.y;
  __shared__ float sm[2];
  if (threadIdx.x == 0) {
    double t1 = 0.0, t2 = 0.0;
    for (int k = 0; k < G; ++k) { t1 += rows[((size_t)k * C + c) * 2]; t2 += rows[((size_t)k * C + c) * 2 + 1]; }
    const double M = *count;
    sm[0] = (float)(t1 / M); sm[1] = (float)(t2 / M);
  }
  __syncthreads();
  const float mu = mean[c], r = rsqrtf(var[c] + eps), g = gamma[c], b = beta[c], a = slope[c], m1 = sm[0], m2 = sm[1];
  const size_t off = ((size_t)n * C + c) * HW;
  for (int i = threadIdx.x; i < HW; i += kT) {
    const float xh = (f32(z[off + i]) - mu) * r, u = g * xh + b, d = f32(dy[off + i]);
    const float du = u > 0.f ? d : a * d;
    dz[off + i] = tf::store_as<T>(g * r * (du - m1 - xh * m2));
  }
}

template <class T>
__global__ void __launch_bounds__(kT) bn_sync_partial_kernel(const T* __restrict__ z, int N, int C, int HW, int S, double* row, float* ws,
                                                             unsigned* cnt) {
  partial_body(z, N, C, HW, S, row, ws, cnt);
}

__global__ void __launch_bounds__(kT) bn_sync_merge_kernel(const double* __restrict__ rows, int G, int C, float* mean, float* var, double* count) {
  const int c = blockIdx.x * kT + threadIdx.x;
  if (c >= C) return;
  double n = 0.0, mu = 0.0, m2 = 0.0;
  for (int k = 0; k < G; ++k) {
    const double* p = rows + ((size_t)k * C + c) * 3;
    const double nb = p[0];
    if (!(nb > 0.0)) continue;                               // an empty shard adds nothing
    const double t = n + nb, d = p[1] - mu, f = nb / t;
    mu += d * f;
    m2 += p[2] + d * d * n * f;                              // Chan et al.: M2 = M2_a + M2_b + d^2 n_a n_b / (n_a + n_b)
    n = t;
  }
  const double v = n > 0.0 ? m2 / n : 0.0;
  mean[c] = (float)mu;
  var[c] = (float)(v > 0.0 ? v : 0.0);
  if (c == 0) *count = n;
}

template <class T>
__global__ void __launch_bounds__(kT) bn_sync_bwd_reduce_kernel(const T* __restrict__ z, const T* __restrict__ dy, int N, int C, int HW, int S,
                                                                const float* mean, const float* var, const float* gamma, const float* beta,
                                                                const float* slope, float eps, float* dgamma, float* dbeta, float* dslope,
                                                                double* row, float* ws, unsigned* cnt) {
  bwd_reduce_body(z, dy, N, C, HW, S, mean, var, gamma, beta, slope, eps, dgamma, dbeta, dslope, row, ws, cnt);
}

template <class T>
__global__ void __launch_bounds__(kT) bn_sync_bwd_apply_kernel(const T* __restrict__ z, const T* __restrict__ dy, T* __restrict__ dz, int C, int HW,
                                                               const float* mean, const float* var, const float* gamma, const float* beta,
                                                               const float* slope, float eps, const double* rows, int G, const double* count) {
  bwd_apply_body(z, dy, dz, C, HW, mean, var, gamma, beta, slope, eps, rows, G, count);
}

// ---- host ------------------------------------------------------------------------------------------------------------------------
int fail(int code, const std::string& msg) {
  train_set_error(msg.c_str());
  return code;
}

#define BS_CHECK(expr)                                                                              \
  do {                                                                                              \
    cudaError_t e_ = (expr);                                                                        \
    if (e_ != cudaSuccess) return fail(CSNET_E_CUDA, std::string(#expr) + ": " + cudaGetErrorString(e_)); \
  } while (0)

bool bad_shape(int dtype, int N, int C, int HW) { return (dtype != CSNET_F32 && dtype != CSNET_BF16) || N < 1 || C < 1 || HW < 1; }

}  // namespace bs
}  // namespace csnet

using namespace csnet::bs;
using csnet::tf::bf16;

extern "C" {

int csnet_train_bn_sync_partial(const void* z, int32_t dtype, int32_t N, int32_t C, int32_t HW, int32_t rank, double* rows, void* stream) {
  if (!z || !rows || bad_shape(dtype, N, C, HW) || rank < 0) return fail(CSNET_E_INVALID, "csnet_train_bn_sync_partial: bad arguments");
  const int S = csnet::tr::reduce_segments(N, C, HW);
  float* ws = nullptr;
  unsigned* cnt = nullptr;
  if (int rc = csnet::tr::reduce_workspace(C, N * S, (cudaStream_t)stream, &ws, &cnt)) return rc;
  double* row = rows + (size_t)rank * C * 3;
  const dim3 grid(C, N * S);
  if (dtype == CSNET_BF16)
    bn_sync_partial_kernel<bf16><<<grid, kT, 0, (cudaStream_t)stream>>>(static_cast<const bf16*>(z), N, C, HW, S, row, ws, cnt);
  else
    bn_sync_partial_kernel<float><<<grid, kT, 0, (cudaStream_t)stream>>>(static_cast<const float*>(z), N, C, HW, S, row, ws, cnt);
  BS_CHECK(cudaGetLastError());
  return CSNET_OK;
}

int csnet_train_bn_sync_merge(const double* rows, int32_t G, int32_t C, float* mean, float* var, double* count, void* stream) {
  if (!rows || !mean || !var || !count || G < 1 || C < 1) return fail(CSNET_E_INVALID, "csnet_train_bn_sync_merge: bad arguments");
  bn_sync_merge_kernel<<<(C + kT - 1) / kT, kT, 0, (cudaStream_t)stream>>>(rows, G, C, mean, var, count);
  BS_CHECK(cudaGetLastError());
  return CSNET_OK;
}

int csnet_train_bn_sync_bwd_reduce(const void* z, const void* dy, int32_t dtype, int32_t N, int32_t C, int32_t HW, const float* mean,
                                   const float* var, const float* gamma, const float* beta, const float* slope, float eps, float* dgamma,
                                   float* dbeta, float* dslope, int32_t rank, double* rows, void* stream) {
  if (!z || !dy || !rows || bad_shape(dtype, N, C, HW) || rank < 0) return fail(CSNET_E_INVALID, "csnet_train_bn_sync_bwd_reduce: bad arguments");
  const int S = csnet::tr::reduce_segments(N, C, HW);
  float* ws = nullptr;
  unsigned* cnt = nullptr;
  if (int rc = csnet::tr::reduce_workspace(C, N * S, (cudaStream_t)stream, &ws, &cnt)) return rc;
  double* row = rows + (size_t)rank * C * 2;
  const dim3 grid(C, N * S);
  if (dtype == CSNET_BF16)
    bn_sync_bwd_reduce_kernel<bf16><<<grid, kT, 0, (cudaStream_t)stream>>>(static_cast<const bf16*>(z), static_cast<const bf16*>(dy), N, C, HW, S,
                                                                           mean, var, gamma, beta, slope, eps, dgamma, dbeta, dslope, row, ws, cnt);
  else
    bn_sync_bwd_reduce_kernel<float><<<grid, kT, 0, (cudaStream_t)stream>>>(static_cast<const float*>(z), static_cast<const float*>(dy), N, C, HW,
                                                                            S, mean, var, gamma, beta, slope, eps, dgamma, dbeta, dslope, row, ws,
                                                                            cnt);
  BS_CHECK(cudaGetLastError());
  return CSNET_OK;
}

int csnet_train_bn_sync_bwd_apply(const void* z, const void* dy, void* dz, int32_t dtype, int32_t N, int32_t C, int32_t HW, const float* mean,
                                  const float* var, const float* gamma, const float* beta, const float* slope, float eps, const double* rows,
                                  int32_t G, const double* count, void* stream) {
  if (!z || !dy || !dz || !rows || !count || bad_shape(dtype, N, C, HW) || G < 1)
    return fail(CSNET_E_INVALID, "csnet_train_bn_sync_bwd_apply: bad arguments");
  const dim3 grid(C, N);
  if (dtype == CSNET_BF16)
    bn_sync_bwd_apply_kernel<bf16><<<grid, kT, 0, (cudaStream_t)stream>>>(static_cast<const bf16*>(z), static_cast<const bf16*>(dy),
                                                                          static_cast<bf16*>(dz), C, HW, mean, var, gamma, beta, slope, eps, rows, G,
                                                                          count);
  else
    bn_sync_bwd_apply_kernel<float><<<grid, kT, 0, (cudaStream_t)stream>>>(static_cast<const float*>(z), static_cast<const float*>(dy),
                                                                           static_cast<float*>(dz), C, HW, mean, var, gamma, beta, slope, eps, rows,
                                                                           G, count);
  BS_CHECK(cudaGetLastError());
  return CSNET_OK;
}

}  // extern "C"
