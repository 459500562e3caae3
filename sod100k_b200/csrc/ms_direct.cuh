// ms_direct.cuh — one dilated 3x3 path of an MSBlock (CSNet/model/csnet.py:116-149: five dilated Conv2dX100, concat, BN,
// PReLU) on 16-bit activations: few output channels (1..8 per dilation), so it is a depthwise-like problem for the FP32 pipe,
// not for the tensor cores.  A thread owns PX output pixels of one row for all of the path's output channels; per (input
// channel, tap row) it loads the needed 8-pixel groups once (16-byte read-only loads, L1-resident across the taps and the
// neighbouring rows), one row ahead of its FMAs, and converts the pixels the taps read to fp32 once.  The weights sit in
// shared memory as the fp32 values of their 16-bit rounding, so every tap is one FFMA on registers and a broadcast shared
// load: the products and their order (ci, ky, kx) are those of a 16-bit x 16-bit + fp32 FMA.  The dilation is a template
// parameter, so every register index is static.
#pragma once
#include "il_stream.cuh"

namespace csnet {

constexpr int kMsdThreads = 128;

struct MsdArgs {
  const uint16_t* src;
  uint16_t* dst;
  const float* w;             // [cin][9][cout] fp32 (BN scale and x100 folded)
  const float* bias;          // [Ctot] (nullptr: none)
  const float* slope;         // [Ctot] (nullptr: none)
  int32_t N, Cin, H, W, Ctot, cout0, cout;
};

template <int D, int PX> struct MsdGeom {
  static constexpr bool kSparse = (D == 16 && PX == 8);                  // only the groups at -16, 0, +16 are needed
  static constexpr int kFirst = D == 16 ? -16 : -8;                      // pixel offset of group 0
  static constexpr int kStep = kSparse ? 16 : 8;
  static constexpr int kGroups = kSparse ? 3 : (D == 16 ? PX / 8 + 4 : PX / 8 + 2);
  __host__ __device__ static constexpr int grp(int i) { return (i - kFirst) / kStep; }       // i: pixel offset from x0
  __host__ __device__ static constexpr int pix(int i) { return (i - kFirst) & 7; }
};

template <typename T, int D, int PX, int COMAX>
__global__ void __launch_bounds__(kMsdThreads) msd_kernel(const __grid_constant__ MsdArgs A) {
  using GEO = MsdGeom<D, PX>;
  static_assert(COMAX % 2 == 0, "weights are read as fp32 pairs");
  extern __shared__ __align__(16) float sw[];                             // [cin][9][COMAX] fp32 values of the 16-bit weights
  const int tid = threadIdx.x;
  for (int i = tid; i < A.Cin * 9 * COMAX; i += kMsdThreads) {
    const int co = i % COMAX, ct = i / COMAX;
    sw[i] = co < A.cout ? Pack<T>::to_f(Pack<T>::bits(__ldg(A.w + (size_t)ct * A.cout + co))) : 0.f;
  }
  __syncthreads();
  const int strips = A.W / PX;
  const long long task = (long long)blockIdx.x * kMsdThreads + tid;
  if (task >= (long long)A.N * A.H * strips) return;
  const int s = (int)(task % strips), y = (int)((task / strips) % A.H), n = (int)(task / ((long long)strips * A.H));
  const int x0 = s * PX, H = A.H, W = A.W;
  float acc[COMAX][PX];
#pragma unroll
  for (int co = 0; co < COMAX; ++co)
#pragma unroll
    for (int p = 0; p < PX; ++p) acc[co][p] = 0.f;
  bool gin[GEO::kGroups];                                                  // group inside the row?
#pragma unroll
  for (int g = 0; g < GEO::kGroups; ++g) {
    const int gx = x0 + GEO::kFirst + g * GEO::kStep;
    gin[g] = gx >= 0 && gx < W;
  }
  const size_t plane = (size_t)H * W;
  const uint16_t* img = A.src + (size_t)n * A.Cin * plane + x0 + GEO::kFirst;
  bool rin[3];                                                             // tap row inside the image? (else zero padding)
#pragma unroll
  for (int ky = 0; ky < 3; ++ky) rin[ky] = y + D * (ky - 1) >= 0 && y + D * (ky - 1) < H;
  // software pipeline over the (ci, ky) rows: the groups of the next row are in flight while this row's FMAs run; a row
  // outside the image is not read
  uint4 cur[GEO::kGroups];
#pragma unroll
  for (int g = 0; g < GEO::kGroups; ++g)
    cur[g] = rin[0] && gin[g] ? __ldg(reinterpret_cast<const uint4*>(img + (ptrdiff_t)(y - D) * W + g * GEO::kStep))
                              : make_uint4(0u, 0u, 0u, 0u);
  for (int ci = 0; ci < A.Cin; ++ci, img += plane) {
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
      const int kn = ky < 2 ? ky + 1 : 0;                                  // next row: (ci, ky + 1) or (ci + 1, 0)
      const uint16_t* next = (ky < 2 ? img : img + plane) + (ptrdiff_t)(y + D * (kn - 1)) * W;
      const bool nin = rin[kn] && (ky < 2 || ci + 1 < A.Cin);
      uint4 nxt[GEO::kGroups];
#pragma unroll
      for (int g = 0; g < GEO::kGroups; ++g)
        nxt[g] = nin && gin[g] ? __ldg(reinterpret_cast<const uint4*>(next + g * GEO::kStep)) : make_uint4(0u, 0u, 0u, 0u);
      if (rin[ky]) {
        float xf[GEO::kGroups * 8];                                          // pixels no tap reads are never converted
#pragma unroll
        for (int g = 0; g < GEO::kGroups; ++g) {
          const uint32_t u[4] = {cur[g].x, cur[g].y, cur[g].z, cur[g].w};
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float2 f = Pack<T>::to_f2(u[j]);
            xf[g * 8 + 2 * j] = f.x; xf[g * 8 + 2 * j + 1] = f.y;
          }
        }
        const float* wrow = sw + (ci * 9 + ky * 3) * COMAX;
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
          float wk[COMAX];
#pragma unroll
          for (int j = 0; j < COMAX; j += 2) {
            const float2 w2 = reinterpret_cast<const float2*>(wrow + kx * COMAX)[j / 2];
            wk[j] = w2.x; wk[j + 1] = w2.y;
          }
#pragma unroll
          for (int co = 0; co < COMAX; ++co) {
            if (co < A.cout) {                                               // uniform
#pragma unroll
              for (int p = 0; p < PX; ++p) {
                const int i = p + D * (kx - 1);                              // static after unrolling
                acc[co][p] = fmaf(xf[GEO::grp(i) * 8 + GEO::pix(i)], wk[co], acc[co][p]);
              }
            }
          }
        }
      }
#pragma unroll
      for (int g = 0; g < GEO::kGroups; ++g) cur[g] = nxt[g];
    }
  }
  uint16_t* out = A.dst + (((size_t)n * A.Ctot + A.cout0) * H + y) * W + x0;
#pragma unroll
  for (int co = 0; co < COMAX; ++co) {
    if (co < A.cout) {
      const float b = A.bias ? __ldg(A.bias + A.cout0 + co) : 0.f, m = A.slope ? __ldg(A.slope + A.cout0 + co) - 1.f : 0.f;
#pragma unroll
      for (int p8 = 0; p8 < PX; p8 += 8) {
        uint4 o;
        o.x = Pack<T>::from_f2(prelu_m1(acc[co][p8 + 0] + b, m), prelu_m1(acc[co][p8 + 1] + b, m));
        o.y = Pack<T>::from_f2(prelu_m1(acc[co][p8 + 2] + b, m), prelu_m1(acc[co][p8 + 3] + b, m));
        o.z = Pack<T>::from_f2(prelu_m1(acc[co][p8 + 4] + b, m), prelu_m1(acc[co][p8 + 5] + b, m));
        o.w = Pack<T>::from_f2(prelu_m1(acc[co][p8 + 6] + b, m), prelu_m1(acc[co][p8 + 7] + b, m));
        *reinterpret_cast<uint4*>(out + (size_t)co * H * W + p8) = o;
      }
    }
  }
}

template <typename T, int PX, int COMAX>
inline void msd_launch_d(int dil, const MsdArgs& A, cudaStream_t st) {
  const long long tasks = (long long)A.N * A.H * (A.W / PX);
  const unsigned grid = (unsigned)((tasks + kMsdThreads - 1) / kMsdThreads);
  const size_t smem = (size_t)A.Cin * 9 * COMAX * sizeof(float);
  switch (dil) {
    case 1: msd_kernel<T, 1, PX, COMAX><<<grid, kMsdThreads, smem, st>>>(A); break;
    case 2: msd_kernel<T, 2, PX, COMAX><<<grid, kMsdThreads, smem, st>>>(A); break;
    case 4: msd_kernel<T, 4, PX, COMAX><<<grid, kMsdThreads, smem, st>>>(A); break;
    case 8: msd_kernel<T, 8, PX, COMAX><<<grid, kMsdThreads, smem, st>>>(A); break;
    default: msd_kernel<T, 16, PX, COMAX><<<grid, kMsdThreads, smem, st>>>(A); break;
  }
}

// one dilated path; cout <= 8.  Wide strips (16 px) for 1-2 output channels: more FMAs per loaded group.
template <typename T>
inline void msd_launch(int dil, const MsdArgs& A, cudaStream_t st) {
  if (A.cout <= 2 && A.W % 16 == 0) msd_launch_d<T, 16, 2>(dil, A, st);
  else if (A.cout <= 4) msd_launch_d<T, 8, 4>(dil, A, st);
  else msd_launch_d<T, 8, 8>(dil, A, st);
}

}  // namespace csnet
