// train_body.cuh — the per-thread bodies of the CSNet training kernels, templated on the element type of the activations they read
// and write (float or __nv_bfloat16).  Weights, weight gradients, BatchNorm statistics, partial sums and every accumulator stay fp32.
//
// The fp32 kernels (train_fast.cuh, train_ops.cu) and the bf16-storage kernels (train_bf16.cu) are thin __global__ wrappers around
// the same bodies, so both storage modes share one reduction order.  With T = float every helper below is the plain fp32 access
// the kernels were written with, so the fp32 instances compile to the same SASS as before the split.
//
// bf16 rounding is round-to-nearest-even (__float2bfloat16_rn) at every store; a bf16 load is exact.  Where an fp32 kernel takes
// one 16-byte vector of 4 pixels, its bf16 instance takes one 8-byte vector of 4 bf16; cp.async tiles hold the storage type.
//
//   conv_fwd_body<KS>     3x3 (KS = 3, dil 1) and dilated (KS = 0) mixes: dst = sum over conv paths (K-concatenated in the loop) + bilinear
//                         resample-add paths; with `transposed` the data gradient of one path (weights read as [co][flipped tap][ci]
//                         while staging); input tile with halo staged by cp.async.
//   conv1x1_body          every 1x1 mix and its data gradient: inputs global -> registers (each input element is needed by exactly one
//                         thread), weights in shared memory, several channels of loads issued ahead of their FMAs.
//   conv_wgrad_body<KS>   dw[ci][tap][co] = sum_{n,y,x} in[n][ci][y+ky-1][x+kx-1] * ddst[n][co][y][x]: per-block partials over a
//                         share of the (image, row band) units, two cp.async stages in flight, interleaved 4 x 4 thread tiles on a
//                         bank-conflict-free channel pitch, merged IN ORDER by reduce_partials_kernel (no atomics).
//   dw3_body / dw3_bwd_body (dw3_wgrad_body)   depthwise 3x3 (Conv2dX100 groups=C): a 4-pixel column strip per thread sliding down
//                         the rows; the backward produces dx and the dw partials in one pass over dy.
//   pool_fwd / pool2_fwd / pool_bwd(4), resample_bwd   the pooling a path carries (with arg-max) and the bilinear adjoint.
//   bn_*                  train-mode BatchNorm + PReLU: statistics, forward (+ the per-image channel means), backward reduce / apply.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <cmath>
#include <cstdint>

namespace csnet {
namespace tf {

using bf16 = __nv_bfloat16;

constexpr int kT = 256;
constexpr int kCoT = 16;            // output channels per thread (forward / dgrad)
constexpr int kMaxConv = 5;         // conv paths of one mix (MSBlock: five dilations)
constexpr int kMaxRs = 3;

// Activation pointers are `void*`: the instance's element type says what they hold.
struct ConvPath {
  const void* src;                  // [N][Cs][H][W]
  const float* w;                   // [cin][k*k][cout]  (forward layout; dgrad reads it transposed)
  int32_t Cs, c0, cin, cout0, cout, dil;
  int32_t halo, Wp, rows, chunk;    // staged tile: rows = R + 2 halo rows of Wp elements (image column x at x + hp), chunk = ci per stage
  int32_t hp;                       // column pad (multiple of 4, >= halo)
};

struct RsPath {
  const void* src;                  // [N][Cs][Hs][Ws], the element type of the conv sources
  int32_t Cs, c0, Hs, Ws, up, cout0, cout;
};

struct ConvArgs {
  void* dst;
  int32_t N, C, H, W;               // destination
  int32_t ksize, transposed;
  int32_t n_conv, n_rs;
  int32_t R, ipb, quads;            // tile: ipb images x R rows; quads = ceil(W / 4)
  int32_t vec;                      // W % 4 == 0: vector global loads / stores
  int32_t tile_floats;              // 4-byte words of shared memory taken by the input tile region (a multiple of 4)
  ConvPath p[kMaxConv];
  RsPath rs[kMaxRs];
};

struct C1Path {
  const void* src;
  const float* w;
  int32_t Cs, c0, cin, cout0, cout, woff;          // woff: first weight row of this path in shared memory
};

struct C1Args {
  void* dst;
  int32_t N, C, H, W, quads, vec, transposed, n_conv, n_rs, Cpad, wrows;
  C1Path p[kMaxConv];
  RsPath rs[kMaxRs];
};

struct WgradArgs {
  const void* in;                   // [N][Cs][H][W], channels [c0, c0 + cin)
  const void* dd;                   // [N][Cd][H][W], channels [cout0, cout0 + cout)
  float* part;                      // [grid][cin * kk * cout] partial sums (block order)
  int32_t N, Cs, c0, cin, Cd, cout0, cout, H, W;
  int32_t R, units;                 // row band; units = N * ceil(H / R)
  int32_t Wp, quads;                // shared-memory pitch (W + 8, multiple of 4), quads = ceil(W / 4)
  int32_t mt, nt, tiles, splits;    // thread tiles: mt = ceil(cin / 4) (x 3 tap rows for 3x3), nt = ceil(cout / 4); splits = pixel splits
  int32_t tpad;                     // tiles per block (grid.y groups of tpad tiles): a multiple of 32, or a power of two < 32
  int32_t cin4, cout4;              // channel counts rounded up to 4 (zero rows)
  int32_t vec;
  int32_t dil, hp;                  // dilation (KS == 0 form) and the column pad of the input tile (multiple of 4, >= dil)
  int32_t cpi, cpd;                 // channel pitches of the two tiles in elements, == 4 (mod 32): the 4-channel thread tiles are interleaved
                                    // (tile t owns channels t, t + M, t + 2M, t + 3M), so the lanes of a warp read distinct bank groups
};

// ---- element access ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float f32(float v) { return v; }
__device__ __forceinline__ float f32(bf16 v) { return __bfloat162float(v); }
template <class T> __device__ __forceinline__ T store_as(float v);
template <> __device__ __forceinline__ float store_as<float>(float v) { return v; }
template <> __device__ __forceinline__ bf16 store_as<bf16>(float v) { return __float2bfloat16_rn(v); }

__device__ __forceinline__ float4 bf4_to_f4(uint2 u) {
  return make_float4(__uint_as_float(u.x << 16), __uint_as_float(u.x & 0xffff0000u), __uint_as_float(u.y << 16),
                     __uint_as_float(u.y & 0xffff0000u));
}
__device__ __forceinline__ uint32_t f2_to_bf2(float a, float b) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);            // a in the low half: the lower address
  return *reinterpret_cast<const uint32_t*>(&h);
}

__device__ __forceinline__ float ldg1(const float* p) { return __ldg(p); }
__device__ __forceinline__ float ldg1(const bf16* p) { return __uint_as_float((uint32_t)__ldg(reinterpret_cast<const unsigned short*>(p)) << 16); }
// one element in its own type (the read-only path)
__device__ __forceinline__ float ldg_raw(const float* p) { return __ldg(p); }
__device__ __forceinline__ bf16 ldg_raw(const bf16* p) { return __ushort_as_bfloat16(__ldg(reinterpret_cast<const unsigned short*>(p))); }
// four consecutive elements: one 16-byte (fp32) or 8-byte (bf16) load
__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ float4 ldg4(const bf16* p) { return bf4_to_f4(__ldg(reinterpret_cast<const uint2*>(p))); }
__device__ __forceinline__ float2 ldg2(const float* p) { return __ldg(reinterpret_cast<const float2*>(p)); }
__device__ __forceinline__ float2 ldg2(const bf16* p) {
  const uint32_t u = __ldg(reinterpret_cast<const unsigned int*>(p));
  return make_float2(__uint_as_float(u << 16), __uint_as_float(u & 0xffff0000u));
}
// four consecutive elements of shared memory
__device__ __forceinline__ float4 lds4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ float4 lds4(const bf16* p) { return bf4_to_f4(*reinterpret_cast<const uint2*>(p)); }
__device__ __forceinline__ void st4(float* p, float a, float b, float c, float d) { *reinterpret_cast<float4*>(p) = make_float4(a, b, c, d); }
__device__ __forceinline__ void st4(bf16* p, float a, float b, float c, float d) { *reinterpret_cast<uint2*>(p) = make_uint2(f2_to_bf2(a, b), f2_to_bf2(c, d)); }
__device__ __forceinline__ void st2(float* p, float a, float b) { *reinterpret_cast<float2*>(p) = make_float2(a, b); }
__device__ __forceinline__ void st2(bf16* p, float a, float b) { *reinterpret_cast<uint32_t*>(p) = f2_to_bf2(a, b); }

// four elements as one vector: float4 / 4 x bf16 in a uint2
template <class T> struct Vec4;
template <> struct Vec4<float> { using type = float4; };
template <> struct Vec4<bf16> { using type = uint2; };
__device__ __forceinline__ float4 to_f4(float4 v) { return v; }
__device__ __forceinline__ float4 to_f4(uint2 u) { return bf4_to_f4(u); }

// 4-byte words taken by n elements (n even for bf16)
template <class T, class N> __host__ __device__ constexpr N words(N n) { return sizeof(T) == 4 ? n : n / 2; }

__device__ __forceinline__ void cp_async16(float* dst_smem, const float* src, bool valid) {
  const uint32_t d = (uint32_t)__cvta_generic_to_shared(dst_smem);
  const int sz = valid ? 16 : 0;                                   // src-size 0: the 16 bytes are zero-filled
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(d), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async4(float* dst_smem, const float* src, bool valid) { cp_async16(dst_smem, src, valid); }
// four bf16: an 8-byte copy (cp.async.cg takes 16 bytes only)
__device__ __forceinline__ void cp_async4(bf16* dst_smem, const bf16* src, bool valid) {
  const uint32_t d = (uint32_t)__cvta_generic_to_shared(dst_smem);
  const int sz = valid ? 8 : 0;
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;\n" ::"r"(d), "l"(src), "r"(sz) : "memory");
}

__device__ __forceinline__ void bilin(int H, int W, int up, int oy, int ox, int& o00, int& o01, int& o10, int& o11, float& w00,
                                      float& w01, float& w10, float& w11) {
  const float inv = 1.f / (float)up;
  float sy = ((float)oy + 0.5f) * inv - 0.5f, sx = ((float)ox + 0.5f) * inv - 0.5f;
  sy = sy < 0.f ? 0.f : sy; sx = sx < 0.f ? 0.f : sx;
  const int y0 = (int)sy, x0 = (int)sx, y1 = y0 + (y0 < H - 1 ? 1 : 0), x1 = x0 + (x0 < W - 1 ? 1 : 0);
  const float ly = sy - (float)y0, lx = sx - (float)x0;
  o00 = y0 * W + x0; o01 = y0 * W + x1; o10 = y1 * W + x0; o11 = y1 * W + x1;
  w00 = (1.f - ly) * (1.f - lx); w01 = (1.f - ly) * lx; w10 = ly * (1.f - lx); w11 = ly * lx;
}

// ---- conv_fwd: KS 3 with dil == 1 (vector shared-memory reads); 0: any ksize / dilation (scalar reads; the MSBlock's dilated
// paths).  Sources (and resample-add sources) are TI, the destination TO; the tile holds TI.
template <int KS, class TI, class TO>
__device__ __forceinline__ void conv_fwd_body(const ConvArgs& A, float* smem) {
  TI* tile = reinterpret_cast<TI*>(smem);                // [chunk][ipb][rows][Wp]
  float* wsm = smem + A.tile_floats;                    // [chunk][kk][kCoT]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int kk = A.ksize * A.ksize, H = A.H, W = A.W, R = A.R, ipb = A.ipb;
  const int bands = (H + R - 1) / R;
  const int n0 = (blockIdx.x / bands) * ipb, r0 = (blockIdx.x % bands) * R;
  const int tasks = ipb * R * A.quads;
  const bool live = tid < tasks;
  const int ti = live ? tid / (R * A.quads) : 0, tr = live ? (tid / A.quads) % R : 0, tq = live ? tid % A.quads : 0;
  const int n = n0 + ti, y = r0 + tr, x0 = 4 * tq;
  const bool ok = live && n < A.N && y < H;
  const size_t plane = (size_t)H * W;

  // one path whose channels fit one stage: the input tile is staged once and reused by every output-channel group
  const bool once = A.n_conv == 1 && A.p[0].chunk >= A.p[0].cin;
  for (int cg = 0; cg * kCoT < A.C; ++cg) {
    const int cb = cg * kCoT;
    float acc[kCoT][4];
#pragma unroll
    for (int c = 0; c < kCoT; ++c) { acc[c][0] = acc[c][1] = acc[c][2] = acc[c][3] = 0.f; }
    for (int pi = 0; pi < A.n_conv; ++pi) {
      const ConvPath& P = A.p[pi];
      if (P.cout0 >= cb + kCoT || P.cout0 + P.cout <= cb) continue;
      const int trows = ipb * P.rows;                                      // staged rows per input channel
      for (int ci0 = 0; ci0 < P.cin; ci0 += P.chunk) {
        const int nc = P.cin - ci0 < P.chunk ? P.cin - ci0 : P.chunk;
        __syncthreads();
        // ---- stage the input tile: one warp per (channel, image, row), zero outside the image -------------------------------
        for (int rr = warp; rr < ((once && cg > 0) ? 0 : nc * trows); rr += kT / 32) {
          const int c = rr / trows, ir = rr - c * trows, i = ir / P.rows, row = ir - i * P.rows;
          const int gy = r0 + row - P.halo, gn = n0 + i;
          TI* d = tile + (size_t)rr * P.Wp;
          const bool inside = gy >= 0 && gy < H && gn < A.N;
          const TI* s = static_cast<const TI*>(P.src) + (((size_t)gn * P.Cs + P.c0 + ci0 + c) * H + (inside ? gy : 0)) * W;
          if (A.vec) {
            for (int v = lane; v * 4 < P.Wp; v += 32) {
              const int xx = v * 4 - P.hp;
              const bool ld = inside && xx >= 0 && xx < W;
              cp_async4(d + v * 4, ld ? s + xx : static_cast<const TI*>(P.src), ld);                 // asynchronous: every row of the stage is in flight at once
            }
          } else {
            for (int v = lane; v < P.Wp; v += 32) {
              const int xx = v - P.hp;
              d[v] = (inside && xx >= 0 && xx < W) ? ldg_raw(s + xx) : TI(0.f);
            }
          }
        }
        asm volatile("cp.async.commit_group;\n" ::: "memory");
        // ---- stage the weights of this (channel chunk, output-channel group); zero outside the path's slice ------------------
        for (int i = tid; i < nc * kk * kCoT; i += kT) {
          const int c = i / (kk * kCoT), t = (i / kCoT) % kk, co = cb + (i % kCoT) - P.cout0;
          float v = 0.f;
          if (co >= 0 && co < P.cout)
            v = A.transposed ? __ldg(P.w + ((size_t)co * kk + (kk - 1 - t)) * P.cin + ci0 + c)       // dgrad: w'[ci'=co][flip t][co'=ci]
                             : __ldg(P.w + ((size_t)(ci0 + c) * kk + t) * P.cout + co);
          wsm[i] = v;
        }
        asm volatile("cp.async.wait_group 0;\n" ::: "memory");
        __syncthreads();
        if (!live) continue;
        // ---- accumulate ---------------------------------------------------------------------------------------------------
        const TI* tb = tile + ((size_t)ti * P.rows + tr) * P.Wp + x0 + P.hp;             // tap (0, 0) of a 1x1; (ky, kx) offsets below
        for (int c = 0; c < nc; ++c) {
          const TI* tc = tb + (size_t)c * trows * P.Wp;
          const float* wc = wsm + c * kk * kCoT;
          if (KS == 3) {
#pragma unroll
            for (int ky = 0; ky < 3; ++ky) {
              const TI* tr_ = tc + (ky * P.Wp) - 4;                                 // halo == 1: rows y-1..y+1 are tile rows tr..tr+2
              const float l = f32(tr_[3]);
              const float4 m = lds4(tr_ + 4);
              const float r = f32(tr_[8]);
              const float in[6] = {l, m.x, m.y, m.z, m.w, r};
#pragma unroll
              for (int kx = 0; kx < 3; ++kx) {
#pragma unroll
                for (int q = 0; q < kCoT / 4; ++q) {
                  const float4 w4 = *reinterpret_cast<const float4*>(wc + (ky * 3 + kx) * kCoT + 4 * q);
                  const float wv[4] = {w4.x, w4.y, w4.z, w4.w};
#pragma unroll
                  for (int j = 0; j < 4; ++j) {
#pragma unroll
                    for (int px = 0; px < 4; ++px) acc[4 * q + j][px] = fmaf(in[px + kx], wv[j], acc[4 * q + j][px]);
                  }
                }
              }
            }
          } else {
            const int ks = A.ksize, hk = ks / 2;
            for (int ky = 0; ky < ks; ++ky) {
              for (int kx = 0; kx < ks; ++kx) {
                const TI* tp = tc + ((ky - hk) * P.dil + P.halo) * P.Wp + (kx - hk) * P.dil;
                const float in[4] = {f32(tp[0]), f32(tp[1]), f32(tp[2]), f32(tp[3])};
#pragma unroll
                for (int q = 0; q < kCoT / 4; ++q) {
                  const float4 w4 = *reinterpret_cast<const float4*>(wc + (ky * ks + kx) * kCoT + 4 * q);
                  const float wv[4] = {w4.x, w4.y, w4.z, w4.w};
#pragma unroll
                  for (int j = 0; j < 4; ++j) {
#pragma unroll
                    for (int px = 0; px < 4; ++px) acc[4 * q + j][px] = fmaf(in[px], wv[j], acc[4 * q + j][px]);
                  }
                }
              }
            }
          }
        }
      }
    }
    if (!ok) continue;
    // ---- resample-add paths (bilinear x up of a low-resolution tensor; align_corners=False, F.interpolate semantics) ------------
    for (int ri = 0; ri < A.n_rs; ++ri) {
      const RsPath& Q = A.rs[ri];
      if (Q.cout0 >= cb + kCoT || Q.cout0 + Q.cout <= cb) continue;
      const size_t lp = (size_t)Q.Hs * Q.Ws;
#pragma unroll
      for (int px = 0; px < 4; ++px) {
        if (x0 + px >= W) continue;
        int o00, o01, o10, o11;
        float w00, w01, w10, w11;
        bilin(Q.Hs, Q.Ws, Q.up, y, x0 + px, o00, o01, o10, o11, w00, w01, w10, w11);
#pragma unroll
        for (int c = 0; c < kCoT; ++c) {
          const int co = cb + c - Q.cout0;
          if (co < 0 || co >= Q.cout) continue;
          const TI* s = static_cast<const TI*>(Q.src) + ((size_t)n * Q.Cs + Q.c0 + co) * lp;
          acc[c][px] += w00 * ldg1(s + o00) + w01 * ldg1(s + o01) + w10 * ldg1(s + o10) + w11 * ldg1(s + o11);
        }
      }
    }
    TO* o = static_cast<TO*>(A.dst) + (((size_t)n * A.C + cb) * H + y) * W + x0;
#pragma unroll
    for (int c = 0; c < kCoT; ++c) {
      if (cb + c >= A.C) break;
      if (A.vec) {
        st4(o + (size_t)c * plane, acc[c][0], acc[c][1], acc[c][2], acc[c][3]);
      } else {
#pragma unroll
        for (int px = 0; px < 4; ++px)
          if (x0 + px < W) o[(size_t)c * plane + px] = store_as<TO>(acc[c][px]);
      }
    }
  }
}

// ---- 1x1 convolution mix, direct form ------------------------------------------------------------------------------------------------
// A 1x1 path needs each input element in exactly one thread (the one that owns its pixel, for every output channel), so the inputs go
// global -> registers as vector loads (re-reads for a second output-channel group hit L1) and only the weights live in shared
// memory: no tile staging, no barriers after the prologue.  Also runs a mix that has only resample-add paths (n_conv == 0).
template <int CT, int PX, bool VEC, int U, class TI, class TO>     // U: input channels loaded ahead of their FMAs (memory-level parallelism)
__device__ __forceinline__ void c1_group(const C1Args& A, const float* wsm, int cb, int n, int y, int x0) {
  const int H = A.H, W = A.W;
  const size_t plane = (size_t)H * W;
  float acc[CT][PX];
#pragma unroll
  for (int c = 0; c < CT; ++c)
#pragma unroll
    for (int px = 0; px < PX; ++px) acc[c][px] = 0.f;
  for (int pi = 0; pi < A.n_conv; ++pi) {
    const C1Path& P = A.p[pi];
    if (P.cout0 >= cb + CT || P.cout0 + P.cout <= cb) continue;
    const TI* s = static_cast<const TI*>(P.src) + (((size_t)n * P.Cs + P.c0) * H + y) * W + x0;
    const float* wr = wsm + (size_t)P.woff * A.Cpad + cb;
    for (int ci0 = 0; ci0 < P.cin; ci0 += U) {
      float v[U][PX];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const TI* q = s + (size_t)(ci0 + u) * plane;
        const bool on = ci0 + u < P.cin;
        if (VEC) {
          if (PX == 4) {
            float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
            if (on) t = ldg4(q);
            v[u][0] = t.x; v[u][1] = t.y; v[u][PX - 2] = t.z; v[u][PX - 1] = t.w;
          } else {
            float2 t = make_float2(0.f, 0.f);
            if (on) t = ldg2(q);
            v[u][0] = t.x; v[u][1] = t.y;
          }
        } else {
#pragma unroll
          for (int px = 0; px < PX; ++px) v[u][px] = (on && x0 + px < W) ? ldg1(q + px) : 0.f;
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (ci0 + u >= P.cin) break;
#pragma unroll
        for (int q4 = 0; q4 < CT / 4; ++q4) {
          const float4 w4 = *reinterpret_cast<const float4*>(wr + (size_t)(ci0 + u) * A.Cpad + 4 * q4);
          const float wv[4] = {w4.x, w4.y, w4.z, w4.w};
#pragma unroll
          for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int px = 0; px < PX; ++px) acc[4 * q4 + j][px] = fmaf(v[u][px], wv[j], acc[4 * q4 + j][px]);
        }
      }
    }
  }
  for (int ri = 0; ri < A.n_rs; ++ri) {
    const RsPath& Q = A.rs[ri];
    if (Q.cout0 >= cb + CT || Q.cout0 + Q.cout <= cb) continue;
    const size_t lp = (size_t)Q.Hs * Q.Ws;
#pragma unroll
    for (int px = 0; px < PX; ++px) {
      if (x0 + px >= W) continue;
      int o00, o01, o10, o11;
      float w00, w01, w10, w11;
      bilin(Q.Hs, Q.Ws, Q.up, y, x0 + px, o00, o01, o10, o11, w00, w01, w10, w11);
#pragma unroll
      for (int c = 0; c < CT; ++c) {
        const int co = cb + c - Q.cout0;
        if (co < 0 || co >= Q.cout) continue;
        const TI* sp = static_cast<const TI*>(Q.src) + ((size_t)n * Q.Cs + Q.c0 + co) * lp;
        acc[c][px] += w00 * ldg1(sp + o00) + w01 * ldg1(sp + o01) + w10 * ldg1(sp + o10) + w11 * ldg1(sp + o11);
      }
    }
  }
  TO* o = static_cast<TO*>(A.dst) + (((size_t)n * A.C + cb) * H + y) * W + x0;
#pragma unroll
  for (int c = 0; c < CT; ++c) {
    if (cb + c >= A.C) break;
    if (VEC) {
      if (PX == 4) st4(o + (size_t)c * plane, acc[c][0], acc[c][1], acc[c][PX - 2], acc[c][PX - 1]);
      else st2(o + (size_t)c * plane, acc[c][0], acc[c][1]);
    } else {
#pragma unroll
      for (int px = 0; px < PX; ++px)
        if (x0 + px < W) o[(size_t)c * plane + px] = store_as<TO>(acc[c][px]);
    }
  }
}

// every path's weights into shared memory [wrows][Cpad], zero outside its slice
__device__ __forceinline__ void c1_stage_weights(const C1Args& A, float* wsm) {
  for (int i = threadIdx.x; i < A.wrows * A.Cpad; i += kT) {
    const int row = i / A.Cpad, col = i - row * A.Cpad;
    float v = 0.f;
    for (int pi = 0; pi < A.n_conv; ++pi) {
      const C1Path& P = A.p[pi];
      const int ci = row - P.woff, co = col - P.cout0;
      if (ci >= 0 && ci < P.cin && co >= 0 && co < P.cout)
        v = A.transposed ? __ldg(P.w + (size_t)co * P.cin + ci) : __ldg(P.w + (size_t)ci * P.cout + co);
    }
    wsm[i] = v;
  }
  __syncthreads();
}

// PX == 4: 4 pixels x (16 | 8) channels per pass (<= 16 output channels: one pass over the input);  PX == 2: 2 pixels x (32 | 16 | 8)
// channels (17..32 output channels in ONE pass).  quads = ceil(W / PX), vec = W % PX == 0.
template <int PX, bool VEC, class TI, class TO, int U = 6>
__device__ __forceinline__ void conv1x1_body(const C1Args& A, float* wsm) {
  c1_stage_weights(A, wsm);
  const size_t task = (size_t)blockIdx.x * kT + threadIdx.x;
  if (task >= (size_t)A.N * A.H * A.quads) return;
  const int q = (int)(task % A.quads), y = (int)((task / A.quads) % A.H), n = (int)(task / ((size_t)A.quads * A.H));
  for (int cb = 0; cb < A.C;) {
    const int left = A.C - cb;
    if (left <= 8) { c1_group<8, PX, VEC, U, TI, TO>(A, wsm, cb, n, y, PX * q); cb += 8; }
    else if (PX == 4 || left <= 16) { c1_group<16, PX, VEC, U, TI, TO>(A, wsm, cb, n, y, PX * q); cb += 16; }
    else { c1_group<32, PX, VEC, U, TI, TO>(A, wsm, cb, n, y, PX * q); cb += 32; }
  }
}

// narrow form: 8 output channels per pass and 8 channels of loads in flight, <= 85 registers so three CTAs fit an SM
template <class TI, class TO, int U = 8>
__device__ __forceinline__ void conv1x1_narrow_body(const C1Args& A, float* wsm) {
  c1_stage_weights(A, wsm);
  const size_t task = (size_t)blockIdx.x * kT + threadIdx.x;
  if (task >= (size_t)A.N * A.H * A.quads) return;
  const int q = (int)(task % A.quads), y = (int)((task / A.quads) % A.H), n = (int)(task / ((size_t)A.quads * A.H));
  for (int cb = 0; cb < A.C; cb += 8) c1_group<8, 4, true, U, TI, TO>(A, wsm, cb, n, y, 4 * q);
}

// ---- weight gradient ---------------------------------------------------------------------------------------------------------
// KS == 1: thread tile 4 ci x 4 co;  KS == 3: 4 ci x 4 co x the 3 taps of one kernel row (dil 1);  KS == 0: 3x3 with any dilation —
// the input tile holds the three row bands r0 + (ky - 1) dil ... of a kernel row each, scalar shared-memory reads.  The source is TI,
// the destination gradient TD; the weight-gradient partials are fp32.
template <int KS, class TI, class TD>
__device__ __forceinline__ void conv_wgrad_body(const WgradArgs& A, float* smem) {
  constexpr int KX = KS == 1 ? 1 : 3, KY = KS == 1 ? 1 : 3;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int H = A.H, W = A.W, R = A.R, Wp = A.Wp, rows_in = KS == 0 ? 3 * R : R + (KS == 3 ? 2 : 0), hp = A.hp;
  const int buf_floats = words<TI>(A.cin4 * A.cpi) + words<TD>(A.cout4 * A.cpd);   // one stage: input tile [cin4][rows_in][Wp] (image column
  const int bands = (H + R - 1) / R;                               // x at x + hp), gradient tile [cout4][R][Wp] (column x at x)
  // task of this thread: (pixel split, tile); tiles beyond A.tiles idle.  Threads of one warp share the split when tiles >= 32.
  const int ltile = tid % A.tpad, split = tid / A.tpad, tile = blockIdx.y * A.tpad + ltile;
  const bool active = tile < A.tiles && split < A.splits;
  const int tm = active ? tile / A.nt : 0, tn = active ? tile % A.nt : 0;
  const int ci_t = tm / KY, ky = tm % KY, co_t = tn, Mi = A.cin4 / 4, Mo = A.nt;     // channels ci_t + i * Mi, co_t + j * Mo
  float acc[KX][4][4];
#pragma unroll
  for (int a = 0; a < KX; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) acc[a][b][0] = acc[a][b][1] = acc[a][b][2] = acc[a][b][3] = 0.f;

  // stage unit u into `base` with vector cp.async (zero-filled outside the image / the channel range); rows that are not 4-element
  // multiples take the synchronous scalar route
  auto stage = [&](int u, float* base) {
    const int n = u / bands, r0 = (u % bands) * R;
    TI* tin = reinterpret_cast<TI*>(base);
    TD* tdd = reinterpret_cast<TD*>(base + words<TI>((size_t)A.cin4 * A.cpi));
    for (int rr = warp; rr < A.cin4 * rows_in; rr += kT / 32) {
      const int c = rr / rows_in, row = rr - c * rows_in;
      const int gy = KS == 0 ? r0 + row % R + (row / R - 1) * A.dil : r0 + row - (KS == 3 ? 1 : 0);
      const bool inside = c < A.cin && gy >= 0 && gy < H && (KS != 0 || r0 + row % R < H);
      const TI* s = static_cast<const TI*>(A.in) + (((size_t)n * A.Cs + A.c0 + (inside ? c : 0)) * H + (inside ? gy : 0)) * W;
      TI* d = tin + (size_t)c * A.cpi + (size_t)row * Wp;
      if (A.vec) {
        for (int v = lane; v * 4 < Wp; v += 32) {
          const int xx = v * 4 - hp;
          const bool ld = inside && xx >= 0 && xx < W;
          cp_async4(d + v * 4, ld ? s + xx : static_cast<const TI*>(A.in), ld);
        }
      } else {
        for (int v = lane; v < Wp; v += 32) {
          const int xx = v - hp;
          d[v] = (inside && xx >= 0 && xx < W) ? ldg_raw(s + xx) : TI(0.f);
        }
      }
    }
    for (int rr = warp; rr < A.cout4 * R; rr += kT / 32) {
      const int c = rr / R, row = rr - c * R, gy = r0 + row;
      const bool inside = c < A.cout && gy < H;
      const TD* s = static_cast<const TD*>(A.dd) + (((size_t)n * A.Cd + A.cout0 + (inside ? c : 0)) * H + (inside ? gy : 0)) * W;
      TD* d = tdd + (size_t)c * A.cpd + (size_t)row * Wp;
      if (A.vec) {
        for (int v = lane; v * 4 < Wp; v += 32) {
          const int xx = v * 4;
          const bool ld = inside && xx < W;
          cp_async4(d + v * 4, ld ? s + xx : static_cast<const TD*>(A.dd), ld);
        }
      } else {
        for (int v = lane; v < Wp; v += 32) d[v] = (inside && v < W) ? ldg_raw(s + v) : TD(0.f);
      }
    }
  };

  // two stages in flight: unit u+grid is copied while unit u is consumed
  int cur = 0;
  if ((int)blockIdx.x < A.units) stage(blockIdx.x, smem);
  asm volatile("cp.async.commit_group;\n" ::: "memory");
  for (int u = blockIdx.x; u < A.units; u += gridDim.x, cur ^= 1) {
    const int un = u + gridDim.x;
    if (un < A.units) stage(un, smem + (size_t)(cur ^ 1) * buf_floats);
    asm volatile("cp.async.commit_group;\n" ::: "memory");
    asm volatile("cp.async.wait_group 1;\n" ::: "memory");
    __syncthreads();
    const float* tbuf = smem + (size_t)cur * buf_floats;
    const TI* tin = reinterpret_cast<const TI*>(tbuf);
    const TD* tdd = reinterpret_cast<const TD*>(tbuf + words<TI>((size_t)A.cin4 * A.cpi));
    if (active) {
    const int nq = R * A.quads;
    for (int q = split; q < nq; q += A.splits) {
      const int row = q / A.quads, x0 = 4 * (q - row * A.quads);
      float4 d4[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) d4[j] = lds4(tdd + (size_t)(co_t + j * Mo) * A.cpd + (size_t)row * Wp + x0);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const TI* ip = tin + (size_t)(ci_t + i * Mi) * A.cpi + (size_t)(KS == 0 ? ky * R + row : row + ky) * Wp + x0 + hp;
        if (KS == 0) {
#pragma unroll
          for (int kx = 0; kx < 3; ++kx) {
            const TI* tp = ip + (kx - 1) * A.dil;
            const float i0 = f32(tp[0]), i1 = f32(tp[1]), i2 = f32(tp[2]), i3 = f32(tp[3]);
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[kx][i][j] += i0 * d4[j].x + i1 * d4[j].y + i2 * d4[j].z + i3 * d4[j].w;
          }
        } else if (KS == 1) {
          const float4 v = lds4(ip);
#pragma unroll
          for (int j = 0; j < 4; ++j)
            acc[0][i][j] += v.x * d4[j].x + v.y * d4[j].y + v.z * d4[j].z + v.w * d4[j].w;
        } else {
          const float l = f32(ip[-1]);
          const float4 m = lds4(ip);
          const float r = f32(ip[4]);
          const float in6[6] = {l, m.x, m.y, m.z, m.w, r};
#pragma unroll
          for (int kx = 0; kx < 3; ++kx)
#pragma unroll
            for (int j = 0; j < 4; ++j)
              acc[kx][i][j] += in6[kx] * d4[j].x + in6[kx + 1] * d4[j].y + in6[kx + 2] * d4[j].z + in6[kx + 3] * d4[j].w;
        }
      }
    }
    }
    __syncthreads();                                               // everyone is done with this stage before the next copy lands in it
  }
  asm volatile("cp.async.wait_group 0;\n" ::: "memory");
  // ---- merge the pixel splits of the block in split order, write the block's partial ---------------------------------------------
  __syncthreads();
  float* red = smem;                                              // [splits][tpad][KX*16]
  constexpr int TA = KX * 16;
  if (active) {
    float* o = red + ((size_t)split * A.tpad + ltile) * TA;
#pragma unroll
    for (int a = 0; a < KX; ++a)
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) o[(a * 4 + i) * 4 + j] = acc[a][i][j];
  }
  __syncthreads();
  const int kk = KS == 1 ? 1 : 9;
  float* out = A.part + (size_t)blockIdx.x * A.cin * kk * A.cout;
  for (int e = tid; e < A.tpad * TA; e += kT) {
    const int lt = e / TA, t = blockIdx.y * A.tpad + lt, r = e - lt * TA, a = r / 16, i = (r / 4) % 4, j = r % 4;
    if (t >= A.tiles) continue;
    const int tm2 = t / A.nt, tn2 = t % A.nt, ci = tm2 / KY + i * (A.cin4 / 4), ky2 = tm2 % KY, co = tn2 + j * A.nt;
    if (ci >= A.cin || co >= A.cout) continue;
    float s = 0.f;
    for (int sp = 0; sp < A.splits; ++sp) s += red[((size_t)sp * A.tpad + lt) * TA + r];
    out[((size_t)ci * kk + ky2 * KX + a) * A.cout + co] = s;
  }
}

// ---- pooling prep (forward) and its routing (backward); the pooled copy has its source's element type ---------------------------
// dst[n][ci][yc][xc] = max over pool x pool of (pre_avg ? 2x2 mean : value) of src channels [c0, c0 + cin); idx = position of the
// FIRST maximum (row-major), as max_pool2d's backward uses it.
template <class T>
__device__ __forceinline__ void pool_fwd_body(const T* __restrict__ src, int N, int Cs, int c0, int cin, int Hs, int Ws, int pre_avg, int pool,
                                              T* __restrict__ dst, uint8_t* __restrict__ idx) {
  const int f = pre_avg ? 2 : 1, Hc = Hs / (f * pool), Wc = Ws / (f * pool);
  const size_t i = (size_t)blockIdx.x * kT + threadIdx.x, total = (size_t)N * cin * Hc * Wc;
  if (i >= total) return;
  const int xc = (int)(i % Wc), yc = (int)((i / Wc) % Hc), c = (int)((i / ((size_t)Wc * Hc)) % cin), n = (int)(i / ((size_t)Wc * Hc * cin));
  const T* s = src + ((size_t)n * Cs + c0 + c) * Hs * Ws;
  float best = -INFINITY;
  int bi = 0;
  for (int py = 0; py < pool; ++py)
    for (int px = 0; px < pool; ++px) {
      const int ya = yc * pool + py, xa = xc * pool + px;
      float v;
      if (pre_avg) {
        const T* b = s + (size_t)(2 * ya) * Ws + 2 * xa;
        v = (((f32(b[0]) + f32(b[1])) + f32(b[Ws])) + f32(b[Ws + 1])) * 0.25f;
      } else {
        v = f32(s[(size_t)ya * Ws + xa]);
      }
      if (v > best) { best = v; bi = py * pool + px; }
    }
  dst[i] = store_as<T>(best);
  if (idx) idx[i] = (uint8_t)bi;
}

// pool == 2 without the average, Ws % 4 == 0: two outputs per thread from two 4-element vector loads
template <class T>
__device__ __forceinline__ void pool2_fwd_body(const T* __restrict__ src, int N, int Cs, int c0, int cin, int Hs, int Ws,
                                               T* __restrict__ dst, uint8_t* __restrict__ idx) {
  const int Hc = Hs >> 1, Wc = Ws >> 1, W2 = Wc >> 1;
  const unsigned t = blockIdx.x * kT + threadIdx.x, total = (unsigned)N * cin * Hc * W2;        // < 2^32: checked by the host
  if (t >= total) return;
  const int x2 = (int)(t % (unsigned)W2), yc = (int)((t / (unsigned)W2) % (unsigned)Hc);
  const unsigned nc = t / ((unsigned)W2 * (unsigned)Hc);
  const int c = (int)(nc % (unsigned)cin), n = (int)(nc / (unsigned)cin);
  const T* s = src + (((size_t)n * Cs + c0 + c) * Hs + 2 * yc) * Ws + 4 * x2;
  const float4 a = ldg4(s), b = ldg4(s + Ws);
  float m0 = a.x; int i0 = 0;
  if (a.y > m0) { m0 = a.y; i0 = 1; }
  if (b.x > m0) { m0 = b.x; i0 = 2; }
  if (b.y > m0) { m0 = b.y; i0 = 3; }
  float m1 = a.z; int i1 = 0;
  if (a.w > m1) { m1 = a.w; i1 = 1; }
  if (b.z > m1) { m1 = b.z; i1 = 2; }
  if (b.w > m1) { m1 = b.w; i1 = 3; }
  const size_t o = ((size_t)nc * Hc + yc) * Wc + 2 * x2;
  st2(dst + o, m0, m1);
  *reinterpret_cast<uchar2*>(idx + o) = make_uchar2((unsigned char)i0, (unsigned char)i1);
}

// dsrc[n][ci][ys][xs] (exactly cin channels) from the gradient of the pooled tensor
template <class T>
__device__ __forceinline__ void pool_bwd_body(const T* __restrict__ dpool, const uint8_t* __restrict__ idx, int N, int cin, int Hs, int Ws,
                                              int pre_avg, int pool, T* __restrict__ dsrc) {
  const int f = pre_avg ? 2 : 1, Hc = Hs / (f * pool), Wc = Ws / (f * pool);
  const size_t i = (size_t)blockIdx.x * kT + threadIdx.x, total = (size_t)N * cin * Hs * Ws;
  if (i >= total) return;
  const int xs = (int)(i % Ws), ys = (int)((i / Ws) % Hs);
  const size_t nc = i / ((size_t)Ws * Hs);
  const int ya = ys / f, xa = xs / f, yc = ya / pool, xc = xa / pool;
  float g = 0.f;
  if (yc < Hc && xc < Wc) {
    const size_t j = (nc * Hc + yc) * Wc + xc;
    const bool hit = pool == 1 || (int)idx[j] == (ya - yc * pool) * pool + (xa - xc * pool);
    if (hit) g = f32(dpool[j]) * (pre_avg ? 0.25f : 1.f);
  }
  dsrc[i] = store_as<T>(g);
}

// four consecutive source pixels per thread (Ws % 4 == 0)
template <class T>
__device__ __forceinline__ void pool_bwd4_body(const T* __restrict__ dpool, const uint8_t* __restrict__ idx, int N, int cin, int Hs, int Ws,
                                               int pre_avg, int pool, T* __restrict__ dsrc) {
  const int f = pre_avg ? 2 : 1, Hc = Hs / (f * pool), Wc = Ws / (f * pool), W4 = Ws >> 2;
  const unsigned t = blockIdx.x * kT + threadIdx.x, total = (unsigned)N * cin * Hs * W4;     // < 2^32: checked by the host
  if (t >= total) return;
  const int x4 = (int)(t % (unsigned)W4), ys = (int)((t / (unsigned)W4) % (unsigned)Hs);
  const size_t nc = t / ((unsigned)W4 * (unsigned)Hs);
  const int ya = ys / f, yc = ya / pool;
  float g[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int xs = 4 * x4 + j, xa = xs / f, xc = xa / pool;
    g[j] = 0.f;
    if (yc < Hc && xc < Wc) {
      const size_t k = (nc * Hc + yc) * Wc + xc;
      const bool hit = pool == 1 || (int)__ldg(idx + k) == (ya - yc * pool) * pool + (xa - xc * pool);
      if (hit) g[j] = ldg1(dpool + k) * (pre_avg ? 0.25f : 1.f);
    }
  }
  st4(dsrc + (nc * Hs + ys) * Ws + 4 * x4, g[0], g[1], g[2], g[3]);
}

// adjoint of the bilinear x UP resample (align_corners=False, source index clamped at 0): dsrc[n][c][ys][xs] for c < cin gathers the
// (2 UP)^2 destination pixels that can feed it — rows UP ys - UP/2 ... UP ys + 3 UP/2 - 1, which also covers the clamped borders —
// with separable weights computed once per thread.
template <int UP, class T>
__device__ __forceinline__ void resample_bwd_body(const T* __restrict__ ddst, int N, int C, int H, int W, int cout0, int cin, int Hs, int Ws,
                                                  T* __restrict__ dsrc) {
  const unsigned t = blockIdx.x * kT + threadIdx.x, total = (unsigned)N * cin * Hs * Ws;         // < 2^32: checked by the host
  if (t >= total) return;
  const int xs = (int)(t % (unsigned)Ws), ys = (int)((t / (unsigned)Ws) % (unsigned)Hs);
  const unsigned ncq = t / ((unsigned)Ws * (unsigned)Hs);
  const int c = (int)(ncq % (unsigned)cin), n = (int)(ncq / (unsigned)cin);
  constexpr float inv = 1.f / (float)UP;
  constexpr int K = 2 * UP;
  float wy[K], wx[K];
  const int yb = ys * UP - UP / 2, xb = xs * UP - UP / 2;
#pragma unroll
  for (int k = 0; k < K; ++k) {
    wy[k] = 0.f; wx[k] = 0.f;
    const int oy = yb + k, ox = xb + k;
    if (oy >= 0 && oy < H) {
      float sy = ((float)oy + 0.5f) * inv - 0.5f;
      sy = sy < 0.f ? 0.f : sy;
      const int y0 = (int)sy, y1 = y0 + (y0 < Hs - 1 ? 1 : 0);
      const float ly = sy - (float)y0;
      wy[k] = (y0 == ys ? 1.f - ly : 0.f) + (y1 == ys ? ly : 0.f);
    }
    if (ox >= 0 && ox < W) {
      float sx = ((float)ox + 0.5f) * inv - 0.5f;
      sx = sx < 0.f ? 0.f : sx;
      const int x0 = (int)sx, x1 = x0 + (x0 < Ws - 1 ? 1 : 0);
      const float lx = sx - (float)x0;
      wx[k] = (x0 == xs ? 1.f - lx : 0.f) + (x1 == xs ? lx : 0.f);
    }
  }
  const T* d = ddst + ((size_t)n * C + cout0 + c) * H * W;
  float g = 0.f;
#pragma unroll
  for (int ky = 0; ky < K; ++ky) {
    const int oy = yb + ky;
    if (oy < 0 || oy >= H) continue;
    const T* row = d + (size_t)oy * W;
    float r = 0.f;
#pragma unroll
    for (int kx = 0; kx < K; ++kx) {
      const int ox = xb + kx;
      if (ox >= 0 && ox < W) r = fmaf(wx[kx], ldg1(row + ox), r);
    }
    g = fmaf(wy[ky], r, g);
  }
  dsrc[t] = store_as<T>(g);
}

// ---- depthwise 3x3 ------------------------------------------------------------------------------------------------------------------
// columns x0 - 1 ... x0 + 4 of row r of a plane (zero outside)
template <class T>
__device__ __forceinline__ void dw_load_row(const T* p, int r, int H, int W, int x0, bool vec, float* d) {
  if (r < 0 || r >= H) { d[0] = d[1] = d[2] = d[3] = d[4] = d[5] = 0.f; return; }
  const T* s = p + (size_t)r * W + x0;
  if (vec) {
    const float4 m = ldg4(s);
    d[1] = m.x; d[2] = m.y; d[3] = m.z; d[4] = m.w;
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j) d[1 + j] = x0 + j < W ? ldg1(s + j) : 0.f;
  }
  d[0] = x0 > 0 ? ldg1(s - 1) : 0.f;
  d[5] = x0 + 4 < W ? ldg1(s + 4) : 0.f;
}

template <class T>
__device__ __forceinline__ void dw_store4(T* d, int x0, int W, bool vec, const float* a) {
  if (vec) st4(d, a[0], a[1], a[2], a[3]);
  else {
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (x0 + j < W) d[j] = store_as<T>(a[j]);
  }
}

// y = scale * conv3x3(x, w[c]) (flip: the data gradient); a thread owns a 4-pixel column strip of `rows` consecutive rows.
template <class T>
__device__ __forceinline__ void dw3_body(const T* __restrict__ x, const float* __restrict__ w, T* __restrict__ y, int N, int C, int H, int W,
                                         float scale, int flip, int quads, int rows) {
  const int bands = (H + rows - 1) / rows;
  const size_t t = (size_t)blockIdx.x * kT + threadIdx.x;
  if (t >= (size_t)N * C * bands * quads) return;
  const int q = (int)(t % quads), b = (int)((t / quads) % bands);
  const size_t nc = t / ((size_t)quads * bands);
  const int c = (int)(nc % C), x0 = 4 * q, r0 = b * rows, r1 = r0 + rows < H ? r0 + rows : H;
  float k[9];
#pragma unroll
  for (int i = 0; i < 9; ++i) k[i] = __ldg(w + c * 9 + (flip ? 8 - i : i)) * scale;
  const T* p = x + nc * H * W;
  T* o = y + nc * H * W;
  const bool vec = (W & 3) == 0;
  float win[3][6];
  dw_load_row(p, r0 - 1, H, W, x0, vec, win[0]);
  dw_load_row(p, r0, H, W, x0, vec, win[1]);
  for (int r = r0; r < r1; ++r) {
    dw_load_row(p, r + 1, H, W, x0, vec, win[2]);
    float a[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float s = 0.f;
#pragma unroll
      for (int ky = 0; ky < 3; ++ky)
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) s = fmaf(win[ky][j + kx], k[ky * 3 + kx], s);
      a[j] = s;
    }
    dw_store4(o + (size_t)r * W + x0, x0, W, vec, a);
#pragma unroll
    for (int j = 0; j < 6; ++j) { win[0][j] = win[1][j]; win[1][j] = win[2][j]; }
  }
}

// block reduction of the 9 tap sums in a fixed order (warp shuffles, then the 8 warp results): part[block][c][9]
__device__ __forceinline__ void dw_block_partial(const float* acc, float* __restrict__ part, int C, int c) {
  __shared__ float sh[kT / 32][9];
#pragma unroll
  for (int i = 0; i < 9; ++i) {
    float v = acc[i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5][i] = v;
  }
  __syncthreads();
  if (threadIdx.x < 9) {
    float s = 0.f;
#pragma unroll
    for (int wv = 0; wv < kT / 32; ++wv) s += sh[wv][threadIdx.x];
    part[((size_t)blockIdx.x * C + c) * 9 + threadIdx.x] = s;
  }
}

// partial[block][c][9]: the block's share of sum_{n,y,x} dy[y][x] * x[y+ky-1][x+kx-1]; grid = (blocks per channel, C); a block walks
// (image, band) units of its channel, a thread a 4-pixel strip of the band.
template <class T>
__device__ __forceinline__ void dw3_wgrad_body(const T* __restrict__ x, const T* __restrict__ dy, float* __restrict__ part, int N, int C, int H,
                                               int W, int quads, int rows) {
  const int c = blockIdx.y, bands = (H + rows - 1) / rows;
  const size_t tasks = (size_t)N * bands * quads;
  const bool vec = (W & 3) == 0;
  float acc[9];
#pragma unroll
  for (int i = 0; i < 9; ++i) acc[i] = 0.f;
  for (size_t t = (size_t)blockIdx.x * kT + threadIdx.x; t < tasks; t += (size_t)gridDim.x * kT) {
    const int q = (int)(t % quads), b = (int)((t / quads) % bands), n = (int)(t / ((size_t)quads * bands));
    const int x0 = 4 * q, r0 = b * rows, r1 = r0 + rows < H ? r0 + rows : H;
    const T* p = x + ((size_t)n * C + c) * H * W;
    const T* g = dy + ((size_t)n * C + c) * H * W;
    float win[3][6];
    dw_load_row(p, r0 - 1, H, W, x0, vec, win[0]);
    dw_load_row(p, r0, H, W, x0, vec, win[1]);
    for (int r = r0; r < r1; ++r) {
      dw_load_row(p, r + 1, H, W, x0, vec, win[2]);
      float d[4];
      const T* gs = g + (size_t)r * W + x0;
      if (vec) {
        const float4 m = ldg4(gs);
        d[0] = m.x; d[1] = m.y; d[2] = m.z; d[3] = m.w;
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) d[j] = x0 + j < W ? ldg1(gs + j) : 0.f;
      }
#pragma unroll
      for (int ky = 0; ky < 3; ++ky)
#pragma unroll
        for (int kx = 0; kx < 3; ++kx)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[ky * 3 + kx] = fmaf(d[j], win[ky][j + kx], acc[ky * 3 + kx]);
#pragma unroll
      for (int j = 0; j < 6; ++j) { win[0][j] = win[1][j]; win[1][j] = win[2][j]; }
    }
  }
  dw_block_partial(acc, part, C, c);
}

// backward of the depthwise 3x3 in ONE pass over dy: dx = scale * conv3x3(dy, flipped w) and the block partials of
// dw[c][tap] = sum dy[y][x] * x[y+ky-1][x+kx-1]; grid = (blocks per channel, C) as dw3_wgrad_body.
template <class T>
__device__ __forceinline__ void dw3_bwd_body(const T* __restrict__ x, const T* __restrict__ dy, const float* __restrict__ w, T* __restrict__ dx,
                                             float* __restrict__ part, int N, int C, int H, int W, float scale, int quads, int rows) {
  const int c = blockIdx.y, bands = (H + rows - 1) / rows;
  const size_t tasks = (size_t)N * bands * quads;
  const bool vec = (W & 3) == 0;
  float k[9], acc[9];
#pragma unroll
  for (int i = 0; i < 9; ++i) { k[i] = __ldg(w + c * 9 + 8 - i) * scale; acc[i] = 0.f; }
  for (size_t t = (size_t)blockIdx.x * kT + threadIdx.x; t < tasks; t += (size_t)gridDim.x * kT) {
    const int q = (int)(t % quads), b = (int)((t / quads) % bands), n = (int)(t / ((size_t)quads * bands));
    const int x0 = 4 * q, r0 = b * rows, r1 = r0 + rows < H ? r0 + rows : H;
    const size_t plane = ((size_t)n * C + c) * H * W;
    const T* p = x + plane;
    const T* g = dy + plane;
    T* o = dx + plane;
    float wx[3][6], wg[3][6];                                     // 3-row windows of x and dy, columns x0 - 1 ... x0 + 4
    dw_load_row(p, r0 - 1, H, W, x0, vec, wx[0]); dw_load_row(p, r0, H, W, x0, vec, wx[1]);
    dw_load_row(g, r0 - 1, H, W, x0, vec, wg[0]); dw_load_row(g, r0, H, W, x0, vec, wg[1]);
    for (int r = r0; r < r1; ++r) {
      dw_load_row(p, r + 1, H, W, x0, vec, wx[2]);
      dw_load_row(g, r + 1, H, W, x0, vec, wg[2]);
      float a[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float s = 0.f;
#pragma unroll
        for (int ky = 0; ky < 3; ++ky)
#pragma unroll
          for (int kx = 0; kx < 3; ++kx) s = fmaf(wg[ky][j + kx], k[ky * 3 + kx], s);
        a[j] = s;
      }
      dw_store4(o + (size_t)r * W + x0, x0, W, vec, a);
#pragma unroll
      for (int ky = 0; ky < 3; ++ky)
#pragma unroll
        for (int kx = 0; kx < 3; ++kx)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[ky * 3 + kx] = fmaf(wg[1][1 + j], wx[ky][j + kx], acc[ky * 3 + kx]);
#pragma unroll
      for (int j = 0; j < 6; ++j) { wx[0][j] = wx[1][j]; wx[1][j] = wx[2][j]; wg[0][j] = wg[1][j]; wg[1][j] = wg[2][j]; }
    }
  }
  dw_block_partial(acc, part, C, c);
}

// ---- BatchNorm (train) + PReLU ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// block-wide sum of up to 3 values; result valid in thread 0
__device__ __forceinline__ void block_sum3(float& a, float& b, float& c) {
  __shared__ float sh[3][kT / 32];
  a = warp_sum(a); b = warp_sum(b); c = warp_sum(c);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) { sh[0][w] = a; sh[1][w] = b; sh[2][w] = c; }
  __syncthreads();
  if (w == 0) {
    a = l < kT / 32 ? sh[0][l] : 0.f; b = l < kT / 32 ? sh[1][l] : 0.f; c = l < kT / 32 ? sh[2][l] : 0.f;
    a = warp_sum(a); b = warp_sum(b); c = warp_sum(c);
  }
  __syncthreads();
}

// Per-channel reductions over (N, H*W) run on a (C, parts) grid — a channel-per-block grid would leave most of the 132 SMs
// idle for 8..79-channel layers.  A block reduces one segment of one image plane, publishes its partial to a workspace,
// and the last block to arrive for a channel (ticket counter) merges the partials IN PART ORDER, so the result does not
// depend on scheduling.  Segments: S per plane, parts = N * S.
__device__ __forceinline__ bool last_block_of(unsigned* counter, unsigned parts) {
  __shared__ bool is_last;
  if (threadIdx.x == 0) {
    __threadfence();
    is_last = atomicAdd(counter, 1u) == parts - 1;
  }
  __syncthreads();
  return is_last;
}

// stats: per channel mean and biased variance in ONE pass over z: sums of (z - K) and (z - K)^2 with the shift K = the mean of 32 fixed
// samples spread over the channel's images and planes (every block of the channel computes the same K), so (mean - K)^2 ~ var / 32
// and the subtraction S2 - S1^2 / M loses no more than a few ulps.  (A single sample is not enough: the corner pixel of a zero-padded
// conv sits many sigma from the mean and cost 6e-3 on one weight gradient.)  Block partials in fp32 over <= a few hundred elements per
// thread, merged in part order in double by the last block.
template <class T>
__device__ __forceinline__ void bn_stats_body(const T* __restrict__ z, int N, int C, int HW, int S, float* mean, float* var, float* ws,
                                              unsigned* cnt) {
  const int c = blockIdx.x, part = blockIdx.y, parts = gridDim.y, n = part / S, sg = part - n * S;
  const int seg = (HW + S - 1) / S, i0 = sg * seg, i1 = (i0 + seg) < HW ? (i0 + seg) : HW;
  const T* p = z + ((size_t)n * C + c) * HW;
  __shared__ float Ks;
  if (threadIdx.x < 32) {
    const int l = threadIdx.x, img = l % N, off = (int)(((long long)l * HW) / 32 + 17) % HW;
    const float v = warp_sum(ldg1(z + ((size_t)img * C + c) * HW + off)) * (1.f / 32.f);
    if (l == 0) Ks = v;
  }
  __syncthreads();
  const float K = Ks;
  float s = 0.f, q = 0.f, d1 = 0.f;
  if (((HW | i0) & 3) == 0 && ((i1 - i0) & 3) == 0) {
    const typename Vec4<T>::type* p4 = reinterpret_cast<const typename Vec4<T>::type*>(p + i0);
    for (int i = threadIdx.x; i < (i1 - i0) / 4; i += kT) {
      const float4 v = to_f4(__ldg(p4 + i));
      const float a = v.x - K, b = v.y - K, cc = v.z - K, d = v.w - K;
      s += (a + b) + (cc + d);
      q += (a * a + b * b) + (cc * cc + d * d);
    }
  } else {
    for (int i = i0 + threadIdx.x; i < i1; i += kT) { const float d = f32(p[i]) - K; s += d; q += d * d; }
  }
  block_sum3(s, q, d1);
  float* w = ws + ((size_t)c * parts + part) * 3;
  if (threadIdx.x == 0) { w[0] = s; w[1] = q; w[2] = (float)(i1 > i0 ? i1 - i0 : 0); }
  if (!last_block_of(cnt + c, parts)) return;
  if (threadIdx.x == 0) {
    __threadfence();
    const volatile float* v = ws + (size_t)c * parts * 3;
    double S1 = 0.0, S2 = 0.0, M = 0.0;
    for (int k = 0; k < parts; ++k) { S1 += (double)v[3 * k]; S2 += (double)v[3 * k + 1]; M += (double)v[3 * k + 2]; }
    const double m1 = S1 / M, vv = (S2 - S1 * m1) / M;
    mean[c] = (float)((double)K + m1); var[c] = (float)(vv > 0.0 ? vv : 0.0);
    cnt[c] = 0u;                                            // ready for the next call on this stream
  }
}

// y = prelu(gamma * (z - mean) * rsqrt(var + eps) + beta);  gap[n*C+c] = mean over HW of y before its rounding to T (optional)
template <class T>
__device__ __forceinline__ void bn_prelu_fwd_body(const T* __restrict__ z, T* __restrict__ y, int C, int HW, const float* mean, const float* var,
                                                  const float* gamma, const float* beta, const float* slope, float eps, float* gap) {
  const int c = blockIdx.x, n = blockIdx.y;
  const float r = rsqrtf(var[c] + eps), g = gamma[c] * r, b = beta[c] - mean[c] * g, a = slope[c];
  const T* p = z + ((size_t)n * C + c) * HW;
  T* o = y + ((size_t)n * C + c) * HW;
  float s = 0.f, d0 = 0.f, d1 = 0.f;
  for (int i = threadIdx.x; i < HW; i += kT) {
    const float u = f32(p[i]) * g + b;
    const float v = u > 0.f ? u : a * u;
    o[i] = store_as<T>(v);
    s += v;
  }
  if (gap) {
    block_sum3(s, d0, d1);
    if (threadIdx.x == 0) gap[(size_t)n * C + c] = s / (float)HW;
  }
}

// backward reductions per channel: S1 = sum du, S2 = sum du * xhat, S3 = sum dy * u * [u <= 0]   (du = dy * prelu'(u));
// same (C, parts) grid and ordered merge as bn_stats_body
template <class T>
__device__ __forceinline__ void bn_prelu_bwd_reduce_body(const T* __restrict__ z, const T* __restrict__ dy, int N, int C, int HW, int S,
                                                         const float* mean, const float* var, const float* gamma, const float* beta,
                                                         const float* slope, float eps, float* dgamma, float* dbeta, float* dslope,
                                                         float* ws, unsigned* cnt) {
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
  block_sum3(s1, s2, s3);
  float* w = ws + ((size_t)c * parts + part) * 3;
  if (threadIdx.x == 0) { w[0] = s1; w[1] = s2; w[2] = s3; }
  if (!last_block_of(cnt + c, parts)) return;
  if (threadIdx.x == 0) {
    __threadfence();
    const volatile float* v = ws + (size_t)c * parts * 3;
    float t1 = 0.f, t2 = 0.f, t3 = 0.f;
    for (int k = 0; k < parts; ++k) { t1 += v[3 * k]; t2 += v[3 * k + 1]; t3 += v[3 * k + 2]; }
    dbeta[c] = t1; dgamma[c] = t2; dslope[c] = t3;
    cnt[c] = 0u;
  }
}

// dz = gamma * r * (du - S1/M - xhat * S2/M)
template <class T>
__device__ __forceinline__ void bn_prelu_bwd_apply_body(const T* __restrict__ z, const T* __restrict__ dy, T* __restrict__ dz, int N, int C, int HW,
                                                        const float* mean, const float* var, const float* gamma, const float* beta,
                                                        const float* slope, float eps, const float* dgamma, const float* dbeta, int frozen) {
  const int c = blockIdx.x, n = blockIdx.y;
  const float mu = mean[c], r = rsqrtf(var[c] + eps), g = gamma[c], b = beta[c], a = slope[c];
  // frozen statistics (eval-mode BN inside a training graph): mean / var are constants, no batch terms
  const float invM = frozen ? 0.f : 1.f / ((float)N * (float)HW), m1 = dbeta[c] * invM, m2 = dgamma[c] * invM;
  const size_t off = ((size_t)n * C + c) * HW;
  for (int i = threadIdx.x; i < HW; i += kT) {
    const float xh = (f32(z[off + i]) - mu) * r, u = g * xh + b, d = f32(dy[off + i]);
    const float du = u > 0.f ? d : a * d;
    dz[off + i] = store_as<T>(g * r * (du - m1 - xh * m2));
  }
}

}  // namespace tf
}  // namespace csnet
