// il_stream.cuh — the 1x1-kind ILBlock as ONE persistent, streaming kernel on the Hopper data path (TMA + wgmma)
// (reference: ILBlock.forward, CSNet/model/csnet.py:72-76 = gOctaveCBR :778-792 over gOctaveConv.forward :664-726,
// then two SimplifiedGOctConvBR.forward :838-851).
//
// A CTA walks a contiguous range of the batch's (image, 4-row chunk) sequence top to bottom, full image width:
//
//   TMA        x_h rows [4c, 4c+4) and x_l rows [2c, 2c+2) arrive by cp.async.bulk.tensor.5d straight in the
//              tensor-core operand layout  [row][8-pixel group][channel slot][8 px]  (a core matrix of the MN-major
//              A operand = 8 channel slots x 16 bytes); the map splits W into (W/8, 8), channel slots past the
//              tensor's C are zero-filled by the TMA unit = the K padding of the GEMM.  2 hi / 3 lo stages.
//   resample   bilinear x2 of x_l -> slots [Chi, Chi+Cli) of the hi chunk (lo -> hi path, csnet.py:702-707; the
//              up-sample commutes with the 1x1 conv), max-pool 2x2 of x_h -> slots [Cli, Cli+Chi) of the lo chunk
//              (hi -> lo path, :709-712).
//   GEMM       a warpgroup issues wgmma.mma_async (f16 x f16 -> f32, M = 64 pixels, N = ru16(Cout), K = 16 per
//              instruction) per 8 pixel groups straight from the shared-memory tiles; fp32 accumulators in registers.
//   epilogue   from the accumulator fragment: + bias, PReLU, 16-bit, written IN PLACE over the chunk (T1).
//   dw tail    a thread owns (channel, two 8-pixel groups) for the whole walk and keeps the open rows of both 3x3 layers
//              as fp32 running sums in registers: dw3x3+BN+PReLU twice with no halo recomputation in y, no shared-memory
//              round trip for T2, 16-byte coalesced stores of the block output.  (mixed-precision FMA: fp16 x fp16 + fp32.)
//
// Stem form (kStem; the first block, csnet.py:60-71: both branches are 3x3 convs of the fp32 image, the lo one of its 2x2
// max-pool): the TMA ring holds 4-row blocks of the fp32 image (4-D map, zero fill outside the image = the conv padding);
// instead of the resample pass the threads build the im2col operand (27 slots: ci, ky, kx) of the hi chunk and of the
// lo chunk (pooling on the fly) in the same [row][group][slot][8 px] layout; GEMM, epilogue and depthwise tail are shared.
//
// An image is cut into `ns` column strips of gsn 8-pixel groups (gsn even); a CTA's tile of a strip carries one halo
// group on each side when ns > 1 (hl = 1: the TMA box starts one group early, out-of-image groups arrive as zeros).
// Narrow strips shrink a CTA's shared memory and threads.  No row halo is ever re-read from HBM (except one
// warm-up chunk where a CTA's range starts inside an image); the work split is a flat division of the
// N * ns * H/4 chunks over the CTAs.  Needs W % 16 == 0, H % 4 == 0, K = Chi + Cli <= 64.  Other shapes: il_block.cuh.
#pragma once
#include <cuda.h>

#include "il_block.cuh"

namespace csnet {

constexpr int kIlsMaxThreads = 384;   // 168 registers a thread: the tail's fp32 sums of 16 pixels stay out of local memory
constexpr int kIlsMaxC = 64;          // output channels per branch (epilogue parameter tables in the kernel arguments)
constexpr int kIlsHiStages = 2, kIlsLoStages = 3;

struct IlsArgs {
  void* yh;
  void* yl;                           // nullptr when Clo == 0
  const uint32_t* wh;                 // packed 16-bit [NH][K8]  columns [x_h | up(x_l)]
  const uint32_t* wl;                 // packed 16-bit [NL][K8]  columns [x_l | pool(x_h)]
  DwParams dw1h, dw1l, dw2h, dw2l;
  float bias_h[kIlsMaxC], sm1_h[kIlsMaxC], bias_l[kIlsMaxC], sm1_l[kIlsMaxC];   // conv bias, PReLU slope - 1
  int32_t N, H, W;
  int32_t Chi, Cli, Cho, Clo;
  int32_t K8, K16, NH, NL;            // NH / NL = ru16(Cho / Clo): the N of the MMAs (NL = 0 without a lo output)
  int32_t SH, SL, ST;                 // channel slots per pixel group: hi chunk, lo chunk, T1L buffer (all odd)
  int32_t GH, GL;                     // pixel groups per image row: W/8, W/16
  int32_t ns, gsn, hl;                // column strips per image, hi groups per strip (even), halo groups per side (0 / 1)
  int32_t GR, GLR;                    // groups per row of a CTA's tile: gsn + 2 hl, gsn/2 + 2 hl
  int32_t Ci, BW;                     // stem form: image channels; width in floats of an image block in shared memory (8 GR + 8)
  int32_t off_xlo;                    // stem form: the lo chunk's GEMM operand buffer
  int32_t cpi, total_chunks;          // chunks per image strip (H/4), N * ns * cpi
  int32_t dw_warps;                   // warps of the CTA = warps of the depthwise tail (tasks packed: hi group pairs, then lo)
  int32_t hi_stage_bytes, lo_stage_bytes;
  int32_t off_xl, off_xh, off_t1l, off_wbh, off_wbl, off_bar, off_zero, off_epi, off_dwp, smem_bytes;
};

__device__ __forceinline__ void tma_load_5d(uint32_t dst, const CUtensorMap* tm, uint32_t bar, int c0, int c1, int c2, int c3, int c4) {
  asm volatile("cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];\n"
               ::"r"(dst), "l"(tm), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4) : "memory");
}
__device__ __forceinline__ void tma_load_4d_a(uint32_t dst, const CUtensorMap* tm, uint32_t bar, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];\n"
               ::"r"(dst), "l"(tm), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx_a(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(bar), "r"(bytes) : "memory");
}
// parity wait with a wall-clock bound: a lost TMA / MMA must trap, not hang the GPU
__device__ __forceinline__ void mbar_wait_a(uint32_t bar, uint32_t parity) {
  uint32_t ok = 0;
  const long long t0 = clock64();
  while (true) {
    asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}\n"
                 : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    if (ok) break;
    if (clock64() - t0 > 4000000000LL) __trap();
  }
}
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  // wgmma shared-memory matrix descriptor, no swizzle: start / LBO / SBO in 16-byte units.  LBO = the stride between
  // core matrices along K, SBO = along M / N (for the MN-major A operand as for the K-major B operand).
  return (uint64_t)((saddr & 0x3FFFF) >> 4) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16) |
         ((uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32);
}
// wgmma.m64nNk16, fp32 += f16 x f16: A (64 pixels x 16 channels) MN-major from shared memory (transposed: pixels are the
// contiguous dimension of a core matrix), B (N output channels x 16) K-major; d: the warpgroup's accumulator fragment.
// mma0 starts a group (scale-d = 0, d write-only): no other instruction defines the accumulator registers before the MMAs,
// which would make ptxas serialize the group's wgmmas.
template <int N> struct Wgmma;
template <> struct Wgmma<16> {
  static __device__ __forceinline__ void mma(float (&d)[8], uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %10, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 1, 0;\n}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
                 : "l"(da), "l"(db), "r"(acc));
  }
  static __device__ __forceinline__ void mma0(float (&d)[8], uint64_t da, uint64_t db) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %10, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 1, 0;\n}\n"
                 : "=f"(d[0]), "=f"(d[1]), "=f"(d[2]), "=f"(d[3]), "=f"(d[4]), "=f"(d[5]), "=f"(d[6]), "=f"(d[7])
                 : "l"(da), "l"(db), "r"(0u));
  }
};
template <> struct Wgmma<32> {
  static __device__ __forceinline__ void mma(float (&d)[16], uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 1, 0;\n}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                 : "l"(da), "l"(db), "r"(acc));
  }
  static __device__ __forceinline__ void mma0(float (&d)[16], uint64_t da, uint64_t db) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 1, 0;\n}\n"
                 : "=f"(d[0]), "=f"(d[1]), "=f"(d[2]), "=f"(d[3]), "=f"(d[4]), "=f"(d[5]), "=f"(d[6]), "=f"(d[7]), "=f"(d[8]), "=f"(d[9]), "=f"(d[10]), "=f"(d[11]), "=f"(d[12]), "=f"(d[13]), "=f"(d[14]), "=f"(d[15])
                 : "l"(da), "l"(db), "r"(0u));
  }
};
template <> struct Wgmma<48> {
  static __device__ __forceinline__ void mma(float (&d)[24], uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %26, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n48k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, %24, %25, p, 1, 1, 1, 0;\n}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
                 : "l"(da), "l"(db), "r"(acc));
  }
  static __device__ __forceinline__ void mma0(float (&d)[24], uint64_t da, uint64_t db) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %26, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n48k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, %24, %25, p, 1, 1, 1, 0;\n}\n"
                 : "=f"(d[0]), "=f"(d[1]), "=f"(d[2]), "=f"(d[3]), "=f"(d[4]), "=f"(d[5]), "=f"(d[6]), "=f"(d[7]), "=f"(d[8]), "=f"(d[9]), "=f"(d[10]), "=f"(d[11]), "=f"(d[12]), "=f"(d[13]), "=f"(d[14]), "=f"(d[15]), "=f"(d[16]), "=f"(d[17]), "=f"(d[18]), "=f"(d[19]), "=f"(d[20]), "=f"(d[21]), "=f"(d[22]), "=f"(d[23])
                 : "l"(da), "l"(db), "r"(0u));
  }
};
template <> struct Wgmma<64> {
  static __device__ __forceinline__ void mma(float (&d)[32], uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 1, 0;\n}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "l"(da), "l"(db), "r"(acc));
  }
  static __device__ __forceinline__ void mma0(float (&d)[32], uint64_t da, uint64_t db) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 1, 0;\n}\n"
                 : "=f"(d[0]), "=f"(d[1]), "=f"(d[2]), "=f"(d[3]), "=f"(d[4]), "=f"(d[5]), "=f"(d[6]), "=f"(d[7]), "=f"(d[8]), "=f"(d[9]), "=f"(d[10]), "=f"(d[11]), "=f"(d[12]), "=f"(d[13]), "=f"(d[14]), "=f"(d[15]), "=f"(d[16]), "=f"(d[17]), "=f"(d[18]), "=f"(d[19]), "=f"(d[20]), "=f"(d[21]), "=f"(d[22]), "=f"(d[23]), "=f"(d[24]), "=f"(d[25]), "=f"(d[26]), "=f"(d[27]), "=f"(d[28]), "=f"(d[29]), "=f"(d[30]), "=f"(d[31])
                 : "l"(da), "l"(db), "r"(0u));
  }
};
template <> struct Wgmma<80> {
  static __device__ __forceinline__ void mma(float (&d)[40], uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %42, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n80k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39}, %40, %41, p, 1, 1, 1, 0;\n}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39])
                 : "l"(da), "l"(db), "r"(acc));
  }
  static __device__ __forceinline__ void mma0(float (&d)[40], uint64_t da, uint64_t db) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %42, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n80k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39}, %40, %41, p, 1, 1, 1, 0;\n}\n"
                 : "=f"(d[0]), "=f"(d[1]), "=f"(d[2]), "=f"(d[3]), "=f"(d[4]), "=f"(d[5]), "=f"(d[6]), "=f"(d[7]), "=f"(d[8]), "=f"(d[9]), "=f"(d[10]), "=f"(d[11]), "=f"(d[12]), "=f"(d[13]), "=f"(d[14]), "=f"(d[15]), "=f"(d[16]), "=f"(d[17]), "=f"(d[18]), "=f"(d[19]), "=f"(d[20]), "=f"(d[21]), "=f"(d[22]), "=f"(d[23]), "=f"(d[24]), "=f"(d[25]), "=f"(d[26]), "=f"(d[27]), "=f"(d[28]), "=f"(d[29]), "=f"(d[30]), "=f"(d[31]), "=f"(d[32]), "=f"(d[33]), "=f"(d[34]), "=f"(d[35]), "=f"(d[36]), "=f"(d[37]), "=f"(d[38]), "=f"(d[39])
                 : "l"(da), "l"(db), "r"(0u));
  }
};
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit_wait() {
  asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory");
  asm volatile("wgmma.wait_group.sync.aligned 0;\n" ::: "memory");
}
__device__ __forceinline__ void warpgroup_bar(int wg) { asm volatile("bar.sync %0, 128;\n" ::"r"(1 + wg) : "memory"); }
// One 64-pixel block of the warpgroup: d = A[64][K16] . B[N][K16]^T over K16 / 16 instructions.
template <int N>
__device__ __forceinline__ void wgmma_block(float (&d)[N / 2], uint64_t da, uint64_t db, int K16) {
  wgmma_fence();
  Wgmma<N>::mma0(d, da, db);
  for (int ks = 1; ks < (K16 >> 4); ++ks) Wgmma<N>::mma(d, da + (uint64_t)(16 * ks), db + (uint64_t)(16 * ks), 1u);
  wgmma_commit_wait();
}
__device__ __forceinline__ uint32_t lds32(uint32_t a) { uint32_t v; asm volatile("ld.shared.b32 %0, [%1];\n" : "=r"(v) : "r"(a)); return v; }
__device__ __forceinline__ uint2 lds64(uint32_t a) { uint2 v; asm volatile("ld.shared.v2.b32 {%0, %1}, [%2];\n" : "=r"(v.x), "=r"(v.y) : "r"(a)); return v; }
__device__ __forceinline__ uint4 lds128(uint32_t a) {
  uint4 v;
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];\n" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a));
  return v;
}
__device__ __forceinline__ uint16_t lds16(uint32_t a) { uint16_t v; asm volatile("ld.shared.u16 %0, [%1];\n" : "=h"(v) : "r"(a)); return v; }
__device__ __forceinline__ void sts128(uint32_t a, uint4 v) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};\n" ::"r"(a), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ void sts16(uint32_t a, uint16_t v) { asm volatile("st.shared.u16 [%0], %1;\n" ::"r"(a), "h"(v) : "memory"); }

// The depthwise tail.  A thread owns one channel and two 8-pixel groups A, B (x0 .. x0+15) of a strip row for the whole
// walk and keeps running sums instead of windows of its inputs: a 3x3 output row is finished by its third input row, so per
// layer the thread holds the two output rows still open (one started by one input row, one by two).  Each input value is
// converted to fp32 once, when its row arrives, and every sum still runs  bias, taps dy = 0, 1, 2 (dx = 0, 1, 2 within)  in
// that order: the chain of the mixed-precision FMA (fp16 x fp16 + fp32), operand for operand.
// Parameters: per tail channel in shared memory, for dw1 then dw2, three float4 {3 weights of tap row dy (rounded through
// the 16-bit type), x}, x = bias, slope - 1, 0: one 16-byte load right before each tap row is used.
constexpr int kIlsDwpBytes = 96;
constexpr int kIlsTX = 20, kIlsT2 = 18, kIlsTO = 16;   // a T1 row of a task (x0-2 .. x0+17), its T2 row (x0-1 .. x0+16), output

// acc[i] += row[i + dx] * w[dx], dx = 0, 1, 2 (one tap row of a 3x3 over NO outputs); kStart: acc[i] = w.w (the bias) first
template <int NO, bool kStart = false>
__device__ __forceinline__ void ils_dw_taps(float (&acc)[NO], const float* row, float4 w) {
#pragma unroll
  for (int i = 0; i < NO; ++i) {
    acc[i] = fmaf(row[i], w.x, kStart ? w.w : acc[i]);
    acc[i] = fmaf(row[i + 1], w.y, acc[i]);
    acc[i] = fmaf(row[i + 2], w.z, acc[i]);
  }
}
__device__ __forceinline__ float4 ils_dw_param(uint32_t a) {
  const uint4 v = lds128(a);
  return make_float4(__uint_as_float(v.x), __uint_as_float(v.y), __uint_as_float(v.z), __uint_as_float(v.w));
}
struct IlsTail {
  float s2a[kIlsT2], s2b[kIlsT2];    // T2 rows r-1 (two input rows in), r (one)
  float soa[kIlsTO], sob[kIlsTO];    // output rows r-2 (two T2 rows in), r-1 (one)
};
// The sums of a walk's start: the rows above its first T1 row are zero (as if the windows started from zero).  The zero
// is opaque to the compiler: folding 0 * w + acc to acc would differ for a -0 bias or a non-finite weight.
__device__ __forceinline__ void ils_dw_start(IlsTail& t, uint32_t prm) {
  float z0;
  asm("mov.b32 %0, 0;\n" : "=f"(z0));
  float z[kIlsTX];
#pragma unroll
  for (int i = 0; i < kIlsTX; ++i) z[i] = z0;
  float4 w0 = ils_dw_param(prm), w1 = ils_dw_param(prm + 16u);
  ils_dw_taps<kIlsT2, true>(t.s2a, z, w0); ils_dw_taps<kIlsT2>(t.s2a, z, w1); ils_dw_taps<kIlsT2, true>(t.s2b, z, w0);
  w0 = ils_dw_param(prm + 48u); w1 = ils_dw_param(prm + 64u);
  ils_dw_taps<kIlsTO, true>(t.soa, z, w0); ils_dw_taps<kIlsTO>(t.soa, z, w1); ils_dw_taps<kIlsTO, true>(t.sob, z, w0);
}
// Per-task constants of the tail: T2 at x0-1, x0+8, x0+16 is conv padding (x 0) at the image's edges; B may lie past the
// strip (its outputs are not stored) or past the image (zeros).
struct IlsTaskEdges {
  float m0, m9, m17;
  bool outB;
};
// One step: T1 row r arrives (x) and finishes T2 row r-1 (s2a), which finishes the block output row r-2 (soa).  On return
// s2a / soa hold the rows just started (T2 row r+1, output row r); s2b / sob swap roles with them: the caller passes the
// sums of even and odd rows in turn (a = s2a/soa, b = s2b/sob of the row).
template <typename T>
__device__ __forceinline__ void ils_dw_push(float (&s2a)[kIlsT2], float (&s2b)[kIlsT2], float (&soa)[kIlsTO], float (&sob)[kIlsTO],
                                            const float (&x)[kIlsTX], uint32_t prm, bool make_t2, const IlsTaskEdges& e, bool make_out,
                                            uint16_t* out) {
  ils_dw_taps<kIlsT2>(s2a, x, ils_dw_param(prm + 32u));
  const float4 w1 = ils_dw_param(prm + 16u);
  float q[kIlsT2];                   // T2 row r-1, rounded through the 16-bit type (zero: conv padding / not needed)
#pragma unroll
  for (int i = 0; i < kIlsT2; i += 2) {
    float v0 = prelu_m1(s2a[i], w1.w), v1 = prelu_m1(s2a[i + 1], w1.w);
    if (i == 0) v0 *= e.m0;
    if (i == 8) v1 *= e.m9;
    if (i == 16) v1 *= e.m17;
    const float2 r = Pack<T>::to_f2(Pack<T>::from_f2(v0, v1));
    q[i] = make_t2 ? r.x : 0.f;
    q[i + 1] = make_t2 ? r.y : 0.f;
  }
  ils_dw_taps<kIlsT2>(s2b, x, w1);
  ils_dw_taps<kIlsTO>(soa, q, ils_dw_param(prm + 80u));
  const float4 v1 = ils_dw_param(prm + 64u);
  ils_dw_taps<kIlsTO>(sob, q, v1);
  if (make_out) {
    uint32_t o[8];
#pragma unroll
    for (int k = 0; k < kIlsTO; k += 2) o[k >> 1] = Pack<T>::from_f2(prelu_m1(soa[k], v1.w), prelu_m1(soa[k + 1], v1.w));
    *reinterpret_cast<uint4*>(out) = make_uint4(o[0], o[1], o[2], o[3]);
    if (e.outB) *reinterpret_cast<uint4*>(out + 8) = make_uint4(o[4], o[5], o[6], o[7]);
  }
  ils_dw_taps<kIlsTO, true>(soa, q, ils_dw_param(prm + 48u));
  ils_dw_taps<kIlsT2, true>(s2a, x, ils_dw_param(prm));
}
// A T1 row of the tail from shared memory, converted to fp32: pA = group A's 16 bytes, pB = group B's (or zeros), pL / pR
// the neighbour groups' edge pairs (or zeros at the image's edges).
template <typename T>
__device__ __forceinline__ void ils_dw_load(float (&x)[kIlsTX], uint32_t pA, uint32_t pB, uint32_t pL, uint32_t pR) {
  const uint4 a = lds128(pA), b = lds128(pB);
  const uint32_t u[10] = {lds32(pL), a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w, lds32(pR)};
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    const float2 f = Pack<T>::to_f2(u[i]);
    x[2 * i] = f.x; x[2 * i + 1] = f.y;
  }
}

__device__ __forceinline__ void stsm_x4_trans(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.trans.shared.b16 [%0], {%1, %2, %3, %4};\n" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}

// GEMM and epilogue of one 64-pixel block (8 pixel groups) by a warpgroup.  Warp qd of the group holds accumulator rows
// [16 qd, 16 qd + 16) = pixel groups g0, g0 + 1 (g0 = 8 b + 2 qd); the m64nNk16 fragment gives a thread rows lane/4 and
// lane/4 + 8, columns 2 (lane % 4) + {0, 1} of every 8-column slab = pixel rows x channel pairs.  + bias, PReLU, pack to 16
// bits, then stmatrix.trans writes each 8 px x 8 channel fragment as 8 channel rows of 8 contiguous pixels — exactly the
// [group][slot][8 px] tile.  ngroups: groups of the chunk (later ones are MMA padding: stored to `dummy`), gstride = slots *
// 16 bytes.  eb / es: shared-memory tables of bias and (slope - 1) per channel.  The tile may be the A operand itself (T1
// written in place): the warpgroup barrier keeps every warp's stores behind the whole group's MMAs.
template <typename T, int N>
__device__ __forceinline__ void ils_block(uint64_t da, uint64_t db, int K16, int wg, uint32_t tile, uint32_t gstride, int g0, int ngroups,
                                          uint32_t eb, uint32_t es, uint32_t dummy, int lane) {
  float d[N / 2];
  wgmma_block<N>(d, da, db, K16);
  warpgroup_bar(wg);
  const int q = lane & 3, mrow = lane & 7, mat = lane >> 3;
#pragma unroll
  for (int cc = 0; cc < N / 16; ++cc) {
    const uint32_t co = (uint32_t)(cc * 16 + 2 * q) * 4u;
    const uint2 bA = lds64(eb + co), bB = lds64(eb + co + 32u), sA = lds64(es + co), sB = lds64(es + co + 32u);
    const float b0 = __uint_as_float(bA.x), b1 = __uint_as_float(bA.y), b2 = __uint_as_float(bB.x), b3 = __uint_as_float(bB.y);
    const float s0 = __uint_as_float(sA.x), s1 = __uint_as_float(sA.y), s2 = __uint_as_float(sB.x), s3 = __uint_as_float(sB.y);
    const float* r = d + 8 * cc;
    const uint32_t m0 = Pack<T>::from_f2(prelu_m1(r[0] + b0, s0), prelu_m1(r[1] + b1, s1));
    const uint32_t m1 = Pack<T>::from_f2(prelu_m1(r[2] + b0, s0), prelu_m1(r[3] + b1, s1));
    const uint32_t m2 = Pack<T>::from_f2(prelu_m1(r[4] + b2, s2), prelu_m1(r[5] + b3, s3));
    const uint32_t m3 = Pack<T>::from_f2(prelu_m1(r[6] + b2, s2), prelu_m1(r[7] + b3, s3));
    // matrix `mat` of the x4 store: pixel group g0 + (mat & 1), channels 16 cc + 8 (mat >> 1) ..; this lane addresses row mrow
    const int pg = g0 + (mat & 1);
    const uint32_t addr = pg < ngroups ? tile + (uint32_t)pg * gstride + (uint32_t)(cc * 16 + 8 * (mat >> 1) + mrow) * 16u
                                       : dummy + (uint32_t)(mat * 8 + mrow) * 16u;
    stsm_x4_trans(addr, m0, m1, m2, m3);
  }
}
template <typename T>
__device__ __forceinline__ void ils_block_n(int N, uint64_t da, uint64_t db, int K16, int wg, uint32_t tile, uint32_t gstride, int g0,
                                            int ngroups, uint32_t eb, uint32_t es, uint32_t dummy, int lane) {
  switch (N) {
    case 16: ils_block<T, 16>(da, db, K16, wg, tile, gstride, g0, ngroups, eb, es, dummy, lane); break;
    case 32: ils_block<T, 32>(da, db, K16, wg, tile, gstride, g0, ngroups, eb, es, dummy, lane); break;
    case 48: ils_block<T, 48>(da, db, K16, wg, tile, gstride, g0, ngroups, eb, es, dummy, lane); break;
    default: ils_block<T, 64>(da, db, K16, wg, tile, gstride, g0, ngroups, eb, es, dummy, lane); break;
  }
}

template <typename T, bool kStem = false>
__global__ void __launch_bounds__(kIlsMaxThreads, 1)
il_stream_kernel(const __grid_constant__ IlsArgs A, const __grid_constant__ CUtensorMap tmH, const __grid_constant__ CUtensorMap tmL) {
  extern __shared__ uint8_t smem_raw[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nthreads = blockDim.x, nwarps = nthreads >> 5;
  const uint32_t sbase = (smem_u32(smem_raw) + 127u) & ~127u;
  const uint32_t XL = sbase + A.off_xl, XH = sbase + A.off_xh, T1L = sbase + A.off_t1l, WBH = sbase + A.off_wbh,
                 WBL = sbase + A.off_wbl, BAR = sbase + A.off_bar, ZERO = sbase + A.off_zero;
  uint8_t* gbase = smem_raw + (sbase - smem_u32(smem_raw));      // generic pointer to the same place
  // barriers: [0,2) hi stage full, [2,5) lo stage full
  const uint32_t bar_h = BAR, bar_l = BAR + 16;
  const uint32_t EPI = sbase + A.off_epi, DUMMY = EPI + 1024;     // bias_h, sm1_h, bias_l, sm1_l (64 floats each); scratch rows

  const int H = A.H, W = A.W, Hl = H >> 1, Wl = W >> 1;
  const int Chi = A.Chi, Cli = A.Cli, Cho = A.Cho, Clo = A.Clo;
  const int GH = A.GH, GL = A.GL, SH = A.SH, SL = A.SL, ST = A.ST, NH = A.NH, NL = A.NL, K16 = A.K16;
  const int GR = A.GR, GLR = A.GLR, hl = A.hl, gsn = A.gsn;
  const int cpi = A.cpi;

  // ---- one-time setup -----------------------------------------------------------------------------------
  if (tid == 0) {
    for (int i = 0; i < 6; ++i) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;\n" ::"r"(BAR + 8 * i) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  }
  // weights -> K-major B operand: core matrices [n group][k group][8 n][8 k]
  {
    uint16_t* wb = reinterpret_cast<uint16_t*>(gbase + A.off_wbh);
    const uint16_t* src = reinterpret_cast<const uint16_t*>(A.wh);
    for (int i = tid; i < NH * K16; i += nthreads) {
      const int n = i / K16, k = i - n * K16;
      wb[(((n >> 3) * (K16 >> 3) + (k >> 3)) * 8 + (n & 7)) * 8 + (k & 7)] = k < A.K8 ? src[n * A.K8 + k] : (uint16_t)0;
    }
    if (NL > 0) {
      wb = reinterpret_cast<uint16_t*>(gbase + A.off_wbl);
      src = reinterpret_cast<const uint16_t*>(A.wl);
      for (int i = tid; i < NL * K16; i += nthreads) {
        const int n = i / K16, k = i - n * K16;
        wb[(((n >> 3) * (K16 >> 3) + (k >> 3)) * 8 + (n & 7)) * 8 + (k & 7)] = k < A.K8 ? src[n * A.K8 + k] : (uint16_t)0;
      }
    }
    if (tid < 16) reinterpret_cast<uint32_t*>(gbase + A.off_zero)[tid] = 0u;
    if (kStem) {
      // K-padding slots [Chi, K16) of both operand buffers: zero once (the im2col build never touches them, the in-place
      // epilogue only writes slots < NH <= Chi)
      // (both hi buffers: the build alternates between them so that it never overwrites the T1 the depthwise tail still reads)
      const int per = K16 - Chi, padh = per * 4 * GR, padl = per * 2 * GLR;
      for (int i = tid; i < 2 * padh + padl; i += nthreads) {
        const bool hb = i < 2 * padh;
        const int st = hb ? i / padh : 0, j = hb ? i - st * padh : i - 2 * padh, g_ = j / per, k_ = Chi + (j - g_ * per);
        sts128((hb ? XH + (uint32_t)st * (uint32_t)A.hi_stage_bytes + (uint32_t)(g_ * SH + k_) * 16u
                   : sbase + A.off_xlo + (uint32_t)(g_ * SL + k_) * 16u), make_uint4(0u, 0u, 0u, 0u));
      }
    }
    if (tid < kIlsMaxC) {
      float* ep = reinterpret_cast<float*>(gbase + A.off_epi);
      ep[tid] = A.bias_h[tid]; ep[kIlsMaxC + tid] = A.sm1_h[tid]; ep[2 * kIlsMaxC + tid] = A.bias_l[tid]; ep[3 * kIlsMaxC + tid] = A.sm1_l[tid];
    }
    // depthwise-tail parameter records: hi channels, then lo ones
    float* dp = reinterpret_cast<float*>(gbase + A.off_dwp);
    for (int i = tid; i < (Cho + Clo) * 24; i += nthreads) {
      const int ch = i / 24, j = i - ch * 24, lyr = j / 12, dy = (j >> 2) % 3, k = j & 3;
      const bool hi = ch < Cho;
      const int cc = hi ? ch : ch - Cho;
      const DwParams& P = lyr ? (hi ? A.dw2h : A.dw2l) : (hi ? A.dw1h : A.dw1l);
      float v = 0.f;
      if (k < 3) v = Pack<T>::to_f2(Pack<T>::from_f2(__ldg(P.w + cc * 9 + dy * 3 + k), 0.f)).x;
      else if (dy == 0) v = __ldg(P.b + cc);
      else if (dy == 1) v = __ldg(P.s + cc) - 1.f;
      dp[i] = v;
    }
  }
  asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
  __syncthreads();

  // depthwise-tail role of this thread (fixed for the whole kernel): a channel and two 8-pixel groups of a strip row
  // tail tasks are packed: threads [0, Cho * gsn / 2) own a hi (channel, group pair), the next Clo * ceil(gsn / 4) a lo one
  const int n_hi_tasks = Cho * (gsn >> 1);
  const bool dw_hi = tid < n_hi_tasks;
  const int dwt = dw_hi ? tid : tid - n_hi_tasks;
  const int Gs = dw_hi ? gsn : gsn >> 1;                  // this role's groups per strip row
  const int Gd = (Gs + 1) >> 1, Cd = dw_hi ? Cho : Clo, Sd = dw_hi ? SH : ST;   // Gd: tasks per channel of a strip row
  const bool dw_live = dwt < Cd * Gd;
  const int dc = dw_live ? dwt / Gd : 0, dg = dw_live ? 2 * (dwt - dc * Gd) : 0;  // dg: group A in the strip row
  const uint32_t prm = sbase + A.off_dwp + (uint32_t)((dw_hi ? dc : Cho + dc) * kIlsDwpBytes);
  const int dw_rows = dw_hi ? 4 : 2;                      // T1 rows per chunk of this role
  const int dHd = dw_hi ? H : Hl, dWd = dw_hi ? W : Wl;
  // byte offset inside a T1 chunk of group A's 16-byte row (row 0)
  const uint32_t dw_off = (uint32_t)((dg + hl) * Sd + dc) * 16u, dw_rowstep = (uint32_t)((dw_hi ? GR : GLR) * Sd) * 16u;
  const int Gimg = dw_hi ? GH : GL;                       // groups per image row of this role

  const int nbh = (4 * GR + 7) >> 3, nbl = NL > 0 ? (2 * GLR + 7) >> 3 : 0;     // 64-pixel GEMM blocks of a chunk
  const uint64_t db_h = gmma_desc(WBH, 128u, (uint32_t)(K16 >> 3) * 128u), db_l = gmma_desc(WBL, 128u, (uint32_t)(K16 >> 3) * 128u);
  const uint32_t hi_tx = (uint32_t)(64 * SH * GR), lo_tx = kStem ? (uint32_t)(A.BW * 4 * A.Ci * 4) : (uint32_t)(32 * SL * GLR);
  const uint32_t XLO = sbase + A.off_xlo;

  // ---- the CTA's range of the (image, chunk) sequence ------------------------------------------------
  int ra = (int)((long long)blockIdx.x * A.total_chunks / gridDim.x);
  const int rb = (int)((long long)(blockIdx.x + 1) * A.total_chunks / gridDim.x);
  uint32_t hq = 0, lq = 0;                               // running counts: hi loads, lo loads

  while (ra < rb) {
    const int item = ra / cpi, ca = ra - item * cpi;
    const int n = item / A.ns, gs0 = (item - n * A.ns) * gsn;                      // image, first hi group of the column strip
    const int cb = (ca + (rb - ra)) < cpi ? (ca + (rb - ra)) : cpi;
    ra += cb - ca;
    const int c0 = ca > 0 ? ca - 1 : 0, c1 = cb < cpi ? cb : cpi - 1;              // hi chunks walked (warm-up / look-ahead)
    const int cl0 = c0 > 0 ? c0 - 1 : 0, cl1 = c1 + 1 < cpi ? c1 + 1 : cpi - 1;    // lo chunks loaded
    const int out_lo = dw_hi ? 4 * ca : 2 * ca, out_hi = dw_hi ? 4 * cb : 2 * cb;  // rows this role stores
    const uint32_t hq0 = hq, lq0 = lq;
    hq += (uint32_t)(c1 - c0 + 1);
    lq += (uint32_t)(cl1 - cl0 + 1);
    auto hi_stage = [&](int c) { return XH + ((hq0 + (uint32_t)(c - c0)) & 1u) * (uint32_t)A.hi_stage_bytes; };
    auto lo_stage = [&](int cl) { return XL + ((lq0 + (uint32_t)(cl - cl0)) % 3u) * (uint32_t)A.lo_stage_bytes; };
    auto issue_hi = [&](int c) {
      const uint32_t q = hq0 + (uint32_t)(c - c0), bar = bar_h + 8 * (q & 1u);
      mbar_expect_tx_a(bar, hi_tx);
      tma_load_5d(hi_stage(c), &tmH, bar, 0, 0, gs0 - hl, 4 * c, n);
    };
    auto issue_lo = [&](int cl) {
      const uint32_t q = lq0 + (uint32_t)(cl - cl0), bar = bar_l + 8 * (q % 3u);
      mbar_expect_tx_a(bar, lo_tx);
      if (kStem) tma_load_4d_a(lo_stage(cl), &tmL, bar, 8 * (gs0 - hl) - 4, 4 * cl, 0, n);     // image block: rows [4 cl, 4 cl + 4), all channels
      else tma_load_5d(lo_stage(cl), &tmL, bar, 0, 0, (gs0 >> 1) - hl, 2 * cl, n);
    };
    if (tid == 0) {
      asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
      if (!kStem) {
        issue_hi(c0);
        if (c0 + 1 <= c1) issue_hi(c0 + 1);
      }
      for (int cl = cl0; cl <= cl1 && cl <= c0 + 1; ++cl) issue_lo(cl);
    }
    int lo_waited = 0;
    IlsTail tl;                                                                    // the tail's open rows (ils_dw_push)
    if (dw_live) ils_dw_start(tl, prm);
    const int gimg = (dw_hi ? gs0 : gs0 >> 1) + dg;                                // group A in the image row
    // group B: in the image (else zeros, T2 at x0+8 is padding); in the strip (else its outputs belong to the next one)
    // the neighbour pair right of B: zeros past the image, and past the tile (then B is the halo and not stored)
    const bool hasB = gimg + 1 < Gimg, zeroL = gimg == 0, zeroR = gimg + 2 >= Gimg || dg + 2 >= Gs + hl;
    IlsTaskEdges edg;
    edg.m0 = zeroL ? 0.f : 1.f;
    edg.m9 = hasB ? 1.f : 0.f;
    edg.m17 = gimg + 2 >= Gimg ? 0.f : 1.f;
    edg.outB = dg + 1 < Gs;
    const uint32_t sd = (uint32_t)Sd * 16u;
    uint16_t* ybase = reinterpret_cast<uint16_t*>(dw_hi ? A.yh : A.yl) + ((size_t)n * Cd + dc) * dHd * dWd + 8 * gimg;

    for (int c = c0; c <= c1; ++c) {
      // ---- 1. the chunk's inputs have landed -----------------------------------------------------------
      {
        const uint32_t q = hq0 + (uint32_t)(c - c0);
        if (!kStem) mbar_wait_a(bar_h + 8 * (q & 1u), (q >> 1) & 1u);
        const int need = (c + 1 < cpi ? c + 1 : cpi - 1) - cl0 + 1;
        while (lo_waited < need) {
          const uint32_t ql = lq0 + (uint32_t)lo_waited;
          mbar_wait_a(bar_l + 8 * (ql % 3u), (ql / 3u) & 1u);
          ++lo_waited;
        }
      }
      const uint32_t xh = hi_stage(c), xl = kStem ? XLO : lo_stage(c);
      if (kStem) {
        // ---- 2s. im2col of the image chunk (hi) and of its 2x2 max-pool (lo): a task = one (row, group, ci, ky) and makes
        //          the three kx slots from one 10-pixel window -----------------------------------------------------------
        const int Ci = A.Ci, BW = A.BW;
        const int n_hi = 4 * GR * Ci * 3, n_lo = Clo > 0 ? 2 * GLR * Ci * 3 : 0;
        for (int task = tid; task < n_hi + n_lo; task += nthreads) {
          const bool hb = task < n_hi;
          const int t = hb ? task : task - n_hi, Gt = hb ? GR : GLR;
          const int ck = t % (Ci * 3), rg = t / (Ci * 3);               // ck = ci * 3 + ky; rg = row * Gt + group
          const int ci = ck / 3, ky = ck - ci * 3, r = rg / Gt, g = rg - r * Gt;
          float f[10];
          if (hb) {
            const int yy = 4 * c + r + ky - 1;                           // image row of this tap row
            if (yy >= 0 && yy < H) {
              const uint32_t a = lo_stage(yy >> 2) + (uint32_t)(((ci * 4 + (yy & 3)) * BW + 8 * g + 3) * 4);
              const uint4 m0 = lds128(a + 4u), m1 = lds128(a + 20u);
              f[0] = __uint_as_float(lds32(a)); f[9] = __uint_as_float(lds32(a + 36u));
              f[1] = __uint_as_float(m0.x); f[2] = __uint_as_float(m0.y); f[3] = __uint_as_float(m0.z); f[4] = __uint_as_float(m0.w);
              f[5] = __uint_as_float(m1.x); f[6] = __uint_as_float(m1.y); f[7] = __uint_as_float(m1.z); f[8] = __uint_as_float(m1.w);
            } else {
#pragma unroll
              for (int j = 0; j < 10; ++j) f[j] = 0.f;
            }
          } else {
            const int yl = 2 * c + r + ky - 1;                           // lo row of this tap row: max of image rows 2 yl, 2 yl + 1
            const int col0 = 16 * g - 8 * hl + 2;                        // block column of image x = 2 (xl0 - 1)
            if (yl >= 0 && yl < Hl) {
              const uint32_t a = lo_stage(yl >> 1) + (uint32_t)(((ci * 4 + ((2 * yl) & 3)) * BW) * 4);
#pragma unroll
              for (int j = 0; j < 10; ++j) {
                const int col = col0 + 2 * j;
                float v = 0.f;
                if (col >= 0 && col + 1 < BW) {                          // outside: the never-read outer half of a halo group
                  const uint2 u0 = lds64(a + (uint32_t)col * 4u), u1 = lds64(a + (uint32_t)(col + BW) * 4u);
                  v = fmaxf(fmaxf(__uint_as_float(u0.x), __uint_as_float(u0.y)), fmaxf(__uint_as_float(u1.x), __uint_as_float(u1.y)));
                }
                f[j] = v;
              }
            } else {
#pragma unroll
              for (int j = 0; j < 10; ++j) f[j] = 0.f;
            }
          }
          const uint32_t e0 = Pack<T>::from_f2(f[0], f[1]), e1 = Pack<T>::from_f2(f[2], f[3]), e2 = Pack<T>::from_f2(f[4], f[5]),
                         e3 = Pack<T>::from_f2(f[6], f[7]), e4 = Pack<T>::from_f2(f[8], f[9]);
          const uint32_t o0 = Pack<T>::from_f2(f[1], f[2]), o1 = Pack<T>::from_f2(f[3], f[4]), o2 = Pack<T>::from_f2(f[5], f[6]),
                         o3 = Pack<T>::from_f2(f[7], f[8]);
          const uint32_t dst = (hb ? xh + (uint32_t)(rg * SH) * 16u : xl + (uint32_t)(rg * SL) * 16u) + (uint32_t)(ck * 3) * 16u;
          sts128(dst, make_uint4(e0, e1, e2, e3));                       // kx = 0: pixels x-1 .. x+6
          sts128(dst + 16u, make_uint4(o0, o1, o2, o3));                 // kx = 1: x .. x+7
          sts128(dst + 32u, make_uint4(e1, e2, e3, e4));                 // kx = 2: x+1 .. x+8
        }
      } else {
      // ---- 2. resample both ways ------------------------------------------------------------------------
        const int n_up = Cli * GR, n_pool = Clo > 0 ? Chi * GLR : 0;
        for (int task = tid; task < n_up + n_pool; task += nthreads) {
          if (task < n_up) {
            // bilinear x2 (align_corners=False): hi pixel 2j = 1/4 lo[j-1] + 3/4 lo[j], 2j+1 = 3/4 lo[j] + 1/4 lo[j+1], clamped
            const int cl_ = task / GR, gr = task - cl_ * GR;                    // gr: group in the tile row; g: in the image row
            const int g = gs0 - hl + gr;
            if (g < 0 || g >= GH) continue;                                       // halo group outside the image: stays zero, never read
            const int glr = (g >> 1) - (gs0 >> 1) + hl, hf = g & 1;               // lo group in the lo tile row
            const uint32_t offM = (uint32_t)(glr * SL + cl_) * 16u + 8u * hf;
            const uint32_t offL = hf ? offM - 2u : (g == 0 ? offM : offM - (uint32_t)SL * 16u + 14u);
            const uint32_t offR = hf ? (g == GH - 1 ? offM + 6u : offM + (uint32_t)SL * 16u - 8u) : offM + 8u;
            float hrow[4][8];
            const uint16_t w25 = Pack<T>::bits(0.25f), w75 = Pack<T>::bits(0.75f);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              int R = 2 * c - 1 + k;
              R = R < 0 ? 0 : (R > Hl - 1 ? Hl - 1 : R);
              const uint32_t rowb = lo_stage(R >> 1) + (uint32_t)((R & 1) * GLR * SL) * 16u;
              const uint2 m = lds64(rowb + offM);
              const uint16_t vl = lds16(rowb + offL), vr = lds16(rowb + offR);
              const uint16_t v0 = (uint16_t)m.x, v1 = (uint16_t)(m.x >> 16), v2 = (uint16_t)m.y, v3 = (uint16_t)(m.y >> 16);
              hrow[k][0] = Pack<T>::fma16(v0, w75, Pack<T>::fma16(vl, w25, 0.f));
              hrow[k][1] = Pack<T>::fma16(v0, w75, Pack<T>::fma16(v1, w25, 0.f));
              hrow[k][2] = Pack<T>::fma16(v1, w75, Pack<T>::fma16(v0, w25, 0.f));
              hrow[k][3] = Pack<T>::fma16(v1, w75, Pack<T>::fma16(v2, w25, 0.f));
              hrow[k][4] = Pack<T>::fma16(v2, w75, Pack<T>::fma16(v1, w25, 0.f));
              hrow[k][5] = Pack<T>::fma16(v2, w75, Pack<T>::fma16(v3, w25, 0.f));
              hrow[k][6] = Pack<T>::fma16(v3, w75, Pack<T>::fma16(v2, w25, 0.f));
              hrow[k][7] = Pack<T>::fma16(v3, w75, Pack<T>::fma16(vr, w25, 0.f));
            }
            const uint32_t dst = xh + (uint32_t)(gr * SH + Chi + cl_) * 16u;
#pragma unroll
            for (int rr = 0; rr < 4; ++rr) {
              // hi row 4c+rr: rr 0: (k0 1/4, k1 3/4); 1: (k1 3/4, k2 1/4); 2: (k1 1/4, k2 3/4); 3: (k2 3/4, k3 1/4)
              const int km = rr < 2 ? 1 : 2, ko = rr == 0 ? 0 : (rr == 3 ? 3 : (rr == 1 ? 2 : 1));
              uint4 o;
              o.x = Pack<T>::from_f2(0.75f * hrow[km][0] + 0.25f * hrow[ko][0], 0.75f * hrow[km][1] + 0.25f * hrow[ko][1]);
              o.y = Pack<T>::from_f2(0.75f * hrow[km][2] + 0.25f * hrow[ko][2], 0.75f * hrow[km][3] + 0.25f * hrow[ko][3]);
              o.z = Pack<T>::from_f2(0.75f * hrow[km][4] + 0.25f * hrow[ko][4], 0.75f * hrow[km][5] + 0.25f * hrow[ko][5]);
              o.w = Pack<T>::from_f2(0.75f * hrow[km][6] + 0.25f * hrow[ko][6], 0.75f * hrow[km][7] + 0.25f * hrow[ko][7]);
              sts128(dst + (uint32_t)(rr * GR * SH) * 16u, o);
            }
          } else {
            // max_pool2d 2x2: lo group glr of lo rows 2c, 2c+1 from the two hi groups under it, 4 hi rows.  With a halo the
            // outer hi group of the tile's first / last lo group is not in the tile: that half is never read downstream.
            const int t = task - n_up, ch = t / GLR, glr = t - ch * GLR;
            const int ga = 2 * glr - hl;                                          // tile index of the left hi group
            const bool okA = ga >= 0, okB = ga + 1 < GR;
            const uint32_t src = xh + (uint32_t)(ga * SH + ch) * 16u;
            const uint32_t dst = xl + (uint32_t)(glr * SL + Cli + ch) * 16u;
#pragma unroll
            for (int lr = 0; lr < 2; ++lr) {
              const uint32_t r0 = src + (uint32_t)(2 * lr * GR * SH) * 16u, r1 = r0 + (uint32_t)(GR * SH) * 16u;
              const uint4 a0 = lds128(okA ? r0 : ZERO), a1 = lds128(okB ? r0 + (uint32_t)SH * 16u : ZERO), c0_ = lds128(okA ? r1 : ZERO),
                          c1_ = lds128(okB ? r1 + (uint32_t)SH * 16u : ZERO);
              auto hmax = [](uint32_t u, uint32_t v) {       // two lo pixels from the vertical maxima of 4 hi pixels
                return __byte_perm(Pack<T>::max2(u, __byte_perm(u, 0u, 0x1032)), Pack<T>::max2(v, __byte_perm(v, 0u, 0x1032)), 0x5410);
              };
              uint4 o;
              o.x = hmax(Pack<T>::max2(a0.x, c0_.x), Pack<T>::max2(a0.y, c0_.y));
              o.y = hmax(Pack<T>::max2(a0.z, c0_.z), Pack<T>::max2(a0.w, c0_.w));
              o.z = hmax(Pack<T>::max2(a1.x, c1_.x), Pack<T>::max2(a1.y, c1_.y));
              o.w = hmax(Pack<T>::max2(a1.z, c1_.z), Pack<T>::max2(a1.w, c1_.w));
              sts128(dst + (uint32_t)(lr * GLR * SL) * 16u, o);
            }
          }
        }
      }
      asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");    // generic writes -> visible to the tensor core / TMA
      __syncthreads();                                                    // (A)
      // ---- 3. next loads (one thread of the last warp) ------------------------------------------------------
      if (warp == nwarps - 1 && lane == 0) {
        asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
        if (!kStem && c >= c0 + 1 && c + 1 <= c1) issue_hi(c + 1);       // stage of chunk c-1: its T1 was consumed
        if (c + 2 <= cl1) issue_lo(c + 2);                               // stage of lo chunk c-1: last read by this chunk's up-sample
      }
      // ---- 4. GEMM + epilogue: warpgroup w takes the 64-pixel blocks w, w + wgs, ..; fp32 accumulators in registers ->
      //         bias, PReLU, 16-bit -> T1 (hi: in place over the block's own pixel groups; lo: its own buffer) ----------------
      if (warp < (nwarps & ~3)) {
        const int wg = warp >> 2, qd = warp & 3, wgs = nwarps >> 2;
        for (int b = wg; b < nbh + nbl; b += wgs) {
          if (b < nbh)
            ils_block_n<T>(NH, gmma_desc(xh + (uint32_t)(b * 8 * SH) * 16u, 128u, (uint32_t)SH * 16u), db_h, K16, wg, xh, (uint32_t)SH * 16u,
                           b * 8 + qd * 2, 4 * GR, EPI, EPI + 256u, DUMMY, lane);
          else
            ils_block_n<T>(NL, gmma_desc(xl + (uint32_t)((b - nbh) * 8 * SL) * 16u, 128u, (uint32_t)SL * 16u), db_l, K16, wg, T1L,
                           (uint32_t)ST * 16u, (b - nbh) * 8 + qd * 2, 2 * GLR, EPI + 512u, EPI + 768u, DUMMY, lane);
        }
      }
      __syncthreads();                                                    // (B)
      // ---- 5. depthwise tail over the chunk's rows --------------------------------------------------------
      if (dw_live) {
        const uint32_t t1b = (dw_hi ? xh : T1L) + dw_off;
        // T1 row r arriving; T2 row r-1; output row r-2.  Rows come in pairs (dw_rows is 4 or 2): the open rows swap roles
        auto row = [&](float (&a2)[kIlsT2], float (&b2)[kIlsT2], float (&ao)[kIlsTO], float (&bo)[kIlsTO], int rr) {
          const int r = dw_rows * c + rr, tr = r - 1, orow = r - 2;
          const bool make_t2 = tr >= 0 && tr >= out_lo - 1 && tr <= out_hi;
          const bool make_out = orow >= out_lo && orow < out_hi;
          const uint32_t p = t1b + (uint32_t)rr * dw_rowstep;
          float x[kIlsTX];
          ils_dw_load<T>(x, p, hasB ? p + sd : ZERO, zeroL ? ZERO : p - sd + 12u, zeroR ? ZERO : p + 2u * sd);
          ils_dw_push<T>(a2, b2, ao, bo, x, prm, make_t2, edg, make_out, ybase + (size_t)orow * dWd);
        };
        for (int rr = 0; rr < dw_rows; rr += 2) {
          row(tl.s2a, tl.s2b, tl.soa, tl.sob, rr);
          row(tl.s2b, tl.s2a, tl.sob, tl.soa, rr + 1);
        }
      }
    }
    // ---- image bottom: two rows of zero padding flush the last two output rows ----------------------------
    if (cb == cpi && dw_live) {
      float z[kIlsTX];
#pragma unroll
      for (int i = 0; i < kIlsTX; ++i) z[i] = 0.f;
      ils_dw_push<T>(tl.s2a, tl.s2b, tl.soa, tl.sob, z, prm, true, edg, dHd - 2 >= out_lo, ybase + (size_t)(dHd - 2) * dWd);
      ils_dw_push<T>(tl.s2b, tl.s2a, tl.sob, tl.soa, z, prm, false, edg, dHd - 1 >= out_lo, ybase + (size_t)(dHd - 1) * dWd);
    }
    __syncthreads();          // every shared-memory read of this piece is done before the next piece's loads overwrite it
  }
}

}  // namespace csnet
