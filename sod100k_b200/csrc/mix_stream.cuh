// mix_stream.cuh — a 1x1 CSNET_OP_MIX / CSNET_OP_MIXPROJ op as a persistent, warp-specialised TMA -> wgmma -> epilogue
// pipeline (reference: the 1x1 gOctaveCBR calls of CSFHead.forward, CSNet/model/csnet.py:202-206 over gOctaveConv.forward
// :664-726, and cls_layer :383 folded into the epilogue).
//
//   dst[c] = PReLU( bias[c] + sum_i W_i . x_i  +  sum_r bilinear_up(low_r)[c] )          (then, MIXPROJ: dot with proj_w)
//
//   * every conv path is a plain 1x1 over a 16-bit tensor at the destination's resolution (W % 8 == 0).  A chunk of A.rows
//     rows (chosen per op by the plan) of each input arrives by cp.async.bulk.tensor.5d in the tensor-core operand layout
//     [row][8-px group][slot][8 px] (channel slots past C zero-filled = the K padding): the threads never touch the operands.
//     Under the same barrier, cp.async.bulk.tensor.4d brings the fp32 rows of each resample-add source that the chunk's
//     bilinear taps reach.
//   * warp 0 (one lane) is the TMA producer over a ring of stages; kMsGroups consumer warpgroups share the 64-pixel blocks
//     of each chunk: wgmma.mma_async (M = 64 pixels, N = ru16(Cout), K = 16 per instruction, the paths of the op accumulate
//     into the same registers = K-concatenation), then the epilogue from the accumulator fragment: bias, the op's
//     resample-add paths (fp32 low-resolution conv results of the up-paths, gathered bilinearly from shared memory), PReLU, then
//     either stores of the Cout planes or the projection onto one fp32 channel (cls_layer) — the Cout-channel tensor is
//     never written.  While one warpgroup runs its epilogue, the others' MMAs and the producer's loads are in flight.
// 3x3 form (k3: every conv path a 3x3, pad 1 — the stage-entry gOctaveCBR of stride-2 ILBlocks, csnet.py:60-71 with the
// avg-pooled inputs): the TMA box carries one halo row above and below (zero fill = the conv padding), two builder warps
// derive the x-1 / x+1 shifted copies of the tile in shared memory (one 16-byte funnel shift per group), and the nine taps are
// nine accumulating MMAs whose A descriptors differ only by a row offset (ky) and the copy (kx) — no im2col.
// HBM traffic = the op's algorithmic bytes (inputs once, output once; the 3x3 form re-reads its two halo rows per chunk from L2).
#pragma once
#include "il_stream.cuh"

namespace csnet {

constexpr int kMsMaxIn = 3, kMsMaxRs = 2, kMsMaxC = 80, kMsRows = 2;   // kMsRows: the chunk height the kernel choice is judged by
constexpr int kMsGroups = 3, kMsThreads = (4 + 4 * kMsGroups) * 32;   // warp 0: TMA; 2, 3: 3x3 builders; 4..: consumer warpgroups

struct MsArgs {
  void* dst;
  const float* w[kMsMaxIn];             // fp32 [cin][cout] of each conv path
  float bias[kMsMaxC], sm1[kMsMaxC], proj[kMsMaxC];
  float proj_b;
  int32_t has_proj, has_slope, dst_f32;
  int32_t n_in, cin[kMsMaxIn], cout0[kMsMaxIn], cout[kMsMaxIn], S[kMsMaxIn], K16[kMsMaxIn], in_off[kMsMaxIn];
  int32_t n_rs, r_dtype[kMsMaxRs], r_up[kMsMaxRs], r_H[kMsMaxRs], r_W[kMsMaxRs], r_C[kMsMaxRs], r_c0[kMsMaxRs], r_cout0[kMsMaxRs], r_n[kMsMaxRs];
  int32_t r_rows[kMsMaxRs], r_off[kMsMaxRs];   // low-resolution rows a chunk's taps reach; their tile's offset in a stage
  int32_t N, H, W, C, NN, G, nb, rows;  // destination dims; NN = ru16(C); G = W / 8; nb = 64-pixel GEMM blocks per chunk of `rows` rows
  int32_t k3, copy_bytes[kMsMaxIn];     // 3x3 form; bytes of one of the three copies (centre, x-1, x+1) of input i's tile
  int32_t cpi, total_chunks, n_stages, stage_bytes, tx_bytes;
  int32_t off_stage, off_wb[kMsMaxIn], off_bar, off_tab, smem_bytes;
};

struct MsTap {                           // bilinear taps of one destination pixel in a low-resolution plane
  int32_t o00, o01, o10, o11;
  float w00, w01, w10, w11;
};
__host__ __device__ __forceinline__ MsTap ms_tap(int Hs, int Ws, int up, int oy, int ox) {
  // F.interpolate(bilinear, align_corners=False): source index (dst + 0.5) / up - 0.5, clamped at 0; the +1 neighbour clamped
  const float inv = 1.0f / (float)up;
  float sy = ((float)oy + 0.5f) * inv - 0.5f, sx = ((float)ox + 0.5f) * inv - 0.5f;
  sy = sy < 0.f ? 0.f : sy;
  sx = sx < 0.f ? 0.f : sx;
  const int y0 = (int)sy, x0 = (int)sx;
  const int y1 = y0 + (y0 < Hs - 1 ? 1 : 0), x1 = x0 + (x0 < Ws - 1 ? 1 : 0);
  const float ly = sy - (float)y0, lx = sx - (float)x0, hy = 1.f - ly, hx = 1.f - lx;
  MsTap t;
  t.o00 = y0 * Ws + x0; t.o01 = y0 * Ws + x1; t.o10 = y1 * Ws + x0; t.o11 = y1 * Ws + x1;
  t.w00 = hy * hx; t.w01 = hy * lx; t.w10 = ly * hx; t.w11 = ly * lx;
  return t;
}
__device__ __forceinline__ float ldsf(uint32_t a) { return __uint_as_float(lds32(a)); }
// The first low-resolution row that the taps of destination row oy reach: the top row of a chunk's staged source tile.
__host__ __device__ __forceinline__ int ms_row0(int Hs, int Ws, int up, int oy) { return ms_tap(Hs, Ws, up, oy, 0).o00 / Ws; }

// Consumer warpgroup `wg`: the (chunk, block) tasks t = k * nb + blk with t % kMsGroups == wg.  A task = one 64-pixel
// block: wgmma over every conv path (and tap) of the op into one fp32 accumulator fragment, then the epilogue from the
// fragment (rows lane/4 and lane/4 + 8 of the warp's 16 pixels, channel pairs 2 (lane % 4) + {0, 1} of every 8-channel slab):
// bias, NRS resample-add paths (fp32 sources), PReLU, then 16-bit (or fp32) stores of the C planes, or (PROJ) the projection
// onto one fp32 channel, summed over the four lanes that share a pixel.  tab: shared-memory float4 {bias, slope-1, proj, 0}.
// Every warpgroup waits for every chunk and releases its stage once (bar_empty counts kMsGroups arrivals), so the
// barriers' phases never run ahead of a warpgroup that has no task in a chunk.
template <typename T, int NRS, bool PROJ, int NN>
__device__ __forceinline__ void ms_consume(const MsArgs& A, uint32_t sbase, uint32_t STG, uint32_t tab, uint32_t bar_full, uint32_t bar_ready,
                                           uint32_t bar_empty, int ra, int rb, int wg, int qd, int lane) {
  const int H = A.H, W = A.W, C = A.C, G = A.G, nb = A.nb, NS = A.n_stages, taps = A.k3 ? 9 : 1;
  const size_t plane = (size_t)H * W;
  const int q = lane & 3;
  for (int idx = ra, k = 0; idx < rb; ++idx, ++k) {
    const int s = k % NS, n = idx / A.cpi, c = idx - n * A.cpi;
    const uint32_t st = STG + (uint32_t)s * (uint32_t)A.stage_bytes;
    mbar_wait_a(bar_ready + 8 * s, (uint32_t)(k / NS) & 1u);
    if (NRS > 0 && A.k3) mbar_wait_a(bar_full + 8 * s, (uint32_t)(k / NS) & 1u);   // the source tiles, read by these threads
    // staged source tile j: [r_n channels][r_rows rows from ms_row0][r_W]; rsb[j] addresses its (virtual) row 0
    uint32_t rsb[NRS > 0 ? NRS : 1], rcs[NRS > 0 ? NRS : 1];
#pragma unroll
    for (int j = 0; j < NRS; ++j) {
      rcs[j] = (uint32_t)(A.r_rows[j] * A.r_W[j]) * 4u;
      rsb[j] = st + (uint32_t)A.r_off[j] - (uint32_t)(ms_row0(A.r_H[j], A.r_W[j], A.r_up[j], c * A.rows) * A.r_W[j]) * 4u;
    }
    for (int blk = 0; blk < nb; ++blk) {
      if ((k * nb + blk) % kMsGroups != wg) continue;                      // warpgroup-uniform
      float d[NN / 2];
#pragma unroll
      for (int i = 0; i < NN / 2; ++i) d[i] = 0.f;
      wgmma_fence();
      uint32_t acc = 0;
      for (int i = 0; i < A.n_in; ++i) {
        for (int tap = 0; tap < taps; ++tap) {
          // 3x3: tap (ky, kx) reads copy kx (x-1 / centre / x+1 = copies 1 / 0 / 2) ky tile rows down
          const int ky = tap / 3, kx = tap - 3 * ky, cp = kx == 1 ? 0 : (kx == 0 ? 1 : 2);
          const uint32_t abase = st + (uint32_t)A.in_off[i] + (A.k3 ? (uint32_t)cp * (uint32_t)A.copy_bytes[i] + (uint32_t)(ky * G * A.S[i]) * 16u : 0u);
          const uint64_t da = gmma_desc(abase + (uint32_t)(blk * 8 * A.S[i]) * 16u, 128u, (uint32_t)A.S[i] * 16u);
          const uint64_t db = gmma_desc(sbase + (uint32_t)A.off_wb[i] + (uint32_t)(tap * NN * A.K16[i] * 2), 128u, (uint32_t)(A.K16[i] >> 3) * 128u);
          for (int ks = 0; ks < (A.K16[i] >> 4); ++ks) {
            Wgmma<NN>::mma(d, da + (uint64_t)(16 * ks), db + (uint64_t)(16 * ks), acc);
            acc = 1;
          }
        }
      }
      wgmma_commit_wait();
      // ---- epilogue: this thread's two pixels (h = 0, 1), one at a time ---------------------------------------------------
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int p = blk * 64 + qd * 16 + (lane >> 2) + 8 * h, pg = p >> 3;
        const bool valid = pg < A.rows * G;
        const int r = pg / G, g = pg - r * G;
        const int y = valid ? c * A.rows + r : c * A.rows, x = valid ? 8 * g + (p & 7) : 0;   // (invalid: a row of the tile)
        MsTap tp[NRS > 0 ? NRS : 1];
#pragma unroll
        for (int j = 0; j < NRS; ++j) tp[j] = ms_tap(A.r_H[j], A.r_W[j], A.r_up[j], y, x);
        float proj_acc = 0.f;
#pragma unroll
        for (int i = 0; i < NN / 8; ++i) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int ch = 8 * i + 2 * q + e;                                 // channels >= C: zero weights, zero tables -> harmless work
            const uint4 t4 = lds128(tab + (uint32_t)ch * 16u);
            float v = d[4 * i + 2 * h + e] + __uint_as_float(t4.x);
#pragma unroll
            for (int t = 0; t < NRS; ++t) {
              if (ch < A.r_n[t]) {                                            // (resample-add paths cover channels [0, r_n): checked by the host)
                const uint32_t s_ = rsb[t] + (uint32_t)ch * rcs[t];
                v += tp[t].w00 * ldsf(s_ + 4u * (uint32_t)tp[t].o00) + tp[t].w01 * ldsf(s_ + 4u * (uint32_t)tp[t].o01) +
                     tp[t].w10 * ldsf(s_ + 4u * (uint32_t)tp[t].o10) + tp[t].w11 * ldsf(s_ + 4u * (uint32_t)tp[t].o11);
              }
            }
            v = prelu_m1(v, __uint_as_float(t4.y));
            if (PROJ) proj_acc = fmaf(__uint_as_float(t4.z), v, proj_acc);
            else if (valid && ch < C) {
              const size_t o = ((size_t)n * C + (size_t)ch) * plane + (size_t)y * W + x;
              if (A.dst_f32) reinterpret_cast<float*>(A.dst)[o] = v;
              else reinterpret_cast<uint16_t*>(A.dst)[o] = Pack<T>::bits(v);
            }
          }
        }
        if (PROJ) {
          proj_acc += __shfl_xor_sync(0xffffffffu, proj_acc, 1);
          proj_acc += __shfl_xor_sync(0xffffffffu, proj_acc, 2);
          if (q == 0 && valid) reinterpret_cast<float*>(A.dst)[((size_t)n * H + y) * W + x] = proj_acc + A.proj_b;
        }
      }
    }
    warpgroup_bar(wg);                                                      // the group's MMAs of this chunk have all completed
    if (qd == 0 && lane == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(bar_empty + 8 * s) : "memory");
  }
}

template <typename T, int NRS, bool PROJ>
__device__ __forceinline__ void ms_consume_n(const MsArgs& A, uint32_t sbase, uint32_t STG, uint32_t tab, uint32_t bar_full, uint32_t bar_ready,
                                             uint32_t bar_empty, int ra, int rb, int wg, int qd, int lane) {
  switch (A.NN) {
    case 16: ms_consume<T, NRS, PROJ, 16>(A, sbase, STG, tab, bar_full, bar_ready, bar_empty, ra, rb, wg, qd, lane); break;
    case 32: ms_consume<T, NRS, PROJ, 32>(A, sbase, STG, tab, bar_full, bar_ready, bar_empty, ra, rb, wg, qd, lane); break;
    case 48: ms_consume<T, NRS, PROJ, 48>(A, sbase, STG, tab, bar_full, bar_ready, bar_empty, ra, rb, wg, qd, lane); break;
    case 64: ms_consume<T, NRS, PROJ, 64>(A, sbase, STG, tab, bar_full, bar_ready, bar_empty, ra, rb, wg, qd, lane); break;
    default: ms_consume<T, NRS, PROJ, 80>(A, sbase, STG, tab, bar_full, bar_ready, bar_empty, ra, rb, wg, qd, lane); break;
  }
}

// PROJ_RS: the instantiation for projected (MIXPROJ) ops that also carry resample-add paths.  It is a kernel of its own so
// that its consumers do not enlarge the register / spill footprint of the instantiation every other op runs.
template <typename T, bool PROJ_RS = false>
__global__ void __launch_bounds__(kMsThreads, 1)
mix_stream_kernel(const __grid_constant__ MsArgs A, const __grid_constant__ CUtensorMap tm0, const __grid_constant__ CUtensorMap tm1,
                  const __grid_constant__ CUtensorMap tm2, const __grid_constant__ CUtensorMap tr0, const __grid_constant__ CUtensorMap tr1) {
  extern __shared__ uint8_t smem_raw[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t sbase = (smem_u32(smem_raw) + 127u) & ~127u;
  uint8_t* gbase = smem_raw + (sbase - smem_u32(smem_raw));
  const uint32_t STG = sbase + A.off_stage, BAR = sbase + A.off_bar;
  // barriers: full[8] at +0, empty[8] at +64, built[8] at +128
  const uint32_t bar_full = BAR, bar_empty = BAR + 64, bar_built = BAR + 128;
  const uint32_t TAB = sbase + A.off_tab;                                 // float4 {bias, slope - 1, proj, 0} per channel (kMsMaxC)
  float* tab = reinterpret_cast<float*>(gbase + A.off_tab);
  const int NS = A.n_stages, NN = A.NN;

  if (tid == 0) {
    for (int i = 0; i < NS; ++i) {
      asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;\n" ::"r"(bar_full + 8 * i) : "memory");
      asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(bar_empty + 8 * i), "r"(kMsGroups) : "memory");   // one per consumer warpgroup
      asm volatile("mbarrier.init.shared::cta.b64 [%0], 2;\n" ::"r"(bar_built + 8 * i) : "memory");      // the two builder warps
    }
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  }
  // weights of every conv path -> K-major B operand [n group][k group][8 n][8 k], zero outside the path's cout slice / cin
  for (int i = 0; i < A.n_in; ++i) {
    uint16_t* wb = reinterpret_cast<uint16_t*>(gbase + A.off_wb[i]);
    const int K16 = A.K16[i], taps = A.k3 ? 9 : 1;
    for (int e = tid; e < taps * NN * K16; e += kMsThreads) {
      const int tap = e / (NN * K16), r_ = e - tap * NN * K16, n = r_ / K16, k = r_ - n * K16;
      const int nn = n - A.cout0[i];
      const float v = (nn >= 0 && nn < A.cout[i] && k < A.cin[i]) ? __ldg(A.w[i] + ((size_t)k * taps + tap) * A.cout[i] + nn) : 0.f;   // blob: [cin][taps][cout]
      wb[tap * NN * K16 + (((n >> 3) * (K16 >> 3) + (k >> 3)) * 8 + (n & 7)) * 8 + (k & 7)] = Pack<T>::bits(v);
    }
    if (A.k3) {
      // K-padding slots [cin, S) of the two shifted copies of every stage: zero once (the builders only write real channels)
      const int tg = (A.rows + 2) * A.G, per = A.S[i] - A.cin[i];
      for (int e = tid; e < NS * 2 * tg * per; e += kMsThreads) {
        const int st = e / (2 * tg * per), r2 = e - st * 2 * tg * per, cp = r2 / (tg * per), r3 = r2 - cp * tg * per, g_ = r3 / per, k_ = A.cin[i] + (r3 - g_ * per);
        sts128(STG + (uint32_t)st * (uint32_t)A.stage_bytes + (uint32_t)A.in_off[i] + (uint32_t)(cp + 1) * (uint32_t)A.copy_bytes[i] + (uint32_t)(g_ * A.S[i] + k_) * 16u,
               make_uint4(0u, 0u, 0u, 0u));
      }
    }
  }
  for (int i = tid; i < kMsMaxC; i += kMsThreads) { tab[4 * i] = A.bias[i]; tab[4 * i + 1] = A.has_slope ? A.sm1[i] : 0.f; tab[4 * i + 2] = A.proj[i]; tab[4 * i + 3] = 0.f; }
  asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
  __syncthreads();

  const int ra = (int)((long long)blockIdx.x * A.total_chunks / gridDim.x), rb = (int)((long long)(blockIdx.x + 1) * A.total_chunks / gridDim.x);

  if (warp == 0) {
    // ---- TMA producer ------------------------------------------------------------------------------------------
    if (lane == 0) {
      for (int idx = ra, k = 0; idx < rb; ++idx, ++k) {
        const int s = k % NS, n = idx / A.cpi, c = idx - n * A.cpi;
        if (k >= NS) mbar_wait_a(bar_empty + 8 * s, ((uint32_t)(k / NS) - 1u) & 1u);      // every consumer is done with the stage
        const uint32_t bar = bar_full + 8 * s, st = STG + (uint32_t)s * (uint32_t)A.stage_bytes;
        mbar_expect_tx_a(bar, (uint32_t)A.tx_bytes);
        const int y0 = A.rows * c - (A.k3 ? 1 : 0);                        // 3x3: one halo row above (and below: the box is 2 rows taller)
        tma_load_5d(st + (uint32_t)A.in_off[0], &tm0, bar, 0, 0, 0, y0, n);
        if (A.n_in > 1) tma_load_5d(st + (uint32_t)A.in_off[1], &tm1, bar, 0, 0, 0, y0, n);
        if (A.n_in > 2) tma_load_5d(st + (uint32_t)A.in_off[2], &tm2, bar, 0, 0, 0, y0, n);
        // resample-add sources: the low-resolution rows this chunk's bilinear taps reach (rows past the bottom: zero fill, never read)
        if (A.n_rs > 0) tma_load_4d_a(st + (uint32_t)A.r_off[0], &tr0, bar, 0, ms_row0(A.r_H[0], A.r_W[0], A.r_up[0], A.rows * c), A.r_c0[0], n);
        if (A.n_rs > 1) tma_load_4d_a(st + (uint32_t)A.r_off[1], &tr1, bar, 0, ms_row0(A.r_H[1], A.r_W[1], A.r_up[1], A.rows * c), A.r_c0[1], n);
      }
    }
  } else if (warp == 2 || warp == 3) {
    // ---- 3x3 form: builders of the shifted copies.  Copy 1 holds x-1 (pixel j of a group = pixel j-1 of the centre tile),
    //      copy 2 holds x+1; zeros enter at the image's left / right edge ---------------------------------------------------
    if (A.k3) {
      const int bt = (warp - 2) * 32 + lane, G = A.G, tg = (A.rows + 2) * G;
      for (int idx = ra, k = 0; idx < rb; ++idx, ++k) {
        const int s = k % NS;
        mbar_wait_a(bar_full + 8 * s, (uint32_t)(k / NS) & 1u);
        const uint32_t st = STG + (uint32_t)s * (uint32_t)A.stage_bytes;
        for (int i = 0; i < A.n_in; ++i) {
          const int S_ = A.S[i], cin = A.cin[i];
          const uint32_t c0 = st + (uint32_t)A.in_off[i], cb = (uint32_t)A.copy_bytes[i];
          for (int t = bt; t < tg * cin; t += 64) {
            const int pg = t / cin, ch = t - pg * cin, g = pg % G;
            const uint32_t a = c0 + (uint32_t)(pg * S_ + ch) * 16u;
            const uint4 cur = lds128(a);
            const uint32_t prev7 = g > 0 ? (uint32_t)lds16(a - (uint32_t)S_ * 16u + 14u) : 0u;
            const uint32_t next0 = g < G - 1 ? (uint32_t)lds16(a + (uint32_t)S_ * 16u) : 0u;
            sts128(a + cb, make_uint4((cur.x << 16) | prev7, __byte_perm(cur.x, cur.y, 0x5432), __byte_perm(cur.y, cur.z, 0x5432), __byte_perm(cur.z, cur.w, 0x5432)));
            sts128(a + 2 * cb, make_uint4(__byte_perm(cur.x, cur.y, 0x5432), __byte_perm(cur.y, cur.z, 0x5432), __byte_perm(cur.z, cur.w, 0x5432), (cur.w >> 16) | (next0 << 16)));
          }
        }
        asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");     // generic writes -> visible to the tensor core
        __syncwarp();
        if (lane == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(bar_built + 8 * s) : "memory");
      }
    }
  } else if (warp >= 4) {
    const int e = warp - 4, qd = e & 3, wg = e >> 2;
    const uint32_t ready = A.k3 ? bar_built : bar_full;
    // a projected op adds its resample paths before the PReLU like any other (the host launches PROJ_RS for those)
    if constexpr (PROJ_RS) {
      if (A.n_rs == 1) ms_consume_n<T, 1, true>(A, sbase, STG, TAB, bar_full, ready, bar_empty, ra, rb, wg, qd, lane);
      else ms_consume_n<T, 2, true>(A, sbase, STG, TAB, bar_full, ready, bar_empty, ra, rb, wg, qd, lane);
    } else if (A.has_proj) ms_consume_n<T, 0, true>(A, sbase, STG, TAB, bar_full, ready, bar_empty, ra, rb, wg, qd, lane);
    else if (A.n_rs == 0) ms_consume_n<T, 0, false>(A, sbase, STG, TAB, bar_full, ready, bar_empty, ra, rb, wg, qd, lane);
    else if (A.n_rs == 1) ms_consume_n<T, 1, false>(A, sbase, STG, TAB, bar_full, ready, bar_empty, ra, rb, wg, qd, lane);
    else ms_consume_n<T, 2, false>(A, sbase, STG, TAB, bar_full, ready, bar_empty, ra, rb, wg, qd, lane);
  }
}

}  // namespace csnet
