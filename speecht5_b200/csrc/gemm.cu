// Batched bf16 GEMM on the Hopper tensor cores (wgmma, fp32 accumulators in registers), operands staged by TMA into
// 128B-swizzled shared memory through an mbarrier ring. One CTA computes a 128 x BN output tile.
//
// Warp roles (512 threads): warpgroup 0 = TMA producer (one elected thread), warpgroups 1..2 = MMA: each issues the
// wgmma of 64 rows of the tile and hands the accumulators over through a swizzled fp32 tile in shared memory,
// warpgroup 3 = epilogue (one row x 32 columns per thread -> fused bias / activation / dropout / residual -> global).
// The handoff is a pair of mbarriers, so the MMA warpgroups start the next tile's main loop while the epilogue drains
// this one; on a CTA's last tile they have nothing left to multiply and join the epilogue (12 warps).
//
// This one kernel is the contraction engine for every dense op on the SpeechT5 path: the q/k/v/out projections
// (reference: speecht5/models/modules/multihead_attention.py:213-231,397), the FFN (transformer_layer.py:127-132,
// 385-391), pre-/post-net Linear layers, the post-net Conv1d stack expressed as an overlapping-window GEMM, and all
// of their backward contractions (MN-major operands avoid explicit transposes).
#include "gemm.cuh"
#include "ptx.cuh"
#include "kernels.cuh"
#include <cuda.h>
#include "tma_map.cuh"
#include <mutex>
#include <stdlib.h>
#include <string.h>
#include <unordered_map>

namespace st5 {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;  // 64 bf16 = 128 bytes = one swizzle row
constexpr int MMA_K = 16;
constexpr int MMA_WARPS = 8;  // two warpgroups, rows [0, 64) and [64, 128) of the tile
constexpr int EPI_WARPS = 4;  // one warpgroup: warp w takes row quarter w and every 32-column chunk
constexpr int GEMM_THREADS = 128 + 32 * (MMA_WARPS + EPI_WARPS);
// Registers per thread after setmaxnreg (producer / MMA / epilogue warpgroup): 40 + 2 * 160 + 152 = 4 * 128, the file
// of one 512-thread CTA.
constexpr int REGS_PRODUCER = 40, REGS_MMA = 160, REGS_EPI = 152;
static_assert(REGS_PRODUCER + 2 * REGS_MMA + REGS_EPI <= 65536 / 128, "register plan exceeds the register file");

struct EpiParams {
  int M, N, nb1;
  void* C; int c_fp32; long c_ld, c_bs1, c_bs2;
  void* C_pre;
  const float* bias;
  const float* bias2; int bias2_rows;
  const void* residual;
  int act; float alpha; int accumulate;
  uint32_t drop_thr; float drop_scale; uint64_t drop_seed, drop_offset;
  int num_k_blocks;
  int a_m1, a_m2, b_m1, b_m2;  // 0 when the operand is broadcast over that batch dim (stride 0), else 1
  int c_m1, c_m2;              // the same for the output (accumulate == 2: split-K batches share one output)
  const void* ag_pre; int ag_act;   // optional: multiply by act'(ag_pre[m][n]) (activation backward fused into dX)
  int tma_store;                    // 1: outputs leave through shared memory + TMA store (maps map_c / map_cpre)
  int tiles_m, tiles_n, num_tiles;  // persistent schedule: tile = (z * tiles_n + n_blk) * tiles_m + m_blk
};

// Activation / activation-derivative over one 32-column chunk with the kind fixed at compile time: the runtime switch
// sits outside the unrolled element loop (one uniform branch per chunk instead of three per element).
template <int ACT>
__device__ __forceinline__ void act_chunk(float (&v)[32]) {
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    if constexpr (ACT == ACT_RELU) v[j] = fmaxf(v[j], 0.f);
    if constexpr (ACT == ACT_GELU) v[j] = gelu_fwd(v[j]);
    if constexpr (ACT == ACT_TANH) v[j] = tanhf(v[j]);
    if constexpr (ACT == ACT_GELU_TANH) v[j] = gelu_tanh_fwd(v[j]);
  }
}
template <int ACT>
__device__ __forceinline__ void actgrad8(float* v, const uint4 u) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const float2 f = __bfloat1622float2(h[t]);
    if constexpr (ACT == ACT_GATE) {  // the forward epilogue stored keep * scale * act'(pre): one multiply per output
      v[2 * t] *= f.x;
      v[2 * t + 1] *= f.y;
    } else {
      v[2 * t] *= act_grad(f.x, ACT);
      v[2 * t + 1] *= act_grad(f.y, ACT);
    }
  }
}

template <int BN, bool A_MN, bool B_MN>
__device__ __forceinline__ void gemm_mainloop(float (&acc)[BN / 2], const uint8_t* smem_a, const uint8_t* smem_b,
                                              uint64_t* full_bar, uint64_t* empty_bar, int& stage, uint32_t& phase,
                                              int nkb, int wg, int STAGES) {
  constexpr uint32_t A_BYTES = BLOCK_M * BLOCK_K * 2;
  constexpr uint32_t B_BYTES = BN * BLOCK_K * 2;
  constexpr uint32_t CHUNK_BYTES = 64 * BLOCK_K * 2;  // one 64(mn) x 64(k) MN-major box
  const bool leader = (threadIdx.x & 127) == 0;
  int prev = -1;
  for (int kb = 0; kb < nkb; ++kb) {
    mbar_wait_quiet(&full_bar[stage], phase);
    const uint32_t sa = smem_u32(smem_a + stage * A_BYTES) + (uint32_t)wg * 8192u;  // this warpgroup's 64 rows
    const uint32_t sb = smem_u32(smem_b + stage * B_BYTES);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BLOCK_K / MMA_K; ++k) {
      // K-major: advance 16 elements (32 B) along the swizzled row. MN-major: advance 16 k-rows (2 KB).
      const uint64_t da = A_MN ? wgmma_smem_desc(sa + k * (MMA_K * 128), CHUNK_BYTES, 1024)
                               : wgmma_smem_desc(sa + k * (MMA_K * 2), 16, 1024);
      const uint64_t db = B_MN ? wgmma_smem_desc(sb + k * (MMA_K * 128), CHUNK_BYTES, 1024)
                               : wgmma_smem_desc(sb + k * (MMA_K * 2), 16, 1024);
      if constexpr (BN == 128) wgmma_m64n128<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, da, db, (kb | k) != 0 ? 1u : 0u);
      else wgmma_m64n64<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, da, db, (kb | k) != 0 ? 1u : 0u);
    }
    wgmma_commit();
    // keep one k-block of MMAs in flight: the slot of the previous one is free once it has retired
    wgmma_wait<1>();
    wgmma_fence_regs(acc);
    if (prev >= 0 && leader) mbar_arrive(&empty_bar[prev]);
    prev = stage;
    if (++stage == STAGES) { stage = 0; phase ^= 1; }
  }
  wgmma_wait<0>();
  wgmma_fence_regs(acc);
  if (leader) mbar_arrive(&empty_bar[prev]);
}

// fp32 accumulator tile in shared memory, chunk-major [BN / 32][BLOCK_M][32], the 16-byte column groups of row r XOR-ed
// by r % 8: the epilogue's row-per-lane float4 reads are conflict-free, and the 32 x 32 block of one row quarter and
// one 32-column chunk is 4 KB of contiguous, 1 KB-aligned memory. That block is the staging buffer of the warp that
// finishes it: the fp32 TMA store box (128B swizzle) has exactly this layout, a bf16 one (64B swizzle) fits in either
// 2 KB half, so two bf16 outputs of one chunk (C_pre and C, or the gate epilogue's pair) take one half each.
__device__ __forceinline__ int acc_idx(int row, int col) {
  return (col >> 5) * (BLOCK_M * 32) + row * 32 + (((((col >> 2) ^ row) & 7) << 2) | (col & 3));
}

// The fused epilogue of one output tile for one warp: rows [32 q, 32 q + 32) of the tile (one per lane), 32-column
// chunks c = grp, grp + ngrp, ... Every output block leaves by TMA from its own 32 x 32 block of `sacc`; the caller
// waits for those bulk stores to have read shared memory before the tile's accumulators may be overwritten.
template <int BN>
__device__ __forceinline__ void epilogue_tile(const EpiParams& p, float* sacc, const CUtensorMap& map_c,
                                              const CUtensorMap& map_cpre, int tile, int q, int grp, int ngrp,
                                              uint64_t dseed, uint64_t doffset) {
    const int tiles_mn = p.tiles_m * p.tiles_n;
    const int z = tile / tiles_mn, rmn = tile - z * tiles_mn;
    const int m0 = (rmn % p.tiles_m) * BLOCK_M, n0 = (rmn / p.tiles_m) * BN;
    const int b1 = z % p.nb1, b2 = z / p.nb1;
    const int row = m0 + q * 32 + (int)lane_id();
    const bool row_ok = row < p.M;
    const long zoff = (long)b1 * p.c_bs1 + (long)b2 * p.c_bs2;
    const long roff = zoff + (long)row * p.c_ld;
    const float* bias2_row = (p.bias2 != nullptr && row_ok) ? p.bias2 + (long)(row / p.bias2_rows) * p.N : nullptr;
    const uint64_t drop_row = ((uint64_t)z * (uint64_t)p.M + (uint64_t)row) * (uint64_t)p.N;
#pragma unroll 1
    for (int c = grp; c < BN / 32; c += ngrp) {
      const int nb = n0 + c * 32;
      if (nb >= p.N) continue;  // warp-uniform; rows beyond M keep going (their loads are guarded, stores clipped)
      uint8_t* const blk = reinterpret_cast<uint8_t*>(sacc + acc_idx(q * 32, c * 32));  // this warp's 32 x 32 block
      bool staged = false;  // a bulk store of this chunk is reading the block
      float v[32];
      {
        const int tr = q * 32 + (int)lane_id();
#pragma unroll
        for (int j = 0; j < 32; j += 4) {
          const float4 a4 = *reinterpret_cast<const float4*>(sacc + acc_idx(tr, c * 32 + j));
          v[j] = a4.x; v[j + 1] = a4.y; v[j + 2] = a4.z; v[j + 3] = a4.w;
        }
      }
      if (p.alpha != 1.f) {
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] *= p.alpha;
      }
      const bool full = (nb + 32 <= p.N);
      if (p.accumulate == 1 && row_ok) {  // partial sums of a multi-pass (split-precision) product live in C (fp32)
        const float* src = reinterpret_cast<const float*>(p.C) + roff + nb;
        if (full && ((p.c_ld & 3) == 0) && ((zoff & 3) == 0) && ((reinterpret_cast<uintptr_t>(p.C) & 15) == 0)) {
#pragma unroll
          for (int j = 0; j < 32; j += 4) {
            const float4 o = *reinterpret_cast<const float4*>(src + j);
            v[j] += o.x; v[j + 1] += o.y; v[j + 2] += o.z; v[j + 3] += o.w;
          }
        } else {
#pragma unroll
          for (int j = 0; j < 32; ++j)
            if (full || nb + j < p.N) v[j] += src[j];
        }
      }
      if (p.bias != nullptr) {
        if (full && ((reinterpret_cast<uintptr_t>(p.bias + nb) & 15) == 0)) {
          // every lane needs the same 32 values: eight 16-byte loads of one address per warp (L1 broadcast)
          const float4* bp = reinterpret_cast<const float4*>(p.bias + nb);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float4 b4 = __ldg(bp + j);
            v[4 * j] += b4.x; v[4 * j + 1] += b4.y; v[4 * j + 2] += b4.z; v[4 * j + 3] += b4.w;
          }
        } else {  // ragged edge: one coalesced load per warp, then register shuffles
          const int jn = nb + (int)lane_id();
          const float bl = jn < p.N ? __ldg(p.bias + jn) : 0.f;
#pragma unroll
          for (int j = 0; j < 32; ++j) v[j] += __shfl_sync(0xffffffffu, bl, j);
        }
      }
      if (bias2_row != nullptr) {
#pragma unroll
        for (int j = 0; j < 32; ++j)
          if (full || nb + j < p.N) v[j] += __ldg(bias2_row + nb + j);
      }
      const bool vec_ok = full && ((p.c_ld & 7) == 0) && ((zoff & 7) == 0) &&
                          ((reinterpret_cast<uintptr_t>(p.C) & 15) == 0) &&
                          ((reinterpret_cast<uintptr_t>(p.C_pre) & 15) == 0);
      // ---- output path: stage the 32x32 block in shared memory and let TMA write it (coalesced, asynchronous,
      // clipped at the tensor edges); fall back to per-thread stores when the output layout is not TMA-addressable.
      auto emit = [&](void* base, const CUtensorMap* tmap) {
        if (p.tma_store) {
          // The second output of a chunk (C after C_pre): bf16 takes the free second half of the block, fp32 waits
          // until the C_pre store has read the block.
          uint8_t* const stg = staged && !p.c_fp32 ? blk + 2048 : blk;
          if (staged && p.c_fp32 && lane_id() == 0) bulk_wait_read0();
          __syncwarp();  // (also: every lane has read its accumulators out of the block)
          staged = true;
          const int rr = (int)lane_id();
          if (p.c_fp32) {
#pragma unroll
            for (int g = 0; g < 8; ++g)
              *reinterpret_cast<float4*>(stg + rr * 128 + ((g ^ (rr & 7)) << 4)) =
                  make_float4(v[4 * g], v[4 * g + 1], v[4 * g + 2], v[4 * g + 3]);
          } else {
#pragma unroll
            for (int g = 0; g < 4; ++g) {
              uint4 pk;
              __nv_bfloat162 t0 = __floats2bfloat162_rn(v[8 * g], v[8 * g + 1]);
              __nv_bfloat162 t1 = __floats2bfloat162_rn(v[8 * g + 2], v[8 * g + 3]);
              __nv_bfloat162 t2 = __floats2bfloat162_rn(v[8 * g + 4], v[8 * g + 5]);
              __nv_bfloat162 t3 = __floats2bfloat162_rn(v[8 * g + 6], v[8 * g + 7]);
              pk.x = *reinterpret_cast<uint32_t*>(&t0); pk.y = *reinterpret_cast<uint32_t*>(&t1);
              pk.z = *reinterpret_cast<uint32_t*>(&t2); pk.w = *reinterpret_cast<uint32_t*>(&t3);
              *reinterpret_cast<uint4*>(stg + rr * 64 + ((g ^ ((rr >> 1) & 3)) << 4)) = pk;
            }
          }
          fence_proxy_async();
          __syncwarp();
          if (lane_id() == 0) {
            if (p.accumulate == 2) tma_reduce_add_4d(tmap, stg, nb, m0 + q * 32, b1 * p.c_m1, b2 * p.c_m2);  // C += tile, at the L2
            else tma_store_4d(tmap, stg, nb, m0 + q * 32, b1 * p.c_m1, b2 * p.c_m2);
            bulk_commit();
          }
          return;
        }
        if (!row_ok) return;
        if (p.c_fp32) {
          float* dst = reinterpret_cast<float*>(base) + roff + nb;
          if (full && ((p.c_ld & 3) == 0) && ((zoff & 3) == 0) && ((reinterpret_cast<uintptr_t>(base) & 15) == 0)) {
#pragma unroll
            for (int j = 0; j < 32; j += 4)
              *reinterpret_cast<float4*>(dst + j) = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
          } else {
#pragma unroll
            for (int j = 0; j < 32; ++j)
              if (full || nb + j < p.N) dst[j] = v[j];
          }
        } else {
          __nv_bfloat16* dst = reinterpret_cast<__nv_bfloat16*>(base) + roff + nb;
          if (vec_ok) {
#pragma unroll
            for (int j = 0; j < 32; j += 8) {
              uint4 pk;
              __nv_bfloat162 t0 = __floats2bfloat162_rn(v[j], v[j + 1]);
              __nv_bfloat162 t1 = __floats2bfloat162_rn(v[j + 2], v[j + 3]);
              __nv_bfloat162 t2 = __floats2bfloat162_rn(v[j + 4], v[j + 5]);
              __nv_bfloat162 t3 = __floats2bfloat162_rn(v[j + 6], v[j + 7]);
              pk.x = *reinterpret_cast<uint32_t*>(&t0); pk.y = *reinterpret_cast<uint32_t*>(&t1);
              pk.z = *reinterpret_cast<uint32_t*>(&t2); pk.w = *reinterpret_cast<uint32_t*>(&t3);
              *reinterpret_cast<uint4*>(dst + j) = pk;
            }
          } else {
#pragma unroll
            for (int j = 0; j < 32; ++j)
              if (full || nb + j < p.N) dst[j] = __float2bfloat16(v[j]);
          }
        }
      };
      if (p.act == ACT_GELU_TANH_GATE) {
        // fc1 of the FFN in throughput mode: out = drop(gelu_tanh(x)), and INSTEAD of the pre-activation the second
        // output is the multiplier the backward pass needs, gate = keep * scale * gelu_tanh'(x) (tanh(u) is shared by
        // both). The dH = dO.W2 GEMM of the backward then multiplies by it -- no Philox, no tanh in that epilogue.
        // Eight columns at a time straight into the two halves of this warp's staging block (bf16: 2 KB each), so
        // the chunk is never held twice in registers. Launcher guarantees: bf16 output, TMA-store layout, N % 8 == 0.
        __syncwarp();  // every lane has read its accumulators out of the block
        const int rr = (int)lane_id();
        const uint64_t e0 = drop_row + (uint64_t)nb;
#pragma unroll
        for (int g = 0; g < 4; ++g) {
          float o[8], d[8];
#pragma unroll
          for (int t = 0; t < 8; ++t) {
            const float x = v[8 * g + t];
            const float x2 = x * x;
            const float th = fast_tanh(x * fmaf(0.0356774081f, x2, 0.7978845608f));
            const float hx = 0.5f * x;
            o[t] = fmaf(hx, th, hx);
            d[t] = fmaf(hx * fmaf(-th, th, 1.f), fmaf(0.1070322243f, x2, 0.7978845608f), fmaf(0.5f, th, 0.5f));
          }
          if (p.drop_thr != 0) {
            const Philox4 r4 = philox4x32(dseed, doffset, (e0 + 8 * g) >> 3);
            const uint32_t w[4] = {r4.x, r4.y, r4.z, r4.w};
#pragma unroll
            for (int t = 0; t < 4; ++t) {
              const float k0 = (w[t] & 0xFFFFu) >= p.drop_thr ? p.drop_scale : 0.f;
              const float k1 = (w[t] >> 16) >= p.drop_thr ? p.drop_scale : 0.f;
              o[2 * t] *= k0; d[2 * t] *= k0;
              o[2 * t + 1] *= k1; d[2 * t + 1] *= k1;
            }
          }
          uint4 po, pd;
          {
            __nv_bfloat162 t0 = __floats2bfloat162_rn(o[0], o[1]), t1 = __floats2bfloat162_rn(o[2], o[3]);
            __nv_bfloat162 t2 = __floats2bfloat162_rn(o[4], o[5]), t3 = __floats2bfloat162_rn(o[6], o[7]);
            po.x = *reinterpret_cast<uint32_t*>(&t0); po.y = *reinterpret_cast<uint32_t*>(&t1);
            po.z = *reinterpret_cast<uint32_t*>(&t2); po.w = *reinterpret_cast<uint32_t*>(&t3);
            __nv_bfloat162 u0 = __floats2bfloat162_rn(d[0], d[1]), u1 = __floats2bfloat162_rn(d[2], d[3]);
            __nv_bfloat162 u2 = __floats2bfloat162_rn(d[4], d[5]), u3 = __floats2bfloat162_rn(d[6], d[7]);
            pd.x = *reinterpret_cast<uint32_t*>(&u0); pd.y = *reinterpret_cast<uint32_t*>(&u1);
            pd.z = *reinterpret_cast<uint32_t*>(&u2); pd.w = *reinterpret_cast<uint32_t*>(&u3);
          }
          const int so = rr * 64 + ((g ^ ((rr >> 1) & 3)) << 4);
          *reinterpret_cast<uint4*>(blk + so) = po;
          *reinterpret_cast<uint4*>(blk + 2048 + so) = pd;
        }
        fence_proxy_async();
        __syncwarp();
        if (lane_id() == 0) {
          tma_store_4d(&map_c, blk, nb, m0 + q * 32, b1, b2);
          tma_store_4d(&map_cpre, blk + 2048, nb, m0 + q * 32, b1, b2);
          bulk_commit();
        }
        continue;
      }
      if (p.C_pre != nullptr) emit(p.C_pre, &map_cpre);
      if (p.act == ACT_GELU_TANH) act_chunk<ACT_GELU_TANH>(v);
      else if (p.act == ACT_GELU) act_chunk<ACT_GELU>(v);
      else if (p.act == ACT_RELU) act_chunk<ACT_RELU>(v);
      else if (p.act == ACT_TANH) act_chunk<ACT_TANH>(v);
      if (p.drop_thr != 0) {
        const uint64_t e0 = drop_row + (uint64_t)nb;
        if ((e0 & 7) == 0) {  // aligned: one Philox call per 8 elements
#pragma unroll
          for (int j = 0; j < 32; j += 8) dropout8_apply(v + j, e0 + j, p.drop_thr, p.drop_scale, dseed, doffset);
        } else {  // odd row pitch: assemble the 32 keep bits from at most five calls
          const uint32_t keep = dropout_keep_mask32(dseed, doffset, e0, p.drop_thr);
#pragma unroll
          for (int j = 0; j < 32; ++j) v[j] = ((keep >> j) & 1u) ? v[j] * p.drop_scale : 0.f;
        }
      }
      if (p.ag_pre != nullptr && row_ok) {
        if (p.c_fp32) {
          const float* pr = reinterpret_cast<const float*>(p.ag_pre) + roff + nb;
#pragma unroll
          for (int j = 0; j < 32; ++j)
            if (full || nb + j < p.N) v[j] *= p.ag_act == ACT_GATE ? pr[j] : act_grad(pr[j], p.ag_act);
        } else {
          const __nv_bfloat16* pr = reinterpret_cast<const __nv_bfloat16*>(p.ag_pre) + roff + nb;
          if (vec_ok && ((reinterpret_cast<uintptr_t>(p.ag_pre) & 15) == 0)) {
#pragma unroll
            for (int j = 0; j < 32; j += 8) {
              const uint4 u = *reinterpret_cast<const uint4*>(pr + j);
              if (p.ag_act == ACT_GATE) actgrad8<ACT_GATE>(v + j, u);
              else if (p.ag_act == ACT_GELU_TANH) actgrad8<ACT_GELU_TANH>(v + j, u);
              else if (p.ag_act == ACT_GELU) actgrad8<ACT_GELU>(v + j, u);
              else if (p.ag_act == ACT_RELU) actgrad8<ACT_RELU>(v + j, u);
              else actgrad8<ACT_TANH>(v + j, u);
            }
          } else {
#pragma unroll
            for (int j = 0; j < 32; ++j)
              if (full || nb + j < p.N)
                v[j] *= p.ag_act == ACT_GATE ? __bfloat162float(pr[j]) : act_grad(__bfloat162float(pr[j]), p.ag_act);
          }
        }
      }
      if (p.residual != nullptr && row_ok) {
        if (p.c_fp32) {
          const float* rs = reinterpret_cast<const float*>(p.residual) + roff + nb;
#pragma unroll
          for (int j = 0; j < 32; ++j)
            if (full || nb + j < p.N) v[j] += rs[j];
        } else {
          const __nv_bfloat16* rs = reinterpret_cast<const __nv_bfloat16*>(p.residual) + roff + nb;
          if (vec_ok && ((reinterpret_cast<uintptr_t>(p.residual) & 15) == 0)) {
#pragma unroll
            for (int j = 0; j < 32; j += 8) {
              const uint4 u = *reinterpret_cast<const uint4*>(rs + j);
              const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
              for (int t = 0; t < 4; ++t) {
                const float2 f = __bfloat1622float2(h[t]);
                v[j + 2 * t] += f.x;
                v[j + 2 * t + 1] += f.y;
              }
            }
          } else {
#pragma unroll
            for (int j = 0; j < 32; ++j)
              if (full || nb + j < p.N) v[j] += __bfloat162float(rs[j]);
          }
        }
      }
      emit(p.C, &map_c);
    }
}

template <int BN, int STAGES, bool A_MN, bool B_MN>
__global__ void __launch_bounds__(GEMM_THREADS, 1) gemm_bf16_wgmma(const __grid_constant__ CUtensorMap map_a,
                                                                const __grid_constant__ CUtensorMap map_b,
                                                                const __grid_constant__ CUtensorMap map_c,
                                                                const __grid_constant__ CUtensorMap map_cpre,
                                                                const __grid_constant__ EpiParams p) {
  constexpr uint32_t A_BYTES = BLOCK_M * BLOCK_K * 2;
  constexpr uint32_t B_BYTES = BN * BLOCK_K * 2;
  constexpr uint32_t CHUNK_BYTES = 64 * BLOCK_K * 2;  // one 64(mn) x 64(k) MN-major box
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + STAGES * A_BYTES;
  float* sacc = reinterpret_cast<float*>(smem_b + STAGES * B_BYTES);  // BLOCK_M x BN fp32 accumulators
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(sacc + BLOCK_M * BN);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* sacc_full = empty_bar + STAGES;  // a tile's accumulators are in sacc (one arrive per MMA warp)
  uint64_t* sacc_empty = sacc_full + 1;      // the epilogue is done with them (one arrive per epilogue warp)

  // Persistent CTA: loops over output tiles (m fastest, so concurrently running CTAs share the B/weight tile in L2);
  // the producer runs ahead into the next tile, and the MMA warps start it while the epilogue drains this one. Every
  // role walks the same tile sequence; the i-th tile of a CTA is the i-th phase of sacc_full and sacc_empty.
  const int warp = threadIdx.x >> 5;
  const int nkb = p.num_k_blocks;
  const int tiles_mn = p.tiles_m * p.tiles_n;

  if (warp == 0 && elect_one()) {
    tma_prefetch_desc(&map_a);
    tma_prefetch_desc(&map_b);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);  // one arrive per MMA warpgroup
    }
    mbar_init(sacc_full, MMA_WARPS);
    mbar_init(sacc_empty, EPI_WARPS);
    fence_mbar_init();
  }
  __syncthreads();
  // Programmatic dependent launch: everything above touched only this CTA's shared memory, so it may run while the
  // preceding grid drains. Wait for that grid's memory here, before the first global access, and let the grid behind
  // us start its own prologue (both are no-ops when the launch carries no programmatic attribute).
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

  if (warp < 4) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<REGS_PRODUCER>();
    if (warp == 0 && elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
      const int z = tile / tiles_mn, rmn = tile - z * tiles_mn;
      const int m0 = (rmn % p.tiles_m) * BLOCK_M, n0 = (rmn / p.tiles_m) * BN;
      const int b1 = z % p.nb1, b2 = z / p.nb1;
      for (int kb = 0; kb < nkb; ++kb) {
        mbar_wait_quiet(&empty_bar[stage], phase ^ 1);
        uint8_t* sa = smem_a + stage * A_BYTES;
        uint8_t* sb = smem_b + stage * B_BYTES;
        const int k0 = kb * BLOCK_K;
        mbar_expect_tx(&full_bar[stage], A_BYTES + B_BYTES);
        if (A_MN) {
#pragma unroll
          for (int c = 0; c < BLOCK_M / 64; ++c)
            tma_load_4d(sa + c * CHUNK_BYTES, &map_a, &full_bar[stage], m0 + c * 64, k0, b1 * p.a_m1, b2 * p.a_m2);
        } else {
          tma_load_4d(sa, &map_a, &full_bar[stage], k0, m0, b1 * p.a_m1, b2 * p.a_m2);
        }
        if (B_MN) {
#pragma unroll
          for (int c = 0; c < BN / 64; ++c)
            tma_load_4d(sb + c * CHUNK_BYTES, &map_b, &full_bar[stage], n0 + c * 64, k0, b1 * p.b_m1, b2 * p.b_m2);
        } else {
          tma_load_4d(sb, &map_b, &full_bar[stage], k0, n0, b1 * p.b_m1, b2 * p.b_m2);
        }
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      }
    }
  } else if (warp < 4 + MMA_WARPS) {
    // ===================== MMA: wgmma main loop, accumulators -> sacc =====================
    setmaxnreg_inc<REGS_MMA>();
    const int mw = warp - 4;  // MMA warp 0..7
    const int wg = mw >> 2;   // MMA warpgroup: rows [64 wg, 64 wg + 64) of the tile
    const int ntiles = (p.num_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;  // >= 1: grid <= tiles
    int stage = 0;
    uint32_t phase = 0;
    for (int it = 0; it < ntiles; ++it) {
      float acc[BN / 2];
      gemm_mainloop<BN, A_MN, B_MN>(acc, smem_a, smem_b, full_bar, empty_bar, stage, phase, nkb, wg, STAGES);
      mbar_wait_quiet(sacc_empty, (it & 1) ^ 1);  // the epilogue of the previous tile is done with sacc
      // acc[i], acc[i + 1] -> acc_idx(row, col), row = 16 w + l / 4 + 8 ((i >> 1) & 1), col = 8 (i >> 2) + 2 (l % 4),
      // spelled as one lane base plus compile-time offsets (the 16-byte group (col / 4) % 8 = (2 (i >> 2)) % 8 ^ (l / 2)
      // % 2, XOR-ed by row % 8 = (l / 4) % 8): few live registers across the main loop.
      const int l = (int)lane_id();
      const int sw = ((l >> 1) & 1) ^ ((l >> 2) & 7);
      float* const abase = sacc + (wg * 64 + (mw & 3) * 16 + (l >> 2)) * 32 + 2 * (l & 1);
#pragma unroll
      for (int i = 0; i < BN / 2; i += 2)
        *reinterpret_cast<float2*>(abase + (i >> 4) * (BLOCK_M * 32) + 256 * ((i >> 1) & 1) +
                                   ((((2 * (i >> 2)) & 7) ^ sw) << 2)) = make_float2(acc[i], acc[i + 1]);
      __syncwarp();
      if (l == 0) mbar_arrive(sacc_full);
    }
    // The CTA's last tile: nothing left to multiply, so these 8 warps join the epilogue warpgroup -- 12 warps, 4 row
    // quarters x 3 column groups (a CTA with a single tile, e.g. a split-K weight gradient, would otherwise drain it on
    // 4 warps). Outside the tile loop, so that the epilogue's registers do not compete with the main loop's.
    uint64_t dseed = p.drop_seed, doffset = p.drop_offset;
    if (p.drop_thr != 0) resolve_seed(dseed, doffset);
    mbar_wait_quiet(sacc_full, (ntiles - 1) & 1);
    epilogue_tile<BN>(p, sacc, map_c, map_cpre, (int)blockIdx.x + (ntiles - 1) * (int)gridDim.x, mw & 3, mw >> 2, 3,
                      dseed, doffset);
    if (lane_id() == 0) bulk_wait_read0();  // sacc must outlive the last bulk store
  } else {
    // ===================== epilogue: sacc -> fused epilogue -> global =====================
    setmaxnreg_inc<REGS_EPI>();
    const int ew = warp - 4 - MMA_WARPS;  // row quarter of this warp
    uint64_t dseed = p.drop_seed, doffset = p.drop_offset;
    if (p.drop_thr != 0) resolve_seed(dseed, doffset);
    for (int tile = blockIdx.x, it = 0; tile < p.num_tiles; tile += gridDim.x, ++it) {
      mbar_wait_quiet(sacc_full, it & 1);
      const bool last = tile + (int)gridDim.x >= p.num_tiles;  // then the MMA warps take column groups 0 and 1
      epilogue_tile<BN>(p, sacc, map_c, map_cpre, tile, ew, last ? 2 : 0, last ? 3 : 1, dseed, doffset);
      if (lane_id() == 0) bulk_wait_read0();  // this warp's bulk stores have read their staging out of sacc
      __syncwarp();
      if (!last && lane_id() == 0) mbar_arrive(sacc_empty);
    }
  }
}

// ---------------------------------------------------------------------------------------------- host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// cuTensorMapEncodeTiled is a driver-API call and needs a current context on the calling thread. The runtime binds its
// primary context to a thread only at that thread's first runtime call, so on a thread whose first CUDA work is a GEMM
// (autograd's device thread when a backward pass starts with a projection) the encode failed with
// CUDA_ERROR_INVALID_CONTEXT. cudaSetDevice binds the primary context of the thread's current device (no synchronisation).
static EncodeTiledFn get_encode_fn() {
  static thread_local bool bound = false;
  if (!bound) {
    int dev = 0;
    if (cudaGetDevice(&dev) == cudaSuccess) cudaSetDevice(dev);
    bound = true;
  }
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(ptr);
  });
  return fn;
}

static int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
  }
  return n;
}

int device_sm_count() { return num_sms(); }

int encode_map_4d(CUtensorMap* map, const void* ptr, int is_f32, const uint64_t dims[4],
                  const uint64_t strides_bytes[3], const uint32_t box[4], int swizzle_bytes) {
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) return -10;
  cuuint64_t d[4] = {dims[0], dims[1], dims[2], dims[3]};
  cuuint64_t s[3] = {strides_bytes[0], strides_bytes[1], strides_bytes[2]};
  cuuint32_t bx[4] = {box[0], box[1], box[2], box[3]};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) || (s[0] & 15) || (s[1] & 15) || (s[2] & 15)) return -11;
  const CUtensorMapSwizzle sw = swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                                : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                : swizzle_bytes == 32 ? CU_TENSOR_MAP_SWIZZLE_32B : CU_TENSOR_MAP_SWIZZLE_NONE;
  CUresult r = enc(map, is_f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4,
                   const_cast<void*>(ptr), d, s, bx, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : -12;
}

int encode_bf16_map_4d(CUtensorMap* map, const void* ptr, const uint64_t dims[4], const uint64_t strides_bytes[3],
                       const uint32_t box[4]) {
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) return -10;
  cuuint64_t d[4] = {dims[0], dims[1], dims[2], dims[3]};
  cuuint64_t s[3] = {strides_bytes[0], strides_bytes[1], strides_bytes[2]};
  cuuint32_t bx[4] = {box[0], box[1], box[2], box[3]};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) || (s[0] & 15) || (s[1] & 15) || (s[2] & 15)) return -11;
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(ptr), d, s, bx, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : -12;
}

// rows x K operand. K-major: memory [rows][ld] (k contiguous). MN-major: memory [K][ld] (row index contiguous).
static int make_operand_map(CUtensorMap* map, const void* ptr, int mn_major, int rows, int K, long ld, int nb1,
                            long bs1, int nb2, long bs2, int box_rows) {
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) return -10;
  cuuint64_t dims[4];
  cuuint64_t strides[3];
  cuuint32_t box[4];
  cuuint32_t estr[4] = {1, 1, 1, 1};
  if (mn_major) {
    dims[0] = (cuuint64_t)rows; dims[1] = (cuuint64_t)K;
    box[0] = 64; box[1] = BLOCK_K;
  } else {
    dims[0] = (cuuint64_t)K; dims[1] = (cuuint64_t)rows;
    box[0] = BLOCK_K; box[1] = (cuuint32_t)box_rows;
  }
  if (nb1 > 1 && bs1 == 0) nb1 = 1;  // broadcast operand: the kernel pins that coordinate to 0
  if (nb2 > 1 && bs2 == 0) nb2 = 1;
  dims[2] = (cuuint64_t)nb1; dims[3] = (cuuint64_t)nb2;
  box[2] = 1; box[3] = 1;
  strides[0] = (cuuint64_t)ld * 2;
  strides[1] = (cuuint64_t)(nb1 > 1 ? bs1 : ld) * 2;
  strides[2] = (cuuint64_t)(nb2 > 1 ? bs2 : ld) * 2;
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) || (strides[0] & 15) || (strides[1] & 15) || (strides[2] & 15))
    return -11;  // TMA needs 16-byte aligned base and strides
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(ptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : -12;
}

template <int BN, int STAGES, bool A_MN, bool B_MN>
static int launch_variant(const GemmDesc& g, const EpiParams& ep, cudaStream_t stream) {
  CUtensorMap ma, mb;
  int rc = make_operand_map(&ma, g.A, g.a_mn, g.M, g.K, g.a_ld, g.nb1, g.a_bs1, g.nb2, g.a_bs2, BLOCK_M);
  if (rc) return rc;
  rc = make_operand_map(&mb, g.B, g.b_mn, g.N, g.K, g.b_ld, g.nb1, g.b_bs1, g.nb2, g.b_bs2, BN);
  if (rc) return rc - 10;
  constexpr size_t smem = (size_t)STAGES * (BLOCK_M * BLOCK_K * 2 + BN * BLOCK_K * 2) + BLOCK_M * BN * 4 +
                          (2 * STAGES + 2) * 8 + 1024;
  static_assert(smem <= 227 * 1024, "GEMM tile does not fit the 227 KB of shared memory of a block");
  auto kern = gemm_bf16_wgmma<BN, STAGES, A_MN, B_MN>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    attr_set = true;
  }
  EpiParams e2 = ep;
  e2.tiles_m = (g.M + BLOCK_M - 1) / BLOCK_M;
  e2.tiles_n = (g.N + BN - 1) / BN;
  const long total = (long)e2.tiles_m * e2.tiles_n * g.nb1 * g.nb2;
  if (total > 0x7fffffffL) return -4;
  e2.num_tiles = (int)total;
  // Output maps for the TMA-store epilogue: 32x32 element boxes, 64B (bf16) / 128B (fp32) swizzle. Needs 16-byte
  // aligned bases and row / batch pitches, and a row length of whole 16-byte units: the bulk store clips a box at the
  // edge of the tensor in 16-byte units, so with a ragged N it also writes the columns [N, c_ld) up to the next 16-byte
  // boundary (zeros, over whatever the caller keeps there). Otherwise the epilogue falls back to per-thread stores.
  CUtensorMap mc, mcp;
  memset(&mc, 0, sizeof(mc));
  memset(&mcp, 0, sizeof(mcp));
  e2.tma_store = 0;
  {
    const long es = g.c_fp32 ? 4 : 2;
    const bool ok = (((long)g.N * es) % 16 == 0) && ((g.c_ld * es) % 16 == 0) &&
                    (g.nb1 <= 1 || (g.c_bs1 * es) % 16 == 0) &&
                    (g.nb2 <= 1 || (g.c_bs2 * es) % 16 == 0) && (reinterpret_cast<uintptr_t>(g.C) % 16 == 0) &&
                    (g.C_pre == nullptr || reinterpret_cast<uintptr_t>(g.C_pre) % 16 == 0);
    if (ok) {
      const int cn1 = (g.nb1 > 1 && g.c_bs1 != 0) ? g.nb1 : 1, cn2 = (g.nb2 > 1 && g.c_bs2 != 0) ? g.nb2 : 1;
      const uint64_t dims[4] = {(uint64_t)g.N, (uint64_t)g.M, (uint64_t)cn1, (uint64_t)cn2};
      const uint64_t strides[3] = {(uint64_t)(g.c_ld * es), (uint64_t)((cn1 > 1 ? g.c_bs1 : g.c_ld) * es),
                                   (uint64_t)((cn2 > 1 ? g.c_bs2 : g.c_ld) * es)};
      const uint32_t box[4] = {32, 32, 1, 1};
      int r2 = encode_map_4d(&mc, g.C, g.c_fp32, dims, strides, box, g.c_fp32 ? 128 : 64);
      if (!r2 && g.C_pre != nullptr) r2 = encode_map_4d(&mcp, g.C_pre, g.c_fp32, dims, strides, box, g.c_fp32 ? 128 : 64);
      e2.tma_store = r2 == 0 ? 1 : 0;
    }
  }
  if (g.accumulate == 2 && !e2.tma_store) return -6;  // the L2-side accumulate is a TMA reduce: needs that output layout
  if (e2.act == ACT_GELU_TANH_GATE &&
      (!e2.tma_store || g.c_fp32 || g.C_pre == nullptr || (g.N & 7) != 0 || g.residual != nullptr || g.ag_pre != nullptr))
    return -5;  // the gate epilogue needs the TMA-store layout, bf16 outputs and an 8-aligned row length
  const long slots = num_sms();
  const int grid = (int)(total < slots ? total : slots);  // one persistent CTA per SM
  static const bool pdl = [] {
    const char* e = getenv("ST5_PDL");
    return e == nullptr || atoi(e) != 0;
  }();
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(GEMM_THREADS);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  int na = 0;
  if (pdl) {
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  cfg.attrs = attr;
  cfg.numAttrs = na;
  cudaError_t le = cudaLaunchKernelEx(&cfg, kern, ma, mb, mc, mcp, e2);
  if (le != cudaSuccess) return (int)le;
  return (int)cudaGetLastError();
}

template <int BN, int STAGES>
static int launch_major(const GemmDesc& g, const EpiParams& ep, cudaStream_t stream) {
  if (g.a_mn) {
    if (g.b_mn) return launch_variant<BN, STAGES, true, true>(g, ep, stream);
    return launch_variant<BN, STAGES, true, false>(g, ep, stream);
  }
  if (g.b_mn) return launch_variant<BN, STAGES, false, true>(g, ep, stream);
  return launch_variant<BN, STAGES, false, false>(g, ep, stream);
}

int gemm_launch(const GemmDesc& g, cudaStream_t stream) {
  if (g.M <= 0 || g.N <= 0 || g.nb1 <= 0 || g.nb2 <= 0) return 0;
  if (g.K <= 0) return -2;
  if (g.accumulate && !g.c_fp32) return -3;
  // a batch dimension with output stride 0 (split-K: several partial products into ONE output) is only sound with the
  // L2-side accumulate
  if (g.accumulate != 2 && ((g.nb1 > 1 && g.c_bs1 == 0) || (g.nb2 > 1 && g.c_bs2 == 0))) return -7;
  EpiParams ep;
  ep.M = g.M; ep.N = g.N; ep.nb1 = g.nb1;
  ep.C = g.C; ep.c_fp32 = g.c_fp32; ep.c_ld = g.c_ld; ep.c_bs1 = g.c_bs1; ep.c_bs2 = g.c_bs2;
  ep.C_pre = g.C_pre; ep.bias = g.bias; ep.bias2 = g.bias2; ep.bias2_rows = g.bias2_rows > 0 ? g.bias2_rows : 1;
  ep.ag_pre = g.ag_pre; ep.ag_act = g.ag_act;
  ep.residual = g.residual; ep.act = g.act; ep.alpha = g.alpha; ep.accumulate = g.accumulate;
  ep.drop_thr = drop_threshold(g.drop_p);
  ep.drop_scale = g.drop_p > 0.f ? 1.f / (1.f - g.drop_p) : 1.f;
  ep.drop_seed = g.drop_seed; ep.drop_offset = g.drop_offset;
  ep.num_k_blocks = (g.K + BLOCK_K - 1) / BLOCK_K;
  ep.a_m1 = (g.nb1 > 1 && g.a_bs1 == 0) ? 0 : 1; ep.a_m2 = (g.nb2 > 1 && g.a_bs2 == 0) ? 0 : 1;
  ep.b_m1 = (g.nb1 > 1 && g.b_bs1 == 0) ? 0 : 1; ep.b_m2 = (g.nb2 > 1 && g.b_bs2 == 0) ? 0 : 1;
  ep.c_m1 = (g.nb1 > 1 && g.c_bs1 == 0) ? 0 : 1; ep.c_m2 = (g.nb2 > 1 && g.c_bs2 == 0) ? 0 : 1;
  // Tile width: minimise (rounds of the persistent grid) x (time per tile); a 128 x 64 tile moves more operand bytes
  // per FLOP than a 128 x 128 one, hence its > 1 factor.
  const long tiles_m = (g.M + BLOCK_M - 1) / BLOCK_M;
  const long batch = (long)g.nb1 * g.nb2;
  const long sms = num_sms();
  auto cost = [&](int bn, double factor) {
    const long tiles = tiles_m * ((g.N + bn - 1) / bn) * batch;
    const long rounds = (tiles + sms - 1) / sms;
    return (double)rounds * (bn * factor + 24.0);
  };
  static const int force_bn = [] {  // tuning / profiling knob: ST5_GEMM_BN=64|128 pins the tile width
    const char* e = getenv("ST5_GEMM_BN");
    return e ? atoi(e) : 0;
  }();
  if (force_bn == 128) return launch_major<128, 4>(g, ep, stream);
  if (force_bn == 64) return launch_major<64, 6>(g, ep, stream);
  const double c128 = g.N > 64 ? cost(128, 1.0) : 1e30;
  const double c64 = cost(64, 1.25);
  if (c128 <= c64) return launch_major<128, 4>(g, ep, stream);
  return launch_major<64, 6>(g, ep, stream);
}

}  // namespace st5
