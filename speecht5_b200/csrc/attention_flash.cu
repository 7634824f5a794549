// Streaming attention forward on the Hopper tensor cores (wgmma) for ANY Tq / Tk, with clipped relative positions.
// It serves both forward entry points: st5_attn_fused_fwd (Tk <= 320, the relative-position variant without clipping)
// and st5_attn_flash_fwd (any length); the outputs and the psave / inv_l / out_f32 contract are the same.
//
// One CTA = (64 query rows, head, utterance). The keys are walked in blocks of 64; nothing of size Tq x Tk stays on
// chip. The output accumulator lives in the registers of the MMA warpgroup and is never rescaled: the kernel makes the
// row maximum FINAL before the first exponential, sweeping the key blocks twice (three times when the caller wants
// normalised probabilities back) and re-issuing the cheap 64 x 64 x 64 score MMA in every sweep:
//
//   sweep 0   S_kb = Q K_kb^T (+ bias)  -> running row maximum
//   sweep 1   S_kb again -> e = exp2(s - max), row sum, dropout, P -> smem (bf16) -> O += P V_kb  (registers)
//             and, for the backward pass, e (bf16, sign bit = dropped) -> psave
//   sweep 2   (only with `probs`) S_kb again -> e / rowsum -> probabilities
//   epilogue  O / rowsum -> bf16 out (+ fp32 copy), lse, 1 / rowsum
//
// Warps: 0..3 = MMA warpgroup (wgmma; S, QP and the finished O leave through shared memory as fp32 rows), 4 = TMA
// producer, 5..8 = softmax (thread = one query row, one of the two 32-key chunks of a block).
//
// Relative positions (encoder.py:40-59, 239-246; multihead_attention.py:346-353) with clipping:
//   bias[i][j] = q_i . pe[clamp(i - j, -maxpos, maxpos - 1) + maxpos]
// Per key block the kernel computes QPw = Q PEw^T for the 128-row window PEw of the table this (query tile, key block)
// pair can reach; every softmax thread reads its row of QPw skewed by the key (clamped at the table ends).
// Reference semantics: speecht5/models/modules/multihead_attention.py:340-389.
#include "../../include/speecht5_b200.h"
#include "kernels.cuh"
#include "ptx.cuh"
#include "tma_map.cuh"

namespace st5 {

int set_error(int code, const char* where);

constexpr int FL_T = 64;              // query tile == key block
constexpr int FL_THREADS = 9 * 32;    // MMA warpgroup, TMA warp, 4 softmax warps
constexpr int FL_PE_ROWS = 128;       // table rows per window (i - j spans 127 values per tile pair)
constexpr int FL_SP = FL_T + 4;       // floats per row of the S / O tiles (row-per-lane float4 reads: conflict-free)
constexpr int FL_QPP = FL_PE_ROWS + 4;
constexpr int FL_MAX_TK_RESIDENT = 320;
constexpr int FL_MAX_T_RPE_RESIDENT = 160;
// Q 8K | K 2 x 8K | V 8K | P 8K | S 17K | O 17K | (PEw 2 x 16K | QPw 33K) | barriers + row reductions | slack
template <bool RPE> constexpr size_t fl_smem() {
  return 8192 + 2 * 8192 + 8192 + 8192 + 2 * (size_t)FL_T * FL_SP * 4 +
         (RPE ? 2 * 16384 + (size_t)FL_T * FL_QPP * 4 : 0) + 128 + 512 + 1024;
}

struct FlashFwdParams {
  int B, H, Tq, Tk, causal, maxpos;
  float scale_log2;
  const uint8_t* key_pad;
  __nv_bfloat16* out; long o_ld, o_bs;
  float* out_f32;
  float* lse; float* inv_l;
  __nv_bfloat16* psave;
  void* probs; int probs_fp32; long p_ld;
  uint32_t drop_thr; float drop_scale; uint64_t seed, offset;
  int probs_heads;  // > 0: only heads < probs_heads get their probabilities written (no third sweep for the others)
};

__device__ __forceinline__ uint32_t fl_pack(float a, float b) {
  __nv_bfloat162 t = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&t);
}
// first table row of the window a (query tile at i0, key block at j0) pair uses: i - j + maxpos spans
// [i0 - j0 - 63 + maxpos, i0 - j0 + 63 + maxpos]; clamped so that the window stays inside the table
__host__ __device__ __forceinline__ int fl_window_row0(int i0, int j0, int maxpos) {
  int w = i0 - j0 - (FL_T - 1) + maxpos;
  const int hi = 2 * maxpos - FL_PE_ROWS;
  if (w > hi) w = hi;
  if (w < 0) w = 0;
  return w;
}
// m64nN accumulator fragment -> fp32 rows in shared memory (pitch in floats)
template <int NR>
__device__ __forceinline__ void fl_store_acc(float* dst, int pitch, const float (&d)[NR]) {
  const int l = (int)lane_id(), w = (threadIdx.x >> 5) & 3;
  const int r0 = 16 * w + (l >> 2);
#pragma unroll
  for (int i = 0; i < NR; i += 2) {
    const int r = r0 + 8 * ((i >> 1) & 1), c = 8 * (i >> 2) + 2 * (l & 3);
    *reinterpret_cast<float2*>(dst + r * pitch + c) = make_float2(d[i], d[i + 1]);
  }
}

template <bool RPE>
__global__ void __launch_bounds__(FL_THREADS, 1)
    attn_flash_fwd_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k,
                          const __grid_constant__ CUtensorMap map_v, const __grid_constant__ CUtensorMap map_pe,
                          const FlashFwdParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;                     // [64 rows][128 B]
  uint8_t* sK = sQ + 8192;                // 2 x [64 keys][128 B]  (K-major B operand of S)
  uint8_t* sV = sK + 2 * 8192;            // [64 keys][128 B]      (MN-major B operand of O)
  uint8_t* sP = sV + 8192;                // [64 rows][64 keys]    (K-major A operand of O)
  float* sS = reinterpret_cast<float*>(sP + 8192);  // [64][FL_SP] scores of the current step
  float* sO = sS + FL_T * FL_SP;                    // [64][FL_SP] finished output accumulator
  uint8_t* sPE = reinterpret_cast<uint8_t*>(sO + FL_T * FL_SP);  // RPE: 2 x [128 table rows][128 B]
  float* sQP = reinterpret_cast<float*>(sPE + (RPE ? 2 * 16384 : 0));  // RPE: [64][FL_QPP]
  uint64_t* bar_q = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(sQP) + (RPE ? FL_T * FL_QPP * 4 : 0));
  uint64_t* bar_k = bar_q + 1;        // [2] K (+ PEw) of a step landed
  uint64_t* bar_kfree = bar_q + 3;    // [2] the score MMAs that read this K stage have completed
  uint64_t* bar_s = bar_q + 5;        // scores of a step are in sS (+ sQP)
  uint64_t* bar_sfree = bar_q + 6;    // softmax warps have read the scores of a step
  uint64_t* bar_v = bar_q + 7;        // V block landed
  uint64_t* bar_p = bar_q + 8;        // P tile written
  uint64_t* bar_pv = bar_q + 9;       // P V MMAs of a block complete (sP and sV may be rewritten)
  uint64_t* bar_o = bar_q + 10;       // O is in sO
  float* red = reinterpret_cast<float*>(bar_q + 16);  // [2][64] row partials of the two column halves

  const int warp = threadIdx.x >> 5;
  const int nqt = (p.Tq + FL_T - 1) / FL_T;
  const int qt = nqt - 1 - (int)blockIdx.x;  // late (long, when causal) tiles first
  const int h = blockIdx.y, b = blockIdx.z;
  const int i0 = qt * FL_T;
  int tk = p.Tk;
  if (p.causal && i0 + FL_T < tk) tk = i0 + FL_T;
  const int nkb = (tk + FL_T - 1) / FL_T;
  void* const probs = (p.probs_heads > 0 && h >= p.probs_heads) ? nullptr : p.probs;  // (uniform over the CTA)
  const int nsweep = probs != nullptr ? 3 : 2;
  const int NS = nsweep * nkb;

  if (warp == 4 && elect_one()) {
    tma_prefetch_desc(&map_q);
    tma_prefetch_desc(&map_k);
    tma_prefetch_desc(&map_v);
    if constexpr (RPE) tma_prefetch_desc(&map_pe);
    mbar_init(bar_q, 1);
    for (int s = 0; s < 2; ++s) {
      mbar_init(&bar_k[s], 1);
      mbar_init(&bar_kfree[s], 1);
    }
    mbar_init(bar_s, 128);
    mbar_init(bar_sfree, 4);
    mbar_init(bar_v, 1);
    mbar_init(bar_p, 4);
    mbar_init(bar_pv, 1);
    mbar_init(bar_o, 128);
    fence_mbar_init();
  }
  __syncthreads();
  pdl_sync();  // (prologue done: nothing above touched global memory)

  if (warp == 4) {
    // ===================== TMA producer =====================
    if (elect_one()) {
      mbar_expect_tx(bar_q, 8192);
      tma_load_4d(sQ, &map_q, bar_q, 0, i0, h, b);
      int pv = 0;
      for (int s = 0; s < NS; ++s) {
        const int sweep = s / nkb, kb = s - sweep * nkb;
        const int st = s & 1;
        if (s >= 2) mbar_wait_quiet(&bar_kfree[st], (uint32_t)(((s >> 1) - 1) & 1));
        mbar_expect_tx(&bar_k[st], 8192u + (RPE ? 16384u : 0u));
        tma_load_4d(sK + st * 8192, &map_k, &bar_k[st], 0, kb * FL_T, h, b);
        if constexpr (RPE)
          tma_load_4d(sPE + st * 16384, &map_pe, &bar_k[st], 0, fl_window_row0(i0, kb * FL_T, p.maxpos), 0, 0);
        if (sweep == 1) {
          if (pv > 0) mbar_wait_quiet(bar_pv, (uint32_t)((pv - 1) & 1));  // P V of the previous block has read sV
          mbar_expect_tx(bar_v, 8192);
          tma_load_4d(sV, &map_v, bar_v, 0, kb * FL_T, h, b);
          ++pv;
        }
      }
    }
  } else if (warp < 4) {
    // ===================== MMA warpgroup =====================
    mbar_wait_quiet(bar_q, 0);
    const uint32_t aq = smem_u32(sQ), ap = smem_u32(sP), av = smem_u32(sV);
    float o[32];
#pragma unroll
    for (int t = 0; t < 32; ++t) o[t] = 0.f;
    int pv = 0;
    for (int s = 0; s < NS; ++s) {
      const int sweep = s / nkb;
      const int st = s & 1;
      mbar_wait_quiet(&bar_k[st], (uint32_t)((s >> 1) & 1));
      if (s > 0) mbar_wait_quiet(bar_sfree, (uint32_t)((s - 1) & 1));
      {
        float sc[32];
        const uint32_t ak = smem_u32(sK + st * 8192);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k)  // head dim 64 = 4 x 16
          wgmma_m64n64<0, 0>(sc, wgmma_smem_desc(aq + k * 32, 16, 1024), wgmma_smem_desc(ak + k * 32, 16, 1024),
                             k != 0 ? 1u : 0u);
        wgmma_commit();
        if constexpr (RPE) {
          float qp[64];
          const uint32_t ape = smem_u32(sPE + st * 16384);
#pragma unroll
          for (int k = 0; k < 4; ++k)
            wgmma_m64n128<0, 0>(qp, wgmma_smem_desc(aq + k * 32, 16, 1024), wgmma_smem_desc(ape + k * 32, 16, 1024),
                                k != 0 ? 1u : 0u);
          wgmma_commit();
          wgmma_wait<0>();
          wgmma_fence_regs(qp);
          fl_store_acc(sQP, FL_QPP, qp);
        } else {
          wgmma_wait<0>();
        }
        wgmma_fence_regs(sc);
        if (threadIdx.x == 0) mbar_arrive(&bar_kfree[st]);
        fl_store_acc(sS, FL_SP, sc);
      }
      mbar_arrive(bar_s);
      if (sweep == 1) {
        mbar_wait_quiet(bar_v, (uint32_t)(pv & 1));
        mbar_wait_quiet(bar_p, (uint32_t)(pv & 1));
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k)  // 64 keys = 4 x 16
          wgmma_m64n64<0, 1>(o, wgmma_smem_desc(ap + k * 32, 16, 1024), wgmma_smem_desc(av + k * 2048, 8192, 1024),
                             (pv | k) != 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(o);
        if (threadIdx.x == 0) mbar_arrive(bar_pv);
        ++pv;
      }
    }
    fl_store_acc(sO, FL_SP, o);
    mbar_arrive(bar_o);
  } else {
    // ===================== softmax warps: thread = (query row, 32-key chunk `half` of every block) =====================
    const int sw = warp - 5;
    const int q = sw & 1;                   // rows [32 q, 32 q + 32) of the tile
    const int half = sw >> 1;               // 0 / 1
    const int lane = (int)lane_id();
    const int r = q * 32 + lane;
    const int i = i0 + r;
    const bool row_ok = i < p.Tq;
    const bool warp_live = i0 + q * 32 < p.Tq;
    const uint8_t* kp = p.key_pad != nullptr ? p.key_pad + (int64_t)b * p.Tk : nullptr;
    const int64_t prow = ((int64_t)b * p.H + h) * p.Tq + i;
    uint64_t dseed = p.seed, doffset = p.offset;
    if (p.drop_thr != 0) resolve_seed(dseed, doffset);
    float* probs_f = reinterpret_cast<float*>(probs);
    __nv_bfloat16* probs_h = reinterpret_cast<__nv_bfloat16*>(probs);

    float m = -INFINITY, mm = 0.f, sum = 0.f, inv = 0.f;
    int pv = 0;
    for (int sweep = 0; sweep < nsweep; ++sweep) {
      for (int kb = 0; kb < nkb; ++kb) {
        const int s = sweep * nkb + kb;
        const int j0 = kb * FL_T;
        mbar_wait_quiet(bar_s, (uint32_t)(s & 1));
        if (sweep == 1 && pv > 0) mbar_wait_quiet(bar_pv, (uint32_t)((pv - 1) & 1));  // sP is free again
        const int c = half;  // 32-key chunk of the block
        const int jc = j0 + c * 32;
        // warp-uniform: does any (row, key) pair of this 32 x 32 chunk exist and pass the causal mask?
        const bool live = warp_live && jc < tk && !(p.causal && jc > i0 + q * 32 + 31);
        uint8_t* blk = sP + r * 128;
        const int cbase = c * 4;
        if (!live) {
          if (sweep == 1) {  // the P V MMA contracts over these keys and the backward reads psave: zeros
#pragma unroll
            for (int g = 0; g < 4; ++g) {
              *reinterpret_cast<uint4*>(blk + (((cbase + g) ^ (r & 7)) << 4)) = make_uint4(0u, 0u, 0u, 0u);
              if (p.psave != nullptr && row_ok && jc + 8 * g + 8 <= p.p_ld)
                *reinterpret_cast<uint4*>(p.psave + prow * p.p_ld + jc + 8 * g) = make_uint4(0u, 0u, 0u, 0u);
            }
          } else if (sweep == 2 && row_ok) {
            for (int t = 0; t < 32; ++t)
              if (jc + t < p.p_ld) {
                if (p.probs_fp32) probs_f[prow * p.p_ld + jc + t] = 0.f;
                else probs_h[prow * p.p_ld + jc + t] = __float2bfloat16(0.f);
              }
          }
        } else {
          float v[32];
          {
            const float* src = sS + r * FL_SP + c * 32;
#pragma unroll
            for (int t = 0; t < 32; t += 4) {
              const float4 f = *reinterpret_cast<const float4*>(src + t);
              v[t] = f.x; v[t + 1] = f.y; v[t + 2] = f.z; v[t + 3] = f.w;
            }
          }
          // validity bits of this row's 32 keys: key exists, not padded (one byte load per lane + ballot), causal
          uint32_t vb;
          {
            const int j = jc + lane;
            const bool ok = j < tk && !(kp != nullptr && kp[j] != 0);
            vb = __ballot_sync(0xffffffffu, ok);
            if (p.causal) {
              const int lim = i - jc;  // keys 0..lim of the chunk are visible
              vb &= lim >= 31 ? 0xffffffffu : (lim < 0 ? 0u : ((2u << lim) - 1u));
            }
          }
          if constexpr (RPE) {
            // row i, key j = jc + u  ->  window column i - j + maxpos - w0, clamped to [0, colmax] (the table ends)
            const int w0 = fl_window_row0(i0, j0, p.maxpos);
            int colmax = 2 * p.maxpos - 1 - w0;
            if (colmax > FL_PE_ROWS - 1) colmax = FL_PE_ROWS - 1;
            const int off = i - jc + p.maxpos - w0;
            const float* qrow = sQP + r * FL_QPP;
#pragma unroll
            for (int t = 0; t < 32; ++t) {
              int col = off - t;
              col = col < 0 ? 0 : (col > colmax ? colmax : col);
              v[t] += qrow[col];
            }
          }
          if (sweep == 0) {
#pragma unroll
            for (int t = 0; t < 32; ++t)
              if ((vb >> t) & 1u) m = fmaxf(m, v[t] * p.scale_log2);
          } else if (sweep == 1) {
            uint32_t kb_ = 0xffffffffu;
            if (p.drop_thr != 0)
              kb_ = dropout_keep_mask32(dseed, doffset, (uint64_t)prow * attn_drop_pitch(p.Tk) + (uint64_t)jc, p.drop_thr);
            __nv_bfloat16* psv = (p.psave != nullptr && row_ok) ? p.psave + prow * p.p_ld + jc : nullptr;
#pragma unroll
            for (int g = 0; g < 4; ++g) {
              float ev[8];
#pragma unroll
              for (int t = 0; t < 8; ++t) {
                const int u = 8 * g + t;
                ev[t] = ((vb >> u) & 1u) ? fast_ex2(v[u] * p.scale_log2 - mm) : 0.f;
                sum += ev[t];
              }
              const uint32_t k8 = kb_ >> (8 * g);
              uint4 pk, ps;
              pk.x = fl_pack((k8 & 1u) ? ev[0] * p.drop_scale : 0.f, (k8 & 2u) ? ev[1] * p.drop_scale : 0.f);
              pk.y = fl_pack((k8 & 4u) ? ev[2] * p.drop_scale : 0.f, (k8 & 8u) ? ev[3] * p.drop_scale : 0.f);
              pk.z = fl_pack((k8 & 16u) ? ev[4] * p.drop_scale : 0.f, (k8 & 32u) ? ev[5] * p.drop_scale : 0.f);
              pk.w = fl_pack((k8 & 64u) ? ev[6] * p.drop_scale : 0.f, (k8 & 128u) ? ev[7] * p.drop_scale : 0.f);
              *reinterpret_cast<uint4*>(blk + (((cbase + g) ^ (r & 7)) << 4)) = pk;
              if (psv != nullptr && jc + 8 * g + 8 <= p.p_ld) {
                ps.x = fl_pack((k8 & 1u) ? ev[0] : -ev[0], (k8 & 2u) ? ev[1] : -ev[1]);
                ps.y = fl_pack((k8 & 4u) ? ev[2] : -ev[2], (k8 & 8u) ? ev[3] : -ev[3]);
                ps.z = fl_pack((k8 & 16u) ? ev[4] : -ev[4], (k8 & 32u) ? ev[5] : -ev[5]);
                ps.w = fl_pack((k8 & 64u) ? ev[6] : -ev[6], (k8 & 128u) ? ev[7] : -ev[7]);
                *reinterpret_cast<uint4*>(psv + 8 * g) = ps;
              }
            }
          } else if (row_ok) {  // sweep 2: normalised, undropped probabilities for the caller
            if (p.probs_fp32) {
              float* dst = probs_f + prow * p.p_ld + jc;
              if (jc + 32 <= p.p_ld && (p.p_ld & 3) == 0) {
#pragma unroll
                for (int t = 0; t < 32; t += 4) {
                  float4 o4;
                  o4.x = ((vb >> t) & 1u) ? fast_ex2(v[t] * p.scale_log2 - mm) * inv : 0.f;
                  o4.y = ((vb >> (t + 1)) & 1u) ? fast_ex2(v[t + 1] * p.scale_log2 - mm) * inv : 0.f;
                  o4.z = ((vb >> (t + 2)) & 1u) ? fast_ex2(v[t + 2] * p.scale_log2 - mm) * inv : 0.f;
                  o4.w = ((vb >> (t + 3)) & 1u) ? fast_ex2(v[t + 3] * p.scale_log2 - mm) * inv : 0.f;
                  *reinterpret_cast<float4*>(dst + t) = o4;
                }
              } else {
#pragma unroll
                for (int t = 0; t < 32; ++t)
                  if (jc + t < p.p_ld) dst[t] = ((vb >> t) & 1u) ? fast_ex2(v[t] * p.scale_log2 - mm) * inv : 0.f;
              }
            } else {
              __nv_bfloat16* dst = probs_h + prow * p.p_ld + jc;
#pragma unroll
              for (int t = 0; t < 32; ++t)
                if (jc + t < p.p_ld)
                  dst[t] = __float2bfloat16(((vb >> t) & 1u) ? fast_ex2(v[t] * p.scale_log2 - mm) * inv : 0.f);
            }
          }
        }
        if (sweep == 1) {
          fence_proxy_async();  // generic-proxy smem writes -> visible to the tensor core (async proxy)
          __syncwarp();
          if (lane == 0) mbar_arrive(bar_p);
          ++pv;
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_sfree);
      }
      if (sweep == 0) {  // the row maximum over all keys: combine the two column halves
        red[half * FL_T + r] = m;
        asm volatile("bar.sync 1, 128;" ::: "memory");
        m = fmaxf(red[r], red[FL_T + r]);
        mm = m == -INFINITY ? 0.f : m;
        asm volatile("bar.sync 1, 128;" ::: "memory");
      } else if (sweep == 1) {
        red[half * FL_T + r] = sum;
        asm volatile("bar.sync 1, 128;" ::: "memory");
        sum = red[r] + red[FL_T + r];
        inv = sum > 0.f ? 1.f / sum : 0.f;
        if (half == 0 && row_ok) {
          if (p.lse != nullptr) p.lse[prow] = sum > 0.f ? (mm + log2f(sum)) * 0.6931471805599453f : -INFINITY;
          if (p.inv_l != nullptr) p.inv_l[prow] = inv;
        }
        asm volatile("bar.sync 1, 128;" ::: "memory");
      } else if (p.causal && half == 0 && row_ok) {  // probabilities right of the last visible block
        for (int j = nkb * FL_T; j < (int)p.p_ld; ++j) {
          if (p.probs_fp32) probs_f[prow * p.p_ld + j] = 0.f;
          else probs_h[prow * p.p_ld + j] = __float2bfloat16(0.f);
        }
      }
    }
    // ---- epilogue: O / rowsum; this thread owns channels [32 half, 32 half + 32) of its row
    mbar_wait_quiet(bar_o, 0);
    if (row_ok) {
      float v[32];
      const float* src = sO + r * FL_SP + half * 32;
#pragma unroll
      for (int t = 0; t < 32; t += 4) {
        const float4 f = *reinterpret_cast<const float4*>(src + t);
        v[t] = f.x * inv; v[t + 1] = f.y * inv; v[t + 2] = f.z * inv; v[t + 3] = f.w * inv;
      }
      if (p.out_f32 != nullptr) {
        float* d32 = p.out_f32 + ((int64_t)b * p.Tq + i) * (p.H * 64) + h * 64 + half * 32;
#pragma unroll
        for (int t = 0; t < 32; t += 4) *reinterpret_cast<float4*>(d32 + t) = make_float4(v[t], v[t + 1], v[t + 2], v[t + 3]);
      }
      __nv_bfloat16* dst = p.out + (int64_t)b * p.o_bs + (int64_t)i * p.o_ld + h * 64 + half * 32;
#pragma unroll
      for (int t = 0; t < 32; t += 8) {
        uint4 pk;
        pk.x = fl_pack(v[t], v[t + 1]);
        pk.y = fl_pack(v[t + 2], v[t + 3]);
        pk.z = fl_pack(v[t + 4], v[t + 5]);
        pk.w = fl_pack(v[t + 6], v[t + 7]);
        *reinterpret_cast<uint4*>(dst + t) = pk;
      }
    }
  }
}

static int fl_make_map(CUtensorMap* m, const void* ptr, int64_t rows, int64_t ld, int64_t bs, int H, int B) {
  const uint64_t dims[4] = {64, (uint64_t)rows, (uint64_t)H, (uint64_t)B};
  const uint64_t strides[3] = {(uint64_t)ld * 2, 128, (uint64_t)bs * 2};
  const uint32_t box[4] = {64, FL_T, 1, 1};
  return encode_bf16_map_4d(m, ptr, dims, strides, box);
}

static int fl_launch(const st5_attn_args* a, float* lse, void* psave, float* inv_l, float* out_f32, void* stream,
                     const char* who) {
  const bool rpe = a->pe_k != nullptr;
  CUtensorMap mq, mk, mv;
  int rc = fl_make_map(&mq, a->q, a->Tq, a->q_ld, a->q_bs, a->H, a->B);
  if (!rc) rc = fl_make_map(&mk, a->k, a->Tk, a->k_ld, a->k_bs, a->H, a->B);
  if (!rc) rc = fl_make_map(&mv, a->v, a->Tk, a->v_ld, a->v_bs, a->H, a->B);
  CUtensorMap mpe = mq;
  if (!rc && rpe) {  // the bf16 table [2*maxpos][64] as a rank-4 map with unit outer dimensions; rows past its end read 0
    const uint64_t dims[4] = {64, (uint64_t)(2 * a->maxpos), 1, 1};
    const uint64_t strides[3] = {128, (uint64_t)(2 * a->maxpos) * 128, (uint64_t)(2 * a->maxpos) * 128};
    const uint32_t box[4] = {64, FL_PE_ROWS, 1, 1};
    rc = encode_bf16_map_4d(&mpe, a->pe_k, dims, strides, box);
  }
  if (rc) return set_error(rc, who);
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(attn_flash_fwd_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)fl_smem<false>());
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(attn_flash_fwd_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                               (int)fl_smem<true>());
    if (e != cudaSuccess) return set_error((int)e, who);
    attr_set = true;
  }
  FlashFwdParams p;
  p.B = a->B; p.H = a->H; p.Tq = a->Tq; p.Tk = a->Tk; p.causal = a->causal; p.maxpos = a->maxpos;
  p.scale_log2 = a->scale * 1.4426950408889634f;
  p.key_pad = a->key_pad;
  p.out = (__nv_bfloat16*)a->out; p.o_ld = a->o_ld; p.o_bs = a->o_bs;
  p.out_f32 = out_f32;
  p.lse = lse; p.inv_l = inv_l;
  p.psave = reinterpret_cast<__nv_bfloat16*>(psave);
  p.probs = a->probs; p.probs_fp32 = a->probs_dtype == ST5_F32; p.p_ld = a->p_ld;
  p.probs_heads = a->probs_heads;
  p.drop_thr = drop_threshold(a->drop_p);
  p.drop_scale = a->drop_p > 0.f ? 1.f / (1.f - a->drop_p) : 1.f;
  p.seed = a->seed; p.offset = a->offset;
  dim3 grid((a->Tq + FL_T - 1) / FL_T, a->H, a->B);
  if (rpe)
    launch_pdl(attn_flash_fwd_kernel<true>, grid, dim3(FL_THREADS), fl_smem<true>(), (cudaStream_t)stream, mq, mk, mv, mpe, p);
  else
    launch_pdl(attn_flash_fwd_kernel<false>, grid, dim3(FL_THREADS), fl_smem<false>(), (cudaStream_t)stream, mq, mk, mv, mpe, p);
  return set_error((int)cudaGetLastError(), who);
}

static int fl_check_common(const st5_attn_args* a, void* psave, const float* inv_l, const char* who) {
  if ((a->probs != nullptr || psave != nullptr) && a->p_ld < a->Tk) return set_error(-3, who);
  if (psave != nullptr && ((a->p_ld & 7) || (reinterpret_cast<uintptr_t>(psave) & 15) || inv_l == nullptr))
    return set_error(-3, "attention forward: psave needs a row pitch that is a multiple of 8, 16-byte alignment and inv_l");
  if ((a->o_ld & 7) || (a->o_bs & 7) || (reinterpret_cast<uintptr_t>(a->out) & 15))
    return set_error(-4, "attention forward: out must be 16-byte aligned");
  return 0;
}

}  // namespace st5

using namespace st5;

extern "C" int st5_attn_fused_fwd(const st5_attn_args* a, float* lse, void* psave, float* inv_l, float* out_f32,
                                  void* stream) {
  const bool rpe = a->pe_k != nullptr;
  if (a->dtype != ST5_BF16 || a->Tk > FL_MAX_TK_RESIDENT || a->Tk <= 0 || a->Tq <= 0)
    return set_error(-2, "st5_attn_fused_fwd: needs bf16 and Tk <= 320");
  if (rpe && (a->causal || a->maxpos <= 0 || a->maxpos > FL_MAX_T_RPE_RESIDENT || a->Tk > a->maxpos || a->Tq > a->maxpos))
    return set_error(-5, "st5_attn_fused_fwd: relative positions need Tq, Tk <= maxpos <= 160 (no clipping), no causal mask");
  const int rc = fl_check_common(a, psave, inv_l, "st5_attn_fused_fwd");
  if (rc) return rc;
  return fl_launch(a, lse, psave, inv_l, out_f32, stream, "st5_attn_fused_fwd");
}

extern "C" int st5_attn_flash_fwd(const st5_attn_args* a, float* lse, void* psave, float* inv_l, float* out_f32,
                                  void* stream) {
  const bool rpe = a->pe_k != nullptr;
  if (a->dtype != ST5_BF16 || a->Tk <= 0 || a->Tq <= 0) return set_error(-2, "st5_attn_flash_fwd: needs bf16");
  if (rpe && (a->causal || a->maxpos <= 0)) return set_error(-5, "st5_attn_flash_fwd: relative positions take no causal mask");
  if (a->probs != nullptr && a->probs_dtype != ST5_F32)
    return set_error(-3, "st5_attn_flash_fwd: returned probabilities are fp32");
  const int rc = fl_check_common(a, psave, inv_l, "st5_attn_flash_fwd");
  if (rc) return rc;
  return fl_launch(a, lse, psave, inv_l, out_f32, stream, "st5_attn_flash_fwd");
}
