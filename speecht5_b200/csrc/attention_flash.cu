// Streaming attention forward on the Hopper tensor cores (wgmma) for ANY Tq / Tk, with clipped relative positions.
// It serves both forward entry points: st5_attn_fused_fwd (Tk <= 320, the relative-position variant without clipping)
// and st5_attn_flash_fwd (any length); the outputs and the psave / inv_l / out_f32 contract are the same.
//
// One CTA = (two 64-row query tiles, head, utterance). The keys are walked in blocks of 64; nothing of size Tq x Tk
// stays on chip. The output accumulator lives in registers and is never rescaled: the kernel makes the row maximum
// FINAL before the first exponential, sweeping the key blocks twice (three times when the caller wants normalised
// probabilities back) and re-issuing the cheap 64 x 64 x 64 score MMA in every sweep:
//
//   sweep 0   S_kb = Q K_kb^T (+ bias)  -> running row maximum
//   sweep 1   S_kb again -> e = exp2(s - max), row sum, dropout, P (bf16, registers) -> O += P V_kb
//             and, for the backward pass, e (bf16, sign bit = dropped) -> psave
//   sweep 2   (only with `probs`) S_kb again -> e / rowsum -> probabilities
//   epilogue  O / rowsum -> bf16 out (+ fp32 copy), lse, 1 / rowsum
//
// Warps: 0..3 and 4..7 = two MMA warpgroups, one query tile each; 8 = TMA producer. Each warpgroup does its softmax on
// its own accumulator fragments (a row is spread over one quad of lanes) and feeds P to the P V wgmma as its register
// A operand, so scores and probabilities never go through shared memory. K and V arrive in a ring of stages that both
// warpgroups read, so each key block is loaded once per 128 query rows. While one warpgroup forms its exponentials the
// other's MMAs run. Causal CTAs pair tile n-1-x with tile x, so that every CTA does the same work; otherwise tiles 2x
// and 2x+1 share a CTA. A lone last tile runs with the second warpgroup idle.
//
// Relative positions (encoder.py:40-59, 239-246; multihead_attention.py:346-353) with clipping:
//   bias[i][j] = q_i . pe[clamp(i - j, -maxpos, maxpos - 1) + maxpos]
// Per key block each warpgroup computes QPw = Q PEw^T for the 128-row window PEw of the table its (query tile, key
// block) pair can reach; the skewed read (row i, key j -> column i - j, clamped at the table ends) needs other lanes'
// columns, so QPw goes through shared memory, one window per warpgroup.
// Reference semantics: speecht5/models/modules/multihead_attention.py:340-389.
#include "../../include/speecht5_b200.h"
#include "kernels.cuh"
#include "ptx.cuh"
#include "tma_map.cuh"

namespace st5 {

int set_error(int code, const char* where);

constexpr int FL_T = 64;              // query tile == key block
constexpr int FL_THREADS = 9 * 32;    // two MMA warpgroups, TMA warp
constexpr int FL_PE_ROWS = 128;       // table rows per window (i - j spans 127 values per tile pair)
constexpr int FL_QPP = FL_PE_ROWS + 4;
constexpr int FL_MAX_TK_RESIDENT = 320;
constexpr int FL_MAX_T_RPE_RESIDENT = 160;
// K / V ring depth: three stages without relative positions; two with them (a stage also holds both PE windows).
template <bool RPE> constexpr int fl_stages() { return RPE ? 2 : 3; }
// one stage: K 8K | V 8K | (PEw of each warpgroup 2 x 16K)
template <bool RPE> constexpr uint32_t fl_stage_bytes() { return 2 * 8192 + (RPE ? 2 * 16384 : 0); }
// Q 2 x 8K | stages | (QPw 2 x 33K) | barriers | alignment slack
template <bool RPE> constexpr size_t fl_smem() {
  return 2 * 8192 + (size_t)fl_stages<RPE>() * fl_stage_bytes<RPE>() + (RPE ? 2 * (size_t)FL_T * FL_QPP * 4 : 0) +
         128 + 1024;
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
// query tiles of CTA x (tb = -1: none): causal CTAs pair the long tile n-1-x with the short tile x, so that all do the
// same work and ta is the longer one; otherwise neighbours 2x, 2x+1
__device__ __forceinline__ void fl_tiles(int x, int nqt, bool causal, int& ta, int& tb) {
  if (causal) {
    ta = nqt - 1 - x;
    tb = x < ta ? x : -1;
  } else {
    ta = 2 * x;
    tb = 2 * x + 1 < nqt ? 2 * x + 1 : -1;
  }
}
__device__ __forceinline__ int fl_tile_nkb(int t, int Tk, bool causal) {
  int tk = Tk;
  if (causal && (t + 1) * FL_T < tk) tk = (t + 1) * FL_T;
  return (tk + FL_T - 1) / FL_T;
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
__device__ __forceinline__ void fl_bar_wg(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }
__device__ __forceinline__ void fl_fence_u32(uint32_t (&a)[4][4]) {
#pragma unroll
  for (int k = 0; k < 4; ++k)
#pragma unroll
    for (int i = 0; i < 4; ++i) asm volatile("" : "+r"(a[k][i])::"memory");
}
// Dropout keep bits of this thread's 32 accumulator elements of one key block (bit i <-> d[i]), at the element index
// the row-per-thread kernels use (prow * attn_drop_pitch(Tk) + key). e0/e1: index of key j0 in rows r0 and r0 + 8.
// Lane qd of a quad draws the Philox groups 2qd and 2qd + 1 (keys 16 qd .. 16 qd + 15) of both rows; the quad then
// exchanges them, since every lane holds two keys of each of the eight groups.
__device__ __forceinline__ uint32_t fl_keep_bits(uint64_t seed, uint64_t offset, uint64_t e0, uint64_t e1,
                                                 uint32_t thr) {
  const int lane = (int)lane_id(), qd = lane & 3;
  uint32_t mine = 0;  // byte 2 ri + cc = the eight keep bits of group 2 qd + cc, row ri
#pragma unroll
  for (int ri = 0; ri < 2; ++ri)
#pragma unroll
    for (int cc = 0; cc < 2; ++cc) {
      const Philox4 r = philox4x32(seed, offset, ((ri ? e1 : e0) + 16 * qd + 8 * cc) >> 3);
#pragma unroll
      for (int l = 0; l < 8; ++l)
        if (philox_lane16(r, l) >= thr) mine |= 1u << (8 * (2 * ri + cc) + l);
    }
  uint32_t keep = 0;
#pragma unroll
  for (int src = 0; src < 4; ++src) {
    const uint32_t x = __shfl_sync(0xffffffffu, mine, (lane & ~3) | src);
#pragma unroll
    for (int cc = 0; cc < 2; ++cc)
#pragma unroll
      for (int ri = 0; ri < 2; ++ri) {
        const uint32_t bits = (x >> (8 * (2 * ri + cc) + 2 * qd)) & 3u;  // keys 2 qd, 2 qd + 1 of group 2 src + cc
        keep |= bits << (4 * (2 * src + cc) + 2 * ri);
      }
  }
  return keep;
}

template <bool RPE>
__global__ void __launch_bounds__(FL_THREADS, 1)
    attn_flash_fwd_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k,
                          const __grid_constant__ CUtensorMap map_v, const __grid_constant__ CUtensorMap map_pe,
                          const FlashFwdParams p) {
  constexpr int ST = fl_stages<RPE>();
  constexpr uint32_t SB = fl_stage_bytes<RPE>();
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;             // 2 x [64 rows][128 B], one tile per warpgroup
  uint8_t* sStage = sQ + 2 * 8192;  // ST x { K [64 keys][128 B] (K-major B of S) | V [64 keys][128 B] (MN-major B of O)
                                    //        | RPE: 2 x PEw [128 table rows][128 B] }
  float* sQP = reinterpret_cast<float*>(sStage + ST * SB);  // RPE: 2 x [64][FL_QPP]
  uint64_t* bar_q = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(sQP) + (RPE ? 2 * FL_T * FL_QPP * 4 : 0));
  uint64_t* bar_full = bar_q + 1;       // [ST] K (+ V in sweep 1, + PEw) of a stage landed
  uint64_t* bar_free = bar_full + ST;   // [ST] every warpgroup's MMAs that read the stage have completed

  const int warp = threadIdx.x >> 5;
  const int nqt = (p.Tq + FL_T - 1) / FL_T;
  int ta, tb;
  fl_tiles((int)blockIdx.x, nqt, p.causal != 0, ta, tb);
  const int nwg = tb >= 0 ? 2 : 1;
  const int h = blockIdx.y, b = blockIdx.z;
  const int nkbm = fl_tile_nkb(ta, p.Tk, p.causal != 0);  // key blocks the longer tile needs
  void* const probs = (p.probs_heads > 0 && h >= p.probs_heads) ? nullptr : p.probs;  // (uniform over the CTA)
  const int nsweep = probs != nullptr ? 3 : 2;

  if (warp == 8 && elect_one()) {
    tma_prefetch_desc(&map_q);
    tma_prefetch_desc(&map_k);
    tma_prefetch_desc(&map_v);
    if constexpr (RPE) tma_prefetch_desc(&map_pe);
    mbar_init(bar_q, 1);
    for (int s = 0; s < ST; ++s) {
      mbar_init(&bar_full[s], 1);
      mbar_init(&bar_free[s], nwg);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_sync();  // (prologue done: nothing above touched global memory)

  if (warp == 8) {
    // ===================== TMA producer =====================
    if (elect_one()) {
      mbar_expect_tx(bar_q, 8192u * nwg);
      tma_load_4d(sQ, &map_q, bar_q, 0, ta * FL_T, h, b);
      if (tb >= 0) tma_load_4d(sQ + 8192, &map_q, bar_q, 0, tb * FL_T, h, b);
      const int NS = nsweep * nkbm;
      for (int s = 0; s < NS; ++s) {
        const int sweep = s / nkbm, kb = s - sweep * nkbm, st = s % ST;
        if (s >= ST) mbar_wait_quiet(&bar_free[st], (uint32_t)((s / ST - 1) & 1));
        uint8_t* stg = sStage + st * SB;
        mbar_expect_tx(&bar_full[st], (sweep == 1 ? 16384u : 8192u) + (RPE ? 16384u * nwg : 0u));
        tma_load_4d(stg, &map_k, &bar_full[st], 0, kb * FL_T, h, b);
        if (sweep == 1) tma_load_4d(stg + 8192, &map_v, &bar_full[st], 0, kb * FL_T, h, b);
        if constexpr (RPE) {
          tma_load_4d(stg + 16384, &map_pe, &bar_full[st], 0, fl_window_row0(ta * FL_T, kb * FL_T, p.maxpos), 0, 0);
          if (tb >= 0)
            tma_load_4d(stg + 32768, &map_pe, &bar_full[st], 0, fl_window_row0(tb * FL_T, kb * FL_T, p.maxpos), 0, 0);
        }
      }
    }
    return;
  }

  // ===================== MMA warpgroups: thread = rows r0, r0 + 8 x 16 keys of every block =====================
  const int wg = warp >> 2, wl = warp & 3;
  const int t = wg == 0 ? ta : tb;
  if (t < 0) return;  // second warpgroup of a lone tile
  const bool lead = (threadIdx.x & 127) == 0;
  const int i0 = t * FL_T;
  int tk = p.Tk;
  if (p.causal && i0 + FL_T < tk) tk = i0 + FL_T;
  const int nkb = (tk + FL_T - 1) / FL_T;
  const int lane = (int)lane_id(), qd = lane & 3;
  const int r0 = 16 * wl + (lane >> 2);                      // local rows r0 and r0 + 8
  const bool row_ok[2] = {i0 + r0 < p.Tq, i0 + r0 + 8 < p.Tq};
  const int64_t prow0 = ((int64_t)b * p.H + h) * p.Tq + i0 + r0;  // row r0 + 8 ri: prow0 + 8 ri
  const int rh = i0 + 32 * (wl >> 1);  // first row of this warp's 32-row half (the psave zero-fill granularity)
  const uint8_t* kp = p.key_pad != nullptr ? p.key_pad + (int64_t)b * p.Tk : nullptr;
  uint64_t dseed = p.seed, doffset = p.offset;
  if (p.drop_thr != 0) resolve_seed(dseed, doffset);
  const uint64_t dpitch = attn_drop_pitch(p.Tk);
  float* probs_f = reinterpret_cast<float*>(probs);
  __nv_bfloat16* probs_h = reinterpret_cast<__nv_bfloat16*>(probs);
  const uint32_t aq = smem_u32(sQ + wg * 8192);
  float* qpw = sQP + wg * FL_T * FL_QPP;

  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, mm[2] = {0.f, 0.f}, sum[2] = {0.f, 0.f}, inv[2] = {0.f, 0.f};
  mbar_wait_quiet(bar_q, 0);
  for (int sweep = 0; sweep < nsweep; ++sweep) {
    for (int kb = 0; kb < nkbm; ++kb) {
      const int s = sweep * nkbm + kb, st = s % ST;
      mbar_wait_quiet(&bar_full[st], (uint32_t)((s / ST) & 1));
      if (kb >= nkb) {  // a block only the other (longer, causal) tile needs
        if (lead) mbar_arrive(&bar_free[st]);
        continue;
      }
      const int j0 = kb * FL_T;
      const uint32_t astg = smem_u32(sStage + st * SB);
      // which of this thread's elements count: key exists and is not padded (a byte per lane + ballot), causal, and
      // the element's 32 x 32 chunk (rows of this warp's half, 32 keys) is live
      uint32_t vm = 0;
      bool live[2];
      {
        const int ja = j0 + lane, jb = j0 + 32 + lane;
        const uint32_t oka = __ballot_sync(0xffffffffu, ja < p.Tk && !(kp != nullptr && kp[ja] != 0));
        const uint32_t okb = __ballot_sync(0xffffffffu, jb < p.Tk && !(kp != nullptr && kp[jb] != 0));
#pragma unroll
        for (int ch = 0; ch < 2; ++ch) {
          const int jc = j0 + 32 * ch;
          live[ch] = rh < p.Tq && jc < tk && !(p.causal && jc > rh + 31);
        }
        const uint64_t okk = (live[0] ? (uint64_t)oka : 0ull) | (live[1] ? (uint64_t)okb << 32 : 0ull);
#pragma unroll
        for (int ri = 0; ri < 2; ++ri) {
          uint64_t rm = okk;  // bit j: key j0 + j counts for row r0 + 8 ri
          if (p.causal) {
            const int lim = i0 + r0 + 8 * ri - j0;  // keys j0 .. j0 + lim are visible
            rm &= lim >= 63 ? ~0ull : (lim < 0 ? 0ull : (2ull << lim) - 1ull);
          }
          const uint32_t lo = (uint32_t)(rm >> (2 * qd)), hi = (uint32_t)(rm >> (32 + 2 * qd));
#pragma unroll
          for (int c = 0; c < 8; ++c)
            vm |= (((c < 4 ? lo : hi) >> (8 * (c & 3))) & 3u) << (4 * c + 2 * ri);
        }
      }
      // dropout keep bits (sweep 1), drawn before the MMAs so that no score fragment is live meanwhile
      uint32_t keep = 0xffffffffu;
      if (sweep == 1 && p.drop_thr != 0)
        keep = fl_keep_bits(dseed, doffset, (uint64_t)prow0 * dpitch + j0, (uint64_t)(prow0 + 8) * dpitch + j0,
                            p.drop_thr);
      if constexpr (RPE) {  // QPw first, so that its fragment and the score fragment are never live together
        float qp[64];
        const uint32_t ape = astg + 16384 + wg * 16384;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wgmma_m64n128<0, 0>(qp, wgmma_smem_desc(aq + k * 32, 16, 1024), wgmma_smem_desc(ape + k * 32, 16, 1024),
                              k != 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(qp);
        fl_bar_wg(1 + wg);  // every lane has read the previous block's window
        fl_store_acc(qpw, FL_QPP, qp);
      }
      float sc[32];
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k)  // head dim 64 = 4 x 16
        wgmma_m64n64<0, 0>(sc, wgmma_smem_desc(aq + k * 32, 16, 1024), wgmma_smem_desc(astg + k * 32, 16, 1024),
                           k != 0 ? 1u : 0u);
      wgmma_commit();
      if constexpr (RPE) fl_bar_wg(1 + wg);  // the window is complete (while the score MMAs run)
      wgmma_wait<0>();
      wgmma_fence_regs(sc);
      if (sweep != 1 && lead) mbar_arrive(&bar_free[st]);
      if constexpr (RPE) {
        // row i, key j  ->  window column i - j + maxpos - w0, clamped to [0, colmax] (the table ends)
        const int w0 = fl_window_row0(i0, j0, p.maxpos);
        int colmax = 2 * p.maxpos - 1 - w0;
        if (colmax > FL_PE_ROWS - 1) colmax = FL_PE_ROWS - 1;
        const int off = i0 + r0 - j0 - 2 * qd + p.maxpos - w0;  // column of row r0, key j0 + 2 qd
        const float* qrow = qpw + r0 * FL_QPP;
#pragma unroll
        for (int i = 0; i < 32; ++i) {
          const int ri = (i >> 1) & 1;
          int col = off + 8 * ri - 8 * (i >> 2) - (i & 1);
          col = col < 0 ? 0 : (col > colmax ? colmax : col);
          sc[i] += qrow[8 * ri * FL_QPP + col];
        }
      }
      if (sweep == 0) {
#pragma unroll
        for (int i = 0; i < 32; ++i)
          if ((vm >> i) & 1u) m[(i >> 1) & 1] = fmaxf(m[(i >> 1) & 1], sc[i] * p.scale_log2);
      } else if (sweep == 1) {
        uint32_t pa[4][4];  // P as the A operand of P V: 16 keys per four registers
#pragma unroll
        for (int i = 0; i < 32; i += 2) {
          const int ri = (i >> 1) & 1, c = i >> 2;
          const float e0 = ((vm >> i) & 1u) ? fast_ex2(sc[i] * p.scale_log2 - mm[ri]) : 0.f;
          const float e1 = ((vm >> (i + 1)) & 1u) ? fast_ex2(sc[i + 1] * p.scale_log2 - mm[ri]) : 0.f;
          sum[ri] += e0;
          sum[ri] += e1;
          const bool k0 = (keep >> i) & 1u, k1 = (keep >> (i + 1)) & 1u;
          pa[c >> 1][(c & 1) << 1 | ri] =
              fl_pack(k0 ? e0 * p.drop_scale : 0.f, k1 ? e1 * p.drop_scale : 0.f);
          const int jcol = j0 + 8 * c;
          if (p.psave != nullptr && row_ok[ri] && jcol + 8 <= p.p_ld)
            *reinterpret_cast<uint32_t*>(p.psave + (prow0 + 8 * ri) * p.p_ld + jcol + 2 * qd) =
                live[c >> 2] ? fl_pack(k0 ? e0 : -e0, k1 ? e1 : -e1) : 0u;
        }
        const uint32_t av = astg + 8192;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k)  // 64 keys = 4 x 16
          wgmma_m64n64_rs<1>(o, pa[k], wgmma_smem_desc(av + k * 2048, 8192, 1024), 1u);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(o);
        fl_fence_u32(pa);
        if (lead) mbar_arrive(&bar_free[st]);  // K and V of the stage are both read
      } else {  // sweep 2: normalised, undropped probabilities for the caller
#pragma unroll
        for (int i = 0; i < 32; ++i) {
          const int ri = (i >> 1) & 1;
          const int j = j0 + 8 * (i >> 2) + 2 * qd + (i & 1);
          if (row_ok[ri] && j < p.p_ld) {
            const float pr = ((vm >> i) & 1u) ? fast_ex2(sc[i] * p.scale_log2 - mm[ri]) * inv[ri] : 0.f;
            if (p.probs_fp32) probs_f[(prow0 + 8 * ri) * p.p_ld + j] = pr;
            else probs_h[(prow0 + 8 * ri) * p.p_ld + j] = __float2bfloat16(pr);
          }
        }
      }
    }
    // end of a sweep: combine each row over its quad
    if (sweep == 0) {
#pragma unroll
      for (int ri = 0; ri < 2; ++ri) {
        m[ri] = fmaxf(m[ri], __shfl_xor_sync(0xffffffffu, m[ri], 1));
        m[ri] = fmaxf(m[ri], __shfl_xor_sync(0xffffffffu, m[ri], 2));
        mm[ri] = m[ri] == -INFINITY ? 0.f : m[ri];
      }
    } else if (sweep == 1) {
#pragma unroll
      for (int ri = 0; ri < 2; ++ri) {
        sum[ri] += __shfl_xor_sync(0xffffffffu, sum[ri], 1);
        sum[ri] += __shfl_xor_sync(0xffffffffu, sum[ri], 2);
        inv[ri] = sum[ri] > 0.f ? 1.f / sum[ri] : 0.f;
        if (qd == 0 && row_ok[ri]) {
          const int64_t pr = prow0 + 8 * ri;
          if (p.lse != nullptr) p.lse[pr] = sum[ri] > 0.f ? (mm[ri] + log2f(sum[ri])) * 0.6931471805599453f : -INFINITY;
          if (p.inv_l != nullptr) p.inv_l[pr] = inv[ri];
        }
      }
    } else if (p.causal) {  // probabilities right of the last visible block
#pragma unroll
      for (int ri = 0; ri < 2; ++ri)
        if (row_ok[ri])
          for (int j = nkb * FL_T + qd; j < (int)p.p_ld; j += 4) {
            if (p.probs_fp32) probs_f[(prow0 + 8 * ri) * p.p_ld + j] = 0.f;
            else probs_h[(prow0 + 8 * ri) * p.p_ld + j] = __float2bfloat16(0.f);
          }
    }
  }
  // ---- epilogue: O / rowsum straight from the fragments
#pragma unroll
  for (int ri = 0; ri < 2; ++ri) {
    if (!row_ok[ri]) continue;
    const int i = i0 + r0 + 8 * ri;
    float* d32 = p.out_f32 != nullptr ? p.out_f32 + ((int64_t)b * p.Tq + i) * (p.H * 64) + h * 64 + 2 * qd : nullptr;
    __nv_bfloat16* dst = p.out + (int64_t)b * p.o_bs + (int64_t)i * p.o_ld + h * 64 + 2 * qd;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      const float v0 = o[4 * c + 2 * ri] * inv[ri], v1 = o[4 * c + 2 * ri + 1] * inv[ri];
      if (d32 != nullptr) *reinterpret_cast<float2*>(d32 + 8 * c) = make_float2(v0, v1);
      *reinterpret_cast<uint32_t*>(dst + 8 * c) = fl_pack(v0, v1);
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
  dim3 grid(((a->Tq + FL_T - 1) / FL_T + 1) / 2, a->H, a->B);  // two query tiles per CTA
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
