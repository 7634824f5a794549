// Fused attention backward on the Hopper tensor cores (wgmma). The probabilities come from the forward pass -- bf16
// exp(s - rowmax) with the dropout decision in the sign bit, normalised here by the saved 1/rowsum -- so one step needs
// a single score-sized MMA, no exponential and no random numbers.
//
// One CTA per (head, utterance). Loop: key block kb (64 keys) outer, query tile qt (64 rows) inner; step it:
//   MMA warpgroup  dP = dO_qt V_kb^T -> shared memory (fp32 rows)
//   threads        (4 warps, 1 thread = 1 query row x 32 keys): dS = P * (dP_masked + dP_ext - delta);
//                  dropout(P) and dS -> shared memory tiles (bf16, 128B-swizzled [q][key])
//   MMA warpgroup  dV_kb += dropout(P)^T dO_qt, dK_kb += dS^T Q_qt (registers, the tiles read MN-major),
//                  dQ_qt(kb) = dS K_kb -> fp32 accumulator in HBM straight from the fragments (plain RMW: the CTA owns
//                  its (b,h)), bf16 on the last key block; dK_kb / dV_kb after the last query tile of the block.
// Q / dO and the saved exponentials are double buffered: TMA fetches those of step it+1 while step it runs.
// Semantics: backward of speecht5/models/modules/multihead_attention.py:340-389. With relative positions the two table
// contractions dQ += dQP PE and dPE = dQP^T Q run on the batched GEMM from the dS written here.
#include "../../include/speecht5_b200.h"
#include "kernels.cuh"
#include "ptx.cuh"
#include "tma_map.cuh"

namespace st5 {

int set_error(int code, const char* where);

constexpr int FB_T = 64;                 // query tile == key block
constexpr int FB_THREADS = 9 * 32;       // MMA warpgroup, TMA warp, 4 compute warps
constexpr int FB_DPP = FB_T + 4;         // floats per row of the dP tile (row-per-lane float4 reads: conflict-free)
// K V | Q x2 | dO x2 | dropout(P) x2 | dS | dP | barriers
constexpr size_t FB_SMEM = 2 * 8192 + 4 * 8192 + 2 * 8192 + 8192 + (size_t)FB_T * FB_DPP * 4 + 256 + 1024;

struct FusedBwdParams {
  int B, H, Tq, Tk, causal;
  float scale, scale_log2;
  const uint8_t* key_pad;
  const float* inv_l; const float* delta;
  const float* dp_ext; long p_ld;
  __nv_bfloat16* dq; long q_ld, q_bs;
  __nv_bfloat16* dk; long k_ld, k_bs;
  __nv_bfloat16* dv; long v_ld, v_bs;
  float* dq_acc;  // [B][Tq][H*64] fp32 scratch
  const __nv_bfloat16* psave;  // [B][H][Tq][p_ld] from the forward pass: exp(s - rowmax), sign bit = dropped element
  __nv_bfloat16* ds_out;          // optional [B][H][Tq][p_ld]: dS for the relative-position contractions
  float drop_scale;
  int ext_heads;  // dp_ext is non-zero only for heads < ext_heads
};

__device__ __forceinline__ uint32_t pack2(float a, float b) {
  __nv_bfloat162 t = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&t);
}

// delta[row] = sum_c dO*O (+ sum_j P*dP_ext): the softmax-backward row constant.
// Plain case: 8 lanes per (b,h,i) row (one 16-byte load of dO and O each), 4 rows per warp. With an external dP the
// row also needs sum_j P*dP_ext over Tk fp32 pairs: one warp per row.
__global__ void attn_delta_kernel(const __nv_bfloat16* __restrict__ dO, const __nv_bfloat16* __restrict__ O,
                                  const float* __restrict__ O32, long o_ld, long o_bs, const float* __restrict__ probs,
                                  const float* __restrict__ dpx, long p_ld, float* __restrict__ delta, int B, int H,
                                  int Tq, int Tk, int ext_heads) {
  pdl_sync();
  const int lane = threadIdx.x & 31;
  const int64_t nrows = (int64_t)B * H * Tq;
  const int64_t gw = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (dpx == nullptr) {
    const int64_t row = gw * 4 + (lane >> 3);
    float acc = 0.f;
    if (row < nrows) {
      const int i = (int)(row % Tq), h = (int)((row / Tq) % H), b = (int)(row / ((int64_t)Tq * H));
      const int64_t off = (int64_t)b * o_bs + (int64_t)i * o_ld + h * 64 + (lane & 7) * 8;
      const uint4 ua = *reinterpret_cast<const uint4*>(dO + off);
      const __nv_bfloat162* ha = reinterpret_cast<const __nv_bfloat162*>(&ua);
      if (O32 != nullptr) {  // the forward's un-rounded output: dS = P (dP - delta) cancels, delta must not carry bf16 error
        const float* o32 = O32 + ((int64_t)b * Tq + i) * (H * 64) + h * 64 + (lane & 7) * 8;
        const float4 o0 = *reinterpret_cast<const float4*>(o32), o1 = *reinterpret_cast<const float4*>(o32 + 4);
        const float2 a0 = __bfloat1622float2(ha[0]), a1 = __bfloat1622float2(ha[1]), a2 = __bfloat1622float2(ha[2]),
                     a3 = __bfloat1622float2(ha[3]);
        acc = a0.x * o0.x + a0.y * o0.y + a1.x * o0.z + a1.y * o0.w + a2.x * o1.x + a2.y * o1.y + a3.x * o1.z + a3.y * o1.w;
      } else {
        const uint4 uo = *reinterpret_cast<const uint4*>(O + off);
        const __nv_bfloat162* ho = reinterpret_cast<const __nv_bfloat162*>(&uo);
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const float2 a = __bfloat1622float2(ha[t]), o = __bfloat1622float2(ho[t]);
          acc += a.x * o.x + a.y * o.y;
        }
      }
    }
    acc += __shfl_xor_sync(0xffffffffu, acc, 1);
    acc += __shfl_xor_sync(0xffffffffu, acc, 2);
    acc += __shfl_xor_sync(0xffffffffu, acc, 4);
    if ((lane & 7) == 0 && row < nrows) delta[row] = acc;
    return;
  }
  const int64_t row = gw;
  if (row >= nrows) return;
  const int i = (int)(row % Tq), h = (int)((row / Tq) % H), b = (int)(row / ((int64_t)Tq * H));
  const bool ext = h < ext_heads;  // the caller's gradient on the probabilities is zero for the other heads (contract)
  const int64_t off = (int64_t)b * o_bs + (int64_t)i * o_ld + h * 64 + lane * 2;
  const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(dO + off));
  float2 o;
  if (O32 != nullptr) o = *reinterpret_cast<const float2*>(O32 + ((int64_t)b * Tq + i) * (H * 64) + h * 64 + lane * 2);
  else o = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(O + off));
  float acc = a.x * o.x + a.y * o.y;
  const float* pr = probs + row * p_ld;
  const float* dx = dpx + row * p_ld;
  if (ext)
    for (int j = lane; j < Tk; j += 32) acc += pr[j] * dx[j];
  acc = warp_sum(acc);
  if (lane == 0) delta[row] = acc;
}

// delta[b][h][i] += sum_j P[b][h][i][j] * dP_ext[b][h][i][j] for the heads that carry an external gradient on their
// probabilities (h < ext_heads): one warp per (b, h < ext_heads, i) row. With the guided-attention loss that is 2 of 12
// heads -- the other rows take the 8-lanes-per-row path of attn_delta_kernel and are not visited here.
__global__ void attn_delta_ext_kernel(const float* __restrict__ probs, const float* __restrict__ dpx, long p_ld,
                                      float* __restrict__ delta, int B, int H, int Tq, int Tk, int ext_heads) {
  pdl_sync();
  const int lane = threadIdx.x & 31;
  const int64_t w = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (w >= (int64_t)B * ext_heads * Tq) return;
  const int i = (int)(w % Tq), h = (int)((w / Tq) % ext_heads), b = (int)(w / ((int64_t)Tq * ext_heads));
  const int64_t row = ((int64_t)b * H + h) * Tq + i;
  const float* pr = probs + row * p_ld;
  const float* dx = dpx + row * p_ld;
  float acc = 0.f;
  for (int j = lane; j < Tk; j += 32) acc += pr[j] * dx[j];
  acc = warp_sum(acc);
  if (lane == 0) delta[row] += acc;
}

__global__ void __launch_bounds__(FB_THREADS, 1)
    attn_fused_bwd_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k,
                          const __grid_constant__ CUtensorMap map_v, const __grid_constant__ CUtensorMap map_do,
                          const __grid_constant__ CUtensorMap map_p, const FusedBwdParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sK = smem;             // [64 keys][128 B]
  uint8_t* sV = sK + 8192;
  uint8_t* sQ = sV + 8192;        // 2 x [64 rows][128 B]
  uint8_t* sdO = sQ + 16384;      // 2 x [64 rows][128 B]
  uint8_t* sPd = sdO + 16384;     // 2 x [64 rows][64 keys]: the saved exponentials, overwritten in place by dropout(P)
  uint8_t* sdS = sPd + 16384;     // [64 rows][64 keys]
  float* sDP = reinterpret_cast<float*>(sdS + 8192);  // [64][FB_DPP]
  uint64_t* bar_kv = reinterpret_cast<uint64_t*>(sDP + FB_T * FB_DPP);  // K/V of a key block landed
  uint64_t* bar_kvfree = bar_kv + 1;  // every MMA that reads this key block's K/V tiles has completed
  uint64_t* bar_qdo = bar_kv + 2;     // [2] Q/dO buffer filled
  uint64_t* bar_qfree = bar_kv + 4;   // [2] Q/dO/exponential buffers consumed by the step's MMAs
  uint64_t* bar_pin = bar_kv + 6;     // [2] the saved exponentials of a step have landed in sPd[buf] (TMA)
  uint64_t* bar_dp = bar_kv + 8;      // dP of the step is in sDP
  uint64_t* bar_pds = bar_kv + 9;     // threads: dropout(P)/dS tiles written, dP read

  const int warp = threadIdx.x >> 5;
  const int h = blockIdx.x, b = blockIdx.y;
  const int nkb = (p.Tk + FB_T - 1) / FB_T, nqt = (p.Tq + FB_T - 1) / FB_T;

  if (warp == 4 && elect_one()) {
    tma_prefetch_desc(&map_q); tma_prefetch_desc(&map_k); tma_prefetch_desc(&map_v); tma_prefetch_desc(&map_do);
    tma_prefetch_desc(&map_p);
    mbar_init(bar_kv, 1); mbar_init(bar_kvfree, 1);
    for (int s = 0; s < 2; ++s) {
      mbar_init(&bar_qdo[s], 1); mbar_init(&bar_qfree[s], 1); mbar_init(&bar_pin[s], 1);
    }
    mbar_init(bar_dp, 128);
    mbar_init(bar_pds, 4);
    fence_mbar_init();
  }
  __syncthreads();
  pdl_sync();  // (prologue done: nothing above touched global memory)

  if (warp == 4) {
    // ===================== TMA producer =====================
    if (elect_one()) {
      int it = 0, kbc = 0;
      for (int kb = 0; kb < nkb; ++kb) {
        const int qt0 = p.causal ? kb : 0;
        for (int qt = qt0; qt < nqt; ++qt, ++it) {
          const int buf = it & 1;
          if (qt == qt0) {
            if (kbc > 0) mbar_wait_quiet(bar_kvfree, (uint32_t)((kbc - 1) & 1));  // MMAs of the previous key block are done
            ++kbc;
            mbar_expect_tx(bar_kv, 16384);
            tma_load_4d(sK, &map_k, bar_kv, 0, kb * FB_T, h, b);
            tma_load_4d(sV, &map_v, bar_kv, 0, kb * FB_T, h, b);
          }
          if (it >= 2) mbar_wait_quiet(&bar_qfree[buf], (uint32_t)(((it >> 1) - 1) & 1));  // step it-2 has read this buffer
          mbar_expect_tx(&bar_qdo[buf], 16384);
          tma_load_4d(sQ + buf * 8192, &map_q, &bar_qdo[buf], 0, qt * FB_T, h, b);
          tma_load_4d(sdO + buf * 8192, &map_do, &bar_qdo[buf], 0, qt * FB_T, h, b);
          // the saved exponentials of this (query tile, key block) go straight into the operand tile the threads will
          // overwrite in place with dropout(P): [64 rows][64 keys], 128B-swizzled
          mbar_expect_tx(&bar_pin[buf], 8192u);
          tma_load_4d(sPd + buf * 8192, &map_p, &bar_pin[buf], kb * FB_T, qt * FB_T, h, b);
        }
      }
    }
  } else if (warp < 4) {
    // ===================== MMA warpgroup =====================
    const uint32_t aK = smem_u32(sK), aV = smem_u32(sV), aQ0 = smem_u32(sQ), adO0 = smem_u32(sdO);
    const uint32_t aPd0 = smem_u32(sPd), adS = smem_u32(sdS);
    const int l = (int)lane_id(), w = warp;
    const int r0 = 16 * w + (l >> 2);  // fragment rows r0, r0 + 8; columns 8 (i >> 2) + 2 (l & 3) + (i & 1)
    float dk[32], dv[32];
#pragma unroll
    for (int t = 0; t < 32; ++t) dk[t] = dv[t] = 0.f;
    int it = 0, kbc = 0;
    for (int kb = 0; kb < nkb; ++kb) {
      const int qt0 = p.causal ? kb : 0;
      if (qt0 >= nqt) {  // causal, Tk > Tq: no query row sees the keys of this block, their gradients are zero
#pragma unroll
        for (int i = 0; i < 32; i += 2) {
          const int key = kb * FB_T + r0 + 8 * ((i >> 1) & 1), col = 8 * (i >> 2) + 2 * (l & 3);
          if (key < p.Tk) {
            *reinterpret_cast<uint32_t*>(p.dk + (int64_t)b * p.k_bs + (int64_t)key * p.k_ld + h * 64 + col) = 0u;
            *reinterpret_cast<uint32_t*>(p.dv + (int64_t)b * p.v_bs + (int64_t)key * p.v_ld + h * 64 + col) = 0u;
          }
        }
        continue;
      }
      mbar_wait_quiet(bar_kv, (uint32_t)(kbc & 1));
      ++kbc;
      for (int qt = qt0; qt < nqt; ++qt, ++it) {
        const int buf = it & 1;
        const uint32_t aQ = aQ0 + (uint32_t)buf * 8192u, adO = adO0 + (uint32_t)buf * 8192u;
        const uint32_t aPd = aPd0 + (uint32_t)buf * 8192u;
        mbar_wait_quiet(&bar_qdo[buf], (uint32_t)((it >> 1) & 1));
        {  // dP = dO V^T (A = dO, B = V: both K-major over the head dimension)
          float dp[32];
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < 4; ++k)
            wgmma_m64n64<0, 0>(dp, wgmma_smem_desc(adO + k * 32, 16, 1024), wgmma_smem_desc(aV + k * 32, 16, 1024),
                               k != 0 ? 1u : 0u);
          wgmma_commit();
          wgmma_wait<0>();
          wgmma_fence_regs(dp);
#pragma unroll
          for (int i = 0; i < 32; i += 2) {
            const int rr = r0 + 8 * ((i >> 1) & 1), cc = 8 * (i >> 2) + 2 * (l & 3);
            *reinterpret_cast<float2*>(sDP + rr * FB_DPP + cc) = make_float2(dp[i], dp[i + 1]);
          }
        }
        mbar_arrive(bar_dp);
        mbar_wait_quiet(bar_pds, (uint32_t)(it & 1));
        float dq[32];
        wgmma_fence();
        const uint32_t acc = qt != qt0;
#pragma unroll
        for (int k = 0; k < 4; ++k) {  // contraction over the 64 query rows: A = P^T / dS^T, B = dO / Q (all MN-major)
          wgmma_m64n64<1, 1>(dv, wgmma_smem_desc(aPd + k * 2048, 8192, 1024), wgmma_smem_desc(adO + k * 2048, 8192, 1024),
                             acc | (uint32_t)(k != 0));
          wgmma_m64n64<1, 1>(dk, wgmma_smem_desc(adS + k * 2048, 8192, 1024), wgmma_smem_desc(aQ + k * 2048, 8192, 1024),
                             acc | (uint32_t)(k != 0));
        }
#pragma unroll
        for (int k = 0; k < 4; ++k)  // contraction over the 64 keys: A = dS (K-major), B = K (MN-major)
          wgmma_m64n64<0, 1>(dq, wgmma_smem_desc(adS + k * 32, 16, 1024), wgmma_smem_desc(aK + k * 2048, 8192, 1024),
                             k != 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(dq);
        wgmma_fence_regs(dk);
        wgmma_fence_regs(dv);
        if (threadIdx.x == 0) {
          mbar_arrive(&bar_qfree[buf]);
          if (qt == nqt - 1) mbar_arrive(bar_kvfree);
        }
        // ---- dQ partial of (kb, qt): running fp32 sum over the key blocks, bf16 after the last one
        const int kb_last = p.causal ? (qt < nkb - 1 ? qt : nkb - 1) : nkb - 1;
#pragma unroll
        for (int i = 0; i < 32; i += 2) {
          const int row = qt * FB_T + r0 + 8 * ((i >> 1) & 1), col = 8 * (i >> 2) + 2 * (l & 3);
          if (row < p.Tq) {
            float2 f = make_float2(dq[i] * p.scale, dq[i + 1] * p.scale);
            float* accp = p.dq_acc + ((int64_t)b * p.Tq + row) * (p.H * 64) + h * 64 + col;
            if (kb > 0) {
              const float2 o = *reinterpret_cast<const float2*>(accp);
              f.x += o.x; f.y += o.y;
            }
            if (kb == kb_last)
              *reinterpret_cast<uint32_t*>(p.dq + (int64_t)b * p.q_bs + (int64_t)row * p.q_ld + h * 64 + col) = pack2(f.x, f.y);
            else
              *reinterpret_cast<float2*>(accp) = f;
          }
        }
        if (qt == nqt - 1) {  // dK / dV of the key block
#pragma unroll
          for (int i = 0; i < 32; i += 2) {
            const int key = kb * FB_T + r0 + 8 * ((i >> 1) & 1), col = 8 * (i >> 2) + 2 * (l & 3);
            if (key < p.Tk) {
              *reinterpret_cast<uint32_t*>(p.dk + (int64_t)b * p.k_bs + (int64_t)key * p.k_ld + h * 64 + col) =
                  pack2(dk[i] * p.scale, dk[i + 1] * p.scale);
              *reinterpret_cast<uint32_t*>(p.dv + (int64_t)b * p.v_bs + (int64_t)key * p.v_ld + h * 64 + col) =
                  pack2(dv[i], dv[i + 1]);
            }
          }
        }
      }
    }
  } else {
    // ===================== compute threads (thread = query row x 32-key chunk) =====================
    const int sw = warp - 5;
    const int q = sw & 1;
    const int c = sw >> 1;  // this warp's 32-key chunk of the block
    const int r = q * 32 + (int)lane_id();
    const int cbase = c * 4;
    int it = 0;
    for (int kb = 0; kb < nkb; ++kb) {
      const int qt0 = p.causal ? kb : 0;
      const int k0 = kb * FB_T;
      for (int qt = qt0; qt < nqt; ++qt, ++it) {
        const int buf = it & 1;
        const int i = qt * FB_T + r;
        const bool row_ok = i < p.Tq;
        const int64_t prow = ((int64_t)b * p.H + h) * p.Tq + i;
        const float delta = row_ok ? p.delta[prow] : 0.f, invl = row_ok ? p.inv_l[prow] : 0.f;
        const float* dpx = (p.dp_ext != nullptr && row_ok && h < p.ext_heads) ? p.dp_ext + prow * p.p_ld : nullptr;
        const int col0 = k0 + c * 32;
        mbar_wait_quiet(bar_dp, (uint32_t)(it & 1));
        mbar_wait_quiet(&bar_pin[buf], (uint32_t)((it >> 1) & 1));  // the exponentials are in sPd[buf] (every warp:
                                                                    // nobody may write the tile before the TMA has)
        uint8_t* bp = sPd + buf * 8192 + r * 128;
        uint8_t* bs = sdS + r * 128;
        // warp-uniform fast path: no live query row in this warp's 32 rows, or the whole key chunk lies beyond Tk --
        // P is zero there, so both operand tiles get zeros (they are contracted over, so they must be written)
        const bool dead = (qt * FB_T + q * 32 >= p.Tq) || (col0 >= p.Tk);
        if (dead) {
#pragma unroll
          for (int g = 0; g < 4; ++g) {
            const int swz = ((cbase + g) ^ (r & 7)) << 4;
            *reinterpret_cast<uint4*>(bp + swz) = make_uint4(0u, 0u, 0u, 0u);
            *reinterpret_cast<uint4*>(bs + swz) = make_uint4(0u, 0u, 0u, 0u);
            if (p.ds_out != nullptr && row_ok && col0 + 8 * g + 8 <= p.p_ld)
              *reinterpret_cast<uint4*>(p.ds_out + prow * p.p_ld + col0 + 8 * g) = make_uint4(0u, 0u, 0u, 0u);
          }
        } else {
        // (dP is finite everywhere: V rows beyond Tk and dO rows beyond Tq arrive as zeros from TMA)
        float dvv[32];
        {
          const float* src = sDP + r * FB_DPP + c * 32;
#pragma unroll
          for (int t = 0; t < 32; t += 4) {
            const float4 f = *reinterpret_cast<const float4*>(src + t);
            dvv[t] = f.x; dvv[t + 1] = f.y; dvv[t + 2] = f.z; dvv[t + 3] = f.w;
          }
        }
#pragma unroll
        for (int g = 0; g < 4; ++g) {
          const int swz = ((cbase + g) ^ (r & 7)) << 4;
          const uint4 praw = *reinterpret_cast<const uint4*>(bp + swz);  // this row's 8 saved exponentials (in place)
          const uint32_t w4[4] = {praw.x, praw.y, praw.z, praw.w};
          float xd[8];
          xd[0] = xd[1] = xd[2] = xd[3] = xd[4] = xd[5] = xd[6] = xd[7] = 0.f;
          if (dpx != nullptr) {  // the caller's gradient on the probabilities: this row's 8 floats of the chunk (keys
                                 // < Tk only: the padding columns [Tk, p_ld) are not part of the contract)
            if ((p.p_ld & 3) == 0 && (reinterpret_cast<uintptr_t>(p.dp_ext) & 15) == 0 && col0 + 8 * g + 8 <= p.Tk) {
              const float4 x0 = __ldg(reinterpret_cast<const float4*>(dpx + col0 + 8 * g));
              const float4 x1 = __ldg(reinterpret_cast<const float4*>(dpx + col0 + 8 * g + 4));
              xd[0] = x0.x; xd[1] = x0.y; xd[2] = x0.z; xd[3] = x0.w;
              xd[4] = x1.x; xd[5] = x1.y; xd[6] = x1.z; xd[7] = x1.w;
            } else {
#pragma unroll
              for (int t = 0; t < 8; ++t)
                if (col0 + 8 * g + t < p.Tk) xd[t] = dpx[col0 + 8 * g + t];
            }
          }
          float pd8[8], ds8[8];
#pragma unroll
          for (int e = 0; e < 4; ++e) {
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
              const int t = 2 * e + hh;
              const uint32_t raw = hh ? (w4[e] & 0xffff0000u) : (w4[e] << 16);  // bf16 -> fp32 bit pattern
              const float keepf = (int32_t)raw < 0 ? 0.f : p.drop_scale;      // sign bit = dropped by the forward pass
              const float pv = fabsf(__uint_as_float(raw)) * invl;           // the probability
              // dP as the softmax sees it: dropout backward of dO V^T, plus the caller's gradient
              const float dp = dvv[8 * g + t] * keepf + xd[t];
              pd8[t] = pv * keepf;
              ds8[t] = pv * (dp - delta);
            }
          }
          uint4 a, d;
          a.x = pack2(pd8[0], pd8[1]); a.y = pack2(pd8[2], pd8[3]); a.z = pack2(pd8[4], pd8[5]); a.w = pack2(pd8[6], pd8[7]);
          d.x = pack2(ds8[0], ds8[1]); d.y = pack2(ds8[2], ds8[3]); d.z = pack2(ds8[4], ds8[5]); d.w = pack2(ds8[6], ds8[7]);
          *reinterpret_cast<uint4*>(bp + swz) = a;
          *reinterpret_cast<uint4*>(bs + swz) = d;
          if (p.ds_out != nullptr && row_ok && col0 + 8 * g + 8 <= p.p_ld)
            *reinterpret_cast<uint4*>(p.ds_out + prow * p.p_ld + col0 + 8 * g) = d;
        }
        }
        fence_proxy_async();
        __syncwarp();
        if (lane_id() == 0) mbar_arrive(bar_pds);
      }
    }
  }
}

static int make_map64(CUtensorMap* m, const void* ptr, int64_t rows, int64_t ld, int64_t bs, int H, int B) {
  const uint64_t dims[4] = {64, (uint64_t)rows, (uint64_t)H, (uint64_t)B};
  const uint64_t strides[3] = {(uint64_t)ld * 2, 128, (uint64_t)bs * 2};
  const uint32_t box[4] = {64, FB_T, 1, 1};
  return encode_bf16_map_4d(m, ptr, dims, strides, box);
}

}  // namespace st5

using namespace st5;

extern "C" int st5_attn_fused_bwd(const st5_attn_args* a, const void* psave, const float* inv_l, const float* out_f32,
                                  float* delta, float* dq_acc, int32_t ext_heads, void* stream) {
  const bool rpe = a->pe_k != nullptr;
  if (a->dtype != ST5_BF16 || a->Tk <= 0 || a->Tq <= 0) return set_error(-2, "st5_attn_fused_bwd: needs bf16");
  if (psave == nullptr || inv_l == nullptr || (a->p_ld & 7) || a->p_ld < a->Tk || (reinterpret_cast<uintptr_t>(psave) & 15))
    return set_error(-5, "st5_attn_fused_bwd: needs psave / inv_l written by st5_attn_fused_fwd (16-byte aligned, row "
                         "pitch a multiple of 8)");
  if (rpe && (a->ds == nullptr || a->dprobs_ext != nullptr || a->causal || (reinterpret_cast<uintptr_t>(a->ds) & 15)))
    return set_error(-5, "st5_attn_fused_bwd: relative positions need a dS buffer and take no external dP");
  if (a->dprobs_ext != nullptr && (a->probs_dtype != ST5_F32 || a->probs == nullptr))
    return set_error(-3, "st5_attn_fused_bwd: dprobs_ext needs the fp32 probabilities the forward returned");
  if (!a->dout || !a->out || !a->dq || !a->dk || !a->dv || !delta || !dq_acc)
    return set_error(-4, "st5_attn_fused_bwd: null argument");
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t nrows = (int64_t)a->B * a->H * a->Tq;
  const bool ext = a->dprobs_ext != nullptr;
  if (!ext && ((a->o_ld & 7) || (a->o_bs & 7) || (reinterpret_cast<uintptr_t>(a->dout) & 15) ||
               (reinterpret_cast<uintptr_t>(a->out) & 15)))
    return set_error(-4, "st5_attn_fused_bwd: out / dout must be 16-byte aligned");
  const int eh = ext_heads > 0 && ext_heads < a->H ? ext_heads : a->H;
  // external dP on a few heads only (and vector-loadable outputs): every row takes the cheap dO.O path, a second small
  // launch adds sum_j P dP_ext on the rows of those heads only
  const bool split = ext && eh < a->H && !((a->o_ld & 7) || (a->o_bs & 7) || (reinterpret_cast<uintptr_t>(a->dout) & 15) ||
                                           (reinterpret_cast<uintptr_t>(a->out) & 15));
  const int64_t warps_needed = (ext && !split) ? nrows : (nrows + 3) / 4;
  launch_pdl(attn_delta_kernel, dim3((unsigned)((warps_needed + 7) / 8)), dim3(256), 0, s, (const __nv_bfloat16*)a->dout,
             (const __nv_bfloat16*)a->out, out_f32, a->o_ld, a->o_bs,
             (ext && !split) ? (const float*)a->probs : (const float*)nullptr, split ? (const float*)nullptr : a->dprobs_ext,
             a->p_ld, delta, a->B, a->H, a->Tq, a->Tk, eh);
  if (split) {
    const int64_t wext = (int64_t)a->B * eh * a->Tq;
    launch_pdl(attn_delta_ext_kernel, dim3((unsigned)((wext + 7) / 8)), dim3(256), 0, s, (const float*)a->probs, a->dprobs_ext,
               a->p_ld, delta, a->B, a->H, a->Tq, a->Tk, eh);
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error((int)e, "st5_attn_fused_bwd(delta)");
  CUtensorMap mq, mk, mv, mdo, mp;
  int rc = make_map64(&mq, a->q, a->Tq, a->q_ld, a->q_bs, a->H, a->B);
  if (!rc) rc = make_map64(&mk, a->k, a->Tk, a->k_ld, a->k_bs, a->H, a->B);
  if (!rc) rc = make_map64(&mv, a->v, a->Tk, a->v_ld, a->v_bs, a->H, a->B);
  if (!rc) rc = make_map64(&mdo, a->dout, a->Tq, a->o_ld, a->o_bs, a->H, a->B);
  if (!rc) {  // psave [B][H][Tq][p_ld] bf16: boxes of 64 keys x 64 query rows, out-of-range rows / columns read as zero
    const uint64_t dims[4] = {(uint64_t)a->p_ld, (uint64_t)a->Tq, (uint64_t)a->H, (uint64_t)a->B};
    const uint64_t strides[3] = {(uint64_t)a->p_ld * 2, (uint64_t)a->Tq * a->p_ld * 2, (uint64_t)a->H * a->Tq * a->p_ld * 2};
    const uint32_t box[4] = {64, FB_T, 1, 1};
    rc = encode_bf16_map_4d(&mp, psave, dims, strides, box);
  }
  if (rc) return set_error(rc, "st5_attn_fused_bwd: tensor map");
  static bool attr_set = false;
  if (!attr_set) {
    e = cudaFuncSetAttribute(attn_fused_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FB_SMEM);
    if (e != cudaSuccess) return set_error((int)e, "st5_attn_fused_bwd");
    attr_set = true;
  }
  FusedBwdParams p;
  p.B = a->B; p.H = a->H; p.Tq = a->Tq; p.Tk = a->Tk; p.causal = a->causal;
  p.scale = a->scale; p.scale_log2 = a->scale * 1.4426950408889634f;
  p.key_pad = a->key_pad; p.inv_l = inv_l; p.delta = delta;
  p.dp_ext = a->dprobs_ext; p.p_ld = a->p_ld;
  p.dq = (__nv_bfloat16*)a->dq; p.q_ld = a->q_ld; p.q_bs = a->q_bs;
  p.dk = (__nv_bfloat16*)a->dk; p.k_ld = a->k_ld; p.k_bs = a->k_bs;
  p.dv = (__nv_bfloat16*)a->dv; p.v_ld = a->v_ld; p.v_bs = a->v_bs;
  p.dq_acc = dq_acc;
  p.psave = reinterpret_cast<const __nv_bfloat16*>(psave);
  p.ds_out = rpe ? reinterpret_cast<__nv_bfloat16*>(a->ds) : nullptr;
  p.drop_scale = a->drop_p > 0.f ? 1.f / (1.f - a->drop_p) : 1.f;
  p.ext_heads = ext_heads > 0 ? ext_heads : a->H;
  launch_pdl(attn_fused_bwd_kernel, dim3(a->H, a->B), dim3(FB_THREADS), FB_SMEM, s, mq, mk, mv, mdo, mp, p);
  return set_error((int)cudaGetLastError(), "st5_attn_fused_bwd");
}
