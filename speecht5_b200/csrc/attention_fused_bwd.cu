// Fused attention backward on the Hopper tensor cores (wgmma). The probabilities come from the forward pass -- bf16
// exp(s - rowmax) with the dropout decision in the sign bit, normalised here by the saved 1/rowsum -- so one step needs
// a single score-sized MMA, no exponential and no random numbers.
//
// One CTA per (head, utterance), two MMA warpgroups: in round j, A owns key block 2j and B key block 2j+1 (dK / dV in
// registers); both walk the query tiles qt (64 rows; causal: from qt = 2j) over one shared Q / dO tile per step:
//   each warpgroup  dP = dO_qt V_kb^T (registers); on the fragments: dS = P * (dP_masked + dP_ext - delta) and
//                   dropout(P) -> its shared memory tiles (bf16, 128B-swizzled [q][key]);
//                   dQ_qt(kb) = dS K_kb, then dV_kb += dropout(P)^T dO_qt, dK_kb += dS^T Q_qt (tiles read MN-major).
//   dQ_qt          running fp32 sum over the key blocks in ascending order: A adds block 2j to the sum of the blocks
//                   before it (prefetched from the dq_acc scratch by the producer warp a step ahead), B adds 2j+1 and
//                   stores the sum back to dq_acc -- bf16 into dq after the last block that reaches the tile.
// While one warpgroup forms dS the other's MMAs run. Q / dO / the saved exponentials and the prefetched running sum
// are double buffered per step, K / V per round.
// Semantics: backward of speecht5/models/modules/multihead_attention.py:340-389. With relative positions the two table
// contractions dQ += dQP PE and dPE = dQP^T Q run on the batched GEMM from the dS written here.
#include "../../include/speecht5_b200.h"
#include "kernels.cuh"
#include "ptx.cuh"
#include "tma_map.cuh"

namespace st5 {

int set_error(int code, const char* where);

constexpr int FB_T = 64;                 // query tile == key block
constexpr int FB_THREADS = 9 * 32;       // MMA warpgroups A and B, TMA / prefetch warp
// K V x2 x2 | Q x2 | dO x2 | dropout(P) x2 x2 | dS x2 | dQ running sum x2 | dQ handoff | barriers
constexpr size_t FB_SMEM = 8 * 8192 + 2 * 8192 + 2 * 8192 + 4 * 8192 + 2 * 8192 + 2 * 16384 + 16384 + 256 + 1024;

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

// named barrier of one warpgroup (ids 1 and 2; 0 is __syncthreads)
__device__ __forceinline__ void wg_bar_sync(int g) {
  if (g == 0) asm volatile("bar.sync 1, 128;" ::: "memory");
  else asm volatile("bar.sync 2, 128;" ::: "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.cta.shared::cta.u32 %0, [%1];" : "=r"(v) : "r"(smem_u32(p)) : "memory");
  return v;
}
__device__ __forceinline__ void red_release_add(uint32_t* p, uint32_t v) {
  asm volatile("red.release.cta.shared::cta.add.u32 [%0], %1;" ::"r"(smem_u32(p)), "r"(v) : "memory");
}
__device__ __forceinline__ void cp_async8(void* dst, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
// the barrier receives this thread's arrival once all of its earlier cp.async copies have landed
__device__ __forceinline__ void cp_async_arrive(uint64_t* bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}

__global__ void __launch_bounds__(FB_THREADS, 1)
    attn_fused_bwd_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k,
                          const __grid_constant__ CUtensorMap map_v, const __grid_constant__ CUtensorMap map_do,
                          const __grid_constant__ CUtensorMap map_p, const FusedBwdParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sK = smem;             // [round buffer][warpgroup] x [64 keys][128 B]
  uint8_t* sV = sK + 4 * 8192;
  uint8_t* sQ = sV + 4 * 8192;    // [step buffer] x [64 rows][128 B]
  uint8_t* sdO = sQ + 2 * 8192;
  uint8_t* sP = sdO + 2 * 8192;   // [step buffer][warpgroup] x [64 rows][64 keys]: exponentials, overwritten by dropout(P)
  uint8_t* sdS = sP + 4 * 8192;   // [warpgroup] x [64 rows][64 keys]
  float2* sAcc = reinterpret_cast<float2*>(sdS + 2 * 8192);  // [step buffer] x [16][128]: dQ running sum, fragment order
  float2* sX = sAcc + 2 * 2048;                              // [16][128]: warpgroup A's partial dQ sum for B
  uint64_t* bar_kv = reinterpret_cast<uint64_t*>(sX + 2048);  // [2] K/V of a round landed
  uint64_t* bar_kvfree = bar_kv + 2;   // [2] both warpgroups are done with a round's K/V buffer
  uint64_t* bar_qdo = bar_kv + 4;      // [2] Q, dO and both exponential tiles of a step landed
  uint64_t* bar_qfree = bar_kv + 6;    // [2] both warpgroups' MMAs of the step have completed
  uint64_t* bar_acc = bar_kv + 8;      // [2] dQ running sum of the step is in sAcc
  uint64_t* bar_accfree = bar_kv + 10; // [2] warpgroup A has read sAcc
  uint64_t* bar_x = bar_kv + 12;       // sX written by A
  uint64_t* bar_xfree = bar_kv + 13;   // sX read by B
  uint32_t* acc_done = reinterpret_cast<uint32_t*>(bar_kv + 14);  // 4 x steps B has finished (dq_acc stored)

  const int warp = threadIdx.x >> 5;
  const int h = blockIdx.x, b = blockIdx.y;
  const int nkb = (p.Tk + FB_T - 1) / FB_T, nqt = (p.Tq + FB_T - 1) / FB_T;

  if (warp == 8 && elect_one()) {
    tma_prefetch_desc(&map_q); tma_prefetch_desc(&map_k); tma_prefetch_desc(&map_v); tma_prefetch_desc(&map_do);
    tma_prefetch_desc(&map_p);
    for (int s = 0; s < 2; ++s) {
      mbar_init(&bar_kv[s], 1); mbar_init(&bar_kvfree[s], 2);
      mbar_init(&bar_qdo[s], 1); mbar_init(&bar_qfree[s], 2);
      mbar_init(&bar_acc[s], 32); mbar_init(&bar_accfree[s], 128);
    }
    mbar_init(bar_x, 128); mbar_init(bar_xfree, 128);
    *acc_done = 0u;
    fence_mbar_init();
  }
  __syncthreads();
  pdl_sync();  // (prologue done: nothing above touched global memory)

  if (warp == 8) {
    // ===================== TMA producer + dQ running-sum prefetch =====================
    const int lane = (int)lane_id();
    int s = 0, rc = 0;
    for (int j = 0; 2 * j < nkb; ++j) {
      const int qt0 = p.causal ? 2 * j : 0;
      if (qt0 >= nqt) break;  // causal, Tk > Tq: no later round has a step either
      const bool hasB = 2 * j + 1 < nkb;
      const int kbuf = rc & 1;
      if (lane == 0) {
        if (rc >= 2) mbar_wait_quiet(&bar_kvfree[kbuf], (uint32_t)(((rc >> 1) - 1) & 1));
        mbar_expect_tx(&bar_kv[kbuf], hasB ? 32768u : 16384u);
        tma_load_4d(sK + (2 * kbuf) * 8192, &map_k, &bar_kv[kbuf], 0, 2 * j * FB_T, h, b);
        tma_load_4d(sV + (2 * kbuf) * 8192, &map_v, &bar_kv[kbuf], 0, 2 * j * FB_T, h, b);
        if (hasB) {
          tma_load_4d(sK + (2 * kbuf + 1) * 8192, &map_k, &bar_kv[kbuf], 0, (2 * j + 1) * FB_T, h, b);
          tma_load_4d(sV + (2 * kbuf + 1) * 8192, &map_v, &bar_kv[kbuf], 0, (2 * j + 1) * FB_T, h, b);
        }
      }
      ++rc;
      for (int qt = qt0; qt < nqt; ++qt, ++s) {
        const int buf = s & 1;
        const bool bOn = hasB && (!p.causal || qt > 2 * j);  // key block 2j+1 reaches this query tile
        if (lane == 0) {
          if (s >= 2) mbar_wait_quiet(&bar_qfree[buf], (uint32_t)(((s >> 1) - 1) & 1));  // step s-2 is done with it
          mbar_expect_tx(&bar_qdo[buf], bOn ? 32768u : 24576u);
          tma_load_4d(sQ + buf * 8192, &map_q, &bar_qdo[buf], 0, qt * FB_T, h, b);
          tma_load_4d(sdO + buf * 8192, &map_do, &bar_qdo[buf], 0, qt * FB_T, h, b);
          tma_load_4d(sP + (2 * buf) * 8192, &map_p, &bar_qdo[buf], 2 * j * FB_T, qt * FB_T, h, b);
          if (bOn) tma_load_4d(sP + (2 * buf + 1) * 8192, &map_p, &bar_qdo[buf], (2 * j + 1) * FB_T, qt * FB_T, h, b);
        }
        __syncwarp();
        if (s >= 2) mbar_wait_quiet(&bar_accfree[buf], (uint32_t)(((s >> 1) - 1) & 1));
        if (j > 0) {
          // The running sum of this tile was stored to dq_acc by warpgroup B in step (j-1, qt), nqt - qt0 steps back:
          // wait until B has counted that step (release after its stores), then copy the tile in fragment order.
          const uint32_t need = 4u * (uint32_t)(s - (nqt - qt0) + 1);
          if (ld_acquire_u32(acc_done) < need) {
            const long long t0 = clock64();
            while (ld_acquire_u32(acc_done) < need)
              if (clock64() - t0 > 4000000000LL) __trap();
          }
          float2* dst = sAcc + buf * 2048;
#pragma unroll 4
          for (int w = 0; w < 4; ++w)
#pragma unroll
            for (int i2 = 0; i2 < 16; ++i2) {
              const int row = qt * FB_T + 16 * w + (lane >> 2) + 8 * (i2 & 1), col = 8 * (i2 >> 1) + 2 * (lane & 3);
              if (row < p.Tq)
                cp_async8(dst + i2 * 128 + w * 32 + lane, p.dq_acc + ((int64_t)b * p.Tq + row) * (p.H * 64) + h * 64 + col);
            }
        }
        cp_async_arrive(&bar_acc[buf]);
      }
    }
    asm volatile("cp.async.wait_all;" ::: "memory");
  } else {
    // ===================== MMA warpgroups: A (g = 0) even key blocks, B (g = 1) odd ones =====================
    const int g = warp >> 2;
    const int tid = threadIdx.x & 127;
    const int l = (int)lane_id(), w = warp & 3;
    const int r0 = 16 * w + (l >> 2);  // fragment rows r0, r0 + 8; columns 8 (i >> 2) + 2 (l & 3) + (i & 1)
    const uint32_t aQ0 = smem_u32(sQ), adO0 = smem_u32(sdO), adS = smem_u32(sdS + g * 8192);
    uint8_t* tS = sdS + g * 8192;
    float dk[32], dv[32];
#pragma unroll
    for (int t = 0; t < 32; ++t) dk[t] = dv[t] = 0.f;
    int s = 0, rc = 0, nx = 0;
    for (int j = 0; 2 * j < nkb; ++j) {
      const int kb = 2 * j + g;
      const int qt0 = p.causal ? 2 * j : 0;
      const int qtm = p.causal ? kb : 0;  // first query tile this warpgroup's key block reaches
      const bool active = kb < nkb && qtm < nqt;
      if (qt0 < nqt) {
        const int kbuf = rc & 1;
        if (active) mbar_wait_quiet(&bar_kv[kbuf], (uint32_t)((rc >> 1) & 1));
        ++rc;
        const uint32_t aK = smem_u32(sK + (2 * kbuf + g) * 8192), aV = smem_u32(sV + (2 * kbuf + g) * 8192);
        for (int qt = qt0; qt < nqt; ++qt, ++s) {
          const int buf = s & 1;
          if (kb < nkb && qt >= qtm) {
            const uint32_t aQ = aQ0 + (uint32_t)buf * 8192u, adO = adO0 + (uint32_t)buf * 8192u;
            uint8_t* tP = sP + (2 * buf + g) * 8192;
            const uint32_t aP = smem_u32(tP);
            const int i0 = qt * FB_T + r0;
            const bool ok0 = i0 < p.Tq, ok1 = i0 + 8 < p.Tq;
            const int64_t prow0 = ((int64_t)b * p.H + h) * p.Tq + i0;
            const float invl0 = ok0 ? p.inv_l[prow0] : 0.f, delta0 = ok0 ? p.delta[prow0] : 0.f;
            const float invl1 = ok1 ? p.inv_l[prow0 + 8] : 0.f, delta1 = ok1 ? p.delta[prow0 + 8] : 0.f;
            mbar_wait_quiet(&bar_qdo[buf], (uint32_t)((s >> 1) & 1));
            float dp[32];
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k)  // dP = dO V^T (A = dO, B = V: both K-major over the head dimension)
              wgmma_m64n64<0, 0>(dp, wgmma_smem_desc(adO + k * 32, 16, 1024), wgmma_smem_desc(aV + k * 32, 16, 1024),
                                 k != 0 ? 1u : 0u);
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_regs(dp);
            // ---- softmax gradient on the fragment: dropout(P) in place of the exponentials, dS into its own tile.
            // Rows beyond Tq / keys beyond Tk in a live 32 x 32 quadrant compute to zero (their exponentials, dO and
            // V rows arrive as zeros); a quadrant with no live row or key is written as +0 without being read.
            const bool rows_dead = qt * FB_T + (w >= 2 ? 32 : 0) >= p.Tq;
            const bool ext = p.dp_ext != nullptr && h < p.ext_heads;
            const float* dpx0 = ext && ok0 ? p.dp_ext + prow0 * p.p_ld : nullptr;
            const float* dpx1 = ext && ok1 ? p.dp_ext + (prow0 + 8) * p.p_ld : nullptr;
            const bool x_vec = (reinterpret_cast<uintptr_t>(p.dp_ext) & 7) == 0;
#pragma unroll
            for (int i = 0; i < 32; i += 2) {
              const int hr = (i >> 1) & 1;
              const int rr = r0 + 8 * hr, key = kb * FB_T + 8 * (i >> 2) + 2 * (l & 3);
              const int off = rr * 128 + ((((i >> 2) ^ (l >> 2)) << 4) | ((l & 3) << 2));  // 128B swizzle
              uint32_t pdw = 0u, dsw = 0u;
              if (!rows_dead && kb * FB_T + (i >= 16 ? 32 : 0) < p.Tk) {
                const uint32_t e2 = *reinterpret_cast<const uint32_t*>(tP + off);  // two saved exponentials
                const float* dpx = hr ? dpx1 : dpx0;
                float xd0 = 0.f, xd1 = 0.f;
                if (dpx != nullptr) {  // the caller's gradient on the probabilities (keys < Tk only)
                  if (x_vec && key + 1 < p.Tk) {
                    const float2 x = __ldg(reinterpret_cast<const float2*>(dpx + key));
                    xd0 = x.x; xd1 = x.y;
                  } else {
                    if (key < p.Tk) xd0 = dpx[key];
                    if (key + 1 < p.Tk) xd1 = dpx[key + 1];
                  }
                }
                const float invl = hr ? invl1 : invl0, delta = hr ? delta1 : delta0;
                const uint32_t raw0 = e2 << 16, raw1 = e2 & 0xffff0000u;  // bf16 -> fp32 bit patterns
                const float keep0 = (int32_t)raw0 < 0 ? 0.f : p.drop_scale;  // sign bit = dropped by the forward pass
                const float keep1 = (int32_t)raw1 < 0 ? 0.f : p.drop_scale;
                const float pv0 = fabsf(__uint_as_float(raw0)) * invl, pv1 = fabsf(__uint_as_float(raw1)) * invl;
                // dP as the softmax sees it: dropout backward of dO V^T, plus the caller's gradient
                const float dp0 = dp[i] * keep0 + xd0, dp1 = dp[i + 1] * keep1 + xd1;
                pdw = pack2(pv0 * keep0, pv1 * keep1);
                dsw = pack2(pv0 * (dp0 - delta), pv1 * (dp1 - delta));
              }
              *reinterpret_cast<uint32_t*>(tP + off) = pdw;
              *reinterpret_cast<uint32_t*>(tS + off) = dsw;
              if (p.ds_out != nullptr && (hr ? ok1 : ok0) && key < p.p_ld)
                *reinterpret_cast<uint32_t*>(p.ds_out + (prow0 + 8 * hr) * p.p_ld + key) = dsw;
            }
            fence_proxy_async();
            wg_bar_sync(g);  // the whole warpgroup's tiles are written before its MMAs read them
            float dq[32];
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k)  // contraction over the 64 keys: A = dS (K-major), B = K (MN-major)
              wgmma_m64n64<0, 1>(dq, wgmma_smem_desc(adS + k * 32, 16, 1024), wgmma_smem_desc(aK + k * 2048, 8192, 1024),
                                 k != 0 ? 1u : 0u);
            wgmma_commit();
            const uint32_t acc = qt != qtm;
#pragma unroll
            for (int k = 0; k < 4; ++k) {  // contraction over the 64 query rows: A = P^T / dS^T, B = dO / Q (MN-major)
              wgmma_m64n64<1, 1>(dv, wgmma_smem_desc(aP + k * 2048, 8192, 1024), wgmma_smem_desc(adO + k * 2048, 8192, 1024),
                                 acc | (uint32_t)(k != 0));
              wgmma_m64n64<1, 1>(dk, wgmma_smem_desc(adS + k * 2048, 8192, 1024), wgmma_smem_desc(aQ + k * 2048, 8192, 1024),
                                 acc | (uint32_t)(k != 0));
            }
            wgmma_commit();
            wgmma_wait<1>();  // dQ is ready; dV / dK keep the tensor pipe busy meanwhile
            wgmma_fence_regs(dq);
            // ---- dQ of (kb, qt): running fp32 sum over the key blocks in ascending order, bf16 after the last one.
            // A adds the sum of blocks < 2j (prefetched) and hands it to B, which adds block 2j+1 and stores it --
            // unless 2j is the last block that reaches the tile, then A stores.
            const int kb_last = p.causal ? (qt < nkb - 1 ? qt : nkb - 1) : nkb - 1;
            const bool last = kb == kb_last;
            const float2* src;
            if (g == 0) {
              mbar_wait_quiet(&bar_acc[buf], (uint32_t)((s >> 1) & 1));
              src = sAcc + buf * 2048 + tid;
              if (!last && nx > 0) mbar_wait_quiet(bar_xfree, (uint32_t)((nx - 1) & 1));
            } else {
              mbar_wait_quiet(bar_x, (uint32_t)(nx & 1));
              src = sX + tid;
            }
            const bool add = g == 1 || kb > 0;
            const bool keep = g == 0 && !last;
#pragma unroll
            for (int i = 0; i < 32; i += 2) {
              const int row = qt * FB_T + r0 + 8 * ((i >> 1) & 1), col = 8 * (i >> 2) + 2 * (l & 3);
              float2 f = make_float2(dq[i] * p.scale, dq[i + 1] * p.scale);
              if (add) {
                const float2 o = src[(i >> 1) * 128];
                f.x += o.x; f.y += o.y;
              }
              if (keep) {
                sX[(i >> 1) * 128 + tid] = f;
              } else if (row < p.Tq) {
                if (last)
                  *reinterpret_cast<uint32_t*>(p.dq + (int64_t)b * p.q_bs + (int64_t)row * p.q_ld + h * 64 + col) =
                      pack2(f.x, f.y);
                else
                  *reinterpret_cast<float2*>(p.dq_acc + ((int64_t)b * p.Tq + row) * (p.H * 64) + h * 64 + col) = f;
              }
            }
            if (g == 0) {
              mbar_arrive(&bar_accfree[buf]);
              if (!last) { mbar_arrive(bar_x); ++nx; }
            } else {
              mbar_arrive(bar_xfree); ++nx;
            }
            wgmma_wait<0>();
            wgmma_fence_regs(dk);
            wgmma_fence_regs(dv);
          } else {
            // B without a block for this tile still releases the step: not before the step's tiles have landed,
            // i.e. after step s-2 was released by both warpgroups -- its arrival must not complete an earlier phase
            mbar_wait_quiet(&bar_qdo[buf], (uint32_t)((s >> 1) & 1));
          }
          if (tid == 0) mbar_arrive(&bar_qfree[buf]);
          if (g == 1) {  // publish this step's dq_acc stores to the prefetching warp
            __threadfence_block();
            __syncwarp();
            if (l == 0) red_release_add(acc_done, 1u);
          }
        }
        if (tid == 0) mbar_arrive(&bar_kvfree[kbuf]);
      }
      if (kb < nkb) {  // dK / dV of the key block (zero when no query row sees it: causal, Tk > Tq)
#pragma unroll
        for (int i = 0; i < 32; i += 2) {
          const int key = kb * FB_T + r0 + 8 * ((i >> 1) & 1), col = 8 * (i >> 2) + 2 * (l & 3);
          if (key < p.Tk) {
            *reinterpret_cast<uint32_t*>(p.dk + (int64_t)b * p.k_bs + (int64_t)key * p.k_ld + h * 64 + col) =
                active ? pack2(dk[i] * p.scale, dk[i + 1] * p.scale) : 0u;
            *reinterpret_cast<uint32_t*>(p.dv + (int64_t)b * p.v_bs + (int64_t)key * p.v_ld + h * 64 + col) =
                active ? pack2(dv[i], dv[i + 1]) : 0u;
          }
        }
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
