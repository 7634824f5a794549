// CTC negative log-likelihood and its gradient with respect to the LOGITS of the encoder's CTC head, log-softmax fused in
// (reference: speecht5/criterions/speech_to_text_loss.py:303-335 -- F.log_softmax via get_normalized_probs_for_ctc, then
// F.ctc_loss(reduction="sum", zero_infinity=...) with cuDNN off). Extended label sequence l' = (blank, l1, blank, ...,
// lL, blank), S = 2L+1 states. Only the two T-step recursions are sequential; everything else is spread over the GPU:
//   1 ctc_rows_kernel   (warp per (t, b) row)  lse_t = logsumexp_k logits[t,b,k];  lp[b,t,s] = logits[t,b,l'_s] - lse_t
//   2 ctc_sweeps_kernel (CTA per utterance)    alpha (forward) and beta (backward) recursions run CONCURRENTLY in the two
//                       halves of the CTA, one thread per state, one barrier per time step; the emission terms lp are
//                       fetched a group of steps ahead (a global round trip per step would dominate the recursion);
//                         alpha_t(s) = lp_t(s) + lse(alpha_{t-1}(s), alpha_{t-1}(s-1), [alpha_{t-1}(s-2) if l'_s != blank, != l'_{s-2}])
//                         beta_t(s)  = lp_t(s) + lse(beta_{t+1}(s),  beta_{t+1}(s+1),  [beta_{t+1}(s+2)  if l'_s != blank, != l'_{s+2}])
//                       nll = -lse of the two final alpha states
//   3 ctc_grad_kernel   (warp per (t, b) row)  dlogits[t,k] = softmax_t(k) - sum_{s: l'_s = k} exp(alpha_t(s) + beta_t(s) - lp_t(s) + nll)
//                       (per-symbol sums in shared memory in the linear domain: every term is <= 1; the blank states,
//                       half of all, are summed in registers).
// Rows t >= input_length get a zero gradient; an infeasible utterance gives nll = +inf, or 0 with zero gradient under
// zero_infinity. The algorithm is restated and checked against torch on the CPU in tests/test_kernel_algorithms_cpu.py.
#include "kernels.cuh"
#include <math_constants.h>

namespace st5 {

__device__ __forceinline__ float lse2(float a, float b) {
  const float m = fmaxf(a, b);
  if (m == -CUDART_INF_F) return -CUDART_INF_F;
  return m + log1pf(__expf(-fabsf(a - b)));
}

constexpr int CTC_ROW_WARPS = 8;
constexpr int CTC_GROUP = 4;  // time steps whose emission terms are fetched together, one group ahead

// one warp per (t, b): lse[t * B + b] and the emission row lp[b][t][0..S)
__global__ void __launch_bounds__(CTC_ROW_WARPS * 32)
    ctc_rows_kernel(const float* __restrict__ logits, int64_t ld_t, int64_t ld_b, const int64_t* __restrict__ targets,
                    const int64_t* __restrict__ tgt_offsets, const int64_t* __restrict__ input_lengths,
                    const int64_t* __restrict__ target_lengths, float* __restrict__ lse, float* __restrict__ lp, int T,
                    int B, int V, int S_max, int blank) {
  const int row = blockIdx.x * CTC_ROW_WARPS + (threadIdx.x >> 5);
  if (row >= T * B) return;
  const int t = row / B, b = row - t * B;
  const float* x = logits + (int64_t)t * ld_t + (int64_t)b * ld_b;
  const int lane = threadIdx.x & 31;
  float m = -CUDART_INF_F;
  for (int k = lane; k < V; k += 32) m = fmaxf(m, x[k]);
  m = warp_max(m);
  float s = 0.f;
  for (int k = lane; k < V; k += 32) s += __expf(x[k] - m);
  s = warp_sum(s);
  const float l = m + __logf(s);
  if (lane == 0) lse[row] = l;
  const int L = (int)target_lengths[b];
  const int S = 2 * L + 1;
  if (S > S_max || t >= input_lengths[b]) return;
  const int64_t* tg = targets + tgt_offsets[b];
  float* dst = lp + ((int64_t)b * T + t) * S_max;
  for (int st = lane; st < S; st += 32) dst[st] = x[(st & 1) ? (int)tg[st >> 1] : blank] - l;
}

// One CTA per utterance, blockDim = 2 * SP (concurrent: threads [0, SP) run alpha, [SP, 2 SP) run beta) or SP (the two
// sweeps one after the other, S_max > 512). Both sweeps take exactly Tn steps, so they share every barrier.
__global__ void __launch_bounds__(1024)
    ctc_sweeps_kernel(const float* __restrict__ lp, const int64_t* __restrict__ targets,
                      const int64_t* __restrict__ tgt_offsets, const int64_t* __restrict__ input_lengths,
                      const int64_t* __restrict__ target_lengths, float* __restrict__ nll_out, float* __restrict__ nll_raw,
                      float* __restrict__ alpha_ws, float* __restrict__ beta_ws, int T, int S_max, int SP, int blank,
                      int zero_infinity) {
  extern __shared__ float sm[];  // [2 roles][2 buffers][SP]
  const int b = blockIdx.x;
  const int Tn = (int)min((int64_t)T, input_lengths[b]);
  const int L = (int)target_lengths[b];
  const int S = 2 * L + 1;
  const bool feasible_len = Tn >= 1 && S <= S_max;  // (an utterance longer than the scratch pitch is reported as infeasible)
  if (!feasible_len) {
    if (threadIdx.x == 0) {
      nll_raw[b] = CUDART_INF_F;
      nll_out[b] = zero_infinity ? 0.f : CUDART_INF_F;
    }
    return;
  }
  const int64_t* tg = targets + tgt_offsets[b];
  const bool concurrent = (int)blockDim.x == 2 * SP;
  const float* lpb = lp + (int64_t)b * T * S_max;
  for (int pass = 0; pass < (concurrent ? 1 : 2); ++pass) {
    const int role = concurrent ? (int)threadIdx.x / SP : pass;  // 0 = alpha, 1 = beta
    const int s = concurrent ? (int)threadIdx.x - role * SP : (int)threadIdx.x;
    float* prev = sm + role * 2 * SP;
    float* cur = prev + SP;
    float* out = (role == 0 ? alpha_ws : beta_ws) + (int64_t)b * T * S_max;
    const bool on = s < S;
    const int sym = on && (s & 1) ? (int)tg[s >> 1] : blank;
    // the second neighbour: alpha from s-2, beta from s+2 (only between two different non-blank labels)
    bool skip = false;
    if (on && (s & 1)) skip = role == 0 ? (s >= 2 && (int)tg[(s >> 1) - 1] != sym) : (s + 2 < S && (int)tg[(s >> 1) + 1] != sym);
    const int d1 = role == 0 ? -1 : 1;
    const bool has1 = role == 0 ? s >= 1 : s + 1 < S;
    auto t_of = [&](int step) { return role == 0 ? step : Tn - 1 - step; };
    float e_cur[CTC_GROUP], e_nxt[CTC_GROUP];
#pragma unroll
    for (int u = 0; u < CTC_GROUP; ++u) e_cur[u] = (on && u < Tn) ? lpb[(int64_t)t_of(u) * S_max + s] : 0.f;
    for (int g0 = 0; g0 < Tn; g0 += CTC_GROUP) {
#pragma unroll
      for (int u = 0; u < CTC_GROUP; ++u) {
        const int step = g0 + CTC_GROUP + u;
        e_nxt[u] = (on && step < Tn) ? lpb[(int64_t)t_of(step) * S_max + s] : 0.f;
      }
#pragma unroll
      for (int u = 0; u < CTC_GROUP; ++u) {
        const int step = g0 + u;
        if (step < Tn) {  // (uniform over the CTA)
          float v = -CUDART_INF_F;
          if (on) {
            if (step == 0) {
              // alpha_0: the first blank and the first label; beta_{Tn-1}: the last blank and the last label
              v = (role == 0 ? s < 2 : s >= S - 2) ? 0.f : -CUDART_INF_F;
            } else {
              v = prev[s];
              if (has1) v = lse2(v, prev[s + d1]);
              if (skip) v = lse2(v, prev[s + 2 * d1]);
            }
            v += e_cur[u];
            out[(int64_t)t_of(step) * S_max + s] = v;
          }
          if (s < SP) cur[s] = v;
          __syncthreads();
          float* tmp = prev; prev = cur; cur = tmp;
        }
      }
#pragma unroll
      for (int u = 0; u < CTC_GROUP; ++u) e_cur[u] = e_nxt[u];
    }
    if (role == 0 && s == 0) {  // prev = alpha_{Tn-1} (written before the last barrier)
      const float ll = S >= 2 ? lse2(prev[S - 1], prev[S - 2]) : prev[0];
      const float nll = -ll;
      nll_raw[b] = nll;
      nll_out[b] = nll < CUDART_INF_F ? nll : (zero_infinity ? 0.f : CUDART_INF_F);
    }
    __syncthreads();
  }
}

// one warp per (t, b) row of the gradient
__global__ void __launch_bounds__(CTC_ROW_WARPS * 32)
    ctc_grad_kernel(const float* __restrict__ logits, int64_t ld_t, int64_t ld_b, const float* __restrict__ lse,
                    const float* __restrict__ lp, const float* __restrict__ alpha_ws, const float* __restrict__ beta_ws,
                    const float* __restrict__ nll_raw, const int64_t* __restrict__ targets,
                    const int64_t* __restrict__ tgt_offsets, const int64_t* __restrict__ input_lengths,
                    const int64_t* __restrict__ target_lengths, float* __restrict__ grad, int T, int B, int V, int S_max,
                    int blank, int warps) {
  extern __shared__ float acc_all[];  // [warps][V]
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row = blockIdx.x * warps + w;
  if (row >= T * B) return;
  const int t = row / B, b = row - t * B;
  float* g = grad + (int64_t)t * ld_t + (int64_t)b * ld_b;
  const float nll = nll_raw[b];
  const int Tn = (int)min((int64_t)T, input_lengths[b]);
  if (!(nll < CUDART_INF_F) || t >= Tn) {
    for (int k = lane; k < V; k += 32) g[k] = 0.f;
    return;
  }
  float* acc = acc_all + (size_t)w * V;
  for (int k = lane; k < V; k += 32) acc[k] = 0.f;
  __syncwarp();
  const int S = 2 * (int)target_lengths[b] + 1;
  const int64_t* tg = targets + tgt_offsets[b];
  const int64_t base = ((int64_t)b * T + t) * S_max;
  float blank_mass = 0.f;
  for (int s = lane; s < S; s += 32) {
    const float e = alpha_ws[base + s] + beta_ws[base + s] - lp[base + s] + nll;
    if (e > -80.f) {
      const float pm = __expf(e);
      if (s & 1) atomicAdd(&acc[(int)tg[s >> 1]], pm);
      else blank_mass += pm;
    }
  }
  blank_mass = warp_sum(blank_mass);
  __syncwarp();
  if (lane == 0) acc[blank] += blank_mass;
  __syncwarp();
  const float* x = logits + (int64_t)t * ld_t + (int64_t)b * ld_b;
  const float l = lse[row];
  for (int k = lane; k < V; k += 32) g[k] = __expf(x[k] - l) - acc[k];
}

// lse [T*B] | raw nll [B] | lp, alpha, beta [B][T][S_max] each
int64_t ctc_ws_floats(int32_t T, int32_t B, int32_t S_max) { return (int64_t)T * B + B + 3 * (int64_t)B * T * S_max; }

int ctc_loss_launch(const float* logits, int64_t ld_t, int64_t ld_b, const int64_t* targets, const int64_t* tgt_offsets,
                    const int64_t* input_lengths, const int64_t* target_lengths, float* nll, float* grad, float* ws,
                    int32_t T, int32_t B, int32_t V, int32_t S_max, int32_t blank, int32_t zero_infinity,
                    cudaStream_t st) {
  if (T <= 0 || B <= 0 || V <= 0 || S_max <= 0 || S_max > 1024 || blank < 0 || blank >= V) return -2;
  // the gradient kernel keeps one fp32 row of V per-symbol sums per warp in 48 KiB of shared memory; checked before any
  // launch so that a rejected call writes nothing
  int warps = CTC_ROW_WARPS;
  while (warps > 1 && (size_t)warps * V * sizeof(float) > 48 * 1024) warps >>= 1;
  if (grad != nullptr && (size_t)warps * V * sizeof(float) > 48 * 1024) return -2;
  float* lse = ws;
  float* nll_raw = ws + (int64_t)T * B;
  float* lp = nll_raw + B;
  float* alpha = lp + (int64_t)B * T * S_max;
  float* beta = alpha + (int64_t)B * T * S_max;
  const int rows = T * B;
  ctc_rows_kernel<<<(rows + CTC_ROW_WARPS - 1) / CTC_ROW_WARPS, CTC_ROW_WARPS * 32, 0, st>>>(
      logits, ld_t, ld_b, targets, tgt_offsets, input_lengths, target_lengths, lse, lp, T, B, V, S_max, blank);
  const int SP = (S_max + 31) / 32 * 32;
  const int threads = 2 * SP <= 1024 ? 2 * SP : SP;
  ctc_sweeps_kernel<<<B, threads, (size_t)4 * SP * sizeof(float), st>>>(lp, targets, tgt_offsets, input_lengths,
                                                                       target_lengths, nll, nll_raw, alpha, beta, T, S_max,
                                                                       SP, blank, zero_infinity);
  if (grad != nullptr) {
    ctc_grad_kernel<<<(rows + warps - 1) / warps, warps * 32, (size_t)warps * V * sizeof(float), st>>>(
        logits, ld_t, ld_b, lse, lp, alpha, beta, nll_raw, targets, tgt_offsets, input_lengths, target_lengths, grad, T, B,
        V, S_max, blank, warps);
  }
  return (int)cudaGetLastError();
}

}  // namespace st5
