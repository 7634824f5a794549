// Beam search over the text decoder's vocabulary: candidate selection and the per-sentence bookkeeping of one step.
//
// Reference: speecht5/sequence_generator.py:430-636 (score masking, search.step, finalize, active-hypothesis selection)
// with finalize_hypos / is_finished (:690-816) and fairseq/search.py:117-144 (BeamSearch.step), ctc_weight 0, no prefix
// tokens; with or without a language model's log-probabilities added before the masking (:420-426).
//
// Candidate selection is exact: each row's top n (the sentence needs n = min(2K, F - 1)) is found by n rounds of a
// CTA-wide arg-max over the row's masked log-probabilities, each round taking the best element strictly after the
// previous one in the order (score descending, index ascending); a per-sentence pass then merges the K row lists the
// same way. The sentence's top n lies inside the union of its rows' top n, so the merge is exact, and the order makes
// ties go to the lower flat index.
//
// Bookkeeping never moves the decoder's key/value cache: cell (slot, position) is written once, and a lineage table
// lin[slot][position] names the slot whose cells hold each position of the hypothesis now in a slot. A reorder rewrites
// the table of the sentence's K slots (column by column, staged through shared memory), not the cache.
#include "kernels.cuh"

namespace st5 {

constexpr int BT = 256;      // threads of the per-row selection
constexpr int BKMAX = 16;    // beams per sentence
constexpr int BVMAX = 32768; // vocabulary
constexpr int UT = 128;      // threads of the per-sentence update
constexpr int UCH = 64;      // lineage columns staged per pass

struct Cand {
  float s;
  int i;
};

// a before b in (score descending, index ascending)
__device__ __forceinline__ bool cand_before(float as, int ai, float bs, int bi) {
  return as > bs || (as == bs && ai < bi);
}

__device__ __forceinline__ Cand warp_best(Cand c) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float s = __shfl_xor_sync(0xffffffffu, c.s, o);
    const int i = __shfl_xor_sync(0xffffffffu, c.i, o);
    if (cand_before(s, i, c.s, c.i)) c = Cand{s, i};
  }
  return c;
}

__device__ __forceinline__ int beam_n(int t, int K, int V) {
  const int F = t == 0 ? V : K * V;
  return min(2 * K, F - 1);
}

// the language model's row of a fused step (sequence_generator.py:420-426): logits y[r * ld + v] for v < V
struct LmRow {
  const void* y;
  int64_t ld;
  int dtype;
  int V;
  float w;
};

__device__ __forceinline__ float lm_ld(const LmRow& lm, int64_t i) {
  return lm.dtype == ST5_F32 ? ldf(static_cast<const float*>(lm.y) + i)
                             : ldf(static_cast<const __nv_bfloat16*>(lm.y) + i);
}

// CTA-wide max (sum when !MAX) of one value per thread; every thread gets the result
template <bool MAX>
__device__ __forceinline__ float cta_reduce(float v, float (&red)[BT / 32], int lane, int w) {
  v = MAX ? warp_max(v) : warp_sum(v);
  if (lane == 0) red[w] = v;
  __syncthreads();
  v = MAX ? red[0] : 0.f;
#pragma unroll
  for (int i = MAX ? 1 : 0; i < BT / 32; ++i) v = MAX ? fmaxf(v, red[i]) : v + red[i];
  __syncthreads();
  return v;
}

// one CTA per row: the row's best n candidates into ws; with LM the row's score gains lm.w * log_softmax(y)[v], v < lm.V
template <typename T, bool LM>
__device__ __forceinline__ void row_topk(const T* logits, int64_t ld, int K, int V, const float* cum, const float* mask,
                                         float inv_temp, int eos, const int64_t* tp, const int64_t* minp,
                                         const int64_t* maxp, float* ws, float (&red)[BT / 32], Cand (&best)[BT / 32],
                                         const LmRow lm) {
  const int r = blockIdx.x, tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int64_t t = *tp;
  if (t == 0 && r % K != 0) return;  // (search.py:119-122: step 0 reads beam 0 only)
  const int n = min(beam_n((int)t, K, V), V);
  const T* x = logits + (int64_t)r * ld;
  float m = -INFINITY;
  for (int v = tid; v < V; v += BT) m = fmaxf(m, ldf(x + v) * inv_temp);
  m = warp_max(m);
  if (lane == 0) red[w] = m;
  __syncthreads();
  m = red[0];
#pragma unroll
  for (int i = 1; i < BT / 32; ++i) m = fmaxf(m, red[i]);
  __syncthreads();
  float l = 0.f;  // (a NaN logit makes the sum NaN and so every log-probability NaN -> -inf, as log_softmax does)
  for (int v = tid; v < V; v += BT) l += expf(ldf(x + v) * inv_temp - m);
  l = warp_sum(l);
  if (lane == 0) red[w] = l;
  __syncthreads();
  l = 0.f;
#pragma unroll
  for (int i = 0; i < BT / 32; ++i) l += red[i];
  const float lse = logf(l);
  // the LM's log-softmax over its own vocabulary, in fp32, without the temperature (:420-425)
  float ym = 0.f, ylse = 0.f;
  if constexpr (LM) {
    const int64_t yo = (int64_t)r * lm.ld;
    __syncthreads();  // (red is reused)
    ym = -INFINITY;
    for (int v = tid; v < lm.V; v += BT) ym = fmaxf(ym, lm_ld(lm, yo + v));
    ym = cta_reduce<true>(ym, red, lane, w);
    float yl = 0.f;
    for (int v = tid; v < lm.V; v += BT) yl += expf(lm_ld(lm, yo + v) - ym);
    ylse = logf(cta_reduce<false>(yl, red, lane, w));
  }
  const bool no_eos = t < *minp, only_eos = t >= *maxp;
  const float c0 = t > 0 ? cum[r] : 0.f;
  float* ws_s = ws + (int64_t)r * 2 * BKMAX * 2;
  int* ws_i = reinterpret_cast<int*>(ws_s + 2 * BKMAX);
  float ps = INFINITY;
  int pi = -1;
  for (int k = 0; k < n; ++k) {
    Cand c{-INFINITY, 0x7fffffff};
    for (int v = tid; v < V; v += BT) {
      float lp = (ldf(x + v) * inv_temp - m) - lse;
      if constexpr (LM) {
        if (v < lm.V) lp += lm.w * ((lm_ld(lm, (int64_t)r * lm.ld + v) - ym) - ylse);  // (:426, before any masking)
      }
      if (no_eos && v == eos) lp = -INFINITY;
      if (lp != lp) lp = -INFINITY;
      lp += mask[v];
      if (only_eos && v != eos) lp = -INFINITY;
      if (t > 0) lp += c0;
      if (cand_before(ps, pi, lp, v) && cand_before(lp, v, c.s, c.i)) c = Cand{lp, v};
    }
    c = warp_best(c);
    if (lane == 0) best[w] = c;
    __syncthreads();
    c = best[0];
#pragma unroll
    for (int i = 1; i < BT / 32; ++i)
      if (cand_before(best[i].s, best[i].i, c.s, c.i)) c = best[i];
    __syncthreads();
    if (tid == 0) {
      ws_s[k] = c.s;
      ws_i[k] = c.i;
    }
    ps = c.s;
    pi = c.i;
  }
}

template <typename T>
__global__ void __launch_bounds__(BT) beam_row_topk(const T* logits, int64_t ld, int K, int V, const float* cum,
                                                    const float* mask, float inv_temp, int eos, const int64_t* tp,
                                                    const int64_t* minp, const int64_t* maxp, float* ws) {
  __shared__ float red[BT / 32];
  __shared__ Cand best[BT / 32];
  row_topk<T, false>(logits, ld, K, V, cum, mask, inv_temp, eos, tp, minp, maxp, ws, red, best, LmRow{});
}

template <typename T>
__global__ void __launch_bounds__(BT) lm_fused_row_topk(const T* logits, int64_t ld, int K, int V, const float* cum,
                                                        const float* mask, float inv_temp, int eos, const int64_t* tp,
                                                        const int64_t* minp, const int64_t* maxp, float* ws,
                                                        const LmRow lm) {
  __shared__ float red[BT / 32];
  __shared__ Cand best[BT / 32];
  row_topk<T, true>(logits, ld, K, V, cum, mask, inv_temp, eos, tp, minp, maxp, ws, red, best, lm);
}

// one warp per sentence: the best n of the union of its rows' lists, flat index beam * V + token
__global__ void __launch_bounds__(32) beam_merge_topk(int K, int V, const int64_t* tp, const float* ws,
                                                      float* cand_score, int32_t* cand_token, int32_t* cand_beam) {
  const int s = blockIdx.x, lane = threadIdx.x;
  const int t = (int)*tp;
  const int n = beam_n(t, K, V), nr = min(n, V), nb = t == 0 ? 1 : K;
  float ps = INFINITY;
  int pi = -1;
  for (int k = 0; k < n; ++k) {
    Cand c{-INFINITY, 0x7fffffff};
    for (int e = lane; e < nb * nr; e += 32) {
      const int b = e / nr, q = e - b * nr;
      const float* row = ws + (int64_t)(s * K + b) * 2 * BKMAX * 2;
      const float sc = row[q];
      const int fi = b * V + reinterpret_cast<const int*>(row + 2 * BKMAX)[q];
      if (cand_before(ps, pi, sc, fi) && cand_before(sc, fi, c.s, c.i)) c = Cand{sc, fi};
    }
    c = warp_best(c);
    if (lane == 0) {
      cand_score[s * 2 * K + k] = c.s;
      cand_token[s * 2 * K + k] = c.i % V;
      cand_beam[s * 2 * K + k] = c.i / V;
    }
    ps = c.s;
    pi = c.i;
  }
}

struct BeamState {
  int B, K, V, T, eos, normalize;
  float len_penalty;
  const int64_t *t, *max_len;
  const float* cand_score;
  const int32_t *cand_token, *cand_beam;
  int32_t *lin, *tok;
  float* score;
  int32_t *ignore, *finished, *parent;
  int64_t* cur_tok;
  float* cur_score;
  int32_t *fin_n, *fin_tok;
  float* fin_pos;
  int32_t* fin_len;
  float* fin_score;
  int32_t* stop;
};

__global__ void __launch_bounds__(UT) beam_update_kernel(const BeamState a) {
  __shared__ int eos_c[BKMAX];     // candidate positions finalized this step, in order
  __shared__ int active[BKMAX];    // candidate position continued in slot k
  __shared__ int new_ignore[BKMAX];
  __shared__ int n_fin, fin0, done;
  __shared__ int stage[BKMAX][UCH];
  const int s = blockIdx.x, tid = threadIdx.x, K = a.K, T = a.T;
  if (a.finished[s]) return;
  const int t = (int)*a.t, maxl = (int)*a.max_len;
  const int n = beam_n(t, K, a.V);
  const float* cs = a.cand_score + s * 2 * K;
  const int32_t* ct = a.cand_token + s * 2 * K;
  const int32_t* cb = a.cand_beam + s * 2 * K;
  if (tid == 0) {
    // (:491-505) eos candidates among the first K, cands_to_ignore by candidate position
    uint32_t em = 0;  // bit c: candidate c ends in eos
    int ne = 0;
    for (int c = 0; c < n; ++c) {
      const bool e = ct[c] == a.eos && cs[c] != -INFINITY && !(c < K && a.ignore[s * K + c]);
      em |= (uint32_t)e << c;
      if (c < K && e) eos_c[ne++] = c;
    }
    // (:766-784) appended in candidate order while fewer than K are held
    const int held = a.fin_n[s];
    fin0 = held;
    n_fin = min(ne, K - held);
    a.fin_n[s] = held + n_fin;
    // (:800-816) finished at K hypotheses or at max_len; past max_len the reference asserts, here the sentence ends
    done = (ne > 0 && (held + n_fin == K || t == maxl)) || t >= maxl;
    if (done) a.finished[s] = 1;
    // (:572-596) active_mask: the first K candidates that neither end in eos nor are ignored, then those that do
    int na = 0;
    for (int pass = 0; pass < 2 && na < K; ++pass) {
      for (int c = 0; c < n && na < K; ++c) {
        const bool m2 = ((em >> c) & 1u) || (c < K && a.ignore[s * K + c] != 0);
        if (m2 == (pass == 1)) {
          active[na] = c;
          new_ignore[na] = pass;
          ++na;
        }
      }
    }
  }
  __syncthreads();
  // finalize (:714-735): tokens 1..t of the beam's hypothesis then eos, cumulative scores differenced
  for (int f = 0; f < n_fin; ++f) {
    const int c = eos_c[f], x = s * K + cb[c], slot = fin0 + f;
    int32_t* ft = a.fin_tok + ((int64_t)s * K + slot) * T;
    float* fp = a.fin_pos + ((int64_t)s * K + slot) * T;
    const int32_t* lx = a.lin + (int64_t)x * T;
    for (int j = tid; j <= t; j += UT) {
      const float cj = j < t ? a.score[(int64_t)lx[j + 1] * T + j + 1] : cs[c];
      const float cp = j == 0 ? 0.f : a.score[(int64_t)lx[j] * T + j];
      ft[j] = j < t ? a.tok[(int64_t)lx[j + 1] * T + j + 1] : a.eos;
      fp[j] = j == 0 ? cj : cj - cp;
    }
    if (tid == 0) {
      a.fin_len[s * K + slot] = t + 1;
      a.fin_score[s * K + slot] = a.normalize ? cs[c] / (float)pow((double)(t + 1), (double)a.len_penalty) : cs[c];
    }
  }
  if (done) return;
  // reorder (:598-636): lin[r][0..t] = lin[parent][0..t], column blocks staged so the gather may read rows it writes
  int32_t* lin = a.lin + (int64_t)s * K * T;
  for (int j0 = 0; j0 <= t; j0 += UCH) {
    const int w = min(UCH, t + 1 - j0);
    for (int e = tid; e < K * UCH; e += UT) {
      const int k = e / UCH, jj = e - k * UCH;
      if (jj < w) stage[k][jj] = lin[(int64_t)k * T + j0 + jj];
    }
    __syncthreads();
    for (int e = tid; e < K * UCH; e += UT) {
      const int k = e / UCH, jj = e - k * UCH;
      if (jj < w) lin[(int64_t)k * T + j0 + jj] = stage[cb[active[k]]][jj];
    }
    __syncthreads();
  }
  if (tid < K) {
    const int c = active[tid], r = s * K + tid;
    const int64_t cell = (int64_t)r * T + t + 1;
    a.parent[r] = s * K + cb[c];
    a.cur_tok[r] = ct[c];
    a.cur_score[r] = cs[c];
    a.ignore[r] = new_ignore[tid];
    a.lin[cell] = r;
    a.tok[cell] = ct[c];
    a.score[cell] = cs[c];
  }
}

__global__ void __launch_bounds__(32) beam_stop_kernel(int B, const int64_t* tp, const int32_t* finished, int32_t* stop) {
  int all = 1;
  for (int s = threadIdx.x; s < B; s += 32) all &= finished[s] != 0;
  all = __all_sync(0xffffffffu, all);
  if (threadIdx.x == 0) stop[*tp] = all;
}

int64_t beam_topk_ws_floats(int B, int K) { return (int64_t)B * K * 2 * BKMAX * 2; }

int beam_topk_launch(const void* logits, int64_t ld, int dtype, int B, int K, int V, const float* cum,
                     const float* mask, float inv_temp, int eos, const int64_t* t, const int64_t* min_len,
                     const int64_t* max_len, float* cand_score, int32_t* cand_token, int32_t* cand_beam, float* ws,
                     cudaStream_t st) {
  if (B <= 0 || K < 1 || K > BKMAX || V < 2 || V > BVMAX || eos < 0 || eos >= V) return -2;
  if (!logits || !cum || !mask || !t || !min_len || !max_len || !cand_score || !cand_token || !cand_beam || !ws) return -3;
  if (ld < V) return -6;
  if (dtype == ST5_F32)
    beam_row_topk<float><<<B * K, BT, 0, st>>>((const float*)logits, ld, K, V, cum, mask, inv_temp, eos, t, min_len,
                                              max_len, ws);
  else
    beam_row_topk<__nv_bfloat16><<<B * K, BT, 0, st>>>((const __nv_bfloat16*)logits, ld, K, V, cum, mask, inv_temp,
                                                      eos, t, min_len, max_len, ws);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return (int)e;
  beam_merge_topk<<<B, 32, 0, st>>>(K, V, t, ws, cand_score, cand_token, cand_beam);
  return (int)cudaGetLastError();
}

int beam_topk_lm_launch(const void* logits, int64_t ld, int dtype, int B, int K, int V, const float* cum,
                        const float* mask, float inv_temp, int eos, const int64_t* t, const int64_t* min_len,
                        const int64_t* max_len, const void* lm_logits, int64_t lm_ld, int lm_dtype, int V_lm,
                        float lm_weight, float* cand_score, int32_t* cand_token, int32_t* cand_beam, float* ws,
                        cudaStream_t st) {
  if (B <= 0 || K < 1 || K > BKMAX || V < 2 || V > BVMAX || eos < 0 || eos >= V || V_lm < 1 || V_lm > V) return -2;
  if (!logits || !cum || !mask || !t || !min_len || !max_len || !lm_logits || !cand_score || !cand_token ||
      !cand_beam || !ws)
    return -3;
  if (ld < V || lm_ld < V_lm) return -6;
  const LmRow lm{lm_logits, lm_ld, lm_dtype, V_lm, lm_weight};
  if (dtype == ST5_F32)
    lm_fused_row_topk<float><<<B * K, BT, 0, st>>>((const float*)logits, ld, K, V, cum, mask, inv_temp, eos, t,
                                                   min_len, max_len, ws, lm);
  else
    lm_fused_row_topk<__nv_bfloat16><<<B * K, BT, 0, st>>>((const __nv_bfloat16*)logits, ld, K, V, cum, mask,
                                                           inv_temp, eos, t, min_len, max_len, ws, lm);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return (int)e;
  beam_merge_topk<<<B, 32, 0, st>>>(K, V, t, ws, cand_score, cand_token, cand_beam);
  return (int)cudaGetLastError();
}

int beam_update_launch(int B, int K, int V, int T, int eos, const int64_t* t, const int64_t* max_len, int normalize,
                       float len_penalty, const float* cand_score, const int32_t* cand_token, const int32_t* cand_beam,
                       int32_t* lin, int32_t* tok, float* score, int32_t* ignore, int32_t* finished, int32_t* parent,
                       int64_t* cur_tok, float* cur_score, int32_t* fin_n, int32_t* fin_tok, float* fin_pos,
                       int32_t* fin_len, float* fin_score, int32_t* stop, cudaStream_t st) {
  // (V > K: step 0 offers n = min(2K, V - 1) candidates, and K of them must continue)
  if (B <= 0 || K < 1 || K > BKMAX || V <= K || V > BVMAX || T < 2) return -2;
  if (!t || !max_len || !cand_score || !cand_token || !cand_beam || !lin || !tok || !score || !ignore || !finished ||
      !parent || !cur_tok || !cur_score || !fin_n || !fin_tok || !fin_pos || !fin_len || !fin_score || !stop)
    return -3;
  const BeamState a{B, K, V, T, eos, normalize, len_penalty, t, max_len, cand_score, cand_token, cand_beam, lin, tok,
                    score, ignore, finished, parent, cur_tok, cur_score, fin_n, fin_tok, fin_pos, fin_len, fin_score,
                    stop};
  beam_update_kernel<<<B, UT, 0, st>>>(a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return (int)e;
  beam_stop_kernel<<<1, 32, 0, st>>>(B, t, finished, stop);
  return (int)cudaGetLastError();
}

}  // namespace st5
