/*
 * speecht5_b200 -- C ABI of the H100 (sm_90a) kernel library for the SpeechT5 forward/backward hot path.
 *
 * The reference (microsoft/SpeechT5, SpeechT5/speecht5/models/modules/*.py) has no FFI of its own: every device op is
 * a PyTorch library call made from the nn.Module forward()s. This header is the boundary a maintainer binds instead
 * (ctypes stub shown in INTEGRATION.md); each entry point names the reference code it replaces (file:line under
 * /root/reference/SpeechT5/).
 *
 * Conventions
 *   - every pointer is a DEVICE pointer owned by the caller (PyTorch); nothing is allocated or freed here;
 *   - `stream` is a cudaStream_t (pass torch.cuda.current_stream().cuda_stream);
 *   - return value 0 = ok, >0 = cudaError_t, <0 = library argument error; st5_last_error() gives the text
 *     (allocation failures contain the literal "out of memory", which fairseq/trainer.py:725 greps for);
 *   - `dtype`: ST5_F32 = 0, ST5_BF16 = 1 is the activation storage type; statistics, biases, LayerNorm/BatchNorm
 *     parameters, probabilities returned to the caller and all gradients of parameters are fp32;
 *   - dropout is counter based: one Philox4x32-7(seed, offset, i/8) call yields eight 16-bit lanes; element i is kept
 *     iff lane i%8 >= p*65536, i = linear index in the logical tensor (attention probabilities: row pitch rounded up
 *     to a multiple of 32 keys), so forward and backward regenerate identical masks without storing them.
 *     If bit 63 of `offset` is set, `seed` is the device address of a uint64 holding the seed (lets a captured CUDA
 *     graph draw fresh masks on every replay).
 */
#ifndef SPEECHT5_B200_H
#define SPEECHT5_B200_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define ST5_F32 0
#define ST5_BF16 1
#define ST5_ACT_NONE 0
#define ST5_ACT_RELU 1
#define ST5_ACT_GELU 2      /* x Phi(x), Phi from the Abramowitz-Stegun 7.1.26 erf (|error| <= 1.5e-7 in erf) with
                               approximate rcp / ex2: |error| <= 2.5e-7 |x| + a few fp32 ulps of the result */
#define ST5_ACT_TANH 3
#define ST5_ACT_GELU_TANH 4 /* tanh-form GELU on the MUFU unit: |error| <= 4.8e-4 vs the erf form (4.74e-4 measured over
                               every bf16 input, at x = 2.7; below half a bf16 ulp of the result wherever |y| > 0.13);
                               bf16 throughput mode */
/* Non-finite inputs of st5_act_fwd / st5_act_bwd: RELU maps NaN to 0 (fmaxf) and its derivative is 0 at NaN and x <= 0;
 * TANH gives +-1 at +-inf, derivative 0; GELU / GELU_TANH give +inf at +inf and NaN at -inf and NaN, and their
 * derivatives NaN at +-inf and NaN (GELU_TANH's also for finite |x| >= 2^64, where x * x overflows). */
#define ST5_ACT_GATE 5      /* actgrad_act only: actgrad_pre already holds the multiplier (written by ..._GATE below) */
#define ST5_ACT_GELU_TANH_GATE 6 /* act only (bf16 output, N % 8 == 0, c_pre != NULL): C = dropout(gelu_tanh(x)) and c_pre
                                    receives keep * scale * gelu_tanh'(x), the factor of the FFN's dH GEMM in backward */
#define ST5_MARGIN_NONE 0 /* speaker head: plain logits */
#define ST5_MARGIN_AM 1   /* s (cos - m) on the margin column (AngularMargin) */
#define ST5_MARGIN_AAM 2  /* s phi(cos) on the margin column (AdditiveAngularMargin) */

int st5_version(void);
const char* st5_last_error(void);
/* sm_90a only: returns 0 when the current device can run the library, else a negative code. */
int st5_device_ok(void);

/* ------------------------------------------------------------------------------------------------- GEMM
 * D[z][m][n] = epi( alpha * sum_k A[z][m][k] * B[z][n][k] ), bf16 operands, fp32 accumulation in registers
 * (TMA + wgmma). Replaces every nn.Linear / torch.bmm / F.conv1d on the path:
 *   models/modules/multihead_attention.py:213-231 (q/k/v), :340 (QK^T), :389 (PV), :397 (out_proj);
 *   models/modules/transformer_layer.py:127-132, 385-391 (fc1/fc2);
 *   models/modules/speech_decoder_prenet.py:41-47,69-72; speech_decoder_postnet.py:31-32,39-51 (Conv1d as an
 *   overlapping-window GEMM over a zero-padded channels-last buffer); and their backward contractions.
 * Operand storage: *_mn = 0 -> row-major [rows][ld] with k contiguous; *_mn = 1 -> [K][ld] with the row index
 * contiguous (the operand is used transposed without a copy). ld / batch strides are in elements and must be
 * multiples of 8 (16 bytes); base pointers 16-byte aligned. Batch index z = b2 * nb1 + b1.
 * epi(v) = dropout(act(v + c_old*accumulate + bias[n] + bias2[m / bias2_rows][n])) + residual[m][n]; the value before
 * act() is also stored to c_pre when non-null.
 * accumulate: 0 = overwrite; 1 = c += (read-modify-write in the epilogue, FP32 c); 2 = c += as a TMA reduce-add at the
 * L2 (FP32 c, 16-byte aligned rows, N a multiple of 4): batch entries may then SHARE one output (c_bs = 0) -- a contraction split over the
 * batch dimension (weight gradients: a_bs / b_bs step along K) -- and nothing reads c first. */
typedef struct st5_gemm_args {
  int32_t M, N, K, nb1, nb2;
  int32_t a_mn, b_mn, c_fp32, act, accumulate, bias2_rows;
  const void* a; int64_t a_ld, a_bs1, a_bs2;
  const void* b; int64_t b_ld, b_bs1, b_bs2;
  void* c; int64_t c_ld, c_bs1, c_bs2;
  void* c_pre;
  const float* bias;
  const float* bias2;
  const void* residual;
  float alpha;
  float drop_p;
  uint64_t drop_seed, drop_offset;
  const void* actgrad_pre;   /* optional: result *= act'(actgrad_pre[m][n]) (type actgrad_act), applied after the */
  int32_t actgrad_act;       /* dropout mask: fuses the activation backward into the dX GEMM of the next layer   */
} st5_gemm_args;
int st5_gemm_bf16(const st5_gemm_args* args, void* stream);

/* fp32 -> bf16 cast of a strided 2-D view: hi = round-to-nearest-even(x). lo != NULL additionally writes the bf16
 * residual round-to-nearest-even(x - float(hi(x))), which
 * lets callers form hi*hi + hi*lo + lo*hi with three accumulate passes of st5_gemm_bf16 (fp32-grade "parity mode"). */
int st5_cast_bf16(const float* src, int64_t src_ld, void* hi, void* lo, int64_t dst_ld, int64_t rows, int64_t cols,
                  void* stream);

/* ------------------------------------------------------------------------------------------------- pre-nets
 * y[b,t,:] = dropout( (tokens ? E[tokens[b,t]] : x[b,t,:]) + alpha * pe[t,:] ); pe has at least T rows of C floats.
 * text_encoder_prenet.py:36-45 (Embedding -> espnet ScaledPositionalEncoding), speech_decoder_prenet.py:52-67. */
int st5_posenc_fwd(const int64_t* tokens, const float* emb, const void* x, const float* pe, const float* alpha,
                   void* y, int dtype, int64_t B, int64_t T, int64_t C, float drop_p, uint64_t seed, uint64_t offset,
                   void* stream);
/* Backward: dx (same dtype, may be NULL), demb += (fp32 scatter-add, skipping padding_idx), dalpha += sum(dy*pe). */
int st5_posenc_bwd(const void* dy, const int64_t* tokens, int64_t padding_idx, const float* pe, void* dx, float* demb,
                   float* dalpha, int dtype, int64_t B, int64_t T, int64_t C, float drop_p, uint64_t seed,
                   uint64_t offset, void* stream);

/* ------------------------------------------------------------------------------------------------- LayerNorm
 * s = residual + dropout(x); y = LN(s) * gamma + beta (biased variance, eps inside the square root). Saves s (for
 * backward), mean and rstd (each may be NULL). C % 8 == 0 and 0 < C <= 1024; every row tensor and gamma / beta are read
 * and written as 16-byte vectors, so their base pointers must be 16-byte aligned (mean / rstd / dgamma / dbeta / dxsum
 * need only float alignment). Anything else returns -2 before any launch.
 * transformer_layer.py:112-132 (post-LN encoder layer), :343-391 (decoder layer), encoder.py:226-227. */
int st5_ln_fwd(const void* x, const void* residual, const float* gamma, const float* beta, void* y, void* s_out,
               float* mean, float* rstd, int dtype, int64_t rows, int64_t C, float eps, float drop_p, uint64_t seed,
               uint64_t offset, void* stream);
/* Same with an fp32 RESIDUAL STREAM next to the bf16 activations (throughput mode): residual_f32 (may be NULL) replaces
 * `residual` as the addend, y_f32 (may be NULL) receives the un-rounded output. The GEMMs keep reading the bf16 `y`; the
 * next block's residual add reads y_f32, so the post-LN stream of transformer_layer.py:112-132 / :343-391 is never
 * rounded to bf16 between layers (the reference keeps it in fp32 on the CPU path / fp16 storage + fp32 LayerNorm on GPU). */
int st5_ln_fwd_stream(const void* x, const void* residual, const float* residual_f32, const float* gamma,
                      const float* beta, void* y, float* y_f32, void* s_out, float* mean, float* rstd, int dtype,
                      int64_t rows, int64_t C, float eps, float drop_p, uint64_t seed, uint64_t offset, void* stream);
/* Forward only, for rows wider than st5_ln_fwd takes (the 1280-wide pre-LN layers of transformer_lm_t5,
 * speecht5/models/t5_transformer_lm.py:16-25): y = LN(x + residual) * gamma + beta with the arithmetic of
 * st5_ln_fwd (fp32 statistics, two-pass variance) for 8 <= C <= 2048, C % 8 == 0, no dropout and no saved sum. residual,
 * mean and rstd may be NULL; x, residual, y, gamma and beta must be 16-byte aligned. Anything else returns -2 before any
 * launch. st5_ln_fwd, st5_ln_fwd_stream and st5_ln_bwd keep C <= 1024: rows this wide have no backward. */
int st5_ln_fwd_wide(const void* x, const void* residual, const float* gamma, const float* beta, void* y, float* mean,
                    float* rstd, int dtype, int64_t rows, int64_t C, float eps, void* stream);
/* ds = LN backward wrt s; dx = dropout-backward(ds) (may alias / be NULL when drop_p == 0 and caller reuses ds);
 * dgamma/dbeta are accumulated (+=) in fp32. `dxsum` (may be NULL; fp32 [C], accumulated +=) receives the column sums
 * of dx (of ds when dx is NULL): in the post-LN tail y = LN(residual + dropout(W a + b)) that is the gradient of b, so
 * the bias gradient of out_proj / fc2 (transformer_layer.py:112-132) costs no launch of its own.
 * st5_ln_bwd_blocks is kept for ABI stability (returns 1; no scratch is needed). */
int64_t st5_ln_bwd_blocks(int64_t rows);
int st5_ln_bwd(const void* dy, const void* s, const float* mean, const float* rstd, const float* gamma, void* ds,
               void* dx, float* dgamma, float* dbeta, float* dxsum, int dtype, int64_t rows, int64_t C, float drop_p,
               uint64_t seed, uint64_t offset, void* stream);

/* HiFi-GAN operand staging (SpeechUT/fairseq/fairseq/models/text_to_speech/hifigan.py:70-100, 154-170: F.leaky_relu
 * before every convolution): out[b][m][:] = leaky_relu(x[b][ph + d*m - pad][:], slope) for source frames inside [0, T),
 * zeros outside -- the zero-padded (d = 1) or de-interleaved (phase ph of dilation d) bf16 operand of the window GEMM in
 * one pass. x [B, T, C], out [B, n_in, C], C a multiple of 8; slope = 1 copies. */
int st5_lrelu_pad(const void* x, void* out, int64_t B, int64_t T, int64_t C, int64_t n_in, int32_t d, int32_t ph,
                  int32_t pad, float slope, void* stream);
/* st5_lrelu_pad over a padded batch of ragged utterances: source frames are limited to [0, L_b) with
 * L_b = clamp(lengths[b] * len_mult, 0, T) (int64), so row b is staged exactly as utterance b alone would be, and x is
 * never read at or past L_b. lengths: int32 [B] in device memory (a captured graph replays for any lengths; NULL:
 * L_b = T, i.e. st5_lrelu_pad); len_mult: the up-sampling factor between the lengths' resolution and x's.
 * Returns -2 for C % 8 != 0, d < 1, ph outside [0, d), len_mult < 1 or the shape / alignment errors of st5_lrelu_pad;
 * -3 for a NULL x or out. Nothing is launched on an error. */
int st5_lrelu_pad_len(const void* x, void* out, int64_t B, int64_t T, int64_t C, int64_t n_in, int32_t d, int32_t ph,
                      int32_t pad, float slope, const int32_t* lengths, int32_t len_mult, void* stream);

/* y = dropout(x) (also its own backward when applied to the gradient). fairseq/modules/fairseq_dropout.py:23-37
 * (F.dropout semantics: keep with probability 1-p, scale by 1/(1-p)); mask = the counter-based generator above. */
int st5_dropout(const void* x, void* y, int dtype, int64_t n, float drop_p, uint64_t seed, uint64_t offset,
                void* stream);
/* y = act(x), stand-alone: the GELU behind the per-frame LayerNorm of layers 1..6 of the "layer_norm" waveform
 * extractor (speech_encoder_prenet.py:308-318). x, y 16-byte aligned. */
int st5_act_fwd(const void* x, void* y, int dtype, int act, int64_t n, void* stream);
/* dpre = dropout-backward(dy) * act'(pre): backward of activation_fn + activation dropout
 * (transformer_layer.py:127-129, speech_decoder_prenet.py:41-47 via espnet Prenet). */
int st5_act_bwd(const void* dy, const void* pre, void* dpre, int dtype, int act, int64_t n, float drop_p, uint64_t seed,
                uint64_t offset, void* stream);
/* out[g][n] (+)= sum_{m in group g} x[m][n], groups of `group_rows` consecutive rows: bias gradients of every
 * nn.Linear on the path (and, per utterance, of the x-vector term of speech_decoder_prenet.py:69-72); also the reduction
 * of split-K partial products. */
int st5_colsum(const void* x, int64_t ld, float* out, int dtype, int64_t rows, int64_t cols, int64_t group_rows,
               int accumulate, void* stream);

/* ------------------------------------------------------------------------------------------------- attention
 * multihead_attention.py:232-405. q/k/v are read in place from the fused projection outputs:
 *   element (b, t, h, c) of q lives at q[b * q_bs + t * q_ld + h * 64 + c] (same for k, v with their strides).
 * scores = scale * q.(k + pe_k[clamp(i-j,-maxpos,maxpos-1)+maxpos]) (RPE, encoder.py:40-59,239-246) ;
 * causal => j <= i; key_pad[b][j] != 0 => -inf; P = softmax_fp32; out = dropout(P) v.
 * probs (optional) receives P: [B,H,Tq,p_ld] in `probs_dtype` (fp32 when returned to the user: need_head_weights).
 * Head dim is fixed at 64 (Base and Large).
 * A query row whose keys are all masked is produced by no caller; the entry points differ there: st5_attn_fwd returns
 * NaN for it (softmax of an all -inf row, as the reference does), st5_attn_fused_fwd / st5_attn_flash_fwd return zeros
 * (inv_l = 0, lse = -inf). Keys no query row sees (masked, or j >= Tq under the causal mask) get exactly zero dK / dV.
 * dprobs_ext: only columns j < Tk are read (the padding columns [Tk, p_ld) may hold anything). */
typedef struct st5_attn_args {
  int32_t B, H, Tq, Tk, dtype, causal, maxpos, probs_dtype;
  const void* q; int64_t q_ld, q_bs;
  const void* k; int64_t k_ld, k_bs;
  const void* v; int64_t v_ld, v_bs;
  const uint8_t* key_pad;      /* [B][Tk] or NULL */
  const float* pe_k;           /* [2*maxpos][64] fp32 or NULL */
  void* out; int64_t o_ld, o_bs;
  void* probs; int64_t p_ld;   /* may be NULL in forward only */
  float scale, drop_p;
  uint64_t seed, offset;
  /* backward only */
  const void* dout;            /* same layout as out */
  const float* dprobs_ext;     /* optional external gradient wrt P, [B,H,Tq,p_ld] fp32 */
  float* ds;                   /* scratch [B,H,Tq,p_ld] fp32 */
  void* dq; void* dk; void* dv;/* same layouts as q, k, v */
  float* dpe_k;                /* [2*maxpos][64] fp32, accumulated (+=) */
  /* fused / flash forward only: > 0 = write `probs` for heads < probs_heads only (the caller reads no others: the
   * guided-attention loss, text_to_speech_loss.py:210-212); the rest of the buffer is left untouched */
  int32_t probs_heads;
} st5_attn_args;
int st5_attn_fwd(const st5_attn_args* args, void* stream);
int st5_attn_bwd(const st5_attn_args* args, void* stream);

/* One-query-row attention of incremental decoding (forward only, fp32 math): the incremental path of
 * multihead_attention.py:255-330 as the synthesis loop speecht5.py:1222-1245 runs it -- the decoder's self-attention
 * over its key/value cache and its cross-attention over the encoder, one new row per (utterance b, head h).
 *   q row of (b, h) at q[b * q_bs + h * 64 + c]; keys / values at k[b * k_bs + j * k_ld + h * 64 + c] (same for v);
 *   out[b * o_bs + h * 64 + c] in `dtype` (ST5_F32 or ST5_BF16; q, k, v share it).
 * key_pad [B][Tk] uint8 (or NULL): != 0 masks key j of utterance b; masked keys are never loaded. No relative positions,
 * no causal mask, no dropout. probs (optional): the normalised fp32 probabilities, [B][H][Tk].
 * Keys are reduced in fixed splits of 64 (split-KV over grid (splits, H, B), merged by a second launch when Tk > 64):
 * a masked key adds an exact zero, so an utterance's result is bit-identical at any B and any key span Tk that holds
 * its valid keys. ws: st5_attn_decode_ws_floats(B, H, Tk, probs != NULL) floats of scratch (none for Tk <= 64).
 * An utterance whose keys are all masked is produced by no caller; its output and probabilities are zeros (at any Tk).
 * Returns -2 for B, H or Tk <= 0, -5 for ws == NULL with Tk > 64, and -6 unless k, v, k_ld, v_ld, k_bs and v_bs are
 * 16-byte aligned (pointers, and strides in bytes); nothing is written then. */
typedef struct st5_attn_decode_args {
  int32_t B, H, Tk, dtype;
  const void* q; int64_t q_bs;
  const void* k; int64_t k_ld, k_bs;
  const void* v; int64_t v_ld, v_bs;
  const uint8_t* key_pad;      /* [B][Tk] or NULL */
  void* out; int64_t o_bs;
  float* probs;                /* [B][H][Tk] or NULL */
  float scale;
  float* ws;
} st5_attn_decode_args;
int64_t st5_attn_decode_ws_floats(int32_t B, int32_t H, int32_t Tk, int32_t with_probs);
int st5_attn_decode_fwd(const st5_attn_decode_args* args, void* stream);

/* One-query-row attention for beam search (sequence_generator.py:327-361, reorder_incremental_state): the same kernel and
 * contract as st5_attn_decode_fwd, except that key / value j of query row b is read from batch row
 *   kv_rows[b * kv_rows_ld + j]   when kv_rows != NULL (kv_div must then be 1, kv_rows_ld >= Tk), else
 *   b / kv_div                     (kv_div >= 1).
 * The first form is the decoder self-attention over a lineage table (each cache cell is written once; a beam reorder
 * rewrites the table, not the cache), the second the cross-attention of K beams over one copy of their sentence's encoder
 * keys / values (kv_div = K). base.B is the number of query rows; key_pad is indexed by query row. Returns -2 for a bad
 * kv_div / kv_rows_ld, otherwise the codes of st5_attn_decode_fwd. */
typedef struct st5_attn_lineage_args {
  st5_attn_decode_args base;
  const int32_t* kv_rows;      /* [B][kv_rows_ld] or NULL */
  int64_t kv_rows_ld;
  int32_t kv_div;
} st5_attn_lineage_args;
int st5_attn_lineage_fwd(const st5_attn_lineage_args* args, void* stream);

/* The two one-row attentions above for a head width `head_dim` of 64 or 80 (transformer_lm_t5, 1280 channels in 16
 * heads: speecht5/models/t5_transformer_lm.py:16-25): every "64" of their index formulas reads head_dim, and the
 * argument structs, the split-KV contract and the error codes are theirs. head_dim 64 launches exactly the kernels of
 * st5_attn_decode_fwd / st5_attn_lineage_fwd (bit-identical results); head_dim 80 launches their 80-wide counterparts:
 * splits of 64 keys, key j in split j / 64 at a fixed position, masked keys never loaded and adding an exact zero, so a
 * row's result is bit-identical at any B and any key span that holds its valid keys; a row whose keys are all masked
 * gives zeros. Any other head_dim returns -2 before any launch (and st5_attn_decode_hd_ws_floats returns -2 for it);
 * ws: st5_attn_decode_hd_ws_floats(B, H, Tk, probs != NULL, head_dim) floats (none for Tk <= 64). */
int64_t st5_attn_decode_hd_ws_floats(int32_t B, int32_t H, int32_t Tk, int32_t with_probs, int32_t head_dim);
int st5_attn_decode_hd_fwd(const st5_attn_decode_args* args, int32_t head_dim, void* stream);
int st5_attn_lineage_hd_fwd(const st5_attn_lineage_args* args, int32_t head_dim, void* stream);

/* Beam search candidate selection (sequence_generator.py:430-454 with fairseq/search.py:117-144, BeamSearch.step) for B
 * sentences of K beams (1 <= K <= 16, rows r = s * K + k), vocabulary V (1 < V <= 32768). Per row, fp32:
 *   lp = x / T - logsumexp(x / T)   (x = logits[r * ld + v], ST5_F32 or ST5_BF16; inv_temp = 1 / T)
 *   eos -> -inf while *t < *min_len; NaN -> -inf; lp += mask[v]; every v != eos -> -inf once *t >= *max_len;
 *   lp += cum[r] for *t > 0 (at *t == 0 only beam 0 of each sentence takes part).
 * Per sentence the best n = min(2K, F - 1) of the F = (t == 0 ? V : K * V) flat candidates (beam * V + v), in
 * descending score, ties to the lower flat index: cand_score / cand_token / cand_beam[s * 2K + i], i < n; entries
 * i >= n are not written. t, min_len, max_len are device scalars (a captured graph replays any step).
 * ws: st5_beam_topk_ws_floats(B, K) floats of scratch. Returns -2 for K, V or B out of range, -3 for a NULL pointer,
 * -6 unless ld >= V; nothing is launched then. */
int64_t st5_beam_topk_ws_floats(int32_t B, int32_t K);
int st5_beam_topk(const void* logits, int64_t ld, int dtype, int32_t B, int32_t K, int32_t V, const float* cum,
                  const float* mask, float inv_temp, int32_t eos, const int64_t* t, const int64_t* min_len,
                  const int64_t* max_len, float* cand_score, int32_t* cand_token, int32_t* cand_beam, float* ws,
                  void* stream);

/* st5_beam_topk with a language model's log-probabilities fused in (sequence_generator.py:420-426, lm_weight w): per row,
 * fp32, before any of st5_beam_topk's masking,
 *   lp = (x / T - logsumexp(x / T)) + w * (y - logsumexp_{u < V_lm}(y_u))   for v < V_lm  (y = lm_logits[r * lm_ld + v],
 *   ST5_F32 or ST5_BF16 per lm_dtype; no temperature on the LM), lp = x / T - logsumexp(x / T) for V_lm <= v < V;
 * then eos -> -inf while *t < *min_len, NaN -> -inf (so w = 0 against an LM log-probability of -inf, or a NaN LM row,
 * gives -inf), mask, max_len and cum exactly as st5_beam_topk, and the same selection into cand_*. Returns -2 for V_lm
 * outside [1, V], -6 unless lm_ld >= V_lm, otherwise the codes of st5_beam_topk; nothing is launched on an error. */
int st5_beam_topk_lm(const void* logits, int64_t ld, int dtype, int32_t B, int32_t K, int32_t V, const float* cum,
                     const float* mask, float inv_temp, int32_t eos, const int64_t* t, const int64_t* min_len,
                     const int64_t* max_len, float* cand_score, int32_t* cand_token, int32_t* cand_beam, float* ws,
                     const void* lm_logits, int64_t lm_ld, int lm_dtype, int32_t V_lm, float lm_weight, void* stream);

/* Beam search bookkeeping for step *t (sequence_generator.py:487-636 with finalize_hypos / is_finished :690-816), one
 * CTA per sentence; a sentence with finished[s] != 0 is skipped. State of slot r (= s * K + k), capacity T positions:
 *   lin[r][j]  the slot whose cells hold position j of the hypothesis now in slot r (lin[r][t] == r on entry);
 *   tok[r][j], score[r][j]  the token at position j (j >= 1; position 0 is the initial eos) and the cumulative score
 *   after it, stored in the cell (lin, j) of the slot that chose it.
 * ignore[s][K]: cands_to_ignore (by candidate position). Finalized hypotheses: fin_n[s] (count), fin_tok[s][K][T],
 * fin_pos[s][K][T] (positional scores = differences of the cumulative fp32 scores), fin_len[s][K], fin_score[s][K]
 * (eos score / (t + 1) ** len_penalty when normalize). For each eos candidate among the first K (score > -inf, not
 * ignored) the hypothesis is appended while fin_n < K; the sentence is finished at fin_n == K or t == max_len.
 * Otherwise the first K non-eos candidates (then eos ones, which become ignored) continue: parent[r], cur_tok[r],
 * cur_score[r], lin[r][0..t] = lin[parent][0..t], lin[r][t+1] = r, tok / score[r][t+1]. stop[*t] = 1 when every
 * sentence is finished. t + 2 <= T is required (the caller sizes T). Returns -2 for K / T out of range or V <= K (step
 * 0 has n = V - 1 < K candidates then, too few to continue K slots), -3 for a NULL pointer. */
int st5_beam_update(int32_t B, int32_t K, int32_t V, int32_t T, int32_t eos, const int64_t* t, const int64_t* max_len,
                    int32_t normalize, float len_penalty, const float* cand_score, const int32_t* cand_token,
                    const int32_t* cand_beam, int32_t* lin, int32_t* tok, float* score, int32_t* ignore,
                    int32_t* finished, int32_t* parent, int64_t* cur_tok, float* cur_score, int32_t* fin_n,
                    int32_t* fin_tok, float* fin_pos, int32_t* fin_len, float* fin_score, int32_t* stop, void* stream);

/* Fused wgmma attention forward (bf16, Tk <= 320): QK^T -> masks -> softmax -> dropout -> PV in ONE launch, no score
 * or probability round trip through HBM. Uses the q/k/v/out/probs/key_pad/scale/dropout fields of st5_attn_args exactly
 * like st5_attn_fwd; additionally writes lse[b][h][i] = log sum_j exp(s_ij) over the keys row i sees (natural log, the
 * masked scores s of the contract above; may be NULL -- no caller passes it today). probs (optional,
 * only when the caller wants them: need_head_weights) receives the undropped normalised probabilities in probs_dtype.
 * What the backward pass reads back (both optional, but together): psave [B,H,Tq,p_ld] BF16 = exp(s - rowmax), NOT
 * normalised, with the SIGN BIT set on elements dropout removed (probabilities are non-negative; a dropped zero is -0),
 * and inv_l [B,H,Tq] = 1 / rowsum. p_ld must be a multiple of 8, psave 16-byte aligned. psave holds zeros on every
 * masked key and in the columns [Tk, p_ld) of every key block the backward reads (under the causal mask: the blocks up
 * to the row's own 64-row tile; later blocks are neither written nor read). out_f32 (optional)
 * [B,Tq,H*64] FP32 receives the un-rounded output: the backward's row constant delta = dO.O is the subtrahend of a
 * cancelling difference (dS = P (dP - delta)) and must not carry the BF16 rounding of `out`.
 * Relative positions (encoder.py:239-246): pe_k != NULL selects the skewed-bias variant; here pe_k must point to a
 * BF16 copy of the [2*maxpos][64] table, and Tq, Tk <= maxpos <= 160 (clamp(i-j) never clips), no causal mask. */
int st5_attn_fused_fwd(const st5_attn_args* args, float* lse, void* psave, float* inv_l, float* out_f32, void* stream);
/* Streaming ("flash") wgmma attention forward for ANY Tq / Tk (bf16): 64-key blocks, the row maximum is made final
 * in a first sweep over the key blocks (scores only), a second sweep computes exp / dropout / P V with the output
 * accumulating in registers, a third one (only when args->probs != NULL, which must then be FP32) writes the normalised
 * probabilities. Same arguments, outputs and psave / inv_l / out_f32 contract as st5_attn_fused_fwd, so
 * st5_attn_fused_bwd is its backward. Relative positions: pe_k = BF16 copy of the [2*maxpos][64] table, any Tq / Tk --
 * clamp(i - j, -maxpos, maxpos - 1) clips as encoder.py:40-59 does; no causal mask together with pe_k. */
int st5_attn_flash_fwd(const st5_attn_args* args, float* lse, void* psave, float* inv_l, float* out_f32, void* stream);
/* Fused wgmma attention backward (multihead_attention.py:340-389 differentiated). psave / inv_l are what
 * st5_attn_fused_fwd wrote: probabilities and dropout decisions are read back instead of recomputed (no exponential, no
 * Philox), so every step needs one score-sized MMA (dP = dO V^T); the Q / dO tiles and the saved exponentials are
 * double buffered. Reads q/k/v, out (forward result), dout and drop_p; optional dprobs_ext (then
 * args->probs must be the FP32 probabilities the forward returned); writes dq/dk/dv (same layouts as q/k/v).
 * ext_heads > 0: dprobs_ext is known to be zero for heads >= ext_heads (the guided-attention loss reads the first two
 * heads of every layer, text_to_speech_loss.py:210-212) -- those heads skip its loads. out_f32 (optional): what the
 * forward wrote there. Scratch: delta [B*H*Tq] floats, dq_acc [B*Tq*H*64] floats (any contents: written before read).
 * dprobs_ext: columns [Tk, p_ld) and heads >= ext_heads (when 0 < ext_heads < H) are never read.
 * Relative positions (pe_k != NULL): args->ds additionally receives dS as BF16 [B,H,Tq,p_ld] for st5_attn_dqp_scatter
 * and the two table GEMMs; dq then holds only the q.k part of the gradient. */
int st5_attn_fused_bwd(const st5_attn_args* args, const void* psave, const float* inv_l, const float* out_f32,
                       float* delta, float* dq_acc, int32_t ext_heads, void* stream);

/* Tensor-core (bf16) attention path: the contractions run on st5_gemm_bf16 (batched over heads and utterances, q/k/v
 * read in place from the fused projection buffers); these three row kernels are the non-GEMM steps between them.
 * Row index = (b*H + h)*Tq + i everywhere; row pitch p_ld (multiple of 8, >= Tk); dropout indices as in st5_attn_fwd.
 *   softmax_fwd: P = softmax(S + QP[i][clamp(i-j)+maxpos] + masks); writes P (bf16), optionally fp32 probabilities
 *                (may alias s) and dropout(P) (bf16). s already holds scale*q.k, qp (optional) scale*q.pe_k^T [rows][2*maxpos].
 *   ds:          dS = P * (dropout_bwd(dP) + dP_ext - rowsum(P * (...))) (bf16); optionally re-emits dropout(P).
 *   dqp_scatter: dQP[row][r] = sum over keys j with clamp(i-j)+maxpos == r of dS[row][j]  (gradient wrt QP); output rows
 *                in the order of dS ((b, h, i)), or with h_major != 0 as (h, b, i). */
int st5_attn_softmax_fwd(const float* s, const float* qp, int64_t qp_ld, const uint8_t* key_pad, void* p_bf16,
                         float* probs_f32, void* pdrop_bf16, int32_t B, int32_t H, int32_t Tq, int32_t Tk, int64_t p_ld,
                         int32_t causal, int32_t maxpos, float drop_p, uint64_t seed, uint64_t offset, void* stream);
int st5_attn_ds(const void* p_bf16, const float* dp, const float* dp_ext, void* ds_bf16, void* pdrop_bf16, int32_t B,
                int32_t H, int32_t Tq, int32_t Tk, int64_t p_ld, float drop_p, uint64_t seed, uint64_t offset,
                void* stream);
int st5_attn_dqp_scatter(const void* ds_bf16, void* dqp_bf16, int32_t B, int32_t H, int32_t Tq, int32_t Tk,
                         int64_t p_ld, int32_t maxpos, int32_t h_major, void* stream);

/* ------------------------------------------------------------------------------------------------- BatchNorm1d
 * espnet Tacotron2 Postnet block (speech_decoder_postnet.py:39-51): y = dropout(act(BN(x))) on channels-last
 * rows [rows][C] (row pitches x_ld, y_ld, dy_ld, dx_ld); training statistics over all rows (padded frames included, as
 * in the reference): save_mean / save_rstd from the biased variance (eps inside the square root), running_var updated
 * with the unbiased one. rows == 1 (torch refuses it) uses var = 0 and moves running_var towards that biased 0.
 * Eval (training == 0): save_mean / save_rstd are derived from the running statistics, which are only read.
 * y_pre (optional in forward, required by the backward when act != ST5_ACT_NONE, else it returns -2) is contiguous
 * [rows][C]: the value before act(). Dropout index = row * C + c. act: NONE, RELU or TANH. scratch: 2 * C floats (any
 * contents). Backward: dgamma / dbeta are accumulated (+=). */
int st5_bn_fwd(const void* x, int64_t x_ld, const float* gamma, const float* beta, float* running_mean,
               float* running_var, float* save_mean, float* save_rstd, void* y, int64_t y_ld, void* y_pre, int dtype,
               int64_t rows, int64_t C, int training, float momentum, float eps, int act, float drop_p, uint64_t seed,
               uint64_t offset, float* scratch, void* stream);
int st5_bn_bwd(const void* dy, int64_t dy_ld, const void* x, int64_t x_ld, const void* y_pre, const float* gamma,
               const float* save_mean, const float* save_rstd, void* dx, int64_t dx_ld, float* dgamma, float* dbeta,
               int dtype, int64_t rows, int64_t C, int act, float drop_p, uint64_t seed, uint64_t offset,
               float* scratch, void* stream);

/* ------------------------------------------------------------------------------------------------- waveform front end
 * (speech-input branch, SURVEY section 8a row 2)
 * Layer 0 of ConvFeatureExtractionModel in mode "default" (speech_encoder_prenet.py:290-327,349-354): Conv1d(1 -> C, K
 * taps, `stride`, no bias) + Fp32GroupNorm(C groups: statistics per utterance and channel over time) + GELU
 * (fairseq/modules/gelu.py:24), fused. wave [B, n_samples] fp32; w [C, K]; y [B, T0, C] channels-last in `dtype`,
 * T0 = (n_samples - K) / stride + 1; mean / rstd [B, C] are saved for the backward. The convolution is recomputed from
 * the waveform in every pass, so the [B, T0, C] tensor is written once (forward) and dy read twice (backward).
 * Samples past (T0 - 1) * stride + K of each row are not read. ws: st5_conv0_ws_floats(...) floats of scratch (any
 * contents). act: ST5_ACT_GELU or ST5_ACT_GELU_TANH. GroupNorm: biased variance over the T0 frames, eps inside the
 * square root (a constant channel gets rstd = eps^-1/2). Backward: dw [C, K], dgamma [C], dbeta [C] are ACCUMULATED
 * (+=); the input is the waveform: no input gradient. Returns, with nothing written: -2 unless B >= 1, 1 <= C <= 1024,
 * 1 <= K <= 16 and stride >= 1; -3 for another act; -4 when T0 < 1 (n_samples < K); -5 when a block's waveform segment,
 * (127 * stride + K) floats, exceeds 48 KiB (stride > 96). */
int64_t st5_conv0_ws_floats(int32_t B, int64_t n_samples, int32_t C, int32_t K, int32_t stride);
int st5_conv0_gn_gelu_fwd(const float* wave, const float* w, const float* gamma, const float* beta, void* y, int dtype,
                          float* mean, float* rstd, float* ws, int32_t B, int64_t n_samples, int32_t C, int32_t K,
                          int32_t stride, float eps, int act, void* stream);
int st5_conv0_gn_gelu_bwd(const void* dy, const float* wave, const float* w, const float* gamma, const float* beta,
                          const float* mean, const float* rstd, float* dw, float* dgamma, float* dbeta, float* ws,
                          int dtype, int32_t B, int64_t n_samples, int32_t C, int32_t K, int32_t stride, int act,
                          void* stream);

/* Layer 0 in extractor mode "layer_norm" (t5_transformer_large, models/speecht5.py:1421; block builder
 * speech_encoder_prenet.py:308-318): Conv1d(1 -> C, K taps, `stride`, no bias) + Fp32LayerNorm over the C channels of
 * each frame + GELU, fused in ONE pass (a warp per frame). y [B, T0, C] channels-last in `dtype`; mean / rstd [B * T0]
 * are saved for the backward. C even, C <= 512, K <= 16. Backward: dw [C, K], dgamma [C], dbeta [C] are ACCUMULATED
 * (+=); ws: st5_conv0_ln_ws_floats(...) floats of scratch (any contents); no input gradient (the input is the
 * waveform). Returns, with nothing written: -2 unless B >= 1, C even in [2, 512], 1 <= K <= 16 and stride >= 1; -3 for
 * another act; -4 when T0 < 1. No stride limit. */
int64_t st5_conv0_ln_ws_floats(int32_t B, int64_t n_samples, int32_t C, int32_t K, int32_t stride);
int st5_conv0_ln_gelu_fwd(const float* wave, const float* w, const float* gamma, const float* beta, void* y, int dtype,
                          float* mean, float* rstd, int32_t B, int64_t n_samples, int32_t C, int32_t K, int32_t stride,
                          float eps, int act, void* stream);
int st5_conv0_ln_gelu_bwd(const void* dy, const float* wave, const float* w, const float* gamma, const float* beta,
                          const float* mean, const float* rstd, float* dw, float* dgamma, float* dbeta, float* ws,
                          int dtype, int32_t B, int64_t n_samples, int32_t C, int32_t K, int32_t stride, int act,
                          void* stream);

/* ------------------------------------------------------------------------------------------------- CTC
 * (speech-input branch, SURVEY section 8a row 18)
 * Replaces F.log_softmax + F.ctc_loss(reduction="sum") of speech_to_text_loss.py:303-335 on the encoder's CTC head.
 * logits fp32, element (t, b, k) at t*ld_t + b*ld_b + k; targets: flat int64 labels, utterance b's at
 * targets[tgt_offsets[b] .. + target_lengths[b]); nll [B] receives the per-utterance negative log-likelihood (+inf for
 * an infeasible utterance, or 0 with zero_infinity); grad (optional, same addressing as logits) receives
 * d(sum_b nll_b)/d logits, zero for t >= input_lengths[b] and for infeasible utterances. S_max >= 2*max(target_lengths)+1
 * (<= 1024) is the scratch pitch; ws: st5_ctc_ws_floats(T, B, S_max) floats (row log-sum-exps, emission terms, alpha
 * and beta lattices). Three launches: row pass, the two recursions side by side in one CTA per utterance, gradient rows.
 * Utterances with input_lengths[b] <= 0 or 2*target_lengths[b]+1 > S_max are reported infeasible; rows t >= T are never
 * read (input_lengths > T counts as T). With grad != NULL, V <= 12288 (the gradient's per-symbol sums of a row live in
 * 48 KiB of shared memory), else -2 before any launch. */
int64_t st5_ctc_ws_floats(int32_t T, int32_t B, int32_t S_max);
int st5_ctc_loss(const float* logits, int64_t ld_t, int64_t ld_b, const int64_t* targets, const int64_t* tgt_offsets,
                 const int64_t* input_lengths, const int64_t* target_lengths, float* nll, float* grad, float* ws,
                 int32_t T, int32_t B, int32_t V, int32_t S_max, int32_t blank, int32_t zero_infinity, void* stream);

/* ------------------------------------------------------------------------------------------------- TTS criterion
 * The reductions of speecht5/criterions/text_to_speech_loss.py and their gradients (SURVEY section 8a row 17).
 * st5_tts_loss_fwd: Tacotron2Loss with use_masking (:217-345). after / before [B, L, D] fp32 contiguous, logits [B, L],
 * ys: element (b, l, c) at b*y_bs + l*D + c (the target tensor may be longer than L), labels: (b, l) at b*lab_bs + l,
 * olens int64 [B] (frames; the valid region of utterance b is l < olens[b] - olens[b] % r, and for r > 1 the stop label
 * of its last valid frame counts as 1, :161-166). out[0..2] = l1, l2, bce (means over valid frames, l1 / l2 also over D);
 * sums: scratch of st5_tts_loss_ws_floats(B, L) floats that st5_tts_loss_bwd reads back (sums[3] = number of valid
 * frames; the rest holds per-CTA partials, added in a fixed order: same inputs, same bits).
 * st5_tts_loss_bwd (gradient of text_to_speech_loss.py:288-330): g[3] = upstream gradients of (l1, l2, bce) in device memory; writes d_after, d_before [B, L, D] and
 * d_logits [B, L] everywhere (zeros outside the masks); sign(0) = 0 in the L1 gradient.
 * D % 4 == 0 selects 16-byte vector accesses: then after, before, ys (and d_after, d_before) must be 16-byte aligned
 * and y_bs a multiple of 4, else -2 before any launch. */
int64_t st5_tts_loss_ws_floats(int32_t B, int32_t L);
int64_t st5_guided_attn_ws_floats(int32_t n_layers, int32_t B, int32_t heads, int32_t T_out);
int st5_tts_loss_fwd(const float* after, const float* before, const float* logits, const float* ys, int64_t y_bs,
                     const float* labels, int64_t lab_bs, const int64_t* olens, int32_t B, int32_t L, int32_t D,
                     int32_t r, float pos_weight, float* sums, float* out, void* stream);
int st5_tts_loss_bwd(const float* after, const float* before, const float* logits, const float* ys, int64_t y_bs,
                     const float* labels, int64_t lab_bs, const int64_t* olens, const float* sums, const float* g,
                     int32_t B, int32_t L, int32_t D, int32_t r, float pos_weight, float* d_after, float* d_before,
                     float* d_logits, void* stream);
/* GuidedMultiHeadAttentionLoss (text_to_speech_loss.py:370-427) over the first `heads` heads of n_layers (<= 8) returned cross-attention
 * probability tensors att[i] = [B, H, T_out, p_ld] fp32: out[0] = alpha * sum_valid W * A / (sum_b il_b * ol_b * heads *
 * n_layers), W = 1 - exp(-(t_in / il - t_out / ol)^2 / (2 sigma^2)), ol = olens[b] / r, il = ilens[b]. The valid region
 * (t_out < min(T_out, ol), t_in < min(T_in, il)) and the normaliser take the clamped lengths; W divides by the unclamped
 * il and ol. gsum: scratch of
 * st5_guided_attn_ws_floats(n_layers, B, heads, T_out) floats (fixed-order partial sums)
 * read back by the backward, which writes datt[i] (same layout) = g[0] * d out / d att on heads < `heads`; the other
 * heads are cleared only with zero_rest != 0 (st5_attn_fused_bwd with ext_heads never reads them). */
int st5_guided_attn_fwd(const float* const* att, int32_t n_layers, int32_t B, int32_t H, int32_t heads, int32_t T_out,
                        int32_t T_in, int64_t p_ld, const int64_t* ilens, const int64_t* olens, int32_t r, float sigma,
                        float alpha, float* gsum, float* out, void* stream);
int st5_guided_attn_bwd(float* const* datt, int32_t n_layers, int32_t B, int32_t H, int32_t heads, int32_t T_out,
                        int32_t T_in, int64_t p_ld, const int64_t* ilens, const int64_t* olens, int32_t r, float sigma,
                        float alpha, const float* gsum, const float* g, int32_t zero_rest, void* stream);

/* ------------------------------------------------------------------------------------------------- speaker head
 * Speaker identification (s2c): SpeakerDecoderPostnet (speaker_decoder_postnet.py:129-197) with its margin layers
 * AngularMargin / AdditiveAngularMargin (speaker_decoder_postnet.py:16-126), and the s2c branch of SpeechtoTextLoss
 * (speech_to_text_loss.py:93-110 label_smoothed_nll_loss, :340-372 compute_loss / compute_accuracy).
 * st5_l2norm_rows_fwd: F.normalize(x, p=2, dim=1) (speaker_decoder_postnet.py:190-191): y[r] = x[r] / max(||x[r]||,
 * 1e-12) into fp32 y [rows, E] (contiguous); nrm [rows] receives ||x[r]|| for the backward. x: row r at x + r * x_ld in
 * `dtype`. st5_l2norm_rows_bwd: dx[r] = (dy[r] - y[r] <dy[r], y[r]>) / ||x[r]|| (dy[r] / 1e-12 on clamped rows), written
 * in `dtype` at dx + r * dx_ld, or ADDED to it with accumulate != 0 (fp32 only: a weight gradient buffer). */
int st5_l2norm_rows_fwd(const void* x, int64_t x_ld, int dtype, float* y, float* nrm, int64_t rows, int64_t E,
                        void* stream);
int st5_l2norm_rows_bwd(const float* dy, const float* y, const float* nrm, void* dx, int64_t dx_ld, int dtype,
                        int accumulate, int64_t rows, int64_t E, void* stream);
/* st5_margin_ce_fwd: one CTA per row b of x [B, N] fp32 (row pitch x_ld). Logits z: with mtarget == NULL, z = x; else
 * column mtarget[b] gets the margin of `mode` (AM: s (x - m); AAM: s phi with sine = sqrt(clamp(1 - x^2, 0, 1)),
 * phi = x cos m - sine sin m, kept where x > th = cos(pi - m) else x - mm, mm = sin(pi - m) m; easy_margin: kept where
 * x > 0 else x, speaker_decoder_postnet.py:118-126) and every other column s x. z_out (optional, pitch z_ld) receives z.
 * With target != NULL: log-softmax of z, then per row stats[4 b + 0..3] = label-smoothed loss (weights 1 - eps - eps_i
 * on the target, eps_i = eps / (N - 1) on every class), nll, arg-max correct (lowest index among equal maxima), valid;
 * all 0 on a row whose target is ignore_index; a target outside [0, N) (and not ignore_index) gives NaN loss and nll.
 * lse [B] is saved for the backward.
 * st5_margin_ce_bwd: d z from the loss (target != NULL: gstat[0] d loss + gstat[1] d nll per valid row, both device
 * floats) or given (dz_in, pitch dz_ld); dx [B, N] fp32 (pitch dx_ld) = d z . d z / d x, including d phi / d x on the
 * margin column (AAM: d sine / d x = -x / sine, taken as 0 where sine = 0, i.e. at |x| >= 1). Same margin arguments as
 * the forward. */
int st5_margin_ce_fwd(const float* x, int64_t x_ld, int32_t B, int32_t N, const int64_t* mtarget, int mode, float scale,
                      float margin, int easy_margin, float* z_out, int64_t z_ld, const int64_t* target, float eps,
                      int64_t ignore_index, float* stats, float* lse, void* stream);
int st5_margin_ce_bwd(const float* x, int64_t x_ld, int32_t B, int32_t N, const int64_t* mtarget, int mode, float scale,
                      float margin, int easy_margin, const int64_t* target, float eps, int64_t ignore_index,
                      const float* lse, const float* gstat, const float* dz_in, int64_t dz_ld, float* dx, int64_t dx_ld,
                      void* stream);
/* st5_time_mean_fwd: y[b, c] = mean over ALL t < T of x[b, t, c] (contiguous [B, T, C] in `dtype`; the reference pools
 * `encoder_out.transpose(0, 1).mean(1)` with padded frames included, models/speecht5.py:836-838). st5_time_mean_bwd:
 * dx[b, t, c] = dy[b, c] / T. */
int st5_time_mean_fwd(const void* x, void* y, int dtype, int64_t B, int64_t T, int64_t C, void* stream);
int st5_time_mean_bwd(const void* dy, void* dx, int dtype, int64_t B, int64_t T, int64_t C, void* stream);

/* ------------------------------------------------------------------------------------------------- optimizer
 * Replaces fairseq/optim/adam.py + fp16_optimizer.py:106-218 on a flat fp32 parameter buffer: one pass applies the
 * gradient scale (grad_mul x clip coefficient max_norm / (norm + 1e-6) capped at 1: fairseq/utils.py clip_grad_norm_,
 * fairseq/trainer.py:796-826), Adam as fairseq/optim/adam.py:Adam.step writes it (denominator sqrt(v) + eps, step size
 * lr * sqrt(1 - b2^t) / (1 - b1^t), weight decay p -= wd * lr * p) and refreshes the bf16 shadow copy the GEMMs read.
 * The clip norm is that of the grad_mul-scaled gradient: sqrt(*grad_norm_sq) * grad_mul (no clip when max_norm <= 0 or
 * grad_norm_sq is NULL). When *grad_norm_sq is NaN, inf or above 3e38 the launch changes nothing (p, m, v, shadow).
 * st5_sumsq accumulates sum(x^2) (the squared gradient norm) into *out; x must be 16-byte aligned (else -2).
 * lr_dev / step_dev: device-resident schedule state so that a captured CUDA graph stays valid across updates. lr_dev
 * replaces `lr` everywhere (also in the weight decay); step_dev replaces `step` (then `step` is not read, else it must
 * be >= 1: -2). p_bf16 may be NULL; p, g, m, v 16-byte aligned and p_bf16 8-byte aligned take the vector path. */
int st5_sumsq(const float* x, int64_t n, float* out /* 1 float, accumulated */, void* stream);
int st5_adam_step(float* p, const float* g, float* m, float* v, void* p_bf16, int64_t n, float lr, float beta1,
                  float beta2, float eps, float weight_decay, int64_t step, const float* grad_norm_sq, float max_norm,
                  float grad_mul, const float* lr_dev /* optional device lr */,
                  const int64_t* step_dev /* optional device step counter */, void* stream);

#ifdef __cplusplus
}
#endif
#endif
