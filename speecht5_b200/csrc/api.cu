// C-ABI entry points (include/speecht5_b200.h). Pure argument marshalling; kernels live in the other .cu files.
#include "../../include/speecht5_b200.h"
#include "gemm.cuh"
#include "kernels.cuh"
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

namespace st5 {
static thread_local char g_err[512] = "";
int set_error(int code, const char* where) {
  if (code == 0) return 0;
  if (code > 0) {
    const char* s = cudaGetErrorString((cudaError_t)code);
    if (code == (int)cudaErrorMemoryAllocation)
      snprintf(g_err, sizeof(g_err), "%s: CUDA out of memory (%s)", where, s);
    else
      snprintf(g_err, sizeof(g_err), "%s: CUDA error %d (%s)", where, code, s);
    cudaGetLastError();
  } else {
    snprintf(g_err, sizeof(g_err), "%s: invalid argument (code %d)", where, code);
  }
  return code;
}
bool pdl_enabled() {
  static const bool on = [] {
    const char* e = getenv("ST5_PDL");
    return e == nullptr || atoi(e) != 0;
  }();
  return on;
}
}  // namespace st5

using namespace st5;

extern "C" {

int st5_version(void) { return 100; }
const char* st5_last_error(void) { return g_err; }

int st5_device_ok(void) {
  int dev = 0;
  cudaDeviceProp prop;
  if (cudaGetDevice(&dev) != cudaSuccess) return set_error(-1, "st5_device_ok");
  if (cudaGetDeviceProperties(&prop, dev) != cudaSuccess) return set_error(-1, "st5_device_ok");
  if (prop.major != 9) return set_error(-2, "st5_device_ok: library is built for sm_90a only");
  return 0;
}

int st5_gemm_bf16(const st5_gemm_args* a, void* stream) {
  GemmDesc g;
  g.M = a->M; g.N = a->N; g.K = a->K; g.nb1 = a->nb1; g.nb2 = a->nb2;
  g.A = a->a; g.a_mn = a->a_mn; g.a_ld = a->a_ld; g.a_bs1 = a->a_bs1; g.a_bs2 = a->a_bs2;
  g.B = a->b; g.b_mn = a->b_mn; g.b_ld = a->b_ld; g.b_bs1 = a->b_bs1; g.b_bs2 = a->b_bs2;
  g.C = a->c; g.c_fp32 = a->c_fp32; g.c_ld = a->c_ld; g.c_bs1 = a->c_bs1; g.c_bs2 = a->c_bs2;
  g.C_pre = a->c_pre; g.bias = a->bias; g.bias2 = a->bias2; g.bias2_rows = a->bias2_rows;
  g.residual = a->residual; g.act = a->act; g.alpha = a->alpha; g.accumulate = a->accumulate;
  g.drop_p = a->drop_p; g.drop_seed = a->drop_seed; g.drop_offset = a->drop_offset;
  g.ag_pre = a->actgrad_pre; g.ag_act = a->actgrad_act;
  return set_error(gemm_launch(g, (cudaStream_t)stream), "st5_gemm_bf16");
}

int st5_cast_bf16(const float* src, int64_t src_ld, void* hi, void* lo, int64_t dst_ld, int64_t rows, int64_t cols,
                  void* stream) {
  return set_error(cast_bf16_launch(src, src_ld, hi, lo, dst_ld, rows, cols, (cudaStream_t)stream), "st5_cast_bf16");
}

int st5_posenc_fwd(const int64_t* tokens, const float* emb, const void* x, const float* pe, const float* alpha,
                   void* y, int dtype, int64_t B, int64_t T, int64_t C, float drop_p, uint64_t seed, uint64_t offset,
                   void* stream) {
  return set_error(posenc_fwd_launch(tokens, emb, x, pe, alpha, y, dtype, B, T, C, drop_p, seed, offset,
                                     (cudaStream_t)stream),
                   "st5_posenc_fwd");
}
int st5_posenc_bwd(const void* dy, const int64_t* tokens, int64_t padding_idx, const float* pe, void* dx, float* demb,
                   float* dalpha, int dtype, int64_t B, int64_t T, int64_t C, float drop_p, uint64_t seed,
                   uint64_t offset, void* stream) {
  return set_error(posenc_bwd_launch(dy, tokens, padding_idx, pe, dx, demb, dalpha, dtype, B, T, C, drop_p, seed,
                                     offset, (cudaStream_t)stream),
                   "st5_posenc_bwd");
}

int st5_ln_fwd(const void* x, const void* residual, const float* gamma, const float* beta, void* y, void* s_out,
               float* mean, float* rstd, int dtype, int64_t rows, int64_t C, float eps, float drop_p, uint64_t seed,
               uint64_t offset, void* stream) {
  return set_error(ln_fwd_launch(x, residual, nullptr, gamma, beta, y, nullptr, s_out, mean, rstd, dtype, rows, C, eps,
                                 drop_p, seed, offset, (cudaStream_t)stream),
                   "st5_ln_fwd");
}
int st5_ln_fwd_stream(const void* x, const void* residual, const float* residual_f32, const float* gamma,
                      const float* beta, void* y, float* y_f32, void* s_out, float* mean, float* rstd, int dtype,
                      int64_t rows, int64_t C, float eps, float drop_p, uint64_t seed, uint64_t offset, void* stream) {
  return set_error(ln_fwd_launch(x, residual, residual_f32, gamma, beta, y, y_f32, s_out, mean, rstd, dtype, rows, C,
                                 eps, drop_p, seed, offset, (cudaStream_t)stream),
                   "st5_ln_fwd_stream");
}
int st5_ln_fwd_wide(const void* x, const void* residual, const float* gamma, const float* beta, void* y, float* mean,
                    float* rstd, int dtype, int64_t rows, int64_t C, float eps, void* stream) {
  return set_error(ln_fwd_wide_launch(x, residual, gamma, beta, y, mean, rstd, dtype, rows, C, eps, (cudaStream_t)stream),
                   "st5_ln_fwd_wide");
}
int64_t st5_ln_bwd_blocks(int64_t rows) { return ln_bwd_blocks(rows); }
int st5_ln_bwd(const void* dy, const void* s, const float* mean, const float* rstd, const float* gamma, void* ds,
               void* dx, float* dgamma, float* dbeta, float* dxsum, int dtype, int64_t rows, int64_t C, float drop_p,
               uint64_t seed, uint64_t offset, void* stream) {
  return set_error(ln_bwd_launch(dy, s, mean, rstd, gamma, ds, dx, dgamma, dbeta, dxsum, dtype, rows, C, drop_p,
                                 seed, offset, (cudaStream_t)stream),
                   "st5_ln_bwd");
}

int st5_lrelu_pad(const void* x, void* out, int64_t B, int64_t T, int64_t C, int64_t n_in, int32_t d, int32_t ph,
                  int32_t pad, float slope, void* stream) {
  return set_error(lrelu_pad_launch(x, out, B, T, C, n_in, d, ph, pad, slope, nullptr, 1, (cudaStream_t)stream),
                   "st5_lrelu_pad");
}
int st5_lrelu_pad_len(const void* x, void* out, int64_t B, int64_t T, int64_t C, int64_t n_in, int32_t d, int32_t ph,
                      int32_t pad, float slope, const int32_t* lengths, int32_t len_mult, void* stream) {
  return set_error(lrelu_pad_launch(x, out, B, T, C, n_in, d, ph, pad, slope, lengths, len_mult, (cudaStream_t)stream),
                   "st5_lrelu_pad_len");
}

int st5_dropout(const void* x, void* y, int dtype, int64_t n, float drop_p, uint64_t seed, uint64_t offset,
                void* stream) {
  return set_error(dropout_launch(x, y, dtype, n, drop_p, seed, offset, (cudaStream_t)stream), "st5_dropout");
}
int st5_act_bwd(const void* dy, const void* pre, void* dpre, int dtype, int act, int64_t n, float drop_p, uint64_t seed,
                uint64_t offset, void* stream) {
  return set_error(act_bwd_launch(dy, pre, dpre, dtype, act, n, drop_p, seed, offset, (cudaStream_t)stream),
                   "st5_act_bwd");
}
int st5_colsum(const void* x, int64_t ld, float* out, int dtype, int64_t rows, int64_t cols, int64_t group_rows,
               int accumulate, void* stream) {
  return set_error(colsum_launch(x, ld, out, dtype, rows, cols, group_rows, accumulate, (cudaStream_t)stream),
                   "st5_colsum");
}

int st5_attn_fwd(const st5_attn_args* a, void* stream) {
  return set_error(attn_fwd_launch(*a, (cudaStream_t)stream), "st5_attn_fwd");
}
int st5_attn_bwd(const st5_attn_args* a, void* stream) {
  return set_error(attn_bwd_launch(*a, (cudaStream_t)stream), "st5_attn_bwd");
}
int64_t st5_attn_decode_ws_floats(int32_t B, int32_t H, int32_t Tk, int32_t with_probs) {
  return attn_decode_ws_floats(B, H, Tk, with_probs);
}
int st5_attn_decode_fwd(const st5_attn_decode_args* a, void* stream) {
  return set_error(attn_decode_launch(*a, (cudaStream_t)stream), "st5_attn_decode_fwd");
}
int st5_attn_lineage_fwd(const st5_attn_lineage_args* a, void* stream) {
  return set_error(attn_lineage_launch(*a, (cudaStream_t)stream), "st5_attn_lineage_fwd");
}
int64_t st5_attn_decode_hd_ws_floats(int32_t B, int32_t H, int32_t Tk, int32_t with_probs, int32_t head_dim) {
  return attn_decode_hd_ws_floats(B, H, Tk, with_probs, head_dim);
}
int st5_attn_decode_hd_fwd(const st5_attn_decode_args* a, int32_t head_dim, void* stream) {
  return set_error(attn_decode_hd_launch(*a, head_dim, (cudaStream_t)stream), "st5_attn_decode_hd_fwd");
}
int st5_attn_lineage_hd_fwd(const st5_attn_lineage_args* a, int32_t head_dim, void* stream) {
  return set_error(attn_lineage_hd_launch(*a, head_dim, (cudaStream_t)stream), "st5_attn_lineage_hd_fwd");
}

int64_t st5_beam_topk_ws_floats(int32_t B, int32_t K) { return beam_topk_ws_floats(B, K); }
int st5_beam_topk(const void* logits, int64_t ld, int dtype, int32_t B, int32_t K, int32_t V, const float* cum,
                  const float* mask, float inv_temp, int32_t eos, const int64_t* t, const int64_t* min_len,
                  const int64_t* max_len, float* cand_score, int32_t* cand_token, int32_t* cand_beam, float* ws,
                  void* stream) {
  return set_error(beam_topk_launch(logits, ld, dtype, B, K, V, cum, mask, inv_temp, eos, t, min_len, max_len,
                                    cand_score, cand_token, cand_beam, ws, (cudaStream_t)stream),
                   "st5_beam_topk");
}
int st5_beam_topk_lm(const void* logits, int64_t ld, int dtype, int32_t B, int32_t K, int32_t V, const float* cum,
                     const float* mask, float inv_temp, int32_t eos, const int64_t* t, const int64_t* min_len,
                     const int64_t* max_len, float* cand_score, int32_t* cand_token, int32_t* cand_beam, float* ws,
                     const void* lm_logits, int64_t lm_ld, int lm_dtype, int32_t V_lm, float lm_weight, void* stream) {
  return set_error(beam_topk_lm_launch(logits, ld, dtype, B, K, V, cum, mask, inv_temp, eos, t, min_len, max_len,
                                       lm_logits, lm_ld, lm_dtype, V_lm, lm_weight, cand_score, cand_token, cand_beam,
                                       ws, (cudaStream_t)stream),
                   "st5_beam_topk_lm");
}
int st5_beam_update(int32_t B, int32_t K, int32_t V, int32_t T, int32_t eos, const int64_t* t, const int64_t* max_len,
                    int32_t normalize, float len_penalty, const float* cand_score, const int32_t* cand_token,
                    const int32_t* cand_beam, int32_t* lin, int32_t* tok, float* score, int32_t* ignore,
                    int32_t* finished, int32_t* parent, int64_t* cur_tok, float* cur_score, int32_t* fin_n,
                    int32_t* fin_tok, float* fin_pos, int32_t* fin_len, float* fin_score, int32_t* stop, void* stream) {
  return set_error(beam_update_launch(B, K, V, T, eos, t, max_len, normalize, len_penalty, cand_score, cand_token,
                                      cand_beam, lin, tok, score, ignore, finished, parent, cur_tok, cur_score, fin_n,
                                      fin_tok, fin_pos, fin_len, fin_score, stop, (cudaStream_t)stream),
                   "st5_beam_update");
}

int st5_bn_fwd(const void* x, int64_t x_ld, const float* gamma, const float* beta, float* running_mean,
               float* running_var, float* save_mean, float* save_rstd, void* y, int64_t y_ld, void* y_pre, int dtype,
               int64_t rows, int64_t C, int training, float momentum, float eps, int act, float drop_p, uint64_t seed,
               uint64_t offset, float* scratch, void* stream) {
  return set_error(bn_fwd_launch(x, x_ld, gamma, beta, running_mean, running_var, save_mean, save_rstd, y, y_ld, y_pre,
                                 dtype, rows, C, training, momentum, eps, act, drop_p, seed, offset, scratch,
                                 (cudaStream_t)stream),
                   "st5_bn_fwd");
}
int st5_bn_bwd(const void* dy, int64_t dy_ld, const void* x, int64_t x_ld, const void* y_pre, const float* gamma,
               const float* save_mean, const float* save_rstd, void* dx, int64_t dx_ld, float* dgamma, float* dbeta,
               int dtype, int64_t rows, int64_t C, int act, float drop_p, uint64_t seed, uint64_t offset,
               float* scratch, void* stream) {
  return set_error(bn_bwd_launch(dy, dy_ld, x, x_ld, y_pre, gamma, save_mean, save_rstd, dx, dx_ld, dgamma, dbeta,
                                 dtype, rows, C, act, drop_p, seed, offset, scratch, (cudaStream_t)stream),
                   "st5_bn_bwd");
}

int64_t st5_conv0_ln_ws_floats(int32_t B, int64_t n_samples, int32_t C, int32_t K, int32_t stride) {
  return conv0_ln_ws_floats(B, n_samples, C, K, stride);
}
int st5_conv0_ln_gelu_fwd(const float* wave, const float* w, const float* gamma, const float* beta, void* y, int dtype,
                          float* mean, float* rstd, int32_t B, int64_t n_samples, int32_t C, int32_t K, int32_t stride,
                          float eps, int act, void* stream) {
  return set_error(conv0_ln_fwd_launch(wave, w, gamma, beta, y, dtype, mean, rstd, B, n_samples, C, K, stride, eps, act,
                                       (cudaStream_t)stream),
                   "st5_conv0_ln_gelu_fwd");
}
int st5_conv0_ln_gelu_bwd(const void* dy, const float* wave, const float* w, const float* gamma, const float* beta,
                          const float* mean, const float* rstd, float* dw, float* dgamma, float* dbeta, float* ws,
                          int dtype, int32_t B, int64_t n_samples, int32_t C, int32_t K, int32_t stride, int act,
                          void* stream) {
  return set_error(conv0_ln_bwd_launch(dy, wave, w, gamma, beta, mean, rstd, dw, dgamma, dbeta, ws, dtype, B, n_samples,
                                       C, K, stride, act, (cudaStream_t)stream),
                   "st5_conv0_ln_gelu_bwd");
}
int st5_act_fwd(const void* x, void* y, int dtype, int act, int64_t n, void* stream) {
  return set_error(act_fwd_launch(x, y, dtype, act, n, (cudaStream_t)stream), "st5_act_fwd");
}

int64_t st5_conv0_ws_floats(int32_t B, int64_t n_samples, int32_t C, int32_t K, int32_t stride) {
  return conv0_ws_floats(B, n_samples, C, K, stride);
}
int st5_conv0_gn_gelu_fwd(const float* wave, const float* w, const float* gamma, const float* beta, void* y, int dtype,
                          float* mean, float* rstd, float* ws, int32_t B, int64_t n_samples, int32_t C, int32_t K,
                          int32_t stride, float eps, int act, void* stream) {
  return set_error(conv0_fwd_launch(wave, w, gamma, beta, y, dtype, mean, rstd, ws, B, n_samples, C, K, stride, eps, act,
                                    (cudaStream_t)stream),
                   "st5_conv0_gn_gelu_fwd");
}
int st5_conv0_gn_gelu_bwd(const void* dy, const float* wave, const float* w, const float* gamma, const float* beta,
                          const float* mean, const float* rstd, float* dw, float* dgamma, float* dbeta, float* ws,
                          int dtype, int32_t B, int64_t n_samples, int32_t C, int32_t K, int32_t stride, int act,
                          void* stream) {
  return set_error(conv0_bwd_launch(dy, wave, w, gamma, beta, mean, rstd, dw, dgamma, dbeta, ws, dtype, B, n_samples, C,
                                    K, stride, act, (cudaStream_t)stream),
                   "st5_conv0_gn_gelu_bwd");
}

int64_t st5_tts_loss_ws_floats(int32_t B, int32_t L) { return 4 + 4 * tts_loss_blocks(B, L); }
int64_t st5_guided_attn_ws_floats(int32_t n_layers, int32_t B, int32_t heads, int32_t T_out) {
  return 2 + guided_attn_blocks(n_layers, B, heads, T_out);
}
int st5_tts_loss_fwd(const float* after, const float* before, const float* logits, const float* ys, int64_t y_bs,
                     const float* labels, int64_t lab_bs, const int64_t* olens, int32_t B, int32_t L, int32_t D,
                     int32_t r, float pos_weight, float* sums, float* out, void* stream) {
  return set_error(tts_loss_fwd_launch(after, before, logits, ys, y_bs, labels, lab_bs, olens, B, L, D, r, pos_weight, sums,
                                       out, (cudaStream_t)stream),
                   "st5_tts_loss_fwd");
}
int st5_tts_loss_bwd(const float* after, const float* before, const float* logits, const float* ys, int64_t y_bs,
                     const float* labels, int64_t lab_bs, const int64_t* olens, const float* sums, const float* g,
                     int32_t B, int32_t L, int32_t D, int32_t r, float pos_weight, float* d_after, float* d_before,
                     float* d_logits, void* stream) {
  return set_error(tts_loss_bwd_launch(after, before, logits, ys, y_bs, labels, lab_bs, olens, sums, g, B, L, D, r,
                                       pos_weight, d_after, d_before, d_logits, (cudaStream_t)stream),
                   "st5_tts_loss_bwd");
}
int st5_guided_attn_fwd(const float* const* att, int32_t n_layers, int32_t B, int32_t H, int32_t heads, int32_t T_out,
                        int32_t T_in, int64_t p_ld, const int64_t* ilens, const int64_t* olens, int32_t r, float sigma,
                        float alpha, float* gsum, float* out, void* stream) {
  return set_error(guided_attn_fwd_launch(att, n_layers, B, H, heads, T_out, T_in, p_ld, ilens, olens, r, sigma, alpha,
                                          gsum, out, (cudaStream_t)stream),
                   "st5_guided_attn_fwd");
}
int st5_guided_attn_bwd(float* const* datt, int32_t n_layers, int32_t B, int32_t H, int32_t heads, int32_t T_out,
                        int32_t T_in, int64_t p_ld, const int64_t* ilens, const int64_t* olens, int32_t r, float sigma,
                        float alpha, const float* gsum, const float* g, int32_t zero_rest, void* stream) {
  return set_error(guided_attn_bwd_launch(datt, n_layers, B, H, heads, T_out, T_in, p_ld, ilens, olens, r, sigma, alpha,
                                          gsum, g, zero_rest, (cudaStream_t)stream),
                   "st5_guided_attn_bwd");
}

int64_t st5_ctc_ws_floats(int32_t T, int32_t B, int32_t S_max) { return ctc_ws_floats(T, B, S_max); }
int st5_ctc_loss(const float* logits, int64_t ld_t, int64_t ld_b, const int64_t* targets, const int64_t* tgt_offsets,
                 const int64_t* input_lengths, const int64_t* target_lengths, float* nll, float* grad, float* ws,
                 int32_t T, int32_t B, int32_t V, int32_t S_max, int32_t blank, int32_t zero_infinity, void* stream) {
  return set_error(ctc_loss_launch(logits, ld_t, ld_b, targets, tgt_offsets, input_lengths, target_lengths, nll, grad,
                                   ws, T, B, V, S_max, blank, zero_infinity, (cudaStream_t)stream),
                   "st5_ctc_loss");
}

int st5_l2norm_rows_fwd(const void* x, int64_t x_ld, int dtype, float* y, float* nrm, int64_t rows, int64_t E,
                        void* stream) {
  return set_error(l2norm_rows_fwd_launch(x, x_ld, dtype, y, nrm, rows, E, (cudaStream_t)stream), "st5_l2norm_rows_fwd");
}
int st5_l2norm_rows_bwd(const float* dy, const float* y, const float* nrm, void* dx, int64_t dx_ld, int dtype,
                        int accumulate, int64_t rows, int64_t E, void* stream) {
  return set_error(l2norm_rows_bwd_launch(dy, y, nrm, dx, dx_ld, dtype, accumulate, rows, E, (cudaStream_t)stream),
                   "st5_l2norm_rows_bwd");
}
int st5_margin_ce_fwd(const float* x, int64_t x_ld, int32_t B, int32_t N, const int64_t* mtarget, int mode, float scale,
                      float margin, int easy_margin, float* z_out, int64_t z_ld, const int64_t* target, float eps,
                      int64_t ignore_index, float* stats, float* lse, void* stream) {
  return set_error(margin_ce_fwd_launch(x, x_ld, B, N, mtarget, mode, scale, margin, easy_margin, z_out, z_ld, target,
                                        eps, ignore_index, stats, lse, (cudaStream_t)stream),
                   "st5_margin_ce_fwd");
}
int st5_margin_ce_bwd(const float* x, int64_t x_ld, int32_t B, int32_t N, const int64_t* mtarget, int mode, float scale,
                      float margin, int easy_margin, const int64_t* target, float eps, int64_t ignore_index,
                      const float* lse, const float* gstat, const float* dz_in, int64_t dz_ld, float* dx, int64_t dx_ld,
                      void* stream) {
  return set_error(margin_ce_bwd_launch(x, x_ld, B, N, mtarget, mode, scale, margin, easy_margin, target, eps,
                                        ignore_index, lse, gstat, dz_in, dz_ld, dx, dx_ld, (cudaStream_t)stream),
                   "st5_margin_ce_bwd");
}
int st5_time_mean_fwd(const void* x, void* y, int dtype, int64_t B, int64_t T, int64_t C, void* stream) {
  return set_error(time_mean_fwd_launch(x, y, dtype, B, T, C, (cudaStream_t)stream), "st5_time_mean_fwd");
}
int st5_time_mean_bwd(const void* dy, void* dx, int dtype, int64_t B, int64_t T, int64_t C, void* stream) {
  return set_error(time_mean_bwd_launch(dy, dx, dtype, B, T, C, (cudaStream_t)stream), "st5_time_mean_bwd");
}

int st5_sumsq(const float* x, int64_t n, float* out, void* stream) {
  return set_error(sumsq_launch(x, n, out, (cudaStream_t)stream), "st5_sumsq");
}
int st5_adam_step(float* p, const float* g, float* m, float* v, void* p_bf16, int64_t n, float lr, float beta1,
                  float beta2, float eps, float weight_decay, int64_t step, const float* grad_norm_sq, float max_norm,
                  float grad_mul, const float* lr_dev, const int64_t* step_dev, void* stream) {
  return set_error(adam_launch(p, g, m, v, p_bf16, n, lr, beta1, beta2, eps, weight_decay, step, grad_norm_sq, max_norm,
                               grad_mul, lr_dev, step_dev, (cudaStream_t)stream),
                   "st5_adam_step");
}

}  // extern "C"
