// The TTS criterion's reductions and their gradients as four launches instead of ~100 elementwise / reduction ATen
// kernels per update (speecht5/criterions/text_to_speech_loss.py):
//   Tacotron2Loss with use_masking (:217-345)   l1 = mean_valid |after - y| + |before - y|, l2 likewise with squares,
//                                               bce = mean_valid BCEWithLogits(stop logit, label; pos_weight)
//       over the frames l < olens[b] - olens[b] % r of utterance b; for r > 1 the stop label at the last valid frame
//       is forced to 1 (:161-166). Means run over valid frames (x odim for l1 / l2) like masked_select + mean.
//   GuidedMultiHeadAttentionLoss (:370-427)     alpha * sum_{valid} W * A / (sum_b il_b * ol_b * n_heads_total),
//       W[t_out, t_in] = 1 - exp(-(t_in / il - t_out / ol)^2 / (2 sigma^2)), over the first `heads` heads of the given
//       layers' returned cross-attention probabilities, ol = olens / r (decoder steps), il = text length.
// HBM-bound passes: forward reads after, before, y once (3 x B*L*odim fp32) -- warp per frame row, 16-byte loads.
#include "kernels.cuh"
#include <initializer_list>
#include <math_constants.h>

namespace st5 {

constexpr int CR_WARPS = 8;

__device__ __forceinline__ float softplus(float x) { return fmaxf(x, 0.f) + log1pf(__expf(-fabsf(x))); }

// Reductions are two-stage and ORDER-FIXED (the same inputs give the same bits: a training step is reproducible from its
// seed): every CTA writes its partial sums to its own slot, one CTA adds the slots in a fixed tree.
// sums: [0] sum |da| + |db|, [1] sum da^2 + db^2, [2] sum bce, [3] number of valid frames; sums[4 + 4*cta + i] = partials
__global__ void __launch_bounds__(CR_WARPS * 32)
    tts_loss_fwd_kernel(const float* __restrict__ after, const float* __restrict__ before,
                        const float* __restrict__ logits, const float* __restrict__ ys, int64_t y_bs,
                        const float* __restrict__ labels, int64_t lab_bs, const int64_t* __restrict__ olens, int B, int L,
                        int D, int r, float pos_weight, float* __restrict__ sums) {
  pdl_sync();
  __shared__ float red[4][CR_WARPS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * CR_WARPS + warp;
  float s1 = 0.f, s2 = 0.f, sb = 0.f, cnt = 0.f;
  if (row < (int64_t)B * L) {
    const int b = (int)(row / L), l = (int)(row - (int64_t)b * L);
    const int ol = (int)(olens[b] - olens[b] % r);
    if (l < ol) {
      const float* a = after + row * D;
      const float* bf = before + row * D;
      const float* y = ys + (int64_t)b * y_bs + (int64_t)l * D;
      if ((D & 3) == 0) {
        for (int c = lane * 4; c < D; c += 128) {
          const float4 va = *reinterpret_cast<const float4*>(a + c), vb = *reinterpret_cast<const float4*>(bf + c);
          const float4 vy = *reinterpret_cast<const float4*>(y + c);
          const float d0 = va.x - vy.x, d1 = va.y - vy.y, d2 = va.z - vy.z, d3 = va.w - vy.w;
          const float e0 = vb.x - vy.x, e1 = vb.y - vy.y, e2 = vb.z - vy.z, e3 = vb.w - vy.w;
          s1 += fabsf(d0) + fabsf(d1) + fabsf(d2) + fabsf(d3) + fabsf(e0) + fabsf(e1) + fabsf(e2) + fabsf(e3);
          s2 += d0 * d0 + d1 * d1 + d2 * d2 + d3 * d3 + e0 * e0 + e1 * e1 + e2 * e2 + e3 * e3;
        }
      } else {
        for (int c = lane; c < D; c += 32) {
          const float d0 = a[c] - y[c], e0 = bf[c] - y[c];
          s1 += fabsf(d0) + fabsf(e0);
          s2 += d0 * d0 + e0 * e0;
        }
      }
      if (lane == 0) {
        const float x = logits[row];
        const float t = (r > 1 && l == ol - 1) ? 1.f : labels[(int64_t)b * lab_bs + l];
        sb = pos_weight * t * softplus(-x) + (1.f - t) * softplus(x);
        cnt = 1.f;
      }
    }
  }
  s1 = warp_sum(s1); s2 = warp_sum(s2);
  if (lane == 0) { red[0][warp] = s1; red[1][warp] = s2; red[2][warp] = sb; red[3][warp] = cnt; }
  __syncthreads();
  if (threadIdx.x < 4) {
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < CR_WARPS; ++w) v += red[threadIdx.x][w];
    sums[4 + 4 * (int64_t)blockIdx.x + threadIdx.x] = v;
  }
}

// fixed-order sum of n partial vectors of width W (W <= 4) laid out [n][W] -> dst[0..W): one CTA of 256 threads
template <int W>
__device__ __forceinline__ void fixed_order_sum(const float* __restrict__ part, int64_t n, float* __restrict__ dst) {
  __shared__ float buf[W][256];
  float v[W];
#pragma unroll
  for (int i = 0; i < W; ++i) v[i] = 0.f;
  for (int64_t k = threadIdx.x; k < n; k += 256)
#pragma unroll
    for (int i = 0; i < W; ++i) v[i] += part[k * W + i];
#pragma unroll
  for (int i = 0; i < W; ++i) buf[i][threadIdx.x] = v[i];
  __syncthreads();
  for (int st = 128; st > 0; st >>= 1) {
    if ((int)threadIdx.x < st)
#pragma unroll
      for (int i = 0; i < W; ++i) buf[i][threadIdx.x] += buf[i][threadIdx.x + st];
    __syncthreads();
  }
  if (threadIdx.x == 0)
#pragma unroll
    for (int i = 0; i < W; ++i) dst[i] = buf[i][0];
  __syncthreads();
}

// out: [0] l1, [1] l2, [2] bce  (means over the valid frames; an empty batch gives zeros)
__global__ void __launch_bounds__(256)
    tts_loss_finalize_kernel(float* __restrict__ sums, int64_t nblk, int D, float* __restrict__ out) {
  pdl_sync();
  fixed_order_sum<4>(sums + 4, nblk, sums);
  if (threadIdx.x == 0) {
    const float n = sums[3];
    const float inv = n > 0.f ? 1.f / n : 0.f;
    out[0] = sums[0] * inv / (float)D;
    out[1] = sums[1] * inv / (float)D;
    out[2] = sums[2] * inv;
  }
}

// g: upstream gradients of (l1, l2, bce). d_after / d_before / d_logits are written everywhere (zeros outside the masks).
__global__ void __launch_bounds__(CR_WARPS * 32)
    tts_loss_bwd_kernel(const float* __restrict__ after, const float* __restrict__ before,
                        const float* __restrict__ logits, const float* __restrict__ ys, int64_t y_bs,
                        const float* __restrict__ labels, int64_t lab_bs, const int64_t* __restrict__ olens,
                        const float* __restrict__ sums, const float* __restrict__ g, int B, int L, int D, int r,
                        float pos_weight, float* __restrict__ d_after, float* __restrict__ d_before,
                        float* __restrict__ d_logits) {
  pdl_sync();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * CR_WARPS + warp;
  if (row >= (int64_t)B * L) return;
  const int b = (int)(row / L), l = (int)(row - (int64_t)b * L);
  const int ol = (int)(olens[b] - olens[b] % r);
  const bool valid = l < ol;
  const float n = sums[3];
  const float inv_n = n > 0.f ? 1.f / n : 0.f;
  const float k1 = g[0] * inv_n / (float)D, k2 = 2.f * g[1] * inv_n / (float)D;
  const float* a = after + row * D;
  const float* bf = before + row * D;
  const float* y = ys + (int64_t)b * y_bs + (int64_t)l * D;
  float* da = d_after + row * D;
  float* db = d_before + row * D;
  auto grad1 = [&](float d) { return valid ? (d > 0.f ? k1 : (d < 0.f ? -k1 : 0.f)) + k2 * d : 0.f; };
  if ((D & 3) == 0) {
    for (int c = lane * 4; c < D; c += 128) {
      float4 oa = make_float4(0.f, 0.f, 0.f, 0.f), ob = oa;
      if (valid) {
        const float4 va = *reinterpret_cast<const float4*>(a + c), vb = *reinterpret_cast<const float4*>(bf + c);
        const float4 vy = *reinterpret_cast<const float4*>(y + c);
        oa = make_float4(grad1(va.x - vy.x), grad1(va.y - vy.y), grad1(va.z - vy.z), grad1(va.w - vy.w));
        ob = make_float4(grad1(vb.x - vy.x), grad1(vb.y - vy.y), grad1(vb.z - vy.z), grad1(vb.w - vy.w));
      }
      *reinterpret_cast<float4*>(da + c) = oa;
      *reinterpret_cast<float4*>(db + c) = ob;
    }
  } else {
    for (int c = lane; c < D; c += 32) {
      da[c] = valid ? grad1(a[c] - y[c]) : 0.f;
      db[c] = valid ? grad1(bf[c] - y[c]) : 0.f;
    }
  }
  if (lane == 0) {
    float dl = 0.f;
    if (valid) {
      const float x = logits[row];
      const float t = (r > 1 && l == ol - 1) ? 1.f : labels[(int64_t)b * lab_bs + l];
      const float sg = 1.f / (1.f + __expf(-x));
      dl = g[2] * inv_n * (sg * (pos_weight * t + 1.f - t) - pos_weight * t);
    }
    d_logits[row] = dl;
  }
}

struct GuidedArgs {
  const float* att[8];   // per layer: [B][H][T_out][p_ld] fp32
  float* datt[8];        // backward only
  int n_layers, B, H, heads, T_out, T_in, r;
  int64_t p_ld;
  float inv_2sigma2, alpha;
};

// gsum[0] += sum W * A over the valid region of (layer, b, h < heads); one warp per (layer, b, h, t_out) row
__global__ void __launch_bounds__(CR_WARPS * 32)
    guided_attn_fwd_kernel(const GuidedArgs p, const int64_t* __restrict__ ilens, const int64_t* __restrict__ olens,
                           float* __restrict__ gsum) {
  pdl_sync();
  __shared__ float red[CR_WARPS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t nrows = (int64_t)p.n_layers * p.B * p.heads * p.T_out;
  const int64_t row = (int64_t)blockIdx.x * CR_WARPS + warp;
  float s = 0.f;
  if (row < nrows) {
    const int to = (int)(row % p.T_out);
    const int h = (int)((row / p.T_out) % p.heads);
    const int b = (int)((row / ((int64_t)p.T_out * p.heads)) % p.B);
    const int ly = (int)(row / ((int64_t)p.T_out * p.heads * p.B));
    const int ol = (int)min((int64_t)p.T_out, olens[b] / p.r), il = (int)min((int64_t)p.T_in, ilens[b]);
    if (to < ol) {
      const float* a = p.att[ly] + (((int64_t)b * p.H + h) * p.T_out + to) * p.p_ld;
      const float gx = (float)to / (float)(olens[b] / p.r);
      const float inv_il = 1.f / (float)ilens[b];
      for (int ti = lane; ti < il; ti += 32) {
        const float dlt = (float)ti * inv_il - gx;
        s += (1.f - __expf(-dlt * dlt * p.inv_2sigma2)) * a[ti];
      }
    }
  }
  s = warp_sum(s);
  if (lane == 0) red[warp] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < CR_WARPS; ++w) v += red[w];
    gsum[2 + (int64_t)blockIdx.x] = v;  // (summed in a fixed order by the finalize kernel)
  }
}

// gsum[0] = sum of the per-CTA partials gsum[2..], gsum[1] = normaliser sum_b il_b * ol_b * (heads * layers);
// out[0] = alpha * gsum[0] / gsum[1]
__global__ void __launch_bounds__(256)
    guided_attn_finalize_kernel(const GuidedArgs p, const int64_t* __restrict__ ilens, const int64_t* __restrict__ olens,
                                float* __restrict__ gsum, int64_t nblk, float* __restrict__ out) {
  pdl_sync();
  fixed_order_sum<1>(gsum + 2, nblk, gsum);
  if (threadIdx.x >= 32) return;
  float n = 0.f;
  for (int b = threadIdx.x; b < p.B; b += 32)
    n += (float)min((int64_t)p.T_out, olens[b] / p.r) * (float)min((int64_t)p.T_in, ilens[b]);
  n = warp_sum(n) * (float)(p.heads * p.n_layers);
  if (threadIdx.x == 0) {
    gsum[1] = n;
    out[0] = n > 0.f ? p.alpha * gsum[0] / n : 0.f;
  }
}

// dA = g * alpha * W / normaliser on the valid region of heads < `heads`, zero on the rest of those heads; heads >= `heads`
// are cleared only when zero_rest != 0 (a consumer that reads the first `heads` heads only -- st5_attn_fused_bwd with
// ext_heads -- does not need them touched)
__global__ void __launch_bounds__(CR_WARPS * 32)
    guided_attn_bwd_kernel(const GuidedArgs p, const int64_t* __restrict__ ilens, const int64_t* __restrict__ olens,
                           const float* __restrict__ gsum, const float* __restrict__ g, int zero_rest) {
  pdl_sync();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int hh = zero_rest ? p.H : p.heads;
  const int64_t nrows = (int64_t)p.n_layers * p.B * hh * p.T_out;
  const int64_t row = (int64_t)blockIdx.x * CR_WARPS + warp;
  if (row >= nrows) return;
  const int to = (int)(row % p.T_out);
  const int h = (int)((row / p.T_out) % hh);
  const int b = (int)((row / ((int64_t)p.T_out * hh)) % p.B);
  const int ly = (int)(row / ((int64_t)p.T_out * hh * p.B));
  float* d = p.datt[ly] + (((int64_t)b * p.H + h) * p.T_out + to) * p.p_ld;
  const int ol = (int)min((int64_t)p.T_out, olens[b] / p.r), il = (int)min((int64_t)p.T_in, ilens[b]);
  const bool live = h < p.heads && to < ol;
  const float n = gsum[1];
  const float k = (live && n > 0.f) ? g[0] * p.alpha / n : 0.f;
  const float gx = live ? (float)to / (float)(olens[b] / p.r) : 0.f;
  const float inv_il = live ? 1.f / (float)ilens[b] : 0.f;
  for (int ti = lane; ti < (int)p.p_ld; ti += 32) {
    float v = 0.f;
    if (live && ti < il) {
      const float dlt = (float)ti * inv_il - gx;
      v = k * (1.f - __expf(-dlt * dlt * p.inv_2sigma2));
    }
    d[ti] = v;
  }
}

int64_t tts_loss_blocks(int B, int L) { return ((int64_t)B * L + CR_WARPS - 1) / CR_WARPS; }

// D % 4 == 0 selects the float4 path, which needs every [B, L, D] operand 16-byte aligned and the ys batch pitch a
// multiple of 4; a misaligned call is rejected before any launch instead of faulting in the kernel. NULL passes.
static bool tts_vec_ok(int D, int64_t y_bs, std::initializer_list<const void*> ptrs) {
  if (D & 3) return true;
  if (y_bs & 3) return false;
  for (const void* q : ptrs)
    if (reinterpret_cast<uintptr_t>(q) & 15) return false;
  return true;
}
int64_t guided_attn_blocks(int n_layers, int B, int heads, int T_out) {
  return ((int64_t)n_layers * B * heads * T_out + CR_WARPS - 1) / CR_WARPS;
}

int tts_loss_fwd_launch(const float* after, const float* before, const float* logits, const float* ys, int64_t y_bs,
                        const float* labels, int64_t lab_bs, const int64_t* olens, int B, int L, int D, int r,
                        float pos_weight, float* sums, float* out, cudaStream_t s) {
  if (B <= 0 || L <= 0 || D <= 0 || r <= 0 || !tts_vec_ok(D, y_bs, {after, before, ys})) return -2;
  const int64_t nblk = tts_loss_blocks(B, L);
  launch_pdl(tts_loss_fwd_kernel, dim3((unsigned)nblk), dim3(CR_WARPS * 32), 0, s, after, before, logits, ys, y_bs, labels, lab_bs, olens, B, L, D, r, pos_weight, sums);
  launch_pdl(tts_loss_finalize_kernel, dim3(1), dim3(256), 0, s, sums, nblk, D, out);
  return (int)cudaGetLastError();
}

int tts_loss_bwd_launch(const float* after, const float* before, const float* logits, const float* ys, int64_t y_bs,
                        const float* labels, int64_t lab_bs, const int64_t* olens, const float* sums, const float* g,
                        int B, int L, int D, int r, float pos_weight, float* d_after, float* d_before, float* d_logits,
                        cudaStream_t s) {
  if (B <= 0 || L <= 0 || D <= 0 || r <= 0 || !tts_vec_ok(D, y_bs, {after, before, ys, d_after, d_before})) return -2;
  const int64_t rows = (int64_t)B * L;
  launch_pdl(tts_loss_bwd_kernel, dim3((unsigned)((rows + CR_WARPS - 1) / CR_WARPS)), dim3(CR_WARPS * 32), 0, s, after, before, logits, ys, y_bs, labels, lab_bs, olens, sums, g, B, L, D, r, pos_weight, d_after, d_before, d_logits);
  return (int)cudaGetLastError();
}

static int guided_fill(GuidedArgs& p, const float* const* att, float* const* datt, int n_layers, int B, int H, int heads,
                       int T_out, int T_in, int64_t p_ld, int r, float sigma, float alpha) {
  if (n_layers <= 0 || n_layers > 8 || B <= 0 || H <= 0 || heads <= 0 || heads > H || T_out <= 0 || T_in <= 0 ||
      p_ld < T_in || r <= 0 || !(sigma > 0.f))
    return -2;
  for (int i = 0; i < 8; ++i) {
    p.att[i] = i < n_layers && att != nullptr ? att[i] : nullptr;
    p.datt[i] = i < n_layers && datt != nullptr ? datt[i] : nullptr;
  }
  p.n_layers = n_layers; p.B = B; p.H = H; p.heads = heads; p.T_out = T_out; p.T_in = T_in; p.r = r; p.p_ld = p_ld;
  p.inv_2sigma2 = 1.f / (2.f * sigma * sigma);
  p.alpha = alpha;
  return 0;
}

int guided_attn_fwd_launch(const float* const* att, int n_layers, int B, int H, int heads, int T_out, int T_in,
                           int64_t p_ld, const int64_t* ilens, const int64_t* olens, int r, float sigma, float alpha,
                           float* gsum, float* out, cudaStream_t s) {
  GuidedArgs p;
  int rc = guided_fill(p, att, nullptr, n_layers, B, H, heads, T_out, T_in, p_ld, r, sigma, alpha);
  if (rc != 0) return rc;
  const int64_t nblk = guided_attn_blocks(n_layers, B, heads, T_out);
  launch_pdl(guided_attn_fwd_kernel, dim3((unsigned)nblk), dim3(CR_WARPS * 32), 0, s, p, ilens, olens, gsum);
  launch_pdl(guided_attn_finalize_kernel, dim3(1), dim3(256), 0, s, p, ilens, olens, gsum, nblk, out);
  return (int)cudaGetLastError();
}

int guided_attn_bwd_launch(float* const* datt, int n_layers, int B, int H, int heads, int T_out, int T_in, int64_t p_ld,
                           const int64_t* ilens, const int64_t* olens, int r, float sigma, float alpha,
                           const float* gsum, const float* g, int zero_rest, cudaStream_t s) {
  GuidedArgs p;
  int rc = guided_fill(p, nullptr, datt, n_layers, B, H, heads, T_out, T_in, p_ld, r, sigma, alpha);
  if (rc != 0) return rc;
  const int64_t rows = (int64_t)n_layers * B * (zero_rest ? H : heads) * T_out;
  launch_pdl(guided_attn_bwd_kernel, dim3((unsigned)((rows + CR_WARPS - 1) / CR_WARPS)), dim3(CR_WARPS * 32), 0, s, p, ilens, olens, gsum, g, zero_rest);
  return (int)cudaGetLastError();
}

}  // namespace st5
