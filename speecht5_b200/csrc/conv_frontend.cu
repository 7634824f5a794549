// First layer of the waveform feature extractor, fused: Conv1d(1 -> C, k, stride, no bias) + GroupNorm(C groups, i.e.
// per-(utterance, channel) statistics over time, fp32) + GELU, channels-last output for the window GEMMs of the next
// layers. Reference: speecht5/models/modules/speech_encoder_prenet.py:290-327,349-354 (block builder, mode "default"),
// fairseq Fp32GroupNorm, fairseq/modules/gelu.py:24. SURVEY section 8a row 2: in the reference this layer makes ~4 full
// passes over a 65 MB/utterance fp32 tensor (conv write, GroupNorm read x2, GELU read/write); here the k-tap
// convolution is cheap enough (k MACs per output) to be RECOMPUTED from the waveform in every pass, so nothing but the
// final bf16 activations (and 2 floats of statistics per utterance and channel) ever touches HBM:
//   forward : pass 1 statistics (reads the waveform only), pass 2 normalise + GELU + store  -> 1 write of [B, T, C]
//   backward: pass 1 sums of g and g*xhat (reads dy), pass 2 weight gradient (reads dy)      -> 2 reads of [B, T, C]
// The input is the waveform, so there is no input gradient. One thread per channel, TCH output frames per block, the
// waveform segment of the block staged in shared memory (every thread reads the same address: broadcast). A block holds
// at most C0_CMAX channels (grid.z walks the channel groups of wider layers): the backward kernels need up to ~80
// registers per thread, so a 1024-thread block would not fit the 64 K register file and would not launch.
// Checked on the device against oracle/speecht5_oracle_asr.py (tests/test_frontend_gpu.py) and, as an algorithm, through
// its CPU restatement (tests/test_kernel_algorithms_cpu.py).
#include "kernels.cuh"

namespace st5 {

constexpr int C0_TCH = 128;   // output frames per block
constexpr int C0_KMAX = 16;   // taps held in registers
constexpr int C0_CMAX = 512;  // channels per block (launch bounds of the one-thread-per-channel kernels: <= 128 regs)

__device__ __forceinline__ float c0_act(float z, int act) { return act == 4 ? gelu_tanh_fwd(z) : gelu_fwd(z); }

// stages wave[b][t0*S .. t0*S + (nt-1)*S + K) and this thread's taps; returns the number of frames of the block
__device__ __forceinline__ int c0_stage(const float* __restrict__ wave, const float* __restrict__ w, float* seg,
                                        float (&wr)[C0_KMAX], int64_t n, int T0, int C, int K, int S, int& t0) {
  const int b = blockIdx.y, c = blockIdx.z * blockDim.x + threadIdx.x;
  t0 = blockIdx.x * C0_TCH;
  const int nt = min(C0_TCH, T0 - t0);
  const int len = (nt - 1) * S + K;
  const float* src = wave + (int64_t)b * n + (int64_t)t0 * S;
  for (int i = threadIdx.x; i < len; i += blockDim.x) seg[i] = src[i];
#pragma unroll
  for (int k = 0; k < C0_KMAX; ++k) wr[k] = (k < K && c < C) ? w[c * K + k] : 0.f;
  __syncthreads();
  return nt;
}
__device__ __forceinline__ float c0_conv(const float* seg, const float (&wr)[C0_KMAX], int t, int K, int S) {
  float v = 0.f;
#pragma unroll
  for (int k = 0; k < C0_KMAX; ++k)
    if (k < K) v = fmaf(wr[k], seg[t * S + k], v);
  return v;
}

// part[((b * chunks + chunk) * 2 + {0: sum, 1: centred sum of squares}) * C + c]
__global__ void __launch_bounds__(C0_CMAX)
    conv0_stats_kernel(const float* __restrict__ wave, const float* __restrict__ w, float* __restrict__ part, int64_t n,
                       int T0, int C, int K, int S) {
  extern __shared__ float seg[];
  float wr[C0_KMAX];
  int t0;
  const int nt = c0_stage(wave, w, seg, wr, n, T0, C, K, S, t0);
  const int c = blockIdx.z * blockDim.x + threadIdx.x;
  if (c >= C) return;
  // one pass: sums of (v - pilot) and (v - pilot)^2 with the chunk's first value as the pilot, so the centred sum of
  // squares M2 = Q - S^2 / n is formed from numbers of the size of the deviations, not of the mean (the convolution
  // is the dominant cost of this kernel: a second, centred pass over the same frames doubled it)
  const float pilot = c0_conv(seg, wr, 0, K, S);
  float sh = 0.f, qh = 0.f;
  for (int t = 1; t < nt; ++t) {
    const float d = c0_conv(seg, wr, t, K, S) - pilot;
    sh += d;
    qh = fmaf(d, d, qh);
  }
  const float sum = fmaf((float)nt, pilot, sh);
  const float m2 = fmaxf(qh - sh * sh / (float)nt, 0.f);
  float* dst = part + ((int64_t)blockIdx.y * gridDim.x + blockIdx.x) * 2 * C;
  dst[c] = sum;
  dst[C + c] = m2;
}

// Chan's pairwise combination of the per-chunk (sum, M2) in double: mean / rstd per (utterance, channel).
// block (64 channels, 8 chunk groups), grid (B, C / 64): the ~250 chunks of a 10 s utterance are walked by 8 threads per
// channel and met in shared memory (one thread per channel would leave the grid at 8 CTAs).
constexpr int C0_FG = 8;
__global__ void __launch_bounds__(64 * C0_FG)
    conv0_finalize_kernel(const float* __restrict__ part, float* __restrict__ mean, float* __restrict__ rstd, int T0,
                          int C, int chunks, float eps) {
  __shared__ double red[C0_FG][64];
  const int b = blockIdx.x, c = blockIdx.y * 64 + threadIdx.x, g = threadIdx.y;
  const bool on = c < C;
  const float* p = part + (int64_t)b * chunks * 2 * C;
  double tot = 0.0;
  if (on)
    for (int i = g; i < chunks; i += C0_FG) tot += (double)p[(int64_t)i * 2 * C + c];
  red[g][threadIdx.x] = tot;
  __syncthreads();
  tot = 0.0;
#pragma unroll
  for (int k = 0; k < C0_FG; ++k) tot += red[k][threadIdx.x];
  __syncthreads();
  const double mu = tot / (double)T0;
  double m2 = 0.0;
  if (on)
    for (int i = g; i < chunks; i += C0_FG) {
      const int ni = min(C0_TCH, T0 - i * C0_TCH);
      const double d = (double)p[(int64_t)i * 2 * C + c] / (double)ni - mu;
      m2 += (double)p[(int64_t)i * 2 * C + C + c] + (double)ni * d * d;
    }
  red[g][threadIdx.x] = m2;
  __syncthreads();
  if (g == 0 && on) {
    m2 = 0.0;
#pragma unroll
    for (int k = 0; k < C0_FG; ++k) m2 += red[k][threadIdx.x];
    mean[b * C + c] = (float)mu;
    rstd[b * C + c] = (float)(1.0 / sqrt(m2 / (double)T0 + (double)eps));  // biased variance, as GroupNorm
  }
}

template <typename T>
__global__ void __launch_bounds__(C0_CMAX)
    conv0_apply_kernel(const float* __restrict__ wave, const float* __restrict__ w, const float* __restrict__ gamma,
                       const float* __restrict__ beta, const float* __restrict__ mean, const float* __restrict__ rstd,
                       T* __restrict__ y, int64_t n, int T0, int C, int K, int S, int act) {
  extern __shared__ float seg[];
  float wr[C0_KMAX];
  int t0;
  const int nt = c0_stage(wave, w, seg, wr, n, T0, C, K, S, t0);
  const int b = blockIdx.y, c = blockIdx.z * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float mu = mean[b * C + c];
  const float sc = rstd[b * C + c] * gamma[c];
  const float sh = beta[c];
  T* dst = y + ((int64_t)b * T0 + t0) * C + c;
  for (int t = 0; t < nt; ++t) {
    const float z = fmaf(c0_conv(seg, wr, t, K, S) - mu, sc, sh);
    stf<T>(dst + (int64_t)t * C, c0_act(z, act));
  }
}

// backward pass 1: part[.. * 2 + {0: sum g, 1: sum g * xhat}], g = dy * act'(z)
template <typename T>
__global__ void __launch_bounds__(C0_CMAX)
    conv0_bwd_sums_kernel(const T* __restrict__ dy, const float* __restrict__ wave, const float* __restrict__ w,
                          const float* __restrict__ gamma, const float* __restrict__ beta,
                          const float* __restrict__ mean, const float* __restrict__ rstd, float* __restrict__ part,
                          int64_t n, int T0, int C, int K, int S, int act) {
  extern __shared__ float seg[];
  float wr[C0_KMAX];
  int t0;
  const int nt = c0_stage(wave, w, seg, wr, n, T0, C, K, S, t0);
  const int b = blockIdx.y, c = blockIdx.z * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float mu = mean[b * C + c], rs = rstd[b * C + c], ga = gamma[c], be = beta[c];
  const T* src = dy + ((int64_t)b * T0 + t0) * C + c;
  float s1 = 0.f, s2 = 0.f;
  for (int t = 0; t < nt; ++t) {
    const float xh = (c0_conv(seg, wr, t, K, S) - mu) * rs;
    const float g = ldf<T>(src + (int64_t)t * C) * act_grad(fmaf(xh, ga, be), act);
    s1 += g;
    s2 = fmaf(g, xh, s2);
  }
  float* dst = part + ((int64_t)blockIdx.y * gridDim.x + blockIdx.x) * 2 * C;
  dst[c] = s1;
  dst[C + c] = s2;
}

// totals per (utterance, channel) + the affine gradients: dbeta[c] += sum_b S1, dgamma[c] += sum_b S2 (same block shape
// as conv0_finalize_kernel)
__global__ void __launch_bounds__(64 * C0_FG)
    conv0_bwd_finalize_kernel(const float* __restrict__ part, float* __restrict__ sums, float* __restrict__ dgamma,
                              float* __restrict__ dbeta, int C, int chunks) {
  __shared__ double red[2][C0_FG][64];
  const int b = blockIdx.x, c = blockIdx.y * 64 + threadIdx.x, g = threadIdx.y;
  const bool on = c < C;
  const float* p = part + (int64_t)b * chunks * 2 * C;
  double s1 = 0.0, s2 = 0.0;
  if (on)
    for (int i = g; i < chunks; i += C0_FG) {
      s1 += (double)p[(int64_t)i * 2 * C + c];
      s2 += (double)p[(int64_t)i * 2 * C + C + c];
    }
  red[0][g][threadIdx.x] = s1;
  red[1][g][threadIdx.x] = s2;
  __syncthreads();
  if (g == 0 && on) {
    s1 = s2 = 0.0;
#pragma unroll
    for (int k = 0; k < C0_FG; ++k) {
      s1 += red[0][k][threadIdx.x];
      s2 += red[1][k][threadIdx.x];
    }
    sums[(b * 2) * C + c] = (float)s1;
    sums[(b * 2 + 1) * C + c] = (float)s2;
    atomicAdd(dbeta + c, (float)s1);
    atomicAdd(dgamma + c, (float)s2);
  }
}

// backward pass 2: dv = rstd * gamma * (g - S1/T - xhat * S2/T); per-block partial dW[c][k] = sum_t dv[t] * wave[t*S + k]
template <typename T>
__global__ void __launch_bounds__(C0_CMAX)
    conv0_bwd_w_kernel(const T* __restrict__ dy, const float* __restrict__ wave, const float* __restrict__ w,
                       const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ mean,
                       const float* __restrict__ rstd, const float* __restrict__ sums, float* __restrict__ part,
                       int64_t n, int T0, int C, int K, int S, int act) {
  extern __shared__ float seg[];
  float wr[C0_KMAX];
  int t0;
  const int nt = c0_stage(wave, w, seg, wr, n, T0, C, K, S, t0);
  const int b = blockIdx.y, c = blockIdx.z * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float mu = mean[b * C + c], rs = rstd[b * C + c], ga = gamma[c], be = beta[c];
  const float inv_t = 1.f / (float)T0;
  const float m1 = sums[(b * 2) * C + c] * inv_t, m2 = sums[(b * 2 + 1) * C + c] * inv_t;
  const T* src = dy + ((int64_t)b * T0 + t0) * C + c;
  float acc[C0_KMAX];
#pragma unroll
  for (int k = 0; k < C0_KMAX; ++k) acc[k] = 0.f;
  for (int t = 0; t < nt; ++t) {
    const float xh = (c0_conv(seg, wr, t, K, S) - mu) * rs;
    const float g = ldf<T>(src + (int64_t)t * C) * act_grad(fmaf(xh, ga, be), act);
    const float dv = rs * ga * (g - m1 - xh * m2);
#pragma unroll
    for (int k = 0; k < C0_KMAX; ++k)
      if (k < K) acc[k] = fmaf(dv, seg[t * S + k], acc[k]);
  }
  float* dst = part + ((int64_t)blockIdx.y * gridDim.x + blockIdx.x) * (int64_t)C * K + (int64_t)c * K;
#pragma unroll
  for (int k = 0; k < C0_KMAX; ++k)
    if (k < K) dst[k] = acc[k];
}

// dw[i] += sum over the per-block partial rows (row range split over blockIdx.y, one atomic per thread)
__global__ void __launch_bounds__(128)
    conv0_reduce_w_kernel(const float* __restrict__ part, float* __restrict__ dw, int rows, int cols, int64_t ld) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= cols) return;
  const int per = (rows + gridDim.y - 1) / gridDim.y;
  const int r0 = blockIdx.y * per, r1 = min(rows, r0 + per);
  float s = 0.f;
  for (int r = r0; r < r1; ++r) s += part[(int64_t)r * ld + i];
  if (r1 > r0) atomicAdd(dw + i, s);
}

// ------------------------------------------------------------------------------------------------------------------
// Layer 0 in extractor mode "layer_norm" (the Large recipes, speech_encoder_prenet.py:308-318 + models/speecht5.py:1421):
// Conv1d(1 -> C, k, stride, no bias) + LayerNorm over the C channels of each frame (fairseq Fp32LayerNorm between two
// TransposeLast) + GELU. The statistics are per FRAME, so one pass suffices: a warp owns a frame, lane l holds the channel
// pairs (2l + 64j, 2l + 64j + 1), j < C0L_NP (C <= 512, even); the k taps of the frame are the same k waveform samples
// for every lane (broadcast loads), the transposed weights [k][C] sit in shared memory (float2 reads, conflict free);
// mean and centred variance by two rounds of warp shuffles on registers. HBM traffic: the waveform once, one store of
// [B, T0, C] and 2 floats per frame of statistics for the backward -- the store is the bound (SURVEY 8d conv FE row).
// Backward (no input gradient -- the input is the waveform): a PAIR of warps per frame recomputes the convolution and the
// normalised value; both form g = dy * act'(z) and the two LayerNorm sums (no exchange between them), warp r of the
// pair accumulates the weight-gradient taps k = r (mod 2) and one of dgamma / dbeta in registers over all its frames.
// Per-pair partial rows are summed by conv0_reduce_w_kernel.
constexpr int C0L_WARPS = 8;
constexpr int C0L_NP = 8;

template <typename T> __device__ __forceinline__ void st_pair(T* p, float a, float b);
template <> __device__ __forceinline__ void st_pair<float>(float* p, float a, float b) {
  *reinterpret_cast<float2*>(p) = make_float2(a, b);
}
template <> __device__ __forceinline__ void st_pair<__nv_bfloat16>(__nv_bfloat16* p, float a, float b) {
  *reinterpret_cast<__nv_bfloat162*>(p) = __floats2bfloat162_rn(a, b);
}
template <typename T> __device__ __forceinline__ float2 ld_pair(const T* p);
template <> __device__ __forceinline__ float2 ld_pair<float>(const float* p) { return *reinterpret_cast<const float2*>(p); }
template <> __device__ __forceinline__ float2 ld_pair<__nv_bfloat16>(const __nv_bfloat16* p) {
  return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(p));
}

// shared: wT[k * C + c] (K * C floats), then gamma[C], beta[C]
__device__ __forceinline__ void c0l_stage(const float* __restrict__ w, const float* __restrict__ gamma,
                                          const float* __restrict__ beta, float* sm, int C, int K) {
  for (int i = threadIdx.x; i < C * K; i += blockDim.x) {
    const int c = i / K, k = i - c * K;
    sm[k * C + c] = w[i];
  }
  for (int i = threadIdx.x; i < C; i += blockDim.x) {
    sm[K * C + i] = gamma[i];
    sm[K * C + C + i] = beta[i];
  }
  __syncthreads();
}
// the frame's taps (every lane the same addresses) and this lane's convolution outputs
__device__ __forceinline__ void c0l_conv(const float* __restrict__ src, const float* sm, float (&x)[C0_KMAX],
                                         float2 (&v)[C0L_NP], int C, int K, int lane) {
#pragma unroll
  for (int k = 0; k < C0_KMAX; ++k) x[k] = k < K ? __ldg(src + k) : 0.f;
#pragma unroll
  for (int j = 0; j < C0L_NP; ++j) {
    const int c = 2 * lane + 64 * j;
    float2 a = make_float2(0.f, 0.f);
    if (c < C) {
#pragma unroll
      for (int k = 0; k < C0_KMAX; ++k)
        if (k < K) {
          const float2 wk = *reinterpret_cast<const float2*>(sm + k * C + c);
          a.x = fmaf(wk.x, x[k], a.x);
          a.y = fmaf(wk.y, x[k], a.y);
        }
    }
    v[j] = a;
  }
}

template <typename T>
__global__ void __launch_bounds__(32 * C0L_WARPS)
    conv0_ln_fwd_kernel(const float* __restrict__ wave, const float* __restrict__ w, const float* __restrict__ gamma,
                        const float* __restrict__ beta, T* __restrict__ y, float* __restrict__ mean,
                        float* __restrict__ rstd, int64_t n, int T0, int64_t frames, int C, int K, int S, float eps,
                        int act) {
  extern __shared__ float sm[];
  c0l_stage(w, gamma, beta, sm, C, K);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float inv_c = 1.f / (float)C;
  for (int64_t f = (int64_t)blockIdx.x * C0L_WARPS + warp; f < frames; f += (int64_t)gridDim.x * C0L_WARPS) {
    const int64_t b = f / T0;
    const int t = (int)(f - b * T0);
    float x[C0_KMAX];
    float2 v[C0L_NP];
    c0l_conv(wave + b * n + (int64_t)t * S, sm, x, v, C, K, lane);
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < C0L_NP; ++j) s += v[j].x + v[j].y;  // (channels beyond C hold 0)
    const float mu = warp_sum(s) * inv_c;
    float q = 0.f;
#pragma unroll
    for (int j = 0; j < C0L_NP; ++j)
      if (2 * lane + 64 * j < C) {
        const float dx = v[j].x - mu, dy = v[j].y - mu;
        q = fmaf(dx, dx, fmaf(dy, dy, q));
      }
    const float rs = rsqrtf(warp_sum(q) * inv_c + eps);
    if (lane == 0) {
      mean[f] = mu;
      rstd[f] = rs;
    }
    T* dst = y + f * C;
#pragma unroll
    for (int j = 0; j < C0L_NP; ++j) {
      const int c = 2 * lane + 64 * j;
      if (c < C) {
        const float2 ga = *reinterpret_cast<const float2*>(sm + K * C + c);
        const float2 be = *reinterpret_cast<const float2*>(sm + K * C + C + c);
        st_pair<T>(dst + c, c0_act(fmaf((v[j].x - mu) * rs, ga.x, be.x), act),
                   c0_act(fmaf((v[j].y - mu) * rs, ga.y, be.y), act));
      }
    }
  }
}

// part row (pair p of CTA x): [C * K] weight-gradient taps (layout c * K + k), [C] dgamma, [C] dbeta
template <typename T, int KH>
__global__ void __launch_bounds__(32 * C0L_WARPS)
    conv0_ln_bwd_kernel(const T* __restrict__ dy, const float* __restrict__ wave, const float* __restrict__ w,
                        const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ mean,
                        const float* __restrict__ rstd, float* __restrict__ part, int64_t n, int T0, int64_t frames,
                        int C, int K, int S, int act) {
  extern __shared__ float sm[];
  c0l_stage(w, gamma, beta, sm, C, K);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int pair = warp >> 1, role = warp & 1;
  constexpr int PAIRS = C0L_WARPS / 2;
  const float inv_c = 1.f / (float)C;
  float2 aw[C0L_NP][KH], aff[C0L_NP];
#pragma unroll
  for (int j = 0; j < C0L_NP; ++j) {
    aff[j] = make_float2(0.f, 0.f);
#pragma unroll
    for (int i = 0; i < KH; ++i) aw[j][i] = make_float2(0.f, 0.f);
  }
  for (int64_t f = (int64_t)blockIdx.x * PAIRS + pair; f < frames; f += (int64_t)gridDim.x * PAIRS) {
    const int64_t b = f / T0;
    const int t = (int)(f - b * T0);
    const float* src = wave + b * n + (int64_t)t * S;
    float x[C0_KMAX], xr[KH];
    float2 v[C0L_NP];
    c0l_conv(src, sm, x, v, C, K, lane);
#pragma unroll
    for (int i = 0; i < KH; ++i) xr[i] = (2 * i + role < K) ? __ldg(src + 2 * i + role) : 0.f;
    const float mu = mean[f], rs = rstd[f];
    const T* g_in = dy + f * C;
    float s1 = 0.f, s2 = 0.f;
    float2 dxh[C0L_NP];
#pragma unroll
    for (int j = 0; j < C0L_NP; ++j) {
      const int c = 2 * lane + 64 * j;
      dxh[j] = make_float2(0.f, 0.f);
      if (c < C) {
        const float2 ga = *reinterpret_cast<const float2*>(sm + K * C + c);
        const float2 be = *reinterpret_cast<const float2*>(sm + K * C + C + c);
        const float2 d = ld_pair<T>(g_in + c);
        const float xh0 = (v[j].x - mu) * rs, xh1 = (v[j].y - mu) * rs;
        const float g0 = d.x * act_grad(fmaf(xh0, ga.x, be.x), act), g1 = d.y * act_grad(fmaf(xh1, ga.y, be.y), act);
        aff[j].x += role ? g0 : g0 * xh0;  // role 0: dgamma, role 1: dbeta
        aff[j].y += role ? g1 : g1 * xh1;
        dxh[j] = make_float2(g0 * ga.x, g1 * ga.y);
        s1 += dxh[j].x + dxh[j].y;
        s2 = fmaf(dxh[j].x, xh0, fmaf(dxh[j].y, xh1, s2));
        v[j] = make_float2(xh0, xh1);
      }
    }
    const float m1 = warp_sum(s1) * inv_c, m2 = warp_sum(s2) * inv_c;
#pragma unroll
    for (int j = 0; j < C0L_NP; ++j) {
      const float du0 = rs * (dxh[j].x - m1 - v[j].x * m2), du1 = rs * (dxh[j].y - m1 - v[j].y * m2);
      if (2 * lane + 64 * j < C) {
#pragma unroll
        for (int i = 0; i < KH; ++i) {
          aw[j][i].x = fmaf(du0, xr[i], aw[j][i].x);
          aw[j][i].y = fmaf(du1, xr[i], aw[j][i].y);
        }
      }
    }
  }
  float* row = part + ((int64_t)blockIdx.x * PAIRS + pair) * ((int64_t)C * K + 2 * C);
#pragma unroll
  for (int j = 0; j < C0L_NP; ++j) {
    const int c = 2 * lane + 64 * j;
    if (c < C) {
#pragma unroll
      for (int i = 0; i < KH; ++i) {
        const int k = 2 * i + role;
        if (k < K) {
          row[(int64_t)c * K + k] = aw[j][i].x;
          row[(int64_t)(c + 1) * K + k] = aw[j][i].y;
        }
      }
      float* a = row + (int64_t)C * K + (role ? C : 0);
      a[c] = aff[j].x;
      a[c + 1] = aff[j].y;
    }
  }
}

static inline int c0_frames(int64_t n, int K, int S) { return n < K ? 0 : (int)((n - K) / S + 1); }
// grid (chunks, B, channel groups), block: the channels of one group rounded up to whole warps
static inline dim3 c0_grid(int chunks, int B, int C) { return dim3(chunks, B, (C + C0_CMAX - 1) / C0_CMAX); }
static inline dim3 c0_block(int C) {
  const int groups = (C + C0_CMAX - 1) / C0_CMAX;
  return dim3(((C + groups - 1) / groups + 31) / 32 * 32);
}

int64_t conv0_ws_floats(int32_t B, int64_t n, int32_t C, int32_t K, int32_t S) {
  const int T0 = c0_frames(n, K, S);
  const int64_t chunks = (T0 + C0_TCH - 1) / C0_TCH;
  return (int64_t)B * chunks * C * (K > 2 ? K : 2) + 2 * (int64_t)B * C;
}

static int c0_check(int32_t B, int64_t n, int32_t C, int32_t K, int32_t S, int act) {
  if (B <= 0 || C <= 0 || C > 1024 || K <= 0 || K > C0_KMAX || S <= 0) return -2;
  if (act != 2 && act != 4) return -3;
  if (c0_frames(n, K, S) <= 0) return -4;
  return 0;
}

int conv0_fwd_launch(const float* wave, const float* w, const float* gamma, const float* beta, void* y, int dtype,
                     float* mean, float* rstd, float* ws, int32_t B, int64_t n, int32_t C, int32_t K, int32_t S,
                     float eps, int act, cudaStream_t st) {
  const int rc = c0_check(B, n, C, K, S, act);
  if (rc) return rc;
  const int T0 = c0_frames(n, K, S);
  const int chunks = (T0 + C0_TCH - 1) / C0_TCH;
  const dim3 grid = c0_grid(chunks, B, C), block = c0_block(C);
  const size_t smem = ((size_t)(C0_TCH - 1) * S + K) * sizeof(float);
  if (smem > 48 * 1024) return -5;
  conv0_stats_kernel<<<grid, block, smem, st>>>(wave, w, ws, n, T0, C, K, S);
  conv0_finalize_kernel<<<dim3(B, (C + 63) / 64), dim3(64, C0_FG), 0, st>>>(ws, mean, rstd, T0, C, chunks, eps);
  if (dtype == ST5_BF16)
    conv0_apply_kernel<__nv_bfloat16><<<grid, block, smem, st>>>(wave, w, gamma, beta, mean, rstd,
                                                                 reinterpret_cast<__nv_bfloat16*>(y), n, T0, C, K, S, act);
  else
    conv0_apply_kernel<float><<<grid, block, smem, st>>>(wave, w, gamma, beta, mean, rstd, reinterpret_cast<float*>(y),
                                                        n, T0, C, K, S, act);
  return (int)cudaGetLastError();
}

int conv0_bwd_launch(const void* dy, const float* wave, const float* w, const float* gamma, const float* beta,
                     const float* mean, const float* rstd, float* dw, float* dgamma, float* dbeta, float* ws, int dtype,
                     int32_t B, int64_t n, int32_t C, int32_t K, int32_t S, int act, cudaStream_t st) {
  const int rc = c0_check(B, n, C, K, S, act);
  if (rc) return rc;
  const int T0 = c0_frames(n, K, S);
  const int chunks = (T0 + C0_TCH - 1) / C0_TCH;
  const dim3 grid = c0_grid(chunks, B, C), block = c0_block(C);
  const size_t smem = ((size_t)(C0_TCH - 1) * S + K) * sizeof(float);
  if (smem > 48 * 1024) return -5;
  float* sums = ws + (int64_t)B * chunks * C * (K > 2 ? K : 2);
  if (dtype == ST5_BF16) {
    const __nv_bfloat16* g = reinterpret_cast<const __nv_bfloat16*>(dy);
    conv0_bwd_sums_kernel<__nv_bfloat16><<<grid, block, smem, st>>>(g, wave, w, gamma, beta, mean, rstd, ws, n, T0, C, K,
                                                                    S, act);
    if (const cudaError_t e = cudaGetLastError()) return (int)e;  // nothing accumulated yet
    conv0_bwd_finalize_kernel<<<dim3(B, (C + 63) / 64), dim3(64, C0_FG), 0, st>>>(ws, sums, dgamma, dbeta, C, chunks);
    conv0_bwd_w_kernel<__nv_bfloat16><<<grid, block, smem, st>>>(g, wave, w, gamma, beta, mean, rstd, sums, ws, n, T0, C,
                                                                 K, S, act);
  } else {
    const float* g = reinterpret_cast<const float*>(dy);
    conv0_bwd_sums_kernel<float><<<grid, block, smem, st>>>(g, wave, w, gamma, beta, mean, rstd, ws, n, T0, C, K, S, act);
    if (const cudaError_t e = cudaGetLastError()) return (int)e;  // nothing accumulated yet
    conv0_bwd_finalize_kernel<<<dim3(B, (C + 63) / 64), dim3(64, C0_FG), 0, st>>>(ws, sums, dgamma, dbeta, C, chunks);
    conv0_bwd_w_kernel<float><<<grid, block, smem, st>>>(g, wave, w, gamma, beta, mean, rstd, sums, ws, n, T0, C, K, S,
                                                         act);
  }
  const int cols = C * K;
  conv0_reduce_w_kernel<<<dim3((cols + 127) / 128, 32), 128, 0, st>>>(ws, dw, B * chunks, cols, cols);
  return (int)cudaGetLastError();
}

// ---- layer_norm mode launchers
static inline int c0l_grid(int64_t frames, int per_cta) {
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int64_t want = (frames + per_cta - 1) / per_cta;
  return (int)(want < 2LL * sms ? (want > 0 ? want : 1) : 2LL * sms);
}
static int c0l_check(int32_t B, int64_t n, int32_t C, int32_t K, int32_t S, int act) {
  if (B <= 0 || C <= 0 || C > 64 * C0L_NP || (C & 1) || K <= 0 || K > C0_KMAX || S <= 0) return -2;
  if (act != 2 && act != 4) return -3;
  if (c0_frames(n, K, S) <= 0) return -4;
  return 0;
}
int64_t conv0_ln_ws_floats(int32_t B, int64_t n, int32_t C, int32_t K, int32_t S) {
  const int64_t frames = (int64_t)B * c0_frames(n, K, S);
  return (int64_t)c0l_grid(frames, C0L_WARPS / 2) * (C0L_WARPS / 2) * ((int64_t)C * K + 2 * C);
}

int conv0_ln_fwd_launch(const float* wave, const float* w, const float* gamma, const float* beta, void* y, int dtype,
                        float* mean, float* rstd, int32_t B, int64_t n, int32_t C, int32_t K, int32_t S, float eps,
                        int act, cudaStream_t st) {
  const int rc = c0l_check(B, n, C, K, S, act);
  if (rc) return rc;
  const int T0 = c0_frames(n, K, S);
  const int64_t frames = (int64_t)B * T0;
  const size_t smem = ((size_t)C * K + 2 * C) * sizeof(float);
  const int grid = c0l_grid(frames, C0L_WARPS);
  if (dtype == ST5_BF16)
    conv0_ln_fwd_kernel<__nv_bfloat16><<<grid, 32 * C0L_WARPS, smem, st>>>(
        wave, w, gamma, beta, reinterpret_cast<__nv_bfloat16*>(y), mean, rstd, n, T0, frames, C, K, S, eps, act);
  else
    conv0_ln_fwd_kernel<float><<<grid, 32 * C0L_WARPS, smem, st>>>(wave, w, gamma, beta, reinterpret_cast<float*>(y),
                                                                   mean, rstd, n, T0, frames, C, K, S, eps, act);
  return (int)cudaGetLastError();
}

template <typename T>
static void c0l_bwd_run(const void* dy, const float* wave, const float* w, const float* gamma, const float* beta,
                        const float* mean, const float* rstd, float* ws, int64_t n, int T0, int64_t frames, int C, int K,
                        int S, int act, int grid, size_t smem, cudaStream_t st) {
  const T* g = reinterpret_cast<const T*>(dy);
  if (K <= 10)
    conv0_ln_bwd_kernel<T, 5><<<grid, 32 * C0L_WARPS, smem, st>>>(g, wave, w, gamma, beta, mean, rstd, ws, n, T0, frames,
                                                                  C, K, S, act);
  else
    conv0_ln_bwd_kernel<T, C0_KMAX / 2><<<grid, 32 * C0L_WARPS, smem, st>>>(g, wave, w, gamma, beta, mean, rstd, ws, n,
                                                                            T0, frames, C, K, S, act);
}

int conv0_ln_bwd_launch(const void* dy, const float* wave, const float* w, const float* gamma, const float* beta,
                        const float* mean, const float* rstd, float* dw, float* dgamma, float* dbeta, float* ws,
                        int dtype, int32_t B, int64_t n, int32_t C, int32_t K, int32_t S, int act, cudaStream_t st) {
  const int rc = c0l_check(B, n, C, K, S, act);
  if (rc) return rc;
  const int T0 = c0_frames(n, K, S);
  const int64_t frames = (int64_t)B * T0;
  const size_t smem = ((size_t)C * K + 2 * C) * sizeof(float);
  const int grid = c0l_grid(frames, C0L_WARPS / 2);
  if (dtype == ST5_BF16)
    c0l_bwd_run<__nv_bfloat16>(dy, wave, w, gamma, beta, mean, rstd, ws, n, T0, frames, C, K, S, act, grid, smem, st);
  else
    c0l_bwd_run<float>(dy, wave, w, gamma, beta, mean, rstd, ws, n, T0, frames, C, K, S, act, grid, smem, st);
  const int rows = grid * (C0L_WARPS / 2);
  const int64_t ld = (int64_t)C * K + 2 * C;
  conv0_reduce_w_kernel<<<dim3((C * K + 127) / 128, 32), 128, 0, st>>>(ws, dw, rows, C * K, ld);
  conv0_reduce_w_kernel<<<dim3((C + 127) / 128, 32), 128, 0, st>>>(ws + (int64_t)C * K, dgamma, rows, C, ld);
  conv0_reduce_w_kernel<<<dim3((C + 127) / 128, 32), 128, 0, st>>>(ws + (int64_t)C * K + C, dbeta, rows, C, ld);
  return (int)cudaGetLastError();
}

}  // namespace st5
