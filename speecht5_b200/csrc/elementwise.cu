// Memory-bound helpers around the GEMMs: casts, (embedding +) scaled positional encoding, dropout, activation
// backward, column sums (bias gradients). All are HBM-bound streaming kernels: one pass, coalesced, fp32 math.
#include "kernels.cuh"
#include "vec8.cuh"
#include "ptx.cuh"
#include "gemm.cuh"

namespace st5 {

static inline int grid_for(int64_t n, int threads) {
  int64_t g = (n + threads - 1) / threads;
  return (int)(g > 132 * 32 ? 132 * 32 : (g < 1 ? 1 : g));
}

// ------------------------------------------------------------------ fp32 -> bf16 (hi [, lo])
__global__ void cast_bf16_kernel(const float* __restrict__ src, int64_t src_ld, __nv_bfloat16* __restrict__ hi,
                                 __nv_bfloat16* __restrict__ lo, int64_t dst_ld, int64_t rows, int64_t cols) {
  pdl_sync();
  const int64_t n = rows * cols;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / cols, c = i - r * cols;
    const float v = src[r * src_ld + c];
    const __nv_bfloat16 h = __float2bfloat16(v);
    hi[r * dst_ld + c] = h;
    if (lo != nullptr) lo[r * dst_ld + c] = __float2bfloat16(v - __bfloat162float(h));
  }
}
int cast_bf16_launch(const float* src, int64_t src_ld, void* hi, void* lo, int64_t dst_ld, int64_t rows, int64_t cols,
                     cudaStream_t s) {
  if (rows * cols == 0) return 0;
  launch_pdl(cast_bf16_kernel, dim3(grid_for(rows * cols, 256)), dim3(256), 0, s, src, src_ld, (__nv_bfloat16*)hi, (__nv_bfloat16*)lo, dst_ld, rows, cols);
  return (int)cudaGetLastError();
}

// ------------------------------------------------------------------ (embedding +) alpha * PE, dropout
template <typename T>
__global__ void posenc_fwd_kernel(const int64_t* __restrict__ tokens, const float* __restrict__ emb,
                                  const T* __restrict__ x, const float* __restrict__ pe,
                                  const float* __restrict__ alpha, T* __restrict__ y, int64_t B, int64_t T_, int64_t C,
                                  uint32_t thr, float dscale, uint64_t seed, uint64_t offset) {
  resolve_seed(seed, offset);
  const int64_t n = B * T_ * C;
  const float a = *alpha;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t bt = i / C, c = i - bt * C;
    const int64_t t = bt % T_;
    float v = tokens != nullptr ? emb[tokens[bt] * C + c] : ldf(x + i);
    v += a * pe[t * C + c];
    if (thr != 0) v = dropout_keep(seed, offset, (uint64_t)i, thr) ? v * dscale : 0.f;
    stf(y + i, v);
  }
}
// Eight channels per thread (C % 8 == 0, 16-byte aligned rows): one Philox call per 8 elements instead of one per element
// (the same decisions: dropout_keep(i) is lane i & 7 of the call at i >> 3), 16 / 32-byte accesses, no per-element div.
template <typename T>
__global__ void posenc_fwd_vec_kernel(const int64_t* __restrict__ tokens, const float* __restrict__ emb,
                                      const T* __restrict__ x, const float* __restrict__ pe,
                                      const float* __restrict__ alpha, T* __restrict__ y, int64_t B, int64_t T_, int64_t C,
                                      uint32_t thr, float dscale, uint64_t seed, uint64_t offset) {
  pdl_sync();
  resolve_seed(seed, offset);
  const int64_t cpr = C >> 3, n8 = B * T_ * cpr;
  const float a = *alpha;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n8; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t bt = i / cpr, c = (i - bt * cpr) * 8;
    const int64_t t = bt % T_, e0 = bt * C + c;
    float v[8], pv[8];
    if (tokens != nullptr) load8<float>(emb + tokens[bt] * C + c, v);
    else load8<T>(x + e0, v);
    load8<float>(pe + t * C + c, pv);
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = fmaf(a, pv[k], v[k]);
    if (thr != 0) dropout8_apply(v, (uint64_t)e0, thr, dscale, seed, offset);
    store8<T>(y + e0, v);
  }
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

int posenc_fwd_launch(const int64_t* tokens, const float* emb, const void* x, const float* pe, const float* alpha,
                      void* y, int dtype, int64_t B, int64_t T, int64_t C, float drop_p, uint64_t seed, uint64_t offset,
                      cudaStream_t s) {
  const int64_t n = B * T * C;
  if (n == 0) return 0;
  const uint32_t thr = drop_threshold(drop_p);
  const float ds = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  if ((C & 7) == 0 && aligned16(emb) && aligned16(x) && aligned16(pe) && aligned16(y)) {
    if (dtype == ST5_F32)
      launch_pdl(posenc_fwd_vec_kernel<float>, dim3(grid_for(n / 8, 256)), dim3(256), 0, s, tokens, emb, (const float*)x, pe,
                 alpha, (float*)y, B, T, C, thr, ds, seed, offset);
    else
      launch_pdl(posenc_fwd_vec_kernel<__nv_bfloat16>, dim3(grid_for(n / 8, 256)), dim3(256), 0, s, tokens, emb,
                 (const __nv_bfloat16*)x, pe, alpha, (__nv_bfloat16*)y, B, T, C, thr, ds, seed, offset);
    return (int)cudaGetLastError();
  }
  if (dtype == ST5_F32)
    posenc_fwd_kernel<float><<<grid_for(n, 256), 256, 0, s>>>(tokens, emb, (const float*)x, pe, alpha, (float*)y, B, T,
                                                              C, thr, ds, seed, offset);
  else
    posenc_fwd_kernel<__nv_bfloat16><<<grid_for(n, 256), 256, 0, s>>>(
        tokens, emb, (const __nv_bfloat16*)x, pe, alpha, (__nv_bfloat16*)y, B, T, C, thr, ds, seed, offset);
  return (int)cudaGetLastError();
}

template <typename T>
__global__ void posenc_bwd_kernel(const T* __restrict__ dy, const int64_t* __restrict__ tokens, int64_t padding_idx,
                                  const float* __restrict__ pe, T* __restrict__ dx, float* __restrict__ demb,
                                  float* __restrict__ dalpha, int64_t B, int64_t T_, int64_t C, uint32_t thr,
                                  float dscale, uint64_t seed, uint64_t offset) {
  resolve_seed(seed, offset);
  const int64_t n = B * T_ * C;
  float acc = 0.f;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t bt = i / C, c = i - bt * C;
    const int64_t t = bt % T_;
    float g = ldf(dy + i);
    if (thr != 0) g = dropout_keep(seed, offset, (uint64_t)i, thr) ? g * dscale : 0.f;
    acc += g * pe[t * C + c];
    if (dx != nullptr) stf(dx + i, g);
    if (tokens != nullptr) {
      const int64_t tok = tokens[bt];
      if (tok != padding_idx) atomicAdd(demb + tok * C + c, g);
    }
  }
  __shared__ float red[32];
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    v = warp_sum(v);
    if (threadIdx.x == 0) atomicAdd(dalpha, v);
  }
}
template <typename T>
__global__ void posenc_bwd_vec_kernel(const T* __restrict__ dy, const int64_t* __restrict__ tokens, int64_t padding_idx,
                                      const float* __restrict__ pe, T* __restrict__ dx, float* __restrict__ demb,
                                      float* __restrict__ dalpha, int64_t B, int64_t T_, int64_t C, uint32_t thr,
                                      float dscale, uint64_t seed, uint64_t offset) {
  pdl_sync();
  resolve_seed(seed, offset);
  const int64_t cpr = C >> 3, n8 = B * T_ * cpr;
  float acc = 0.f;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n8; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t bt = i / cpr, c = (i - bt * cpr) * 8;
    const int64_t t = bt % T_, e0 = bt * C + c;
    float g[8], pv[8];
    load8<T>(dy + e0, g);
    if (thr != 0) dropout8_apply(g, (uint64_t)e0, thr, dscale, seed, offset);
    load8<float>(pe + t * C + c, pv);
#pragma unroll
    for (int k = 0; k < 8; ++k) acc = fmaf(g[k], pv[k], acc);
    if (dx != nullptr) store8<T>(dx + e0, g);
    if (tokens != nullptr) {
      const int64_t tok = tokens[bt];
      if (tok != padding_idx) {
        float* d = demb + tok * C + c;
        if ((reinterpret_cast<uintptr_t>(d) & 15) == 0) {
          asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(d), "f"(g[0]), "f"(g[1]), "f"(g[2]), "f"(g[3]) : "memory");
          asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(d + 4), "f"(g[4]), "f"(g[5]), "f"(g[6]), "f"(g[7]) : "memory");
        } else {
#pragma unroll
          for (int k = 0; k < 8; ++k) atomicAdd(d + k, g[k]);
        }
      }
    }
  }
  __shared__ float red[32];
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    v = warp_sum(v);
    if (threadIdx.x == 0) atomicAdd(dalpha, v);
  }
}

int posenc_bwd_launch(const void* dy, const int64_t* tokens, int64_t padding_idx, const float* pe, void* dx,
                      float* demb, float* dalpha, int dtype, int64_t B, int64_t T, int64_t C, float drop_p,
                      uint64_t seed, uint64_t offset, cudaStream_t s) {
  const int64_t n = B * T * C;
  if (n == 0) return 0;
  const uint32_t thr = drop_threshold(drop_p);
  const float ds = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  if ((C & 7) == 0 && aligned16(dy) && aligned16(pe) && aligned16(dx)) {
    if (dtype == ST5_F32)
      launch_pdl(posenc_bwd_vec_kernel<float>, dim3(grid_for(n / 8, 256)), dim3(256), 0, s, (const float*)dy, tokens,
                 padding_idx, pe, (float*)dx, demb, dalpha, B, T, C, thr, ds, seed, offset);
    else
      launch_pdl(posenc_bwd_vec_kernel<__nv_bfloat16>, dim3(grid_for(n / 8, 256)), dim3(256), 0, s, (const __nv_bfloat16*)dy,
                 tokens, padding_idx, pe, (__nv_bfloat16*)dx, demb, dalpha, B, T, C, thr, ds, seed, offset);
    return (int)cudaGetLastError();
  }
  if (dtype == ST5_F32)
    posenc_bwd_kernel<float><<<grid_for(n, 256), 256, 0, s>>>((const float*)dy, tokens, padding_idx, pe, (float*)dx,
                                                              demb, dalpha, B, T, C, thr, ds, seed, offset);
  else
    posenc_bwd_kernel<__nv_bfloat16><<<grid_for(n, 256), 256, 0, s>>>((const __nv_bfloat16*)dy, tokens, padding_idx, pe,
                                                                      (__nv_bfloat16*)dx, demb, dalpha, B, T, C, thr,
                                                                      ds, seed, offset);
  return (int)cudaGetLastError();
}

// ------------------------------------------------------------------ leaky-ReLU into a padded / de-interleaved operand
// HiFi-GAN (SpeechUT/.../hifigan.py:70-100,154-170): every convolution is preceded by a leaky-ReLU and consumed here as a
// window GEMM over a zero-padded copy of its input; dilated convolutions read one PHASE (frames ph, ph+d, ...) of it.
// out[b][m][:] = lrelu(x[b][ph + d*m - pad][:]) for frames inside [0, L_b), zeros outside: one pass instead of the
// activation, the zero fill and the strided copy (three launches, two extra round trips of the activations).
// L_b = clamp(lengths[b] * len_mult, 0, T) (lengths == nullptr: T), so one padded batch of ragged utterances stages
// each utterance exactly as it would be staged alone; frames at or past L_b are never read. LEN = false (no lengths)
// compiles the length test out: st5_lrelu_pad's hot path stays the kernel it was.
template <bool LEN>
__global__ void lrelu_pad_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ out, int64_t B,
                                 int64_t T, int64_t C, int64_t n_in, int d, int ph, int pad, float slope,
                                 const int32_t* __restrict__ lengths, int len_mult) {
  pdl_sync();
  const int64_t cpr = C >> 3, n8 = B * n_in * cpr;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n8; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = i / cpr, c = (i - row * cpr) * 8;
    const int64_t b = row / n_in, m = row - b * n_in;
    const int64_t xi = (int64_t)ph + (int64_t)d * m - pad;
    int64_t L = T;
    if (LEN) {
      const int64_t l = (int64_t)__ldg(lengths + b) * len_mult;
      L = l < 0 ? 0 : (l < T ? l : T);
    }
    uint4 o = make_uint4(0u, 0u, 0u, 0u);
    if (xi >= 0 && xi < L) {
      float v[8];
      load8<__nv_bfloat16>(x + (b * T + xi) * C + c, v);
#pragma unroll
      for (int k = 0; k < 8; ++k) v[k] = v[k] > 0.f ? v[k] : v[k] * slope;
      __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&o);
#pragma unroll
      for (int k = 0; k < 4; ++k) h[k] = __floats2bfloat162_rn(v[2 * k], v[2 * k + 1]);
    }
    *reinterpret_cast<uint4*>(out + row * C + c) = o;
  }
}
int lrelu_pad_launch(const void* x, void* out, int64_t B, int64_t T, int64_t C, int64_t n_in, int d, int ph, int pad,
                     float slope, const int32_t* lengths, int len_mult, cudaStream_t s) {
  if (x == nullptr || out == nullptr) return -3;
  if (B <= 0 || T <= 0 || C <= 0 || (C & 7) || n_in <= 0 || d <= 0 || ph < 0 || ph >= d || len_mult < 1 ||
      !aligned16(x) || !aligned16(out))
    return -2;
  launch_pdl(lengths != nullptr ? lrelu_pad_kernel<true> : lrelu_pad_kernel<false>,
             dim3(grid_for(B * n_in * (C >> 3), 256)), dim3(256), 0, s, (const __nv_bfloat16*)x, (__nv_bfloat16*)out, B,
             T, C, n_in, d, ph, pad, slope, lengths, len_mult);
  return (int)cudaGetLastError();
}

// ------------------------------------------------------------------ dropout
template <typename T>
__global__ void dropout_kernel(const T* __restrict__ x, T* __restrict__ y, int64_t n, uint32_t thr, float dscale,
                               uint64_t seed, uint64_t offset) {
  resolve_seed(seed, offset);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float v = ldf(x + i);
    if (thr != 0) v = dropout_keep(seed, offset, (uint64_t)i, thr) ? v * dscale : 0.f;
    stf(y + i, v);
  }
}
int dropout_launch(const void* x, void* y, int dtype, int64_t n, float drop_p, uint64_t seed, uint64_t offset,
                   cudaStream_t s) {
  if (n == 0) return 0;
  const uint32_t thr = drop_threshold(drop_p);
  const float ds = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  if (dtype == ST5_F32)
    dropout_kernel<float><<<grid_for(n, 256), 256, 0, s>>>((const float*)x, (float*)y, n, thr, ds, seed, offset);
  else
    dropout_kernel<__nv_bfloat16><<<grid_for(n, 256), 256, 0, s>>>((const __nv_bfloat16*)x, (__nv_bfloat16*)y, n, thr,
                                                                   ds, seed, offset);
  return (int)cudaGetLastError();
}

// ------------------------------------------------------------------ activation backward (with dropout backward)
template <typename T>
__global__ void act_bwd_kernel(const T* __restrict__ dy, const T* __restrict__ pre, T* __restrict__ dpre, int act,
                               int64_t n, uint32_t thr, float dscale, uint64_t seed, uint64_t offset) {
  resolve_seed(seed, offset);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float g = ldf(dy + i);
    if (thr != 0) g = dropout_keep(seed, offset, (uint64_t)i, thr) ? g * dscale : 0.f;
    stf(dpre + i, g * act_grad(ldf(pre + i), act));
  }
}
int act_bwd_launch(const void* dy, const void* pre, void* dpre, int dtype, int act, int64_t n, float drop_p,
                   uint64_t seed, uint64_t offset, cudaStream_t s) {
  if (n == 0) return 0;
  const uint32_t thr = drop_threshold(drop_p);
  const float ds = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  if (dtype == ST5_F32)
    act_bwd_kernel<float><<<grid_for(n, 256), 256, 0, s>>>((const float*)dy, (const float*)pre, (float*)dpre, act, n,
                                                           thr, ds, seed, offset);
  else
    act_bwd_kernel<__nv_bfloat16><<<grid_for(n, 256), 256, 0, s>>>(
        (const __nv_bfloat16*)dy, (const __nv_bfloat16*)pre, (__nv_bfloat16*)dpre, act, n, thr, ds, seed, offset);
  return (int)cudaGetLastError();
}

// ------------------------------------------------------------------ activation forward (stand-alone)
// y = act(x): the GELU that follows the per-frame LayerNorm of the "layer_norm" waveform extractor
// (speech_encoder_prenet.py:308-318: conv -> dropout(0) -> LayerNorm -> GELU). 8 (bf16) / 4 (fp32) elements per thread.
__device__ __forceinline__ float act_value(float z, int act) {
  if (act == 4) return gelu_tanh_fwd(z);
  if (act == 2) return gelu_fwd(z);
  if (act == 1) return fmaxf(z, 0.f);
  if (act == 3) return tanhf(z);
  return z;
}
template <typename T, int V>
__global__ void act_fwd_kernel(const T* __restrict__ x, T* __restrict__ y, int act, int64_t n) {
  const int64_t nv = n / V;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nv; i += (int64_t)gridDim.x * blockDim.x) {
    const uint4 in = reinterpret_cast<const uint4*>(x)[i];
    const T* e = reinterpret_cast<const T*>(&in);
    uint4 out;
    T* o = reinterpret_cast<T*>(&out);
#pragma unroll
    for (int k = 0; k < V; ++k) stf<T>(o + k, act_value(ldf<T>(e + k), act));
    reinterpret_cast<uint4*>(y)[i] = out;
  }
  if (blockIdx.x == 0)
    for (int64_t i = nv * V + threadIdx.x; i < n; i += blockDim.x) stf<T>(y + i, act_value(ldf<T>(x + i), act));
}
int act_fwd_launch(const void* x, void* y, int dtype, int act, int64_t n, cudaStream_t s) {
  if (n == 0) return 0;
  if (!aligned16(x) || !aligned16(y)) return -2;
  if (dtype == ST5_F32)
    act_fwd_kernel<float, 4><<<grid_for(n / 4 + 1, 256), 256, 0, s>>>((const float*)x, (float*)y, act, n);
  else
    act_fwd_kernel<__nv_bfloat16, 8><<<grid_for(n / 8 + 1, 256), 256, 0, s>>>((const __nv_bfloat16*)x,
                                                                             (__nv_bfloat16*)y, act, n);
  return (int)cudaGetLastError();
}

// ------------------------------------------------------------------ grouped column sums (bias gradients)
// grid: (col tiles of 32, groups, row splits). block (32, 8). Partial sums are combined with fp32 atomics.
template <typename T>
__global__ void colsum_kernel(const T* __restrict__ x, int64_t ld, float* __restrict__ out, int64_t rows, int64_t cols,
                              int64_t group_rows, int64_t rows_per_split) {
  const int64_t col = (int64_t)blockIdx.x * 32 + threadIdx.x;
  const int64_t g = blockIdx.y;
  const int64_t r0 = g * group_rows + (int64_t)blockIdx.z * rows_per_split;
  int64_t r1 = r0 + rows_per_split;
  const int64_t gend = (g + 1) * group_rows < rows ? (g + 1) * group_rows : rows;
  if (r1 > gend) r1 = gend;
  float acc = 0.f;
  if (col < cols)
    for (int64_t r = r0 + threadIdx.y; r < r1; r += 8) acc += ldf(x + r * ld + col);
  __shared__ float red[8][33];
  red[threadIdx.y][threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.y == 0 && col < cols) {
    float v = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) v += red[k][threadIdx.x];
    atomicAdd(out + g * cols + col, v);
  }
}
// Vector variant: a lane owns VEC consecutive columns (one 16-byte load per row), so a warp reads 512 contiguous bytes
// of every row it visits. Used whenever the layout is 16-byte addressable; also the reduction of split-K partials.
template <typename T, int VEC>
__global__ void colsum_vec_kernel(const T* __restrict__ x, int64_t ld, float* __restrict__ out, int64_t rows,
                                  int64_t cols, int64_t group_rows, int64_t rows_per_split, int mode) {
  pdl_sync();
  const int64_t col = ((int64_t)blockIdx.x * 32 + threadIdx.x) * VEC;
  const int64_t g = blockIdx.y;
  const int64_t r0 = g * group_rows + (int64_t)blockIdx.z * rows_per_split;
  int64_t r1 = r0 + rows_per_split;
  const int64_t gend = (g + 1) * group_rows < rows ? (g + 1) * group_rows : rows;
  if (r1 > gend) r1 = gend;
  float acc[VEC];
#pragma unroll
  for (int k = 0; k < VEC; ++k) acc[k] = 0.f;
  if (col < cols) {
#pragma unroll 4
    for (int64_t r = r0 + threadIdx.y; r < r1; r += 8) {
      const uint4 u = __ldg(reinterpret_cast<const uint4*>(x + r * ld + col));
      if constexpr (VEC == 4) {
        acc[0] += __uint_as_float(u.x); acc[1] += __uint_as_float(u.y);
        acc[2] += __uint_as_float(u.z); acc[3] += __uint_as_float(u.w);
      } else {
        const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 f = __bfloat1622float2(h[k]);
          acc[2 * k] += f.x;
          acc[2 * k + 1] += f.y;
        }
      }
    }
  }
  __shared__ float red[8][32 * VEC + 1];
#pragma unroll
  for (int k = 0; k < VEC; ++k) red[threadIdx.y][threadIdx.x * VEC + k] = acc[k];
  __syncthreads();
  for (int c = threadIdx.y * 32 + threadIdx.x; c < 32 * VEC; c += 256) {
    const int64_t oc = (int64_t)blockIdx.x * 32 * VEC + c;
    if (oc < cols) {
      float v = 0.f;
#pragma unroll
      for (int k = 0; k < 8; ++k) v += red[k][c];
      // mode 0: several row splits share an output (fp32 atomics, output pre-zeroed or accumulated into);
      // mode 1 / 2: this block owns its outputs (store / add) -- no memset, no atomics
      if (mode == 0) atomicAdd(out + g * cols + oc, v);
      else if (mode == 1) out[g * cols + oc] = v;
      else out[g * cols + oc] += v;
    }
  }
}
int colsum_launch(const void* x, int64_t ld, float* out, int dtype, int64_t rows, int64_t cols, int64_t group_rows,
                  int accumulate, cudaStream_t s) {
  if (rows == 0 || cols == 0) return 0;
  if (group_rows <= 0) group_rows = rows;
  const int64_t groups = (rows + group_rows - 1) / group_rows;
  const int vec = dtype == ST5_F32 ? 4 : 8;
  const bool vec_ok = (cols % vec == 0) && (ld % vec == 0) && ((reinterpret_cast<uintptr_t>(x) & 15) == 0);
  const int64_t cw = vec_ok ? 32 * vec : 32;  // columns per block
  const int64_t col_blocks = (cols + cw - 1) / cw;
  // enough row splits to fill the machine a few times over, each split at least 64 rows deep
  int64_t splits = (4 * 132 + col_blocks * groups - 1) / (col_blocks * groups);
  const int64_t max_splits = (group_rows + 63) / 64;
  if (splits > max_splits) splits = max_splits;
  if (splits < 1) splits = 1;
  const int64_t rps = (group_rows + splits - 1) / splits;
  dim3 grid((unsigned)col_blocks, (unsigned)groups, (unsigned)splits), block(32, 8);
  const int mode = (vec_ok && splits == 1) ? (accumulate ? 2 : 1) : 0;
  if (mode == 0 && !accumulate) {
    cudaError_t e = cudaMemsetAsync(out, 0, sizeof(float) * groups * cols, s);
    if (e != cudaSuccess) return (int)e;
  }
  if (vec_ok && dtype == ST5_F32)
    launch_pdl(colsum_vec_kernel<float, 4>, dim3(grid), dim3(block), 0, s, (const float*)x, ld, out, rows, cols, group_rows, rps, mode);
  else if (vec_ok)
    launch_pdl(colsum_vec_kernel<__nv_bfloat16, 8>, dim3(grid), dim3(block), 0, s, (const __nv_bfloat16*)x, ld, out, rows, cols, group_rows, rps, mode);
  else if (dtype == ST5_F32)
    colsum_kernel<float><<<grid, block, 0, s>>>((const float*)x, ld, out, rows, cols, group_rows, rps);
  else
    colsum_kernel<__nv_bfloat16><<<grid, block, 0, s>>>((const __nv_bfloat16*)x, ld, out, rows, cols, group_rows, rps);
  return (int)cudaGetLastError();
}

}  // namespace st5
