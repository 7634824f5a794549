// BatchNorm1d (fused tanh + dropout) forward/backward (LayerNorm lives in layernorm.cu).
// Reference semantics: fairseq LayerNorm == torch.nn.LayerNorm (fairseq/modules/layer_norm.py:30-35), post-LN residual
// blocks of transformer_layer.py:112-132 / :343-391; espnet Tacotron2 Postnet BatchNorm1d blocks
// (speech_decoder_postnet.py:39-51) with training statistics over every row, padded frames included.
#include <initializer_list>
#include "kernels.cuh"
#include "ptx.cuh"
#include "gemm.cuh"
#include "vec8.cuh"

namespace st5 {

// =============================================================================================== BatchNorm1d
// channels-last rows [rows][C]; block (32 channels, 8 row lanes); per-channel partial sums via fp32 atomics.
template <typename T, int MODE>  // MODE 0: sum(x) ; 1: sum((x-mean)^2) with mean = aux[c]
__global__ void bn_stat_kernel(const T* __restrict__ x, int64_t ld, const float* __restrict__ aux,
                               float* __restrict__ out, int64_t rows, int C, int64_t rows_per_block) {
  const int c = blockIdx.x * 32 + threadIdx.x;
  const int64_t r0 = (int64_t)blockIdx.y * rows_per_block;
  const int64_t r1 = r0 + rows_per_block < rows ? r0 + rows_per_block : rows;
  float acc = 0.f;
  if (c < C) {
    const float mu = MODE == 1 ? aux[c] : 0.f;
    for (int64_t r = r0 + threadIdx.y; r < r1; r += 8) {
      const float v = ldf(x + r * ld + c) - mu;
      acc += MODE == 1 ? v * v : v;
    }
  }
  __shared__ float red[8][33];
  red[threadIdx.y][threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    float v = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) v += red[k][threadIdx.x];
    atomicAdd(out + c, v);
  }
}
__global__ void bn_finalize_stats(float* __restrict__ scratch, float* __restrict__ running_mean,
                                  float* __restrict__ running_var, float* __restrict__ save_mean,
                                  float* __restrict__ save_rstd, int64_t rows, int C, float momentum, float eps,
                                  int stage) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  if (stage == 0) {
    scratch[c] = scratch[c] / (float)rows;  // mean
  } else {
    const float mu = scratch[c];
    const float var = scratch[C + c] / (float)rows;
    save_mean[c] = mu;
    save_rstd[c] = rsqrtf(var + eps);
    if (running_mean != nullptr) {
      const float unbiased = rows > 1 ? scratch[C + c] / (float)(rows - 1) : var;
      running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * mu;
      running_var[c] = (1.f - momentum) * running_var[c] + momentum * unbiased;
    }
  }
}
__global__ void bn_eval_stats(const float* __restrict__ running_mean, const float* __restrict__ running_var,
                              float* __restrict__ save_mean, float* __restrict__ save_rstd, int C, float eps) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  save_mean[c] = running_mean[c];
  save_rstd[c] = rsqrtf(running_var[c] + eps);
}
template <typename T>
__global__ void bn_apply_kernel(const T* __restrict__ x, int64_t x_ld, const float* __restrict__ gamma,
                                const float* __restrict__ beta, const float* __restrict__ mean,
                                const float* __restrict__ rstd, T* __restrict__ y, int64_t y_ld, T* __restrict__ y_pre,
                                int64_t rows, int C, int act, uint32_t thr, float dscale, uint64_t seed,
                                uint64_t offset) {
  resolve_seed(seed, offset);
  const int64_t n = rows * C;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / C;
    const int c = (int)(i - r * C);
    float v = (ldf(x + r * x_ld + c) - mean[c]) * rstd[c] * gamma[c] + beta[c];
    if (y_pre != nullptr) { stf(y_pre + i, v); v = ldf(y_pre + i); }
    if (act == ACT_TANH) v = tanhf(v);
    else if (act == ACT_RELU) v = fmaxf(v, 0.f);
    if (thr != 0) v = dropout_keep(seed, offset, (uint64_t)i, thr) ? v * dscale : 0.f;
    stf(y + r * y_ld + c, v);
  }
}

// ---- vector variants (C, every row pitch a multiple of 8, 16-byte aligned bases): a thread owns 8 consecutive channels
// of a row -- one 16-byte access per tensor, ONE Philox call per 8 outputs (the scalar kernels pay one per element),
// MUFU tanh in bf16 mode.
template <typename T> __device__ __forceinline__ float bn_tanh(float v) {
  if constexpr (sizeof(T) == 2) return fast_tanh(v);
  else return tanhf(v);
}
template <typename T>
__global__ void bn_apply_vec_kernel(const T* __restrict__ x, int64_t x_ld, const float* __restrict__ gamma,
                                    const float* __restrict__ beta, const float* __restrict__ mean,
                                    const float* __restrict__ rstd, T* __restrict__ y, int64_t y_ld,
                                    T* __restrict__ y_pre, int64_t rows, int C, int act, uint32_t thr, float dscale,
                                    uint64_t seed, uint64_t offset) {
  if (thr != 0) resolve_seed(seed, offset);
  const int c8n = C >> 3;
  const int64_t ng = rows * c8n;
  for (int64_t gi = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; gi < ng; gi += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = gi / c8n;
    const int c = (int)(gi - r * c8n) * 8;
    float v[8], mu[8], rs[8], ga[8], be[8];
    load8<T>(x + r * x_ld + c, v);
    load8<float>(mean + c, mu); load8<float>(rstd + c, rs); load8<float>(gamma + c, ga); load8<float>(beta + c, be);
#pragma unroll
    for (int t = 0; t < 8; ++t) v[t] = round_to<T>((v[t] - mu[t]) * rs[t] * ga[t] + be[t]);
    if (y_pre != nullptr) store8<T>(y_pre + r * C + c, v);
    if (act == ACT_TANH) {
#pragma unroll
      for (int t = 0; t < 8; ++t) v[t] = bn_tanh<T>(v[t]);
    } else if (act == ACT_RELU) {
#pragma unroll
      for (int t = 0; t < 8; ++t) v[t] = fmaxf(v[t], 0.f);
    }
    if (thr != 0) dropout8(v, (uint64_t)(r * C + c), thr, dscale, seed, offset);
    store8<T>(y + r * y_ld + c, v);
  }
}
// g = dropout_bwd(dy) * act'(y_pre) for 8 channels of row r
template <typename T>
__device__ __forceinline__ void bn_g8(const T* dy, int64_t dy_ld, const T* y_pre, int64_t r, int c, int C, int act,
                                      uint32_t thr, float dscale, uint64_t seed, uint64_t offset, float* g) {
  load8<T>(dy + r * dy_ld + c, g);
  if (thr != 0) dropout8(g, (uint64_t)(r * C + c), thr, dscale, seed, offset);
  if (act == ACT_TANH) {
    float yp[8];
    load8<T>(y_pre + r * C + c, yp);
#pragma unroll
    for (int t = 0; t < 8; ++t) {
      const float th = bn_tanh<T>(yp[t]);
      g[t] *= fmaf(-th, th, 1.f);
    }
  } else if (act == ACT_RELU) {
    float yp[8];
    load8<T>(y_pre + r * C + c, yp);
#pragma unroll
    for (int t = 0; t < 8; ++t) g[t] = yp[t] > 0.f ? g[t] : 0.f;
  }
}
// grid (ceil(C / 256), row blocks), block (32, 8): lane = 8 channels, threadIdx.y strides the rows
template <typename T>
__global__ void bn_bwd_stat_vec_kernel(const T* __restrict__ dy, int64_t dy_ld, const T* __restrict__ x, int64_t x_ld,
                                       const T* __restrict__ y_pre, const float* __restrict__ mean,
                                       const float* __restrict__ rstd, float* __restrict__ scratch, int64_t rows,
                                       int C, int64_t rows_per_block, int act, uint32_t thr, float dscale,
                                       uint64_t seed, uint64_t offset) {
  if (thr != 0) resolve_seed(seed, offset);
  const int c = (blockIdx.x * 32 + threadIdx.x) * 8;
  const int64_t r0 = (int64_t)blockIdx.y * rows_per_block;
  const int64_t r1 = r0 + rows_per_block < rows ? r0 + rows_per_block : rows;
  float a[8], bsum[8];
#pragma unroll
  for (int t = 0; t < 8; ++t) a[t] = bsum[t] = 0.f;
  if (c < C) {
    float mu[8], rs[8];
    load8<float>(mean + c, mu); load8<float>(rstd + c, rs);
    for (int64_t r = r0 + threadIdx.y; r < r1; r += 8) {
      float g[8], xv[8];
      bn_g8<T>(dy, dy_ld, y_pre, r, c, C, act, thr, dscale, seed, offset, g);
      load8<T>(x + r * x_ld + c, xv);
#pragma unroll
      for (int t = 0; t < 8; ++t) {
        a[t] += g[t];
        bsum[t] += g[t] * (xv[t] - mu[t]) * rs[t];
      }
    }
  }
  __shared__ float red[2][8][257];
#pragma unroll
  for (int t = 0; t < 8; ++t) {
    red[0][threadIdx.y][threadIdx.x * 8 + t] = a[t];
    red[1][threadIdx.y][threadIdx.x * 8 + t] = bsum[t];
  }
  __syncthreads();
  const int cc = threadIdx.y * 32 + threadIdx.x;  // 256 threads <-> 256 channels of this block
  const int cg = blockIdx.x * 256 + cc;
  if (cg < C) {
    float va = 0.f, vb = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) { va += red[0][k][cc]; vb += red[1][k][cc]; }
    atomicAdd(scratch + cg, va);
    atomicAdd(scratch + C + cg, vb);
  }
}
template <typename T>
__global__ void bn_bwd_apply_vec_kernel(const T* __restrict__ dy, int64_t dy_ld, const T* __restrict__ x, int64_t x_ld,
                                        const T* __restrict__ y_pre, const float* __restrict__ gamma,
                                        const float* __restrict__ mean, const float* __restrict__ rstd,
                                        const float* __restrict__ scratch, T* __restrict__ dx, int64_t dx_ld,
                                        float* __restrict__ dgamma, float* __restrict__ dbeta, int64_t rows, int C,
                                        int act, uint32_t thr, float dscale, uint64_t seed, uint64_t offset) {
  if (thr != 0) resolve_seed(seed, offset);
  const int c8n = C >> 3;
  const int64_t ng = rows * c8n;
  const float inv_n = 1.f / (float)rows;
  for (int64_t gi = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; gi < ng; gi += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = gi / c8n;
    const int c = (int)(gi - r * c8n) * 8;
    float g[8], xv[8], mu[8], rs[8], ga[8], s0[8], s1[8];
    bn_g8<T>(dy, dy_ld, y_pre, r, c, C, act, thr, dscale, seed, offset, g);
    load8<T>(x + r * x_ld + c, xv);
    load8<float>(mean + c, mu); load8<float>(rstd + c, rs); load8<float>(gamma + c, ga);
    load8<float>(scratch + c, s0); load8<float>(scratch + C + c, s1);
#pragma unroll
    for (int t = 0; t < 8; ++t) {
      const float xh = (xv[t] - mu[t]) * rs[t];
      g[t] = ga[t] * rs[t] * (g[t] - s0[t] * inv_n - xh * s1[t] * inv_n);
    }
    store8<T>(dx + r * dx_ld + c, g);
  }
  if (blockIdx.x == 0)
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
      if (dbeta != nullptr) dbeta[c] += scratch[c];
      if (dgamma != nullptr) dgamma[c] += scratch[C + c];
    }
}
static inline bool bn_vec_ok(int64_t C, std::initializer_list<int64_t> lds, std::initializer_list<const void*> ptrs) {
  if (C & 7) return false;
  for (int64_t l : lds) if (l & 7) return false;
  for (const void* q : ptrs) if (q != nullptr && (reinterpret_cast<uintptr_t>(q) & 15)) return false;
  return true;
}

static inline int bn_row_blocks(int64_t rows, int64_t* rpb) {
  int64_t nb = (rows + 255) / 256;
  if (nb > 128) nb = 128;
  if (nb < 1) nb = 1;
  *rpb = (rows + nb - 1) / nb;
  return (int)nb;
}

int bn_fwd_launch(const void* x, int64_t x_ld, const float* gamma, const float* beta, float* running_mean,
                  float* running_var, float* save_mean, float* save_rstd, void* y, int64_t y_ld, void* y_pre, int dtype,
                  int64_t rows, int64_t C, int training, float momentum, float eps, int act, float drop_p,
                  uint64_t seed, uint64_t offset, float* scratch, cudaStream_t s) {
  if (rows == 0 || C == 0) return 0;
  const unsigned cblk = (unsigned)((C + 127) / 128);
  if (training) {
    cudaError_t e = cudaMemsetAsync(scratch, 0, sizeof(float) * 2 * C, s);
    if (e != cudaSuccess) return (int)e;
    int64_t rpb;
    const int nb = bn_row_blocks(rows, &rpb);
    dim3 grid((unsigned)((C + 31) / 32), (unsigned)nb), block(32, 8);
    if (dtype == ST5_F32) bn_stat_kernel<float, 0><<<grid, block, 0, s>>>((const float*)x, x_ld, nullptr, scratch, rows, (int)C, rpb);
    else bn_stat_kernel<__nv_bfloat16, 0><<<grid, block, 0, s>>>((const __nv_bfloat16*)x, x_ld, nullptr, scratch, rows, (int)C, rpb);
    bn_finalize_stats<<<cblk, 128, 0, s>>>(scratch, nullptr, nullptr, nullptr, nullptr, rows, (int)C, momentum, eps, 0);
    if (dtype == ST5_F32) bn_stat_kernel<float, 1><<<grid, block, 0, s>>>((const float*)x, x_ld, scratch, scratch + C, rows, (int)C, rpb);
    else bn_stat_kernel<__nv_bfloat16, 1><<<grid, block, 0, s>>>((const __nv_bfloat16*)x, x_ld, scratch, scratch + C, rows, (int)C, rpb);
    bn_finalize_stats<<<cblk, 128, 0, s>>>(scratch, running_mean, running_var, save_mean, save_rstd, rows, (int)C, momentum, eps, 1);
  } else {
    bn_eval_stats<<<cblk, 128, 0, s>>>(running_mean, running_var, save_mean, save_rstd, (int)C, eps);
  }
  const uint32_t thr = drop_threshold(drop_p);
  const float ds = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  const int64_t n = rows * C;
  int64_t g = (n + 255) / 256;
  if (g > 132 * 16) g = 132 * 16;
  if (bn_vec_ok(C, {x_ld, y_ld}, {x, y, y_pre, gamma, beta, save_mean, save_rstd})) {
    int64_t gv = (n / 8 + 255) / 256;
    if (gv > 132 * 16) gv = 132 * 16;
    if (dtype == ST5_F32)
      bn_apply_vec_kernel<float><<<(unsigned)gv, 256, 0, s>>>((const float*)x, x_ld, gamma, beta, save_mean, save_rstd,
                                                              (float*)y, y_ld, (float*)y_pre, rows, (int)C, act, thr,
                                                              ds, seed, offset);
    else
      bn_apply_vec_kernel<__nv_bfloat16><<<(unsigned)gv, 256, 0, s>>>(
          (const __nv_bfloat16*)x, x_ld, gamma, beta, save_mean, save_rstd, (__nv_bfloat16*)y, y_ld,
          (__nv_bfloat16*)y_pre, rows, (int)C, act, thr, ds, seed, offset);
    return (int)cudaGetLastError();
  }
  if (dtype == ST5_F32)
    bn_apply_kernel<float><<<(unsigned)g, 256, 0, s>>>((const float*)x, x_ld, gamma, beta, save_mean, save_rstd,
                                                       (float*)y, y_ld, (float*)y_pre, rows, (int)C, act, thr, ds, seed,
                                                       offset);
  else
    bn_apply_kernel<__nv_bfloat16><<<(unsigned)g, 256, 0, s>>>((const __nv_bfloat16*)x, x_ld, gamma, beta, save_mean,
                                                               save_rstd, (__nv_bfloat16*)y, y_ld,
                                                               (__nv_bfloat16*)y_pre, rows, (int)C, act, thr, ds, seed,
                                                               offset);
  return (int)cudaGetLastError();
}

// backward: g = dropout_bwd(dy) * act'(y_pre); pass 1: sum(g), sum(g * xhat) per channel; pass 2: dx.
template <typename T>
__device__ __forceinline__ float bn_g(const T* dy, int64_t dy_ld, const T* y_pre, int64_t r, int c, int C, int act,
                                      uint32_t thr, float dscale, uint64_t seed, uint64_t offset) {
  const int64_t i = r * C + c;
  float g = ldf(dy + r * dy_ld + c);
  if (thr != 0) g = dropout_keep(seed, offset, (uint64_t)i, thr) ? g * dscale : 0.f;
  if (act == ACT_TANH) {
    const float t = tanhf(ldf(y_pre + i));
    g *= 1.f - t * t;
  } else if (act == ACT_RELU) {
    g = ldf(y_pre + i) > 0.f ? g : 0.f;
  }
  return g;
}
template <typename T>
__global__ void bn_bwd_stat_kernel(const T* __restrict__ dy, int64_t dy_ld, const T* __restrict__ x, int64_t x_ld,
                                   const T* __restrict__ y_pre, const float* __restrict__ mean,
                                   const float* __restrict__ rstd, float* __restrict__ scratch, int64_t rows, int C,
                                   int64_t rows_per_block, int act, uint32_t thr, float dscale, uint64_t seed,
                                   uint64_t offset) {
  resolve_seed(seed, offset);
  const int c = blockIdx.x * 32 + threadIdx.x;
  const int64_t r0 = (int64_t)blockIdx.y * rows_per_block;
  const int64_t r1 = r0 + rows_per_block < rows ? r0 + rows_per_block : rows;
  float a = 0.f, b = 0.f;
  if (c < C) {
    const float mu = mean[c], rs = rstd[c];
    for (int64_t r = r0 + threadIdx.y; r < r1; r += 8) {
      const float g = bn_g(dy, dy_ld, y_pre, r, c, C, act, thr, dscale, seed, offset);
      a += g;
      b += g * (ldf(x + r * x_ld + c) - mu) * rs;
    }
  }
  __shared__ float red[2][8][33];
  red[0][threadIdx.y][threadIdx.x] = a;
  red[1][threadIdx.y][threadIdx.x] = b;
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    float va = 0.f, vb = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) { va += red[0][k][threadIdx.x]; vb += red[1][k][threadIdx.x]; }
    atomicAdd(scratch + c, va);
    atomicAdd(scratch + C + c, vb);
  }
}
template <typename T>
__global__ void bn_bwd_apply_kernel(const T* __restrict__ dy, int64_t dy_ld, const T* __restrict__ x, int64_t x_ld,
                                    const T* __restrict__ y_pre, const float* __restrict__ gamma,
                                    const float* __restrict__ mean, const float* __restrict__ rstd,
                                    const float* __restrict__ scratch, T* __restrict__ dx, int64_t dx_ld,
                                    float* __restrict__ dgamma, float* __restrict__ dbeta, int64_t rows, int C, int act,
                                    uint32_t thr, float dscale, uint64_t seed, uint64_t offset) {
  resolve_seed(seed, offset);
  const int64_t n = rows * C;
  const float inv_n = 1.f / (float)rows;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / C;
    const int c = (int)(i - r * C);
    const float g = bn_g(dy, dy_ld, y_pre, r, c, C, act, thr, dscale, seed, offset);
    const float xh = (ldf(x + r * x_ld + c) - mean[c]) * rstd[c];
    stf(dx + r * dx_ld + c, gamma[c] * rstd[c] * (g - scratch[c] * inv_n - xh * scratch[C + c] * inv_n));
  }
  if (blockIdx.x == 0)
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
      if (dbeta != nullptr) dbeta[c] += scratch[c];
      if (dgamma != nullptr) dgamma[c] += scratch[C + c];
    }
}

int bn_bwd_launch(const void* dy, int64_t dy_ld, const void* x, int64_t x_ld, const void* y_pre, const float* gamma,
                  const float* save_mean, const float* save_rstd, void* dx, int64_t dx_ld, float* dgamma, float* dbeta,
                  int dtype, int64_t rows, int64_t C, int act, float drop_p, uint64_t seed, uint64_t offset,
                  float* scratch, cudaStream_t s) {
  if (rows == 0 || C == 0) return 0;
  if (act != ACT_NONE && y_pre == nullptr) return -2;
  cudaError_t e = cudaMemsetAsync(scratch, 0, sizeof(float) * 2 * C, s);
  if (e != cudaSuccess) return (int)e;
  const uint32_t thr = drop_threshold(drop_p);
  const float ds = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  int64_t rpb;
  const int nb = bn_row_blocks(rows, &rpb);
  dim3 grid((unsigned)((C + 31) / 32), (unsigned)nb), block(32, 8);
  const int64_t n = rows * C;
  int64_t g = (n + 255) / 256;
  if (g > 132 * 16) g = 132 * 16;
  if (bn_vec_ok(C, {dy_ld, x_ld, dx_ld}, {dy, x, y_pre, dx, gamma, save_mean, save_rstd, scratch})) {
    // (each block covers 256 channels: split the rows finer than the scalar kernel to keep ~4 blocks per SM busy)
    const int64_t cblocks = (C + 255) / 256;
    int64_t vnb = (592 + cblocks - 1) / cblocks;
    if (vnb > (rows + 31) / 32) vnb = (rows + 31) / 32;
    if (vnb < 1) vnb = 1;
    rpb = (rows + vnb - 1) / vnb;
    dim3 vgrid((unsigned)cblocks, (unsigned)((rows + rpb - 1) / rpb));
    int64_t gv = (n / 8 + 255) / 256;
    if (gv > 132 * 16) gv = 132 * 16;
    if (dtype == ST5_F32) {
      bn_bwd_stat_vec_kernel<float><<<vgrid, block, 0, s>>>((const float*)dy, dy_ld, (const float*)x, x_ld,
                                                            (const float*)y_pre, save_mean, save_rstd, scratch, rows,
                                                            (int)C, rpb, act, thr, ds, seed, offset);
      bn_bwd_apply_vec_kernel<float><<<(unsigned)gv, 256, 0, s>>>(
          (const float*)dy, dy_ld, (const float*)x, x_ld, (const float*)y_pre, gamma, save_mean, save_rstd, scratch,
          (float*)dx, dx_ld, dgamma, dbeta, rows, (int)C, act, thr, ds, seed, offset);
    } else {
      bn_bwd_stat_vec_kernel<__nv_bfloat16><<<vgrid, block, 0, s>>>(
          (const __nv_bfloat16*)dy, dy_ld, (const __nv_bfloat16*)x, x_ld, (const __nv_bfloat16*)y_pre, save_mean,
          save_rstd, scratch, rows, (int)C, rpb, act, thr, ds, seed, offset);
      bn_bwd_apply_vec_kernel<__nv_bfloat16><<<(unsigned)gv, 256, 0, s>>>(
          (const __nv_bfloat16*)dy, dy_ld, (const __nv_bfloat16*)x, x_ld, (const __nv_bfloat16*)y_pre, gamma, save_mean,
          save_rstd, scratch, (__nv_bfloat16*)dx, dx_ld, dgamma, dbeta, rows, (int)C, act, thr, ds, seed, offset);
    }
    return (int)cudaGetLastError();
  }
  if (dtype == ST5_F32) {
    bn_bwd_stat_kernel<float><<<grid, block, 0, s>>>((const float*)dy, dy_ld, (const float*)x, x_ld,
                                                     (const float*)y_pre, save_mean, save_rstd, scratch, rows, (int)C,
                                                     rpb, act, thr, ds, seed, offset);
    bn_bwd_apply_kernel<float><<<(unsigned)g, 256, 0, s>>>((const float*)dy, dy_ld, (const float*)x, x_ld,
                                                           (const float*)y_pre, gamma, save_mean, save_rstd, scratch,
                                                           (float*)dx, dx_ld, dgamma, dbeta, rows, (int)C, act, thr, ds,
                                                           seed, offset);
  } else {
    bn_bwd_stat_kernel<__nv_bfloat16><<<grid, block, 0, s>>>(
        (const __nv_bfloat16*)dy, dy_ld, (const __nv_bfloat16*)x, x_ld, (const __nv_bfloat16*)y_pre, save_mean,
        save_rstd, scratch, rows, (int)C, rpb, act, thr, ds, seed, offset);
    bn_bwd_apply_kernel<__nv_bfloat16><<<(unsigned)g, 256, 0, s>>>(
        (const __nv_bfloat16*)dy, dy_ld, (const __nv_bfloat16*)x, x_ld, (const __nv_bfloat16*)y_pre, gamma, save_mean,
        save_rstd, scratch, (__nv_bfloat16*)dx, dx_ld, dgamma, dbeta, rows, (int)C, act, thr, ds, seed, offset);
  }
  return (int)cudaGetLastError();
}

}  // namespace st5
