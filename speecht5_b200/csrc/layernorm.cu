// LayerNorm with fused residual + dropout, forward and backward. HBM-bound: one warp per row, 16-byte vector accesses
// (8 bf16 / 2x4 fp32 per lane per chunk), fp32 statistics (two-pass variance on registers).
// Reference semantics: fairseq LayerNorm == torch.nn.LayerNorm (fairseq/modules/layer_norm.py:30-35); post-LN residual
// tails of transformer_layer.py:112-132 / :343-391 and encoder.py:226-227.
//   forward : s = residual + dropout(x);  y = (s - mean) * rstd * gamma + beta          (s, mean, rstd saved)
//   backward: ds = rstd * (g - mean(g) - xhat * mean(g * xhat)),  g = dy * gamma ;  dx = dropout_bwd(ds)
//             dgamma += sum_rows dy * xhat ; dbeta += sum_rows dy     (separate column-reduction kernel)
#include "kernels.cuh"
#include <stdlib.h>
#include "ptx.cuh"
#include "vec8.cuh"
#include "tma_map.cuh"  // device_sm_count()

namespace st5 {

constexpr int LN_WARPS = 4;
constexpr int LN_MAX_CHUNKS = 4;  // per lane: C <= 4 * 32 * 8 = 1024

template <typename T>
__global__ void __launch_bounds__(LN_WARPS * 32)
    ln_fwd_kernel(const T* __restrict__ x, const T* __restrict__ residual, const float* __restrict__ residual_f32,
                  const float* __restrict__ gamma, const float* __restrict__ beta, T* __restrict__ y,
                  float* __restrict__ y_f32, T* __restrict__ s_out, float* __restrict__ mean,
                  float* __restrict__ rstd, int64_t rows, int C, float eps, uint32_t thr, float dscale, uint64_t seed,
                  uint64_t offset) {
  pdl_sync();
  if (thr != 0) resolve_seed(seed, offset);
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * LN_WARPS + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int nchunks = C >> 3;
  float v[LN_MAX_CHUNKS][8];
  float sum = 0.f;
#pragma unroll
  for (int k = 0; k < LN_MAX_CHUNKS; ++k) {
    const int ch = k * 32 + lane;
    if (ch < nchunks) {
      const int64_t e0 = row * C + ch * 8;
      load8<T>(x + e0, v[k]);
      if (thr != 0) dropout8(v[k], (uint64_t)e0, thr, dscale, seed, offset);
      if (residual_f32 != nullptr) {  // fp32 residual stream: the un-rounded output of the previous LayerNorm
        float r[8];
        load8<float>(residual_f32 + e0, r);
#pragma unroll
        for (int t = 0; t < 8; ++t) v[k][t] += r[t];
      } else if (residual != nullptr) {
        float r[8];
        load8<T>(residual + e0, r);
#pragma unroll
        for (int t = 0; t < 8; ++t) v[k][t] += r[t];
      }
      // s is saved (in the activation dtype) for the backward pass only; the statistics and the output use the
      // un-rounded sum -- rounding it first would put one more bf16 rounding (1.6e-3 rms) into every LayerNorm
      if (s_out != nullptr) store8<T>(s_out + e0, v[k]);
#pragma unroll
      for (int t = 0; t < 8; ++t) sum += v[k][t];
    }
  }
  sum = warp_sum(sum);
  const float mu = sum / (float)C;
  float sq = 0.f;
#pragma unroll
  for (int k = 0; k < LN_MAX_CHUNKS; ++k) {
    if (k * 32 + lane < nchunks) {
#pragma unroll
      for (int t = 0; t < 8; ++t) {
        const float d = v[k][t] - mu;
        sq += d * d;
      }
    }
  }
  sq = warp_sum(sq);
  const float rs = rsqrtf(sq / (float)C + eps);
  if (lane == 0) {
    if (mean != nullptr) mean[row] = mu;
    if (rstd != nullptr) rstd[row] = rs;
  }
#pragma unroll
  for (int k = 0; k < LN_MAX_CHUNKS; ++k) {
    const int ch = k * 32 + lane;
    if (ch < nchunks) {
      float g[8], b[8], o[8];
      load8<float>(gamma + ch * 8, g);
      load8<float>(beta + ch * 8, b);
#pragma unroll
      for (int t = 0; t < 8; ++t) o[t] = (v[k][t] - mu) * rs * g[t] + b[t];
      store8<T>(y + row * C + ch * 8, o);
      if (y_f32 != nullptr) store8<float>(y_f32 + row * C + ch * 8, o);
    }
  }
}

int ln_fwd_launch(const void* x, const void* residual, const float* residual_f32, const float* gamma, const float* beta,
                  void* y, float* y_f32, void* s_out, float* mean, float* rstd, int dtype, int64_t rows, int64_t C,
                  float eps, float drop_p, uint64_t seed, uint64_t offset, cudaStream_t s) {
  if (rows == 0) return 0;
  if (C > 8 * 32 * LN_MAX_CHUNKS || C <= 0 || (C & 7)) return -2;
  const uint32_t thr = drop_threshold(drop_p);
  const float ds = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  const unsigned grid = (unsigned)((rows + LN_WARPS - 1) / LN_WARPS);
  if (dtype == ST5_F32)
    launch_pdl(ln_fwd_kernel<float>, dim3(grid), dim3(LN_WARPS * 32), 0, s, (const float*)x, (const float*)residual,
               residual_f32, gamma, beta, (float*)y, y_f32, (float*)s_out, mean, rstd, rows, (int)C, eps, thr, ds, seed, offset);
  else
    launch_pdl(ln_fwd_kernel<__nv_bfloat16>, dim3(grid), dim3(LN_WARPS * 32), 0, s, (const __nv_bfloat16*)x, (const __nv_bfloat16*)residual, residual_f32, gamma, beta, (__nv_bfloat16*)y, y_f32,
        (__nv_bfloat16*)s_out, mean, rstd, rows, (int)C, eps, thr, ds, seed, offset);
  return (int)cudaGetLastError();
}

// number of floats of scratch the caller provides (kept for ABI stability; the reduction now uses fp32 atomics)
int64_t ln_bwd_blocks(int64_t rows) { (void)rows; return 1; }

template <typename T>
__global__ void __launch_bounds__(LN_WARPS * 32)
    ln_bwd_dx_kernel(const T* __restrict__ dy, const T* __restrict__ s_in, const float* __restrict__ mean,
                     const float* __restrict__ rstd, const float* __restrict__ gamma, T* __restrict__ ds,
                     T* __restrict__ dx, int64_t rows, int C, uint32_t thr, float dscale, uint64_t seed,
                     uint64_t offset) {
  if (thr != 0) resolve_seed(seed, offset);
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * LN_WARPS + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int nchunks = C >> 3;
  const float mu = mean[row], rs = rstd[row];
  float g[LN_MAX_CHUNKS][8], xh[LN_MAX_CHUNKS][8];
  float c1 = 0.f, c2 = 0.f;
#pragma unroll
  for (int k = 0; k < LN_MAX_CHUNKS; ++k) {
    const int ch = k * 32 + lane;
    if (ch < nchunks) {
      const int64_t e0 = row * C + ch * 8;
      float d[8], sv[8], gm[8];
      load8<T>(dy + e0, d);
      load8<T>(s_in + e0, sv);
      load8<float>(gamma + ch * 8, gm);
#pragma unroll
      for (int t = 0; t < 8; ++t) {
        xh[k][t] = (sv[t] - mu) * rs;
        g[k][t] = d[t] * gm[t];
        c1 += g[k][t];
        c2 += g[k][t] * xh[k][t];
      }
    }
  }
  c1 = warp_sum(c1) / (float)C;
  c2 = warp_sum(c2) / (float)C;
#pragma unroll
  for (int k = 0; k < LN_MAX_CHUNKS; ++k) {
    const int ch = k * 32 + lane;
    if (ch < nchunks) {
      const int64_t e0 = row * C + ch * 8;
      float r[8];
#pragma unroll
      for (int t = 0; t < 8; ++t) r[t] = rs * (g[k][t] - c1 - xh[k][t] * c2);
      if (ds != nullptr) store8<T>(ds + e0, r);
      if (dx != nullptr) {
        if (thr != 0) dropout8(r, (uint64_t)e0, thr, dscale, seed, offset);
        store8<T>(dx + e0, r);
      }
    }
  }
}

// dgamma[c] += sum_r dy[r][c] * xhat[r][c]; dbeta[c] += sum_r dy[r][c].  grid (C/64, row splits), block (32, 8):
// each lane owns two adjacent columns (4-byte / 8-byte loads), partials combined with fp32 atomics.
template <typename T> __device__ __forceinline__ float2 load2(const T* p);
template <> __device__ __forceinline__ float2 load2<float>(const float* p) { return *reinterpret_cast<const float2*>(p); }
template <> __device__ __forceinline__ float2 load2<__nv_bfloat16>(const __nv_bfloat16* p) {
  return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(p));
}
template <typename T>
__global__ void __launch_bounds__(256)
    ln_bwd_param_kernel(const T* __restrict__ dy, const T* __restrict__ s_in, const float* __restrict__ mean,
                        const float* __restrict__ rstd, float* __restrict__ dgamma, float* __restrict__ dbeta,
                        int64_t rows, int C, int64_t rows_per_block) {
  const int c = blockIdx.x * 64 + threadIdx.x * 2;
  const int64_t r0 = (int64_t)blockIdx.y * rows_per_block;
  const int64_t r1 = r0 + rows_per_block < rows ? r0 + rows_per_block : rows;
  float ga = 0.f, gb = 0.f, ba = 0.f, bb = 0.f;
  if (c < C) {
    for (int64_t r = r0 + threadIdx.y; r < r1; r += 8) {
      const float mu = mean[r], rs = rstd[r];
      const float2 d = load2<T>(dy + r * C + c), sv = load2<T>(s_in + r * C + c);
      ga += d.x * (sv.x - mu) * rs; gb += d.y * (sv.y - mu) * rs;
      ba += d.x; bb += d.y;
    }
  }
  __shared__ float red[4][8][33];
  red[0][threadIdx.y][threadIdx.x] = ga; red[1][threadIdx.y][threadIdx.x] = gb;
  red[2][threadIdx.y][threadIdx.x] = ba; red[3][threadIdx.y][threadIdx.x] = bb;
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      s0 += red[0][k][threadIdx.x]; s1 += red[1][k][threadIdx.x];
      s2 += red[2][k][threadIdx.x]; s3 += red[3][k][threadIdx.x];
    }
    if (dgamma != nullptr) { atomicAdd(dgamma + c, s0); atomicAdd(dgamma + c + 1, s1); }
    if (dbeta != nullptr) { atomicAdd(dbeta + c, s2); atomicAdd(dbeta + c + 1, s3); }
  }
}

// Input gradient AND parameter gradients in ONE pass over dy / s (the two-kernel form reads both tensors twice):
// persistent grid, warp per row. The per-channel sums -- dgamma, dbeta and, when asked for, the column sums of dx (= the
// bias gradient of the projection that produced x: its separate column-sum launch disappears) -- live in a PRIVATE
// shared-memory strip per warp (plain read-modify-write of the lane's own 16-byte slots, conflict-free layout), which
// frees the registers for a one-row-ahead prefetch of dy / s: a warp visits only 2-5 rows, so without the prefetch every
// row costs a full exposed HBM round trip; what bounds it then is bytes in flight: 16 warps x 3 KB per SM. The strips
// meet after a CTA barrier and leave as
// 16-byte vector reductions (red.global.add.v4.f32) when the targets are 16-byte aligned. NCH = 16-byte chunks per lane.
constexpr int LNB_WARPS = 8;
constexpr int LNB_NACC = 3;  // dgamma | dbeta | column sums of dx

template <typename T> struct Raw8;
template <> struct Raw8<__nv_bfloat16> {
  uint4 u;
  __device__ __forceinline__ void load(const __nv_bfloat16* p) { u = *reinterpret_cast<const uint4*>(p); }
  __device__ __forceinline__ void decode(float* v) const {
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const float2 f = __bfloat1622float2(h[t]);
      v[2 * t] = f.x; v[2 * t + 1] = f.y;
    }
  }
};
template <> struct Raw8<float> {
  float4 a, b;
  __device__ __forceinline__ void load(const float* p) {
    a = reinterpret_cast<const float4*>(p)[0];
    b = reinterpret_cast<const float4*>(p)[1];
  }
  __device__ __forceinline__ void decode(float* v) const {
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  }
};

__device__ __forceinline__ void red_add_v4(float* p, float4 v) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

template <typename T, int NCH>
__global__ void __launch_bounds__(LNB_WARPS * 32, 2)
    ln_bwd_fused_kernel(const T* __restrict__ dy, const T* __restrict__ s_in, const float* __restrict__ mean,
                        const float* __restrict__ rstd, const float* __restrict__ gamma, T* __restrict__ ds,
                        T* __restrict__ dx, float* __restrict__ dgamma, float* __restrict__ dbeta,
                        float* __restrict__ dxsum, int64_t rows, int C, uint32_t thr, float dscale, uint64_t seed,
                        uint64_t offset) {
  extern __shared__ __align__(16) float ln_acc[];  // [LNB_WARPS][LNB_NACC][C]; channel ch*8+t at (t>>2)*(C/2) + ch*4 + (t&3)
  constexpr bool PF = sizeof(T) == 2;  // one-row-ahead prefetch (24 registers for bf16; fp32 rows would need 48)
  {  // (the strips are this CTA's own shared memory: cleared while the preceding grid drains)
    float4* z = reinterpret_cast<float4*>(ln_acc);
    for (int t = threadIdx.x; t < LNB_WARPS * LNB_NACC * (C >> 2); t += LNB_WARPS * 32) z[t] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  pdl_sync();
  __syncthreads();
  if (thr != 0) resolve_seed(seed, offset);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nchunks = C >> 3;
  const int half4 = C >> 3;  // float4 index of the second half of an accumulator
  float4* acc = reinterpret_cast<float4*>(ln_acc + (size_t)warp * LNB_NACC * C);
  const int acc4 = C >> 2;   // float4 per accumulator
  const int64_t stride = (int64_t)gridDim.x * LNB_WARPS;
  int64_t row = (int64_t)blockIdx.x * LNB_WARPS + warp;
  Raw8<T> cd[NCH], cs[NCH];
  float mu = 0.f, rs = 0.f;
  if (PF && row < rows) {
#pragma unroll
    for (int k = 0; k < NCH; ++k) {
      const int ch = k * 32 + lane;
      if (ch < nchunks) {
        cd[k].load(dy + row * C + ch * 8);
        cs[k].load(s_in + row * C + ch * 8);
      }
    }
    mu = mean[row];
    rs = rstd[row];
  }
  for (; row < rows; row += stride) {
    if constexpr (!PF) {
#pragma unroll
      for (int k = 0; k < NCH; ++k) {
        const int ch = k * 32 + lane;
        if (ch < nchunks) {
          cd[k].load(dy + row * C + ch * 8);
          cs[k].load(s_in + row * C + ch * 8);
        }
      }
      mu = mean[row];
      rs = rstd[row];
    }
    float d[NCH][8], xh[NCH][8];
#pragma unroll
    for (int k = 0; k < NCH; ++k) {
      if (k * 32 + lane < nchunks) {
        cd[k].decode(d[k]);
        cs[k].decode(xh[k]);
#pragma unroll
        for (int t = 0; t < 8; ++t) xh[k][t] = (xh[k][t] - mu) * rs;
      }
    }
    const float rs_cur = rs;
    if constexpr (PF) {  // the raw registers are free again: the next row's loads fly under this row's arithmetic
      const int64_t nxt = row + stride;
      if (nxt < rows) {
#pragma unroll
        for (int k = 0; k < NCH; ++k) {
          const int ch = k * 32 + lane;
          if (ch < nchunks) {
            cd[k].load(dy + nxt * C + ch * 8);
            cs[k].load(s_in + nxt * C + ch * 8);
          }
        }
        mu = mean[nxt];
        rs = rstd[nxt];
      }
    }
    float c1 = 0.f, c2 = 0.f;
#pragma unroll
    for (int k = 0; k < NCH; ++k) {
      const int ch = k * 32 + lane;
      if (ch < nchunks) {
        float gm[8];
        load8<float>(gamma + ch * 8, gm);
        float4 g0 = acc[ch], g1 = acc[half4 + ch], b0 = acc[acc4 + ch], b1 = acc[acc4 + half4 + ch];
        g0.x += d[k][0] * xh[k][0]; g0.y += d[k][1] * xh[k][1]; g0.z += d[k][2] * xh[k][2]; g0.w += d[k][3] * xh[k][3];
        g1.x += d[k][4] * xh[k][4]; g1.y += d[k][5] * xh[k][5]; g1.z += d[k][6] * xh[k][6]; g1.w += d[k][7] * xh[k][7];
        b0.x += d[k][0]; b0.y += d[k][1]; b0.z += d[k][2]; b0.w += d[k][3];
        b1.x += d[k][4]; b1.y += d[k][5]; b1.z += d[k][6]; b1.w += d[k][7];
        acc[ch] = g0; acc[half4 + ch] = g1; acc[acc4 + ch] = b0; acc[acc4 + half4 + ch] = b1;
#pragma unroll
        for (int t = 0; t < 8; ++t) {
          d[k][t] *= gm[t];  // g = dy * gamma from here on
          c1 += d[k][t];
          c2 += d[k][t] * xh[k][t];
        }
      }
    }
    c1 = warp_sum(c1) / (float)C;
    c2 = warp_sum(c2) / (float)C;
#pragma unroll
    for (int k = 0; k < NCH; ++k) {
      const int ch = k * 32 + lane;
      if (ch < nchunks) {
        const int64_t e0 = row * C + ch * 8;
        float r[8];
#pragma unroll
        for (int t = 0; t < 8; ++t) r[t] = rs_cur * (d[k][t] - c1 - xh[k][t] * c2);
        if (ds != nullptr) store8<T>(ds + e0, r);
        if (dx != nullptr) {
          if (thr != 0) dropout8(r, (uint64_t)e0, thr, dscale, seed, offset);
          store8<T>(dx + e0, r);
        }
        if (dxsum != nullptr) {  // (without dropout dx == ds: the sums are those of r either way)
          float4 x0 = acc[2 * acc4 + ch], x1 = acc[2 * acc4 + half4 + ch];
          x0.x += r[0]; x0.y += r[1]; x0.z += r[2]; x0.w += r[3];
          x1.x += r[4]; x1.y += r[5]; x1.z += r[6]; x1.w += r[7];
          acc[2 * acc4 + ch] = x0; acc[2 * acc4 + half4 + ch] = x1;
        }
      }
    }
  }
  __syncthreads();
  // strips -> global: item = (accumulator a, float4 slot q); slot q < C/8 holds channels 8q..8q+3, else 8(q-C/8)+4..+7
  const float4* all = reinterpret_cast<const float4*>(ln_acc);
  for (int it = threadIdx.x; it < LNB_NACC * acc4; it += LNB_WARPS * 32) {
    const int a = it / acc4, q = it - a * acc4;
    float* dst = a == 0 ? dgamma : (a == 1 ? dbeta : dxsum);
    if (dst == nullptr) continue;
    float4 v = all[it];
#pragma unroll
    for (int w = 1; w < LNB_WARPS; ++w) {
      const float4 o = all[(size_t)w * LNB_NACC * acc4 + it];
      v.x += o.x; v.y += o.y; v.z += o.z; v.w += o.w;
    }
    const int c0 = q < half4 ? q * 8 : (q - half4) * 8 + 4;
    if ((reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
      red_add_v4(dst + c0, v);
    } else {
      atomicAdd(dst + c0, v.x); atomicAdd(dst + c0 + 1, v.y); atomicAdd(dst + c0 + 2, v.z); atomicAdd(dst + c0 + 3, v.w);
    }
  }
}

template <typename T, int NCH>
static int ln_bwd_fused_run(const void* dy, const void* s_in, const float* mean, const float* rstd, const float* gamma,
                            void* ds, void* dx, float* dgamma, float* dbeta, float* dxsum, int64_t rows, int C,
                            uint32_t thr, float dsc, uint64_t seed, uint64_t offset, cudaStream_t s) {
  static bool attr_set = false;  // (one per kernel instantiation)
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(ln_bwd_fused_kernel<T, NCH>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         LNB_WARPS * LNB_NACC * NCH * 256 * (int)sizeof(float));
    if (e != cudaSuccess) return (int)e;
    attr_set = true;
  }
  int64_t want = (rows + LNB_WARPS - 1) / LNB_WARPS;
  const int64_t cap = 2 * (int64_t)device_sm_count();
  const unsigned grid = (unsigned)(want < cap ? want : cap);
  const size_t smem = (size_t)LNB_WARPS * LNB_NACC * C * sizeof(float);
  launch_pdl(ln_bwd_fused_kernel<T, NCH>, dim3(grid), dim3(LNB_WARPS * 32), smem, s, (const T*)dy, (const T*)s_in, mean, rstd, gamma, (T*)ds,
                                                                 (T*)dx, dgamma, dbeta, dxsum, rows, C, thr, dsc, seed, offset);
  return 0;
}

template <typename T>
static int ln_bwd_fused_dispatch(const void* dy, const void* s_in, const float* mean, const float* rstd, const float* gamma,
                                 void* ds, void* dx, float* dgamma, float* dbeta, float* dxsum, int64_t rows, int C,
                                 uint32_t thr, float dsc, uint64_t seed, uint64_t offset, cudaStream_t s) {
  if (C <= 768)
    return ln_bwd_fused_run<T, 3>(dy, s_in, mean, rstd, gamma, ds, dx, dgamma, dbeta, dxsum, rows, C, thr, dsc, seed, offset, s);
  return ln_bwd_fused_run<T, LN_MAX_CHUNKS>(dy, s_in, mean, rstd, gamma, ds, dx, dgamma, dbeta, dxsum, rows, C, thr, dsc, seed,
                                            offset, s);
}

int ln_bwd_launch(const void* dy, const void* s_in, const float* mean, const float* rstd, const float* gamma, void* ds,
                  void* dx, float* dgamma, float* dbeta, float* dxsum, int dtype, int64_t rows, int64_t C,
                  float drop_p, uint64_t seed, uint64_t offset, cudaStream_t s) {
  if (rows == 0) return 0;
  if (C > 8 * 32 * LN_MAX_CHUNKS || C <= 0 || (C & 7)) return -2;
  const uint32_t thr = drop_threshold(drop_p);
  const float dsc = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  if ((dgamma != nullptr || dbeta != nullptr || dxsum != nullptr) && (rows >= 64 || dxsum != nullptr)) {
    // one pass over dy / s for dx, the parameter sums and the column sums of dx
    int rc;
    if (dtype == ST5_F32)
      rc = ln_bwd_fused_dispatch<float>(dy, s_in, mean, rstd, gamma, ds, dx, dgamma, dbeta, dxsum, rows, (int)C, thr, dsc,
                                        seed, offset, s);
    else
      rc = ln_bwd_fused_dispatch<__nv_bfloat16>(dy, s_in, mean, rstd, gamma, ds, dx, dgamma, dbeta, dxsum, rows, (int)C, thr,
                                                dsc, seed, offset, s);
    return rc != 0 ? rc : (int)cudaGetLastError();
  }
  const unsigned grid = (unsigned)((rows + LN_WARPS - 1) / LN_WARPS);
  int64_t splits = (rows + 255) / 256;
  if (splits > 96) splits = 96;
  const int64_t rpb = (rows + splits - 1) / splits;
  dim3 pgrid((unsigned)((C + 63) / 64), (unsigned)splits), pblock(32, 8);
  if (dtype == ST5_F32) {
    ln_bwd_dx_kernel<float><<<grid, LN_WARPS * 32, 0, s>>>((const float*)dy, (const float*)s_in, mean, rstd, gamma,
                                                           (float*)ds, (float*)dx, rows, (int)C, thr, dsc, seed, offset);
    if (dgamma != nullptr || dbeta != nullptr)
      ln_bwd_param_kernel<float><<<pgrid, pblock, 0, s>>>((const float*)dy, (const float*)s_in, mean, rstd, dgamma,
                                                          dbeta, rows, (int)C, rpb);
  } else {
    ln_bwd_dx_kernel<__nv_bfloat16><<<grid, LN_WARPS * 32, 0, s>>>(
        (const __nv_bfloat16*)dy, (const __nv_bfloat16*)s_in, mean, rstd, gamma, (__nv_bfloat16*)ds, (__nv_bfloat16*)dx,
        rows, (int)C, thr, dsc, seed, offset);
    if (dgamma != nullptr || dbeta != nullptr)
      ln_bwd_param_kernel<__nv_bfloat16><<<pgrid, pblock, 0, s>>>((const __nv_bfloat16*)dy, (const __nv_bfloat16*)s_in,
                                                                  mean, rstd, dgamma, dbeta, rows, (int)C, rpb);
  }
  return (int)cudaGetLastError();
}

}  // namespace st5
