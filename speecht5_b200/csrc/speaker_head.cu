// Speaker-identification head (speecht5/models/modules/speaker_decoder_postnet.py:16-197) and the speaker criterion
// (SpeechtoTextLoss on the class logits, speecht5/criterions/speech_to_text_loss.py:93-110, 340-372):
//   l2norm_rows     y = x / max(||x||, 1e-12) per row (F.normalize), the embeddings [B, E] and the class weight [N, E]
//   margin_ce       one CTA per row of the logits [B, N]: additive / angular margin on one column, log-softmax,
//                   label-smoothed NLL, arg-max correctness; backward forms d logits including d phi / d cos
//   time_mean       mean over ALL frames of [B, T, C] (the reference's `.mean(1)` keeps padded frames)
// Everything is fp32 arithmetic; row sums run in a fixed order (same inputs, same bits).
#include "kernels.cuh"
#include <math_constants.h>

namespace st5 {

constexpr float L2_EPS = 1e-12f;
constexpr int L2_WARPS = 8;
constexpr int MCE_THREADS = 256;

__device__ __forceinline__ float block_sum(float v, float* red) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = 0.f;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += red[w];
  return t;
}

// ------------------------------------------------------------------------------------------------ row L2 normalisation
template <typename T>
__global__ void __launch_bounds__(L2_WARPS * 32)
    l2norm_rows_fwd_kernel(const T* __restrict__ x, int64_t x_ld, float* __restrict__ y, float* __restrict__ nrm,
                           int64_t rows, int64_t E) {
  pdl_sync();
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * L2_WARPS + (threadIdx.x >> 5);
  if (row >= rows) return;
  const T* xr = x + row * x_ld;
  float ss = 0.f;
  for (int64_t c = lane; c < E; c += 32) {
    const float v = ldf<T>(xr + c);
    ss += v * v;
  }
  const float n = sqrtf(warp_sum(ss));
  const float inv = 1.f / fmaxf(n, L2_EPS);
  for (int64_t c = lane; c < E; c += 32) y[row * E + c] = ldf<T>(xr + c) * inv;
  if (lane == 0) nrm[row] = n;
}

// d x = (dy - y <dy, y>) / ||x|| where ||x|| >= eps (the clamp passes its gradient), else dy / eps
template <typename T>
__global__ void __launch_bounds__(L2_WARPS * 32)
    l2norm_rows_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ y, const float* __restrict__ nrm,
                           T* __restrict__ dx, int64_t dx_ld, int accumulate, int64_t rows, int64_t E) {
  pdl_sync();
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * L2_WARPS + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float* dr = dy + row * E;
  const float* yr = y + row * E;
  const float n = nrm[row];
  const bool clamped = n < L2_EPS;
  float dot = 0.f;
  if (!clamped)
    for (int64_t c = lane; c < E; c += 32) dot += dr[c] * yr[c];
  dot = warp_sum(dot);
  const float inv = 1.f / fmaxf(n, L2_EPS);
  T* xr = dx + row * dx_ld;
  for (int64_t c = lane; c < E; c += 32) {
    float g = (dr[c] - yr[c] * dot) * inv;
    if (accumulate) g += ldf<T>(xr + c);
    stf<T>(xr + c, g);
  }
}

// ------------------------------------------------------------------------------------------------ margin + CE rows
struct Margin {
  int mode;  // ST5_MARGIN_NONE / _AM / _AAM
  float s, m, cos_m, sin_m, th, mm;
  int easy;
};

// logit of column j of a row whose margin column is mt (-1: no margin, plain logits)
__device__ __forceinline__ float margin_logit(const Margin& g, float c, int j, int mt) {
  if (mt < 0) return c;
  if (j != mt) return g.s * c;
  if (g.mode == ST5_MARGIN_AM) return g.s * (c - g.m);
  const float sine = sqrtf(fminf(fmaxf(1.f - c * c, 0.f), 1.f));
  const float phi = c * g.cos_m - sine * g.sin_m;
  const bool keep = g.easy ? (c > 0.f) : (c > g.th);
  return g.s * (keep ? phi : (g.easy ? c : c - g.mm));
}

// d logit / d c of the same column
__device__ __forceinline__ float margin_slope(const Margin& g, float c, int j, int mt) {
  if (mt < 0) return 1.f;
  if (j != mt || g.mode == ST5_MARGIN_AM) return g.s;
  const float q = 1.f - c * c;
  const float sine = sqrtf(fminf(fmaxf(q, 0.f), 1.f));
  // torch: clamp passes the gradient inside [0, 1]; d sqrt(q) / d c = -c / sqrt(q)
  const float dsine = (q >= 0.f && q <= 1.f && sine > 0.f) ? -c / sine : 0.f;
  const bool keep = g.easy ? (c > 0.f) : (c > g.th);
  return g.s * (keep ? (g.cos_m - dsine * g.sin_m) : 1.f);
}

__global__ void __launch_bounds__(MCE_THREADS)
    margin_ce_fwd_kernel(const float* __restrict__ x, int64_t x_ld, int N, const int64_t* __restrict__ mtarget,
                         Margin g, float* __restrict__ z_out, int64_t z_ld, const int64_t* __restrict__ target,
                         float eps, int64_t ignore_index, float* __restrict__ stats, float* __restrict__ lse_out) {
  pdl_sync();
  __shared__ float red[MCE_THREADS / 32];
  __shared__ float redv[MCE_THREADS / 32];
  __shared__ int redi[MCE_THREADS / 32];
  const int b = blockIdx.x;
  const float* xr = x + (int64_t)b * x_ld;
  const int mt = mtarget != nullptr ? (int)mtarget[b] : -1;
  float mx = -CUDART_INF_F, sz = 0.f;
  int ix = N;
  for (int j = threadIdx.x; j < N; j += MCE_THREADS) {
    const float z = margin_logit(g, xr[j], j, mt);
    if (z_out != nullptr) z_out[(int64_t)b * z_ld + j] = z;
    if (z > mx) { mx = z; ix = j; }  // (increasing j per thread: the first maximum is kept)
    sz += z;
  }
  if (target == nullptr) return;
  // arg-max with the lowest index among equal maxima (torch.argmax)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float v2 = __shfl_xor_sync(0xffffffffu, mx, o);
    const int i2 = __shfl_xor_sync(0xffffffffu, ix, o);
    if (v2 > mx || (v2 == mx && i2 < ix)) { mx = v2; ix = i2; }
  }
  if (lane == 0) { redv[warp] = mx; redi[warp] = ix; }
  __syncthreads();
  mx = redv[0];
  ix = redi[0];
  for (int w = 1; w < MCE_THREADS / 32; ++w)
    if (redv[w] > mx || (redv[w] == mx && redi[w] < ix)) { mx = redv[w]; ix = redi[w]; }
  float se = 0.f;
  for (int j = threadIdx.x; j < N; j += MCE_THREADS) se += __expf(margin_logit(g, xr[j], j, mt) - mx);
  se = block_sum(se, red);
  sz = block_sum(sz, red);
  if (threadIdx.x != 0) return;
  const float lse = mx + logf(se);
  const int64_t t = target[b];
  const bool valid = t != ignore_index;
  float loss = 0.f, nll = 0.f;
  if (valid && (t < 0 || t >= N)) {
    loss = nll = CUDART_NAN_F;  // a class index outside the logits: reported, never read out of bounds
  } else if (valid) {
    nll = lse - margin_logit(g, xr[t], (int)t, mt);
    const float smooth = (float)N * lse - sz;  // -sum_j log p_j
    const float eps_i = eps / (float)(N - 1);
    loss = (1.f - eps - eps_i) * nll + eps_i * smooth;
  }
  stats[4 * b + 0] = loss;
  stats[4 * b + 1] = nll;
  stats[4 * b + 2] = (valid && ix == (int)t) ? 1.f : 0.f;
  stats[4 * b + 3] = valid ? 1.f : 0.f;
  lse_out[b] = lse;
}

__global__ void __launch_bounds__(MCE_THREADS)
    margin_ce_bwd_kernel(const float* __restrict__ x, int64_t x_ld, int N, const int64_t* __restrict__ mtarget,
                         Margin g, const int64_t* __restrict__ target, float eps, int64_t ignore_index,
                         const float* __restrict__ lse, const float* __restrict__ gstat,
                         const float* __restrict__ dz_in, int64_t dz_ld, float* __restrict__ dx, int64_t dx_ld) {
  pdl_sync();
  const int b = blockIdx.x;
  const float* xr = x + (int64_t)b * x_ld;
  float* dr = dx + (int64_t)b * dx_ld;
  const int mt = mtarget != nullptr ? (int)mtarget[b] : -1;
  int64_t t = -1;
  float ga = 0.f, gn = 0.f, eps_i = 0.f, l = 0.f;
  if (target != nullptr) {
    t = target[b];
    if (t != ignore_index) {
      eps_i = eps / (float)(N - 1);
      ga = gstat[0];
      gn = gstat[1];
      l = lse[b];
    }
  }
  const bool valid = target != nullptr && t != ignore_index;
  for (int j = threadIdx.x; j < N; j += MCE_THREADS) {
    const float c = xr[j];
    float dz;
    if (target != nullptr) {
      if (valid) {
        const float p = __expf(margin_logit(g, c, j, mt) - l);
        const float hit = j == (int)t ? 1.f : 0.f;
        dz = ga * ((1.f - eps - eps_i) * (p - hit) + eps_i * ((float)N * p - 1.f)) + gn * (p - hit);
      } else {
        dz = 0.f;
      }
    } else {
      dz = dz_in[(int64_t)b * dz_ld + j];
    }
    dr[j] = dz * margin_slope(g, c, j, mt);
  }
}

// ------------------------------------------------------------------------------------------------ mean over time
constexpr int TM_COLS = 32, TM_ROWS = 8;

template <typename T>
__global__ void __launch_bounds__(TM_COLS * TM_ROWS)
    time_mean_fwd_kernel(const T* __restrict__ x, T* __restrict__ y, int64_t Tn, int64_t C) {
  pdl_sync();
  __shared__ float part[TM_ROWS][TM_COLS];
  const int tx = threadIdx.x % TM_COLS, ty = threadIdx.x / TM_COLS;
  const int64_t b = blockIdx.y, c = (int64_t)blockIdx.x * TM_COLS + tx;
  float s = 0.f;
  if (c < C)
    for (int64_t t = ty; t < Tn; t += TM_ROWS) s += ldf<T>(x + (b * Tn + t) * C + c);
  part[ty][tx] = s;
  __syncthreads();
  if (ty == 0 && c < C) {
    float a = 0.f;
#pragma unroll
    for (int r = 0; r < TM_ROWS; ++r) a += part[r][tx];
    stf<T>(y + b * C + c, a / (float)Tn);
  }
}

template <typename T>
__global__ void time_mean_bwd_kernel(const T* __restrict__ dy, T* __restrict__ dx, int64_t Tn, int64_t C, int64_t n) {
  pdl_sync();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int64_t c = i % C, b = i / (Tn * C);
  stf<T>(dx + i, ldf<T>(dy + b * C + c) / (float)Tn);
}

static Margin make_margin(int mode, float scale, float margin, int easy) {
  Margin g;
  g.mode = mode;
  g.s = scale;
  g.m = margin;
  g.cos_m = cosf(margin);
  g.sin_m = sinf(margin);
  g.th = cosf(CUDART_PI_F - margin);
  g.mm = sinf(CUDART_PI_F - margin) * margin;
  g.easy = easy;
  return g;
}

int l2norm_rows_fwd_launch(const void* x, int64_t x_ld, int dtype, float* y, float* nrm, int64_t rows, int64_t E,
                           cudaStream_t s) {
  if (rows < 0 || E <= 0 || x_ld < E || (dtype != ST5_F32 && dtype != ST5_BF16)) return -2;
  if (rows == 0) return 0;
  const dim3 grid((unsigned)((rows + L2_WARPS - 1) / L2_WARPS)), block(L2_WARPS * 32);
  cudaError_t e = dtype == ST5_F32
      ? launch_pdl(l2norm_rows_fwd_kernel<float>, grid, block, 0, s, (const float*)x, x_ld, y, nrm, rows, E)
      : launch_pdl(l2norm_rows_fwd_kernel<__nv_bfloat16>, grid, block, 0, s, (const __nv_bfloat16*)x, x_ld, y, nrm,
                   rows, E);
  return (int)e;
}

int l2norm_rows_bwd_launch(const float* dy, const float* y, const float* nrm, void* dx, int64_t dx_ld, int dtype,
                           int accumulate, int64_t rows, int64_t E, cudaStream_t s) {
  if (rows < 0 || E <= 0 || dx_ld < E || (dtype != ST5_F32 && dtype != ST5_BF16)) return -2;
  if (accumulate && dtype != ST5_F32) return -3;
  if (rows == 0) return 0;
  const dim3 grid((unsigned)((rows + L2_WARPS - 1) / L2_WARPS)), block(L2_WARPS * 32);
  cudaError_t e = dtype == ST5_F32
      ? launch_pdl(l2norm_rows_bwd_kernel<float>, grid, block, 0, s, dy, y, nrm, (float*)dx, dx_ld, accumulate, rows, E)
      : launch_pdl(l2norm_rows_bwd_kernel<__nv_bfloat16>, grid, block, 0, s, dy, y, nrm, (__nv_bfloat16*)dx, dx_ld,
                   accumulate, rows, E);
  return (int)e;
}

static bool margin_ok(int mode, int N) {
  return (mode == ST5_MARGIN_NONE || mode == ST5_MARGIN_AM || mode == ST5_MARGIN_AAM) && N >= 2;
}

int margin_ce_fwd_launch(const float* x, int64_t x_ld, int32_t B, int32_t N, const int64_t* mtarget, int mode,
                         float scale, float margin, int easy, float* z_out, int64_t z_ld, const int64_t* target,
                         float eps, int64_t ignore_index, float* stats, float* lse, cudaStream_t s) {
  if (B < 0 || !margin_ok(mode, N) || x_ld < N || (z_out != nullptr && z_ld < N)) return -2;
  if (mtarget != nullptr && mode == ST5_MARGIN_NONE) return -2;
  if (target != nullptr && (stats == nullptr || lse == nullptr)) return -2;
  if (B == 0) return 0;
  return (int)launch_pdl(margin_ce_fwd_kernel, dim3(B), dim3(MCE_THREADS), 0, s, x, x_ld, N, mtarget,
                         make_margin(mode, scale, margin, easy), z_out, z_ld, target, eps, ignore_index, stats, lse);
}

int margin_ce_bwd_launch(const float* x, int64_t x_ld, int32_t B, int32_t N, const int64_t* mtarget, int mode,
                         float scale, float margin, int easy, const int64_t* target, float eps, int64_t ignore_index,
                         const float* lse, const float* gstat, const float* dz_in, int64_t dz_ld, float* dx,
                         int64_t dx_ld, cudaStream_t s) {
  if (B < 0 || !margin_ok(mode, N) || x_ld < N || dx_ld < N) return -2;
  if (mtarget != nullptr && mode == ST5_MARGIN_NONE) return -2;
  if ((target == nullptr) == (dz_in == nullptr)) return -2;  // exactly one source of d logits
  if (target != nullptr && (lse == nullptr || gstat == nullptr)) return -2;
  if (dz_in != nullptr && dz_ld < N) return -2;
  if (B == 0) return 0;
  return (int)launch_pdl(margin_ce_bwd_kernel, dim3(B), dim3(MCE_THREADS), 0, s, x, x_ld, N, mtarget,
                         make_margin(mode, scale, margin, easy), target, eps, ignore_index, lse, gstat, dz_in, dz_ld,
                         dx, dx_ld);
}

int time_mean_fwd_launch(const void* x, void* y, int dtype, int64_t B, int64_t Tn, int64_t C, cudaStream_t s) {
  if (B < 0 || Tn <= 0 || C <= 0 || (dtype != ST5_F32 && dtype != ST5_BF16)) return -2;
  if (B == 0) return 0;
  const dim3 grid((unsigned)((C + TM_COLS - 1) / TM_COLS), (unsigned)B), block(TM_COLS * TM_ROWS);
  cudaError_t e = dtype == ST5_F32
      ? launch_pdl(time_mean_fwd_kernel<float>, grid, block, 0, s, (const float*)x, (float*)y, Tn, C)
      : launch_pdl(time_mean_fwd_kernel<__nv_bfloat16>, grid, block, 0, s, (const __nv_bfloat16*)x, (__nv_bfloat16*)y,
                   Tn, C);
  return (int)e;
}

int time_mean_bwd_launch(const void* dy, void* dx, int dtype, int64_t B, int64_t Tn, int64_t C, cudaStream_t s) {
  if (B < 0 || Tn <= 0 || C <= 0 || (dtype != ST5_F32 && dtype != ST5_BF16)) return -2;
  const int64_t n = B * Tn * C;
  if (n == 0) return 0;
  const dim3 grid((unsigned)((n + 255) / 256)), block(256);
  cudaError_t e = dtype == ST5_F32
      ? launch_pdl(time_mean_bwd_kernel<float>, grid, block, 0, s, (const float*)dy, (float*)dx, Tn, C, n)
      : launch_pdl(time_mean_bwd_kernel<__nv_bfloat16>, grid, block, 0, s, (const __nv_bfloat16*)dy,
                   (__nv_bfloat16*)dx, Tn, C, n);
  return (int)e;
}

}  // namespace st5
