// Gradient-norm reduction and fused clip + Adam + bf16-shadow refresh over the flat parameter buffer.
// Semantics follow the reference trainer: fairseq/trainer.py:796-826 (multiply_grads -> clip_grad_norm -> step),
// fairseq/utils.py:clip_grad_norm_ (coef = max_norm / (norm + 1e-6), clamped to 1), fairseq/optim/adam.py:Adam.step
// (denom = sqrt(v) + eps; step = lr * sqrt(1 - b2^t) / (1 - b1^t); weight decay p -= wd * lr * p).
#include "kernels.cuh"

namespace st5 {

__global__ void sumsq_kernel(const float* __restrict__ x, int64_t n, float* __restrict__ out) {
  pdl_sync();
  float acc = 0.f;
  const int64_t n4 = n / 4;
  const float4* x4 = reinterpret_cast<const float4*>(x);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 v = x4[i];
    acc += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  }
  for (int64_t i = n4 * 4 + blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    acc += x[i] * x[i];
  __shared__ float red[32];
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    v = warp_sum(v);
    if (threadIdx.x == 0) atomicAdd(out, v);
  }
}
int sumsq_launch(const float* x, int64_t n, float* out, cudaStream_t s) {
  if (n == 0) return 0;
  if (reinterpret_cast<uintptr_t>(x) & 15) return -2;
  int64_t g = (n / 4 + 255) / 256;
  if (g > 132 * 8) g = 132 * 8;
  if (g < 1) g = 1;
  launch_pdl(sumsq_kernel, dim3((unsigned)g), dim3(256), 0, s, x, n, out);
  return (int)cudaGetLastError();
}

__global__ void adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                            float* __restrict__ v, __nv_bfloat16* __restrict__ pb, int64_t n, float lr, float beta1,
                            float beta2, float eps, float wd, float step_size, const float* __restrict__ gnorm_sq,
                            float max_norm, float grad_mul, const float* __restrict__ lr_dev,
                            const int64_t* __restrict__ step_dev) {
  pdl_sync();
  if (lr_dev != nullptr) lr = *lr_dev;
  if (step_dev != nullptr) {  // device-resident schedule state: a captured CUDA graph stays valid across updates
    const float t = (float)(*step_dev);
    step_size = lr * sqrtf(1.f - powf(beta2, t)) / (1.f - powf(beta1, t));
  } else if (lr_dev != nullptr) {
    step_size = lr * step_size;  // host passed the bias-correction factor only
  }
  // fairseq/trainer.py:845-858 raises FloatingPointError on a NaN / Inf gradient norm and the update is not applied;
  // here the whole launch is a no-op (parameters, both moments and the bf16 shadow untouched) and the host reads the
  // overflow counter when it chooses to (B200Trainer.check_overflow) -- nothing to notice it inside a graph replay.
  if (gnorm_sq != nullptr && !(*gnorm_sq <= 3.0e38f)) return;
  float gscale = grad_mul;
  if (gnorm_sq != nullptr && max_norm > 0.f) {
    const float norm = sqrtf(*gnorm_sq) * grad_mul;
    const float coef = max_norm / (norm + 1e-6f);
    gscale *= coef < 1.f ? coef : 1.f;
  }
  const float omb1 = 1.f - beta1, omb2 = 1.f - beta2, wdlr = wd * lr;
  auto upd = [&](float& pi, float gi, float& mi, float& vi) {
    gi *= gscale;
    mi = beta1 * mi + omb1 * gi;
    vi = beta2 * vi + omb2 * gi * gi;
    if (wd != 0.f) pi -= wdlr * pi;
    pi -= step_size * mi / (sqrtf(vi) + eps);
  };
  // 16-byte accesses (30 B of HBM traffic per parameter is the whole cost of this kernel); scalar tail / fallback
  const bool vec = (((uintptr_t)p | (uintptr_t)g | (uintptr_t)m | (uintptr_t)v) & 15) == 0 &&
                   (pb == nullptr || ((uintptr_t)pb & 7) == 0);
  const int64_t n4 = vec ? n >> 2 : 0;
  const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x, nth = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = tid; i < n4; i += nth) {
    const float4 g4 = __ldcs(reinterpret_cast<const float4*>(g) + i);
    float4 m4 = reinterpret_cast<float4*>(m)[i], v4 = reinterpret_cast<float4*>(v)[i], p4 = reinterpret_cast<float4*>(p)[i];
    upd(p4.x, g4.x, m4.x, v4.x); upd(p4.y, g4.y, m4.y, v4.y); upd(p4.z, g4.z, m4.z, v4.z); upd(p4.w, g4.w, m4.w, v4.w);
    reinterpret_cast<float4*>(m)[i] = m4;
    reinterpret_cast<float4*>(v)[i] = v4;
    reinterpret_cast<float4*>(p)[i] = p4;
    if (pb != nullptr) {
      __nv_bfloat162 lo = __floats2bfloat162_rn(p4.x, p4.y), hi = __floats2bfloat162_rn(p4.z, p4.w);
      uint2 pk;
      pk.x = *reinterpret_cast<uint32_t*>(&lo);
      pk.y = *reinterpret_cast<uint32_t*>(&hi);
      reinterpret_cast<uint2*>(pb)[i] = pk;
    }
  }
  for (int64_t i = n4 * 4 + tid; i < n; i += nth) {
    float pi = p[i], mi = m[i], vi = v[i];
    upd(pi, g[i], mi, vi);
    m[i] = mi; v[i] = vi; p[i] = pi;
    if (pb != nullptr) pb[i] = __float2bfloat16(pi);
  }
}
int adam_launch(float* p, const float* g, float* m, float* v, void* p_bf16, int64_t n, float lr, float beta1,
                float beta2, float eps, float weight_decay, int64_t step, const float* grad_norm_sq, float max_norm,
                float grad_mul, const float* lr_dev, const int64_t* step_dev, cudaStream_t s) {
  if (n == 0) return 0;
  if (step < 1 && step_dev == nullptr) return -2;
  float step_size = 0.f;
  if (step_dev == nullptr) {
    const double bc1 = 1.0 - pow((double)beta1, (double)step);
    const double bc2 = 1.0 - pow((double)beta2, (double)step);
    step_size = (float)((lr_dev != nullptr ? 1.0 : (double)lr) * sqrt(bc2) / bc1);
  }
  int64_t gsz = (n + 255) / 256;
  if (gsz > 132 * 16) gsz = 132 * 16;
  launch_pdl(adam_kernel, dim3((unsigned)gsz), dim3(256), 0, s, p, g, m, v, (__nv_bfloat16*)p_bf16, n, lr, beta1, beta2, eps, weight_decay, step_size, grad_norm_sq, max_norm, grad_mul, lr_dev, step_dev);
  return (int)cudaGetLastError();
}

}  // namespace st5
