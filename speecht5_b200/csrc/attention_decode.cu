// One-query-row attention for incremental decoding: the decoder's self-attention over its key/value cache and its
// cross-attention over the encoder, one new row per (utterance, head) and step.
//
// Reference: the incremental path of speecht5/models/modules/multihead_attention.py:255-330 (saved prev_key /
// prev_value, one query row) inside the synthesis loop of speecht5/models/speecht5.py:1222-1245.
//
// Split-KV: the keys of an utterance are cut into fixed splits of DCH keys. Each CTA of grid (splits, H, B) reduces one
// split to (max, sum of exponentials, 64-wide unnormalised accumulator); a combine kernel merges the splits in index
// order. Key j always lands in split j / DCH at the same lane position, and a masked key adds an exact zero (a split
// whose keys are all masked merges with weight zero), so an utterance's result depends only on its own valid keys: not
// on B and not on the buffer's key span (the bucket of a captured graph). An utterance whose keys are all masked has
// l = 0 on both paths; 1 / l is then taken as 0, so its output and probabilities are zeros on both paths alike.
#include "kernels.cuh"
#include "vec8.cuh"

namespace st5 {

constexpr int DT = 128;   // threads per CTA
constexpr int DH = 64;    // head dim
constexpr int DCH = 64;   // keys per split
constexpr int DPART = DH + 2;  // partial record: max, sum, accumulator[64]

__device__ __forceinline__ float* decode_probs(const st5_attn_decode_args& a, int b, int h) {
  return a.probs != nullptr ? a.probs + ((int64_t)b * a.H + h) * a.Tk : nullptr;
}

template <typename T> struct Vec16;
template <> struct Vec16<float> {
  static constexpr int N = 4;
  static __device__ __forceinline__ void load(const float* p, float* o) {
    const float4 v = *reinterpret_cast<const float4*>(p);
    o[0] = v.x; o[1] = v.y; o[2] = v.z; o[3] = v.w;
  }
};
template <> struct Vec16<__nv_bfloat16> {
  static constexpr int N = 8;
  static __device__ __forceinline__ void load(const __nv_bfloat16* p, float* o) {
    const uint4 v = *reinterpret_cast<const uint4*>(p);
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const float2 f = __bfloat1622float2(h[t]);
      o[2 * t] = f.x; o[2 * t + 1] = f.y;
    }
  }
};

__device__ __forceinline__ float cta_reduce(float v, float* red, bool is_max) {
  v = is_max ? warp_max(v) : warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = red[0];
#pragma unroll
  for (int w = 1; w < DT / 32; ++w) r = is_max ? fmaxf(r, red[w]) : r + red[w];
  return r;
}

// Where key / value j of query row b lives. Plain (st5_attn_decode_fwd): batch row b. Lineage (st5_attn_lineage_fwd):
// batch row rows[b * rows_ld + j] when a table is given, else b / div.
struct KvMap {
  const int32_t* rows;
  int64_t rows_ld;
  int div;
};

// direct != 0: the buffer holds at most DCH keys, so there is one split and this CTA writes the final output (and
// probabilities) itself -- bit-identical to what the combine kernel makes of a single split.
template <typename T, bool MAP>
__device__ __forceinline__ void decode_split(const st5_attn_decode_args& a, const KvMap& map, int n_splits, int direct) {
  constexpr int VE = Vec16<T>::N;   // elements per 16-byte load
  constexpr int LPK = DH / VE;      // lanes per key row
  constexpr int KPI = DT / LPK;     // keys per CTA iteration
  __shared__ float q[DH];
  __shared__ float sc[DCH];
  __shared__ float red[DT / 32];
  __shared__ float part[DT / 32][DH];
  const int s = blockIdx.x, h = blockIdx.y, b = blockIdx.z, tid = threadIdx.x;
  const int j0 = s * DCH;
  const int j1 = min(j0 + DCH, a.Tk);
  if (tid < DH) q[tid] = ldf((const T*)a.q + (int64_t)b * a.q_bs + h * DH + tid);
  __syncthreads();
  const int lane = tid & 31, sub = lane % LPK, slot = tid / LPK;
  float qr[VE];
#pragma unroll
  for (int e = 0; e < VE; ++e) qr[e] = q[sub * VE + e];
  const uint8_t* kp = a.key_pad != nullptr ? a.key_pad + (int64_t)b * a.Tk : nullptr;
  const int32_t* rt = MAP && map.rows != nullptr ? map.rows + (int64_t)b * map.rows_ld : nullptr;
  const int64_t kvb = MAP ? (int64_t)(b / map.div) : (int64_t)b;
  const T* kb = (const T*)a.k + h * DH + sub * VE;
#pragma unroll
  for (int it = 0; it < DCH / KPI; ++it) {
    const int j = j0 + it * KPI + slot;
    const bool valid = j < j1 && (kp == nullptr || kp[j] == 0);
    float d = 0.f;
    if (valid) {
      float kr[VE];
      Vec16<T>::load(kb + (MAP && rt != nullptr ? (int64_t)rt[j] : kvb) * a.k_bs + (int64_t)j * a.k_ld, kr);
#pragma unroll
      for (int e = 0; e < VE; ++e) d += qr[e] * kr[e];
    }
#pragma unroll
    for (int o = LPK / 2; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
    if (sub == 0) sc[j - j0] = valid ? d * a.scale : -INFINITY;
  }
  __syncthreads();
  const float sraw = tid < DCH ? sc[tid] : -INFINITY;
  const float m = cta_reduce(sraw, red, true);
  const float ex = sraw == -INFINITY ? 0.f : expf(sraw - m);  // (a split with every key masked: m = -inf, all zero)
  const float l = cta_reduce(ex, red, false);
  if (tid < DCH) sc[tid] = ex;
  const int64_t bh = (int64_t)b * a.H + h;
  if (!direct && a.probs != nullptr && tid < DCH && j0 + tid < a.Tk) a.ws[(int64_t)n_splits * DPART * a.B * a.H + bh * a.Tk + j0 + tid] = sraw;
  __syncthreads();
  // out_c = sum_j e_j v_jc: lane `sub` owns channels sub*VE .. +VE, slots stride over the split's keys
  const T* vb = (const T*)a.v + h * DH + sub * VE;
  float acc[VE];
#pragma unroll
  for (int e = 0; e < VE; ++e) acc[e] = 0.f;
#pragma unroll
  for (int it = 0; it < DCH / KPI; ++it) {
    const int jj = it * KPI + slot;
    const float p = sc[jj];
    if (j0 + jj < j1 && p != 0.f) {
      float vr[VE];
      const int j = j0 + jj;
      Vec16<T>::load(vb + (MAP && rt != nullptr ? (int64_t)rt[j] : kvb) * a.v_bs + (int64_t)j * a.v_ld, vr);
#pragma unroll
      for (int e = 0; e < VE; ++e) acc[e] += p * vr[e];
    }
  }
#pragma unroll
  for (int e = 0; e < VE; ++e) {
#pragma unroll
    for (int o = LPK; o < 32; o <<= 1) acc[e] += __shfl_xor_sync(0xffffffffu, acc[e], o);
  }
  if (lane < LPK) {
#pragma unroll
    for (int e = 0; e < VE; ++e) part[tid >> 5][sub * VE + e] = acc[e];
  }
  __syncthreads();
  if (tid < DH) {
    float r = part[0][tid];
#pragma unroll
    for (int w = 1; w < DT / 32; ++w) r += part[w][tid];
    if (direct) {
      stf((T*)a.out + (int64_t)b * a.o_bs + h * DH + tid, r * (l > 0.f ? 1.f / l : 0.f));
    } else {
      float* pr = a.ws + (bh * n_splits + s) * DPART;
      pr[2 + tid] = r;
      if (tid == 0) { pr[0] = m; pr[1] = l; }
    }
  }
  if (direct) {
    float* pr = decode_probs(a, b, h);
    if (pr != nullptr) {
      const float inv = l > 0.f ? 1.f / l : 0.f;
      for (int j = tid; j < a.Tk; j += DT) pr[j] = sc[j] * inv;
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(DT) attn_decode_split(const st5_attn_decode_args a, int n_splits, int direct) {
  decode_split<T, false>(a, KvMap{nullptr, 0, 1}, n_splits, direct);
}

template <typename T>
__global__ void __launch_bounds__(DT) attn_lineage_split(const st5_attn_lineage_args a, int n_splits, int direct) {
  decode_split<T, true>(a.base, KvMap{a.kv_rows, a.kv_rows_ld, a.kv_div}, n_splits, direct);
}

__global__ void __launch_bounds__(DT) attn_decode_combine(const st5_attn_decode_args a, int n_splits, int dtype) {
  const int h = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  const int ns = n_splits;
  const int64_t bh = (int64_t)b * a.H + h;
  const float* pr = a.ws + bh * n_splits * DPART;
  float M = -INFINITY;
  for (int s = 0; s < ns; ++s) M = fmaxf(M, pr[s * DPART]);
  float L = 0.f;
  for (int s = 0; s < ns; ++s) {
    const float ms = pr[s * DPART];
    L += ms == -INFINITY ? 0.f : pr[s * DPART + 1] * expf(ms - M);
  }
  const float inv = L > 0.f ? 1.f / L : 0.f;
  if (tid < DH) {
    float r = 0.f;
    for (int s = 0; s < ns; ++s) {
      const float ms = pr[s * DPART];
      r += pr[s * DPART + 2 + tid] * (ms == -INFINITY ? 0.f : expf(ms - M));
    }
    r *= inv;
    if (dtype == ST5_F32) stf((float*)a.out + (int64_t)b * a.o_bs + h * DH + tid, r);
    else stf((__nv_bfloat16*)a.out + (int64_t)b * a.o_bs + h * DH + tid, r);
  }
  float* po = decode_probs(a, b, h);
  if (po != nullptr) {
    const float* sr = a.ws + (int64_t)n_splits * DPART * a.B * a.H + bh * a.Tk;
    for (int j = tid; j < a.Tk; j += DT) po[j] = sr[j] == -INFINITY ? 0.f : expf(sr[j] - M) * inv;
  }
}

int64_t attn_decode_ws_floats(int B, int H, int Tk, int with_probs) {
  if (Tk <= DCH) return 0;
  const int64_t ns = (Tk + DCH - 1) / DCH;
  return (int64_t)B * H * (ns * DPART + (with_probs ? Tk : 0));
}

static int decode_check(const st5_attn_decode_args& a) {
  if (a.B <= 0 || a.H <= 0 || a.Tk <= 0) return -2;
  const int esz = a.dtype == ST5_F32 ? 4 : 2;
  if (((a.k_ld * esz) & 15) || ((a.v_ld * esz) & 15) || ((a.k_bs * esz) & 15) || ((a.v_bs * esz) & 15)) return -6;
  if ((reinterpret_cast<uintptr_t>(a.k) & 15) || (reinterpret_cast<uintptr_t>(a.v) & 15)) return -6;
  if (a.Tk > DCH && a.ws == nullptr) return -5;
  return 0;
}

int attn_decode_launch(const st5_attn_decode_args& a, cudaStream_t st) {
  const int rc = decode_check(a);
  if (rc != 0) return rc;
  const int ns = (a.Tk + DCH - 1) / DCH;
  const int direct = ns == 1;
  const dim3 grid(ns, a.H, a.B);
  if (a.dtype == ST5_F32) attn_decode_split<float><<<grid, DT, 0, st>>>(a, ns, direct);
  else attn_decode_split<__nv_bfloat16><<<grid, DT, 0, st>>>(a, ns, direct);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess || direct) return (int)e;
  attn_decode_combine<<<dim3(a.H, a.B), DT, 0, st>>>(a, ns, a.dtype);
  return (int)cudaGetLastError();
}

int attn_lineage_launch(const st5_attn_lineage_args& a, cudaStream_t st) {
  const int rc = decode_check(a.base);
  if (rc != 0) return rc;
  if (a.kv_div < 1 || (a.kv_rows != nullptr && (a.kv_div != 1 || a.kv_rows_ld < a.base.Tk))) return -2;
  const int ns = (a.base.Tk + DCH - 1) / DCH;
  const int direct = ns == 1;
  const dim3 grid(ns, a.base.H, a.base.B);
  if (a.base.dtype == ST5_F32) attn_lineage_split<float><<<grid, DT, 0, st>>>(a, ns, direct);
  else attn_lineage_split<__nv_bfloat16><<<grid, DT, 0, st>>>(a, ns, direct);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess || direct) return (int)e;
  attn_decode_combine<<<dim3(a.base.H, a.base.B), DT, 0, st>>>(a.base, ns, a.base.dtype);
  return (int)cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------- head dim 80
// Heads of 80 channels (fairseq's transformer_lm_t5: 1280 channels / 16 heads), same split-KV contract as above: splits
// of DCH keys over grid (splits, H, B), key j in split j / DCH at a fixed position, masked keys never loaded and adding
// an exact zero, the same combine, the same direct path for Tk <= DCH.
//
// Layout. 80 bf16 values are ten 16-byte vectors (80 fp32 twenty), so the 64-wide layout above -- LPK = DH / VE lanes
// per key row, a power of two, partial sums reduced with __shfl_xor_sync -- does not divide the row: it would leave six
// of sixteen lanes idle or need 8-byte loads. Here TEN threads own a key row, thread `sub` the eight consecutive
// channels sub*8 .. sub*8+7 (one 16-byte bf16 vector or two fp32 ones), so every load stays 16 bytes wide and the ten
// threads of a row read its 160 (320) contiguous bytes. A 128-thread CTA holds twelve such rows (threads 120..127 sit
// out the key loops) and covers a split in six passes, all of whose loads are issued before the first use. Ten is not
// a power of two, so partial dot products and partial value accumulators are combined through shared memory instead of
// shuffles, each in a fixed order (sub 0..9, slot 0..11): the result depends only on the key's data and position.
constexpr int D80 = 80;
constexpr int D80_SUB = 10;                                  // threads per key row
constexpr int D80_SLOTS = DT / D80_SUB;                      // key rows per pass (12)
constexpr int D80_IT = (DCH + D80_SLOTS - 1) / D80_SLOTS;    // passes per split (6)
constexpr int D80_PART = D80 + 2;                            // partial record: max, sum, accumulator[80]

template <typename T, bool MAP>
__device__ __forceinline__ void decode80_split(const st5_attn_decode_args& a, const KvMap& map, int n_splits, int direct) {
  __shared__ float q[D80];
  __shared__ float ps[DCH][D80_SUB + 1];
  __shared__ float sc[DCH];
  __shared__ float red[DT / 32];
  __shared__ float pacc[D80_SLOTS][D80];
  const int s = blockIdx.x, h = blockIdx.y, b = blockIdx.z, tid = threadIdx.x;
  const int j0 = s * DCH;
  const int j1 = min(j0 + DCH, a.Tk);
  if (tid < D80) q[tid] = ldf((const T*)a.q + (int64_t)b * a.q_bs + h * D80 + tid);
  __syncthreads();
  const int slot = tid / D80_SUB, sub = tid - slot * D80_SUB;
  const bool active = slot < D80_SLOTS;
  float qr[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) qr[e] = active ? q[sub * 8 + e] : 0.f;
  const uint8_t* kp = a.key_pad != nullptr ? a.key_pad + (int64_t)b * a.Tk : nullptr;
  const int32_t* rt = MAP && map.rows != nullptr ? map.rows + (int64_t)b * map.rows_ld : nullptr;
  const int64_t kvb = MAP ? (int64_t)(b / map.div) : (int64_t)b;
  const T* kb = (const T*)a.k + h * D80 + sub * 8;
  float kr[D80_IT][8];
  bool ok[D80_IT];
#pragma unroll
  for (int it = 0; it < D80_IT; ++it) {
    const int jj = it * D80_SLOTS + slot;
    const int j = j0 + jj;
    ok[it] = active && jj < DCH && j < j1 && (kp == nullptr || kp[j] == 0);
    if (ok[it]) load8<T>(kb + (MAP && rt != nullptr ? (int64_t)rt[j] : kvb) * a.k_bs + (int64_t)j * a.k_ld, kr[it]);
  }
#pragma unroll
  for (int it = 0; it < D80_IT; ++it) {
    const int jj = it * D80_SLOTS + slot;
    float d = 0.f;
    if (ok[it]) {
#pragma unroll
      for (int e = 0; e < 8; ++e) d += qr[e] * kr[it][e];
    }
    if (active && jj < DCH) ps[jj][sub] = d;
  }
  __syncthreads();
  float sraw = -INFINITY;
  if (tid < DCH && j0 + tid < j1 && (kp == nullptr || kp[j0 + tid] == 0)) {
    float d = ps[tid][0];
#pragma unroll
    for (int u = 1; u < D80_SUB; ++u) d += ps[tid][u];
    sraw = d * a.scale;
  }
  const float m = cta_reduce(sraw, red, true);
  const float ex = sraw == -INFINITY ? 0.f : expf(sraw - m);  // (a split with every key masked: m = -inf, all zero)
  const float l = cta_reduce(ex, red, false);
  if (tid < DCH) sc[tid] = ex;
  const int64_t bh = (int64_t)b * a.H + h;
  if (!direct && a.probs != nullptr && tid < DCH && j0 + tid < a.Tk) a.ws[(int64_t)n_splits * D80_PART * a.B * a.H + bh * a.Tk + j0 + tid] = sraw;
  __syncthreads();
  // out_c = sum_j e_j v_jc: thread `sub` of a slot accumulates channels sub*8 .. +8 over the slot's keys
  const T* vb = (const T*)a.v + h * D80 + sub * 8;
  float vr[D80_IT][8];
  float pj[D80_IT];
#pragma unroll
  for (int it = 0; it < D80_IT; ++it) {
    const int jj = it * D80_SLOTS + slot;
    const int j = j0 + jj;
    pj[it] = active && jj < DCH && j < j1 ? sc[jj] : 0.f;
    if (pj[it] != 0.f) load8<T>(vb + (MAP && rt != nullptr ? (int64_t)rt[j] : kvb) * a.v_bs + (int64_t)j * a.v_ld, vr[it]);
  }
  float acc[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) acc[e] = 0.f;
#pragma unroll
  for (int it = 0; it < D80_IT; ++it) {
    if (pj[it] != 0.f) {
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[e] += pj[it] * vr[it][e];
    }
  }
  if (active) {
#pragma unroll
    for (int e = 0; e < 8; ++e) pacc[slot][sub * 8 + e] = acc[e];
  }
  __syncthreads();
  if (tid < D80) {
    float r = pacc[0][tid];
#pragma unroll
    for (int w = 1; w < D80_SLOTS; ++w) r += pacc[w][tid];
    if (direct) {
      stf((T*)a.out + (int64_t)b * a.o_bs + h * D80 + tid, r * (l > 0.f ? 1.f / l : 0.f));
    } else {
      float* pr = a.ws + (bh * n_splits + s) * D80_PART;
      pr[2 + tid] = r;
      if (tid == 0) { pr[0] = m; pr[1] = l; }
    }
  }
  if (direct) {
    float* pr = decode_probs(a, b, h);
    if (pr != nullptr) {
      const float inv = l > 0.f ? 1.f / l : 0.f;
      for (int j = tid; j < a.Tk; j += DT) pr[j] = sc[j] * inv;
    }
  }
}

// The kernels' arguments travel in a struct of their own (the symbols then name neither st5_attn_decode_args nor
// st5_attn_lineage_args, which identify the 64-wide kernels); MAP: the lineage form.
struct Decode80Launch {
  st5_attn_decode_args a;
  KvMap map;
};

template <typename T, bool MAP>
__global__ void __launch_bounds__(DT) attn_decode80_split(const Decode80Launch p, int n_splits, int direct) {
  decode80_split<T, MAP>(p.a, p.map, n_splits, direct);
}

// attn_decode_combine over 80-wide partial records
__global__ void __launch_bounds__(DT) attn_decode80_combine(const Decode80Launch p, int n_splits, int dtype) {
  const st5_attn_decode_args& a = p.a;
  const int h = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  const int64_t bh = (int64_t)b * a.H + h;
  const float* pr = a.ws + bh * n_splits * D80_PART;
  float M = -INFINITY;
  for (int s = 0; s < n_splits; ++s) M = fmaxf(M, pr[s * D80_PART]);
  float L = 0.f;
  for (int s = 0; s < n_splits; ++s) {
    const float ms = pr[s * D80_PART];
    L += ms == -INFINITY ? 0.f : pr[s * D80_PART + 1] * expf(ms - M);
  }
  const float inv = L > 0.f ? 1.f / L : 0.f;
  if (tid < D80) {
    float r = 0.f;
    for (int s = 0; s < n_splits; ++s) {
      const float ms = pr[s * D80_PART];
      r += pr[s * D80_PART + 2 + tid] * (ms == -INFINITY ? 0.f : expf(ms - M));
    }
    r *= inv;
    if (dtype == ST5_F32) stf((float*)a.out + (int64_t)b * a.o_bs + h * D80 + tid, r);
    else stf((__nv_bfloat16*)a.out + (int64_t)b * a.o_bs + h * D80 + tid, r);
  }
  float* po = decode_probs(a, b, h);
  if (po != nullptr) {
    const float* sr = a.ws + (int64_t)n_splits * D80_PART * a.B * a.H + bh * a.Tk;
    for (int j = tid; j < a.Tk; j += DT) po[j] = sr[j] == -INFINITY ? 0.f : expf(sr[j] - M) * inv;
  }
}

template <bool MAP>
static int decode80_launch(const Decode80Launch& p, cudaStream_t st) {
  const st5_attn_decode_args& a = p.a;
  const int ns = (a.Tk + DCH - 1) / DCH;
  const int direct = ns == 1;
  const dim3 grid(ns, a.H, a.B);
  if (a.dtype == ST5_F32) attn_decode80_split<float, MAP><<<grid, DT, 0, st>>>(p, ns, direct);
  else attn_decode80_split<__nv_bfloat16, MAP><<<grid, DT, 0, st>>>(p, ns, direct);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess || direct) return (int)e;
  attn_decode80_combine<<<dim3(a.H, a.B), DT, 0, st>>>(p, ns, a.dtype);
  return (int)cudaGetLastError();
}

int64_t attn_decode_hd_ws_floats(int B, int H, int Tk, int with_probs, int head_dim) {
  if (head_dim == DH) return attn_decode_ws_floats(B, H, Tk, with_probs);
  if (head_dim != D80) return -2;
  if (Tk <= DCH) return 0;
  const int64_t ns = (Tk + DCH - 1) / DCH;
  return (int64_t)B * H * (ns * D80_PART + (with_probs ? Tk : 0));
}

int attn_decode_hd_launch(const st5_attn_decode_args& a, int head_dim, cudaStream_t st) {
  if (head_dim == DH) return attn_decode_launch(a, st);
  if (head_dim != D80) return -2;
  const int rc = decode_check(a);
  if (rc != 0) return rc;
  return decode80_launch<false>(Decode80Launch{a, KvMap{nullptr, 0, 1}}, st);
}

int attn_lineage_hd_launch(const st5_attn_lineage_args& a, int head_dim, cudaStream_t st) {
  if (head_dim == DH) return attn_lineage_launch(a, st);
  if (head_dim != D80) return -2;
  const int rc = decode_check(a.base);
  if (rc != 0) return rc;
  if (a.kv_div < 1 || (a.kv_rows != nullptr && (a.kv_div != 1 || a.kv_rows_ld < a.base.Tk))) return -2;
  return decode80_launch<true>(Decode80Launch{a.base, KvMap{a.kv_rows, a.kv_rows_ld, a.kv_div}}, st);
}

}  // namespace st5
