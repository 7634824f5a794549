// Thin inline-PTX wrappers for sm_90a: mbarrier, TMA (cp.async.bulk.tensor), wgmma (warpgroup MMA).
// Everything here is device-side and header-only. The bit layout of the wgmma shared-memory descriptor follows the
// PTX ISA "matrix descriptor" table for wgmma (the encoding CUTLASS's cute/arch/mma_sm90_desc.hpp documents).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>

namespace st5 {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n"
      ".reg .b32 rx;\n"
      ".reg .pred px;\n"
      "elect.sync rx|px, 0xffffffff;\n"
      "selp.u32 %0, 1, 0, px;\n"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug must surface as a trap (launch failure), never as a hung GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 4000000000LL) {  // ~2 s at 2 GHz
      printf("st5: mbarrier timeout block(%d,%d,%d) thread %d parity %u\n", blockIdx.x, blockIdx.y, blockIdx.z,
             threadIdx.x, parity);
      __trap();
    }
  }
}

// The same bound without the printf: a call inside a wgmma pipeline would make ptxas serialise the MMAs.
__device__ __forceinline__ void mbar_wait_quiet(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  long long t0 = clock64();
  while (!mbar_try_wait(bar, parity))
    if (clock64() - t0 > 4000000000LL) __trap();
}
// Register reallocation between the warpgroups of a warp-specialised block (the producer gives, the MMA warps take).
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const void* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const void* map, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], "
      "[%2];"
      :
      : "r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// TMA store: shared -> global tile (bulk async group); rows / columns outside the tensor are clipped by the hardware.
__device__ __forceinline__ void tma_store_4d(const void* map, const void* src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
               :
               : "l"(map), "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
// TMA reduce: global tile += shared tile, element type from the tensor map (fp32 here); the read-modify-write happens at
// the L2, so several CTAs may target the same tile (split-K partial products) and nobody has to read C first.
__device__ __forceinline__ void tma_reduce_add_4d(const void* map, const void* src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.reduce.async.bulk.tensor.4d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
               :
               : "l"(map), "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// wait until the shared-memory source of every committed bulk store of this thread has been read
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }

// ---------------------------------------------------------------- wgmma (sm_90a warpgroup MMA)
// D[64 x N] (+)= A[64 x 16] * B[16 x N], bf16 inputs from shared memory (descriptors), fp32 accumulators in the
// registers of the issuing warpgroup. TA / TB = 1 when that operand is MN-major (transposed) in shared memory.
// Accumulator fragment of thread t (warp w = t / 32 of the warpgroup, lane l): d[i] sits at
//   row 16 w + l / 4 + 8 ((i >> 1) & 1), column 8 (i >> 2) + 2 (l % 4) + (i & 1).
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// Keep the compiler from moving accumulator reads / writes across an asynchronous wgmma.
template <int NR>
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[NR]) {
#pragma unroll
  for (int i = 0; i < NR; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n64(float (&d)[32], uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, p, 1, 1, %35, %36;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(desc_a), "l"(desc_b), "r"(scale_d), "n"(TA), "n"(TB));
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n128(float (&d)[64], uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, %67, %68;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(desc_a), "l"(desc_b), "r"(scale_d), "n"(TA), "n"(TB));
}


// Shared-memory matrix descriptor (64-bit, sm_90 layout). Fields in 16-byte units: start address [0,14), leading
// byte offset [16,30), stride byte offset [32,46); layout type at [62,64) (1 = 128B swizzle). K-major 128B-swizzled
// tiles: SBO = 1024 (one 8-row swizzle atom), LBO unused. MN-major: LBO = stride between 64-element MN chunks,
// SBO = 1024 (eight k rows of 128 B).
__host__ __device__ __forceinline__ uint64_t wgmma_smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

// ---------------------------------------------------------------- counter-based RNG (Philox4x32-7)
// Seven rounds: the smallest round count of Philox4x32 that passes BigCrush (Salmon et al., SC'11, table 2); dropout
// needs decorrelated keep decisions, not a cryptographic margin, and the generator sits inside GEMM / attention
// epilogues where every round is ~8 issue slots per 8 outputs.
constexpr int PHILOX_ROUNDS = 7;
struct Philox4 {
  uint32_t x, y, z, w;
};
__host__ __device__ __forceinline__ uint32_t mulhi32(uint32_t a, uint32_t b) {
  return (uint32_t)(((uint64_t)a * (uint64_t)b) >> 32);
}
__host__ __device__ __forceinline__ Philox4 philox4x32(uint64_t seed, uint64_t offset, uint64_t idx) {
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
  uint32_t c0 = (uint32_t)idx, c1 = (uint32_t)(idx >> 32), c2 = (uint32_t)offset, c3 = (uint32_t)(offset >> 32);
#pragma unroll
  for (int i = 0; i < PHILOX_ROUNDS; ++i) {
    uint32_t h0 = mulhi32(0xD2511F53u, c0), l0 = 0xD2511F53u * c0;
    uint32_t h1 = mulhi32(0xCD9E8D57u, c2), l1 = 0xCD9E8D57u * c2;
    uint32_t n0 = h1 ^ c1 ^ k0, n1 = l1, n2 = h0 ^ c3 ^ k1, n3 = l0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return Philox4{c0, c1, c2, c3};
}
// Seeds may be passed by value or -- so that a captured CUDA graph draws fresh masks on every replay -- as the device
// address of a uint64 seed, flagged by bit 63 of `offset`.
constexpr uint64_t SEED_PTR_FLAG = 1ull << 63;
__device__ __forceinline__ void resolve_seed(uint64_t& seed, uint64_t& offset) {
  if (offset & SEED_PTR_FLAG) {
    seed = *reinterpret_cast<const uint64_t*>(seed);
    offset &= ~SEED_PTR_FLAG;
  }
}
// Dropout keep-mask for element `i` of a tensor. One Philox4x32 call yields eight 16-bit lanes, i.e. the decisions of 8
// consecutive elements: keep iff lane >= thr16, thr16 = min(p * 65536, 65535) (p is quantised to 1/65536).
__host__ __device__ __forceinline__ uint32_t philox_lane16(const Philox4& r, int lane) {
  const uint32_t w = (lane >> 1) == 0 ? r.x : (lane >> 1) == 1 ? r.y : (lane >> 1) == 2 ? r.z : r.w;
  return (lane & 1) ? (w >> 16) : (w & 0xFFFFu);
}
__host__ __device__ __forceinline__ bool dropout_keep(uint64_t seed, uint64_t offset, uint64_t i, uint32_t thr) {
  const Philox4 r = philox4x32(seed, offset, i >> 3);
  return philox_lane16(r, (int)(i & 7)) >= thr;
}
// Attention probabilities are indexed with a row pitch rounded up to 32 keys, so that every 32-column chunk of a row
// starts on a Philox group boundary (4 calls per chunk, no ragged head).
__host__ __device__ __forceinline__ uint64_t attn_drop_pitch(int Tk) { return (uint64_t)((Tk + 31) & ~31); }
// keep-bits of 32 consecutive elements e0 .. e0+31 (any alignment): at most 5 Philox calls instead of 32
__device__ __forceinline__ uint32_t dropout_keep_mask32(uint64_t seed, uint64_t offset, uint64_t e0, uint32_t thr) {
  uint32_t mask = 0;
  const int lead = (int)((8 - (e0 & 7)) & 7);  // elements before the first 8-aligned group boundary
  if (lead != 0) {
    const Philox4 r = philox4x32(seed, offset, e0 >> 3);
    for (int t = 0; t < lead; ++t)
      if (philox_lane16(r, (int)((e0 + t) & 7)) >= thr) mask |= 1u << t;
  }
#pragma unroll
  for (int g = 0; g < 4; ++g) {
    const int t0 = lead + 8 * g;
    if (t0 < 32) {
      const Philox4 r = philox4x32(seed, offset, (e0 + t0) >> 3);
      const uint32_t w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
      for (int l = 0; l < 8; ++l) {
        const int t = t0 + l;
        const uint32_t v = (l & 1) ? (w[l >> 1] >> 16) : (w[l >> 1] & 0xFFFFu);
        if (t < 32 && v >= thr) mask |= 1u << t;
      }
    }
  }
  return mask;
}
// eight consecutive elements starting at e0 (a multiple of 8): v[t] = keep ? v[t] * scale : 0
__device__ __forceinline__ void dropout8_apply(float* v, uint64_t e0, uint32_t thr, float dscale, uint64_t seed,
                                               uint64_t offset) {
  const Philox4 r = philox4x32(seed, offset, e0 >> 3);
  v[0] = (r.x & 0xFFFFu) >= thr ? v[0] * dscale : 0.f; v[1] = (r.x >> 16) >= thr ? v[1] * dscale : 0.f;
  v[2] = (r.y & 0xFFFFu) >= thr ? v[2] * dscale : 0.f; v[3] = (r.y >> 16) >= thr ? v[3] * dscale : 0.f;
  v[4] = (r.z & 0xFFFFu) >= thr ? v[4] * dscale : 0.f; v[5] = (r.z >> 16) >= thr ? v[5] * dscale : 0.f;
  v[6] = (r.w & 0xFFFFu) >= thr ? v[6] * dscale : 0.f; v[7] = (r.w >> 16) >= thr ? v[7] * dscale : 0.f;
}

}  // namespace st5
