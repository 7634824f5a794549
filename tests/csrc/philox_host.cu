// Host-side statistics of the counter-based dropout generator (speecht5_b200/csrc/ptx.cuh: Philox4x32-7, 16-bit
// lanes). Built with nvcc and run on the CPU by tests/test_philox_cpu.py -- the functions under test are the very
// __host__ __device__ functions the kernels call.
#include <cmath>
#include <cstdio>
#include <cstdint>
#include <vector>

#include "../../speecht5_b200/csrc/ptx.cuh"

using namespace st5;

int main() {
  const uint64_t seed = 0x1234567ull, offset = 3;
  // 1. keep rate at p = 0.1 / 0.5 over 2^21 consecutive elements
  for (float p : {0.1f, 0.5f}) {
    const uint32_t thr = (uint32_t)(p * 65536.f);
    uint64_t keep = 0;
    const uint64_t n = 1ull << 21;
    for (uint64_t i = 0; i < n; ++i) keep += dropout_keep(seed, offset, i, thr) ? 1 : 0;
    std::printf("keep_rate p=%.2f %.6f\n", p, (double)keep / (double)n);
  }
  // 2. chi-square of the top byte of every 16-bit lane (256 bins) over 2^18 calls
  {
    std::vector<double> bins(256, 0.0);
    const uint64_t calls = 1ull << 18;
    for (uint64_t c = 0; c < calls; ++c) {
      const Philox4 r = philox4x32(seed, offset, c);
      const uint32_t w[4] = {r.x, r.y, r.z, r.w};
      for (int k = 0; k < 4; ++k) {
        bins[(w[k] >> 8) & 0xFF] += 1.0;
        bins[(w[k] >> 24) & 0xFF] += 1.0;
      }
    }
    const double expect = (double)(calls * 8) / 256.0;
    double chi = 0.0;
    for (double b : bins) chi += (b - expect) * (b - expect) / expect;
    std::printf("chi2_256 %.3f\n", chi);  // 255 degrees of freedom: mean 255, sd 22.6
  }
  // 3. serial correlation between the decisions of neighbouring elements and of neighbouring rows (pitch 320)
  {
    const uint32_t thr = (uint32_t)(0.5f * 65536.f);
    const uint64_t n = 1ull << 20;
    double s_adj = 0, s_row = 0;
    for (uint64_t i = 0; i < n; ++i) {
      const int a = dropout_keep(seed, offset, i, thr) ? 1 : -1;
      const int b = dropout_keep(seed, offset, i + 1, thr) ? 1 : -1;
      const int c = dropout_keep(seed, offset, i + 320, thr) ? 1 : -1;
      s_adj += a * b;
      s_row += a * c;
    }
    std::printf("corr_adjacent %.6f\ncorr_row %.6f\n", s_adj / n, s_row / n);
  }
  // 4. different offsets (= different dropout sites) and seeds are decorrelated
  {
    const uint32_t thr = (uint32_t)(0.5f * 65536.f);
    const uint64_t n = 1ull << 20;
    double s_off = 0, s_seed = 0;
    for (uint64_t i = 0; i < n; ++i) {
      const int a = dropout_keep(seed, offset, i, thr) ? 1 : -1;
      s_off += a * (dropout_keep(seed, offset + 1, i, thr) ? 1 : -1);
      s_seed += a * (dropout_keep(seed + 1, offset, i, thr) ? 1 : -1);
    }
    std::printf("corr_offset %.6f\ncorr_seed %.6f\n", s_off / n, s_seed / n);
  }
  // 5. known answers (a change of the generator must be deliberate)
  {
    const Philox4 r = philox4x32(1, 2, 3);
    std::printf("kat %08x %08x %08x %08x\n", r.x, r.y, r.z, r.w);
    std::printf("pitch %llu %llu\n", (unsigned long long)attn_drop_pitch(313), (unsigned long long)attn_drop_pitch(160));
    // wgmma shared-memory descriptors (16-byte units): start address bit 0, leading byte offset bit 16, stride byte
    // offset bit 32, 128B swizzle = layout type 1 at bit 62
    std::printf("desc %016llx %016llx\n", (unsigned long long)wgmma_smem_desc(0x1000, 16, 1024),
                (unsigned long long)wgmma_smem_desc(0x2040, 8192, 1024));
  }
  return 0;
}
