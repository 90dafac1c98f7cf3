// Condition term of the DreamVideo motion adapters (tools/modules/unet/util.py:499-519).
//
// Adapter.forward adds lambda * condition_linear(c) to x before down_linear.  Both are linear, so
//   down(x + lambda (Wc c + bc)) = down(x) + lambda (Wd Wc c + Wd bc)
// and the pack stores the products Wd Wc / Wd bc of every conditioned adapter of the model stacked into one matrix.  One
// launch per forward then yields the fp32 row bias of all of them (vgen_linear_gelu_rowbias adds it before the GELU).
// The problem is a few rows (one per video, or per frame) against a tall matrix: one warp per output column streams its
// weight row once per block of kRows rows with 16-byte loads; the condition rows are re-read from L1.
#include "common.h"

namespace vg {

static constexpr int kRows = 4;

__global__ void __launch_bounds__(256) adapter_condition_kernel(const __half* __restrict__ c, long ldc, int rows, int k,
                                                                const __half* __restrict__ w, const float* __restrict__ v,
                                                                int n, const float* __restrict__ lam, float lam_scalar,
                                                                int groups_per_lam, float* __restrict__ g, long ldg) {
  const int j = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (j >= n) return;
  const __half* wr = w + (long)j * k;
  for (int r0 = 0; r0 < rows; r0 += kRows) {
    float acc[kRows] = {0.f, 0.f, 0.f, 0.f};
    for (int kk = lane * 8; kk < k; kk += 32 * 8) {
      const uint4 wv = __ldg(reinterpret_cast<const uint4*>(wr + kk));
      const __half2* w2 = reinterpret_cast<const __half2*>(&wv);
#pragma unroll
      for (int i = 0; i < kRows; ++i) {
        if (r0 + i < rows) {
          const uint4 cv = __ldg(reinterpret_cast<const uint4*>(c + (long)(r0 + i) * ldc + kk));
          const __half2* c2 = reinterpret_cast<const __half2*>(&cv);
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const float2 a = __half22float2(c2[q]), b = __half22float2(w2[q]);
            acc[i] = fmaf(a.x, b.x, fmaf(a.y, b.y, acc[i]));
          }
        }
      }
    }
#pragma unroll
    for (int i = 0; i < kRows; ++i) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], o);
    }
    if (lane < kRows && r0 + lane < rows) {
      const int r = r0 + lane;
      float s = acc[0];
#pragma unroll
      for (int i = 1; i < kRows; ++i)
        if (lane == i) s = acc[i];
      const float l = lam ? lam[r / groups_per_lam] : lam_scalar;
      g[(long)r * ldg + j] = l * (s + v[j]);
    }
  }
}

}  // namespace vg

using namespace vg;

extern "C" int vgen_adapter_condition(const void* c, int64_t rows, int64_t k, int64_t ldc, const void* w, const float* v,
                                      int64_t n, const float* lam, float lam_scalar, int64_t groups_per_lam, float* g,
                                      int64_t ldg, void* stream) {
  VG_REQUIRE(c && w && v && g, "vgen_adapter_condition: null pointer");
  VG_REQUIRE(rows >= 0 && rows < (1L << 31) && k > 0 && k % 8 == 0 && ldc >= k && ldc % 8 == 0 && n > 0 &&
                 n < (1L << 31) && ldg >= n && groups_per_lam >= 1,
             "vgen_adapter_condition: bad shape (k and ldc must be multiples of 8)");
  VG_REQUIRE((reinterpret_cast<uintptr_t>(c) & 15) == 0 && (reinterpret_cast<uintptr_t>(w) & 15) == 0,
             "vgen_adapter_condition: c and w must be 16-byte aligned");
  if (rows == 0) return 0;
  const int warps = 8;
  launch_kernel(adapter_condition_kernel, dim3((unsigned)((n + warps - 1) / warps)), dim3(32 * warps), 0,
                reinterpret_cast<cudaStream_t>(stream), reinterpret_cast<const __half*>(c), (long)ldc, (int)rows, (int)k,
                reinterpret_cast<const __half*>(w), v, (int)n, lam, lam_scalar, (int)groups_per_lam, g, (long)ldg);
  VG_LAUNCH_CHECK("adapter_condition_kernel");
  return 0;
}
