// LoRA down projection with the per-sample strength folded in (UNetSD_LoRA's runtime mode):
//
//   h[row][j] = fp16(strength[row / rows_per_sample][col_set[j]] * col_scale[j] * (x[row] . d[j]))   j < r
//   h[row][j] = 0                                                                                      r <= j < r_pad
//
// d [r][k] stacks the down weights of every LoRA set and every projection that reads x (q, k and v of a fused projection),
// so one launch serves them all; h is the K tail vgen_linear_lora multiplies by the block-diagonal up weights.  The
// padding columns are written as zeros, so the tail adds exact zeros there.
//
// One warp per row: the row stays packed in registers (16-byte vectors), each of the r dot products is a warp reduction,
// lane jj of the warp keeps column j0 + jj and the warp stores 32 columns at once.  d is a few KB and stays in L1.
#include "common.h"

namespace vg {

static constexpr int kDownMaxV = 10;   // 16-byte vectors per lane: k <= 32 * 8 * 10 = 2560

__global__ void __launch_bounds__(256) lora_down_kernel(const __half* __restrict__ x, long rows, int k, long ldx,
                                                        const __half* __restrict__ d, int r, const int* __restrict__ col_set,
                                                        const float* __restrict__ col_scale, const float* __restrict__ strength,
                                                        int nsets, long rows_per_sample, __half* __restrict__ h, long ldh,
                                                        int r_pad) {
  const int lane = threadIdx.x & 31;
  const int k8 = k / 8;
  const long warps_total = (long)gridDim.x * (blockDim.x >> 5);
  for (long row = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < rows; row += warps_total) {
    uint4 xv[kDownMaxV];
#pragma unroll
    for (int v = 0; v < kDownMaxV; ++v) {
      const int c8 = lane + v * 32;
      xv[v] = c8 < k8 ? __ldg(reinterpret_cast<const uint4*>(x + row * ldx + c8 * 8)) : make_uint4(0u, 0u, 0u, 0u);
    }
    const float* srow = strength + (row / rows_per_sample) * nsets;
    for (int j0 = 0; j0 < r_pad; j0 += 32) {
      float mine = 0.f;
      const int jn = r - j0 < 32 ? r - j0 : 32;
      for (int jj = 0; jj < jn; ++jj) {
        const int j = j0 + jj;
        const __half* dr = d + (long)j * k;
        float s = 0.f;
#pragma unroll
        for (int v = 0; v < kDownMaxV; ++v) {
          const int c8 = lane + v * 32;
          if (c8 < k8) {
            const uint4 dv = __ldg(reinterpret_cast<const uint4*>(dr + c8 * 8));
            const __half2* a2 = reinterpret_cast<const __half2*>(&xv[v]);
            const __half2* b2 = reinterpret_cast<const __half2*>(&dv);
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              const float2 fa = __half22float2(a2[q]), fb = __half22float2(b2[q]);
              s = fmaf(fa.x, fb.x, s);
              s = fmaf(fa.y, fb.y, s);
            }
          }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == jj) mine = srow[col_set[j]] * col_scale[j] * s;
      }
      if (j0 + lane < r_pad) h[row * ldh + j0 + lane] = __float2half_rn(mine);
    }
  }
}

}  // namespace vg

using namespace vg;

extern "C" {

int vgen_lora_down(const void* x, int64_t m, int64_t k, int64_t ldx, const void* d, int64_t r, const int32_t* col_set,
                   const float* col_scale, const float* strength, int64_t nsets, int64_t rows_per_sample, void* h,
                   int64_t ldh, int64_t r_pad, void* stream) {
  VG_REQUIRE(x && d && col_set && col_scale && strength && h, "vgen_lora_down: null pointer");
  VG_REQUIRE(m >= 0 && k > 0 && k % 8 == 0 && k <= 32 * 8 * kDownMaxV && ldx >= k && ldx % 8 == 0 && r > 0 && r <= r_pad &&
                 ldh >= r_pad && nsets > 0 && rows_per_sample > 0,
             "vgen_lora_down: bad shape (k a multiple of 8 up to 2560, 0 < r <= r_pad <= ldh)");
  VG_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(d) & 15) == 0,
             "vgen_lora_down: x and d must be 16-byte aligned");
  if (m == 0) return 0;
  const int wpb = 8;
  long blocks = (m + wpb - 1) / wpb;
  const long cap = 16L * sm_count();
  if (blocks > cap) blocks = cap;
  launch_kernel(lora_down_kernel, dim3((unsigned)blocks), dim3(32 * wpb), 0, reinterpret_cast<cudaStream_t>(stream),
                reinterpret_cast<const __half*>(x), (long)m, (int)k, (long)ldx, reinterpret_cast<const __half*>(d), (int)r,
                reinterpret_cast<const int*>(col_set), col_scale, strength, (int)nsets, (long)rows_per_sample,
                reinterpret_cast<__half*>(h), (long)ldh, (int)r_pad);
  VG_LAUNCH_CHECK("lora_down_kernel");
  return 0;
}

}  // extern "C"
