// SIMT cross-check implementation of tapgemm (same arguments, same epilogue rounding order as
// tapgemm_sm90.cu).  It exists to bisect tensor-core / TMA descriptor bugs on the GPU
// (VGEN_TAPGEMM_IMPL=simt) and to serve channel counts that are not a multiple of 64.
// One thread per (row, n): slow, obviously-correct.
#include "common.h"
#include "ptx.cuh"
#include "tapgemm.h"

namespace vg {

__device__ __forceinline__ float gelu_erf_s(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f)); }

__global__ void tapgemm_simt_kernel(const __half* __restrict__ A, long st1, long st2, long st3,
                                    const __half* __restrict__ W, const __half* __restrict__ H, long ldh,
                                    const __half* __restrict__ U, int r, TapGemmShape s, TapGemmEpilogue e) {
  const long rows = (long)s.d1 * s.d2 * s.d3;
  const int out_n = e.geglu ? s.n / 2 : s.n;
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * out_n) return;
  const int n = (int)(idx % out_n);
  const long row = idx / out_n;
  const int i1 = (int)(row % s.d1);
  const int i2 = (int)((row / s.d1) % s.d2);
  const int i3 = (int)(row / ((long)s.d1 * s.d2));
  const long ktot = (long)s.num_taps * s.c;

  auto dot = [&](int wrow) {
    float acc = 0.f;
    for (int t = 0; t < s.num_taps; ++t) {
      const int j1 = i1 + s.tap1[t], j2 = i2 + s.tap2[t], j3 = i3 + s.tap3[t];
      if (j1 < 0 || j1 >= s.d1 || j2 < 0 || j2 >= s.d2 || j3 < 0 || j3 >= s.d3) continue;
      const __half* ap = A + j1 * st1 + j2 * st2 + j3 * st3;
      const __half* wp = W + (long)wrow * ktot + (long)t * s.c;
      for (int c = 0; c < s.c; ++c) acc += __half2float(ap[c]) * __half2float(wp[c]);
    }
    // K tail (linear only): the same accumulator continues over h[row] . u[wrow]
    for (int j = 0; j < r; ++j) acc += __half2float(H[row * ldh + j]) * __half2float(U[(long)wrow * r + j]);
    return acc;
  };

  // folded LayerNorm (linear only: row = i1): acc * rstd + (-mean rstd) * col_sum
  const float ln_scale = e.row_stats ? e.row_stats[row].x * e.alpha : e.alpha;
  const float ln_shift = e.row_stats ? e.row_stats[row].y * e.alpha : 0.f;
  float a;
  if (!e.geglu) {
    a = dot(n) * ln_scale;
    if (e.bias) a += e.bias[n];
    if (e.row_stats) a = fmaf(ln_shift, e.col_sum[n], a);
    if (e.row_bias) a += e.row_bias[(row / e.rows_per_group) * e.ld_row_bias + n];
    if (e.gelu) a = gelu_erf_s(a);
    if (e.relu) a = fmaxf(a, 0.f);
    if (e.group_bias) a = __half2float(__float2half_rn(a)) + __half2float(e.group_bias[(long)(i3 / e.group_bias_div) * e.ld_group_bias + n]);
    if (e.residual) a = __half2float(__float2half_rn(a)) + __half2float(e.residual[row * e.ldr + n]);
  } else {
    const int hb = s.bn / 2;
    const int blk = n / hb, j = n % hb;
    const int wv = blk * s.bn + j, wg = wv + hb;
    float v = dot(wv) * ln_scale, g = dot(wg) * ln_scale;
    if (e.bias) {
      v += e.bias[wv];
      g += e.bias[wg];
    }
    if (e.row_stats) {
      v = fmaf(ln_shift, e.col_sum[wv], v);
      g = fmaf(ln_shift, e.col_sum[wg], g);
    }
    const float v16 = __half2float(__float2half_rn(v));
    const float g16 = __half2float(__float2half_rn(g));
    a = v16 * __half2float(__float2half_rn(gelu_erf_s(g16)));
  }
  const long ooff = e.out_s2 ? (long)i1 * e.ldo + (long)i2 * e.out_s2 + (long)i3 * e.out_s3 : row * e.ldo;
  e.out[ooff + n] = __float2half_rn(a);
}

int tapgemm_simt_launch(const TapGemmArgs& a, cudaStream_t stream) {
  const TapGemmShape& s = a.shape;
  const long rows = (long)s.d1 * s.d2 * s.d3;
  const long total = rows * (a.epi.geglu ? s.n / 2 : s.n);
  if (total == 0) return 0;
  const int threads = 256;
  const long blocks = (total + threads - 1) / threads;
  VG_REQUIRE(blocks < (1L << 31), "tapgemm_simt: problem too large");
  VG_REQUIRE(!a.r || (s.num_taps == 1 && s.d2 == 1 && s.d3 == 1 && !a.epi.geglu),
             "tapgemm_simt: the K tail goes with a plain linear");
  launch_kernel(tapgemm_simt_kernel, dim3((unsigned)blocks), dim3(threads), 0, stream, a.a, a.a_stride1, a.a_stride2, a.a_stride3, a.w,
                a.h, a.ldh, a.u, a.r, s, a.epi);
  VG_LAUNCH_CHECK("tapgemm_simt_kernel");
  return 0;
}

}  // namespace vg
