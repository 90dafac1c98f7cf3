// The DPT neck and head of the MiDaS v3 depth annotator (tools/annotator/depth/__init__.py:125-293) that the tap-GEMM
// family cannot express by itself.  All three kernels are HBM-bound, channels-last fp16, 16-byte vectors:
//   * the scatter half of a ConvTranspose2d whose kernel equals its stride (stage 1: 4, stage 2: 2): the GEMM half is
//     vgen_linear against the weight repacked to rows (ky, kx, co); this kernel adds the bias and places every
//     (ky, kx) block of a GEMM row at its output pixel;
//   * bilinear x2 upsampling with align_corners=True (FusionBlock, head.1);
//   * the head's tail, ReLU -> ConvTranspose2d(32, 1, 1) + bias -> ReLU, as one per-pixel dot product (an N = 1 GEMM
//     would fill one column of a tile).
#include "common.h"

namespace vg {

static inline unsigned nblk_dpt(long total, int threads) { return (unsigned)((total + threads - 1) / threads); }

// out[b][y*s+ky][x*s+kx][co] = g[(b*hp+y)*wp+x][(ky*s+kx)*cout+co] + bias[co]; one thread per 8 output channels.
__global__ void dpt_tconv_scatter_kernel(const __half* __restrict__ g, long ldg, const float* __restrict__ bias,
                                         __half* __restrict__ out, long nimg, int hp, int wp, int s, int cout) {
  const int c8 = cout / 8;
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const int wo = wp * s, ho = hp * s;
  if (idx >= nimg * ho * wo * c8) return;
  const int cv = (int)(idx % c8);
  const long pix = idx / c8;
  const int ox = (int)(pix % wo);
  const int oy = (int)((pix / wo) % ho);
  const long b = pix / ((long)wo * ho);
  const int y = oy / s, ky = oy - y * s, x = ox / s, kx = ox - x * s;
  const uint4 u = __ldg(reinterpret_cast<const uint4*>(g + ((b * hp + y) * wp + x) * ldg + (long)(ky * s + kx) * cout + cv * 8));
  const __half2* h2 = reinterpret_cast<const __half2*>(&u);
  const float4 b0 = __ldg(reinterpret_cast<const float4*>(bias + cv * 8));
  const float4 b1 = __ldg(reinterpret_cast<const float4*>(bias + cv * 8 + 4));
  const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
  uint4 r;
  __half2* r2 = reinterpret_cast<__half2*>(&r);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 f = __half22float2(h2[i]);
    r2[i] = __floats2half2_rn(f.x + bb[2 * i], f.y + bb[2 * i + 1]);
  }
  reinterpret_cast<uint4*>(out)[idx] = r;
}

// F.interpolate(scale_factor=2, mode='bilinear', align_corners=True) with PyTorch's arithmetic: the source coordinate
// is dst * ((in - 1) / (out - 1)) in fp32, the lower index its truncation, the weights (1 - l, l) with l the fraction.
__global__ void dpt_upsample_bilinear2x_kernel(const __half* __restrict__ x, __half* __restrict__ y, long nimg, int h, int w,
                                               int c8, float ry, float rx) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const int ho = 2 * h, wo = 2 * w;
  if (idx >= nimg * ho * wo * c8) return;
  const int cv = (int)(idx % c8);
  const long pix = idx / c8;
  const int ox = (int)(pix % wo);
  const int oy = (int)((pix / wo) % ho);
  const long b = pix / ((long)wo * ho);
  const float sy = ry * (float)oy, sx = rx * (float)ox;
  const int y0 = (int)sy, x0 = (int)sx;
  const int y1 = y0 + (y0 < h - 1 ? 1 : 0), x1 = x0 + (x0 < w - 1 ? 1 : 0);
  const float ly = sy - (float)y0, lx = sx - (float)x0;
  const float hy = 1.0f - ly, hx = 1.0f - lx;
  const uint4* xv = reinterpret_cast<const uint4*>(x) + b * h * w * c8 + cv;
  const uint4 u00 = __ldg(xv + ((long)y0 * w + x0) * c8), u01 = __ldg(xv + ((long)y0 * w + x1) * c8);
  const uint4 u10 = __ldg(xv + ((long)y1 * w + x0) * c8), u11 = __ldg(xv + ((long)y1 * w + x1) * c8);
  const __half2 *a = reinterpret_cast<const __half2*>(&u00), *bq = reinterpret_cast<const __half2*>(&u01),
                *cq = reinterpret_cast<const __half2*>(&u10), *d = reinterpret_cast<const __half2*>(&u11);
  uint4 r;
  __half2* r2 = reinterpret_cast<__half2*>(&r);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 fa = __half22float2(a[i]), fb = __half22float2(bq[i]), fc = __half22float2(cq[i]), fd = __half22float2(d[i]);
    const float vx = hy * (hx * fa.x + lx * fb.x) + ly * (hx * fc.x + lx * fd.x);
    const float vy = hy * (hx * fa.y + lx * fb.y) + ly * (hx * fc.y + lx * fd.y);
    r2[i] = __floats2half2_rn(vx, vy);
  }
  reinterpret_cast<uint4*>(y)[idx] = r;
}

// out[r] = relu(sum_c relu(x[r][c]) * w[c] + bias[0]), fp32 accumulation, stored as fp16 or fp32; one thread per pixel.
template <typename Tout>
__global__ void dpt_head_out_kernel(const __half* __restrict__ x, long ldx, long rows, int c, const float* __restrict__ w,
                                    const float* __restrict__ bias, Tout* __restrict__ out) {
  const long r = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  const uint4* xr = reinterpret_cast<const uint4*>(x + r * ldx);
  float acc = 0.f;
  for (int k = 0; k < c / 8; ++k) {
    const uint4 u = __ldg(xr + k);
    const __half2* h2 = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = __half22float2(h2[i]);
      acc = fmaf(fmaxf(f.x, 0.f), __ldg(w + 8 * k + 2 * i), acc);
      acc = fmaf(fmaxf(f.y, 0.f), __ldg(w + 8 * k + 2 * i + 1), acc);
    }
  }
  const float v = acc + __ldg(bias);
  out[r] = (Tout)(v < 0.f ? 0.f : v);
}

}  // namespace vg

using namespace vg;

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

extern "C" {

int vgen_dpt_tconv_scatter(const void* g, int64_t ldg, const float* bias, void* out, int64_t nimg, int64_t hp, int64_t wp,
                           int64_t s, int64_t cout, void* stream) {
  VG_REQUIRE(g && bias && out, "vgen_dpt_tconv_scatter: null pointer");
  VG_REQUIRE(nimg >= 0 && hp > 0 && wp > 0 && s >= 1 && cout > 0 && cout % 8 == 0 && ldg >= s * s * cout && ldg % 8 == 0,
             "vgen_dpt_tconv_scatter: bad shape (cout and ldg must be multiples of 8)");
  VG_REQUIRE(aligned16(g) && aligned16(bias) && aligned16(out), "vgen_dpt_tconv_scatter: g, bias and out must be 16-byte aligned");
  const long total = nimg * hp * s * wp * s * (cout / 8);
  if (total == 0) return 0;
  launch_kernel(dpt_tconv_scatter_kernel, dim3(nblk_dpt(total, 256)), dim3(256), 0, reinterpret_cast<cudaStream_t>(stream),
                reinterpret_cast<const __half*>(g), (long)ldg, bias, reinterpret_cast<__half*>(out), (long)nimg, (int)hp,
                (int)wp, (int)s, (int)cout);
  VG_LAUNCH_CHECK("dpt_tconv_scatter_kernel");
  return 0;
}

int vgen_upsample_bilinear2x_ac(const void* x, void* y, int64_t nimg, int64_t h, int64_t w, int64_t c, void* stream) {
  VG_REQUIRE(x && y, "vgen_upsample_bilinear2x_ac: null pointer");
  VG_REQUIRE(nimg >= 0 && h > 0 && w > 0 && c > 0 && c % 8 == 0, "vgen_upsample_bilinear2x_ac: bad shape (C must be a multiple of 8)");
  VG_REQUIRE(aligned16(x) && aligned16(y), "vgen_upsample_bilinear2x_ac: x and y must be 16-byte aligned");
  const long total = nimg * 4 * h * w * (c / 8);
  if (total == 0) return 0;
  // area_pixel_compute_scale(align_corners=True): (in - 1) / (out - 1), computed in fp32 as PyTorch's kernels do
  const float ry = (float)(h - 1) / (float)(2 * h - 1), rx = (float)(w - 1) / (float)(2 * w - 1);
  launch_kernel(dpt_upsample_bilinear2x_kernel, dim3(nblk_dpt(total, 256)), dim3(256), 0,
                reinterpret_cast<cudaStream_t>(stream), reinterpret_cast<const __half*>(x), reinterpret_cast<__half*>(y),
                (long)nimg, (int)h, (int)w, (int)(c / 8), ry, rx);
  VG_LAUNCH_CHECK("dpt_upsample_bilinear2x_kernel");
  return 0;
}

int vgen_dpt_head_out(const void* x, int64_t ldx, int64_t rows, int64_t c, const float* w, const float* bias, void* out,
                      int out_is_f32, void* stream) {
  VG_REQUIRE(x && w && bias && out, "vgen_dpt_head_out: null pointer");
  VG_REQUIRE(rows >= 0 && c > 0 && c % 8 == 0 && c <= 1024 && ldx >= c && ldx % 8 == 0,
             "vgen_dpt_head_out: bad shape (c and ldx must be multiples of 8, c <= 1024)");
  VG_REQUIRE(aligned16(x), "vgen_dpt_head_out: x must be 16-byte aligned");
  if (rows == 0) return 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (out_is_f32)
    launch_kernel(dpt_head_out_kernel<float>, dim3(nblk_dpt(rows, 256)), dim3(256), 0, st, reinterpret_cast<const __half*>(x),
                  (long)ldx, (long)rows, (int)c, w, bias, reinterpret_cast<float*>(out));
  else
    launch_kernel(dpt_head_out_kernel<__half>, dim3(nblk_dpt(rows, 256)), dim3(256), 0, st, reinterpret_cast<const __half*>(x),
                  (long)ldx, (long)rows, (int)c, w, bias, reinterpret_cast<__half*>(out));
  VG_LAUNCH_CHECK("dpt_head_out_kernel");
  return 0;
}

}  // extern "C"
