// The pieces of the VideoComposer sketch annotators (tools/annotator/sketch/pidinet.py, sketch_simplification.py) that
// the tap-GEMM family cannot express by itself.  Activations are channels-last fp16, arithmetic fp32:
//   * PiDiNet's depthwise 3x3 / 5x5 conv + ReLU, optionally on the 2x2 max-pool of its input (the stride-2 blocks), with
//     the pooled tensor written as well for the block's 1x1 shortcut;
//   * CSAM + MapReduce in two per-pixel passes: y = sigmoid(conv2(conv1(relu(x)))) is one value per pixel, so
//     MapReduce(x * y) = y * (w . x) + b;
//   * the final fuse: bilinear resize of the four side maps (align_corners=False), the 4 -> 1 classifier and the sigmoid;
//   * the cleaner's last layer, a 3x3 conv to one channel + sigmoid (an N = 1 GEMM would fill one column of a tile);
//   * the cleaner's input normalisation (x - mean) / std, applied before any zero padding.
#include "common.h"

namespace vg {

static inline unsigned nblk_sk(long total, int threads) { return (unsigned)((total + threads - 1) / threads); }

__device__ __forceinline__ float sigmoid_f(float v) { return 1.0f / (1.0f + expf(-v)); }

// ------------------------------------------------------------------ depthwise conv (+ 2x2 max-pool) + ReLU
// One CTA = an 8 x 16 output tile x 64 channels (8 groups of 8, one 16-byte vector each), the tile and its halo staged in
// shared memory; the output grid is (h, w), or (h/2, w/2) floored with POOL.
static constexpr int kDwTy = 8, kDwTx = 16, kDwThreads = 256;

template <int K, bool POOL>
__global__ void __launch_bounds__(kDwThreads) dwconv_relu_kernel(const __half* __restrict__ x, const float* __restrict__ wgt,
                                                                 __half* __restrict__ pooled, __half* __restrict__ out, int h,
                                                                 int w, int c, int ho, int wo, int tiles_x) {
  constexpr int R = K / 2, HY = kDwTy + 2 * R, HX = kDwTx + 2 * R;
  __shared__ uint4 tile[HY * HX * 8];
  __shared__ float ws[K * K * 64];
  const int n = blockIdx.z, c0 = blockIdx.y * 64;
  const int ty0 = (blockIdx.x / tiles_x) * kDwTy, tx0 = (blockIdx.x % tiles_x) * kDwTx;
  for (int i = threadIdx.x; i < K * K * 64; i += kDwThreads) ws[i] = __ldg(wgt + (long)(i / 64) * c + c0 + i % 64);
  const uint4* xv = reinterpret_cast<const uint4*>(x);
  const int c8 = c / 8;
  for (int i = threadIdx.x; i < HY * HX * 8; i += kDwThreads) {
    const int g = i & 7, p = i >> 3, hy = p / HX, hx = p - hy * HX;
    const int oy = ty0 + hy - R, ox = tx0 + hx - R;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (oy >= 0 && oy < ho && ox >= 0 && ox < wo) {
      if (POOL) {
        const long b = ((long)n * h + 2 * oy) * w + 2 * ox;
        const uint4 a0 = __ldg(xv + b * c8 + c0 / 8 + g), a1 = __ldg(xv + (b + 1) * c8 + c0 / 8 + g);
        const uint4 a2 = __ldg(xv + (b + w) * c8 + c0 / 8 + g), a3 = __ldg(xv + (b + w + 1) * c8 + c0 / 8 + g);
        const __half2 *p0 = reinterpret_cast<const __half2*>(&a0), *p1 = reinterpret_cast<const __half2*>(&a1),
                      *p2 = reinterpret_cast<const __half2*>(&a2), *p3 = reinterpret_cast<const __half2*>(&a3);
        __half2* r = reinterpret_cast<__half2*>(&v);
#pragma unroll
        for (int j = 0; j < 4; ++j) r[j] = __hmax2(__hmax2(p0[j], p1[j]), __hmax2(p2[j], p3[j]));
        if (hy >= R && hy < R + kDwTy && hx >= R && hx < R + kDwTx)
          reinterpret_cast<uint4*>(pooled)[(((long)n * ho + oy) * wo + ox) * c8 + c0 / 8 + g] = v;
      } else {
        v = __ldg(xv + (((long)n * h + oy) * w + ox) * c8 + c0 / 8 + g);
      }
    }
    tile[i] = v;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < kDwTy * kDwTx * 8; i += kDwThreads) {
    const int g = i & 7, p = i >> 3, py = p / kDwTx, px = p - py * kDwTx;
    const int oy = ty0 + py, ox = tx0 + px;
    if (oy >= ho || ox >= wo) continue;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll
    for (int ky = 0; ky < K; ++ky)
#pragma unroll
      for (int kx = 0; kx < K; ++kx) {
        const uint4 u = tile[((py + ky) * HX + px + kx) * 8 + g];
        const __half2* h2 = reinterpret_cast<const __half2*>(&u);
        const float* wk = ws + (ky * K + kx) * 64 + g * 8;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = __half22float2(h2[j]);
          acc[2 * j] = fmaf(f.x, wk[2 * j], acc[2 * j]);
          acc[2 * j + 1] = fmaf(f.y, wk[2 * j + 1], acc[2 * j + 1]);
        }
      }
    uint4 r;
    __half2* r2 = reinterpret_cast<__half2*>(&r);
#pragma unroll
    for (int j = 0; j < 4; ++j) r2[j] = __floats2half2_rn(fmaxf(acc[2 * j], 0.f), fmaxf(acc[2 * j + 1], 0.f));
    reinterpret_cast<uint4*>(out)[(((long)n * ho + oy) * wo + ox) * c8 + c0 / 8 + g] = r;
  }
}

// ------------------------------------------------------------------ CSAM + MapReduce
// pass 1, per pixel: t[r][0..3] = w1 . relu(x[r]) + b1 (CSAM conv1), s[r] = wm . x[r] (MapReduce without its bias)
__global__ void csam_pre_kernel(const __half* __restrict__ x, long rows, int c, const float* __restrict__ w1,
                                const float* __restrict__ b1, const float* __restrict__ wm, float4* __restrict__ t,
                                float* __restrict__ s) {
  const long r = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  const uint4* xr = reinterpret_cast<const uint4*>(x + r * c);
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f, am = 0.f;
  for (int k = 0; k < c / 8; ++k) {
    const uint4 u = __ldg(xr + k);
    const __half2* h2 = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float2 f2 = __half22float2(h2[j / 2]);
      const float v = (j & 1) ? f2.y : f2.x, rv = fmaxf(v, 0.f);
      const int ch = 8 * k + j;
      a0 = fmaf(rv, __ldg(w1 + ch), a0);
      a1 = fmaf(rv, __ldg(w1 + c + ch), a1);
      a2 = fmaf(rv, __ldg(w1 + 2 * c + ch), a2);
      a3 = fmaf(rv, __ldg(w1 + 3 * c + ch), a3);
      am = fmaf(v, __ldg(wm + ch), am);
    }
  }
  t[r] = make_float4(a0 + __ldg(b1), a1 + __ldg(b1 + 1), a2 + __ldg(b1 + 2), a3 + __ldg(b1 + 3));
  s[r] = am;
}

// pass 2, per pixel: e = sigmoid(conv3x3(t; w2 [4][3][3], zero padding)) * s + bm
__global__ void csam_out_kernel(const float4* __restrict__ t, const float* __restrict__ s, long nimg, int h, int w,
                                const float* __restrict__ w2, const float* __restrict__ bm, float* __restrict__ e) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= nimg * h * w) return;
  const int x0 = (int)(idx % w), y0 = (int)((idx / w) % h);
  const long b = idx / ((long)w * h);
  float acc = 0.f;
#pragma unroll
  for (int ky = 0; ky < 3; ++ky)
#pragma unroll
    for (int kx = 0; kx < 3; ++kx) {
      const int yy = y0 + ky - 1, xx = x0 + kx - 1;
      if (yy < 0 || yy >= h || xx < 0 || xx >= w) continue;
      const float4 v = __ldg(t + (b * h + yy) * w + xx);
      acc = fmaf(v.x, __ldg(w2 + 0 * 9 + ky * 3 + kx), acc);
      acc = fmaf(v.y, __ldg(w2 + 1 * 9 + ky * 3 + kx), acc);
      acc = fmaf(v.z, __ldg(w2 + 2 * 9 + ky * 3 + kx), acc);
      acc = fmaf(v.w, __ldg(w2 + 3 * 9 + ky * 3 + kx), acc);
    }
  e[idx] = fmaf(sigmoid_f(acc), s[idx], __ldg(bm));
}

// ------------------------------------------------------------------ final fuse
struct FuseMaps {
  const float* e[4];
  int h[4], w[4];
  float sy[4], sx[4];   // in / out, in fp32 (area_pixel_compute_scale, align_corners=False)
};

// F.interpolate(bilinear, align_corners=False) with PyTorch's arithmetic: src = max(scale * (dst + 0.5) - 0.5, 0), the
// lower index its truncation, the upper one clamped to the last row / column
__device__ __forceinline__ float bilinear_ac0(const float* m, int h, int w, float sy, float sx, int oy, int ox) {
  const float fy = fmaxf(sy * ((float)oy + 0.5f) - 0.5f, 0.f), fx = fmaxf(sx * ((float)ox + 0.5f) - 0.5f, 0.f);
  const int y0 = (int)fy, x0 = (int)fx;
  const int y1 = y0 + (y0 < h - 1 ? 1 : 0), x1 = x0 + (x0 < w - 1 ? 1 : 0);
  const float ly = fy - (float)y0, lx = fx - (float)x0, hy = 1.f - ly, hx = 1.f - lx;
  return hy * (hx * __ldg(m + y0 * w + x0) + lx * __ldg(m + y0 * w + x1)) +
         ly * (hx * __ldg(m + y1 * w + x0) + lx * __ldg(m + y1 * w + x1));
}

template <typename Tout>
__global__ void pidinet_fuse_kernel(const FuseMaps maps, long nimg, int H, int W, const float* __restrict__ cw,
                                    Tout* __restrict__ out) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= nimg * H * W) return;
  const int ox = (int)(idx % W), oy = (int)((idx / W) % H);
  const long b = idx / ((long)W * H);
  float acc = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float v = bilinear_ac0(maps.e[i] + b * maps.h[i] * maps.w[i], maps.h[i], maps.w[i], maps.sy[i], maps.sx[i], oy, ox);
    acc = fmaf(__ldg(cw + i), v, acc);
  }
  out[idx] = (Tout)sigmoid_f(acc + __ldg(cw + 4));
}

// ------------------------------------------------------------------ 3x3 conv to one channel + sigmoid
// out[b][y][x] = sigmoid(sum_{ky,kx,c} x[b][y+ky-1][x+kx-1][c] * w[ky*3+kx][c] + bias), zero padding; one thread per pixel
template <typename Tout>
__global__ void conv3x3_to1_sigmoid_kernel(const __half* __restrict__ x, long nimg, int h, int w, int c,
                                           const float* __restrict__ wgt, const float* __restrict__ bias,
                                           Tout* __restrict__ out) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= nimg * h * w) return;
  const int x0 = (int)(idx % w), y0 = (int)((idx / w) % h);
  const long b = idx / ((long)w * h);
  float acc = 0.f;
  for (int ky = 0; ky < 3; ++ky)
    for (int kx = 0; kx < 3; ++kx) {
      const int yy = y0 + ky - 1, xx = x0 + kx - 1;
      if (yy < 0 || yy >= h || xx < 0 || xx >= w) continue;
      const uint4* xr = reinterpret_cast<const uint4*>(x + ((b * h + yy) * w + xx) * c);
      const float* wk = wgt + (ky * 3 + kx) * c;
      for (int k = 0; k < c / 8; ++k) {
        const uint4 u = __ldg(xr + k);
        const __half2* h2 = reinterpret_cast<const __half2*>(&u);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = __half22float2(h2[j]);
          acc = fmaf(f.x, __ldg(wk + 8 * k + 2 * j), acc);
          acc = fmaf(f.y, __ldg(wk + 8 * k + 2 * j + 1), acc);
        }
      }
    }
  out[idx] = (Tout)sigmoid_f(acc + __ldg(bias));
}

// ------------------------------------------------------------------ (x - mean) / std -> fp16
template <typename Tin>
__global__ void sketch_normalize_kernel(const Tin* __restrict__ x, long count, float mean, float std_, __half* __restrict__ y) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  y[i] = __float2half_rn(((float)x[i] - mean) / std_);
}

}  // namespace vg

using namespace vg;

static bool aligned16_sk(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

extern "C" {

int vgen_dwconv_relu(const void* x, int64_t nimg, int64_t h, int64_t w, int64_t c, int64_t k, const float* wgt, int pool,
                     void* pooled, void* out, void* stream) {
  VG_REQUIRE(x && wgt && out && (!pool || pooled), "vgen_dwconv_relu: null pointer");
  VG_REQUIRE(nimg >= 0 && h > 0 && w > 0 && c > 0 && c % 64 == 0 && (k == 3 || k == 5),
             "vgen_dwconv_relu: bad shape (c a multiple of 64, k 3 or 5)");
  VG_REQUIRE(!pool || (h >= 2 && w >= 2), "vgen_dwconv_relu: a pooled input needs h, w >= 2");
  VG_REQUIRE(aligned16_sk(x) && aligned16_sk(out) && aligned16_sk(pooled), "vgen_dwconv_relu: x, pooled and out must be 16-byte aligned");
  const int ho = (int)(pool ? h / 2 : h), wo = (int)(pool ? w / 2 : w);
  const int tiles_x = (wo + kDwTx - 1) / kDwTx, tiles_y = (ho + kDwTy - 1) / kDwTy;
  if (nimg == 0) return 0;
  VG_REQUIRE(nimg < 65536 && (long)tiles_x * tiles_y < (1L << 31), "vgen_dwconv_relu: too large");
  const dim3 grid((unsigned)(tiles_x * tiles_y), (unsigned)(c / 64), (unsigned)nimg);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const __half* xi = reinterpret_cast<const __half*>(x);
  __half *pi = reinterpret_cast<__half*>(pooled), *oi = reinterpret_cast<__half*>(out);
  if (k == 3 && pool) launch_kernel(dwconv_relu_kernel<3, true>, grid, dim3(kDwThreads), 0, st, xi, wgt, pi, oi, (int)h, (int)w, (int)c, ho, wo, tiles_x);
  if (k == 3 && !pool) launch_kernel(dwconv_relu_kernel<3, false>, grid, dim3(kDwThreads), 0, st, xi, wgt, pi, oi, (int)h, (int)w, (int)c, ho, wo, tiles_x);
  if (k == 5 && pool) launch_kernel(dwconv_relu_kernel<5, true>, grid, dim3(kDwThreads), 0, st, xi, wgt, pi, oi, (int)h, (int)w, (int)c, ho, wo, tiles_x);
  if (k == 5 && !pool) launch_kernel(dwconv_relu_kernel<5, false>, grid, dim3(kDwThreads), 0, st, xi, wgt, pi, oi, (int)h, (int)w, (int)c, ho, wo, tiles_x);
  VG_LAUNCH_CHECK("dwconv_relu_kernel");
  return 0;
}

int vgen_csam_mapreduce(const void* x, int64_t nimg, int64_t h, int64_t w, int64_t c, const float* w1, const float* b1,
                        const float* w2, const float* wm, const float* bm, float* t_ws, float* s_ws, float* e, void* stream) {
  VG_REQUIRE(x && w1 && b1 && w2 && wm && bm && t_ws && s_ws && e, "vgen_csam_mapreduce: null pointer");
  VG_REQUIRE(nimg >= 0 && h > 0 && w > 0 && c > 0 && c % 8 == 0, "vgen_csam_mapreduce: bad shape (c a multiple of 8)");
  VG_REQUIRE(aligned16_sk(x) && aligned16_sk(t_ws), "vgen_csam_mapreduce: x and t_ws must be 16-byte aligned");
  const long rows = nimg * h * w;
  if (rows == 0) return 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  launch_kernel(csam_pre_kernel, dim3(nblk_sk(rows, 256)), dim3(256), 0, st, reinterpret_cast<const __half*>(x), rows, (int)c,
                w1, b1, wm, reinterpret_cast<float4*>(t_ws), s_ws);
  VG_LAUNCH_CHECK("csam_pre_kernel");
  launch_kernel(csam_out_kernel, dim3(nblk_sk(rows, 256)), dim3(256), 0, st, reinterpret_cast<const float4*>(t_ws),
                (const float*)s_ws, (long)nimg, (int)h, (int)w, w2, bm, e);
  VG_LAUNCH_CHECK("csam_out_kernel");
  return 0;
}

int vgen_pidinet_fuse(const float* e1, const float* e2, const float* e3, const float* e4, const int64_t* hw, int64_t nimg,
                      int64_t H, int64_t W, const float* cw, void* out, int out_is_f32, void* stream) {
  VG_REQUIRE(e1 && e2 && e3 && e4 && hw && cw && out, "vgen_pidinet_fuse: null pointer");
  VG_REQUIRE(nimg >= 0 && H > 0 && W > 0, "vgen_pidinet_fuse: bad shape");
  FuseMaps m;
  const float* es[4] = {e1, e2, e3, e4};
  for (int i = 0; i < 4; ++i) {
    VG_REQUIRE(hw[2 * i] > 0 && hw[2 * i + 1] > 0, "vgen_pidinet_fuse: empty side map");
    m.e[i] = es[i];
    m.h[i] = (int)hw[2 * i];
    m.w[i] = (int)hw[2 * i + 1];
    m.sy[i] = (float)m.h[i] / (float)H;
    m.sx[i] = (float)m.w[i] / (float)W;
  }
  const long total = nimg * H * W;
  if (total == 0) return 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (out_is_f32)
    launch_kernel(pidinet_fuse_kernel<float>, dim3(nblk_sk(total, 256)), dim3(256), 0, st, m, (long)nimg, (int)H, (int)W, cw,
                  reinterpret_cast<float*>(out));
  else
    launch_kernel(pidinet_fuse_kernel<__half>, dim3(nblk_sk(total, 256)), dim3(256), 0, st, m, (long)nimg, (int)H, (int)W, cw,
                  reinterpret_cast<__half*>(out));
  VG_LAUNCH_CHECK("pidinet_fuse_kernel");
  return 0;
}

int vgen_conv3x3_to1_sigmoid(const void* x, int64_t nimg, int64_t h, int64_t w, int64_t c, const float* wgt, const float* bias,
                             void* out, int out_is_f32, void* stream) {
  VG_REQUIRE(x && wgt && bias && out, "vgen_conv3x3_to1_sigmoid: null pointer");
  VG_REQUIRE(nimg >= 0 && h > 0 && w > 0 && c > 0 && c % 8 == 0, "vgen_conv3x3_to1_sigmoid: bad shape (c a multiple of 8)");
  VG_REQUIRE(aligned16_sk(x), "vgen_conv3x3_to1_sigmoid: x must be 16-byte aligned");
  const long total = nimg * h * w;
  if (total == 0) return 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (out_is_f32)
    launch_kernel(conv3x3_to1_sigmoid_kernel<float>, dim3(nblk_sk(total, 256)), dim3(256), 0, st, reinterpret_cast<const __half*>(x),
                  (long)nimg, (int)h, (int)w, (int)c, wgt, bias, reinterpret_cast<float*>(out));
  else
    launch_kernel(conv3x3_to1_sigmoid_kernel<__half>, dim3(nblk_sk(total, 256)), dim3(256), 0, st, reinterpret_cast<const __half*>(x),
                  (long)nimg, (int)h, (int)w, (int)c, wgt, bias, reinterpret_cast<__half*>(out));
  VG_LAUNCH_CHECK("conv3x3_to1_sigmoid_kernel");
  return 0;
}

int vgen_sketch_normalize(const void* x, int x_is_f32, int64_t count, float mean, float std_, void* y, void* stream) {
  VG_REQUIRE(x && y && count >= 0 && std_ != 0.f, "vgen_sketch_normalize: bad arguments");
  if (count == 0) return 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (x_is_f32)
    launch_kernel(sketch_normalize_kernel<float>, dim3(nblk_sk(count, 256)), dim3(256), 0, st, reinterpret_cast<const float*>(x),
                  (long)count, mean, std_, reinterpret_cast<__half*>(y));
  else
    launch_kernel(sketch_normalize_kernel<__half>, dim3(nblk_sk(count, 256)), dim3(256), 0, st, reinterpret_cast<const __half*>(x),
                  (long)count, mean, std_, reinterpret_cast<__half*>(y));
  VG_LAUNCH_CHECK("sketch_normalize_kernel");
  return 0;
}

}  // extern "C"
