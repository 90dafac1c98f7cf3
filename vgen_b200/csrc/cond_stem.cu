// VideoComposer condition stem: y = AdaptiveAvgPool_{oh x ow}(SiLU(conv3x3_pad1(x) + bias)) in one pass.
//
// The first three modules of every condition encoder of UNetSD_VideoLCM / UNetSD_TFT2V
// (tools/modules/unet/unet_videolcm.py:295-372, unet_tf2tv.py same lines) run at pixel resolution on every forward.
// Composed from generic ops they would write the 8-channel padded input, a 72-wide im2col matrix and the full-resolution
// 4*concat_dim-channel activation, and read each of them back.  Here each CTA stages its input tile (plus the 1-pixel
// conv halo) in shared memory once, every thread computes the conv + SiLU of the pixels of its own pooling window in
// registers, and only the pooled channels-last map is written.
//
// Work split: a CTA owns an 8 x 8 tile of pooled pixels of one image; thread (g, p) computes channels [8g, 8g+8) of pooled
// pixel p, so the 64 threads of a channel group (two warps) read the same weights (shared-memory broadcast).  Pooling
// windows are PyTorch's adaptive bins, start = floor(i*H/oh), end = ceil((i+1)*H/oh): uneven and overlapping windows are
// recomputed by each bin that covers them, which costs at most one extra row / column per bin.
// Arithmetic: fp32 throughout, one fp16 rounding at the store.
#include "common.h"

namespace {

constexpr int kTile = 8;          // pooled pixels per CTA side
constexpr int kCoPerThread = 8;   // output channels per thread (one 16-byte store)
constexpr int kMaxCout = 64;
constexpr int kMaxCin = 4;

__host__ __device__ inline int bin_start(int i, int in, int out) { return (i * in) / out; }
__host__ __device__ inline int bin_end(int i, int in, int out) { return ((i + 1) * in + out - 1) / out; }

__device__ inline float load_f(const float* p) { return __ldg(p); }
__device__ inline float load_f(const __half* p) { return __half2float(__ldg(p)); }

// x: [b][cin][f][H][W]; w: [cout][cin][3][3] fp32; bias [cout]; y: [(b f)][oh][ow][cout] fp16.
// Dynamic shared memory: cout*cin*9 weights, cout biases, then cin planes of span_h x span_w input values.
template <typename T>
__global__ void __launch_bounds__(kTile * kTile * (kMaxCout / kCoPerThread))
cond_stem_kernel(const T* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias, __half* __restrict__ y,
                 int f, int cin, int H, int W, int cout, int oh, int ow, int span_h, int span_w) {
  extern __shared__ float smem[];
  float* s_w = smem;                                  // [cout][cin*9]
  float* s_b = s_w + cout * cin * 9;                  // [cout]
  float* s_x = s_b + cout;                            // [cin][span_h][span_w]

  const int img = blockIdx.z;                         // (b f) image index
  const int bi = img / f, fi = img - bi * f;
  const int oy0 = blockIdx.y * kTile, ox0 = blockIdx.x * kTile;
  const int oy_last = min(oy0 + kTile, oh) - 1, ox_last = min(ox0 + kTile, ow) - 1;
  // input rows / cols of this tile's windows, with the conv halo
  const int r0 = bin_start(oy0, H, oh) - 1, c0 = bin_start(ox0, W, ow) - 1;
  const int rows = bin_end(oy_last, H, oh) + 1 - r0, cols = bin_end(ox_last, W, ow) + 1 - c0;

  const int nthr = blockDim.x, tid = threadIdx.x;
  for (int i = tid; i < cout * cin * 9; i += nthr) s_w[i] = __ldg(w + i);
  for (int i = tid; i < cout; i += nthr) s_b[i] = __ldg(bias + i);
  const long plane = (long)H * W;
  for (int ci = 0; ci < cin; ++ci) {
    const T* src = x + ((long)(bi * cin + ci) * f + fi) * plane;
    float* dst = s_x + ci * span_h * span_w;
    for (int i = tid; i < rows * cols; i += nthr) {
      const int rr = i / cols, cc = i - rr * cols;
      const int gy = r0 + rr, gx = c0 + cc;
      float v = 0.f;                                  // zero padding of the conv
      if (gy >= 0 && gy < H && gx >= 0 && gx < W) v = load_f(src + (long)gy * W + gx);
      dst[rr * span_w + cc] = v;
    }
  }
  __syncthreads();

  const int p = tid % (kTile * kTile), g = tid / (kTile * kTile);
  const int oy = oy0 + p / kTile, ox = ox0 + p % kTile;
  if (oy >= oh || ox >= ow) return;                   // no barrier follows
  const int y0 = bin_start(oy, H, oh), y1 = bin_end(oy, H, oh);
  const int x0 = bin_start(ox, W, ow), x1 = bin_end(ox, W, ow);
  const int co0 = g * kCoPerThread;
  const float* wg = s_w + co0 * cin * 9;
  const int wstride = cin * 9;

  float acc[kCoPerThread];
#pragma unroll
  for (int j = 0; j < kCoPerThread; ++j) acc[j] = 0.f;

  for (int yy = y0; yy < y1; ++yy) {
    for (int xx = x0; xx < x1; ++xx) {
      float cv[kCoPerThread];
#pragma unroll
      for (int j = 0; j < kCoPerThread; ++j) cv[j] = s_b[co0 + j];
      // window pixel (yy, xx) -> tile coordinates of its top-left conv tap
      const float* xb = s_x + (yy - 1 - r0) * span_w + (xx - 1 - c0);
      for (int ci = 0; ci < cin; ++ci) {
        const float* xc = xb + ci * span_h * span_w;
#pragma unroll
        for (int ky = 0; ky < 3; ++ky) {
#pragma unroll
          for (int kx = 0; kx < 3; ++kx) {
            const float v = xc[ky * span_w + kx];
            const int k = ci * 9 + ky * 3 + kx;
#pragma unroll
            for (int j = 0; j < kCoPerThread; ++j) cv[j] = fmaf(v, wg[j * wstride + k], cv[j]);
          }
        }
      }
#pragma unroll
      for (int j = 0; j < kCoPerThread; ++j) acc[j] += cv[j] / (1.f + __expf(-cv[j]));
    }
  }
  const float inv = 1.f / (float)((y1 - y0) * (x1 - x0));
  __align__(16) __half out[kCoPerThread];
#pragma unroll
  for (int j = 0; j < kCoPerThread; ++j) out[j] = __float2half_rn(acc[j] * inv);
  __half* dst = y + (((long)img * oh + oy) * ow + ox) * cout + co0;
  *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(out);
}

// Largest input span (rows or cols, halo included) of any kTile-bin group along one axis.
int max_span(int in, int out) {
  int m = 0;
  for (int t0 = 0; t0 < out; t0 += kTile) {
    const int t1 = (t0 + kTile < out ? t0 + kTile : out) - 1;
    const int s = bin_end(t1, in, out) - bin_start(t0, in, out) + 2;
    m = s > m ? s : m;
  }
  return m;
}

vg::PerDeviceOnce g_smem_attr;

}  // namespace

using namespace vg;

extern "C" int vgen_cond_stem(const void* x, int x_is_f32, int64_t b, int64_t cin, int64_t f, int64_t h, int64_t w,
                              const float* weight, const float* bias, int64_t cout, void* y, int64_t oh, int64_t ow,
                              void* stream) {
  VG_REQUIRE(x && weight && bias && y, "vgen_cond_stem: null pointer");
  VG_REQUIRE(b >= 0 && f > 0 && h > 0 && w > 0 && oh > 0 && ow > 0 && oh <= h && ow <= w,
             "vgen_cond_stem: bad shape (need 0 < oh <= h, 0 < ow <= w)");
  VG_REQUIRE(cin >= 1 && cin <= kMaxCin, "vgen_cond_stem: cin must be 1..4");
  VG_REQUIRE(cout > 0 && cout % kCoPerThread == 0 && cout <= kMaxCout, "vgen_cond_stem: cout must be a multiple of 8, at most 64");
  VG_REQUIRE(b * f <= 65535, "vgen_cond_stem: b*f must be at most 65535");
  VG_REQUIRE(((uintptr_t)y & 15) == 0, "vgen_cond_stem: y must be 16-byte aligned");
  VG_REQUIRE(h <= 32768 && w <= 32768, "vgen_cond_stem: image too large (h, w <= 32768)");
  if (b == 0) return 0;
  const int span_h = max_span((int)h, (int)oh), span_w = max_span((int)w, (int)ow);
  const size_t smem = sizeof(float) * ((size_t)cout * cin * 9 + cout + (size_t)cin * span_h * span_w);
  VG_REQUIRE(smem <= 200 * 1024, "vgen_cond_stem: pooling windows too large for one shared-memory tile (h/oh, w/ow too big)");
  if (g_smem_attr.need()) {
    VG_CUDA(cudaFuncSetAttribute(cond_stem_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    VG_CUDA(cudaFuncSetAttribute(cond_stem_kernel<__half>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    g_smem_attr.mark();
  }
  const dim3 grid(cdiv(ow, kTile), cdiv(oh, kTile), (unsigned)(b * f));
  const dim3 block(kTile * kTile * (unsigned)(cout / kCoPerThread));
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (x_is_f32)
    launch_kernel(cond_stem_kernel<float>, grid, block, smem, st, reinterpret_cast<const float*>(x), weight, bias,
                  reinterpret_cast<__half*>(y), (int)f, (int)cin, (int)h, (int)w, (int)cout, (int)oh, (int)ow, span_h, span_w);
  else
    launch_kernel(cond_stem_kernel<__half>, grid, block, smem, st, reinterpret_cast<const __half*>(x), weight, bias,
                  reinterpret_cast<__half*>(y), (int)f, (int)cin, (int)h, (int)w, (int)cout, (int)oh, (int)ow, span_h, span_w);
  VG_LAUNCH_CHECK("cond_stem_kernel");
  return 0;
}
