// DreamVideo's evaluation metric (metric/cal_metric_DreamVideo.py), device side: the two image transforms and the scores.
//
// 1. resize_crop_norm_kernel: torchvision's Resize(short side, BICUBIC) -> CenterCrop -> ToTensor -> Normalize of uint8
//    RGB images, bit-exact with Pillow's 8-bit ImagingResample (libImaging/Resample.c).  The host computes Pillow's
//    fixed-point coefficients (22 fractional bits, per output row / column) and passes only the rows and columns inside
//    the crop, so nothing outside the crop is computed.  A block owns a 16 x 32 output tile: it first runs the
//    horizontal pass over the source rows its vertical windows read (int32 sums from 1 << 21, >> 22, clamped to
//    [0, 255], into a uint8 tile in shared memory, exactly Pillow's intermediate image), then the vertical pass from
//    there.  An axis Pillow does not resample arrives as an identity table (one tap of weight 1 << 22), which
//    reproduces the byte.  Normalisation is torchvision's order in IEEE fp32: (u / 255 - mean) / std.
// 2. video_scores_kernel: CLIP-T, CLIP-I, DINO-I and temporal consistency of one video from its fp32 features, in one
//    block, with F.normalize's x / max(||x||, 1e-12) and the reference's un-renormalised frame means.
#include "common.h"
#include "ptx.cuh"

namespace vg {

constexpr int RS_TX = 32, RS_TY = 16, RS_THREADS = 256;
constexpr int RS_BITS = 22;

__device__ __forceinline__ int clip8(int ss) { return min(max(ss >> RS_BITS, 0), 255); }

// src [n][h][w][3] uint8; hb [cw][2] = (first source column, taps), hk [cw][kh]; vb [ch][2] = (first source row, taps),
// vk [ch][kv]; out: fp16 [n][ch][cw][3] (out_f32 = 0) or fp32 [n][3][ch][cw] (out_f32 = 1).
__global__ void __launch_bounds__(RS_THREADS) resize_crop_norm_kernel(
    const uint8_t* __restrict__ src, int h, int w, const int* __restrict__ hb, const int* __restrict__ hk, int kh,
    const int* __restrict__ vb, const int* __restrict__ vk, int kv, int ch, int cw, float m0, float m1, float m2, float s0,
    float s1, float s2, void* __restrict__ out, int out_f32) {
  extern __shared__ uint8_t tile[];                       // [rows][RS_TX][3]: the horizontal pass of this tile's rows
  const int img = blockIdx.z;
  const int ox0 = blockIdx.x * RS_TX, oy0 = blockIdx.y * RS_TY;
  const int ty_n = min(RS_TY, ch - oy0), tx_n = min(RS_TX, cw - ox0);
  const int r0 = __ldg(vb + 2 * oy0);
  const int r1 = __ldg(vb + 2 * (oy0 + ty_n - 1)) + __ldg(vb + 2 * (oy0 + ty_n - 1) + 1);   // windows move monotonically
  const int rows = r1 - r0;
  const uint8_t* im = src + (long)img * h * w * 3;
  for (int i = threadIdx.x; i < rows * RS_TX; i += RS_THREADS) {
    const int r = i / RS_TX, cx = i - r * RS_TX;
    if (cx >= tx_n) continue;
    const int ox = ox0 + cx;
    const int xmin = __ldg(hb + 2 * ox), cnt = __ldg(hb + 2 * ox + 1);
    const int* k = hk + (long)ox * kh;
    const uint8_t* p = im + ((long)(r0 + r) * w + xmin) * 3;
    int s0i = 1 << (RS_BITS - 1), s1i = s0i, s2i = s0i;
    for (int x = 0; x < cnt; ++x) {
      const int kx = __ldg(k + x);
      s0i += (int)__ldg(p + 3 * x) * kx;
      s1i += (int)__ldg(p + 3 * x + 1) * kx;
      s2i += (int)__ldg(p + 3 * x + 2) * kx;
    }
    uint8_t* t = tile + (r * RS_TX + cx) * 3;
    t[0] = (uint8_t)clip8(s0i), t[1] = (uint8_t)clip8(s1i), t[2] = (uint8_t)clip8(s2i);
  }
  __syncthreads();
  const float mean[3] = {m0, m1, m2}, sd[3] = {s0, s1, s2};
  for (int i = threadIdx.x; i < RS_TY * RS_TX; i += RS_THREADS) {
    const int cy = i / RS_TX, cx = i - cy * RS_TX;
    if (cy >= ty_n || cx >= tx_n) continue;
    const int oy = oy0 + cy, ox = ox0 + cx;
    const int ymin = __ldg(vb + 2 * oy) - r0, cnt = __ldg(vb + 2 * oy + 1);
    const int* k = vk + (long)oy * kv;
    int acc[3] = {1 << (RS_BITS - 1), 1 << (RS_BITS - 1), 1 << (RS_BITS - 1)};
    for (int y = 0; y < cnt; ++y) {
      const int ky = __ldg(k + y);
      const uint8_t* t = tile + ((ymin + y) * RS_TX + cx) * 3;
#pragma unroll
      for (int c = 0; c < 3; ++c) acc[c] += (int)t[c] * ky;
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float u = __fdiv_rn((float)clip8(acc[c]), 255.0f);          // ToTensor: byte / 255
      const float v = __fdiv_rn(__fsub_rn(u, mean[c]), sd[c]);          // Normalize: sub_(mean).div_(std)
      if (out_f32)
        reinterpret_cast<float*>(out)[(((long)img * 3 + c) * ch + oy) * cw + ox] = v;
      else
        reinterpret_cast<__half*>(out)[(((long)img * ch + oy) * cw + ox) * 3 + c] = __float2half_rn(v);
    }
  }
}

// ---- scores -----------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float row_dot(const float* a, const float* b, int n, int lane) {
  float s = 0.f;
  for (int c = lane; c < n; c += 32) s += a[c] * b[c];
  return warp_sum(s);
}

// cf [f][e] CLIP frame features, tx [e] text feature, ct [t][e] CLIP target features, df [f][d] / dt [t][d] DINO;
// out[4] = {CLIP-T, CLIP-I, DINO-I, temporal consistency}.
__global__ void __launch_bounds__(256) video_scores_kernel(const float* __restrict__ cf, const float* __restrict__ tx,
                                                           const float* __restrict__ ct, const float* __restrict__ df,
                                                           const float* __restrict__ dt, int f, int e, int t, int d,
                                                           float* __restrict__ out) {
  extern __shared__ float sm[];
  float* nrm = sm;                       // norms: [f] clip frames, [1] text, [t] clip targets, [f] dino frames, [t] dino targets
  float* gm = nrm + 2 * f + 2 * t + 1;   // [e] mean of the normalised CLIP frame features
  float* gdm = gm + e;                   // [d] the same for DINO
  float* pair = gdm + d;                 // [f - 1] consecutive-frame cosines
  float* tdot = pair + f;                // [t] CLIP target . gm, then [t] DINO target . gdm
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int nrows = 2 * f + 2 * t + 1;
  for (int r = wid; r < nrows; r += nw) {
    const float* x;
    int n;
    if (r < f) x = cf + (long)r * e, n = e;
    else if (r == f) x = tx, n = e;
    else if (r < f + 1 + t) x = ct + (long)(r - f - 1) * e, n = e;
    else if (r < 2 * f + 1 + t) x = df + (long)(r - f - 1 - t) * d, n = d;
    else x = dt + (long)(r - 2 * f - 1 - t) * d, n = d;
    const float ss = row_dot(x, x, n, lane);
    if (lane == 0) nrm[r] = fmaxf(sqrtf(ss), 1e-12f);
  }
  __syncthreads();
  const float* nd = nrm + f + 1 + t;
  for (int c = threadIdx.x; c < e + d; c += blockDim.x) {
    float s = 0.f;
    if (c < e)
      for (int i = 0; i < f; ++i) s += cf[(long)i * e + c] / nrm[i];
    else
      for (int i = 0; i < f; ++i) s += df[(long)i * d + (c - e)] / nd[i];
    if (c < e) gm[c] = s / (float)f;
    else gdm[c - e] = s / (float)f;
  }
  __syncthreads();
  for (int i = wid; i < f - 1; i += nw) {
    float s = 0.f;
    for (int c = lane; c < e; c += 32) s += (cf[(long)i * e + c] / nrm[i]) * (cf[(long)(i + 1) * e + c] / nrm[i + 1]);
    s = warp_sum(s);
    if (lane == 0) pair[i] = s;
  }
  for (int j = wid; j < 2 * t; j += nw) {
    float s;
    if (j < t) s = row_dot(ct + (long)j * e, gm, e, lane) / nrm[f + 1 + j];
    else s = row_dot(dt + (long)(j - t) * d, gdm, d, lane) / nd[f + j - t];
    if (lane == 0) tdot[j] = s;
  }
  float clip_t = 0.f;
  if (wid == 0) {
    float s = 0.f;
    for (int c = lane; c < e; c += 32) s += (tx[c] / nrm[f]) * gm[c];
    clip_t = warp_sum(s);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float tc = 0.f, ci = 0.f, di = 0.f;
    for (int i = 0; i < f - 1; ++i) tc += pair[i];
    for (int j = 0; j < t; ++j) ci += tdot[j], di += tdot[t + j];
    out[0] = clip_t;
    out[1] = t > 0 ? ci / (float)t : 0.f;
    out[2] = t > 0 ? di / (float)t : 0.f;
    out[3] = tc / (float)(f - 1);                    // one frame: 0 / 0 = NaN, the mean of an empty tensor
  }
}

}  // namespace vg

using namespace vg;

extern "C" {

int vgen_resize_bicubic_crop_normalize(const uint8_t* src, int64_t n, int64_t h, int64_t w, const int32_t* hbounds,
                                       const int32_t* hcoef, int64_t kh, const int32_t* vbounds, const int32_t* vcoef,
                                       int64_t kv, int64_t ch, int64_t cw, int64_t tile_rows, const float* mean3,
                                       const float* std3, void* out, int out_f32, void* stream) {
  VG_REQUIRE(src && hbounds && hcoef && vbounds && vcoef && mean3 && std3 && out,
             "vgen_resize_bicubic_crop_normalize: null pointer");
  VG_REQUIRE(n >= 0 && h > 0 && w > 0 && kh > 0 && kv > 0 && ch > 0 && cw > 0 && tile_rows > 0,
             "vgen_resize_bicubic_crop_normalize: bad shape");
  VG_REQUIRE(n <= 65535 && h * w * 3 < (1ll << 31), "vgen_resize_bicubic_crop_normalize: too many or too large images");
  const size_t smem = (size_t)tile_rows * RS_TX * 3;
  VG_REQUIRE(smem <= 200 * 1024, "vgen_resize_bicubic_crop_normalize: the vertical windows of a tile span too many rows");
  if (n == 0) return 0;
  static PerDeviceOnce attr;
  if (attr.need()) {
    VG_CUDA(cudaFuncSetAttribute(resize_crop_norm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr.mark();
  }
  dim3 grid((unsigned)cdiv(cw, RS_TX), (unsigned)cdiv(ch, RS_TY), (unsigned)n);
  launch_kernel(resize_crop_norm_kernel, grid, dim3(RS_THREADS), smem, reinterpret_cast<cudaStream_t>(stream), src, (int)h,
                (int)w, hbounds, hcoef, (int)kh, vbounds, vcoef, (int)kv, (int)ch, (int)cw, mean3[0], mean3[1], mean3[2],
                std3[0], std3[1], std3[2], out, out_f32);
  VG_LAUNCH_CHECK("resize_crop_norm_kernel");
  return 0;
}

int vgen_video_scores(const float* clip_frames, int64_t f, int64_t e, const float* text, const float* clip_targets,
                      int64_t t, const float* dino_frames, const float* dino_targets, int64_t d, float* out4, void* stream) {
  VG_REQUIRE(clip_frames && text && dino_frames && out4 && (t == 0 || (clip_targets && dino_targets)),
             "vgen_video_scores: null pointer");
  VG_REQUIRE(f >= 1 && e > 0 && d > 0 && t >= 0, "vgen_video_scores: bad shape");
  const size_t smem = sizeof(float) * (size_t)(2 * f + 2 * t + 1 + e + d + f + 2 * t);
  VG_REQUIRE(smem <= 48 * 1024, "vgen_video_scores: too many frames / targets for one block");
  launch_kernel(video_scores_kernel, dim3(1), dim3(256), smem, reinterpret_cast<cudaStream_t>(stream), clip_frames, text,
                clip_targets, dino_frames, dino_targets, (int)f, (int)e, (int)t, (int)d, out4);
  VG_LAUNCH_CHECK("video_scores_kernel");
  return 0;
}

}  // extern "C"
