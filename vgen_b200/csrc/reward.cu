// InstructVideo's segmental video reward (utils/reward/reward.py DiffRewardModel.reward_scorer), device side: the frame
// preprocess of the HPSv2 image tower and the segment-averaged score.
//
// 1. reward_frames_kernel: for each selected frame, the decoder's x * 0.5 + 0.5 (fp32 input) or x / 255 (uint8 RGB input),
//    clamp(0, 1), torchvision's Resize (F.interpolate bilinear, align_corners=False, antialias off or on) and
//    Normalize((x - mean) / std), in IEEE fp32.  A per-output-frame table names the source frame, so the selected frames
//    are read in place from the full video.  The host computes each axis' taps once per size (first source index, tap
//    count, fp32 weights; F.interpolate's weights, see vgen_b200/reward.py bilinear_taps); a source index past the edge
//    is clamped, which is F.interpolate's i1 = min(i0 + 1, in - 1).  A block owns a 16 x 32 output tile: the horizontal
//    pass over the source rows its vertical windows read lands in a shared fp32 tile, then the vertical pass reads it.
// 2. segment_reward_kernel: one block per video: F.normalize of its s image features and of its text feature (fp32,
//    x / max(||x||, 1e-12)), the per-segment cosines, optionally times exp(-|g - f // 2| * lambda) (the temporally
//    attenuated reward, g the segment's frame index), averaged over the segments.
#include "common.h"
#include "ptx.cuh"

namespace vg {

constexpr int RF_TX = 32, RF_TY = 16, RF_THREADS = 256;

struct FrameSrc {
  const void* p;
  int u8;                                   // 1: uint8 samples, x / 255; 0: fp32 samples, x * 0.5 + 0.5
  int frames_per;                           // frames per video in the source (1 for a [n, ...] frame batch)
  long s_video, s_frame, s_c, s_y, s_x;     // element strides
  int h, w;
};

__device__ __forceinline__ float load_unit(const FrameSrc& s, long off) {
  float v;
  if (s.u8) v = __fdiv_rn((float)__ldg(reinterpret_cast<const uint8_t*>(s.p) + off), 255.0f);
  else v = __fadd_rn(__fmul_rn(__ldg(reinterpret_cast<const float*>(s.p) + off), 0.5f), 0.5f);
  return fminf(fmaxf(v, 0.0f), 1.0f);
}

// idx [n] source frame (video * frames_per + frame); hb [ow][2] = (first source column, taps), hk [ow][kh] fp32;
// vb [oh][2], vk [oh][kv]; out: fp16 [n][oh][ow][3] (out_f32 = 0) or fp32 [n][3][oh][ow] (out_f32 = 1).
__global__ void __launch_bounds__(RF_THREADS) reward_frames_kernel(
    FrameSrc s, const int* __restrict__ idx, const int* __restrict__ hb, const float* __restrict__ hk, int kh,
    const int* __restrict__ vb, const float* __restrict__ vk, int kv, int oh, int ow, float m0, float m1, float m2, float s0,
    float s1, float s2, void* __restrict__ out, int out_f32) {
  extern __shared__ float tile[];                            // [rows][RF_TX][3]: the horizontal pass of this tile's rows
  const int img = blockIdx.z;
  const int j = __ldg(idx + img);
  const long base = (long)(j / s.frames_per) * s.s_video + (long)(j % s.frames_per) * s.s_frame;
  const int ox0 = blockIdx.x * RF_TX, oy0 = blockIdx.y * RF_TY;
  const int ty_n = min(RF_TY, oh - oy0), tx_n = min(RF_TX, ow - ox0);
  const int r0 = __ldg(vb + 2 * oy0);
  const int r1 = __ldg(vb + 2 * (oy0 + ty_n - 1)) + __ldg(vb + 2 * (oy0 + ty_n - 1) + 1);   // windows move monotonically
  const int rows = r1 - r0;
  for (int i = threadIdx.x; i < rows * RF_TX; i += RF_THREADS) {
    const int r = i / RF_TX, cx = i - r * RF_TX;
    if (cx >= tx_n) continue;
    const int ox = ox0 + cx;
    const int xmin = __ldg(hb + 2 * ox), cnt = __ldg(hb + 2 * ox + 1);
    const float* k = hk + (long)ox * kh;
    const long row = base + (long)min(r0 + r, s.h - 1) * s.s_y;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f;
    for (int x = 0; x < cnt; ++x) {
      const float kx = __ldg(k + x);
      const long p = row + (long)min(xmin + x, s.w - 1) * s.s_x;
      a0 = fmaf(load_unit(s, p), kx, a0);
      a1 = fmaf(load_unit(s, p + s.s_c), kx, a1);
      a2 = fmaf(load_unit(s, p + 2 * s.s_c), kx, a2);
    }
    float* t = tile + (r * RF_TX + cx) * 3;
    t[0] = a0, t[1] = a1, t[2] = a2;
  }
  __syncthreads();
  const float mean[3] = {m0, m1, m2}, sd[3] = {s0, s1, s2};
  for (int i = threadIdx.x; i < RF_TY * RF_TX; i += RF_THREADS) {
    const int cy = i / RF_TX, cx = i - cy * RF_TX;
    if (cy >= ty_n || cx >= tx_n) continue;
    const int oy = oy0 + cy, ox = ox0 + cx;
    const int ymin = __ldg(vb + 2 * oy) - r0, cnt = __ldg(vb + 2 * oy + 1);
    const float* k = vk + (long)oy * kv;
    float acc[3] = {0.f, 0.f, 0.f};
    for (int y = 0; y < cnt; ++y) {
      const float ky = __ldg(k + y);
      const float* t = tile + ((ymin + y) * RF_TX + cx) * 3;
#pragma unroll
      for (int c = 0; c < 3; ++c) acc[c] = fmaf(t[c], ky, acc[c]);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float v = __fdiv_rn(__fsub_rn(acc[c], mean[c]), sd[c]);     // Normalize: sub_(mean).div_(std)
      if (out_f32)
        reinterpret_cast<float*>(out)[(((long)img * 3 + c) * oh + oy) * ow + ox] = v;
      else
        reinterpret_cast<__half*>(out)[(((long)img * oh + oy) * ow + ox) * 3 + c] = __float2half_rn(v);
    }
  }
}

// img [b * s][e] (video-major), txt [b][e], gidx [b * s] the segments' frame indices; out [b].
__global__ void __launch_bounds__(128) segment_reward_kernel(const float* __restrict__ img, const float* __restrict__ txt,
                                                             const int* __restrict__ gidx, int s, int e, int f, int tar,
                                                             float lambda, float* __restrict__ out) {
  extern __shared__ float diag[];                            // [s]
  const int k = blockIdx.x;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const float* t = txt + (long)k * e;
  for (int j = wid; j < s; j += nw) {
    const float* x = img + ((long)k * s + j) * e;
    float xx = 0.f, tt = 0.f, xt = 0.f;
    for (int c = lane; c < e; c += 32) {
      const float a = x[c], b = t[c];
      xx = fmaf(a, a, xx), tt = fmaf(b, b, tt), xt = fmaf(a, b, xt);
    }
    xx = warp_sum(xx), tt = warp_sum(tt), xt = warp_sum(xt);
    if (lane == 0) {
      float d = xt / (fmaxf(sqrtf(xx), 1e-12f) * fmaxf(sqrtf(tt), 1e-12f));
      if (tar) d *= expf(-(float)abs(__ldg(gidx + (long)k * s + j) - f / 2) * lambda);
      diag[j] = d;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float m = 0.f;
    for (int j = 0; j < s; ++j) m += diag[j];
    out[k] = m / (float)s;
  }
}

}  // namespace vg

using namespace vg;

extern "C" {

int vgen_reward_frames(const void* src, int src_u8, const int32_t* frame_idx, int64_t n, int64_t frames_per,
                       int64_t s_video, int64_t s_frame, int64_t s_c, int64_t s_y, int64_t s_x, int64_t h, int64_t w,
                       const int32_t* hbounds, const float* hcoef, int64_t kh, const int32_t* vbounds, const float* vcoef,
                       int64_t kv, int64_t oh, int64_t ow, int64_t tile_rows, const float* mean3, const float* std3,
                       void* out, int out_f32, void* stream) {
  VG_REQUIRE(src && frame_idx && hbounds && hcoef && vbounds && vcoef && mean3 && std3 && out,
             "vgen_reward_frames: null pointer");
  VG_REQUIRE(n >= 0 && frames_per > 0 && h > 0 && w > 0 && kh > 0 && kv > 0 && oh > 0 && ow > 0 && tile_rows > 0,
             "vgen_reward_frames: bad shape");
  VG_REQUIRE(n <= 65535 && h < (1 << 30) && w < (1 << 30), "vgen_reward_frames: too many or too large frames");
  const size_t smem = (size_t)tile_rows * RF_TX * 3 * sizeof(float);
  VG_REQUIRE(smem <= 200 * 1024, "vgen_reward_frames: the vertical windows of a tile span too many rows");
  if (n == 0) return 0;
  static PerDeviceOnce attr;
  if (attr.need()) {
    VG_CUDA(cudaFuncSetAttribute(reward_frames_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr.mark();
  }
  FrameSrc s{src, src_u8 ? 1 : 0, (int)frames_per, (long)s_video, (long)s_frame, (long)s_c, (long)s_y, (long)s_x, (int)h, (int)w};
  dim3 grid((unsigned)cdiv(ow, RF_TX), (unsigned)cdiv(oh, RF_TY), (unsigned)n);
  launch_kernel(reward_frames_kernel, grid, dim3(RF_THREADS), smem, reinterpret_cast<cudaStream_t>(stream), s, frame_idx,
                hbounds, hcoef, (int)kh, vbounds, vcoef, (int)kv, (int)oh, (int)ow, mean3[0], mean3[1], mean3[2], std3[0],
                std3[1], std3[2], out, out_f32);
  VG_LAUNCH_CHECK("reward_frames_kernel");
  return 0;
}

int vgen_segment_reward(const float* image_features, const float* text_features, const int32_t* frame_idx, int64_t b,
                        int64_t s, int64_t e, int64_t f, int tar, float lambda_tar, float* out, void* stream) {
  VG_REQUIRE(image_features && text_features && out && (!tar || frame_idx), "vgen_segment_reward: null pointer");
  VG_REQUIRE(b >= 0 && s >= 1 && e > 0 && f >= s && b <= 2147483647, "vgen_segment_reward: bad shape");
  VG_REQUIRE(s <= 12 * 1024, "vgen_segment_reward: too many segments for one block");
  if (b == 0) return 0;
  launch_kernel(segment_reward_kernel, dim3((unsigned)b), dim3(128), (size_t)s * sizeof(float),
                reinterpret_cast<cudaStream_t>(stream), image_features, text_features, frame_idx, (int)s, (int)e, (int)f,
                tar ? 1 : 0, lambda_tar, out);
  VG_LAUNCH_CHECK("segment_reward_kernel");
  return 0;
}

}  // extern "C"
