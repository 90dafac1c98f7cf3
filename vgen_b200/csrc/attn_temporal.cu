// Temporal self-attention: sequences are the f frames of one pixel, head_dim 64.  There are
// tens of thousands of short (L x L) problems per call, so a 64-row wgmma tile would be mostly padding
// (at least half at f <= 32, up to 48% at 33-63 frames); both kernels below use mma.sync.m16n8k16 fragments
// instead (the S accumulator layout IS the A-fragment layout of the P V product).
//  * f <= 32: attn_temporal_kernel, each warp owns one (pixel, head) and keeps the whole problem in registers.
//    It is bound by its q/k/v reads (8 FLOP/B), not by the math.
//  * f > 32: attn_temporal_flash_kernel, one CTA per (pixel, head, 64-query tile), each warp 16 query rows;
//    K/V stream through shared memory in 64-key blocks (cp.async, double-buffered when f > 64) with an online
//    softmax, so shared memory is fixed and any f works.
//
// Replaces xformers.ops.memory_efficient_attention for the TemporalTransformer blocks
// (/root/reference/tools/modules/unet/util.py:231-269 called from :1258-1261, tokens '(b h w) f c');
// the activations stay in the frame-major [f][hw][C] layout, the kernel gathers the f tokens of a pixel
// with a stride instead of materialising the reference's '(b h w) f c' permutation.
#include <algorithm>

#include "common.h"
#include "ptx.cuh"

namespace vg {

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
__device__ __forceinline__ void mma16816(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0,
                                         uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// LP = padded sequence length (16 or 32).  smem per warp: Q, K, V tiles [LP][64+8] fp16 (row padding
// of 16 B keeps ldmatrix conflict-free).
template <int LP>
__global__ void __launch_bounds__(128) attn_temporal_kernel(const __half* __restrict__ q, const __half* __restrict__ k,
                                                            const __half* __restrict__ v, __half* __restrict__ out,
                                                            long nseq, int heads, int L, long tok_stride_q,
                                                            long seq_stride_q, long tok_stride_o, long seq_stride_o,
                                                            float scale_log2, long spb, long batch_stride_q,
                                                            long batch_stride_o) {
  constexpr int kRow = 72;  // halfs per smem row
  constexpr int MT = LP / 16;
  extern __shared__ __align__(16) __half sm_t[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long item = (long)blockIdx.x * 4 + warp;  // (seq, head)
  if (item >= nseq * heads) return;
  const long seq = item / heads;
  const int head = (int)(item % heads);
  __half* sQ = sm_t + (size_t)warp * 3 * LP * kRow;
  __half* sK = sQ + LP * kRow;
  __half* sV = sK + LP * kRow;

  // ---- stage q/k/v rows of this (seq, head): each row is 128 contiguous bytes in HBM
  // videos back to back: sequence s is pixel (s % spb) of video (s / spb)
  const long vid = seq / spb, pix = seq - vid * spb;
  const long base = vid * batch_stride_q + pix * seq_stride_q + head * 64;
  for (int i = lane; i < LP * 8; i += 32) {
    const int t = i >> 3, piece = i & 7;
    uint4 uq = make_uint4(0, 0, 0, 0), uk = uq, uv = uq;
    if (t < L) {
      const long off = base + t * tok_stride_q + piece * 8;
      uq = __ldg(reinterpret_cast<const uint4*>(q + off));
      uk = __ldg(reinterpret_cast<const uint4*>(k + off));
      uv = __ldg(reinterpret_cast<const uint4*>(v + off));
    }
    *reinterpret_cast<uint4*>(sQ + t * kRow + piece * 8) = uq;
    *reinterpret_cast<uint4*>(sK + t * kRow + piece * 8) = uk;
    *reinterpret_cast<uint4*>(sV + t * kRow + piece * 8) = uv;
  }
  __syncwarp();

  const int g = lane >> 2, tq = lane & 3;
  // ---- S = Q K^T : MT m-tiles x (LP/8) n-tiles, k over 64 in 4 steps
  float s[MT][LP / 8][4];
#pragma unroll
  for (int m = 0; m < MT; ++m)
#pragma unroll
    for (int n = 0; n < LP / 8; ++n)
#pragma unroll
      for (int e = 0; e < 4; ++e) s[m][n][e] = 0.f;
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    uint32_t a[MT][4];
#pragma unroll
    for (int m = 0; m < MT; ++m) {
      // A 16x16 block: matrices (rows 0-7,k 0-7) (rows 8-15,k 0-7) (rows 0-7,k 8-15) (rows 8-15,k 8-15)
      const int row = m * 16 + (lane & 15);
      const int col = ks * 16 + ((lane >> 4) << 3);
      ldsm_x4(smem_u32(sQ + row * kRow + col), a[m][0], a[m][1], a[m][2], a[m][3]);
    }
#pragma unroll
    for (int n2 = 0; n2 < LP / 16; ++n2) {
      // B for two n-tiles (16 keys) x 16 k: K rows are keys, contiguous in d  -> non-transposed ldmatrix
      uint32_t b0, b1, b2, b3;
      const int row = n2 * 16 + (lane & 7) + ((lane >> 4) << 3);
      const int col = ks * 16 + (((lane >> 3) & 1) << 3);
      ldsm_x4(smem_u32(sK + row * kRow + col), b0, b1, b2, b3);
#pragma unroll
      for (int m = 0; m < MT; ++m) {
        mma16816(s[m][2 * n2], a[m][0], a[m][1], a[m][2], a[m][3], b0, b1);
        mma16816(s[m][2 * n2 + 1], a[m][0], a[m][1], a[m][2], a[m][3], b2, b3);
      }
    }
  }
  // ---- softmax over keys (row g -> elements 0,1 ; row g+8 -> elements 2,3 ; keys n*8 + 2*tq + {0,1})
  uint32_t pa[MT][LP / 8][2];  // P as packed fp16 pairs: [.][n][0] rows g, [.][n][1] rows g+8
  float inv_l[MT][2];
#pragma unroll
  for (int m = 0; m < MT; ++m) {
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int n = 0; n < LP / 8; ++n) {
      const int key = n * 8 + 2 * tq;
      if (key >= L) s[m][n][0] = s[m][n][2] = -INFINITY;
      if (key + 1 >= L) s[m][n][1] = s[m][n][3] = -INFINITY;
      mx0 = fmaxf(mx0, fmaxf(s[m][n][0], s[m][n][1]));
      mx1 = fmaxf(mx1, fmaxf(s[m][n][2], s[m][n][3]));
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    float l0 = 0.f, l1 = 0.f;
#pragma unroll
    for (int n = 0; n < LP / 8; ++n) {
      const float e0 = fast_exp2((s[m][n][0] - mx0) * scale_log2);
      const float e1 = fast_exp2((s[m][n][1] - mx0) * scale_log2);
      const float e2 = fast_exp2((s[m][n][2] - mx1) * scale_log2);
      const float e3 = fast_exp2((s[m][n][3] - mx1) * scale_log2);
      l0 += e0 + e1;
      l1 += e2 + e3;
      pa[m][n][0] = pack_half2(e0, e1);
      pa[m][n][1] = pack_half2(e2, e3);
    }
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
    l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    inv_l[m][0] = 1.0f / l0;
    inv_l[m][1] = 1.0f / l1;
  }
  // ---- O = P V : k over keys (LP/16 steps), n over d (8 tiles)
  float o[MT][8][4];
#pragma unroll
  for (int m = 0; m < MT; ++m)
#pragma unroll
    for (int n = 0; n < 8; ++n)
#pragma unroll
      for (int e = 0; e < 4; ++e) o[m][n][e] = 0.f;
#pragma unroll
  for (int ks = 0; ks < LP / 16; ++ks) {
#pragma unroll
    for (int n2 = 0; n2 < 4; ++n2) {
      // B (k = key, n = d): V rows are keys -> transposed ldmatrix; two d-tiles (16 d) per x4
      uint32_t b0, b1, b2, b3;
      const int row = ks * 16 + (lane & 7) + (((lane >> 3) & 1) << 3);
      const int col = n2 * 16 + ((lane >> 4) << 3);
      ldsm_x4_t(smem_u32(sV + row * kRow + col), b0, b1, b2, b3);
#pragma unroll
      for (int m = 0; m < MT; ++m) {
        const uint32_t a0 = pa[m][2 * ks][0], a1 = pa[m][2 * ks][1], a2 = pa[m][2 * ks + 1][0], a3 = pa[m][2 * ks + 1][1];
        mma16816(o[m][2 * n2], a0, a1, a2, a3, b0, b1);
        mma16816(o[m][2 * n2 + 1], a0, a1, a2, a3, b2, b3);
      }
    }
  }
  // ---- normalise, stage through smem (reuse sQ), coalesced 16-byte stores
  __syncwarp();
#pragma unroll
  for (int m = 0; m < MT; ++m)
#pragma unroll
    for (int n = 0; n < 8; ++n) {
      const int col = n * 8 + 2 * tq;
      *reinterpret_cast<uint32_t*>(sQ + (m * 16 + g) * kRow + col) = pack_half2(o[m][n][0] * inv_l[m][0], o[m][n][1] * inv_l[m][0]);
      *reinterpret_cast<uint32_t*>(sQ + (m * 16 + g + 8) * kRow + col) = pack_half2(o[m][n][2] * inv_l[m][1], o[m][n][3] * inv_l[m][1]);
    }
  __syncwarp();
  const long obase = vid * batch_stride_o + pix * seq_stride_o + head * 64;
  for (int i = lane; i < L * 8; i += 32) {
    const int t = i >> 3, piece = i & 7;
    *reinterpret_cast<uint4*>(out + obase + t * tok_stride_o + piece * 8) = *reinterpret_cast<const uint4*>(sQ + t * kRow + piece * 8);
  }
}

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool valid) {
  // src-size 0 reads nothing and zero-fills the 16 bytes (rows past L)
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// Any L > 32.  grid (nseq*heads, ceil(L/64)); blockDim 32 * ceil(min(L,64)/16).  smem: Q [64][kRow], then
// nbuf (1 when L <= 64, else 2) K/V block pairs [64][kRow].  Warps whose 16 rows all lie past L still load and
// meet the barriers but skip the math.
__global__ void __launch_bounds__(128) attn_temporal_flash_kernel(
    const __half* __restrict__ q, const __half* __restrict__ k, const __half* __restrict__ v, __half* __restrict__ out,
    int heads, int L, long tok_stride_q, long seq_stride_q, long tok_stride_o, long seq_stride_o, float scale_log2,
    long spb, long batch_stride_q, long batch_stride_o) {
  constexpr int kRow = 72;
  constexpr int kBlk = 64;
  extern __shared__ __align__(16) __half sm_f[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nthr = blockDim.x;
  const long item = blockIdx.x;  // (seq, head)
  const long seq = item / heads;
  const int head = (int)(item % heads);
  const int q0 = blockIdx.y * kBlk;
  const int nblk = (L + kBlk - 1) / kBlk;
  __half* sQ = sm_f;
  __half* sKV = sQ + kBlk * kRow;  // buffer i: K at sKV + 2*i*kBlk*kRow, V right after
  const long vid = seq / spb, pix = seq - vid * spb;
  const long base = vid * batch_stride_q + pix * seq_stride_q + head * 64;

  for (int i = threadIdx.x; i < kBlk * 8; i += nthr) {
    const int t = i >> 3, piece = i & 7;
    const bool ok = q0 + t < L;
    cp_async16(smem_u32(sQ + t * kRow + piece * 8), q + base + (ok ? (long)(q0 + t) * tok_stride_q + piece * 8 : 0), ok);
  }
  auto load_kv = [&](int blk, int buf) {
    __half* sK = sKV + (size_t)buf * 2 * kBlk * kRow;
    __half* sV = sK + kBlk * kRow;
    for (int i = threadIdx.x; i < kBlk * 8; i += nthr) {
      const int t = i >> 3, piece = i & 7, key = blk * kBlk + t;
      const bool ok = key < L;
      const long off = base + (ok ? (long)key * tok_stride_q + piece * 8 : 0);
      cp_async16(smem_u32(sK + t * kRow + piece * 8), k + off, ok);
      cp_async16(smem_u32(sV + t * kRow + piece * 8), v + off, ok);
    }
    cp_async_commit();
  };
  load_kv(0, 0);

  const int g = lane >> 2, tq = lane & 3;
  const int row0 = warp * 16;
  const bool active = q0 + row0 < L;  // warp-uniform
  uint32_t qa[4][4];
  float o[8][4];
#pragma unroll
  for (int n = 0; n < 8; ++n)
#pragma unroll
    for (int e = 0; e < 4; ++e) o[n][e] = 0.f;
  float mx0 = -INFINITY, mx1 = -INFINITY, l0 = 0.f, l1 = 0.f;  // rows g and g+8 (this thread's quad-partial sums)

  for (int blk = 0; blk < nblk; ++blk) {
    if (blk + 1 < nblk) {
      load_kv(blk + 1, (blk + 1) & 1);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    if (active) {
      const __half* sK = sKV + (size_t)(blk & 1) * 2 * kBlk * kRow;
      const __half* sV = sK + kBlk * kRow;
      if (blk == 0) {
#pragma unroll
        for (int ks = 0; ks < 4; ++ks)
          ldsm_x4(smem_u32(sQ + (row0 + (lane & 15)) * kRow + ks * 16 + ((lane >> 4) << 3)), qa[ks][0], qa[ks][1], qa[ks][2],
                  qa[ks][3]);
      }
      // ---- S = Q K^T for this key block: 8 n-tiles of 8 keys
      float s[8][4];
#pragma unroll
      for (int n = 0; n < 8; ++n)
#pragma unroll
        for (int e = 0; e < 4; ++e) s[n][e] = 0.f;
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
#pragma unroll
        for (int n2 = 0; n2 < 4; ++n2) {
          uint32_t b0, b1, b2, b3;
          const int row = n2 * 16 + (lane & 7) + ((lane >> 4) << 3);
          const int col = ks * 16 + (((lane >> 3) & 1) << 3);
          ldsm_x4(smem_u32(sK + row * kRow + col), b0, b1, b2, b3);
          mma16816(s[2 * n2], qa[ks][0], qa[ks][1], qa[ks][2], qa[ks][3], b0, b1);
          mma16816(s[2 * n2 + 1], qa[ks][0], qa[ks][1], qa[ks][2], qa[ks][3], b2, b3);
        }
      }
      // ---- online softmax: mask keys >= L, rescale the running sum and O by exp2((old max - new max) * scale)
      float bm0 = -INFINITY, bm1 = -INFINITY;
#pragma unroll
      for (int n = 0; n < 8; ++n) {
        const int key = blk * kBlk + n * 8 + 2 * tq;
        if (key >= L) s[n][0] = s[n][2] = -INFINITY;
        if (key + 1 >= L) s[n][1] = s[n][3] = -INFINITY;
        bm0 = fmaxf(bm0, fmaxf(s[n][0], s[n][1]));
        bm1 = fmaxf(bm1, fmaxf(s[n][2], s[n][3]));
      }
      bm0 = fmaxf(bm0, __shfl_xor_sync(0xffffffffu, bm0, 1));
      bm0 = fmaxf(bm0, __shfl_xor_sync(0xffffffffu, bm0, 2));
      bm1 = fmaxf(bm1, __shfl_xor_sync(0xffffffffu, bm1, 1));
      bm1 = fmaxf(bm1, __shfl_xor_sync(0xffffffffu, bm1, 2));
      const float nm0 = fmaxf(mx0, bm0), nm1 = fmaxf(mx1, bm1);  // finite: key blk*64 < L is never masked
      const float c0 = fast_exp2((mx0 - nm0) * scale_log2), c1 = fast_exp2((mx1 - nm1) * scale_log2);
      mx0 = nm0;
      mx1 = nm1;
      l0 *= c0;
      l1 *= c1;
#pragma unroll
      for (int n = 0; n < 8; ++n) {
        o[n][0] *= c0;
        o[n][1] *= c0;
        o[n][2] *= c1;
        o[n][3] *= c1;
      }
      uint32_t pa[8][2];
#pragma unroll
      for (int n = 0; n < 8; ++n) {
        const float e0 = fast_exp2((s[n][0] - nm0) * scale_log2);
        const float e1 = fast_exp2((s[n][1] - nm0) * scale_log2);
        const float e2 = fast_exp2((s[n][2] - nm1) * scale_log2);
        const float e3 = fast_exp2((s[n][3] - nm1) * scale_log2);
        l0 += e0 + e1;
        l1 += e2 + e3;
        pa[n][0] = pack_half2(e0, e1);
        pa[n][1] = pack_half2(e2, e3);
      }
      // ---- O += P V: k over the block's 64 keys (4 steps), n over d (8 tiles)
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
#pragma unroll
        for (int n2 = 0; n2 < 4; ++n2) {
          uint32_t b0, b1, b2, b3;
          const int row = ks * 16 + (lane & 7) + (((lane >> 3) & 1) << 3);
          const int col = n2 * 16 + ((lane >> 4) << 3);
          ldsm_x4_t(smem_u32(sV + row * kRow + col), b0, b1, b2, b3);
          mma16816(o[2 * n2], pa[2 * ks][0], pa[2 * ks][1], pa[2 * ks + 1][0], pa[2 * ks + 1][1], b0, b1);
          mma16816(o[2 * n2 + 1], pa[2 * ks][0], pa[2 * ks][1], pa[2 * ks + 1][0], pa[2 * ks + 1][1], b2, b3);
        }
      }
    }
    __syncthreads();  // the next iteration's load overwrites this buffer
  }
  if (!active) return;
  // ---- normalise once, stage through this warp's own Q rows, coalesced 16-byte stores of rows < L
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float i0 = 1.0f / l0, i1 = 1.0f / l1;
#pragma unroll
  for (int n = 0; n < 8; ++n) {
    const int col = n * 8 + 2 * tq;
    *reinterpret_cast<uint32_t*>(sQ + (row0 + g) * kRow + col) = pack_half2(o[n][0] * i0, o[n][1] * i0);
    *reinterpret_cast<uint32_t*>(sQ + (row0 + g + 8) * kRow + col) = pack_half2(o[n][2] * i1, o[n][3] * i1);
  }
  __syncwarp();
  const long obase = vid * batch_stride_o + pix * seq_stride_o + head * 64;
  for (int i = lane; i < 16 * 8; i += 32) {
    const int t = row0 + (i >> 3), piece = i & 7;
    if (q0 + t < L)
      *reinterpret_cast<uint4*>(out + obase + (long)(q0 + t) * tok_stride_o + piece * 8) =
          *reinterpret_cast<const uint4*>(sQ + t * kRow + piece * 8);
  }
}

// Generic small attention (any head_dim <= 64, any L), one thread per (seq, head, query): the frame transformers
// with 4- or 8-channel heads (UNetSD_I2VGen's local temporal encoder, unet_i2vgen.py:122-124, and the VideoComposer
// condition encoders, unet_videolcm.py:121-141; util.py:1396-1424), and head_dim 64 with unaligned operands.
__global__ void attn_small_kernel(const __half* __restrict__ q, const __half* __restrict__ k, const __half* __restrict__ v,
                                  __half* __restrict__ out, long nseq, int heads, int L, int d, long tok_stride,
                                  long seq_stride, long tok_stride_o, long seq_stride_o, float scale, long spb,
                                  long batch_stride, long batch_stride_o) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= nseq * heads * L) return;
  const int i = (int)(idx % L);
  const int head = (int)((idx / L) % heads);
  const long seq = idx / ((long)L * heads);
  const long vid = seq / spb, pix = seq - vid * spb;
  const long base = vid * batch_stride + pix * seq_stride + head * d;
  float qv[64];
  for (int c = 0; c < d; ++c) qv[c] = __half2float(q[base + i * tok_stride + c]);
  float mx = -INFINITY;
  for (int j = 0; j < L; ++j) {
    float sc = 0.f;
    for (int c = 0; c < d; ++c) sc += qv[c] * __half2float(k[base + j * tok_stride + c]);
    mx = fmaxf(mx, sc * scale);
  }
  float l = 0.f;
  float acc[64];
  for (int c = 0; c < d; ++c) acc[c] = 0.f;
  for (int j = 0; j < L; ++j) {
    float sc = 0.f;
    for (int c = 0; c < d; ++c) sc += qv[c] * __half2float(k[base + j * tok_stride + c]);
    const float e = __expf(sc * scale - mx);
    l += e;
    for (int c = 0; c < d; ++c) acc[c] += e * __half2float(v[base + j * tok_stride + c]);
  }
  const long ob = vid * batch_stride_o + pix * seq_stride_o + head * d + i * tok_stride_o;
  for (int c = 0; c < d; ++c) out[ob + c] = __float2half_rn(acc[c] / l);
}

}  // namespace vg

using namespace vg;

extern "C" int vgen_attention_temporal(const void* q, const void* k, const void* v, void* out, int64_t nseq, int64_t heads,
                                       int64_t L, int64_t head_dim, int64_t tok_stride, int64_t seq_stride,
                                       int64_t tok_stride_o, int64_t seq_stride_o, int64_t seqs_per_batch,
                                       int64_t batch_stride, int64_t batch_stride_o, float scale, void* stream) {
  VG_REQUIRE(q && k && v && out, "vgen_attention_temporal: null pointer");
  VG_REQUIRE(nseq >= 0 && heads > 0 && L > 0 && head_dim > 0, "vgen_attention_temporal: bad shape");
  if (seqs_per_batch <= 0) seqs_per_batch = nseq > 0 ? nseq : 1;
  VG_REQUIRE(nseq % seqs_per_batch == 0, "vgen_attention_temporal: nseq must be a multiple of seqs_per_batch");
  const long spb = seqs_per_batch;
  if (nseq == 0) return 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const __half *qp = reinterpret_cast<const __half*>(q), *kp = reinterpret_cast<const __half*>(k),
               *vp = reinterpret_cast<const __half*>(v);
  __half* op = reinterpret_cast<__half*>(out);
  const bool aligned = ((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(k) | reinterpret_cast<uintptr_t>(v) |
                         reinterpret_cast<uintptr_t>(out)) & 15) == 0 &&
                       tok_stride % 8 == 0 && seq_stride % 8 == 0 && tok_stride_o % 8 == 0 && seq_stride_o % 8 == 0 &&
                       batch_stride % 8 == 0 && batch_stride_o % 8 == 0;
  if (head_dim == 64 && L <= 32 && aligned) {
    const long items = nseq * heads;
    const unsigned blocks = (unsigned)((items + 3) / 4);
    const float sl2 = scale * 1.4426950408889634f;
    if (L <= 16) {
      const size_t smem = 4 * 3 * 16 * 72 * sizeof(__half);
      launch_kernel(attn_temporal_kernel<16>, dim3(blocks), dim3(128), smem, st, qp, kp, vp, op, nseq, (int)heads, (int)L, tok_stride, seq_stride,
                                                          tok_stride_o, seq_stride_o, sl2, spb, batch_stride, batch_stride_o);
    } else {
      const size_t smem = 4 * 3 * 32 * 72 * sizeof(__half);
      static PerDeviceOnce attr_once;
      if (attr_once.need()) {
        VG_CUDA(cudaFuncSetAttribute(attn_temporal_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr_once.mark();
      }
      launch_kernel(attn_temporal_kernel<32>, dim3(blocks), dim3(128), smem, st, qp, kp, vp, op, nseq, (int)heads, (int)L, tok_stride, seq_stride,
                                                          tok_stride_o, seq_stride_o, sl2, spb, batch_stride, batch_stride_o);
    }
    VG_LAUNCH_CHECK("attn_temporal_kernel");
    return 0;
  }
  if (head_dim == 64 && aligned) {
    const long items = nseq * heads;
    const long qtiles = (L + 63) / 64;
    VG_REQUIRE(items <= 0x7fffffffL && qtiles <= 65535, "vgen_attention_temporal: too many sequences or frames");
    const int warps = (int)((std::min<long>(L, 64) + 15) / 16);
    const size_t smem = (size_t)(1 + 2 * (L > 64 ? 2 : 1)) * 64 * 72 * sizeof(__half);  // 27 KiB or 45 KiB
    launch_kernel(attn_temporal_flash_kernel, dim3((unsigned)items, (unsigned)qtiles), dim3(32 * warps), smem, st, qp, kp, vp, op,
                  (int)heads, (int)L, tok_stride, seq_stride, tok_stride_o, seq_stride_o, scale * 1.4426950408889634f, spb,
                  batch_stride, batch_stride_o);
    VG_LAUNCH_CHECK("attn_temporal_flash_kernel");
    return 0;
  }
  VG_REQUIRE(head_dim <= 64, "vgen_attention_temporal: unsupported head_dim");
  const long total = nseq * heads * L;
  launch_kernel(attn_small_kernel, dim3((unsigned)((total + 127) / 128)), dim3(128), 0, st, qp, kp, vp, op, nseq, (int)heads, (int)L, (int)head_dim,
                                                                    tok_stride, seq_stride, tok_stride_o, seq_stride_o, scale, spb,
                                                                    batch_stride, batch_stride_o);
  VG_LAUNCH_CHECK("attn_small_kernel");
  return 0;
}
