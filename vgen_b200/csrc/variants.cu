// Kernels that only the model variants of SURVEY.md section 8 row a21 need (UNetSD_HiGen, UNetSD_SR600):
//   * cross attention for arbitrary head_dim <= 256 and ragged (lq, lk) -- HiGen's 16-token context
//     transformer (head_dim 160), far too small for the wgmma kernel;
//   * F.interpolate(mode='linear') over the frame axis of the motion embedding (unet_higen.py:387-396);
//   * the FreeU-style skip filter of UNetSD_SR600 (unet_sr600.py:30-49,271-283): the 2x2 centre block of
//     the shifted 2-D spectrum is scaled.  Only four DFT bins change, so the filter is evaluated as
//     x - (1-s)*Re(L) with L the inverse DFT of those four bins -- two reductions and one rank-4 update,
//     no FFT library;
//   * a scaled strided copy ("x[:, :C/2] *= 1.1" fused with the channel concat).
#include "common.h"
#include "ptx.cuh"

namespace vg {

// ------------------------------------------------------------------ small cross attention
// one warp per (batch, head, query); lanes split head_dim (8 values per lane, head_dim <= 256);
// online softmax over the keys.  q[b][lq][heads*d] with token stride ldq; k/v likewise.
__global__ void attn_cross_small_kernel(const __half* __restrict__ q, const __half* __restrict__ k,
                                        const __half* __restrict__ v, __half* __restrict__ out, long batch, int heads,
                                        int lq, int lk, int d, long ldq, long ldk, long ldv, long ldo, int kv_batch_div,
                                        float scale, int causal) {
  const long warp = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= batch * heads * lq) return;
  const int i = (int)(warp % lq);
  const int head = (int)((warp / lq) % heads);
  const long b = warp / ((long)lq * heads);
  const long bk = b / kv_batch_div;
  const __half* qp = q + (b * lq + i) * ldq + head * d;
  const __half* kp = k + bk * lk * ldk + head * d;
  const __half* vp = v + bk * lk * ldv + head * d;
  float qv[8], acc[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const int ch = lane + 32 * c;
    qv[c] = ch < d ? __half2float(qp[ch]) * scale : 0.f;
    acc[c] = 0.f;
  }
  float mx = -INFINITY, l = 0.f;
  // causal (CLIP text tower, attn_mask of open_clip's build_attention_mask): query i sees keys 0 .. i + (lk - lq)
  const int jend = causal ? min(lk, i + 1 + (lk - lq)) : lk;
  for (int j = 0; j < jend; ++j) {
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      const int ch = lane + 32 * c;
      if (ch < d) s += qv[c] * __half2float(kp[j * ldk + ch]);
    }
    s = warp_sum(s);
    const float mn = fmaxf(mx, s);
    const float corr = __expf(mx - mn), e = __expf(s - mn);
    l = l * corr + e;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      const int ch = lane + 32 * c;
      if (ch < d) acc[c] = acc[c] * corr + e * __half2float(vp[j * ldv + ch]);
    }
    mx = mn;
  }
  __half* op = out + (b * lq + i) * ldo + head * d;
  const float inv = 1.0f / l;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const int ch = lane + 32 * c;
    if (ch < d) op[ch] = __float2half_rn(acc[c] * inv);
  }
}

// ------------------------------------------------------------------ linear interpolation of rows
// x[nseq][lin][c] -> y[nseq][lout][c], F.interpolate(mode='linear', align_corners=False) along the
// middle axis: src = (dst + 0.5) * lin/lout - 0.5 clamped at 0, neighbours clamped at lin-1.
__global__ void interp_linear_rows_kernel(const __half* __restrict__ x, __half* __restrict__ y, long nseq, int lin, int lout,
                                          int c) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= nseq * lout * c) return;
  const int ch = (int)(idx % c);
  const int o = (int)((idx / c) % lout);
  const long s = idx / ((long)c * lout);
  const float ratio = (float)lin / (float)lout;
  float src = ((float)o + 0.5f) * ratio - 0.5f;
  if (src < 0.f) src = 0.f;
  const int i0 = (int)src;
  const int i1 = i0 + (i0 < lin - 1 ? 1 : 0);
  const float w1 = src - (float)i0, w0 = 1.0f - w1;
  const float a = __half2float(x[(s * lin + i0) * c + ch]), b = __half2float(x[(s * lin + i1) * c + ch]);
  y[idx] = __float2half_rn(w0 * a + w1 * b);
}

// ------------------------------------------------------------------ SR600 low-frequency skip filter
// grid (c/64 chunks, nimg); block (64 channels, 4 pixel slices).  Pass 1 accumulates the four DFT bins
// (ky, kx) in {0,-1}x{0,-1} of every (image, channel) plane; pass 2 subtracts (1-scale) * Re(inverse
// DFT of those bins) and stores fp16 into a (possibly wider) destination row.
constexpr int kFfChan = 64;
constexpr int kFfSlices = 4;

__global__ void __launch_bounds__(kFfChan* kFfSlices)
    fourier_lowfreq_kernel(const __half* __restrict__ x, __half* __restrict__ y, int h, int w, int c, long ldx, long ldy,
                           float scale) {
  extern __shared__ float sm[];
  float* cy = sm;            // cos(2 pi y / h)
  float* sy = cy + h;
  float* cx = sy + h;        // cos(2 pi x / w)
  float* sx = cx + w;
  float* red = sx + w;       // [slices][7][64]
  const int tid = threadIdx.y * kFfChan + threadIdx.x;
  for (int i = tid; i < h; i += kFfChan * kFfSlices) sincospif(2.0f * (float)i / (float)h, &sy[i], &cy[i]);
  for (int i = tid; i < w; i += kFfChan * kFfSlices) sincospif(2.0f * (float)i / (float)w, &sx[i], &cx[i]);
  __syncthreads();
  const int ch = blockIdx.x * kFfChan + threadIdx.x;
  const long n = blockIdx.y;
  const bool live = ch < c;
  const __half* xp = x + n * (long)h * w * ldx + ch;
  // X00 (real); X10 = sum x e^{+i ty}; X01 = sum x e^{+i tx}; X11 = sum x e^{+i (ty+tx)}
  float a00 = 0.f, a10r = 0.f, a10i = 0.f, a01r = 0.f, a01i = 0.f, a11r = 0.f, a11i = 0.f;
  if (live) {
    for (int p = threadIdx.y; p < h * w; p += kFfSlices) {
      const int yy = p / w, xx = p - yy * w;
      const float v = __half2float(xp[(long)p * ldx]);
      const float c1 = cy[yy], s1 = sy[yy], c2 = cx[xx], s2 = sx[xx];
      a00 += v;
      a10r += v * c1, a10i += v * s1;
      a01r += v * c2, a01i += v * s2;
      a11r += v * (c1 * c2 - s1 * s2), a11i += v * (s1 * c2 + c1 * s2);
    }
  }
  float vals[7] = {a00, a10r, a10i, a01r, a01i, a11r, a11i};
#pragma unroll
  for (int q = 0; q < 7; ++q) red[(threadIdx.y * 7 + q) * kFfChan + threadIdx.x] = vals[q];
  __syncthreads();
#pragma unroll
  for (int q = 0; q < 7; ++q) {
    float t = 0.f;
#pragma unroll
    for (int s = 0; s < kFfSlices; ++s) t += red[(s * 7 + q) * kFfChan + threadIdx.x];
    vals[q] = t;
  }
  if (!live) return;
  const float g = (1.0f - scale) / (float)(h * w);
  __half* yp = y + n * (long)h * w * ldy + ch;
  for (int p = threadIdx.y; p < h * w; p += kFfSlices) {
    const int yy = p / w, xx = p - yy * w;
    const float c1 = cy[yy], s1 = sy[yy], c2 = cx[xx], s2 = sx[xx];
    const float c12 = c1 * c2 - s1 * s2, s12 = s1 * c2 + c1 * s2;
    // Re(X e^{-i a}) = Xr cos a + Xi sin a
    const float low = vals[0] + vals[1] * c1 + vals[2] * s1 + vals[3] * c2 + vals[4] * s2 + vals[5] * c12 + vals[6] * s12;
    const float v = __half2float(xp[(long)p * ldx]);
    yp[(long)p * ldy] = __float2half_rn(v - g * low);
  }
}

// nearest x2 upsampling keeping output rows [row0, row0 + rows_out) of the 2h rows (UpsampleSR600 drops
// the first and last row, util.py:799-801); 8 channels per thread.
__global__ void upsample2x_rows_kernel(const __half* __restrict__ x, __half* __restrict__ y, long nimg, int h, int w, int cv,
                                       int row0, int rows_out) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const long total = nimg * rows_out * (2L * w) * cv;
  if (idx >= total) return;
  const int c8 = (int)(idx % cv);
  const int ox = (int)((idx / cv) % (2 * w));
  const int oy = (int)((idx / ((long)cv * 2 * w)) % rows_out);
  const long n = idx / ((long)cv * 2 * w * rows_out);
  const int iy = (oy + row0) >> 1, ix = ox >> 1;
  reinterpret_cast<uint4*>(y)[idx] = __ldg(reinterpret_cast<const uint4*>(x) + ((n * h + iy) * w + ix) * cv + c8);
}

__global__ void scale_copy2d_kernel(const __half* __restrict__ src, long lds, __half* __restrict__ dst, long ldd, long rows,
                                    int cols, float s) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * cols) return;
  const long r = idx / cols;
  const int c = (int)(idx % cols);
  dst[r * ldd + c] = __float2half_rn(__half2float(src[r * lds + c]) * s);
}

}  // namespace vg

using namespace vg;

// ------------------------------------------------------------------ CLIP embeddings (clip_embedder.py:190-191)
// out[r][:] = fp16(row(ids[r])[:] + pos[r % L][:]): token_embedding(text) + positional_embedding, fp32 like the
// reference, rounded once.  row(id) = table[id] for id < vocab, else extra[id - vocab] (the learned textual-inversion
// vectors the embedding manager writes over the token embedding, tools/modules/embedding_manager.py:76-116).  Without an
// extra table an id is clamped to the vocabulary; with one the host has range-checked the ids.  One thread per 4 channels.
__global__ void embed_tokens_kernel(const long long* __restrict__ ids, const float* __restrict__ table,
                                    const float* __restrict__ extra, const float* __restrict__ pos, __half* __restrict__ out,
                                    long nrows, int L, int W, long vocab, long n_extra) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const int w4 = W >> 2;
  if (idx >= nrows * w4) return;
  const long r = idx / w4;
  const int c = (int)(idx - r * w4) * 4;
  long id = ids[r];
  const long n = vocab + n_extra;
  id = id < 0 ? 0 : (id >= n ? n - 1 : id);
  const float* row = id < vocab ? table + id * W : extra + (id - vocab) * W;
  const float4 a = __ldg(reinterpret_cast<const float4*>(row + c));
  const float4 b = __ldg(reinterpret_cast<const float4*>(pos + (r % L) * W + c));
  uint2 o;
  o.x = pack_half2(a.x + b.x, a.y + b.y);
  o.y = pack_half2(a.z + b.z, a.w + b.w);
  *reinterpret_cast<uint2*>(out + r * W + c) = o;
}
// x[b][i] = fp16(float(x[b][i]) + add[i]) for i < n: the vision tower's positional embedding broadcast over the batch
__global__ void add_rows_f32_kernel(__half* __restrict__ x, const float* __restrict__ add, long batch, long n) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= batch * n) return;
  x[idx] = __float2half_rn(__half2float(x[idx]) + add[idx % n]);
}

static inline unsigned nblk(long total, int threads) { return (unsigned)((total + threads - 1) / threads); }

extern "C" {

int vgen_attention_cross_small(const void* q, const void* k, const void* v, void* out, int64_t batch, int64_t heads,
                               int64_t lq, int64_t lk, int64_t head_dim, int64_t ldq, int64_t ldk, int64_t ldv, int64_t ldo,
                               int64_t kv_batch_div, int causal, float scale, void* stream) {
  VG_REQUIRE(q && k && v && out, "vgen_attention_cross_small: null pointer");
  VG_REQUIRE(!causal || lk >= lq, "vgen_attention_cross_small: causal needs lk >= lq");
  VG_REQUIRE(batch >= 0 && heads > 0 && lq > 0 && lk > 0 && head_dim > 0 && head_dim <= 256 && kv_batch_div > 0 &&
                 batch % kv_batch_div == 0,
             "vgen_attention_cross_small: bad shape");
  if (batch == 0) return 0;
  const long warps = batch * heads * lq;
  launch_kernel(attn_cross_small_kernel, dim3(nblk(warps * 32, 128)), dim3(128), 0, reinterpret_cast<cudaStream_t>(stream), 
      reinterpret_cast<const __half*>(q), reinterpret_cast<const __half*>(k), reinterpret_cast<const __half*>(v),
      reinterpret_cast<__half*>(out), batch, (int)heads, (int)lq, (int)lk, (int)head_dim, ldq, ldk, ldv, ldo,
      (int)kv_batch_div, scale, causal ? 1 : 0);
  VG_LAUNCH_CHECK("attn_cross_small_kernel");
  return 0;
}

int vgen_interp_linear_rows(const void* x, void* y, int64_t nseq, int64_t lin, int64_t lout, int64_t c, void* stream) {
  VG_REQUIRE(x && y && nseq >= 0 && lin > 0 && lout > 0 && c > 0, "vgen_interp_linear_rows: bad arguments");
  const long total = nseq * lout * c;
  if (total == 0) return 0;
  launch_kernel(interp_linear_rows_kernel, dim3(nblk(total, 256)), dim3(256), 0, reinterpret_cast<cudaStream_t>(stream), 
      reinterpret_cast<const __half*>(x), reinterpret_cast<__half*>(y), nseq, (int)lin, (int)lout, (int)c);
  VG_LAUNCH_CHECK("interp_linear_rows_kernel");
  return 0;
}

int vgen_fourier_lowfreq_filter(const void* x, int64_t ldx, void* y, int64_t ldy, int64_t nimg, int64_t h, int64_t w,
                                int64_t c, float scale, void* stream) {
  VG_REQUIRE(x && y && nimg >= 0 && h >= 2 && w >= 2 && c > 0 && ldx >= c && ldy >= c,
             "vgen_fourier_lowfreq_filter: bad arguments");
  VG_REQUIRE(nimg <= 65535, "vgen_fourier_lowfreq_filter: too many images for one launch");
  if (nimg == 0) return 0;
  const size_t smem = (2 * (h + w) + kFfSlices * 7 * kFfChan) * sizeof(float);
  VG_REQUIRE(smem <= 48 * 1024, "vgen_fourier_lowfreq_filter: plane too large");
  dim3 grid((unsigned)((c + kFfChan - 1) / kFfChan), (unsigned)nimg), block(kFfChan, kFfSlices);
  launch_kernel(fourier_lowfreq_kernel, dim3(grid), dim3(block), smem, reinterpret_cast<cudaStream_t>(stream), 
      reinterpret_cast<const __half*>(x), reinterpret_cast<__half*>(y), (int)h, (int)w, (int)c, ldx, ldy, scale);
  VG_LAUNCH_CHECK("fourier_lowfreq_kernel");
  return 0;
}

int vgen_upsample_nearest2x_rows(const void* x, void* y, int64_t nimg, int64_t h, int64_t w, int64_t c, int64_t row0,
                                 int64_t rows_out, void* stream) {
  VG_REQUIRE(x && y && c % 8 == 0 && row0 >= 0 && rows_out > 0 && row0 + rows_out <= 2 * h,
             "vgen_upsample_nearest2x_rows: bad arguments (C must be a multiple of 8, rows within 2h)");
  const long total = nimg * rows_out * 2 * w * (c / 8);
  if (total == 0) return 0;
  launch_kernel(upsample2x_rows_kernel, dim3(nblk(total, 256)), dim3(256), 0, reinterpret_cast<cudaStream_t>(stream), 
      reinterpret_cast<const __half*>(x), reinterpret_cast<__half*>(y), nimg, (int)h, (int)w, (int)(c / 8), (int)row0,
      (int)rows_out);
  VG_LAUNCH_CHECK("upsample2x_rows_kernel");
  return 0;
}

int vgen_scale_copy2d(const void* src, int64_t lds, void* dst, int64_t ldd, int64_t rows, int64_t cols, float s,
                      void* stream) {
  VG_REQUIRE(src && dst && rows >= 0 && cols > 0 && lds >= cols && ldd >= cols, "vgen_scale_copy2d: bad arguments");
  if (rows == 0) return 0;
  launch_kernel(scale_copy2d_kernel, dim3(nblk(rows * cols, 256)), dim3(256), 0, reinterpret_cast<cudaStream_t>(stream), 
      reinterpret_cast<const __half*>(src), lds, reinterpret_cast<__half*>(dst), ldd, rows, (int)cols, s);
  VG_LAUNCH_CHECK("scale_copy2d_kernel");
  return 0;
}

int vgen_embed_tokens_extra(const int64_t* ids, const float* table, int64_t vocab, const float* extra, int64_t n_extra,
                            const float* pos, void* out, int64_t nrows, int64_t L, int64_t W, void* stream) {
  VG_REQUIRE(ids && table && pos && out && nrows >= 0 && L > 0 && W > 0 && W % 4 == 0 && vocab > 0 && n_extra >= 0 &&
                 (extra != nullptr) == (n_extra > 0),
             "vgen_embed_tokens: bad arguments");
  VG_REQUIRE(((reinterpret_cast<uintptr_t>(table) | reinterpret_cast<uintptr_t>(extra) | reinterpret_cast<uintptr_t>(pos)) &
              15) == 0 && (reinterpret_cast<uintptr_t>(out) & 7) == 0,
             "vgen_embed_tokens: table / extra / pos must be 16-byte aligned");
  if (nrows == 0) return 0;
  launch_kernel(embed_tokens_kernel, dim3(nblk(nrows * (W / 4), 256)), dim3(256), 0, reinterpret_cast<cudaStream_t>(stream),
                reinterpret_cast<const long long*>(ids), table, extra, pos, reinterpret_cast<__half*>(out), nrows, (int)L,
                (int)W, vocab, n_extra);
  VG_LAUNCH_CHECK("embed_tokens_kernel");
  return 0;
}

int vgen_embed_tokens(const int64_t* ids, const float* table, const float* pos, void* out, int64_t nrows, int64_t L, int64_t W,
                      int64_t vocab, void* stream) {
  return vgen_embed_tokens_extra(ids, table, vocab, nullptr, 0, pos, out, nrows, L, W, stream);
}

int vgen_add_rows_f32(void* x, const float* add, int64_t batch, int64_t n, void* stream) {
  VG_REQUIRE(x && add && batch >= 0 && n > 0, "vgen_add_rows_f32: bad arguments");
  if (batch == 0) return 0;
  launch_kernel(add_rows_f32_kernel, dim3(nblk(batch * n, 256)), dim3(256), 0, reinterpret_cast<cudaStream_t>(stream),
                reinterpret_cast<__half*>(x), add, batch, n);
  VG_LAUNCH_CHECK("add_rows_f32_kernel");
  return 0;
}

}  // extern "C"
