// Data-movement and pointwise kernels of the hot path (all HBM-bound, 16-byte vectorised where the
// channel count allows): layout conversion at the model boundary, im2col for the few convs the TMA
// tap-GEMM cannot express (stride 2, C % 64 != 0), nearest-neighbour upsampling, channel concat,
// small linears (timestep MLPs), sinusoidal embedding, row softmax (VAE attention), adaptive average
// pooling, and the fused classifier-free-guidance + DDIM update.
#include "common.h"
#include "ptx.cuh"

namespace vg {

__device__ __forceinline__ float silu_e(float v) { return __fdividef(v, 1.0f + __expf(-v)); }

// ------------------------------------------------------------------ layout: [n][c][p] <-> [n][p][c]
// boundary of MODEL.forward: x arrives as fp32 [b, c, f, h, w] (reference layout, unet_t2v.py:257) and
// the result leaves as fp16 [b, c, f, h, w] (:276).  Inside, everything is channels-last.
template <typename Tin>
__global__ void cp_to_pc_kernel(const Tin* __restrict__ x, __half* __restrict__ y, long n, int c, long p, int c_pad) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * p * c_pad) return;
  const int ci = (int)(idx % c_pad);
  const long pi = (idx / c_pad) % p;
  const long ni = idx / ((long)c_pad * p);
  float v = 0.f;
  if (ci < c) v = (float)x[(ni * c + ci) * p + pi];
  y[idx] = __float2half_rn(v);
}
template <typename Tout>
__global__ void pc_to_cp_kernel(const __half* __restrict__ x, Tout* __restrict__ y, long n, int c, long p, long ldx) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * p * c) return;
  const long pi = idx % p;
  const int ci = (int)((idx / p) % c);
  const long ni = idx / (p * c);
  y[idx] = (Tout)__half2float(x[(ni * p + pi) * ldx + ci]);
}
template <>
__global__ void pc_to_cp_kernel<__half>(const __half* __restrict__ x, __half* __restrict__ y, long n, int c, long p, long ldx) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * p * c) return;
  const long pi = idx % p;
  const int ci = (int)((idx / p) % c);
  const long ni = idx / (p * c);
  y[idx] = x[(ni * p + pi) * ldx + ci];
}

// ------------------------------------------------------------------ im2col (channels-last gather)
// out[(n,oy,ox)][(ky*kw+kx)*c + ci] = act(x[n][oy*s-pt+ky][ox*s-pl+kx][ci]); columns >= kh*kw*c are zero.
__global__ void im2col_kernel(const __half* __restrict__ x, __half* __restrict__ out, long nimg, int h, int w, int c,
                              int kh, int kw, int stride, int pad_t, int pad_l, int ho, int wo, int kpad, int act_silu) {
  const bool vec = (c % 8 == 0);
  const int kv = vec ? kpad / 8 : kpad;
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const long rows = nimg * ho * wo;
  if (idx >= rows * kv) return;
  const int kk = (int)(idx % kv);
  const long row = idx / kv;
  const int ox = (int)(row % wo);
  const int oy = (int)((row / wo) % ho);
  const long n = row / ((long)wo * ho);
  if (vec) {
    const int k0 = kk * 8;
    uint4 u = make_uint4(0, 0, 0, 0);
    if (k0 < kh * kw * c) {
      const int tap = k0 / c, ci = k0 - tap * c;
      const int ky = tap / kw, kx = tap - ky * kw;
      const int iy = oy * stride - pad_t + ky, ix = ox * stride - pad_l + kx;
      if (iy >= 0 && iy < h && ix >= 0 && ix < w) {
        u = __ldg(reinterpret_cast<const uint4*>(x + ((n * h + iy) * w + ix) * c + ci));
        if (act_silu) {
          __half2* h2 = reinterpret_cast<__half2*>(&u);
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            float2 f = __half22float2(h2[i]);
            h2[i] = __floats2half2_rn(silu_e(f.x), silu_e(f.y));
          }
        }
      }
    }
    *reinterpret_cast<uint4*>(out + row * kpad + k0) = u;
  } else {
    float v = 0.f;
    if (kk < kh * kw * c) {
      const int tap = kk / c, ci = kk - tap * c;
      const int ky = tap / kw, kx = tap - ky * kw;
      const int iy = oy * stride - pad_t + ky, ix = ox * stride - pad_l + kx;
      if (iy >= 0 && iy < h && ix >= 0 && ix < w) {
        v = __half2float(x[((n * h + iy) * w + ix) * c + ci]);
        if (act_silu) v = silu_e(v);
      }
    }
    out[row * kpad + kk] = __float2half_rn(v);
  }
}

// ------------------------------------------------------------------ nearest x2 upsample (channels-last)
__global__ void upsample2x_kernel(const __half* __restrict__ x, __half* __restrict__ y, long nimg, int h, int w, int c8) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const long total = nimg * (2L * h) * (2L * w) * c8;
  if (idx >= total) return;
  const int cv = (int)(idx % c8);
  const long pix = idx / c8;
  const int ox = (int)(pix % (2 * w));
  const int oy = (int)((pix / (2 * w)) % (2 * h));
  const long n = pix / (4L * w * h);
  const uint4 u = __ldg(reinterpret_cast<const uint4*>(x) + ((n * h + (oy >> 1)) * w + (ox >> 1)) * c8 + cv);
  reinterpret_cast<uint4*>(y)[idx] = u;
}

// ------------------------------------------------------------------ 2-D strided copy (channel concat)
__global__ void copy2d_kernel(const __half* __restrict__ src, long lds, __half* __restrict__ dst, long ldd, long rows,
                              int cols) {
  const bool vec = (cols % 8 == 0) && (lds % 8 == 0) && (ldd % 8 == 0) &&
                   (((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15) == 0);
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (vec) {
    const int cv = cols / 8;
    if (idx >= rows * cv) return;
    const long r = idx / cv;
    const int c = (int)(idx % cv) * 8;
    *reinterpret_cast<uint4*>(dst + r * ldd + c) = __ldg(reinterpret_cast<const uint4*>(src + r * lds + c));
  } else {
    if (idx >= rows * cols) return;
    const long r = idx / cols;
    const int c = (int)(idx % cols);
    dst[r * ldd + c] = src[r * lds + c];
  }
}

// ------------------------------------------------------------------ pointwise ops
// op: 0 silu(a)  1 a+b  2 gelu(a) (erf)  3 a*s  4 a + s*b  5 relu(a)
__global__ void eltwise_kernel(const __half* __restrict__ a, const __half* __restrict__ b, __half* __restrict__ y, long n,
                               int op, float s) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  const float x = __half2float(a[idx]);
  float r;
  switch (op) {
    case 0: r = silu_e(x); break;
    case 1: r = x + __half2float(b[idx]); break;
    case 2: r = 0.5f * x * (1.0f + erff(x * 0.70710678118654752f)); break;
    case 3: r = x * s; break;
    case 4: r = x + s * __half2float(b[idx]); break;
    default: r = x < 0.f ? 0.f : x; break;  // NaN passes through, as in torch.relu
  }
  y[idx] = __float2half_rn(r);
}
// op 6: QuickGELU x * sigmoid(1.702 x) (OpenAI CLIP's activation, open_clip transformer.py QuickGELU); its own kernel, so
// the ops above keep their code
__global__ void quick_gelu_kernel(const __half* __restrict__ a, __half* __restrict__ y, long n) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  const float x = __half2float(a[idx]);
  y[idx] = __float2half_rn(x / (1.0f + expf(-1.702f * x)));
}

// ------------------------------------------------------------------ small linear (M rows small or K tiny)
// out[m][n] = (act_in(a[m][:]) . w[n][:] + bias[n]) (+ res[m][n]); one warp per output element.
__global__ void linear_small_kernel(const __half* __restrict__ a, long lda, const __half* __restrict__ w,
                                    const float* __restrict__ bias, const __half* __restrict__ res, long ldr,
                                    __half* __restrict__ out, long ldo, long m, int n, int k, int silu_in, int gelu_out) {
  const long warp_id = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp_id >= m * n) return;
  const long mi = warp_id / n;
  const int ni = (int)(warp_id % n);
  const __half* ar = a + mi * lda;
  const __half* wr = w + (long)ni * k;
  float acc = 0.f;
  for (int c = lane; c < k; c += 32) {
    float x = __half2float(ar[c]);
    if (silu_in) x = __half2float(__float2half_rn(silu_e(x)));
    acc += x * __half2float(wr[c]);
  }
  acc = warp_sum(acc);
  if (lane == 0) {
    if (bias) acc += bias[ni];
    if (gelu_out) {
      const float h = __half2float(__float2half_rn(acc));
      acc = 0.5f * h * (1.0f + erff(h * 0.70710678118654752f));
    }
    if (res) acc = __half2float(__float2half_rn(acc)) + __half2float(res[mi * ldr + ni]);
    out[mi * ldo + ni] = __float2half_rn(acc);
  }
}
// K tiny (<= 32): one thread per output element
__global__ void linear_tinyk_kernel(const __half* __restrict__ a, long lda, const __half* __restrict__ w,
                                    const float* __restrict__ bias, const __half* __restrict__ res, long ldr,
                                    __half* __restrict__ out, long ldo, long m, int n, int k, int silu_in, int gelu_out) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= m * n) return;
  const long mi = idx / n;
  const int ni = (int)(idx % n);
  float acc = 0.f;
  for (int c = 0; c < k; ++c) {
    float x = __half2float(a[mi * lda + c]);
    if (silu_in) x = __half2float(__float2half_rn(silu_e(x)));
    acc += x * __half2float(w[(long)ni * k + c]);
  }
  if (bias) acc += bias[ni];
  if (gelu_out) {
    const float h = __half2float(__float2half_rn(acc));
    acc = 0.5f * h * (1.0f + erff(h * 0.70710678118654752f));
  }
  if (res) acc = __half2float(__float2half_rn(acc)) + __half2float(res[mi * ldr + ni]);
  out[mi * ldo + ni] = __float2half_rn(acc);
}

// ------------------------------------------------------------------ sinusoidal embedding
// tools/modules/unet/util.py:178-190: outer(t, 10000^(-i/half)), cat[cos, sin]; fp32 math, fp16 store
__global__ void sinusoidal_kernel(const float* __restrict__ t, __half* __restrict__ out, int b, int dim) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int half = dim / 2;
  if (idx >= b * half) return;
  const int i = idx % half, bi = idx / half;
  const float freq = powf(10000.0f, -((float)i / (float)half));
  const float ang = t[bi] * freq;
  out[(long)bi * dim + i] = __float2half_rn(cosf(ang));
  out[(long)bi * dim + half + i] = __float2half_rn(sinf(ang));
}

// ------------------------------------------------------------------ row softmax (in place, fp16 rows)
__global__ void __launch_bounds__(256) softmax_rows_kernel(__half* __restrict__ x, long ld, int n, float scale) {
  __shared__ float red[8];
  __half* row = x + (long)blockIdx.x * ld;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  float mx = -INFINITY;
  for (int i = tid; i < n; i += 256) mx = fmaxf(mx, __half2float(row[i]));
  mx = warp_max(mx);
  if (lane == 0) red[wid] = mx;
  __syncthreads();
  mx = red[0];
#pragma unroll
  for (int i = 1; i < 8; ++i) mx = fmaxf(mx, red[i]);
  __syncthreads();
  float s = 0.f;
  for (int i = tid; i < n; i += 256) s += __expf((__half2float(row[i]) - mx) * scale);
  s = warp_sum(s);
  if (lane == 0) red[wid] = s;
  __syncthreads();
  s = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) s += red[i];
  const float inv = 1.0f / s;
  for (int i = tid; i < n; i += 256) row[i] = __float2half_rn(__expf((__half2float(row[i]) - mx) * scale) * inv);
}

// ------------------------------------------------------------------ adaptive average pool (channels-last)
__global__ void adaptive_avgpool_kernel(const __half* __restrict__ x, __half* __restrict__ y, long nimg, int h, int w, int c,
                                        int oh, int ow, int silu_in) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= nimg * oh * ow * c) return;
  const int ci = (int)(idx % c);
  const int ox = (int)((idx / c) % ow);
  const int oy = (int)((idx / ((long)c * ow)) % oh);
  const long n = idx / ((long)c * ow * oh);
  // torch: start = floor(o*in/out), end = ceil((o+1)*in/out)
  const int y0 = (oy * h) / oh, y1 = ((oy + 1) * h + oh - 1) / oh;
  const int x0 = (ox * w) / ow, x1 = ((ox + 1) * w + ow - 1) / ow;
  float s = 0.f;
  for (int yy = y0; yy < y1; ++yy)
    for (int xx = x0; xx < x1; ++xx) {
      float v = __half2float(x[((n * h + yy) * w + xx) * c + ci]);
      if (silu_in) v = __half2float(__float2half_rn(silu_e(v)));
      s += v;
    }
  y[idx] = __float2half_rn(s / (float)((y1 - y0) * (x1 - x0)));
}

// ------------------------------------------------------------------ fused CFG + DDIM update
// diffusion_ddim.py:157-162 (classifier-free mix, done in the model's fp16 like the reference under
// autocast), :194-196 (v -> x0), :230-240 (eps, x_{t-1}); xt stays fp32.  y/u: model outputs in the
// reference layout [b, c, f, h, w] fp16.  coef = {sqrt_ab, sqrt_1m_ab, sqrt_recip_ab, sqrt_recipm1_ab,
// sqrt_ab_prev, dir_coef, sigma*mask} already cast to fp32 like _i() does.
struct DdimCoef {
  float c[8];
};
__global__ void ddim_step_kernel(float* __restrict__ xt, const __half* __restrict__ y, const __half* __restrict__ u,
                                 const float* __restrict__ noise, long n, float guide, int has_u, DdimCoef k, int mean_v,
                                 float* __restrict__ x0_out) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  float out;
  if (has_u) {
    const __half yh = y[idx], uh = u[idx];
    const __half d = __float2half_rn(__half2float(yh) - __half2float(uh));   // fp16 tensor ops round each step
    const __half gd = __float2half_rn(guide * __half2float(d));
    out = __half2float(__float2half_rn(__half2float(uh) + __half2float(gd)));
  } else {
    out = __half2float(y[idx]);
  }
  const float x = xt[idx];
  float x0;
  if (mean_v)
    x0 = k.c[0] * x - k.c[1] * out;
  else
    x0 = k.c[2] * x - k.c[3] * out;
  const float eps = (k.c[2] * x - x0) / k.c[3];
  float r = k.c[4] * x0 + k.c[5] * eps;
  if (noise) r += k.c[6] * noise[idx];
  xt[idx] = r;
  if (x0_out) x0_out[idx] = x0;
}

// ------------------------------------------------------------------ VAE posterior sample
// DiagonalGaussianDistribution.sample (autoencoder.py:211-225): moments [n][p][2*zc] fp16 channels-last
// (mean | logvar), logvar clamped to [-30, 20], z = (mean + exp(0.5*logvar) * noise) * scale; noise and z are
// fp32 in the reference layout [n][zc][p].
__global__ void vae_sample_kernel(const __half* __restrict__ mom, const float* __restrict__ noise, float* __restrict__ z,
                                  long n, int zc, long p, float scale) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * zc * p) return;
  const long pi = idx % p;
  const int ci = (int)((idx / p) % zc);
  const long ni = idx / (p * zc);
  const __half* m = mom + (ni * p + pi) * (2 * zc);
  const float mean = __half2float(m[ci]);
  float lv = __half2float(m[zc + ci]);
  lv = fminf(fmaxf(lv, -30.0f), 20.0f);
  z[idx] = (mean + expf(0.5f * lv) * noise[idx]) * scale;
}

static inline unsigned nblk(long total, int threads) { return (unsigned)((total + threads - 1) / threads); }

}  // namespace vg

using namespace vg;

extern "C" {

int vgen_cp_to_pc(const void* x, int x_is_f32, void* y, int64_t n, int64_t c, int64_t p, int64_t c_pad, void* stream) {
  VG_REQUIRE(x && y && n >= 0 && c > 0 && p > 0 && c_pad >= c, "vgen_cp_to_pc: bad arguments");
  const long total = n * p * c_pad;
  if (total == 0) return 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (x_is_f32)
    launch_kernel(cp_to_pc_kernel<float>, dim3(nblk(total, 256)), dim3(256), 0, st, reinterpret_cast<const float*>(x), reinterpret_cast<__half*>(y), n, (int)c, p, (int)c_pad);
  else
    launch_kernel(cp_to_pc_kernel<__half>, dim3(nblk(total, 256)), dim3(256), 0, st, reinterpret_cast<const __half*>(x), reinterpret_cast<__half*>(y), n, (int)c, p, (int)c_pad);
  VG_LAUNCH_CHECK("cp_to_pc_kernel");
  return 0;
}

int vgen_pc_to_cp(const void* x, int64_t ldx, void* y, int y_is_f32, int64_t n, int64_t c, int64_t p, void* stream) {
  VG_REQUIRE(x && y && n >= 0 && c > 0 && p > 0 && ldx >= c, "vgen_pc_to_cp: bad arguments");
  const long total = n * p * c;
  if (total == 0) return 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (y_is_f32)
    launch_kernel(pc_to_cp_kernel<float>, dim3(nblk(total, 256)), dim3(256), 0, st, reinterpret_cast<const __half*>(x), reinterpret_cast<float*>(y), n, (int)c, p, ldx);
  else
    launch_kernel(pc_to_cp_kernel<__half>, dim3(nblk(total, 256)), dim3(256), 0, st, reinterpret_cast<const __half*>(x), reinterpret_cast<__half*>(y), n, (int)c, p, ldx);
  VG_LAUNCH_CHECK("pc_to_cp_kernel");
  return 0;
}

int vgen_im2col(const void* x, void* out, int64_t nimg, int64_t h, int64_t w, int64_t c, int64_t kh, int64_t kw,
                int64_t stride, int64_t pad_t, int64_t pad_l, int64_t ho, int64_t wo, int64_t kpad, int act_silu, void* stream) {
  VG_REQUIRE(x && out && nimg >= 0 && h > 0 && w > 0 && c > 0 && kh > 0 && kw > 0 && stride > 0 && ho > 0 && wo > 0 &&
                 kpad >= kh * kw * c,
             "vgen_im2col: bad arguments");
  if (c % 8 == 0) VG_REQUIRE(kpad % 8 == 0, "vgen_im2col: kpad must be a multiple of 8");
  const long rows = nimg * ho * wo;
  const long total = rows * (c % 8 == 0 ? kpad / 8 : kpad);
  if (total == 0) return 0;
  launch_kernel(im2col_kernel, dim3(nblk(total, 256)), dim3(256), 0, reinterpret_cast<cudaStream_t>(stream), 
      reinterpret_cast<const __half*>(x), reinterpret_cast<__half*>(out), nimg, (int)h, (int)w, (int)c, (int)kh, (int)kw,
      (int)stride, (int)pad_t, (int)pad_l, (int)ho, (int)wo, (int)kpad, act_silu);
  VG_LAUNCH_CHECK("im2col_kernel");
  return 0;
}

int vgen_upsample_nearest2x(const void* x, void* y, int64_t nimg, int64_t h, int64_t w, int64_t c, void* stream) {
  VG_REQUIRE(x && y && c % 8 == 0, "vgen_upsample_nearest2x: C must be a multiple of 8");
  const long total = nimg * 4 * h * w * (c / 8);
  if (total == 0) return 0;
  launch_kernel(upsample2x_kernel, dim3(nblk(total, 256)), dim3(256), 0, reinterpret_cast<cudaStream_t>(stream), 
      reinterpret_cast<const __half*>(x), reinterpret_cast<__half*>(y), nimg, (int)h, (int)w, (int)(c / 8));
  VG_LAUNCH_CHECK("upsample2x_kernel");
  return 0;
}

int vgen_copy2d(const void* src, int64_t lds, void* dst, int64_t ldd, int64_t rows, int64_t cols, void* stream) {
  VG_REQUIRE(src && dst && rows >= 0 && cols > 0 && (lds >= cols || lds == 0) && ldd >= cols, "vgen_copy2d: bad arguments");
  if (rows == 0) return 0;
  const bool vec = (cols % 8 == 0) && (lds % 8 == 0) && (ldd % 8 == 0) &&
                   (((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15) == 0);
  const long total = vec ? rows * (cols / 8) : rows * cols;
  launch_kernel(copy2d_kernel, dim3(nblk(total, 256)), dim3(256), 0, reinterpret_cast<cudaStream_t>(stream), 
      reinterpret_cast<const __half*>(src), lds, reinterpret_cast<__half*>(dst), ldd, rows, (int)cols);
  VG_LAUNCH_CHECK("copy2d_kernel");
  return 0;
}

int vgen_eltwise(int op, const void* a, const void* b, void* y, int64_t n, float s, void* stream) {
  VG_REQUIRE(a && y && op >= 0 && op <= 6, "vgen_eltwise: bad arguments");
  VG_REQUIRE(!(op == 1 || op == 4) || b, "vgen_eltwise: binary op needs b");
  if (n == 0) return 0;
  if (op == 6) {
    launch_kernel(quick_gelu_kernel, dim3(nblk(n, 256)), dim3(256), 0, reinterpret_cast<cudaStream_t>(stream),
                  reinterpret_cast<const __half*>(a), reinterpret_cast<__half*>(y), n);
    VG_LAUNCH_CHECK("quick_gelu_kernel");
    return 0;
  }
  launch_kernel(eltwise_kernel, dim3(nblk(n, 256)), dim3(256), 0, reinterpret_cast<cudaStream_t>(stream), 
      reinterpret_cast<const __half*>(a), reinterpret_cast<const __half*>(b), reinterpret_cast<__half*>(y), n, op, s);
  VG_LAUNCH_CHECK("eltwise_kernel");
  return 0;
}

int vgen_linear_small(const void* a, int64_t m, int64_t k, int64_t lda, const void* w, const float* bias, int64_t n,
                      const void* res, int64_t ldr, void* out, int64_t ldo, int silu_in, int gelu_out, void* stream) {
  VG_REQUIRE(a && w && out && m >= 0 && k > 0 && n > 0, "vgen_linear_small: bad arguments");
  if (m == 0) return 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (k <= 32) {
    launch_kernel(linear_tinyk_kernel, dim3(nblk(m * n, 256)), dim3(256), 0, st, reinterpret_cast<const __half*>(a), lda, reinterpret_cast<const __half*>(w),
                                                         bias, reinterpret_cast<const __half*>(res), ldr,
                                                         reinterpret_cast<__half*>(out), ldo, m, (int)n, (int)k, silu_in, gelu_out);
    VG_LAUNCH_CHECK("linear_tinyk_kernel");
  } else {
    launch_kernel(linear_small_kernel, dim3(nblk(m * n * 32, 256)), dim3(256), 0, st, reinterpret_cast<const __half*>(a), lda, reinterpret_cast<const __half*>(w),
                                                              bias, reinterpret_cast<const __half*>(res), ldr,
                                                              reinterpret_cast<__half*>(out), ldo, m, (int)n, (int)k, silu_in, gelu_out);
    VG_LAUNCH_CHECK("linear_small_kernel");
  }
  return 0;
}

int vgen_sinusoidal_embedding(const float* t, void* out, int64_t b, int64_t dim, void* stream) {
  VG_REQUIRE(t && out && b > 0 && dim > 0 && dim % 2 == 0, "vgen_sinusoidal_embedding: bad arguments");
  launch_kernel(sinusoidal_kernel, dim3(nblk(b * dim / 2, 128)), dim3(128), 0, reinterpret_cast<cudaStream_t>(stream), t, reinterpret_cast<__half*>(out), (int)b, (int)dim);
  VG_LAUNCH_CHECK("sinusoidal_kernel");
  return 0;
}

int vgen_softmax_rows(void* x, int64_t rows, int64_t n, int64_t ld, float scale, void* stream) {
  VG_REQUIRE(x && rows >= 0 && n > 0 && ld >= n, "vgen_softmax_rows: bad arguments");
  if (rows == 0) return 0;
  launch_kernel(softmax_rows_kernel, dim3((unsigned)rows), dim3(256), 0, reinterpret_cast<cudaStream_t>(stream), reinterpret_cast<__half*>(x), ld, (int)n, scale);
  VG_LAUNCH_CHECK("softmax_rows_kernel");
  return 0;
}

int vgen_adaptive_avgpool(const void* x, void* y, int64_t nimg, int64_t h, int64_t w, int64_t c, int64_t oh, int64_t ow,
                          int silu_in, void* stream) {
  VG_REQUIRE(x && y && h > 0 && w > 0 && c > 0 && oh > 0 && ow > 0, "vgen_adaptive_avgpool: bad arguments");
  const long total = nimg * oh * ow * c;
  if (total == 0) return 0;
  launch_kernel(adaptive_avgpool_kernel, dim3(nblk(total, 256)), dim3(256), 0, reinterpret_cast<cudaStream_t>(stream), 
      reinterpret_cast<const __half*>(x), reinterpret_cast<__half*>(y), nimg, (int)h, (int)w, (int)c, (int)oh, (int)ow, silu_in);
  VG_LAUNCH_CHECK("adaptive_avgpool_kernel");
  return 0;
}

int vgen_vae_sample(const void* moments, const float* noise, float* z, int64_t n, int64_t zc, int64_t p, float scale,
                    void* stream) {
  VG_REQUIRE(moments && noise && z && n >= 0 && zc > 0 && p > 0, "vgen_vae_sample: bad arguments");
  const long total = n * zc * p;
  if (total == 0) return 0;
  launch_kernel(vae_sample_kernel, dim3(nblk(total, 256)), dim3(256), 0, reinterpret_cast<cudaStream_t>(stream), 
      reinterpret_cast<const __half*>(moments), noise, z, n, (int)zc, p, scale);
  VG_LAUNCH_CHECK("vae_sample_kernel");
  return 0;
}

int vgen_ddim_step(float* xt, const void* y, const void* u, const float* noise, int64_t n, float guide_scale,
                   const float* coef7, int mean_type_v, float* x0_out, void* stream) {
  VG_REQUIRE(xt && y && coef7 && n >= 0, "vgen_ddim_step: bad arguments");
  if (n == 0) return 0;
  DdimCoef k;
  for (int i = 0; i < 7; ++i) k.c[i] = coef7[i];
  k.c[7] = 0.f;
  launch_kernel(ddim_step_kernel, dim3(nblk(n, 256)), dim3(256), 0, reinterpret_cast<cudaStream_t>(stream), 
      xt, reinterpret_cast<const __half*>(y), reinterpret_cast<const __half*>(u), noise, n, guide_scale, u != nullptr, k,
      mean_type_v, x0_out);
  VG_LAUNCH_CHECK("ddim_step_kernel");
  return 0;
}

}  // extern "C"
