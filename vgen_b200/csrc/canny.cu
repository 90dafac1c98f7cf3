// The VideoComposer canny annotator (tools/annotator/canny/__init__.py CannyDetector: cv2.convertScaleAbs, a median
// threshold, cv2.Canny with aperture 3 and the L1 gradient), device side, for n frames per call.
//
// 1. canny_quantise_kernel: each sample to a byte, |x * 255| rounded to nearest even and saturated (convertScaleAbs of the
//    fp32 frame), or the uint8 sample as it is; planar bytes [n][c][h][w] and a 256-bin histogram per frame.
// 2. canny_threshold_kernel: one block per frame: the exact median of the frame's h * w * c bytes from its histogram
//    (the float64 mean of the two middle values for an even count, as np.median), then the frame's thresholds in
//    float64: explicit, (1 -/+ 0.33) * median, or (1 - r) * median and twice that with the host-drawn r.  Then cv2.Canny's
//    own rule: swap if low > high, floor to integers.
// 3. canny_gradient_kernel: a 32 x 16 tile with a 2-pixel halo of bytes in shared memory: 3x3 Sobel with replicated
//    borders (int), per pixel the channel with the strictly largest |dx| + |dy|, the L1 magnitude on the tile plus a
//    1-pixel ring (0 outside the image), non-maximum suppression with the Q15 tan(22.5 deg) direction test, and the
//    class: 0 no edge, 1 candidate (m > low), 2 strong (m > high).  It also starts the union-find: label = the pixel's
//    own index for a candidate, -1 otherwise.
// 4. Hysteresis as connected-component labelling over the candidates (8-connectivity): canny_merge_kernel joins every
//    candidate with its candidate neighbours above and to the left (lock-free union-find, the smaller index becomes the
//    root), canny_flatten_kernel points every candidate at its root and marks the roots of components holding a strong
//    pixel, canny_output_kernel writes 1.0 for candidates of marked components and 0.0 elsewhere.  The launch count is
//    fixed; a weak chain of any length is joined by the union-find, not by repeated propagation.
#include <algorithm>

#include "common.h"

namespace vg {

constexpr int CN_TX = 32, CN_TY = 16, CN_THREADS = 256;
constexpr int CN_BX = CN_TX + 4, CN_BY = CN_TY + 4;      // bytes: tile + 2-pixel halo
constexpr int CN_MX = CN_TX + 2, CN_MY = CN_TY + 2;      // magnitude: tile + 1-pixel ring
constexpr int CN_TG22 = 13573;                           // round(tan(22.5 deg) * 2^15)

struct CannySrc {
  const void* p;
  int u8;
  long s_n, s_c, s_y, s_x;                               // element strides
};

__global__ void __launch_bounds__(CN_THREADS) canny_quantise_kernel(CannySrc s, int c, int h, int w,
                                                                    uint8_t* __restrict__ bytes, int* __restrict__ hist) {
  __shared__ int bins[256];
  const int img = blockIdx.y;
  const long P = (long)h * w, total = P * c;
  for (int i = threadIdx.x; i < 256; i += CN_THREADS) bins[i] = 0;
  __syncthreads();
  const long base = (long)img * s.s_n;
  for (long i = (long)blockIdx.x * CN_THREADS + threadIdx.x; i < total; i += (long)gridDim.x * CN_THREADS) {
    const int ch = (int)(i / P);
    const long p = i - (long)ch * P;
    const int y = (int)(p / w), x = (int)(p - (long)y * w);
    const long off = base + ch * s.s_c + y * s.s_y + x * s.s_x;
    int v;
    if (s.u8) {
      v = __ldg(reinterpret_cast<const uint8_t*>(s.p) + off);
    } else {
      // convertScaleAbs(img * 255.): an fp32 product, |.|, cvRound (nearest even), saturate; NaN -> 0
      v = __float2int_rn(fabsf(__fmul_rn(__ldg(reinterpret_cast<const float*>(s.p) + off), 255.0f)));
      v = min(max(v, 0), 255);
    }
    bytes[(long)img * total + i] = (uint8_t)v;
    atomicAdd(&bins[v], 1);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 256; i += CN_THREADS)
    if (bins[i]) atomicAdd(hist + img * 256 + i, bins[i]);
}

// mode 0: explicit (lo, hi); 1: (1 - 0.33) * m, (1 + 0.33) * m; 2: (1 - r[img]) * m and twice that.
// thr [n][2] = the integer (low, high) the magnitude is compared with.
__global__ void __launch_bounds__(256) canny_threshold_kernel(const int* __restrict__ hist, long count, int mode,
                                                              const double* __restrict__ r, double lo, double hi,
                                                              int* __restrict__ thr) {
  __shared__ long cum[256];
  __shared__ int mid[2];
  const int img = blockIdx.x, t = threadIdx.x;
  const int own = hist[img * 256 + t];
  cum[t] = own;
  __syncthreads();
  for (int d = 1; d < 256; d <<= 1) {                    // inclusive scan
    const long add = t >= d ? cum[t - d] : 0;
    __syncthreads();
    cum[t] += add;
    __syncthreads();
  }
  const long k[2] = {(count - 1) / 2, count / 2};        // the middle ranks (equal for an odd count)
  const long before = cum[t] - own;
#pragma unroll
  for (int q = 0; q < 2; ++q)
    if (before <= k[q] && k[q] < cum[t]) mid[q] = t;
  __syncthreads();
  if (t != 0) return;
  const double m = __ddiv_rn((double)(mid[0] + mid[1]), 2.0);
  double low = lo, high = hi;
  if (mode == 1) {
    low = trunc(fmax(0.0, __dmul_rn(1.0 - 0.33, m)));
    high = trunc(fmin(255.0, __dmul_rn(1.0 + 0.33, m)));
  } else if (mode == 2) {
    low = trunc(fmax(0.0, __dmul_rn(__dsub_rn(1.0, __ldg(r + img)), m)));
    high = 2.0 * low;
  }
  if (low > high) {
    const double x = low;
    low = high, high = x;
  }
  // the L1 magnitude lies in [0, 2040]: clamping the floors to [-1, 2040] keeps every comparison m > low / m > high
  thr[2 * img] = (int)fmin(fmax(floor(low), -1.0), 2040.0);
  thr[2 * img + 1] = (int)fmin(fmax(floor(high), -1.0), 2040.0);
}

__global__ void __launch_bounds__(CN_THREADS) canny_gradient_kernel(const uint8_t* __restrict__ bytes, int c, int h, int w,
                                                                    const int* __restrict__ thr, uint8_t* __restrict__ cls,
                                                                    int* __restrict__ label, uint8_t* __restrict__ keep) {
  __shared__ uint8_t b[3][CN_BY][CN_BX];
  __shared__ int mag[CN_MY][CN_MX];
  __shared__ short gx[CN_TY][CN_TX], gy[CN_TY][CN_TX];
  const int img = blockIdx.z;
  const int x0 = blockIdx.x * CN_TX, y0 = blockIdx.y * CN_TY;
  const long P = (long)h * w;
  const uint8_t* src = bytes + (long)img * c * P;
  for (int i = threadIdx.x; i < c * CN_BY * CN_BX; i += CN_THREADS) {
    const int ch = i / (CN_BY * CN_BX), r = i - ch * (CN_BY * CN_BX);
    const int ty = r / CN_BX, tx = r - ty * CN_BX;
    const int y = min(max(y0 - 2 + ty, 0), h - 1), x = min(max(x0 - 2 + tx, 0), w - 1);   // replicated border
    b[ch][ty][tx] = __ldg(src + ch * P + (long)y * w + x);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < CN_MY * CN_MX; i += CN_THREADS) {
    const int ty = i / CN_MX, tx = i - ty * CN_MX;
    const int y = y0 - 1 + ty, x = x0 - 1 + tx;
    int best = 0, bdx = 0, bdy = 0;
    if (y >= 0 && y < h && x >= 0 && x < w) {
      for (int ch = 0; ch < c; ++ch) {
        const uint8_t(*q)[CN_BX] = b[ch];
        const int a00 = q[ty][tx], a01 = q[ty][tx + 1], a02 = q[ty][tx + 2];
        const int a10 = q[ty + 1][tx], a12 = q[ty + 1][tx + 2];
        const int a20 = q[ty + 2][tx], a21 = q[ty + 2][tx + 1], a22 = q[ty + 2][tx + 2];
        const int dx = (a02 + 2 * a12 + a22) - (a00 + 2 * a10 + a20);
        const int dy = (a20 + 2 * a21 + a22) - (a00 + 2 * a01 + a02);
        const int m = abs(dx) + abs(dy);
        if (ch == 0 || m > best) best = m, bdx = dx, bdy = dy;
      }
    }
    mag[ty][tx] = best;                                   // 0 outside the image
    if (ty >= 1 && ty <= CN_TY && tx >= 1 && tx <= CN_TX) gx[ty - 1][tx - 1] = (short)bdx, gy[ty - 1][tx - 1] = (short)bdy;
  }
  __syncthreads();
  const int low = __ldg(thr + 2 * img), high = __ldg(thr + 2 * img + 1);
  for (int i = threadIdx.x; i < CN_TY * CN_TX; i += CN_THREADS) {
    const int ty = i / CN_TX, tx = i - ty * CN_TX;
    const int y = y0 + ty, x = x0 + tx;
    if (y >= h || x >= w) continue;
    const int my = ty + 1, mx = tx + 1;
    const int m = mag[my][mx];
    int k = 0;
    if (m > low) {
      const int dx = gx[ty][tx], dy = gy[ty][tx];
      const int ax = abs(dx), ay = abs(dy) << 15;
      const int tg22 = ax * CN_TG22;
      bool peak;
      if (ay < tg22) {                                    // near-horizontal gradient: left / right neighbours
        peak = m > mag[my][mx - 1] && m >= mag[my][mx + 1];
      } else if (ay > tg22 + (ax << 16)) {                // near-vertical: above / below
        peak = m > mag[my - 1][mx] && m >= mag[my + 1][mx];
      } else {                                            // diagonal, along the gradient's sign
        const int sg = (dx ^ dy) < 0 ? -1 : 1;
        peak = m > mag[my - 1][mx - sg] && m > mag[my + 1][mx + sg];
      }
      if (peak) k = m > high ? 2 : 1;
    }
    const long p = (long)y * w + x;
    cls[(long)img * P + p] = (uint8_t)k;
    label[(long)img * P + p] = k ? (int)p : -1;
    keep[(long)img * P + p] = 0;
  }
}

// Labels are read with ld.volatile while other blocks link roots: an L1-cached stale root would never see its link.
__device__ __forceinline__ int uf_find(volatile int* L, int x) {
  for (int y = L[x]; y != x; y = L[x]) x = y;
  return x;
}

// Join the trees of a and b: link the larger root below the smaller one with atomicMin; if that root was linked by
// another thread meanwhile, atomicMin returns its new parent, and the join continues from there.
__device__ __forceinline__ void uf_union(int* L, int a, int b) {
  for (;;) {
    a = uf_find(L, a), b = uf_find(L, b);
    if (a == b) return;
    if (a > b) {
      const int t = a;
      a = b, b = t;
    }
    const int old = atomicMin(L + b, a);
    if (old == b) return;
    b = old;
  }
}

__global__ void __launch_bounds__(CN_THREADS) canny_merge_kernel(const uint8_t* __restrict__ cls, int h, int w,
                                                                 int* __restrict__ label) {
  const long P = (long)h * w;
  const long p = (long)blockIdx.x * CN_THREADS + threadIdx.x;
  if (p >= P) return;
  const uint8_t* C = cls + (long)blockIdx.y * P;
  if (!C[p]) return;
  int* L = label + (long)blockIdx.y * P;
  const int y = (int)(p / w), x = (int)(p - (long)y * w);
  if (x > 0 && C[p - 1]) uf_union(L, (int)p, (int)(p - 1));
  if (y > 0) {
    const long u = p - w;
    if (x > 0 && C[u - 1]) uf_union(L, (int)p, (int)(u - 1));
    if (C[u]) uf_union(L, (int)p, (int)u);
    if (x + 1 < w && C[u + 1]) uf_union(L, (int)p, (int)(u + 1));
  }
}

__global__ void __launch_bounds__(CN_THREADS) canny_flatten_kernel(const uint8_t* __restrict__ cls, long P,
                                                                   int* __restrict__ label, uint8_t* __restrict__ keep) {
  const long p = (long)blockIdx.x * CN_THREADS + threadIdx.x;
  if (p >= P) return;
  const long o = (long)blockIdx.y * P;
  const int k = cls[o + p];
  if (!k) return;
  int* L = label + o;
  int r = (int)p;
  for (int q = L[r]; q != r; q = L[r]) r = q;             // other threads only shorten paths here
  L[p] = r;
  if (k == 2) keep[o + r] = 1;
}

__global__ void __launch_bounds__(CN_THREADS) canny_output_kernel(const uint8_t* __restrict__ cls,
                                                                  const int* __restrict__ label,
                                                                  const uint8_t* __restrict__ keep, long P,
                                                                  float* __restrict__ out) {
  const long p = (long)blockIdx.x * CN_THREADS + threadIdx.x;
  if (p >= P) return;
  const long o = (long)blockIdx.y * P;
  out[o + p] = (cls[o + p] && keep[o + label[o + p]]) ? 1.0f : 0.0f;
}

}  // namespace vg

using namespace vg;

extern "C" {

int vgen_canny(const void* src, int src_u8, int64_t n, int64_t c, int64_t h, int64_t w, int64_t s_n, int64_t s_c,
               int64_t s_y, int64_t s_x, int mode, const double* rand, double low, double high, uint8_t* bytes,
               int32_t* hist, int32_t* thr, uint8_t* cls, int32_t* label, uint8_t* keep, float* out, void* stream) {
  VG_REQUIRE(src && bytes && hist && thr && cls && label && keep && out && (mode != 2 || rand), "vgen_canny: null pointer");
  VG_REQUIRE(n >= 0 && (c == 1 || c == 3) && h > 0 && w > 0 && mode >= 0 && mode <= 2, "vgen_canny: bad shape or mode");
  VG_REQUIRE(n <= 65535 && h * w < (1ll << 31), "vgen_canny: too many or too large frames");
  VG_REQUIRE(mode != 0 || (low == low && high == high), "vgen_canny: NaN threshold");
  if (n == 0) return 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const long P = (long)(h * w);
  VG_CUDA(cudaMemsetAsync(hist, 0, (size_t)n * 256 * sizeof(int32_t), st));
  CannySrc s{src, src_u8 ? 1 : 0, (long)s_n, (long)s_c, (long)s_y, (long)s_x};
  const int qblocks = (int)std::min<long>(cdiv(P * c, CN_THREADS * 8), std::max<long>(1, 4096 / n));
  launch_kernel(canny_quantise_kernel, dim3((unsigned)qblocks, (unsigned)n), dim3(CN_THREADS), 0, st, s, (int)c, (int)h,
                (int)w, bytes, hist);
  VG_LAUNCH_CHECK("canny_quantise_kernel");
  launch_kernel(canny_threshold_kernel, dim3((unsigned)n), dim3(256), 0, st, hist, (long)(P * c), mode, rand, low, high,
                thr);
  VG_LAUNCH_CHECK("canny_threshold_kernel");
  launch_kernel(canny_gradient_kernel, dim3((unsigned)cdiv(w, CN_TX), (unsigned)cdiv(h, CN_TY), (unsigned)n),
                dim3(CN_THREADS), 0, st, bytes, (int)c, (int)h, (int)w, thr, cls, label, keep);
  VG_LAUNCH_CHECK("canny_gradient_kernel");
  const dim3 pgrid((unsigned)cdiv(P, CN_THREADS), (unsigned)n);
  launch_kernel(canny_merge_kernel, pgrid, dim3(CN_THREADS), 0, st, cls, (int)h, (int)w, label);
  VG_LAUNCH_CHECK("canny_merge_kernel");
  launch_kernel(canny_flatten_kernel, pgrid, dim3(CN_THREADS), 0, st, cls, P, label, keep);
  VG_LAUNCH_CHECK("canny_flatten_kernel");
  launch_kernel(canny_output_kernel, pgrid, dim3(CN_THREADS), 0, st, cls, label, keep, P, out);
  VG_LAUNCH_CHECK("canny_output_kernel");
  return 0;
}

}  // extern "C"
