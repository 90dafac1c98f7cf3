// The VideoComposer colour-palette annotator (tools/annotator/histogram/palette.py Palette.histogram / quantize_image:
// skimage rgb2lab, sklearn euclidean_distances against the palette's Lab entries, argmin, bincount, Gaussian smoothing),
// device side, for n frames per call.
//
// 1. palette_nearest_kernel: per pixel, Lab in float64 as skimage 0.22 computes it (sRGB linearisation with the 0.04045
//    threshold and the 2.4 power, or a 256-entry table of it for uint8 input; xyz_from_rgb; D65 2-degree white; cube
//    root or 7.787 t + 16/116), then the nearest palette entry by sklearn's expansion -2 x.y + |x|^2 + |y|^2 clipped at
//    0, the first index on ties (np.argmin).  Every product and sum is rounded on its own (no FMA contraction), in the
//    order the host restatement uses.  The histogram form counts into a per-block shared-memory histogram, then adds it
//    to the frame's global counts; the quantise form writes the chosen entry's host-computed lab2rgb colour.
// 2. palette_finish_kernel: one block per frame: count / (h * w) in float64, the smoothing by the host-built
//    row-normalised exp(-lab_dists / 2 sigma^2) matrix, zeroing below 1e-5 (both only when the matrix is given, as the
//    reference skips both for sigma <= 0), written as fp32 or fp64.
#include <algorithm>

#include "common.h"

namespace vg {

constexpr int PAL_THREADS = 256;
constexpr int PAL_MAX = 156;                               // the UNet's hist_dim: the default 11-hue palette

struct PalSrc {
  const void* p;
  int kind;                                                // 0 fp32, 1 uint8, 2 fp64
  long s_n, s_c, s_y, s_x;                                 // element strides
};

__device__ __forceinline__ double pal_sample(const PalSrc& s, long off, const double* lin) {
  if (s.kind == 1) return lin[__ldg(reinterpret_cast<const uint8_t*>(s.p) + off)];
  const double v = s.kind == 0 ? (double)__ldg(reinterpret_cast<const float*>(s.p) + off)
                               : __ldg(reinterpret_cast<const double*>(s.p) + off);
  return v > 0.04045 ? pow(__ddiv_rn(__dadd_rn(v, 0.055), 1.055), 2.4) : __ddiv_rn(v, 12.92);
}

__device__ __forceinline__ double pal_f(double t) {       // xyz2lab's nonlinearity
  return t > 0.008856 ? cbrt(t) : __dadd_rn(__dmul_rn(7.787, t), 16.0 / 116.0);
}

__device__ __forceinline__ double pal_dot3(double a0, double a1, double a2, double b0, double b1, double b2) {
  return __dadd_rn(__dadd_rn(__dmul_rn(a0, b0), __dmul_rn(a1, b1)), __dmul_rn(a2, b2));
}

// lab4: [npal][4] = (L, a, b, |lab|^2); lin: the uint8 linearisation table [256]; counts [n][npal] (kHist) or
// out fp64 [n][h][w][3] gathered from qrgb [npal][3].
template <bool kHist>
__global__ void __launch_bounds__(PAL_THREADS) palette_nearest_kernel(PalSrc s, int h, int w,
                                                                      const double4* __restrict__ lab4, int npal,
                                                                      const double* __restrict__ lin,
                                                                      unsigned* __restrict__ counts,
                                                                      const double* __restrict__ qrgb,
                                                                      double* __restrict__ out) {
  __shared__ double4 pal[PAL_MAX];
  __shared__ unsigned bins[PAL_MAX];
  __shared__ double tab[256];
  const int img = blockIdx.y;
  for (int i = threadIdx.x; i < npal; i += PAL_THREADS) {
    pal[i] = lab4[i];
    bins[i] = 0;
  }
  if (s.kind == 1)
    for (int i = threadIdx.x; i < 256; i += PAL_THREADS) tab[i] = lin[i];
  __syncthreads();
  const long P = (long)h * w;
  const long base = (long)img * s.s_n;
  for (long p = (long)blockIdx.x * PAL_THREADS + threadIdx.x; p < P; p += (long)gridDim.x * PAL_THREADS) {
    const int y = (int)(p / w), x = (int)(p - (long)y * w);
    const long off = base + y * s.s_y + x * s.s_x;
    const double r = pal_sample(s, off, tab), g = pal_sample(s, off + s.s_c, tab), b = pal_sample(s, off + 2 * s.s_c, tab);
    // rgb2xyz (xyz_from_rgb rows), scaled by the D65 2-degree white, then xyz2lab
    const double fx = pal_f(__ddiv_rn(pal_dot3(r, g, b, 0.412453, 0.357580, 0.180423), 0.95047));
    const double fy = pal_f(pal_dot3(r, g, b, 0.212671, 0.715160, 0.072169));
    const double fz = pal_f(__ddiv_rn(pal_dot3(r, g, b, 0.019334, 0.119193, 0.950227), 1.08883));
    const double L = __dsub_rn(__dmul_rn(116.0, fy), 16.0);
    const double A = __dmul_rn(500.0, __dsub_rn(fx, fy));
    const double B = __dmul_rn(200.0, __dsub_rn(fy, fz));
    const double xx = pal_dot3(L, A, B, L, A, B);
    int best = 0;
    double dbest = 0.0;
    for (int k = 0; k < npal; ++k) {
      const double4 q = pal[k];
      double d = __dadd_rn(__dadd_rn(__dmul_rn(-2.0, pal_dot3(L, A, B, q.x, q.y, q.z)), xx), q.w);
      d = d > 0.0 ? d : 0.0;                               // np.maximum(distances, 0)
      if (k == 0 || d < dbest) {
        dbest = d;
        best = k;
      }
    }
    if (kHist) {
      atomicAdd(&bins[best], 1u);
    } else {
      double* o = out + ((long)img * P + p) * 3;
      o[0] = qrgb[best * 3];
      o[1] = qrgb[best * 3 + 1];
      o[2] = qrgb[best * 3 + 2];
    }
  }
  if (kHist) {
    __syncthreads();
    for (int i = threadIdx.x; i < npal; i += PAL_THREADS)
      if (bins[i]) atomicAdd(counts + (long)img * npal + i, bins[i]);
  }
}

// weight: [npal][npal] row-normalised smoothing matrix, or null (sigma <= 0: the plain normalised counts)
__global__ void __launch_bounds__(PAL_THREADS) palette_finish_kernel(const unsigned* __restrict__ counts, int npal,
                                                                     double npix, const double* __restrict__ weight,
                                                                     void* out, int out_f64) {
  __shared__ double hist[PAL_MAX];
  const int img = blockIdx.x, t = threadIdx.x;
  for (int i = t; i < npal; i += PAL_THREADS) hist[i] = __ddiv_rn((double)counts[(long)img * npal + i], npix);
  __syncthreads();
  for (int i = t; i < npal; i += PAL_THREADS) {
    double v = hist[i];
    if (weight) {
      const double* wr = weight + (long)i * npal;
      v = 0.0;
      for (int j = 0; j < npal; ++j) v = __dadd_rn(v, __dmul_rn(wr[j], hist[j]));
      if (v < 1e-5) v = 0.0;
    }
    if (out_f64)
      reinterpret_cast<double*>(out)[(long)img * npal + i] = v;
    else
      reinterpret_cast<float*>(out)[(long)img * npal + i] = (float)v;
  }
}

static int nearest_blocks(long P, long n) {
  return (int)std::min<long>(cdiv(P, PAL_THREADS * 4), std::max<long>(1, 8192 / n));
}

}  // namespace vg

using namespace vg;

#define PAL_CHECK_COMMON(fn)                                                                                          \
  VG_REQUIRE(src && lab4 && (src_kind != 1 || lin), fn ": null pointer");                                            \
  VG_REQUIRE(n >= 0 && h > 0 && w > 0 && src_kind >= 0 && src_kind <= 2, fn ": bad shape or source type");          \
  VG_REQUIRE(npal >= 1 && npal <= PAL_MAX, fn ": the palette must have 1 to 156 entries");                           \
  VG_REQUIRE(n <= 65535 && h * w < (1ll << 31), fn ": too many or too large frames")

extern "C" {

int vgen_palette_histogram(const void* src, int src_kind, int64_t n, int64_t h, int64_t w, int64_t s_n, int64_t s_c,
                           int64_t s_y, int64_t s_x, const double* lab4, int64_t npal, const double* lin,
                           const double* weight, uint32_t* counts, void* out, int out_f64, void* stream) {
  PAL_CHECK_COMMON("vgen_palette_histogram");
  VG_REQUIRE(counts && out, "vgen_palette_histogram: null pointer");
  if (n == 0) return 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const long P = (long)(h * w);
  VG_CUDA(cudaMemsetAsync(counts, 0, (size_t)n * npal * sizeof(uint32_t), st));
  PalSrc s{src, src_kind, (long)s_n, (long)s_c, (long)s_y, (long)s_x};
  launch_kernel(palette_nearest_kernel<true>, dim3((unsigned)nearest_blocks(P, n), (unsigned)n), dim3(PAL_THREADS), 0,
                st, s, (int)h, (int)w, reinterpret_cast<const double4*>(lab4), (int)npal, lin, counts,
                (const double*)nullptr, (double*)nullptr);
  VG_LAUNCH_CHECK("palette_nearest_kernel");
  launch_kernel(palette_finish_kernel, dim3((unsigned)n), dim3(PAL_THREADS), 0, st, (const unsigned*)counts, (int)npal,
                (double)P, weight, out, out_f64 ? 1 : 0);
  VG_LAUNCH_CHECK("palette_finish_kernel");
  return 0;
}

int vgen_palette_quantize(const void* src, int src_kind, int64_t n, int64_t h, int64_t w, int64_t s_n, int64_t s_c,
                          int64_t s_y, int64_t s_x, const double* lab4, int64_t npal, const double* lin,
                          const double* qrgb, double* out, void* stream) {
  PAL_CHECK_COMMON("vgen_palette_quantize");
  VG_REQUIRE(qrgb && out, "vgen_palette_quantize: null pointer");
  if (n == 0) return 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const long P = (long)(h * w);
  PalSrc s{src, src_kind, (long)s_n, (long)s_c, (long)s_y, (long)s_x};
  launch_kernel(palette_nearest_kernel<false>, dim3((unsigned)nearest_blocks(P, n), (unsigned)n), dim3(PAL_THREADS), 0,
                st, s, (int)h, (int)w, reinterpret_cast<const double4*>(lab4), (int)npal, lin, (unsigned*)nullptr, qrgb,
                out);
  VG_LAUNCH_CHECK("palette_nearest_kernel");
  return 0;
}

}  // extern "C"
