// Internal description of one tap-GEMM problem (see tapgemm_sm90.cu for the maths).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>

namespace vg {

static constexpr int kMaxTaps = 33;   // the 33 distinct taps of PiDiNet's CDCM (four dilated 3x3 convs summed)
static constexpr int kMaxBnGelu = 224;   // widest N tile of the GELU / row-bias epilogue (BN = 256 spills registers)

// Division by a launch-time constant as multiply-high + shift (exact for 0 <= x < 2^31).  The persistent
// kernels decompose a tile index with three div/mod pairs per tile in every warp role; with hardware
// integer division (~40 dependent instructions each) that alone cost more than the MMAs of a short-K tile.
struct FastDiv {
  uint32_t d, mul, shr;
};
inline FastDiv make_fastdiv(int d) {
  FastDiv f;
  f.d = (uint32_t)d;
  f.mul = 0;
  f.shr = 0;
  if (d > 1) {
    int lg = 0;
    while ((1ll << lg) < d) ++lg;
    const int p = 31 + lg;
    f.mul = (uint32_t)(((1ull << p) + (uint64_t)d - 1) / (uint64_t)d);
    f.shr = (uint32_t)(p - 32);
  }
  return f;
}
#ifdef __CUDACC__
__device__ __forceinline__ int fd_div(const FastDiv& f, int x) {
  return f.d == 1 ? x : (int)(__umulhi((uint32_t)x, f.mul) >> f.shr);
}
__device__ __forceinline__ void fd_divmod(const FastDiv& f, int x, int& q, int& r) {
  q = fd_div(f, x);
  r = x - q * (int)f.d;
}
#endif

struct TapGemmShape {
  int c;            // channels of A (K per tap)
  int kc;           // c / 64
  int d1, d2, d3;   // logical extents of A / of the output rows (row = (i3*d2 + i2)*d1 + i1)
  int box1, box2;   // output tile = box1 x box2 positions (<= 128) of one i3
  int t1, t2;       // tiles along d1 / d2
  int num_taps;
  int8_t tap1[kMaxTaps], tap2[kMaxTaps], tap3[kMaxTaps];  // coordinate offsets per tap (bytes keep the kernel parameters
                                                        // about as small as with nine int taps)
  int n;            // output channels (rows of W)
  int bn;           // N tile
  int nb;           // ceil(n / bn)
  int total_tiles;  // d3 * t2 * t1 * nb
  FastDiv f_nb, f_t1, f_t2, f_box1;  // filled by tapgemm_prepare_shape()
};

inline void tapgemm_prepare_shape(TapGemmShape& s) {
  s.f_nb = make_fastdiv(s.nb);
  s.f_t1 = make_fastdiv(s.t1);
  s.f_t2 = make_fastdiv(s.t2);
  s.f_box1 = make_fastdiv(s.box1);
}

struct TapGemmEpilogue {
  __half* out;
  long ldo;                  // elements between consecutive output rows
  float alpha;               // accumulator scale
  const float* bias;         // [n] or null   (GEGLU: indexed like the packed W rows)
  const __half* group_bias;  // [d3][n] or null: added per outermost coordinate (frame) after rounding
  long ld_group_bias;
  int group_bias_div;        // bias row = i3 / group_bias_div
  FastDiv f_group_bias_div;  // filled by the wgmma launcher
  const __half* residual;    // [rows][n] or null: added after rounding
  long ldr;
  int geglu;                 // out has n/2 columns: value * gelu(gate)
  const float2* row_stats;   // [rows] {rstd, -mean * rstd} or null: LayerNorm folded into the epilogue (linear only)
  const float* col_sum;      // [n]: sum_k w[n][k]   (GEGLU: indexed like bias)
  int gelu;                  // out = gelu_erf(acc + bias + row_bias) in fp32, one rounding (adapter down projection)
  const float* row_bias;     // [rows / rows_per_group][n] fp32 or null: added to the accumulator before the activation
  long ld_row_bias;
  int rows_per_group;
  FastDiv f_rows_per_group;  // filled by the wgmma launcher
  int relu;                  // out = relu(acc * alpha + bias) in fp32, one rounding (no residual / per-frame bias)
  long out_s2, out_s3;       // 0: output rows are ldo apart; else element strides of the output along d2 / d3, with
                             // ldo the stride along d1 (one phase of a transposed conv writes a strided sub-grid)
};

struct TapGemmArgs {
  const __half* a;
  long a_stride1, a_stride2, a_stride3;  // element strides of d1, d2, d3 (channel stride is 1)
  const __half* w;                       // [n][num_taps * c], K-major
  // K tail (linear only, vgen_linear_lora): out += h[row][:r] . u[n][:r] accumulated after the main K loop into the same
  // fp32 accumulators; r = 0: none.  h fp16 [rows][r] (row stride ldh), u fp16 [n][r]; r a multiple of 64.
  const __half* h;
  long ldh;
  const __half* u;
  int r;
  TapGemmShape shape;
  TapGemmEpilogue epi;
};

int tapgemm_sm90_launch(const TapGemmArgs& a, cudaStream_t stream);   // wgmma + TMA, one CTA per 128-row tile
int tapgemm_simt_launch(const TapGemmArgs& a, cudaStream_t stream);   // plain SIMT cross-check kernel

}  // namespace vg
