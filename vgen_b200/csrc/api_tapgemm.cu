// C-ABI entry points of the tap-GEMM family: they only describe the problem (extents, taps, tile
// shape) and hand it to the wgmma kernel (or, for debugging, the SIMT cross-check kernel).
#include <stdlib.h>

#include "common.h"
#include "tapgemm.h"

namespace vg {

static int g_tapgemm_impl = 0;  // 0 = auto (wgmma whenever C % 64 == 0, else simt), 1 = simt
static int g_tapgemm_bn = 0;    // 0 = pick_bn; else the N tile of every launch whose epilogue leaves bn at 0 (debug)

// N tile.  With many M tiles the cost is the padded N extent plus a per-tile constant (~24 columns' worth of
// epilogue / pipeline fill).  With FEW M tiles (the coarse levels of the UNet) the persistent grid runs
// ceil(tiles / SMs) waves and the widest tile can leave most of the last wave idle, while a narrower one adds a wave
// of less work each.  So the cost is waves x (BN + overhead), waves counted on this device.
// The widest candidate is 224: on every tap-GEMM shape of bench.py's i2vgen step, BN = 256 measured no faster than the
// best narrower tile except on two 22 x 40 conv3x3s with K >= 17 280 (within 2 % there), and 1.2-1.5x slower on the
// 1280-wide linears and temporal convs (K = 1280 ... 5120), which the model used to give 256 (H100 80GB HBM3, 700 W;
// tools/bench_tapgemm_wide.py).  GEGLU keeps its own rule: its tile is fixed when the weight is packed.
static constexpr int kMaxBnAuto = 224;
static int pick_bn(long n, int geglu, long m_tiles, int ctas) {
  if (geglu) {
    for (int bn = 256; bn >= 64; bn -= 64)
      if (n % bn == 0) return bn;
    return 0;
  }
  if (n <= 96) return (int)((n + 31) / 32) * 32;
  if (ctas < 1) ctas = 1;
  int best = 128;
  double best_cost = 1e30;
  for (int bn = kMaxBnAuto; bn >= 96; bn -= 32) {
    const long nb = (n + bn - 1) / bn;
    const long tiles = nb * (m_tiles > 0 ? m_tiles : 1);
    const long waves = (tiles + ctas - 1) / ctas;
    // many waves: the tail wave is amortised, fall back to total padded work
    const double work = tiles > 8L * ctas ? (double)tiles / ctas : (double)waves;
    const double cost = work * (bn + 24.0);
    if (cost < best_cost - 1e-9) {
      best_cost = cost;
      best = bn;
    }
  }
  return best;
}

// choose the (box1, box2) output tile (<=128 positions) that wastes the fewest MMA rows
static void pick_box(long d1, long d2, int* b1, int* b2) {
  double best = -1;
  int bb1 = 1, bb2 = 1;
  const int max1 = (int)(d1 < 128 ? d1 : 128);
  for (int x = max1; x >= 1; --x) {
    int y = 128 / x;
    if (y > d2) y = (int)d2;
    if (y > 256) y = 256;
    const double tiles = (double)cdiv(d1, x) * cdiv(d2, y);
    const double eff = (double)d1 * d2 / (tiles * 128.0);
    if (eff > best + 1e-9) {
      best = eff;
      bb1 = x;
      bb2 = y;
    }
  }
  *b1 = bb1;
  *b2 = bb2;
}

static int fill_epilogue(TapGemmArgs* t, void* out, long ldo, const vgen_epilogue* epi) {
  TapGemmEpilogue& e = t->epi;
  e.out = reinterpret_cast<__half*>(out);
  e.ldo = ldo;
  e.alpha = epi ? epi->alpha : 1.0f;
  e.bias = epi ? epi->bias : nullptr;
  e.group_bias = epi ? reinterpret_cast<const __half*>(epi->group_bias) : nullptr;
  e.ld_group_bias = epi ? epi->group_bias_ld : 0;
  e.group_bias_div = (epi && epi->group_bias_div > 1) ? (int)epi->group_bias_div : 1;
  e.residual = epi ? reinterpret_cast<const __half*>(epi->residual) : nullptr;
  e.ldr = epi ? epi->residual_ld : 0;
  e.geglu = epi ? epi->geglu : 0;
  // the GEGLU epilogue (wgmma and SIMT alike) computes value * gelu(gate) and nothing after it
  VG_REQUIRE(!e.geglu || (!e.residual && !e.group_bias), "tapgemm: the GEGLU epilogue takes no residual or per-frame bias");
  e.row_stats = epi ? reinterpret_cast<const float2*>(epi->row_stats) : nullptr;
  e.col_sum = epi ? epi->col_sum : nullptr;
  VG_REQUIRE((e.row_stats == nullptr) == (e.col_sum == nullptr), "tapgemm: row_stats and col_sum go together");
  VG_REQUIRE((reinterpret_cast<uintptr_t>(e.row_stats) & 7) == 0 && (reinterpret_cast<uintptr_t>(e.col_sum) & 15) == 0,
             "tapgemm: row_stats must be 8-byte and col_sum 16-byte aligned");
  return 0;
}

static int finish_and_launch(TapGemmArgs* t, const vgen_epilogue* epi, void* stream) {
  static bool env_read = false;
  if (!env_read) {  // VGEN_TAPGEMM_IMPL=0|1 overrides the default once (A/B measurements)
    env_read = true;
    const char* ev = getenv("VGEN_TAPGEMM_IMPL");
    if (ev && ev[0] >= '0' && ev[0] <= '1') g_tapgemm_impl = ev[0] - '0';
  }
  TapGemmShape& s = t->shape;
  s.kc = s.c / 64;
  const long m_tiles_all = (long)s.d3 * cdiv(s.d2, s.box2) * cdiv(s.d1, s.box1);
  int bn = (epi && epi->bn > 0) ? epi->bn
           : g_tapgemm_bn > 0   ? g_tapgemm_bn
                                : pick_bn(s.n, t->epi.geglu, m_tiles_all, sm_count());
  VG_REQUIRE(bn > 0, "tapgemm: no valid N tile (GEGLU needs n % 64 == 0)");
  s.bn = bn;
  s.nb = cdiv(s.n, bn);
  s.t1 = cdiv(s.d1, s.box1);
  s.t2 = cdiv(s.d2, s.box2);
  const long tiles = (long)s.d3 * s.t2 * s.t1 * s.nb;
  VG_REQUIRE(tiles < (1L << 31), "tapgemm: too many tiles");
  s.total_tiles = (int)tiles;
  if (tiles == 0) return 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (g_tapgemm_impl == 1 || (s.c % 64) != 0) return tapgemm_simt_launch(*t, st);
  return tapgemm_sm90_launch(*t, st);
}

}  // namespace vg

using namespace vg;

extern "C" {

int vgen_set_tapgemm_impl(int impl) {
  if (impl < 0 || impl > 1) return fail("vgen_set_tapgemm_impl: impl must be 0 (auto) or 1 (simt)");
  g_tapgemm_impl = impl;
  return 0;
}

int vgen_set_tapgemm_bn(int bn) {
  if (bn != 0 && (bn < 32 || bn > 256 || bn % 32 != 0))
    return fail("vgen_set_tapgemm_bn: bn must be 0 (heuristic) or a multiple of 32 in [32, 256]");
  g_tapgemm_bn = bn;
  return 0;
}

int vgen_linear(const void* a, int64_t m, int64_t k, int64_t lda, const void* w, int64_t n, void* out, int64_t ldo,
                const vgen_epilogue* epi, void* stream) {
  VG_REQUIRE(a && w && out, "vgen_linear: null pointer");
  VG_REQUIRE(m >= 0 && k > 0 && n > 0 && lda >= k, "vgen_linear: bad shape");
  if (m == 0) return 0;
  TapGemmArgs t{};
  t.a = reinterpret_cast<const __half*>(a);
  t.w = reinterpret_cast<const __half*>(w);
  t.a_stride1 = lda;
  t.a_stride2 = lda * m;
  t.a_stride3 = lda * m;
  TapGemmShape& s = t.shape;
  s.c = (int)k;
  s.d1 = (int)m;
  s.d2 = 1;
  s.d3 = 1;
  s.box1 = 128;
  s.box2 = 1;
  s.num_taps = 1;
  s.tap1[0] = s.tap2[0] = s.tap3[0] = 0;
  s.n = (int)n;
  {
    int rc = fill_epilogue(&t, out, ldo, epi);
    if (rc) return rc;
  }
  VG_REQUIRE(!t.epi.group_bias, "vgen_linear: group_bias is only defined for conv entries");
  return finish_and_launch(&t, epi, stream);
}

int vgen_linear_lora(const void* a, int64_t m, int64_t k, int64_t lda, const void* w, int64_t n, const void* h, int64_t r,
                     int64_t ldh, const void* u, void* out, int64_t ldo, const vgen_epilogue* epi, void* stream) {
  VG_REQUIRE(a && w && out && h && u, "vgen_linear_lora: null pointer");
  VG_REQUIRE(m >= 0 && k > 0 && n > 0 && lda >= k && r > 0 && r % 64 == 0 && ldh >= r, "vgen_linear_lora: bad shape");
  if (m == 0) return 0;
  TapGemmArgs t{};
  t.a = reinterpret_cast<const __half*>(a);
  t.w = reinterpret_cast<const __half*>(w);
  t.a_stride1 = lda;
  t.a_stride2 = lda * m;
  t.a_stride3 = lda * m;
  t.h = reinterpret_cast<const __half*>(h);
  t.ldh = ldh;
  t.u = reinterpret_cast<const __half*>(u);
  t.r = (int)r;
  TapGemmShape& s = t.shape;
  s.c = (int)k;
  s.d1 = (int)m;
  s.d2 = 1;
  s.d3 = 1;
  s.box1 = 128;
  s.box2 = 1;
  s.num_taps = 1;
  s.tap1[0] = s.tap2[0] = s.tap3[0] = 0;
  s.n = (int)n;
  {
    int rc = fill_epilogue(&t, out, ldo, epi);
    if (rc) return rc;
  }
  VG_REQUIRE(!t.epi.group_bias && !t.epi.geglu && !t.epi.row_stats,
             "vgen_linear_lora: bias and residual only (no group_bias, GEGLU or folded LayerNorm)");
  return finish_and_launch(&t, epi, stream);
}

int vgen_linear_gelu_rowbias(const void* a, int64_t m, int64_t k, int64_t lda, const void* w, int64_t n, const float* bias,
                             const float* row_bias, int64_t ld_row_bias, int64_t rows_per_group, void* out, int64_t ldo,
                             void* stream) {
  VG_REQUIRE(a && w && out, "vgen_linear_gelu_rowbias: null pointer");
  VG_REQUIRE(m >= 0 && k > 0 && n > 0 && lda >= k && ldo >= n, "vgen_linear_gelu_rowbias: bad shape");
  VG_REQUIRE(row_bias == nullptr || (rows_per_group >= 1 && rows_per_group < (1L << 31) && ld_row_bias >= n &&
                                     ld_row_bias % 2 == 0 && (reinterpret_cast<uintptr_t>(row_bias) & 7) == 0),
             "vgen_linear_gelu_rowbias: row_bias needs rows_per_group >= 1, an even ld_row_bias >= n and 8-byte alignment");
  if (m == 0) return 0;
  TapGemmArgs t{};
  t.a = reinterpret_cast<const __half*>(a);
  t.w = reinterpret_cast<const __half*>(w);
  t.a_stride1 = lda;
  t.a_stride2 = lda * m;
  t.a_stride3 = lda * m;
  TapGemmShape& s = t.shape;
  s.c = (int)k;
  s.d1 = (int)m;
  s.d2 = 1;
  s.d3 = 1;
  s.box1 = 128;
  s.box2 = 1;
  s.num_taps = 1;
  s.tap1[0] = s.tap2[0] = s.tap3[0] = 0;
  s.n = (int)n;
  TapGemmEpilogue& e = t.epi;
  e.out = reinterpret_cast<__half*>(out);
  e.ldo = ldo;
  e.alpha = 1.0f;
  e.bias = bias;
  e.gelu = 1;
  e.row_bias = row_bias;
  e.ld_row_bias = row_bias ? ld_row_bias : 0;
  e.rows_per_group = row_bias ? (int)rows_per_group : 1;
  return finish_and_launch(&t, nullptr, stream);
}

int vgen_conv2d_3x3(const void* x, int64_t nimg, int64_t h, int64_t w_, int64_t c, const void* w, int64_t n, void* out,
                    int64_t ldo, const vgen_epilogue* epi, void* stream) {
  VG_REQUIRE(x && w && out, "vgen_conv2d_3x3: null pointer");
  VG_REQUIRE(nimg >= 0 && h > 0 && w_ > 0 && c > 0 && n > 0, "vgen_conv2d_3x3: bad shape");
  if (nimg == 0) return 0;
  TapGemmArgs t{};
  t.a = reinterpret_cast<const __half*>(x);
  t.w = reinterpret_cast<const __half*>(w);
  t.a_stride1 = c;
  t.a_stride2 = c * w_;
  t.a_stride3 = c * w_ * h;
  TapGemmShape& s = t.shape;
  s.c = (int)c;
  s.d1 = (int)w_;
  s.d2 = (int)h;
  s.d3 = (int)nimg;
  pick_box(w_, h, &s.box1, &s.box2);
  s.num_taps = 9;
  for (int ky = 0; ky < 3; ++ky)
    for (int kx = 0; kx < 3; ++kx) {
      s.tap1[ky * 3 + kx] = kx - 1;
      s.tap2[ky * 3 + kx] = ky - 1;
      s.tap3[ky * 3 + kx] = 0;
    }
  s.n = (int)n;
  {
    int rc = fill_epilogue(&t, out, ldo, epi);
    if (rc) return rc;
  }
  VG_REQUIRE(!t.epi.row_stats, "vgen_conv2d_3x3: row_stats (folded LayerNorm) is only defined for vgen_linear");
  return finish_and_launch(&t, epi, stream);
}

int vgen_conv2d_taps(const void* x, int64_t nimg, int64_t h, int64_t w_, int64_t c, int64_t ntaps, const int32_t* dy,
                     const int32_t* dx, const void* w, int64_t n, void* out, int64_t out_stride_y, int64_t out_stride_x,
                     const vgen_epilogue* epi, int relu, void* stream) {
  VG_REQUIRE(x && w && out && dy && dx, "vgen_conv2d_taps: null pointer");
  VG_REQUIRE(nimg >= 0 && h > 0 && w_ > 0 && c > 0 && n > 0, "vgen_conv2d_taps: bad shape");
  VG_REQUIRE(ntaps >= 1 && ntaps <= kMaxTaps, "vgen_conv2d_taps: 1 to 33 taps");
  VG_REQUIRE(out_stride_x >= n && out_stride_y >= out_stride_x * w_, "vgen_conv2d_taps: output strides overlap");
  for (int i = 0; i < ntaps; ++i)
    VG_REQUIRE(dy[i] >= -127 && dy[i] <= 127 && dx[i] >= -127 && dx[i] <= 127, "vgen_conv2d_taps: tap offsets must be in [-127, 127]");
  if (nimg == 0) return 0;
  TapGemmArgs t{};
  t.a = reinterpret_cast<const __half*>(x);
  t.w = reinterpret_cast<const __half*>(w);
  t.a_stride1 = c;
  t.a_stride2 = c * w_;
  t.a_stride3 = c * w_ * h;
  TapGemmShape& s = t.shape;
  s.c = (int)c;
  s.d1 = (int)w_;
  s.d2 = (int)h;
  s.d3 = (int)nimg;
  pick_box(w_, h, &s.box1, &s.box2);
  s.num_taps = (int)ntaps;
  for (int i = 0; i < ntaps; ++i) {
    s.tap1[i] = (int8_t)dx[i];
    s.tap2[i] = (int8_t)dy[i];
    s.tap3[i] = 0;
  }
  s.n = (int)n;
  {
    int rc = fill_epilogue(&t, out, out_stride_x, epi);
    if (rc) return rc;
  }
  VG_REQUIRE(!t.epi.row_stats && !t.epi.geglu, "vgen_conv2d_taps: no folded LayerNorm or GEGLU");
  VG_REQUIRE(!relu || (!t.epi.residual && !t.epi.group_bias), "vgen_conv2d_taps: the ReLU epilogue goes with bias only");
  t.epi.relu = relu ? 1 : 0;
  if (out_stride_y != out_stride_x * w_) {   // a strided sub-grid (the tile-store kernels serve it with the ReLU epilogue)
    VG_REQUIRE(relu, "vgen_conv2d_taps: a strided output needs relu = 1");
    t.epi.out_s2 = out_stride_y;
    t.epi.out_s3 = out_stride_y * h;
  }
  return finish_and_launch(&t, epi, stream);
}

int vgen_tconv3_batch(const void* x, int64_t batch, int64_t f, int64_t hw, int64_t c, const void* w, int64_t n, void* out,
                      int64_t ldo, const vgen_epilogue* epi, void* stream) {
  VG_REQUIRE(x && w && out, "vgen_tconv3: null pointer");
  VG_REQUIRE(batch >= 0 && f >= 0 && hw > 0 && c > 0 && n > 0, "vgen_tconv3: bad shape");
  if (f == 0 || batch == 0) return 0;
  TapGemmArgs t{};
  t.a = reinterpret_cast<const __half*>(x);
  t.w = reinterpret_cast<const __half*>(w);
  t.a_stride1 = c;
  t.a_stride2 = c * hw;
  t.a_stride3 = c * hw * f;
  TapGemmShape& s = t.shape;
  s.c = (int)c;
  s.d1 = (int)hw;
  s.d2 = (int)f;
  s.d3 = (int)batch;  // videos: the frame taps are zero-padded by the TMA unit at each video's first / last frame
  s.box1 = (int)(hw < 128 ? hw : 128);
  s.box2 = 1;
  if (hw < 128) {  // small planes: put several frames in one tile
    s.box2 = (int)(128 / hw);
    if (s.box2 > f) s.box2 = (int)f;
  }
  s.num_taps = 3;
  for (int kt = 0; kt < 3; ++kt) {
    s.tap1[kt] = 0;
    s.tap2[kt] = kt - 1;
    s.tap3[kt] = 0;
  }
  s.n = (int)n;
  {
    int rc = fill_epilogue(&t, out, ldo, epi);
    if (rc) return rc;
  }
  VG_REQUIRE(!t.epi.group_bias, "vgen_tconv3: group_bias not supported");
  VG_REQUIRE(!t.epi.row_stats, "vgen_tconv3: row_stats (folded LayerNorm) is only defined for vgen_linear");
  return finish_and_launch(&t, epi, stream);
}

int vgen_tconv3(const void* x, int64_t f, int64_t hw, int64_t c, const void* w, int64_t n, void* out, int64_t ldo,
                const vgen_epilogue* epi, void* stream) {
  return vgen_tconv3_batch(x, 1, f, hw, c, w, n, out, ldo, epi, stream);
}

}  // extern "C"
