// FP8 (e4m3) path of the tap-GEMM family: the one-tap (linear) instantiation with 8-bit operands, used by the UNet's
// transformer projections when a model is built with fp8_linear=True.  The fp16 kernels (tapgemm_sm90.cu) are untouched.
//
//   out[r, n] = epilogue( row_scale[r] * col_scale[n] * sum_k A8[r, k] * W8[n, k] )
//
// A8 are the e4m3 codes of the activations, quantised per row (vgen_quantize_rows_e4m3: row_scale = amax / 448), W8 the
// e4m3 codes of the weights, quantised per output channel at pack time (col_scale = amax / 448).
//
// Structure: the persistent, warp-specialised layout of tapgemm_sm90.cu.  One TMA producer warp fills a ring of
// (128 rows x 128 K) A tiles and (BN x 128 K) W tiles; 128 bytes of e4m3 are one 128B-swizzle row, so the tiles and the
// shared-memory descriptors are those of the fp16 kernel with 64 fp16 replaced by 128 e4m3.  Two consumer warpgroups
// each own 64 rows and issue four m64nBNk32 e4m3 wgmmas per stage.
//
// Promotion.  The tensor core adds 8-bit products in an accumulator narrower than fp32.  After every stage (K = 128,
// four wgmmas) the stage's partial sums are added into separate fp32 registers and the next stage starts from zero, so a
// long K (5120 for the FF down projection at 1280 channels) accumulates in full fp32.
//
// Epilogue.  The fp32 sums are multiplied by row_scale * col_scale and handed to tapgemm_epilogue_tile unchanged
// (bias, GEGLU interleave, residual, fp16 rounding, TMA tile stores).
#include <cuda_fp8.h>
#include <string.h>

#include "common.h"
#include "ptx.cuh"
#include "tapgemm.h"
#include "tapgemm_epilogue.cuh"

namespace vg {
namespace {

constexpr int kBM = 128;       // rows per tile
constexpr int kBK = 128;       // K per stage = one 128B swizzle row of e4m3
constexpr int kThreads = 384;  // producer warpgroup + two consumer warpgroups
constexpr int kABytes = kBM * kBK;
constexpr int kMaxStages = 8;

struct alignas(64) Fp8GemmParams {
  CUtensorMap map_a;    // A8 [m][k], box {128, 128}
  CUtensorMap map_b;    // W8 [n][k], box {128, BN}
  CUtensorMap map_out;  // output [out_n, m, 1, 1], box {32, 128, 1, 1}, 64B swizzle
  int out_tma;
  int m, kb;            // rows, K stages (ceil(k / 128); the TMA unit zero-fills the K tail)
  TapGemmShape s;       // n, bn, nb, total_tiles, f_nb (the epilogue reads s.n)
  TapGemmEpilogue e;
  const float* row_scale;
  const float* col_scale;
  int stages;
};

template <int BN, bool kGeglu>
__global__ void __launch_bounds__(kThreads, 1) tapgemm_fp8_kernel(const __grid_constant__ Fp8GemmParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  constexpr int kBBytes = BN * kBK;
  constexpr int kStageBytes = kABytes + kBBytes;
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  const int stages = p.stages;

  uint8_t* tiles = smem;
  uint8_t* staging = smem + (size_t)stages * kStageBytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(staging + kEpiStagingTotal);
  uint64_t* empty_bar = full_bar + stages;
  const TapGemmShape& s = p.s;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&p.map_a);
    tma_prefetch_desc(&p.map_b);
    if (p.out_tma) tma_prefetch_desc(&p.map_out);
    for (int i = 0; i < stages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 8);  // one arrival per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (warp != 0) return;
    // ------------------------------------------------------------------ TMA producer
    int st = 0;
    uint32_t ph = 0;
    for (int tile = blockIdx.x; tile < s.total_tiles; tile += gridDim.x) {
      int mt, nb_i;
      fd_divmod(s.f_nb, tile, mt, nb_i);
      for (int kb = 0; kb < p.kb; ++kb) {
        mbar_wait(&empty_bar[st], ph ^ 1);
        if (elect_one()) {
          mbar_expect_tx(&full_bar[st], (uint32_t)kStageBytes);
          uint8_t* sa = tiles + (size_t)st * kStageBytes;
          tma_load_2d(sa, &p.map_a, &full_bar[st], kb * kBK, mt * kBM);
          tma_load_2d(sa + kABytes, &p.map_b, &full_bar[st], kb * kBK, nb_i * BN);
        }
        __syncwarp();
        if (++st == stages) {
          st = 0;
          ph ^= 1;
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- wgmma consumers + epilogue
  setmaxnreg_inc<232>();
  const TapGemmEpilogue& e = p.e;
  const int cw = wg - 1;
  const int r0 = cw * 64 + (warp & 3) * 16 + (lane >> 2);  // this thread's rows are r0 and r0 + 8
  const int q2 = (lane & 3) * 2;
  const int out_n = kGeglu ? (s.n >> 1) : s.n;
  const bool vec_ok = tapgemm_vec_ok(e, out_n);
  EpiStore est;
  est.tma = p.out_tma != 0;
  est.map = &p.map_out;
  est.stage = smem_u32(staging);
  est.leader = (threadIdx.x == 128);
  est.slot = 0;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const uint32_t r = (uint32_t)(r0 + 8 * h);
    est.row_off[h] = r * 64u + (uint32_t)q2 * 2u;
    est.row_xor[h] = (r >> 1) & 3u;
  }
  const uint32_t tiles_addr = smem_u32(tiles);
  int st = 0;
  uint32_t ph = 0;
  float acc[BN / 2], sum[BN / 2];
  for (int tile = blockIdx.x; tile < s.total_tiles; tile += gridDim.x) {
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) sum[i] = 0.f;
    for (int kb = 0; kb < p.kb; ++kb) {
      mbar_wait(&full_bar[st], ph);
      const uint32_t a_addr = tiles_addr + (uint32_t)st * (uint32_t)kStageBytes;
      const uint64_t a_desc = wgmma_desc_sw128(a_addr + (uint32_t)cw * 64u * 128u, 16, 1024);
      const uint64_t b_desc = wgmma_desc_sw128(a_addr + kABytes, 16, 1024);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kBK / 32; ++k) {
        // advance 32 e4m3 (32 B) along K inside the swizzle atom: +2 in the >>4 address field
        wgmma_ss_e4m3<BN>(acc, a_desc + 2 * k, b_desc + 2 * k, k != 0 ? 1 : 0);
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_pin(acc);
      if (lane == 0) mbar_arrive(&empty_bar[st]);
      // promotion: this stage's partial sums into the fp32 accumulators
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) sum[i] += acc[i];
      if (++st == stages) {
        st = 0;
        ph ^= 1;
      }
    }

    EpiTile t;
    int mt;
    fd_divmod(s.f_nb, tile, mt, t.nb_i);
    t.i3 = 0;
    t.i1_0 = mt * kBM;
    t.i2_0 = 0;
    float rs[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = t.i1_0 + r0 + 8 * h;
      t.row_ok[h] = row < p.m;
      t.row[h] = row;
      t.ooff[h] = (long)row * e.ldo;
      rs[h] = t.row_ok[h] ? __ldg(p.row_scale + row) : 0.f;
    }
    // dequantisation: sum[(j * 4) + 2 h + c] is row h, column n0 + 8 j + q2 + c (GEGLU: packed weight row, like bias)
    const int n0 = t.nb_i * BN;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int n = n0 + j * 8 + q2;
      float2 cs = make_float2(0.f, 0.f);
      if (n + 1 < s.n) {
        cs = __ldg(reinterpret_cast<const float2*>(p.col_scale + n));
      } else if (n < s.n) {
        cs.x = __ldg(p.col_scale + n);
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        sum[j * 4 + 2 * h] *= rs[h] * cs.x;
        sum[j * 4 + 2 * h + 1] *= rs[h] * cs.y;
      }
    }
    tapgemm_epilogue_tile<BN, kGeglu, false, false>(s, e, t, est, vec_ok, out_n, q2, sum);
  }
  epi_stage_drain(est);
}

template <int BN>
int launch_fp8_bn(const Fp8GemmParams& p, bool geglu, int grid, size_t smem, cudaStream_t stream) {
  static PerDeviceOnce attr_once;
  if (attr_once.need()) {
    VG_CUDA(cudaFuncSetAttribute(tapgemm_fp8_kernel<BN, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    VG_CUDA(cudaFuncSetAttribute(tapgemm_fp8_kernel<BN, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    attr_once.mark();
  }
  if (geglu)
    launch_kernel(tapgemm_fp8_kernel<BN, true>, dim3(grid), dim3(kThreads), smem, stream, p);
  else
    launch_kernel(tapgemm_fp8_kernel<BN, false>, dim3(grid), dim3(kThreads), smem, stream, p);
  VG_LAUNCH_CHECK("tapgemm_fp8_kernel");
  return 0;
}

// N tile: 128 unless padding n to a multiple of 128 wastes more than a tenth of the tile work (n = 320: 64).
int pick_bn_fp8(long n, bool geglu) {
  if (geglu) return n % 128 == 0 ? 128 : (n % 64 == 0 ? 64 : 0);
  if (n <= 64) return 64;
  const long pad = (n + 127) / 128 * 128;
  return (pad - n) * 10 > pad && n % 64 == 0 ? 64 : 128;
}

// ------------------------------------------------------------------------------------------- row quantiser
// One warp per row: pass 1 takes the row's amax (fp16 |x|, exact), pass 2 writes e4m3(x / scale) with scale = amax / 448
// in fp32 (IEEE division, round-to-nearest-even conversion with saturation: the codes equal torch's
// (x.float() / scale).to(torch.float8_e4m3fn)).  An all-zero row gets scale 1 (codes 0).  8 elements per lane step.
__global__ void quantize_rows_e4m3_kernel(const __half* __restrict__ x, long m, int k, long ldx, uint8_t* __restrict__ q,
                                          long ldq, float* __restrict__ scale) {
  const long row = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= m) return;
  const __half* xr = x + row * ldx;
  float amax = 0.f;
  for (int c = lane * 8; c < k; c += 256) {
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(xr + c));
    const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = __half22float2(__habs2(h[i]));
      amax = fmaxf(amax, fmaxf(f.x, f.y));
    }
  }
  amax = warp_max(amax);
  const float sc = amax > 0.f ? __fdiv_rn(amax, 448.f) : 1.f;
  if (lane == 0) scale[row] = sc;
  uint8_t* qr = q + row * ldq;
  for (int c = lane * 8; c < k; c += 256) {
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(xr + c));
    const __half2* h = reinterpret_cast<const __half2*>(&v);
    uint32_t w[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const float2 a = __half22float2(h[2 * i]), b = __half22float2(h[2 * i + 1]);
      const uint32_t lo = __nv_cvt_float2_to_fp8x2(make_float2(__fdiv_rn(a.x, sc), __fdiv_rn(a.y, sc)), __NV_SATFINITE, __NV_E4M3);
      const uint32_t hi = __nv_cvt_float2_to_fp8x2(make_float2(__fdiv_rn(b.x, sc), __fdiv_rn(b.y, sc)), __NV_SATFINITE, __NV_E4M3);
      w[i] = lo | (hi << 16);
    }
    *reinterpret_cast<uint2*>(qr + c) = make_uint2(w[0], w[1]);
  }
}

}  // namespace
}  // namespace vg

using namespace vg;

extern "C" {

int vgen_quantize_rows_e4m3(const void* x, int64_t m, int64_t k, int64_t ldx, void* q, int64_t ldq, float* scale,
                            void* stream) {
  VG_REQUIRE(x && q && scale, "vgen_quantize_rows_e4m3: null pointer");
  VG_REQUIRE(m >= 0 && k > 0 && ldx >= k && ldq >= k, "vgen_quantize_rows_e4m3: bad shape");
  VG_REQUIRE(k % 8 == 0 && ldx % 8 == 0 && ldq % 8 == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0 &&
                 (reinterpret_cast<uintptr_t>(q) & 7) == 0,
             "vgen_quantize_rows_e4m3: k and the row strides must be multiples of 8, x 16-byte and q 8-byte aligned");
  if (m == 0) return 0;
  constexpr int kRowsPerBlock = 8;
  launch_kernel(quantize_rows_e4m3_kernel, dim3((unsigned)((m + kRowsPerBlock - 1) / kRowsPerBlock)), dim3(32 * kRowsPerBlock),
                0, reinterpret_cast<cudaStream_t>(stream), reinterpret_cast<const __half*>(x), (long)m, (int)k, (long)ldx,
                reinterpret_cast<uint8_t*>(q), (long)ldq, scale);
  VG_LAUNCH_CHECK("quantize_rows_e4m3_kernel");
  return 0;
}

int vgen_linear_fp8(const void* a, const float* a_scale, int64_t m, int64_t k, int64_t lda, const void* w,
                    const float* w_scale, int64_t n, void* out, int64_t ldo, const vgen_epilogue* epi, void* stream) {
  VG_REQUIRE(a && a_scale && w && w_scale && out, "vgen_linear_fp8: null pointer");
  VG_REQUIRE(m >= 0 && k > 0 && n > 0 && lda >= k, "vgen_linear_fp8: bad shape");
  VG_REQUIRE(k % 16 == 0 && lda % 16 == 0 && (reinterpret_cast<uintptr_t>(a) & 15) == 0 &&
                 (reinterpret_cast<uintptr_t>(w) & 15) == 0 && (reinterpret_cast<uintptr_t>(w_scale) & 7) == 0,
             "vgen_linear_fp8: k and lda must be multiples of 16, A and W 16-byte and w_scale 8-byte aligned");
  VG_REQUIRE(m < (1L << 31) && n < (1L << 24), "vgen_linear_fp8: too large");
  if (epi) {
    VG_REQUIRE(!epi->group_bias && !epi->row_stats && !epi->col_sum,
               "vgen_linear_fp8: the e4m3 GEMM takes bias / residual / GEGLU epilogues only");
    VG_REQUIRE(!(epi->geglu && epi->residual), "vgen_linear_fp8: the GEGLU epilogue takes no residual");
  }
  if (m == 0) return 0;
  const bool geglu = epi && epi->geglu;
  const int bn = (epi && epi->bn > 0) ? epi->bn : pick_bn_fp8(n, geglu);
  VG_REQUIRE(bn == 64 || bn == 128, "vgen_linear_fp8: N tile must be 64 or 128 (GEGLU: n % 64 == 0)");
  if (geglu) VG_REQUIRE(n % bn == 0, "vgen_linear_fp8: GEGLU needs n % bn == 0");
  const long out_n = geglu ? n / 2 : n;
  VG_REQUIRE(ldo >= out_n, "vgen_linear_fp8: ldo < output width");

  Fp8GemmParams p;
  memset(&p, 0, sizeof p);
  p.m = (int)m;
  p.kb = (int)((k + kBK - 1) / kBK);
  p.row_scale = a_scale;
  p.col_scale = w_scale;
  TapGemmShape& s = p.s;
  s.c = (int)k;
  s.d1 = (int)m;
  s.d2 = s.d3 = 1;
  s.box1 = kBM;
  s.box2 = 1;
  s.t1 = cdiv(m, kBM);
  s.t2 = 1;
  s.num_taps = 1;
  s.n = (int)n;
  s.bn = bn;
  s.nb = cdiv(n, bn);
  const long tiles = (long)s.t1 * s.nb;
  VG_REQUIRE(tiles < (1L << 31), "vgen_linear_fp8: too many tiles");
  s.total_tiles = (int)tiles;
  tapgemm_prepare_shape(s);

  TapGemmEpilogue& e = p.e;
  e.out = reinterpret_cast<__half*>(out);
  e.ldo = ldo;
  e.alpha = epi ? epi->alpha : 1.0f;
  e.bias = epi ? epi->bias : nullptr;
  e.residual = epi ? reinterpret_cast<const __half*>(epi->residual) : nullptr;
  e.ldr = epi ? epi->residual_ld : 0;
  e.geglu = geglu ? 1 : 0;
  e.f_group_bias_div = make_fastdiv(1);
  e.group_bias_div = 1;
  e.rows_per_group = 1;
  e.f_rows_per_group = make_fastdiv(1);
  if (geglu) VG_REQUIRE(!e.bias || (reinterpret_cast<uintptr_t>(e.bias) & 15) == 0, "vgen_linear_fp8: GEGLU bias must be 16-byte aligned");
  {
    const uint64_t dims[2] = {(uint64_t)k, (uint64_t)m};
    const uint64_t strides[1] = {(uint64_t)lda};
    const uint32_t box[2] = {(uint32_t)kBK, (uint32_t)kBM};
    int rc = make_tmap_u8(&p.map_a, a, 2, dims, strides, box);
    if (rc) return rc;
  }
  {
    const uint64_t dims[2] = {(uint64_t)k, (uint64_t)n};
    const uint64_t strides[1] = {(uint64_t)k};
    const uint32_t box[2] = {(uint32_t)kBK, (uint32_t)bn};
    int rc = make_tmap_u8(&p.map_b, w, 2, dims, strides, box);
    if (rc) return rc;
  }
  p.out_tma = (tapgemm_out_tma_ok(e) && out_n >= 32) ? 1 : 0;
  if (p.out_tma) {
    const uint64_t ld = (uint64_t)ldo * 2;
    const uint64_t dims[4] = {(uint64_t)out_n, (uint64_t)m, 1, 1};
    const uint64_t strides[3] = {ld, ld * (uint64_t)m, ld * (uint64_t)m};
    const uint32_t box[4] = {32, (uint32_t)kBM, 1, 1};
    int rc = make_tmap_f16(&p.map_out, out, 4, dims, strides, box, 64);
    if (rc) return rc;
  }
  const int stage_bytes = kABytes + bn * kBK;
  int stages = (226 * 1024 - kEpiStagingTotal - 2 * kMaxStages * 8) / stage_bytes;
  if (stages > kMaxStages) stages = kMaxStages;
  p.stages = stages;
  const size_t smem = (size_t)stages * stage_bytes + kEpiStagingTotal + 2 * stages * 8 + 1024;
  int grid = sm_count();
  if (grid > s.total_tiles) grid = s.total_tiles;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return bn == 64 ? launch_fp8_bn<64>(p, geglu, grid, smem, st) : launch_fp8_bn<128>(p, geglu, grid, smem, st);
}

}  // extern "C"
