// tapgemm: the one tensor-core kernel behind every conv / linear of the UNet and the VAE.
//
//   out[row, n] = epilogue( sum_{tap} sum_{c} A[coord(row) + offset(tap), c] * W[n, tap*C + c] )
//
// A is an fp16 activation tensor in channels-last layout, viewed as a rank-4 box-tiled TMA tensor
// {C, d1, d2, d3}.  A "tap" is a coordinate offset (e.g. the 9 taps of a 3x3 conv, the 3 taps of the
// temporal (3,1,1) conv, or the single tap of a linear / 1x1 conv).  Out-of-range coordinates are
// zero-filled by the TMA unit, which IS the conv's zero padding - there is no im2col buffer and no
// halo handling in the kernel.  Per k-iteration the producer issues one 4-D box load of A
// ([box2][box1][64 ch], 128B-swizzled, = the 128-row K-major wgmma A tile) and one 2-D load of W.
//
// Reference ops this replaces (all cuDNN / cuBLAS calls in the reference):
//   nn.Conv2d 3x3 in ResBlock          tools/modules/unet/util.py:845-876
//   nn.Conv3d (3,1,1) TemporalConvBlock_v2                                   util.py:1662-1680
//   nn.Linear (q/k/v/out, GEGLU, FF, proj_in/out)                            util.py:224-229,707-741,338
//   nn.Conv1d k=1 (TemporalTransformer proj)                                 util.py:1213,1229
//   VAE conv3x3 / 1x1                  tools/modules/autoencoder.py:282-335,344-363
//
// Structure (sm_90a): persistent CTAs (one per SM) of three warpgroups, warp-specialised:
//   warpgroup 0    warp 0 is the TMA producer (one elected lane): kStages-deep smem ring, mbarrier full/empty;
//                  the warpgroup hands most of its registers to the other two (setmaxnreg)
//   warpgroups 1-2 wgmma consumers: each owns 64 of the tile's 128 rows, fp32 accumulators in registers
//                  (64 x BN per warpgroup), then the epilogue on those registers: alpha / bias / per-frame bias /
//                  residual / GEGLU -> fp16 -> staging tile -> TMA store
// While the consumers run the epilogue of tile i the producer already fills the ring with tile i+1.
#include "common.h"
#include "ptx.cuh"
#include "tapgemm.h"
#include "tapgemm_epilogue.cuh"

namespace vg {

static constexpr int kBM = 128;       // rows per tile (two wgmma M = 64 halves)
static constexpr int kBK = 64;        // K per pipeline stage = one 128B swizzle row of fp16
static constexpr int kThreads = 384;  // producer warpgroup + two consumer warpgroups
static constexpr int kABytes = kBM * kBK * 2;  // 16 KB
static constexpr int kMaxStages = 8;

struct alignas(64) TapGemmKernelParams {
  CUtensorMap map_a;
  CUtensorMap map_b;
  CUtensorMap map_out;  // output, box {32, box1, box2, 1}, 64B swizzle (TMA tile stores of the epilogue)
  int out_tma;          // 1: map_out is valid
  TapGemmShape s;
  TapGemmEpilogue e;
  int stages;
  CUtensorMap map_h;    // K tail (kEpi bit 4): H [rows][r] as a rank-4 map shaped like map_a, and U [n][r]
  CUtensorMap map_u;
  int tail_iters;       // r / 64
};

// kEpi: bit 0 = GEGLU epilogue, bit 1 = LayerNorm folded into the epilogue (TapGemmEpilogue.row_stats), bit 2 = GELU with the
// fp32 row bias (TapGemmEpilogue.gelu), bit 3 = ReLU (TapGemmEpilogue.relu), bit 4 = K tail (TapGemmArgs.h / u: r / 64 more
// k-iterations after the main loop, H and U tiles loaded through their own maps into the same ring stages); BN (the wgmma N and the accumulator count) is a
// template parameter as well, so every register index of the epilogue is a constant.
template <int BN, int kEpi>
__global__ void __launch_bounds__(kThreads, 1) tapgemm_sm90_kernel(const __grid_constant__ TapGemmKernelParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // 1024B alignment is required by the 128B swizzle atom (8 rows x 128 B).
  constexpr bool kGeglu = (kEpi & 1) != 0, kLn = (kEpi & 2) != 0, kGelu = (kEpi & 4) != 0, kRelu = (kEpi & 8) != 0;
  constexpr bool kTail = (kEpi & 16) != 0;
  constexpr int kBBytes = BN * kBK * 2;                            // multiple of 1024 (BN % 32 == 0)
  constexpr int kStageBytes = kABytes + kBBytes;
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  const int stages = p.stages;

  uint8_t* tiles = smem;
  uint8_t* staging = smem + (size_t)stages * kStageBytes;   // epilogue staging tiles (1024-aligned)
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(staging + kEpiStagingTotal);   // [stages]
  uint64_t* empty_bar = full_bar + stages;                                          // [stages]

  const TapGemmShape& s = p.s;
  const int k_iters = s.num_taps * s.kc + (kTail ? p.tail_iters : 0);
  const uint32_t stage_tx = (uint32_t)(s.box1 * s.box2 * kBK * 2 + kBBytes);

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&p.map_a);
    tma_prefetch_desc(&p.map_b);
    if (p.out_tma) tma_prefetch_desc(&p.map_out);
    if constexpr (kTail) {
      tma_prefetch_desc(&p.map_h);
      tma_prefetch_desc(&p.map_u);
    }
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
    // the whole warp walks the loop (warp-uniform operands); one elected lane issues the TMA
    int st = 0;
    uint32_t ph = 0;  // ring position / phase, carried across tiles
    for (int tile = blockIdx.x; tile < s.total_tiles; tile += gridDim.x) {
      int m, nb_i, rest, t1_i, i3, t2_i;
      fd_divmod(s.f_nb, tile, m, nb_i);
      fd_divmod(s.f_t1, m, rest, t1_i);
      fd_divmod(s.f_t2, rest, i3, t2_i);
      const int i1_0 = t1_i * s.box1, i2_0 = t2_i * s.box2, n0 = nb_i * BN;
      for (int tap = 0; tap < s.num_taps; ++tap) {
        const int c1 = i1_0 + s.tap1[tap], c2 = i2_0 + s.tap2[tap], c3 = i3 + s.tap3[tap];
        const int wk0 = tap * s.c;
        for (int kc_i = 0; kc_i < s.kc; ++kc_i) {
          mbar_wait(&empty_bar[st], ph ^ 1);
          if (elect_one()) {
            mbar_expect_tx(&full_bar[st], stage_tx);
            uint8_t* sa = tiles + (size_t)st * kStageBytes;
            tma_load_4d(sa, &p.map_a, &full_bar[st], kc_i * kBK, c1, c2, c3);
            tma_load_2d(sa + kABytes, &p.map_b, &full_bar[st], wk0 + kc_i * kBK, n0);
          }
          __syncwarp();
          if (++st == stages) {
            st = 0;
            ph ^= 1;
          }
        }
      }
      if constexpr (kTail) {   // the tail tiles have the main loop's A / B tile shapes, so the consumers cannot tell them apart
        for (int r = 0; r < p.tail_iters; ++r) {
          mbar_wait(&empty_bar[st], ph ^ 1);
          if (elect_one()) {
            mbar_expect_tx(&full_bar[st], stage_tx);
            uint8_t* sa = tiles + (size_t)st * kStageBytes;
            tma_load_4d(sa, &p.map_h, &full_bar[st], r * kBK, i1_0, i2_0, i3);
            tma_load_2d(sa + kABytes, &p.map_u, &full_bar[st], r * kBK, n0);
          }
          __syncwarp();
          if (++st == stages) {
            st = 0;
            ph ^= 1;
          }
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- wgmma consumers + epilogue
  setmaxnreg_inc<232>();
  const TapGemmEpilogue& e = p.e;
  const int cw = wg - 1;                                 // consumer warpgroup: rows [64 cw, 64 cw + 64) of the tile
  const int r0 = cw * 64 + (warp & 3) * 16 + (lane >> 2);  // this thread's rows are r0 and r0 + 8
  const int q2 = (lane & 3) * 2;
  const int rows_in_tile = s.box1 * s.box2;
  const int out_n = kGeglu ? (s.n >> 1) : s.n;
  const bool vec_ok = tapgemm_vec_ok(e, out_n);
  int r1[2], r2[2];                 // position of the rows inside the box (tile-invariant)
  fd_divmod(s.f_box1, r0, r2[0], r1[0]);
  fd_divmod(s.f_box1, r0 + 8, r2[1], r1[1]);
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
  float acc[BN / 2];
  for (int tile = blockIdx.x; tile < s.total_tiles; tile += gridDim.x) {
    int prev = -1;   // stage whose wgmmas are still in flight
    for (int it = 0; it < k_iters; ++it) {
      mbar_wait(&full_bar[st], ph);
      const uint32_t a_addr = tiles_addr + (uint32_t)st * (uint32_t)kStageBytes;
      const uint64_t a_desc = wgmma_desc_sw128(a_addr + (uint32_t)cw * 64u * 128u, 16, 1024);
      const uint64_t b_desc = wgmma_desc_sw128(a_addr + kABytes, 16, 1024);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kBK / 16; ++k) {
        // advance 16 elements (32 B) along K inside the swizzle atom: +2 in the >>4 address field
        wgmma_ss<BN>(acc, a_desc + 2 * k, b_desc + 2 * k, (it | k) != 0 ? 1 : 0);
      }
      wgmma_commit();
      if (prev >= 0) {
        wgmma_wait<1>();   // the previous stage has been read: hand it back to the producer
        if (lane == 0) mbar_arrive(&empty_bar[prev]);
      }
      prev = st;
      if (++st == stages) {
        st = 0;
        ph ^= 1;
      }
    }
    wgmma_wait<0>();
    wgmma_pin(acc);
    if (lane == 0) mbar_arrive(&empty_bar[prev]);

    EpiTile t;
    int m, rest, t1_i, t2_i;
    fd_divmod(s.f_nb, tile, m, t.nb_i);
    fd_divmod(s.f_t1, m, rest, t1_i);
    fd_divmod(s.f_t2, rest, t.i3, t2_i);
    t.i1_0 = t1_i * s.box1;
    t.i2_0 = t2_i * s.box2;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int i1 = t.i1_0 + r1[h], i2 = t.i2_0 + r2[h];
      t.row_ok[h] = (r0 + 8 * h < rows_in_tile) && (i1 < s.d1) && (i2 < s.d2);
      t.row[h] = ((long)t.i3 * s.d2 + i2) * s.d1 + i1;
      // strided output (transposed-conv phases) exists only with the ReLU epilogue: the other kinds keep dense rows
      t.ooff[h] = (kRelu && e.out_s2) ? (long)i1 * e.ldo + (long)i2 * e.out_s2 + (long)t.i3 * e.out_s3 : t.row[h] * e.ldo;
    }
    tapgemm_epilogue_tile<BN, kGeglu, kLn, kGelu, kRelu>(s, e, t, est, vec_ok, out_n, q2, acc);
  }
  epi_stage_drain(est);
}

// ------------------------------------------------------------------------------------------- host
template <int BN>
static int launch_bn(const TapGemmKernelParams& p, int kind, int grid, size_t smem, cudaStream_t stream) {
  static PerDeviceOnce attr_once;
  if (attr_once.need()) {
    VG_CUDA(cudaFuncSetAttribute(tapgemm_sm90_kernel<BN, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    VG_CUDA(cudaFuncSetAttribute(tapgemm_sm90_kernel<BN, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    VG_CUDA(cudaFuncSetAttribute(tapgemm_sm90_kernel<BN, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    VG_CUDA(cudaFuncSetAttribute(tapgemm_sm90_kernel<BN, 16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    if constexpr (BN < 256)
      VG_CUDA(cudaFuncSetAttribute(tapgemm_sm90_kernel<BN, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    if constexpr (BN % 64 == 0) {
      VG_CUDA(cudaFuncSetAttribute(tapgemm_sm90_kernel<BN, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
      VG_CUDA(cudaFuncSetAttribute(tapgemm_sm90_kernel<BN, 3>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    }
    attr_once.mark();
  }
  if constexpr (BN % 64 == 0) {
    if (kind == 3) launch_kernel(tapgemm_sm90_kernel<BN, 3>, dim3(grid), dim3(kThreads), smem, stream, p);
    if (kind == 1) launch_kernel(tapgemm_sm90_kernel<BN, 1>, dim3(grid), dim3(kThreads), smem, stream, p);
  }
  if constexpr (BN < 256) {   // the GELU epilogue spills at BN = 256: pick_bn stops at 224, a forced 256 is refused
    if (kind == 4) launch_kernel(tapgemm_sm90_kernel<BN, 4>, dim3(grid), dim3(kThreads), smem, stream, p);
  }
  if (kind == 16) launch_kernel(tapgemm_sm90_kernel<BN, 16>, dim3(grid), dim3(kThreads), smem, stream, p);
  if (kind == 8) launch_kernel(tapgemm_sm90_kernel<BN, 8>, dim3(grid), dim3(kThreads), smem, stream, p);
  if (kind == 2) launch_kernel(tapgemm_sm90_kernel<BN, 2>, dim3(grid), dim3(kThreads), smem, stream, p);
  if (kind == 0) launch_kernel(tapgemm_sm90_kernel<BN, 0>, dim3(grid), dim3(kThreads), smem, stream, p);
  VG_LAUNCH_CHECK("tapgemm_sm90_kernel");
  return 0;
}

int tapgemm_sm90_launch(const TapGemmArgs& a, cudaStream_t stream) {
  const TapGemmShape& s = a.shape;
  VG_REQUIRE(s.c % 64 == 0, "tapgemm_sm90: C must be a multiple of 64");
  VG_REQUIRE(s.bn >= 32 && s.bn <= 256 && s.bn % 32 == 0, "tapgemm_sm90: BN must be in [32,256], multiple of 32");
  VG_REQUIRE(s.box1 >= 1 && s.box2 >= 1 && s.box1 * s.box2 <= kBM && s.box1 <= 256 && s.box2 <= 256,
             "tapgemm_sm90: bad box");
  VG_REQUIRE(s.num_taps >= 1 && s.num_taps <= kMaxTaps, "tapgemm_sm90: bad tap count");
  VG_REQUIRE((reinterpret_cast<uintptr_t>(a.a) & 15) == 0 && (reinterpret_cast<uintptr_t>(a.w) & 15) == 0,
             "tapgemm_sm90: A and W must be 16-byte aligned");
  if (a.epi.geglu) VG_REQUIRE(s.bn % 64 == 0 && s.n % s.bn == 0, "tapgemm_sm90: GEGLU needs BN%64==0 and N%BN==0");
  if (a.epi.geglu) VG_REQUIRE(!a.epi.residual && !a.epi.group_bias && (reinterpret_cast<uintptr_t>(a.epi.bias) & 15) == 0,
                             "tapgemm_sm90: GEGLU takes no residual / per-frame bias and needs a 16-byte aligned bias");
  if (a.epi.row_stats) VG_REQUIRE(!a.epi.residual && !a.epi.group_bias && s.num_taps == 1 && s.d2 == 1 && s.d3 == 1,
                                  "tapgemm: a folded LayerNorm goes with a plain linear (no residual / per-frame bias)");
  if (a.epi.gelu) VG_REQUIRE(s.bn <= kMaxBnGelu, "tapgemm_sm90: the GELU epilogue needs BN <= 224");
  if (a.epi.gelu) VG_REQUIRE(!a.epi.geglu && !a.epi.row_stats && !a.epi.residual && !a.epi.group_bias && s.num_taps == 1 &&
                             s.d2 == 1 && s.d3 == 1, "tapgemm: the GELU / row-bias epilogue goes with a plain linear");
  if (a.epi.relu) VG_REQUIRE(!a.epi.geglu && !a.epi.row_stats && !a.epi.gelu && !a.epi.residual && !a.epi.group_bias,
                             "tapgemm: the ReLU epilogue goes with bias only");
  VG_REQUIRE(!a.epi.out_s2 || a.epi.relu, "tapgemm_sm90: a strided output goes with the ReLU epilogue");
  if (a.r) VG_REQUIRE(a.r % 64 == 0 && s.num_taps == 1 && s.d2 == 1 && s.d3 == 1 && !a.epi.geglu && !a.epi.row_stats &&
                      !a.epi.gelu && !a.epi.relu && !a.epi.group_bias,
                      "tapgemm_sm90: the K tail goes with a plain linear (bias / residual only), r a multiple of 64");

  TapGemmKernelParams p;
  p.s = s;
  tapgemm_prepare_shape(p.s);
  p.e = a.epi;
  p.e.f_group_bias_div = make_fastdiv(p.e.group_bias_div > 1 ? p.e.group_bias_div : 1);
  p.e.f_rows_per_group = make_fastdiv(p.e.rows_per_group > 1 ? p.e.rows_per_group : 1);
  {
    const uint64_t dims[4] = {(uint64_t)s.c, (uint64_t)s.d1, (uint64_t)s.d2, (uint64_t)s.d3};
    const uint64_t strides[3] = {(uint64_t)a.a_stride1 * 2, (uint64_t)a.a_stride2 * 2, (uint64_t)a.a_stride3 * 2};
    const uint32_t box[4] = {64, (uint32_t)s.box1, (uint32_t)s.box2, 1};
    int rc = make_tmap_f16(&p.map_a, a.a, 4, dims, strides, box);
    if (rc) return rc;
  }
  {
    const uint64_t dims[2] = {(uint64_t)s.num_taps * s.c, (uint64_t)s.n};
    const uint64_t strides[1] = {(uint64_t)s.num_taps * s.c * 2};
    const uint32_t box[2] = {64, (uint32_t)s.bn};
    int rc = make_tmap_f16(&p.map_b, a.w, 2, dims, strides, box);
    if (rc) return rc;
  }
  p.tail_iters = a.r / kBK;
  if (a.r) {
    VG_REQUIRE((reinterpret_cast<uintptr_t>(a.h) & 15) == 0 && (reinterpret_cast<uintptr_t>(a.u) & 15) == 0 && a.ldh % 8 == 0,
               "tapgemm_sm90: H and U must be 16-byte aligned, ldh a multiple of 8");
    const uint64_t hdims[4] = {(uint64_t)a.r, (uint64_t)s.d1, 1, 1};
    const uint64_t hstrides[3] = {(uint64_t)a.ldh * 2, (uint64_t)a.ldh * 2 * s.d1, (uint64_t)a.ldh * 2 * s.d1};
    const uint32_t hbox[4] = {64, (uint32_t)s.box1, (uint32_t)s.box2, 1};
    int rc = make_tmap_f16(&p.map_h, a.h, 4, hdims, hstrides, hbox);
    if (rc) return rc;
    const uint64_t udims[2] = {(uint64_t)a.r, (uint64_t)s.n};
    const uint64_t ustrides[1] = {(uint64_t)a.r * 2};
    const uint32_t ubox[2] = {64, (uint32_t)s.bn};
    rc = make_tmap_f16(&p.map_u, a.u, 2, udims, ustrides, ubox);
    if (rc) return rc;
  }
  const int stage_bytes = kABytes + s.bn * kBK * 2;
  const int out_n = a.epi.geglu ? s.n / 2 : s.n;
  p.out_tma = (tapgemm_out_tma_ok(a.epi) && out_n >= 32) ? 1 : 0;
  if (p.out_tma) {
    const uint64_t ld = (uint64_t)a.epi.ldo * 2;
    const uint64_t dims[4] = {(uint64_t)out_n, (uint64_t)s.d1, (uint64_t)s.d2, (uint64_t)s.d3};
    const uint64_t strides[3] = {ld, a.epi.out_s2 ? (uint64_t)a.epi.out_s2 * 2 : ld * s.d1,
                                 a.epi.out_s2 ? (uint64_t)a.epi.out_s3 * 2 : ld * s.d1 * s.d2};
    const uint32_t box[4] = {32, (uint32_t)s.box1, (uint32_t)s.box2, 1};
    int rc = make_tmap_f16(&p.map_out, a.epi.out, 4, dims, strides, box, 64);
    if (rc) return rc;
  }
  // 227 KB of shared memory per block: the ring takes what the staging tiles, the barriers and the alignment slack leave
  int stages = (226 * 1024 - kEpiStagingTotal - 2 * kMaxStages * 8) / stage_bytes;
  if (stages > kMaxStages) stages = kMaxStages;
  p.stages = stages;
  const size_t smem = (size_t)stages * stage_bytes + kEpiStagingTotal + 2 * stages * 8 + 1024;

  int grid = sm_count();
  if (grid > s.total_tiles) grid = s.total_tiles;
  if (grid < 1) return 0;
  const int kind = (a.epi.geglu ? 1 : 0) | (a.epi.row_stats ? 2 : 0) | (a.epi.gelu ? 4 : 0) | (a.epi.relu ? 8 : 0) | (a.r ? 16 : 0);
  switch (s.bn) {
    case 32: return launch_bn<32>(p, kind, grid, smem, stream);
    case 64: return launch_bn<64>(p, kind, grid, smem, stream);
    case 96: return launch_bn<96>(p, kind, grid, smem, stream);
    case 128: return launch_bn<128>(p, kind, grid, smem, stream);
    case 160: return launch_bn<160>(p, kind, grid, smem, stream);
    case 192: return launch_bn<192>(p, kind, grid, smem, stream);
    case 224: return launch_bn<224>(p, kind, grid, smem, stream);
    default: return launch_bn<256>(p, kind, grid, smem, stream);
  }
}

}  // namespace vg
