// Epilogue of the tap-GEMM kernel.  The accumulators of a 128 x BN tile live in the registers of the two MMA
// warpgroups in the wgmma fragment layout: a thread owns two rows (g and g + 8 of its warp's 16) and, of every
// 8-column group, the column pair 2 q, 2 q + 1.  It applies alpha, bias, per-frame bias (ResBlock "h + emb_out"),
// residual, folded LayerNorm or GEGLU to those pairs, rounding to fp16 exactly where the reference materialises an
// fp16 tensor, 32 columns (four groups) at a time.
//
// Stores.  A pair is 4 bytes, so direct stores would touch eight 128-byte lines per warp instruction with 16 bytes
// each.  Instead a 32-column chunk of the whole tile is written to a 64B-swizzled staging tile in shared memory
// (conflict-free 4-byte stores) and leaves the SM as ONE TMA tile store: rows x 64 bytes, clipped by the TMA unit
// at the tensor edges.  Two staging tiles ring so the store of chunk i overlaps the math of chunk i+1.  The direct
// path remains for outputs the TMA cannot address (row stride or base not 16-byte aligned).
#pragma once
#include "ptx.cuh"
#include "tapgemm.h"

namespace vg {

// exact-erf GELU (F.gelu default, util.py:714) with erf from Abramowitz-Stegun 7.1.26 (|error| < 1.5e-7, far below
// the fp16 rounding the result receives).  Written so that no cancellation and no sign fix-up is needed:
//   c = 1 - erf(|x|/sqrt2) = poly(t) * t * exp(-x^2/2),  t = 1 / (1 + p |x|/sqrt2)
//   gelu(x) = max(x, 0) - (|x|/2) * c
// and exp(-z^2) = ex2(-u^2) with u = z * sqrt(log2 e): 2 MUFU (rcp, ex2, both .ftz: no denormal fix-up code) + 13
// FMA-pipe instructions (libm erff: ~30; the straightforward 0.5x(1+erf) form with __expf: ~20).
__device__ __forceinline__ float gelu_erf(float x) {
#ifdef VG_GELU_LIBM
  return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f));
#endif
  constexpr float kU = 0.70710678118654752f * 1.2011224087864498f;   // 1/sqrt2 * sqrt(log2 e)
  constexpr float kP = 0.3275911f / 1.2011224087864498f;             // p / sqrt(log2 e)
  const float ax = fabsf(x);
  const float u = ax * kU;
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(u, kP, 1.0f)));
  float poly = fmaf(1.061405429f, t, -1.453152027f);
  poly = fmaf(poly, t, 1.421413741f);
  poly = fmaf(poly, t, -0.284496736f);
  poly = fmaf(poly, t, 0.254829592f);
  const float c = poly * t * fast_exp2(-u * u);
  return fmaxf(x, 0.f) - (0.5f * ax) * c;
}

static constexpr int kEpiStageBytes = 128 * 64;              // one staging tile: 128 rows x 32 fp16
static constexpr int kEpiStagingTotal = 2 * kEpiStageBytes;  // 2 ring slots
static constexpr int kEpiThreads = 256;                      // the two MMA warpgroups
static constexpr int kEpiBarrier = 1;                        // named barrier of those threads

struct EpiTile {
  int nb_i;          // n-block index of the tile
  int i3;            // outermost coordinate (frame) of the tile
  int i1_0, i2_0;    // origin of the tile along d1 / d2 (TMA store coordinates)
  long row[2];       // output rows of this thread
  long ooff[2];      // element offsets of those rows in the output
  bool row_ok[2];    // those rows are inside the tensor
};

struct EpiStore {
  bool tma;                // TMA tile stores (else direct per-thread stores)
  const CUtensorMap* map;  // output [out_n, d1, d2, d3], box {32, box1, box2, 1}, 64B swizzle
  uint32_t stage;          // shared address of the two staging tiles
  uint32_t row_off[2];     // r * 64 + 4 q: this thread's pair inside a 16-byte piece of its rows
  uint32_t row_xor[2];     // (r >> 1) & 3: 64B-swizzle term of those rows
  bool leader;             // the one thread that issues / tracks the bulk stores
  uint32_t slot;           // ring position, carried across chunks and tiles
};

__device__ __forceinline__ bool tapgemm_vec_ok(const TapGemmEpilogue& e, int out_n) {
  return ((reinterpret_cast<uintptr_t>(e.bias) & 15) == 0) && ((e.ldo & 7) == 0) && ((out_n & 7) == 0) &&
         ((reinterpret_cast<uintptr_t>(e.out) & 15) == 0) && ((reinterpret_cast<uintptr_t>(e.group_bias) & 15) == 0) &&
         ((e.ld_group_bias & 7) == 0) &&
         (e.residual == nullptr || (((e.ldr & 7) == 0) && ((reinterpret_cast<uintptr_t>(e.residual) & 15) == 0)));
}

// host side: can the output be written with TMA tile stores?
inline bool tapgemm_out_tma_ok(const TapGemmEpilogue& e) {
  return (reinterpret_cast<uintptr_t>(e.out) & 15) == 0 && (e.ldo & 7) == 0 && (e.out_s2 & 7) == 0 && (e.out_s3 & 7) == 0;
}

// ---- staging-tile protocol ---------------------------------------------------------------------------
// acquire: the slot written two chunks ago must have been read by its TMA store
__device__ __forceinline__ void epi_stage_acquire(EpiStore& st) {
  if (st.leader) bulk_wait_group_read<1>();
  named_bar_sync(kEpiBarrier, kEpiThreads);
}
// the pair of row h in 8-column group g4 (0..3) of the chunk
__device__ __forceinline__ void epi_stage_put(const EpiStore& st, int h, int g4, uint32_t pair) {
  const uint32_t addr = st.stage + st.slot * kEpiStageBytes + st.row_off[h] + ((((uint32_t)g4) ^ st.row_xor[h]) << 4);
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(pair) : "memory");
}
// publish: make the generic-proxy writes visible to the TMA unit, then one thread stores the tile
__device__ __forceinline__ void epi_stage_publish(EpiStore& st, int col, const EpiTile& t) {
  fence_proxy_async_smem();
  named_bar_sync(kEpiBarrier, kEpiThreads);
  if (st.leader) {
    tma_store_4d(st.map, st.stage + st.slot * kEpiStageBytes, col, t.i1_0, t.i2_0, t.i3);
    bulk_commit_group();
  }
  st.slot ^= 1;
}
// before the kernel exits every bulk store must have completed
__device__ __forceinline__ void epi_stage_drain(const EpiStore& st) {
  if (st.tma && st.leader) bulk_wait_group<0>();
}

__device__ __forceinline__ float round_h(float x) { return __half2float(__float2half_rn(x)); }

// kGeglu / kLn / kGelu are template parameters of the kernel: the epilogues have very different register needs.
// kLn: LayerNorm folded into the GEMM (TapGemmEpilogue.row_stats / col_sum): the accumulator row is scaled by the row's
// rstd and shifted by (-mean * rstd) * col_sum[n]; such launches carry no residual / per-frame bias.
// kGelu: adapter down projection (util.py:512-515): gelu_erf(acc + bias + row_bias[row / rows_per_group]) in fp32 and one
// fp16 rounding at the store (the fp32 row bias carries the adapter's condition term); no residual / per-frame bias.
// kRelu: relu(acc * alpha + bias) in fp32 and one fp16 rounding at the store; no residual / per-frame bias.
// q2 = 2 * (lane % 4): this thread's column pair inside every 8-column group.
template <int BN, bool kGeglu, bool kLn, bool kGelu, bool kRelu = false>
__device__ __forceinline__ void tapgemm_epilogue_tile(const TapGemmShape& s, const TapGemmEpilogue& e, const EpiTile& t,
                                                      EpiStore& st, bool vec_ok, int out_n, int q2, float (&acc)[BN / 2]) {
  float ln_scale[2] = {e.alpha, e.alpha}, ln_shift[2] = {0.f, 0.f};   // kLn: rstd (* alpha) and -mean * rstd of the rows
  if (kLn) {
#pragma unroll
    for (int h = 0; h < 2; ++h)
      if (t.row_ok[h]) {
        const float2 rs = __ldg(e.row_stats + t.row[h]);
        ln_scale[h] = rs.x * e.alpha;
        ln_shift[h] = rs.y * e.alpha;
      }
  }
  __half* orow[2] = {e.out + t.ooff[0], e.out + t.ooff[1]};
  constexpr bool kResidual = !kLn && !kGelu && !kRelu;   // the launchers refuse a residual with the other epilogues
  if constexpr (!kGeglu) {
    const int n0 = t.nb_i * BN;
    const __half* grow = e.group_bias ? e.group_bias + (long)fd_div(e.f_group_bias_div, t.i3) * e.ld_group_bias : nullptr;
    const float* rrb[2] = {nullptr, nullptr};   // kGelu: this thread's rows of the row bias
    if (kGelu && e.row_bias) {
#pragma unroll
      for (int h = 0; h < 2; ++h)
        if (t.row_ok[h]) rrb[h] = e.row_bias + (long)fd_div(e.f_rows_per_group, (int)t.row[h]) * e.ld_row_bias;
    }
#pragma unroll
    for (int c = 0; c < BN / 32; ++c) {
      const int nbase = n0 + c * 32;
      if (nbase >= s.n) break;  // uniform over the CTA
      const bool full = nbase + 32 <= s.n;
      const bool vec = vec_ok && full;               // pairs are loaded / stored as 4- or 8-byte words
      const bool staged = st.tma && vec;             // uniform over the CTA
      // The chunk's residual pairs are loaded up front, all in flight together: the staging stores below carry a
      // "memory" clobber, so a load left in the loop would wait for the previous store and the chunk would pay one
      // DRAM latency per pair.
      __half2 res[4][2];
      if (kResidual && e.residual) {
#pragma unroll
        for (int g4 = 0; g4 < 4; ++g4) {
          const int n = nbase + g4 * 8 + q2;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            res[g4][h] = __float2half2_rn(0.f);
            if (!t.row_ok[h]) continue;
            const __half* rrow = e.residual + t.row[h] * e.ldr;
            if (vec) {
              res[g4][h] = __ldg(reinterpret_cast<const __half2*>(rrow + n));
            } else {
              if (n < s.n) res[g4][h].x = rrow[n];
              if (n + 1 < s.n) res[g4][h].y = rrow[n + 1];
            }
          }
        }
      }
      if (staged) epi_stage_acquire(st);
#pragma unroll
      for (int g4 = 0; g4 < 4; ++g4) {
        const int n = nbase + g4 * 8 + q2;
        float2 b = make_float2(0.f, 0.f), cs = b, gb = b;
        const bool have_g = !kLn && grow != nullptr;
        if (vec) {
          if (e.bias) b = __ldg(reinterpret_cast<const float2*>(e.bias + n));
          if (kLn) cs = __ldg(reinterpret_cast<const float2*>(e.col_sum + n));
          if (have_g) gb = __half22float2(__ldg(reinterpret_cast<const __half2*>(grow + n)));
        } else {
          if (n < s.n) {
            if (e.bias) b.x = e.bias[n];
            if (kLn) cs.x = e.col_sum[n];
            if (have_g) gb.x = __half2float(grow[n]);
          }
          if (n + 1 < s.n) {
            if (e.bias) b.y = e.bias[n + 1];
            if (kLn) cs.y = e.col_sum[n + 1];
            if (have_g) gb.y = __half2float(grow[n + 1]);
          }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float f0 = acc[(c * 4 + g4) * 4 + 2 * h] * ln_scale[h] + b.x;
          float f1 = acc[(c * 4 + g4) * 4 + 2 * h + 1] * ln_scale[h] + b.y;
          if (kLn) {
            f0 = fmaf(ln_shift[h], cs.x, f0);
            f1 = fmaf(ln_shift[h], cs.y, f1);
          }
          if (kGelu) {
            if (rrb[h]) {
              if (vec) {
                const float2 g = __ldg(reinterpret_cast<const float2*>(rrb[h] + n));
                f0 += g.x;
                f1 += g.y;
              } else {
                if (n < s.n) f0 += rrb[h][n];
                if (n + 1 < s.n) f1 += rrb[h][n + 1];
              }
            }
            f0 = gelu_erf(f0);
            f1 = gelu_erf(f1);
          }
          if (kRelu) {
            f0 = fmaxf(f0, 0.f);
            f1 = fmaxf(f1, 0.f);
          }
          if (have_g) {
            // reference: h (fp16 conv output) + emb_out (fp16) -> fp16  (util.py:909-919)
            f0 = round_h(f0) + gb.x;
            f1 = round_h(f1) + gb.y;
          }
          if (kResidual && e.residual && t.row_ok[h]) {
            if (vec || n < s.n) f0 = round_h(f0) + __low2float(res[g4][h]);
            if (vec || n + 1 < s.n) f1 = round_h(f1) + __high2float(res[g4][h]);
          }
          if (staged) {
            epi_stage_put(st, h, g4, pack_half2(f0, f1));   // rows outside the tensor are clipped by the TMA unit
          } else if (t.row_ok[h]) {
            if (vec) {
              *reinterpret_cast<uint32_t*>(orow[h] + n) = pack_half2(f0, f1);
            } else {
              if (n < s.n) orow[h][n] = __float2half_rn(f0);
              if (n + 1 < s.n) orow[h][n + 1] = __float2half_rn(f1);
            }
          }
        }
      }
      if (staged) epi_stage_publish(st, nbase, t);
    }
  } else {
    // GEGLU: columns [0,BN/2) of this tile are "value" j, columns [BN/2,BN) the matching "gate" j
    // (host interleaves the weight rows per BN block).  out = value * gelu(gate)   (util.py:707-714)
    constexpr int hb = BN / 2;
    const int o0 = t.nb_i * hb;
#pragma unroll
    for (int c = 0; c < hb / 32; ++c) {
      const int obase = o0 + c * 32;
      if (obase >= out_n) break;  // uniform over the CTA
      const bool full = obase + 32 <= out_n;
      const bool vec = vec_ok && full;
      const bool staged = st.tma && vec;
      if (staged) epi_stage_acquire(st);
#pragma unroll
      for (int g4 = 0; g4 < 4; ++g4) {
        const int j = c * 32 + g4 * 8 + q2;       // value column inside the tile (gate is + hb)
        const int wv = t.nb_i * BN + j;           // packed weight-row index of the value (bias / col_sum index)
        float2 bv = make_float2(0.f, 0.f), bg = bv, cv = bv, cg = bv;
        if (e.bias) {  // packed bias is 16-byte aligned and wv is even
          bv = __ldg(reinterpret_cast<const float2*>(e.bias + wv));
          bg = __ldg(reinterpret_cast<const float2*>(e.bias + wv + hb));
        }
        if (kLn) {
          cv = __ldg(reinterpret_cast<const float2*>(e.col_sum + wv));
          cg = __ldg(reinterpret_cast<const float2*>(e.col_sum + wv + hb));
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int iv = (c * 4 + g4) * 4 + 2 * h, ig = iv + (hb / 8) * 4;
          // shift = bias + (-mean rstd) * col_sum, per packed weight row
          const float sv0 = fmaf(ln_shift[h], cv.x, bv.x), sv1 = fmaf(ln_shift[h], cv.y, bv.y);
          const float sg0 = fmaf(ln_shift[h], cg.x, bg.x), sg1 = fmaf(ln_shift[h], cg.y, bg.y);
          // reference: the projection is an fp16 tensor, gelu(gate) an fp16 tensor, their product an fp16 tensor.
          // Pairs are kept packed: value and gelu(gate) are rounded by the f32x2 -> f16x2 pack, the product is one
          // HMUL2 (an fp16 x fp16 product is exact in fp32, so rounding it once is what the reference computes).
          const __half2 a2 = __floats2half2_rn(fmaf(acc[iv], ln_scale[h], sv0), fmaf(acc[iv + 1], ln_scale[h], sv1));
          const float2 b2 = __half22float2(__floats2half2_rn(fmaf(acc[ig], ln_scale[h], sg0), fmaf(acc[ig + 1], ln_scale[h], sg1)));
          const __half2 o2 = __hmul2(a2, __floats2half2_rn(gelu_erf(b2.x), gelu_erf(b2.y)));
          const int on = obase + g4 * 8 + q2;
          if (staged) {
            epi_stage_put(st, h, g4, *reinterpret_cast<const uint32_t*>(&o2));
          } else if (t.row_ok[h]) {
            if (vec) {
              *reinterpret_cast<__half2*>(orow[h] + on) = o2;
            } else {
              if (on < out_n) orow[h][on] = __low2half(o2);
              if (on + 1 < out_n) orow[h][on + 1] = __high2half(o2);
            }
          }
        }
      }
      if (staged) epi_stage_publish(st, obase, t);
    }
  }
}

}  // namespace vg
