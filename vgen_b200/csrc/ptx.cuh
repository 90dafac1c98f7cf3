// Thin inline-PTX wrappers for the sm_90a features the kernels use:
// mbarrier, TMA (cp.async.bulk.tensor), wgmma (fence / mma_async / commit / wait), fences.
// Everything here is hand-written for sm_90a; there is no fallback path.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace vg {

// A wait that takes longer than this many SM cycles is a deadlock (a broken pipeline),
// not a slow kernel: trap instead of hanging the GPU.
#ifndef VG_WATCHDOG_CYCLES
#define VG_WATCHDOG_CYCLES (3000000000LL)
#endif

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ----------------------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ uint32_t mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok;
}
// non-blocking probe: has the phase with this parity completed?
__device__ __forceinline__ uint32_t mbar_test_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok;
}
__device__ __forceinline__ void st_shared_v4(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
// (no printf on the way out: a function call inside a wgmma pipeline makes ptxas serialise the wgmmas and drop setmaxnreg)
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > VG_WATCHDOG_CYCLES) __trap();
  }
}

// One lane of a fully-converged warp (elect.sync).  The single-thread TMA instructions are issued
// under this predicate while the WHOLE warp runs the surrounding loop, so their operands stay warp-uniform
// (uniform registers) instead of going through per-instruction R2UR "waterfall" loops.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

// ----------------------------------------------------------------------------- fences
// generic-proxy writes to shared memory -> visible to the async proxy (TMA / wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ----------------------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}
// TMA tile store (shared -> global), tracked by the issuing thread's bulk async-group
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* map, uint32_t smem_src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(map),
               "r"(smem_src), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_group_read() {  // <= N groups may still be READING their smem source
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void bulk_wait_group() {       // <= N groups not yet complete (writes visible)
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0,
                                            int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0,
                                            int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], "
      "[%2];" ::"r"(smem_u32(smem_dst)),
      "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
// same, destination given as a shared-window address (the void* argument is ignored)
__device__ __forceinline__ void tma_load_4d(void*, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3,
                                            uint32_t smem_dst_addr) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, "
      "%6}], [%2];" ::"r"(smem_dst_addr),
      "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0,
                                            int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, "
      "%6}], [%2];" ::"r"(smem_u32(smem_dst)),
      "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// ----------------------------------------------------------------------------- wgmma (sm_90a)
// Shared-memory matrix descriptor, 128-byte swizzle (the layout a SWIZZLE_128B TMA box of 64 fp16 lands in).
//   bits [0,14)  start address >> 4        bits [16,30) leading byte offset >> 4
//   bits [32,46) stride byte offset >> 4   bits [62,64) swizzle (1 = 128 B)
// K-major operand: 8-row groups are `sbo` bytes apart (1024 for dense 128-byte rows), lbo is unused.
// MN-major operand (one 64-element atom wide): 8-row groups along K are 1024 bytes apart.
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}
// Accumulator registers touched by ordinary code -> ordered before the next wgmma of this warpgroup.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {  // <= N committed groups still running
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// Compiler-level pin, no instruction: the accumulators are (re)defined HERE, i.e. after the wgmma_wait that precedes this
// call -- without it the compiler may read them above the wait, whose asm statement does not name them.
template <int N>
__device__ __forceinline__ void wgmma_pin(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// Register budget of a warpgroup (warp-specialised kernels: the TMA warpgroup gives registers to the MMA warpgroups).
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }

// D[64 x N, fp32 registers] (+)= A[64 x 16, smem] * B[N x 16, smem]^T, fp16 operands, both K-major.
// Fragment layout (thread t of the warpgroup, w = t / 32, g = (t % 32) / 4, q = t % 4): d[4 j + e] is row 16 w + g,
// column 8 j + 2 q + e; d[4 j + 2 + e] is row 16 w + g + 8 of the same column.
template <int N>
__device__ __forceinline__ void wgmma_ss(float (&d)[N / 2], uint64_t a_desc, uint64_t b_desc, int accumulate);

#define VG_PH_0 "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15"
#define VG_PH_1 ",%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31"
#define VG_PH_2 ",%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47"
#define VG_PH_3 ",%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63"
#define VG_PH_4 ",%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79"
#define VG_PH_5 ",%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95"
#define VG_PH_6 ",%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111"
#define VG_PH_7 ",%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127"
#define VG_D16(o)                                                                                                   \
  "+f"(d[o + 0]), "+f"(d[o + 1]), "+f"(d[o + 2]), "+f"(d[o + 3]), "+f"(d[o + 4]), "+f"(d[o + 5]), "+f"(d[o + 6]),   \
      "+f"(d[o + 7]), "+f"(d[o + 8]), "+f"(d[o + 9]), "+f"(d[o + 10]), "+f"(d[o + 11]), "+f"(d[o + 12]),            \
      "+f"(d[o + 13]), "+f"(d[o + 14]), "+f"(d[o + 15])
// N: instruction N; PH: placeholder list of the N / 2 accumulators; A, B, S: operand numbers that follow them
#define VG_WGMMA_SS(N, PH, A, B, S, ...)                                                                         \
  template <>                                                                                                    \
  __device__ __forceinline__ void wgmma_ss<N>(float (&d)[N / 2], uint64_t a_desc, uint64_t b_desc, int accumulate) { \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" #S ", 0;\n\t"                                        \
                 "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32.f16.f16 {" PH "}, %" #A ", %" #B ", p, 1, 1, 0, 0;\n\t}" \
                 : __VA_ARGS__                                                                                   \
                 : "l"(a_desc), "l"(b_desc), "r"(accumulate));                                                   \
  }
VG_WGMMA_SS(32, VG_PH_0, 16, 17, 18, VG_D16(0))
VG_WGMMA_SS(64, VG_PH_0 VG_PH_1, 32, 33, 34, VG_D16(0), VG_D16(16))
VG_WGMMA_SS(96, VG_PH_0 VG_PH_1 VG_PH_2, 48, 49, 50, VG_D16(0), VG_D16(16), VG_D16(32))
VG_WGMMA_SS(128, VG_PH_0 VG_PH_1 VG_PH_2 VG_PH_3, 64, 65, 66, VG_D16(0), VG_D16(16), VG_D16(32), VG_D16(48))
VG_WGMMA_SS(160, VG_PH_0 VG_PH_1 VG_PH_2 VG_PH_3 VG_PH_4, 80, 81, 82, VG_D16(0), VG_D16(16), VG_D16(32), VG_D16(48),
            VG_D16(64))
VG_WGMMA_SS(192, VG_PH_0 VG_PH_1 VG_PH_2 VG_PH_3 VG_PH_4 VG_PH_5, 96, 97, 98, VG_D16(0), VG_D16(16), VG_D16(32),
            VG_D16(48), VG_D16(64), VG_D16(80))
VG_WGMMA_SS(224, VG_PH_0 VG_PH_1 VG_PH_2 VG_PH_3 VG_PH_4 VG_PH_5 VG_PH_6, 112, 113, 114, VG_D16(0), VG_D16(16),
            VG_D16(32), VG_D16(48), VG_D16(64), VG_D16(80), VG_D16(96))
VG_WGMMA_SS(256, VG_PH_0 VG_PH_1 VG_PH_2 VG_PH_3 VG_PH_4 VG_PH_5 VG_PH_6 VG_PH_7, 128, 129, 130, VG_D16(0), VG_D16(16),
            VG_D16(32), VG_D16(48), VG_D16(64), VG_D16(80), VG_D16(96), VG_D16(112))
#undef VG_WGMMA_SS

// D[64 x N, fp32 registers] (+)= A[64 x 32, smem] * B[N x 32, smem]^T, e4m3 operands, both K-major (the only operand
// layout wgmma takes for 8-bit types).  Same fragment layout as wgmma_ss; one instruction covers K = 32 (32 bytes).
template <int N>
__device__ __forceinline__ void wgmma_ss_e4m3(float (&d)[N / 2], uint64_t a_desc, uint64_t b_desc, int accumulate);
#define VG_WGMMA_SS_E4M3(N, PH, A, B, S, ...)                                                                           \
  template <>                                                                                                          \
  __device__ __forceinline__ void wgmma_ss_e4m3<N>(float (&d)[N / 2], uint64_t a_desc, uint64_t b_desc, int accumulate) { \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" #S ", 0;\n\t"                                              \
                 "wgmma.mma_async.sync.aligned.m64n" #N "k32.f32.e4m3.e4m3 {" PH "}, %" #A ", %" #B ", p, 1, 1;\n\t}"  \
                 : __VA_ARGS__                                                                                         \
                 : "l"(a_desc), "l"(b_desc), "r"(accumulate));                                                         \
  }
VG_WGMMA_SS_E4M3(64, VG_PH_0 VG_PH_1, 32, 33, 34, VG_D16(0), VG_D16(16))
VG_WGMMA_SS_E4M3(128, VG_PH_0 VG_PH_1 VG_PH_2 VG_PH_3, 64, 65, 66, VG_D16(0), VG_D16(16), VG_D16(32), VG_D16(48))
#undef VG_WGMMA_SS_E4M3

// D[64 x 64] (+)= A[64 x 16, registers] * B[16 x 64, smem, MN-major]: the P V product of the attention kernels.
// a[0..3]: the m16k16 fragment of this thread's warp -- {row g, k 2q..2q+1}, {row g+8, same k}, {row g, k 2q+8..2q+9},
// {row g+8, same k} -- which is what two adjacent 8-column groups of a wgmma accumulator hold once packed to fp16.
__device__ __forceinline__ void wgmma_rs_n64_bt(float (&d)[32], const uint32_t (&a)[4], uint64_t b_desc, int accumulate) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {" VG_PH_0 VG_PH_1 "}, {%32,%33,%34,%35}, %36, p, 1, 1, 1;\n\t}"
               : VG_D16(0), VG_D16(16)
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(accumulate));
}
#undef VG_D16

// ----------------------------------------------------------------------------- misc
__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

}  // namespace vg
