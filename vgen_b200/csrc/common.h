// Host-side helpers shared by every translation unit of libvgen_b200.so.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <string>

#include "../../include/vgen_b200.h"

namespace vg {

// Error plumbing: every C-ABI entry returns 0 on success, non-zero on failure, and the message is
// kept per host thread for vgen_last_error().
void set_error(const std::string& msg);
int fail(const std::string& msg);
int check_cuda(cudaError_t e, const char* what);

#define VG_CUDA(expr)                                   \
  do {                                                  \
    int _rc = ::vg::check_cuda((expr), #expr);          \
    if (_rc) return _rc;                                \
  } while (0)
#define VG_LAUNCH_CHECK(name)                                   \
  do {                                                          \
    ::vg::g_launches.fetch_add(1, std::memory_order_relaxed);   \
    int _rc = ::vg::check_cuda(cudaGetLastError(), name);       \
    if (_rc) return _rc;                                        \
  } while (0)
#define VG_REQUIRE(cond, msg)                                          \
  do {                                                                 \
    if (!(cond)) return ::vg::fail(std::string(msg) + " [" #cond "]"); \
  } while (0)

// Encode a tiled, swizzled (128B default, or 64B) fp16 tensor map (rank <= 4). dims/box are innermost-first;
// strides_bytes has rank-1 entries (dims 1..rank-1). Out-of-bounds elements read as zero / are not written.
int make_tmap_f16(CUtensorMap* map, const void* base, int rank, const uint64_t* dims,
                  const uint64_t* strides_bytes, const uint32_t* box, int swizzle_bytes = 128);
// Same for a tensor of bytes (e4m3 codes): dims / box in elements = bytes.
int make_tmap_u8(CUtensorMap* map, const void* base, int rank, const uint64_t* dims,
                 const uint64_t* strides_bytes, const uint32_t* box, int swizzle_bytes = 128);

int sm_count();            // of the CURRENT device (cached per device)
int current_device();

// "do this once per device" guard for per-device function attributes (cudaFuncSetAttribute is per device: a process that
// drives a second GPU must set the > 48 KB dynamic shared memory opt-in there too).
struct PerDeviceOnce {
  std::atomic<unsigned long long> done{0};
  bool need() const { return ((done.load(std::memory_order_acquire) >> (current_device() & 63)) & 1ull) == 0; }
  void mark() { done.fetch_or(1ull << (current_device() & 63), std::memory_order_release); }
};
extern std::atomic<long long> g_launches;  // kernels launched by this library (vgen_launch_count)

static inline int cdiv(long a, long b) { return (int)((a + b - 1) / b); }

// Every kernel of the library is launched through this (cudaLaunchKernelEx; one place to add launch attributes).
// Programmatic dependent launch is deliberately not set here: no kernel of the library calls griddepcontrol.wait, so a
// kernel started early could read its predecessor's output before it is written.
#ifdef __CUDACC__
template <typename... KArgs, typename... Args>
static inline cudaError_t launch_kernel(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                                        Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cfg.attrs = nullptr;
  cfg.numAttrs = 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}
#endif

}  // namespace vg
