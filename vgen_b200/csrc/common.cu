// Library-wide host state: last error, launch counter, device properties, tensor-map encoding.
#include "common.h"

#include <stdlib.h>

#include <atomic>
#include <mutex>

namespace vg {

static thread_local std::string g_last_error;
std::atomic<long long> g_launches{0};

void set_error(const std::string& msg) { g_last_error = msg; }
int fail(const std::string& msg) {
  g_last_error = msg;
  return 1;
}
int check_cuda(cudaError_t e, const char* what) {
  if (e == cudaSuccess) {
    return 0;
  }
  g_last_error = std::string(what) + ": " + cudaGetErrorName(e) + " (" + cudaGetErrorString(e) + ")";
  return 2;
}
const std::string& last_error() { return g_last_error; }

int current_device() {
  int dev = 0;
  cudaGetDevice(&dev);
  return dev;
}

int sm_count() {
  static std::atomic<int> cache[64];
  const int dev = current_device() & 63;
  int n = cache[dev].load(std::memory_order_relaxed);
  if (n == 0) {
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    cache[dev].store(n, std::memory_order_relaxed);
  }
  return n;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    // the driver entry point is resolved at run time, so the library links against cudart only
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess) {
      fn = reinterpret_cast<EncodeTiledFn>(p);
    }
  });
  return fn;
}

static int make_tmap(CUtensorMapDataType dtype, CUtensorMap* map, const void* base, int rank, const uint64_t* dims,
                     const uint64_t* strides_bytes, const uint32_t* box, int swizzle_bytes);

int make_tmap_f16(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                  const uint32_t* box, int swizzle_bytes) {
  return make_tmap(CU_TENSOR_MAP_DATA_TYPE_FLOAT16, map, base, rank, dims, strides_bytes, box, swizzle_bytes);
}

int make_tmap_u8(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                 const uint32_t* box, int swizzle_bytes) {
  return make_tmap(CU_TENSOR_MAP_DATA_TYPE_UINT8, map, base, rank, dims, strides_bytes, box, swizzle_bytes);
}

static int make_tmap(CUtensorMapDataType dtype, CUtensorMap* map, const void* base, int rank, const uint64_t* dims,
                     const uint64_t* strides_bytes, const uint32_t* box, int swizzle_bytes) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return fail("cuTensorMapEncodeTiled entry point not available (no CUDA driver?)");
  cuuint64_t gdim[5];
  cuuint64_t gstr[4];
  cuuint32_t bdim[5];
  cuuint32_t estr[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bdim[i] = box[i];
    estr[i] = 1;
  }
  for (int i = 0; i + 1 < rank; ++i) {
    gstr[i] = strides_bytes[i];
    if (gstr[i] % 16 != 0) return fail("tensor map: strides must be multiples of 16 bytes");
  }
  CUresult r = enc(map, dtype, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bdim,
                   estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char buf[256];
    snprintf(buf, sizeof buf,
             "cuTensorMapEncodeTiled failed (%d): rank %d dims [%llu %llu %llu %llu] box [%u %u %u %u] stride0 %llu",
             (int)r, rank, (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0),
             (unsigned long long)(rank > 2 ? dims[2] : 0), (unsigned long long)(rank > 3 ? dims[3] : 0), box[0],
             rank > 1 ? box[1] : 0, rank > 2 ? box[2] : 0, rank > 3 ? box[3] : 0,
             (unsigned long long)(rank > 1 ? strides_bytes[0] : 0));
    return fail(buf);
  }
  return 0;
}

}  // namespace vg

extern "C" {
int vgen_abi_version(void) { return VGEN_B200_ABI_VERSION; }
const char* vgen_last_error(void) { return vg::g_last_error.c_str(); }
int64_t vgen_launch_count(void) { return (int64_t)vg::g_launches.load(); }
}
