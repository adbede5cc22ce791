#include "host_util.h"

#include <atomic>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

namespace stego {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int cuda_fail(cudaError_t e, const char* what) {
  set_error("%s: %s (%s)", what, cudaGetErrorName(e), cudaGetErrorString(e));
  return STEGO_ERR_CUDA;
}

static std::atomic<long long> g_launches{0};
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }
long long launch_count() { return g_launches.load(std::memory_order_relaxed); }

int num_sms() {
  static int cached = 0;
  if (cached == 0) {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) return 132;
    cached = n;
  }
  return cached;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
    if (e != cudaSuccess || q != cudaDriverEntryPointSuccess || !p) return nullptr;
    fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

static int make_tmap(CUtensorMapDataType dtype, CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                     const uint64_t* strides_bytes, const uint32_t* box) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) {
    set_error("cuTensorMapEncodeTiled driver entry point unavailable");
    return STEGO_ERR_CUDA;
  }
  if (rank < 2 || rank > 3) {
    set_error("tensor map rank %d unsupported", rank);
    return STEGO_ERR_BAD_ARG;
  }
  if ((reinterpret_cast<uintptr_t>(base) & 15u) != 0) {
    set_error("tensor map base %p not 16-byte aligned", base);
    return STEGO_ERR_BAD_ARG;
  }
  cuuint64_t gdim[3];
  cuuint64_t gstr[2];
  cuuint32_t bdim[3];
  cuuint32_t estr[3] = {1, 1, 1};
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bdim[i] = box[i];
  }
  for (int i = 0; i < rank - 1; ++i) {
    if (strides_bytes[i] % 16 != 0) {
      set_error("tensor map stride %llu not a multiple of 16 bytes", (unsigned long long)strides_bytes[i]);
      return STEGO_ERR_BAD_ARG;
    }
    gstr[i] = strides_bytes[i];
  }
  CUresult r = fn(out, dtype, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bdim,
                  estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed with CUresult %d (rank %d dims %llu,%llu box %u,%u)", (int)r, rank,
              (unsigned long long)dims[0], (unsigned long long)dims[1], box[0], box[1]);
    return STEGO_ERR_CUDA;
  }
  return STEGO_OK;
}

int make_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                   const uint64_t* strides_bytes, const uint32_t* box) {
  return make_tmap(CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, out, base, rank, dims, strides_bytes, box);
}

}  // namespace stego

extern "C" const char* stego_last_error(void) { return stego::g_err; }
extern "C" int stego_version(void) { return 100; }
extern "C" long long stego_launch_count(void) { return stego::launch_count(); }
