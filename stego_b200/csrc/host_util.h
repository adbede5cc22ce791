// Host-side helpers shared by the C-ABI translation units: error reporting, TMA tensor-map
// encoding through the driver entry point (no link-time libcuda dependency), device queries.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <mutex>

namespace stego {

// status codes returned by every extern "C" entry point
enum : int {
  STEGO_OK = 0,
  STEGO_ERR_BAD_ARG = -1,      // shape / alignment / null pointer
  STEGO_ERR_UNSUPPORTED = -2,  // valid request this build has no kernel for
  STEGO_ERR_CUDA = -3,         // a CUDA runtime / driver call failed
};

void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what);  // records the message, returns STEGO_ERR_CUDA
int num_sms();
void count_launch();  // bumps the library-wide kernel launch counter (stego_launch_count)

// Encode a tiled bf16 tensor map (rank 2 or 3) with 128-byte swizzle.
//   dims[i], box[i]: element counts, innermost first; strides_bytes[i]: byte stride of dim i+1.
int make_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                   const uint64_t* strides_bytes, const uint32_t* box);
// The same for fp32 elements (GEMM output / reduce-add tiles).
int make_tmap_f32(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                  const uint64_t* strides_bytes, const uint32_t* box);

// Device ordinals whose per-device state (shared-memory opt-ins, SM counts) is cached; a process that sees more
// devices than this still works, it sets the attribute / queries the count on every call for the ordinals beyond.
constexpr int kMaxCachedDevices = 64;

// Serialises the opt-in slow path of every kernel (rare: once per kernel, device and size increase).
std::mutex& opt_in_mutex();

// Lets Kernel launch with `bytes` of dynamic shared memory on the current device: above the 48 KB default that takes
// an opt-in.  A function attribute belongs to the current device's context, so the configured size is kept per device
// ordinal and set again only when a launch on that device asks for more than before.  Safe from any host thread: the
// check is one atomic load, and the attribute is raised under a mutex so that a smaller concurrent request can never
// lower it below a size already recorded.  Returns STEGO_OK, or cuda_fail(e, what).
template <auto Kernel>
int opt_in_smem(size_t bytes, const char* what) {
  static std::atomic<size_t> configured[kMaxCachedDevices];
  if (bytes <= 48 * 1024) return STEGO_OK;
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return cuda_fail(e, what);
  const bool cached = dev >= 0 && dev < kMaxCachedDevices;
  if (cached && configured[dev].load(std::memory_order_acquire) >= bytes) return STEGO_OK;
  std::lock_guard<std::mutex> lock(opt_in_mutex());
  if (cached && configured[dev].load(std::memory_order_relaxed) >= bytes) return STEGO_OK;
  e = cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  if (e != cudaSuccess) return cuda_fail(e, what);
  if (cached) configured[dev].store(bytes, std::memory_order_release);
  return STEGO_OK;
}

#define STEGO_CHECK_ARG(cond, ...)       \
  do {                                   \
    if (!(cond)) {                       \
      ::stego::set_error(__VA_ARGS__);   \
      return ::stego::STEGO_ERR_BAD_ARG; \
    }                                    \
  } while (0)

#define STEGO_CHECK_LAUNCH(what)                                     \
  do {                                                               \
    cudaError_t _e = cudaGetLastError();                             \
    if (_e != cudaSuccess) return ::stego::cuda_fail(_e, what);      \
    ::stego::count_launch();                                         \
  } while (0)

}  // namespace stego
