// Host-side helpers shared by the C-ABI translation units: error reporting, TMA tensor-map
// encoding through the driver entry point (no link-time libcuda dependency), device queries.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

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
