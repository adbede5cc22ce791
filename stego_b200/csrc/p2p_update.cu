// The data-parallel exchange of the training step as ONE kernel over NVLink peer memory: gradient all-reduce fused into
// the Adam update (replaces Lightning-DDP's bucketed all-reduce behind `manual_backward`, src/train_segmentation.py:227,476,
// followed by the three `optimizer.step()` calls of :228-230).
//
// Every rank owns one peer-visible block (cudaMalloc + CUDA IPC, opened by the other ranks of the node):
//     export[2][n] floats   the rank's local gradient of step e is copied into export[e & 1]
//     flags[world] uint32   flags[r] = last epoch rank r has published
// Per step and rank, on the update stream:
//   1. p2p_publish_kernel      local flat gradient -> export[e & 1]
//   2. p2p_signal_wait_kernel  one warp: store e (release, system scope) into flags[rank] of EVERY rank's block, then spin
//                              (acquire) until its own flags[*] >= e.  32 threads, no shared memory: it co-resides with the
//                              persistent GEMM / attention CTAs of the next step's backbone and holds no SM while ranks skew.
//   3. p2p_adam_kernel         g = sum over ranks (fixed order 0..world-1: every replica adds in the same order, so the
//                              replicas stay bit-identical) of export_r[e & 1][i], read straight from the peers' memory
//                              over NVLink; grad[i] = g (what an all-reduce would have left there); Adam on the local
//                              parameter / moment slices of all optimiser groups in the same launch.
// The 0.8 MB (ViT-S) / 2.8 MB (ViT-B) exchange costs world x that in NVLink reads per GPU (6.6 / 22 MB at 8 GPUs: ~10-30 us)
// and no SM-holding rendezvous.  The double buffer makes a second barrier unnecessary: a rank overwrites export[e & 1] at
// step e + 2, after it has seen every peer's flag e + 1, which a peer only publishes after its own update e (same stream)
// has read export[e & 1].
#include <cstring>

#include "common.cuh"
#include "host_util.h"

namespace stego {

constexpr int P2P_MAX_WORLD = 16;
constexpr int P2P_MAX_GROUPS = 4;

__global__ void __launch_bounds__(256) p2p_publish_kernel(const float* __restrict__ src, float* __restrict__ dst, long long n) {
  const long long i = 4 * (1ll * blockIdx.x * 256 + threadIdx.x);
  if (i + 3 < n) {
    *reinterpret_cast<float4*>(dst + i) = *reinterpret_cast<const float4*>(src + i);
  } else {
    for (long long j = i; j < n; ++j) dst[j] = src[j];
  }
}

struct P2pSignalParams {
  unsigned int* peer_flags[P2P_MAX_WORLD];  // flags array inside rank r's block
  int rank, world;
  unsigned int epoch;
  int* status;                 // set to 1 on time-out
  unsigned long long timeout_ns;
};

__global__ void __launch_bounds__(32) p2p_signal_wait_kernel(P2pSignalParams p) {
  const int t = threadIdx.x;
  if (t < p.world) {
    __threadfence_system();  // the export copy (previous kernel on this stream) is ordered before the flag
    asm volatile("st.release.sys.global.u32 [%0], %1;\n" ::"l"(p.peer_flags[t] + p.rank), "r"(p.epoch) : "memory");
    const unsigned int* mine = p.peer_flags[p.rank] + t;
    const unsigned long long t0 = globaltimer_ns();
    unsigned int v;
    for (;;) {
      asm volatile("ld.acquire.sys.global.u32 %0, [%1];\n" : "=r"(v) : "l"(mine) : "memory");
      if (static_cast<int>(v - p.epoch) >= 0) break;
      if (globaltimer_ns() - t0 > p.timeout_ns) {
        atomicExch(p.status, 1);
        break;
      }
      __nanosleep(200);
    }
  }
}

struct P2pAdamGroup {
  long long start, numel;
  AdamCoef c;
};
struct P2pAdamParams {
  const float* exports[P2P_MAX_WORLD];  // export[e & 1] of every rank
  int world, ngroups;
  P2pAdamGroup groups[P2P_MAX_GROUPS];
  float* param; float* grad; float* m; float* v;  // local flat buffers
  long long n;
  float grad_scale;
};

__global__ void __launch_bounds__(256) p2p_adam_kernel(P2pAdamParams p) {
  const long long i = 1ll * blockIdx.x * 256 + threadIdx.x;
  if (i >= p.n) return;
  float g = 0.f;
#pragma unroll 1
  for (int r = 0; r < p.world; ++r) g += __ldcv(p.exports[r] + i);  // peer memory: never from a stale cache line
  p.grad[i] = g;
#pragma unroll
  for (int k = 0; k < P2P_MAX_GROUPS; ++k) {
    if (k < p.ngroups && i >= p.groups[k].start && i < p.groups[k].start + p.groups[k].numel) {
      float pi = p.param[i], mi = p.m[i], vi = p.v[i];
      adam_elem(pi, mi, vi, __fmul_rn(g, p.grad_scale), p.groups[k].c);
      p.m[i] = mi;
      p.v[i] = vi;
      p.param[i] = pi;
    }
  }
}

}  // namespace stego

using namespace stego;

// Allocate a peer-visible, zero-filled block on the current device; handle_out receives the 64-byte CUDA IPC handle.
extern "C" int stego_p2p_alloc(long long bytes, long long* ptr_out, unsigned char* handle_out) {
  STEGO_CHECK_ARG(bytes > 0 && ptr_out && handle_out, "stego_p2p_alloc: bad args");
  void* ptr = nullptr;
  cudaError_t e = cudaMalloc(&ptr, static_cast<size_t>(bytes));
  if (e != cudaSuccess) return cuda_fail(e, "cudaMalloc(p2p block)");
  e = cudaMemset(ptr, 0, static_cast<size_t>(bytes));
  if (e != cudaSuccess) return cuda_fail(e, "cudaMemset(p2p block)");
  cudaIpcMemHandle_t h;
  e = cudaIpcGetMemHandle(&h, ptr);
  if (e != cudaSuccess) { cudaFree(ptr); return cuda_fail(e, "cudaIpcGetMemHandle"); }
  static_assert(sizeof(h) == 64, "CUDA IPC handle size");
  std::memcpy(handle_out, &h, sizeof(h));
  e = cudaDeviceSynchronize();
  if (e != cudaSuccess) return cuda_fail(e, "cudaDeviceSynchronize(p2p alloc)");
  *ptr_out = reinterpret_cast<long long>(ptr);
  return STEGO_OK;
}

// Map another rank's block (same node) into this process; peer access is enabled by the driver on first use.
extern "C" int stego_p2p_open(const unsigned char* handle, long long* ptr_out) {
  STEGO_CHECK_ARG(handle && ptr_out, "stego_p2p_open: bad args");
  cudaIpcMemHandle_t h;
  std::memcpy(&h, handle, sizeof(h));
  void* ptr = nullptr;
  cudaError_t e = cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess);
  if (e != cudaSuccess) return cuda_fail(e, "cudaIpcOpenMemHandle");
  *ptr_out = reinterpret_cast<long long>(ptr);
  return STEGO_OK;
}

extern "C" int stego_p2p_close(long long ptr) {
  cudaError_t e = cudaIpcCloseMemHandle(reinterpret_cast<void*>(ptr));
  if (e != cudaSuccess) return cuda_fail(e, "cudaIpcCloseMemHandle");
  return STEGO_OK;
}

extern "C" int stego_p2p_free(long long ptr) {
  cudaError_t e = cudaFree(reinterpret_cast<void*>(ptr));
  if (e != cudaSuccess) return cuda_fail(e, "cudaFree(p2p block)");
  return STEGO_OK;
}

// Steps 1 + 2: publish the local gradient of `epoch` and rendezvous.  export_slot = this rank's export[epoch & 1];
// peer_flags[r] = address of the flags array inside rank r's block (host array of `world` addresses);
// status: device int, set to 1 if a peer did not arrive within timeout_ms (the update then proceeds on stale data and
// the host raises at the next flush()).
extern "C" int stego_p2p_publish(const float* grad, long long n, float* export_slot, const long long* peer_flags, int rank,
                                 int world, int epoch, int* status, int timeout_ms, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(grad && export_slot && peer_flags && status && n > 0, "stego_p2p_publish: bad args");
  STEGO_CHECK_ARG(((reinterpret_cast<uintptr_t>(grad) | reinterpret_cast<uintptr_t>(export_slot)) & 15) == 0,
                  "stego_p2p_publish: 16-byte aligned buffers required");
  STEGO_CHECK_ARG(world >= 1 && world <= P2P_MAX_WORLD && rank >= 0 && rank < world && epoch > 0 && timeout_ms > 0,
                  "stego_p2p_publish: world=%d rank=%d epoch=%d", world, rank, epoch);
  const long long n4 = (n + 3) / 4;
  p2p_publish_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, stream>>>(grad, export_slot, n);
  STEGO_CHECK_LAUNCH("p2p_publish_kernel");
  P2pSignalParams p;
  for (int r = 0; r < P2P_MAX_WORLD; ++r) p.peer_flags[r] = r < world ? reinterpret_cast<unsigned int*>(peer_flags[r]) : nullptr;
  p.rank = rank; p.world = world; p.epoch = static_cast<unsigned int>(epoch); p.status = status;
  p.timeout_ns = 1000000ull * static_cast<unsigned long long>(timeout_ms);
  p2p_signal_wait_kernel<<<1, 32, 0, stream>>>(p);
  STEGO_CHECK_LAUNCH("p2p_signal_wait_kernel");
  return STEGO_OK;
}

// Step 3: all-reduce (sum, fixed rank order) fused into Adam.  peer_exports[r] = address of rank r's export[epoch & 1];
// group_desc: ngroups x 7 doubles (start, numel, lr, beta1, beta2, eps, step[1-based]); grad receives the summed gradient.
extern "C" int stego_p2p_adam(const long long* peer_exports, int world, float* param, float* grad, float* exp_avg,
                              float* exp_avg_sq, long long n, const double* group_desc, int ngroups, float grad_scale,
                              void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(peer_exports && param && grad && exp_avg && exp_avg_sq && group_desc && n > 0, "stego_p2p_adam: null pointer");
  STEGO_CHECK_ARG(world >= 1 && world <= P2P_MAX_WORLD && ngroups >= 1 && ngroups <= P2P_MAX_GROUPS,
                  "stego_p2p_adam: world=%d ngroups=%d", world, ngroups);
  P2pAdamParams p;
  for (int r = 0; r < P2P_MAX_WORLD; ++r) p.exports[r] = r < world ? reinterpret_cast<const float*>(peer_exports[r]) : nullptr;
  p.world = world; p.ngroups = ngroups;
  for (int k = 0; k < ngroups; ++k) {
    const double* d = group_desc + 7 * k;
    STEGO_CHECK_ARG(d[0] >= 0 && d[1] > 0 && d[0] + d[1] <= (double)n && d[6] >= 1, "stego_p2p_adam: bad group %d", k);
    p.groups[k].start = static_cast<long long>(d[0]);
    p.groups[k].numel = static_cast<long long>(d[1]);
    p.groups[k].c = adam_coef(d[2], d[3], d[4], d[5], d[6]);
  }
  p.param = param; p.grad = grad; p.m = exp_avg; p.v = exp_avg_sq; p.n = n; p.grad_scale = grad_scale;
  p2p_adam_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(p);
  STEGO_CHECK_LAUNCH("p2p_adam_kernel");
  return STEGO_OK;
}
