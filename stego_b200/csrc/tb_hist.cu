// TensorBoard histograms of fp32 device tensors (SummaryWriter.add_histogram's default buckets, see tb_hist.cuh):
// the bucket table, a generic histogram kernel and the fixed-order finish of the min / max / sum / sum-of-squares
// partials that the correlation-loss histogram variants (corr_loss.cu) share.
#include <math.h>

#include "host_util.h"
#include "tb_hist.cuh"

namespace stego {

void tb_tables(double* edges, float* thresholds) {
  double e[TB_EDGES];
  double v = 1e-12;  // writer.py: buckets / neg_buckets, then neg_buckets[::-1] + [0] + buckets
  for (int j = 0; j < TB_POS; ++j) {
    e[TB_POS + 1 + j] = v;
    e[TB_POS - 1 - j] = -v;
    v *= 1.1;
  }
  e[TB_POS] = 0.0;
  for (int k = 0; k < TB_EDGES; ++k) {
    if (edges) edges[k] = e[k];
    if (thresholds) {
      float f = static_cast<float>(e[k]);
      if (static_cast<double>(f) < e[k]) f = nextafterf(f, INFINITY);
      thresholds[k] = f;
    }
  }
  if (thresholds) {
    float f = static_cast<float>(e[TB_EDGES - 1]);
    if (static_cast<double>(f) > e[TB_EDGES - 1]) f = nextafterf(f, -INFINITY);
    thresholds[TB_EDGES] = f;
  }
}

constexpr int TB_THREADS = 512;
constexpr int TB_CTAS = 264;  // fixed, so that the partial sums (and the result) do not depend on the device

// One CTA: bins in shared memory, then one global atomic per non-empty bin; per-CTA stats partials.
__global__ void __launch_bounds__(TB_THREADS)
tb_histogram_kernel(const float* __restrict__ x, long long n, const float* __restrict__ thr,
                    unsigned long long* __restrict__ counts, double* __restrict__ part) {
  __shared__ float t[TB_THR];
  __shared__ uint32_t bins[TB_BINS];
  __shared__ TbStats wred[TB_THREADS / 32];
  for (int k = threadIdx.x; k < TB_THR; k += TB_THREADS) t[k] = thr[k];
  for (int k = threadIdx.x; k < TB_BINS; k += TB_THREADS) bins[k] = 0;
  __syncthreads();
  TbStats st;
  st.init();
  for (long long i = static_cast<long long>(blockIdx.x) * TB_THREADS + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * TB_THREADS) {
    const float v = x[i];
    const int k = tb_bucket(v, t);
    if (k >= 0) atomicAdd(&bins[k], 1u);
    st.add(v);
  }
  st.warp_reduce();
  if ((threadIdx.x & 31) == 0) wred[threadIdx.x >> 5] = st;
  __syncthreads();
  for (int k = threadIdx.x; k < TB_BINS; k += TB_THREADS)
    if (bins[k]) atomicAdd(&counts[k], static_cast<unsigned long long>(bins[k]));
  if (threadIdx.x == 0) {
    TbStats c = wred[0];
    for (int w = 1; w < TB_THREADS / 32; ++w) {
      c.mn = fminf(c.mn, wred[w].mn);
      c.mx = fmaxf(c.mx, wred[w].mx);
      c.s += wred[w].s;
      c.s2 += wred[w].s2;
    }
    double* o = part + static_cast<size_t>(blockIdx.x) * 4;
    o[0] = c.mn; o[1] = c.mx; o[2] = c.s; o[3] = c.s2;
  }
}

struct TbFinishArgs {
  int first[TB_GROUPS_MAX + 1];
};

// one CTA per group: strided per-thread sums, then a fixed tree
constexpr int TB_FINISH_THREADS = 256;
__global__ void __launch_bounds__(TB_FINISH_THREADS)
tb_finish_kernel(const double* __restrict__ part, TbFinishArgs a, double* __restrict__ stats) {
  const int g = blockIdx.x;
  __shared__ double red[4][TB_FINISH_THREADS];
  double mn = INFINITY, mx = -INFINITY, s = 0.0, s2 = 0.0;
  for (int c = a.first[g] + threadIdx.x; c < a.first[g + 1]; c += TB_FINISH_THREADS) {
    const double* q = part + static_cast<size_t>(c) * 4;
    mn = fmin(mn, q[0]); mx = fmax(mx, q[1]); s += q[2]; s2 += q[3];
  }
  red[0][threadIdx.x] = mn; red[1][threadIdx.x] = mx; red[2][threadIdx.x] = s; red[3][threadIdx.x] = s2;
  __syncthreads();
  for (int w = TB_FINISH_THREADS / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) {
      red[0][threadIdx.x] = fmin(red[0][threadIdx.x], red[0][threadIdx.x + w]);
      red[1][threadIdx.x] = fmax(red[1][threadIdx.x], red[1][threadIdx.x + w]);
      red[2][threadIdx.x] += red[2][threadIdx.x + w];
      red[3][threadIdx.x] += red[3][threadIdx.x + w];
    }
    __syncthreads();
  }
  if (threadIdx.x < 4) stats[g * 4 + threadIdx.x] = red[threadIdx.x][0];
}

int tb_launch_finish(const double* part, const int* first, int ngroups, double* stats, cudaStream_t stream) {
  TbFinishArgs a;
  for (int g = 0; g <= ngroups; ++g) a.first[g] = first[g];
  tb_finish_kernel<<<ngroups, TB_FINISH_THREADS, 0, stream>>>(part, a, stats);
  STEGO_CHECK_LAUNCH("tb_finish_kernel");
  return STEGO_OK;
}

}  // namespace stego

using namespace stego;

extern "C" int stego_tb_tables(double* edges, float* thresholds) {
  tb_tables(edges, thresholds);
  return STEGO_OK;
}

extern "C" int stego_tb_histogram(const float* values, long long n, const float* thresholds, long long* counts,
                                  double* cta_partials, double* stats, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(values && thresholds && counts && cta_partials && stats, "stego_tb_histogram: null pointer");
  STEGO_CHECK_ARG(n > 0, "stego_tb_histogram: n=%lld (needs at least one value)", n);
  cudaError_t e = cudaMemsetAsync(counts, 0, sizeof(long long) * TB_BINS, stream);
  if (e != cudaSuccess) return cuda_fail(e, "stego_tb_histogram: memset");
  const long long blocks = (n + TB_THREADS - 1) / TB_THREADS;
  const int grid = static_cast<int>(blocks < TB_CTAS ? blocks : TB_CTAS);
  tb_histogram_kernel<<<grid, TB_THREADS, 0, stream>>>(values, n, thresholds,
                                                       reinterpret_cast<unsigned long long*>(counts), cta_partials);
  STEGO_CHECK_LAUNCH("tb_histogram_kernel");
  const int first[2] = {0, grid};
  return tb_launch_finish(cta_partials, first, 1, stats, stream);
}
