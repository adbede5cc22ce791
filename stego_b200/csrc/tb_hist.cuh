// TensorBoard's default histogram buckets (SummaryWriter.add_histogram(tag, values), bins="tensorflow") on the GPU.
//
// The edges are torch/utils/tensorboard/writer.py's `default_bins`: v = 1e-12, v *= 1.1 while v < 1e20 (774 values),
// mirrored negative, 0 in the middle: TB_EDGES = 1549 float64 edges, TB_BINS = 1548 buckets.  The counts are those of
// np.histogram(values.astype(float64), default_bins): bucket k is [e_k, e_k+1), the last one [e_1547, e_1548]; values
// outside [e_0, e_1548] (and NaN) are not counted.
//
// Exact decisions on fp32 values: for an fp32 x and a float64 edge e, x >= e holds exactly when x >= RU(e), RU(e) the
// smallest float >= e (no float lies in [e, RU(e)) other than RU(e) itself, and x < e implies x <= RD(e) < RU(e) when e
// is not a float).  The table holds t_k = RU(e_k) for the 1549 edges, then t_1549 = RD(e_1548) for the closed upper
// end.  -0.0 >= t_774 = +0.0, so -0.0 falls in [0, 1e-12), as it does in numpy.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace stego {

constexpr int TB_POS = 774;               // positive edges 1e-12 * 1.1^j (as the writer's loop accumulates them)
constexpr int TB_EDGES = 2 * TB_POS + 1;  // 1549
constexpr int TB_BINS = TB_EDGES - 1;     // 1548
constexpr int TB_THR = TB_EDGES + 1;      // thresholds: RU of each edge, then RD of the last edge
constexpr int TB_GROUPS_MAX = 3;          // histograms one correlation launch fills (intra, inter, negatives)

// Host: the float64 edges (may be null) and the fp32 threshold table described above (may be null).
void tb_tables(double* edges, float* thresholds);

// Bucket of x (0 .. TB_BINS - 1), or -1 when np.histogram does not count it.  `t` is the threshold table (any memory
// space).  A logarithmic first guess, then a fix-up against the table that makes the answer exact whatever the guess.
__device__ __forceinline__ int tb_bucket(float x, const float* t) {
  if (!(x >= t[0] && x <= t[TB_EDGES])) return -1;
  const float ax = fabsf(x);
  int k;
  if (ax < 1e-12f) {
    k = x >= 0.f ? TB_POS : TB_POS - 1;
  } else {
    // j with 1e-12 * 1.1^j <= |x| < 1e-12 * 1.1^(j+1), up to rounding; 1 / log2(1.1) = 7.272540897
    const int j = min(static_cast<int>(__log2f(ax * 1e12f) * 7.272540897f), TB_POS - 1);
    k = x > 0.f ? TB_POS + 1 + j : TB_POS - 2 - j;
  }
  k = max(0, min(k, TB_BINS - 1));
  while (k < TB_BINS - 1 && x >= t[k + 1]) ++k;
  while (k > 0 && x < t[k]) --k;
  return k;
}

// Running min / max / sum / sum of squares of the values one thread has seen; sums in fp64 (x * x is exact in fp64).
struct TbStats {
  float mn, mx;
  double s, s2;
  __device__ __forceinline__ void init() { mn = INFINITY; mx = -INFINITY; s = 0.0; s2 = 0.0; }
  __device__ __forceinline__ void add(float x) {
    mn = fminf(mn, x);
    mx = fmaxf(mx, x);
    const double d = x;
    s += d;
    s2 += d * d;
  }
  // butterfly over the warp: a fixed pattern, so every lane ends with the same, reproducible totals
  __device__ __forceinline__ void warp_reduce() {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      s += __shfl_xor_sync(0xffffffffu, s, o);
      s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    }
  }
};

// Host: per histogram group g, reduce the per-CTA partials part[first_g .. first_g+1)[4] (min, max, sum, sum of
// squares) in a fixed order into stats[g][4].  first has ngroups + 1 entries.
int tb_launch_finish(const double* part, const int* first, int ngroups, double* stats, cudaStream_t stream);

}  // namespace stego
