// Device (and one host) helpers shared by the training probes (probes.cu) and the fused evaluation probes
// (eval_probes.cu): bilinear source indices and the low-res box a tile of output pixels reads, label reads,
// centroid normalisation, the warp-per-pixel channel broadcast and the per-CTA confusion histogram.
#pragma once
#include "common.cuh"

namespace stego {

// ATen area_pixel_compute_source_index (align_corners=False, non-cubic): clamp negative to 0
__device__ __forceinline__ void src_index(int dst, float scale, int in_size, int& i0, int& i1, float& l1) {
  float s = scale * (dst + 0.5f) - 0.5f;
  if (s < 0.f) s = 0.f;
  i0 = static_cast<int>(s);
  if (i0 > in_size - 1) i0 = in_size - 1;
  i1 = i0 + ((i0 < in_size - 1) ? 1 : 0);
  l1 = s - i0;
}

// The low-res cells [lo, lo + cells) that output pixels first..last (one tile side) interpolate from
__device__ __forceinline__ void src_span(int first, int last, float scale, int in_size, int& lo, int& cells) {
  int hi, tmp;
  float ftmp;
  src_index(first, scale, in_size, lo, tmp, ftmp);
  src_index(last, scale, in_size, tmp, hi, ftmp);
  cells = hi - lo + 1;
}

// Host bound on src_span's cells for a tile side of `tile` output pixels, upsampling in_size -> out_size
inline int src_span_max(int tile, int in_size, int out_size) {
  const int cells = (int)((double)tile * in_size / out_size) + 3;
  return cells < in_size ? cells : in_size;
}

// label [B][H][W] element i: int64 / int32 / uint8 by label_bytes = 8 / 4 / 1 (uint8 255 is out of range: ignored)
__device__ __forceinline__ long long read_label(const void* label, int label_bytes, long long i) {
  if (label_bytes == 8) return reinterpret_cast<const long long*>(label)[i];
  if (label_bytes == 4) return reinterpret_cast<const int*>(label)[i];
  return reinterpret_cast<const unsigned char*>(label)[i];
}

// F.normalize (eps 1e-12) of the centroids clusters [n][C] into dst[k * sk + c * sc] (sk, sc = C, 1: [n][C];
// 1, 32: the transposed [C][32] table of the warp-per-pixel kernels).  One warp per centroid, round-robin over
// nwarps warps; the caller synchronises.
__device__ __forceinline__ void normalize_centroids(const float* clusters, int n, int C, int nwarps, float* dst,
                                                    int sk, int sc) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int k = warp; k < n; k += nwarps) {
    float ss = 0.f;
    for (int c = lane; c < C; c += 32) { const float v = clusters[k * C + c]; ss += v * v; }
    ss = warp_sum(ss);
    const float inv = 1.0f / fmaxf(sqrtf(ss), 1e-12f);
    for (int c = lane; c < C; c += 32) dst[k * sk + c * sc] = clusters[k * C + c] * inv;
  }
}

// Warp per pixel (C <= 96): channel c of the pixel at xp goes to lane c % 32 of xr[c / 32] (0 beyond C)
__device__ __forceinline__ void load_channels(const float* xp, int C, int lane, float (&xr)[3]) {
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int c = lane + 32 * k;
    xr[k] = (c < C) ? xp[c] : 0.f;
  }
}

// Broadcasts the pixel's channels to the whole warp in ascending order: f(c, x_c) for c = 0 .. C-1.  Dot products
// with a [C][32] table (lane = class) are f = [&](int c, float x) { d = fmaf(x, table[c * 32 + lane], d); }, one FMA
// chain per accumulator in channel order.
template <class F>
__device__ __forceinline__ void for_each_channel(const float (&xr)[3], int C, F&& f) {
#pragma unroll
  for (int k = 0; k < 3; ++k) {
#pragma unroll 8
    for (int j = 0; j < 32; ++j) {
      const int c = 32 * k + j;
      if (c < C) f(c, __shfl_sync(0xffffffffu, xr[k], j));  // warp-uniform
    }
  }
}

// Per-CTA confusion counts of the two eval probes: hist[probe][pred * 32 + actual], probe 0 linear, 1 cluster.
// (Zeroed by a plain loop in each kernel: moving that loop into a helper costs eval_probe_vec4_kernel 40 B of spills.)
typedef unsigned int ConfHist[2][32 * 32];

// UnsupervisedMetrics.update (src/utils.py:219-229): a pixel counts when 0 <= label < n_cls and pred < n_cls
__device__ __forceinline__ void conf_hist_add(ConfHist& hist, long long lab, int n_cls, int lin_pred, int clu_pred) {
  if (lab >= 0 && lab < n_cls) {
    if (lin_pred >= 0 && lin_pred < n_cls) atomicAdd(&hist[0][lin_pred * 32 + static_cast<int>(lab)], 1u);
    if (clu_pred >= 0 && clu_pred < n_cls) atomicAdd(&hist[1][clu_pred * 32 + static_cast<int>(lab)], 1u);
  }
}

// After the CTA's last conf_hist_add: one 64-bit atomic per non-zero cell into lin_conf [n_lin][n_cls] and
// clu_conf [n_clu][n_cls] (either may be null)
__device__ __forceinline__ void conf_hist_flush(const ConfHist& hist, unsigned long long* lin_conf,
                                                unsigned long long* clu_conf, int n_lin, int n_clu, int n_cls) {
  __syncthreads();
  for (int i = threadIdx.x; i < 2 * 32 * 32; i += blockDim.x) {
    const unsigned int cnt = (&hist[0][0])[i];
    if (cnt == 0u) continue;
    const int probe = i >> 10, pred = (i >> 5) & 31, act = i & 31;
    unsigned long long* dst = probe ? clu_conf : lin_conf;
    if (dst && act < n_cls && pred < (probe ? n_clu : n_lin)) atomicAdd(dst + pred * n_cls + act, (unsigned long long)cnt);
  }
}

}  // namespace stego
