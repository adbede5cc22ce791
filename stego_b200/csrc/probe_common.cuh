// Device (and one host) helpers shared by the training probes (probes.cu) and the fused evaluation probes
// (eval_probes.cu): bilinear source indices and the low-res box a tile of output pixels reads, label reads,
// centroid normalisation, the warp-per-pixel channel broadcast, the K-tiled dots of wide codes and the per-CTA
// confusion histogram.
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

// ---- wide codes: the backbone's 384 / 768 channels (projection_type None, the DINO baseline) --------------------------
// A pixel's channels no longer fit the registers of the warp-per-pixel kernels; the dot products run as 32-channel K
// tiles through shared memory instead, PW_ROWS pixels per CTA of 256 threads.
constexpr int PW_ROWS = 64, PW_KC = 32, PW_SX = PW_KC + 4;  // sX row stride: 16-byte rows, offset banks

// acc[i] += sum_c xat(r0 + 16 rg + i, c) * table(c, o) for the thread's output column o = tid & 63 and pixel group
// rg = tid >> 6, sequential fp32 FMAs in channel order; with kSumSq, ss (threads < 64) += sum_c xat(r0 + tid, c)^2.  xat(r, c): channel
// c of pixel r < rows; table(c, o): the probe table's column o.  C % 32 == 0; sX [PW_ROWS][PW_SX] (16-byte aligned) and
// sT [PW_KC][64] are the caller's shared memory.
// sinv[k] = 1 / max(|c_k|, 1e-12) for the centroids clusters [n][C], as normalize_centroids computes the norms (a warp
// per centroid, 8 warps); the caller synchronises
__device__ __forceinline__ void centroid_inv_norms(const float* clusters, int n, int C, float* sinv) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int k = warp; k < n; k += 8) {
    float ss = 0.f;
    for (int c = lane; c < C; c += 32) { const float v = clusters[1ll * k * C + c]; ss += v * v; }
    ss = warp_sum(ss);
    if (lane == 0) sinv[k] = 1.0f / fmaxf(sqrtf(ss), 1e-12f);
  }
}

template <bool kSumSq, typename XFn, typename TableFn>
__device__ __forceinline__ void wide_tile_dots(XFn xat, long long rows, long long r0, int C, TableFn table, float* sX,
                                               float* sT, float (&acc)[16], float& ss) {
  const int o = threadIdx.x & 63, rg = threadIdx.x >> 6;
  for (int c0 = 0; c0 < C; c0 += PW_KC) {
    __syncthreads();  // the previous K tile has been read
    for (int i = threadIdx.x; i < PW_ROWS * PW_KC; i += blockDim.x) {
      const int rr = i / PW_KC, c = i % PW_KC;
      const long long r = r0 + rr;
      sX[rr * PW_SX + c] = (r < rows) ? xat(r, c0 + c) : 0.f;
    }
    for (int i = threadIdx.x; i < PW_KC * 64; i += blockDim.x) sT[i] = table(c0 + (i >> 6), i & 63);
    __syncthreads();
    if (kSumSq && threadIdx.x < PW_ROWS)
      for (int c = 0; c < PW_KC; ++c) ss = fmaf(sX[threadIdx.x * PW_SX + c], sX[threadIdx.x * PW_SX + c], ss);
#pragma unroll
    for (int c = 0; c < PW_KC; c += 4) {
      const float w0 = sT[c * 64 + o], w1 = sT[(c + 1) * 64 + o], w2 = sT[(c + 2) * 64 + o], w3 = sT[(c + 3) * 64 + o];
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const float4 v = *reinterpret_cast<const float4*>(&sX[(rg * 16 + i) * PW_SX + c]);
        acc[i] = fmaf(v.w, w3, fmaf(v.z, w2, fmaf(v.y, w1, fmaf(v.x, w0, acc[i]))));
      }
    }
  }
}

}  // namespace stego
