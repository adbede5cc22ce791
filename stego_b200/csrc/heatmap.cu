// Dense correspondence heatmaps (sm_90a): the diagnostic of the reference's src/plot_dino_correspondence.py,
// get_heatmaps (:39-58), for a batch of images and P query points per image.
//
//   q   = F.normalize(sample(feats, query_points))                     :43, :45 (eps 1e-12)
//   c   = einsum("nchw,ncij->nhwij", q, F.normalize(target))           :45 / :49
//   c   = clamp(c - c.mean([3, 4]), 0)                                 :46-47 / :50-51
//   out = F.interpolate(c, (H, W), mode="bilinear", align_corners=True)  :53-56
//
// Pipeline (stego_b200/correspondence.py: correspondence_heatmaps):
//   1. heatmap_target_kernel : one pass over the target map (any strides, fp32 or bf16) -> the K-major bf16 GEMM operand
//                              [B][h w][K] and the fp32 inverse norm of every position.  bf16 targets are exact in one
//                              plane, written twice ([t | t]); fp32 targets are split t = hi + lo ([hi | hi | lo]).
//   2. heatmap_query_kernel  : bilinear sample of P listed points per image (taps.cuh), L2 normalise in fp32, split
//                              q = hi + lo: [hi | lo] against a bf16 target, [hi | lo | hi] against an fp32 one.
//   3. stego_gemm_bf16_batched: raw[b] = q_ops[b] . t_ops[b]^T, fp32 [B][P][h w] — with the hi/lo planes folded along K
//                              this is q.t to ~2^-16 relative (the lo.lo term is dropped).
//   4. heatmap_finish_kernel : per (b, p) row: c = raw * inv_norm, fixed-order row mean, clamp(c - mean, 0), in place.
//   5. heatmap_upsample_kernel: [B P][h][w] -> [B P][H][W] fp32, bilinear align_corners=True with ATen's CUDA arithmetic
//                              (upsample_bilinear2d_out_frame), 16-byte streaming stores, 8 rows per thread: the HBM-write-bound step.
#include "common.cuh"
#include "host_util.h"
#include "taps.cuh"

namespace stego {

constexpr int HM_MAX_E = 768;              // channels per lane <= 24 in the query sampler
constexpr int HM_NV = HM_MAX_E / 32;
constexpr float HM_EPS = 1e-12f;           // F.normalize's default eps

__device__ __forceinline__ float load_elem(const void* src, int is_bf16, long long off) {
  return is_bf16 ? __bfloat162float(reinterpret_cast<const bf16*>(src)[off]) : reinterpret_cast<const float*>(src)[off];
}

// One warp per target position (b, j = y w + x): ops[b][j] = [t | t] (bf16 source) or [hi | hi | lo] (fp32 source),
// each segment Epad wide with zeros past E; inv_norm[b][j] = 1 / max(||t||, 1e-12) from the fp32 sum of squares.
__global__ void __launch_bounds__(256)
heatmap_target_kernel(const void* src, int is_bf16, long long sb, long long sc, long long sy, long long sx, int B, int E,
                      int h, int w, int Epad, bf16* ops, float* inv_norm) {
  const long long pos = static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const long long hw = static_cast<long long>(h) * w;
  if (pos >= B * hw) return;
  const int b = static_cast<int>(pos / hw);
  const int j = static_cast<int>(pos - b * hw);
  const long long base = b * sb + static_cast<long long>(j / w) * sy + static_cast<long long>(j % w) * sx;
  const int K = (is_bf16 ? 2 : 3) * Epad;
  bf16* row = ops + pos * K;
  float ss = 0.f;
  for (int c = lane; c < Epad; c += 32) {
    const float v = c < E ? load_elem(src, is_bf16, base + c * sc) : 0.f;
    ss += v * v;
    const bf16 hi = __float2bfloat16_rn(v);
    row[c] = hi;
    row[Epad + c] = hi;
    if (!is_bf16) row[2 * Epad + c] = __float2bfloat16_rn(v - __bfloat162float(hi));
  }
  ss = warp_sum(ss);
  if (lane == 0) inv_norm[pos] = 1.0f / fmaxf(sqrtf(ss), HM_EPS);
}

// One warp per query (b, p): grid_sample(feats, query_points.permute(0, 2, 1, 3), border, align_corners=True) at
// points[b][p] = (x, y), summed nw, ne, sw, se as ATen's grid_sampler_2d, normalised in fp32 (eps 1e-12) and split
// n = hi + lo: ops[b][p] = [hi | lo] (nseg 2) or [hi | lo | hi] (nseg 3), each segment Epad wide, zeros past E.
__global__ void __launch_bounds__(256)
heatmap_query_kernel(const void* src, int is_bf16, long long sb, long long sc, long long sy, long long sx,
                     const float* points, int B, int P, int E, int h, int w, int Epad, int nseg, bf16* ops) {
  const long long q = static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (q >= static_cast<long long>(B) * P) return;
  const int b = static_cast<int>(q / P);
  const Taps t = grid_taps(points[2 * q], points[2 * q + 1], h, w);
  auto off = [&](int pix) { return static_cast<long long>(pix / w) * sy + static_cast<long long>(pix % w) * sx; };
  const long long base = b * sb;
  const long long o00 = base + off(t.i00), o01 = base + off(t.i01), o10 = base + off(t.i10), o11 = base + off(t.i11);
  float v[HM_NV];
  float ss = 0.f;
#pragma unroll
  for (int k = 0; k < HM_NV; ++k) {
    const int c = lane + 32 * k;
    float val = 0.f;
    if (c < E) {
      const long long cc = static_cast<long long>(c) * sc;
      val = load_elem(src, is_bf16, o00 + cc) * t.w00;
      val += load_elem(src, is_bf16, o01 + cc) * t.w01;
      val += load_elem(src, is_bf16, o10 + cc) * t.w10;
      val += load_elem(src, is_bf16, o11 + cc) * t.w11;
    }
    v[k] = val;
    ss += val * val;
  }
  ss = warp_sum(ss);
  const float inv = 1.0f / fmaxf(sqrtf(ss), HM_EPS);
  bf16* row = ops + q * nseg * Epad;
#pragma unroll
  for (int k = 0; k < HM_NV; ++k) {
    const int c = lane + 32 * k;
    if (c < Epad) {
      const float n = v[k] * inv;
      const bf16 hi = __float2bfloat16_rn(n);
      const bf16 lo = __float2bfloat16_rn(n - __bfloat162float(hi));
      row[c] = hi;
      row[Epad + c] = lo;
      if (nseg == 3) row[2 * Epad + c] = hi;
    }
  }
}

// One CTA per (b, p) row of the raw correlations [B P][hw]: c = raw * inv_norm[b], mean over the row, raw <- max(c -
// mean, 0).  The mean is c_0 + mean_j (c_j - c_0), summed per thread over a fixed stride, then a warp tree and the 8
// warp totals in order (the same order every run); shifted by c_0, a constant row has mean c_0 exactly and maps to 0.
__global__ void __launch_bounds__(256)
heatmap_finish_kernel(float* corr, const float* inv_norm, int P, int hw) {
  __shared__ float warp_tot[8];
  const long long r = blockIdx.x;
  float* row = corr + r * hw;
  const float* inv = inv_norm + (r / P) * hw;
  const float c0 = __fmul_rn(row[0], inv[0]);  // __fmul_rn: no fma contraction, c_j is the same rounding everywhere
  float s = 0.f;
  for (int j = threadIdx.x; j < hw; j += 256) s += __fmul_rn(row[j], inv[j]) - c0;
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) warp_tot[threadIdx.x >> 5] = s;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) tot += warp_tot[i];
  const float mean = c0 + tot / static_cast<float>(hw);
  for (int j = threadIdx.x; j < hw; j += 256) row[j] = fmaxf(__fmul_rn(row[j], inv[j]) - mean, 0.f);
}

// F.interpolate(x, (H, W), mode="bilinear", align_corners=True) of rows [n][h][w] -> [n][H][W], fp32, with the
// arithmetic of ATen's CUDA upsample_bilinear2d_out_frame: src = scale * dst (scale = (in - 1) / (out - 1), 0 for
// out = 1), lambda1 = src - floor, lambda0 = 1 - lambda1, the two rows interpolated along w first.  A thread (x index
// over [n][W / V], blockIdx.y = a band of HM_UP_ROWS output rows) forms the taps of its V consecutive columns once and
// writes them on each row of the band with one streaming store (V = 4: 16 bytes); the inputs come from L1 / L2.
constexpr int HM_UP_ROWS = 8;

template <int V>
__global__ void __launch_bounds__(256)
heatmap_upsample_kernel(const float* __restrict__ in, float* __restrict__ out, long long n, int h, int w, int H, int W,
                        float rh, float rw) {
  const int WV = W / V;
  const long long xi = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (xi >= n * WV) return;
  const long long r = xi / WV;
  const int x0 = static_cast<int>(xi - r * WV) * V;
  int c0[V], c1[V];
  float l0[V], l1[V];
#pragma unroll
  for (int v = 0; v < V; ++v) {
    const float w1r = rw * (x0 + v);
    const int w1 = static_cast<int>(w1r);
    c0[v] = w1;
    c1[v] = w1 + ((w1 < w - 1) ? 1 : 0);
    l1[v] = w1r - w1;
    l0[v] = 1.f - l1[v];
  }
  const float* img = in + r * h * w;
  float* dst = out + r * H * W + x0;
#pragma unroll
  for (int k = 0; k < HM_UP_ROWS; ++k) {
    const int y = blockIdx.y * HM_UP_ROWS + k;
    if (y >= H) break;
    const float h1r = rh * y;
    const int h1 = static_cast<int>(h1r);
    const int h1p = (h1 < h - 1) ? 1 : 0;
    const float h1l = h1r - h1;
    const float h0l = 1.f - h1l;
    const float* r0 = img + h1 * w;
    const float* r1 = r0 + h1p * w;
    float o[V];
#pragma unroll
    for (int v = 0; v < V; ++v)
      o[v] = h0l * (l0[v] * __ldg(r0 + c0[v]) + l1[v] * __ldg(r0 + c1[v])) +
             h1l * (l0[v] * __ldg(r1 + c0[v]) + l1[v] * __ldg(r1 + c1[v]));
    float* d = dst + static_cast<long long>(y) * W;
    if constexpr (V == 4) __stcs(reinterpret_cast<float4*>(d), make_float4(o[0], o[1], o[2], o[3]));
    else __stcs(d, o[0]);
  }
}

}  // namespace stego

using namespace stego;

// C-ABI: see include/stego_b200.h for the contracts.
extern "C" int stego_heatmap_prep_target(const void* target, int target_is_bf16, long long stride_b, long long stride_c,
                                         long long stride_y, long long stride_x, int B, int E, int h, int w, int Epad,
                                         void* ops, float* inv_norm, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(target && ops && inv_norm, "stego_heatmap_prep_target: null pointer");
  STEGO_CHECK_ARG(B > 0 && h > 0 && w > 0, "stego_heatmap_prep_target: B=%d h=%d w=%d", B, h, w);
  STEGO_CHECK_ARG(E >= 1 && E <= HM_MAX_E, "stego_heatmap_prep_target: E=%d outside 1..%d", E, HM_MAX_E);
  STEGO_CHECK_ARG(Epad >= E && Epad % 8 == 0, "stego_heatmap_prep_target: Epad=%d (a multiple of 8, >= E=%d)", Epad, E);
  const long long warps = static_cast<long long>(B) * h * w;
  const long long blocks = (warps + 7) / 8;
  STEGO_CHECK_ARG(blocks <= 0x7fffffffll, "stego_heatmap_prep_target: %lld positions", warps);
  heatmap_target_kernel<<<static_cast<unsigned>(blocks), 256, 0, stream>>>(
      target, target_is_bf16 ? 1 : 0, stride_b, stride_c, stride_y, stride_x, B, E, h, w, Epad,
      reinterpret_cast<bf16*>(ops), inv_norm);
  STEGO_CHECK_LAUNCH("heatmap_target_kernel");
  return STEGO_OK;
}

extern "C" int stego_heatmap_sample_queries(const void* feats, int feats_is_bf16, long long stride_b, long long stride_c,
                                            long long stride_y, long long stride_x, const float* points, int B, int P,
                                            int E, int h, int w, int Epad, int nseg, void* ops, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(feats && points && ops, "stego_heatmap_sample_queries: null pointer");
  STEGO_CHECK_ARG(B > 0 && P > 0 && h > 0 && w > 0, "stego_heatmap_sample_queries: B=%d P=%d h=%d w=%d", B, P, h, w);
  STEGO_CHECK_ARG(E >= 1 && E <= HM_MAX_E, "stego_heatmap_sample_queries: E=%d outside 1..%d", E, HM_MAX_E);
  STEGO_CHECK_ARG(Epad >= E && Epad % 8 == 0 && Epad <= HM_MAX_E,
                  "stego_heatmap_sample_queries: Epad=%d (a multiple of 8, E=%d..%d)", Epad, E, HM_MAX_E);
  STEGO_CHECK_ARG(nseg == 2 || nseg == 3, "stego_heatmap_sample_queries: nseg=%d (2 or 3)", nseg);
  const long long blocks = (static_cast<long long>(B) * P + 7) / 8;
  heatmap_query_kernel<<<static_cast<unsigned>(blocks), 256, 0, stream>>>(
      feats, feats_is_bf16 ? 1 : 0, stride_b, stride_c, stride_y, stride_x, points, B, P, E, h, w, Epad, nseg,
      reinterpret_cast<bf16*>(ops));
  STEGO_CHECK_LAUNCH("heatmap_query_kernel");
  return STEGO_OK;
}

extern "C" int stego_heatmap_finish(float* corr, const float* inv_norm, int B, int P, int hw, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(corr && inv_norm, "stego_heatmap_finish: null pointer");
  STEGO_CHECK_ARG(B > 0 && P > 0 && hw > 0, "stego_heatmap_finish: B=%d P=%d hw=%d", B, P, hw);
  const long long rows = static_cast<long long>(B) * P;
  STEGO_CHECK_ARG(rows <= 0x7fffffffll, "stego_heatmap_finish: B * P = %lld rows", rows);
  heatmap_finish_kernel<<<static_cast<unsigned>(rows), 256, 0, stream>>>(corr, inv_norm, P, hw);
  STEGO_CHECK_LAUNCH("heatmap_finish_kernel");
  return STEGO_OK;
}

extern "C" int stego_heatmap_upsample(const float* in, float* out, long long n, int h, int w, int H, int W,
                                      void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(in && out, "stego_heatmap_upsample: null pointer");
  STEGO_CHECK_ARG(n > 0 && h > 0 && w > 0 && H > 0 && W > 0, "stego_heatmap_upsample: n=%lld h=%d w=%d H=%d W=%d", n, h,
                  w, H, W);
  STEGO_CHECK_ARG(H <= 65535, "stego_heatmap_upsample: H=%d exceeds 65535", H);
  const bool vec = W % 4 == 0 && (reinterpret_cast<uintptr_t>(out) & 15u) == 0;
  const int V = vec ? 4 : 1;
  const long long threads = n * (W / V);
  const long long blocks = (threads + 255) / 256;
  STEGO_CHECK_ARG(blocks <= 0x7fffffffll, "stego_heatmap_upsample: %lld x %d outputs per row", n, W);
  // area_pixel_compute_scale (align_corners=True), in fp32 as ATen forms it on the host
  const float rh = H > 1 ? static_cast<float>(h - 1) / static_cast<float>(H - 1) : 0.f;
  const float rw = W > 1 ? static_cast<float>(w - 1) / static_cast<float>(W - 1) : 0.f;
  const dim3 grid(static_cast<unsigned>(blocks), static_cast<unsigned>((H + HM_UP_ROWS - 1) / HM_UP_ROWS));
  if (vec) heatmap_upsample_kernel<4><<<grid, 256, 0, stream>>>(in, out, n, h, w, H, W, rh, rw);
  else heatmap_upsample_kernel<1><<<grid, 256, 0, stream>>>(in, out, n, h, w, H, W, rh, rw);
  STEGO_CHECK_LAUNCH("heatmap_upsample_kernel");
  return STEGO_OK;
}
