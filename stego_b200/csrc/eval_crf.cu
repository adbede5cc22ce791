// Batched, deterministic dense-CRF mean field of the CRF-refined evaluation (stego_b200.eval.fused_eval_crf;
// src/eval_segmentation.py:133-141 with run_crf=True -> src/crf.py:22-45 once per probe and frame).
//
// The same inference as crf.cu (Potts mean field, Gaussian kernel sxy 1 / w 3 and bilateral kernel sxy 67, srgb 3 / w 4,
// NORMALIZE_SYMMETRIC, ten iterations, densecrf's blur stencil and slice scale), organised differently:
//   * both probes ride in one 64-float row per pixel and per lattice point (linear classes in [0, 32), cluster classes
//     in [32, 64)): one splat, one blur and one slice per lattice serve both probes;
//   * every frame of the batch in one launch per stage.  The bilateral lattices of the frames are concatenated (point
//     ids, neighbour tables and slot lists offset by the frame's base) and run as one lattice over B*N pixels.  The
//     position lattice depends only on the frame size: one copy is shared by the B frames, and its values are laid out
//     per frame ([B][M][64]);
//   * the splat is a gather: lattice point i sums its (pixel, vertex) slots in the order of a CSR list built once per
//     lattice (slots sorted by point, ascending slot index within a point).  There are no float atomics, so results
//     are bit-reproducible and a frame's outputs do not depend on the other frames of the batch;
//   * the last update takes both argmaxes, writes the label maps and accumulates the confusion counts
//     (UnsupervisedMetrics.update); the [n][H][W] marginals are written only on request.
// Missing blur neighbours are id -1 (tested in the blur) instead of crf.cu's zero row 0, so that a lattice copy is
// exactly M rows and the frame copies of the position lattice tile the value buffer without gaps.
//
//   ecrf_splat_kernel<D, W>   values[c][i][col] = sum over slots s of point i: bary[s] * v(pixel(s)),
//                             v = norm * Q[col] (W = 64) or 1 (W = 1: the ones-splat of the normalisation)
//   ecrf_blur_kernel<W>       values'[c][i] = values[c][i] + 0.5 (values[c][n1(i)] + values[c][n2(i)])   one axis
//   ecrf_norm_kernel<D>       norm[pixel] = 1 / sqrt(alpha sum_r bary values[offset] + 1e-20)
//   ecrf_update_kernel        slice both lattices, Q <- softmax(-U + w_g n_g K_g + w_b n_b K_b) per probe; last
//                             iteration: argmax, marginals, confusion counts
#include "host_util.h"
#include "probe_common.cuh"

namespace stego {

constexpr int ECRF_LD = 64;  // floats per pixel / lattice-point row: both probes, 32 classes each

// A permutohedral lattice over n_pix pixels with M points, replicated over `copies` consecutive blocks of n_pix pixels
// (pixel gp belongs to copy gp / n_pix; its point i is row (gp / n_pix) * M + i of the value buffer)
struct GatherLattice {
  const int* offset;  // [n_pix][D+1] point of (pixel, vertex)
  const float* bary;  // [n_pix][D+1] barycentric weights
  const int* rowptr;  // [M+1] CSR row pointers into slots
  const int* slots;   // [n_pix*(D+1)] slot = pixel * (D+1) + vertex, sorted by point
  const int* n1;      // [D+1][M] blur neighbours (-1: missing)
  const int* n2;
  const float* norm;  // [n_pix] NORMALIZE_SYMMETRIC factor (null while it is being computed)
  long long n_pix;
  int M;
};

template <int D, int W>
__global__ void __launch_bounds__(256)
ecrf_splat_kernel(GatherLattice L, int copies, const float* __restrict__ Q, float* __restrict__ values) {
  const long long e = 1ll * blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= 1ll * copies * L.M * W) return;
  const int col = static_cast<int>(e % W);
  const long long P = e / W;
  const long long c = P / L.M;
  const int i = static_cast<int>(P % L.M);
  const long long pix0 = c * L.n_pix;
  float s = 0.f;
  const int end = L.rowptr[i + 1];
  for (int k = L.rowptr[i]; k < end; ++k) {
    const int slot = L.slots[k];
    const int pix = slot / (D + 1);
    const float v = (W == 1) ? 1.0f : L.norm[pix] * Q[(pix0 + pix) * ECRF_LD + col];
    s += L.bary[slot] * v;
  }
  values[e] = s;
}

template <int W>
__global__ void __launch_bounds__(256)
ecrf_blur_kernel(const float* __restrict__ old_v, float* __restrict__ new_v, const int* __restrict__ n1,
                 const int* __restrict__ n2, int M, int copies) {
  const long long e = 1ll * blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= 1ll * copies * M * W) return;
  const int col = static_cast<int>(e % W);
  const long long P = e / W;
  const long long base = (P / M) * M;
  const int i = static_cast<int>(P % M);
  const int a = n1[i], b = n2[i];
  const float va = a >= 0 ? old_v[(base + a) * W + col] : 0.f;
  const float vb = b >= 0 ? old_v[(base + b) * W + col] : 0.f;
  new_v[e] = old_v[e] + 0.5f * (va + vb);
}

template <int D>
__global__ void __launch_bounds__(256)
ecrf_norm_kernel(const int* __restrict__ offset, const float* __restrict__ bary, const float* __restrict__ values,
                 float alpha, float* __restrict__ norm_out, long long N) {
  const long long pix = 1ll * blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= N) return;
  float s = 0.f;
#pragma unroll
  for (int r = 0; r <= D; ++r) s += bary[pix * (D + 1) + r] * values[offset[pix * (D + 1) + r]] * alpha;
  norm_out[pix] = 1.0f / sqrtf(s + 1e-20f);  // pairwise.cpp NORMALIZE_SYMMETRIC
}

struct EcrfUpdateParams {
  const float* unary;  // [B*N][64]
  float* Q;            // [B*N][64], in / out
  GatherLattice g;     // position lattice: n_pix = N, copies = B
  GatherLattice b;     // concatenated bilateral lattices: n_pix = B*N, one copy
  const float* val_g;  // blurred values [B*Mg][64]
  const float* val_b;  // blurred values [Mb][64]
  float w_g, w_b;
  long long N;         // pixels per frame
  int B, n_lin, n_clu;
  // last iteration only (each may be null)
  float* lin_q;        // [B][n_lin][N]
  float* clu_q;        // [B][n_clu][N]
  unsigned char* lin_pred;  // [B][N]
  unsigned char* clu_pred;
  const void* label;   // [B][N] int64 / int32 / uint8 by label_bytes
  int label_bytes, n_cls;
  unsigned long long* lin_conf;  // [n_lin][n_cls] +=
  unsigned long long* clu_conf;  // [n_clu][n_cls] +=
};

// argmax over the lanes of a warp (v = -inf on unused lanes), lowest index on ties (torch.argmax / np.argmax)
__device__ __forceinline__ int warp_argmax(float v) {
  int idx = threadIdx.x & 31;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
    if (ov > v || (ov == v && oi < idx)) { v = ov; idx = oi; }
  }
  return idx;
}

// softmax over the lanes < n (0 on the others)
__device__ __forceinline__ float warp_softmax(float t, bool on) {
  const float mx = warp_max(on ? t : -INFINITY);
  const float e = on ? __expf(t - mx) : 0.f;
  return e / warp_sum(e);
}

// warp per pixel, grid-stride (so the last iteration flushes its per-CTA confusion counts once per CTA);
// lane = class of both probes
template <bool LAST>
__global__ void __launch_bounds__(256)
ecrf_update_kernel(EcrfUpdateParams p) {
  __shared__ ConfHist hist;
  const bool want_conf = LAST && p.label != nullptr;
  if (want_conf)
    for (int i = threadIdx.x; i < 2 * 32 * 32; i += blockDim.x) (&hist[0][0])[i] = 0u;
  if (want_conf) __syncthreads();
  const int lane = threadIdx.x & 31;
  const long long total = p.N * p.B;
  const long long warps = 1ll * gridDim.x * (blockDim.x >> 5);
  const float alpha_g = 1.0f / (1.0f + 0.25f), alpha_b = 1.0f / (1.0f + 0.03125f);  // 1 / (1 + 2^-d), d = 2, 5
  for (long long gp = 1ll * blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); gp < total; gp += warps) {
    const long long frame = gp / p.N, pix = gp - frame * p.N;
    float sg0 = 0.f, sg1 = 0.f, sb0 = 0.f, sb1 = 0.f;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const float w = p.g.bary[pix * 3 + r];
      const float* v = p.val_g + (frame * p.g.M + p.g.offset[pix * 3 + r]) * ECRF_LD;
      sg0 += w * v[lane];
      sg1 += w * v[32 + lane];
    }
#pragma unroll
    for (int r = 0; r < 6; ++r) {
      const float w = p.b.bary[gp * 6 + r];
      const float* v = p.val_b + 1ll * p.b.offset[gp * 6 + r] * ECRF_LD;
      sb0 += w * v[lane];
      sb1 += w * v[32 + lane];
    }
    const float ng = p.g.norm[pix], nb = p.b.norm[gp];
    const float* u = p.unary + gp * ECRF_LD;
    const float t0 = -u[lane] + p.w_g * (sg0 * alpha_g * ng) + p.w_b * (sb0 * alpha_b * nb);
    const float t1 = -u[32 + lane] + p.w_g * (sg1 * alpha_g * ng) + p.w_b * (sb1 * alpha_b * nb);
    const bool on0 = lane < p.n_lin, on1 = lane < p.n_clu;
    const float q0 = warp_softmax(t0, on0), q1 = warp_softmax(t1, on1);
    if (!LAST) {
      p.Q[gp * ECRF_LD + lane] = q0;
      p.Q[gp * ECRF_LD + 32 + lane] = q1;
      continue;
    }
    if (p.lin_q && on0) p.lin_q[(frame * p.n_lin + lane) * p.N + pix] = q0;
    if (p.clu_q && on1) p.clu_q[(frame * p.n_clu + lane) * p.N + pix] = q1;
    const int a0 = warp_argmax(on0 ? q0 : -INFINITY), a1 = warp_argmax(on1 ? q1 : -INFINITY);
    if (lane == 0) {
      if (p.lin_pred) p.lin_pred[gp] = static_cast<unsigned char>(a0);
      if (p.clu_pred) p.clu_pred[gp] = static_cast<unsigned char>(a1);
      if (want_conf) conf_hist_add(hist, read_label(p.label, p.label_bytes, gp), p.n_cls, a0, a1);
    }
  }
  if (want_conf) conf_hist_flush(hist, p.lin_conf, p.clu_conf, p.n_lin, p.n_clu, p.n_cls);
}

static unsigned blocks_for(long long threads) { return (unsigned)((threads + 255) / 256); }

// splat (gather) + the d+1 blur passes of one lattice (W floats per row); the blurred values end in values_tmp for
// d = 2 (three passes) and back in values for d = 5 (six passes), as in crf.cu
template <int D, int W>
static int ecrf_filter(const GatherLattice& L, int copies, const float* Q, float* values, float* values_tmp,
                       cudaStream_t stream) {
  const long long n = 1ll * copies * L.M * W;
  ecrf_splat_kernel<D, W><<<blocks_for(n), 256, 0, stream>>>(L, copies, Q, values);
  STEGO_CHECK_LAUNCH("ecrf_splat_kernel");
  float* a = values;
  float* b = values_tmp;
  for (int j = 0; j <= D; ++j) {
    ecrf_blur_kernel<W><<<blocks_for(n), 256, 0, stream>>>(a, b, L.n1 + 1ll * j * L.M, L.n2 + 1ll * j * L.M, L.M, copies);
    STEGO_CHECK_LAUNCH("ecrf_blur_kernel");
    float* t = a; a = b; b = t;
  }
  return STEGO_OK;
}

}  // namespace stego

using namespace stego;

static GatherLattice make_lattice(const int* offset, const float* bary, const int* rowptr, const int* slots, const int* n1,
                                  const int* n2, const float* norm, long long n_pix, int M) {
  GatherLattice L;
  L.offset = offset; L.bary = bary; L.rowptr = rowptr; L.slots = slots; L.n1 = n1; L.n2 = n2; L.norm = norm;
  L.n_pix = n_pix; L.M = M;
  return L;
}

// NORMALIZE_SYMMETRIC factor of a lattice by gathers: norm[pixel] = 1 / sqrt(K 1 + 1e-20).  values, values_tmp: [M] fp32
// scratch.  (rowptr, slots): the CSR list of the (pixel, vertex) slots of every point.
extern "C" int stego_eval_crf_norm(int d, long long N, int M, const int* offset, const float* bary, const int* rowptr,
                                   const int* slots, const int* n1, const int* n2, float* values, float* values_tmp,
                                   float* norm_out, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG((d == 2 || d == 5) && N > 0 && M > 0 && offset && bary && rowptr && slots && n1 && n2 && values &&
                  values_tmp && norm_out, "stego_eval_crf_norm: bad args");
  STEGO_CHECK_ARG(N * (d + 1) < (1ll << 31), "stego_eval_crf_norm: %lld pixels exceed the int32 slot ids", N);
  const GatherLattice L = make_lattice(offset, bary, rowptr, slots, n1, n2, nullptr, N, M);
  int rc = d == 2 ? ecrf_filter<2, 1>(L, 1, nullptr, values, values_tmp, stream)
                  : ecrf_filter<5, 1>(L, 1, nullptr, values, values_tmp, stream);
  if (rc != STEGO_OK) return rc;
  const float* blurred = d == 2 ? values_tmp : values;
  const float alpha = 1.0f / (1.0f + exp2f(-(float)d));
  if (d == 2) ecrf_norm_kernel<2><<<blocks_for(N), 256, 0, stream>>>(offset, bary, blurred, alpha, norm_out, N);
  else ecrf_norm_kernel<5><<<blocks_for(N), 256, 0, stream>>>(offset, bary, blurred, alpha, norm_out, N);
  STEGO_CHECK_LAUNCH("ecrf_norm_kernel");
  return STEGO_OK;
}

// n_iter mean-field iterations of B frames of N pixels, both probes at once (see the top of this file).  unary, Q:
// [B*N][64] (stego_eval_crf_unary; Q is overwritten).  Position lattice (*_g): one frame, Mg points, shared by the B
// frames.  Bilateral lattice (*_b): the frames' lattices concatenated, Mb points over B*N pixels.  Scratch: val_g,
// tmp_g [B*Mg][64], val_b, tmp_b [Mb][64].  Outputs of the last iteration, each optional: marginals lin_q [B][n_lin][N],
// clu_q [B][n_clu][N]; argmax maps lin_pred, clu_pred [B][N] uint8; with label [B][N] (label_bytes 8 / 4 / 1) the
// confusion counts lin_conf [n_lin][n_label_classes], clu_conf [n_clu][n_label_classes] are incremented at
// [pred][actual] for every pixel with 0 <= label < n_label_classes and pred < n_label_classes.
extern "C" int stego_eval_crf_mean_field(int B, long long N, int n_lin, int n_clu, int n_iter, const float* unary, float* Q,
                                         const int* off_g, const float* bary_g, const int* rowptr_g, const int* slots_g,
                                         const int* n1_g, const int* n2_g, const float* norm_g, int Mg,
                                         const int* off_b, const float* bary_b, const int* rowptr_b, const int* slots_b,
                                         const int* n1_b, const int* n2_b, const float* norm_b, int Mb, float w_g,
                                         float w_b, float* val_g, float* tmp_g, float* val_b, float* tmp_b, float* lin_q,
                                         float* clu_q, unsigned char* lin_pred, unsigned char* clu_pred,
                                         const void* label, int label_bytes, int n_label_classes, long long* lin_conf,
                                         long long* clu_conf, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(B > 0 && N > 0 && n_iter > 0 && Mg > 0 && Mb > 0 && n_lin > 0 && n_lin <= 32 && n_clu > 0 &&
                  n_clu <= 32, "stego_eval_crf_mean_field: B=%d N=%lld n_lin=%d n_clu=%d n_iter=%d Mg=%d Mb=%d unsupported "
                  "(classes <= 32, at least one iteration)", B, N, n_lin, n_clu, n_iter, Mg, Mb);
  STEGO_CHECK_ARG(unary && Q && off_g && bary_g && rowptr_g && slots_g && n1_g && n2_g && norm_g && off_b && bary_b &&
                  rowptr_b && slots_b && n1_b && n2_b && norm_b && val_g && tmp_g && val_b && tmp_b,
                  "stego_eval_crf_mean_field: null pointer");
  STEGO_CHECK_ARG(1ll * B * N * 6 < (1ll << 31) && 1ll * B * Mg < (1ll << 31),
                  "stego_eval_crf_mean_field: %d x %lld pixels exceed the int32 slot ids", B, N);
  STEGO_CHECK_ARG(!label || ((label_bytes == 8 || label_bytes == 4 || label_bytes == 1) && n_label_classes > 0 &&
                             n_label_classes <= 32 && (lin_conf || clu_conf)),
                  "stego_eval_crf_mean_field: confusion counts need label_bytes in {8,4,1}, n_label_classes <= 32 and an "
                  "output");
  EcrfUpdateParams p;
  p.unary = unary; p.Q = Q;
  p.g = make_lattice(off_g, bary_g, rowptr_g, slots_g, n1_g, n2_g, norm_g, N, Mg);
  p.b = make_lattice(off_b, bary_b, rowptr_b, slots_b, n1_b, n2_b, norm_b, 1ll * B * N, Mb);
  p.w_g = w_g; p.w_b = w_b; p.N = N; p.B = B; p.n_lin = n_lin; p.n_clu = n_clu;
  p.lin_q = lin_q; p.clu_q = clu_q; p.lin_pred = lin_pred; p.clu_pred = clu_pred;
  p.label = label; p.label_bytes = label_bytes; p.n_cls = n_label_classes;
  p.lin_conf = reinterpret_cast<unsigned long long*>(lin_conf);
  p.clu_conf = reinterpret_cast<unsigned long long*>(clu_conf);
  p.val_g = tmp_g;  // three blur passes: the blurred position values end in tmp_g
  p.val_b = val_b;  // six passes: back in val_b
  const long long warps = 1ll * B * N;
  const long long cap = 8ll * num_sms();
  const long long grid = (warps + 7) / 8 < cap ? (warps + 7) / 8 : cap;
  for (int it = 0; it < n_iter; ++it) {
    int rc;
    if ((rc = ecrf_filter<2, ECRF_LD>(p.g, B, Q, val_g, tmp_g, stream)) != STEGO_OK) return rc;
    if ((rc = ecrf_filter<5, ECRF_LD>(p.b, 1, Q, val_b, tmp_b, stream)) != STEGO_OK) return rc;
    if (it + 1 < n_iter) {
      ecrf_update_kernel<false><<<(unsigned)grid, 256, 0, stream>>>(p);
    } else {
      ecrf_update_kernel<true><<<(unsigned)grid, 256, 0, stream>>>(p);
    }
    STEGO_CHECK_LAUNCH("ecrf_update_kernel");
  }
  return STEGO_OK;
}
