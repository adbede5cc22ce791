// Dense CRF post-processing on the GPU (BASELINE.json configs[4]; SURVEY.md 8(f) rank 2).
//
// Reference: src/crf.py:22-45 hands every frame to pydensecrf on a pool of CPU processes
// (src/eval_segmentation.py:52-54,133-135):
//     d = DenseCRF2D(w, h, c); d.setUnaryEnergy(-log softmax);
//     d.addPairwiseGaussian(sxy=1, compat=3); d.addPairwiseBilateral(sxy=67, srgb=3, rgbim, compat=4); Q = d.inference(10)
// i.e. mean-field inference in a fully connected CRF (Kraehenbuehl & Koltun 2011) whose two Gaussian kernels are applied
// with the permutohedral lattice (Adams et al. 2010).  pydensecrf is third-party C++ that is not in the reference; the
// algorithm below follows its published sources (densecrf.cpp / pairwise.cpp / permutohedral.cpp) as restated by
// oracle/crf_oracle.py — parity with the reference's CRF stage is UNPINNED (DESIGN.md), the CUDA path is tested against
// that restatement.
//
// One mean-field implementation serves dense_crf / batched_crf (one probe: rows of 32 floats per pixel and lattice
// point) and the CRF-refined evaluation fused_eval_crf (two probes: rows of 64 floats, linear classes in [0, 32),
// cluster classes in [32, 64), so one splat, one blur and one slice per lattice serve both probes).  Every frame of a
// batch runs through each stage in one launch: the bilateral lattices of the frames are concatenated (point ids,
// neighbour tables and slot lists offset by the frame's base) and run as one lattice over B*N pixels; the position
// lattice depends only on the frame size, so one copy is shared by the B frames and its values are laid out per frame
// ([B][M][row]).  The splat is a gather: lattice point i sums its (pixel, vertex) slots in the order of a CSR list built
// once per lattice (slots sorted by point, ascending slot index within a point).  There are no float atomics, so results
// are bit-reproducible and a frame's outputs do not depend on the other frames of the batch.  Missing blur neighbours
// are id -1, so a lattice copy is exactly M rows and the frame copies of the position lattice tile the value buffer.
//
// Pieces (all HBM / L2-bound gather work, no tensor cores):
//   crf_lattice_kernel       per pixel: embed the feature (x/sxy, y/sxy[, c0..c2/srgb]) in the permutohedral lattice,
//                            find the enclosing simplex, its d+1 vertices as packed 64-bit keys and the barycentric
//                            weights
//   (host)                   unique keys -> lattice point ids, neighbour tables along the d+1 axes, the CSR slot list
//                            (torch.unique / searchsorted / a stable argsort: construction, once per image)
//   crf_unary_kernel         class scores -> unary energies and Q_0 (dense_crf; the evaluation's unaries come from
//                            eval_crf_unary_kernel in eval_probes.cu)
//   crf_splat_kernel<D, W>   values[c][i][col] = sum over slots s of point i: bary[s] * v(pixel(s)),
//                            v = norm * Q[col] (W = 32 or 64) or 1 (W = 1: the ones-splat of the normalisation)
//   crf_blur_kernel<W>       values'[c][i] = values[c][i] + 0.5 (values[c][n1(i)] + values[c][n2(i)])   one axis
//   crf_norm_kernel<D>       norm[pixel] = 1 / sqrt(alpha sum_r bary values[offset] + 1e-20)
//   crf_update_kernel<NP>    slice both lattices, Q <- softmax(-U + w_g n_g K_g + w_b n_b K_b) per probe, warp per
//                            pixel, lanes = classes; last iteration: argmax, marginals, confusion counts
//                            (UnsupervisedMetrics.update), each on request
#include "host_util.h"
#include "probe_common.cuh"

namespace stego {

constexpr int CRF_LD = 32;  // floats per pixel / lattice-point row: classes padded to one warp

struct LatticeParams {
  int H, W, d;              // d = 2 (position) or 5 (position + colour)
  float inv_sxy, inv_srgb;
  const unsigned char* image;  // [H][W][3] uint8 (d == 5) in the channel order the caller wants (crf.py passes BGR)
  long long* keys;          // [N][d+1]
  float* bary;              // [N][d+1]
  int bits;                 // bits per packed key coordinate
};

template <int D>
__global__ void __launch_bounds__(256)
crf_lattice_kernel(LatticeParams p) {
  const long long N = 1ll * p.H * p.W;
  const long long pix = 1ll * blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= N) return;
  const int x = static_cast<int>(pix % p.W), y = static_cast<int>(pix / p.W);
  float f[D];
  f[0] = x * p.inv_sxy;
  f[1] = y * p.inv_sxy;
  if (D == 5) {
    const unsigned char* c = p.image + pix * 3;
    f[2] = c[0] * p.inv_srgb;
    f[3] = c[1] * p.inv_srgb;
    f[4] = c[2] * p.inv_srgb;
  }
  // permutohedral.cpp Permutohedral::init, one point
  const float inv_std_dev = sqrtf(2.0f / 3.0f) * (D + 1);
  float elevated[D + 1];
  float sm = 0.f;
#pragma unroll
  for (int j = D; j > 0; --j) {
    const float cf = f[j - 1] * (1.0f / sqrtf(static_cast<float>((j + 1) * j)) * inv_std_dev);
    elevated[j] = sm - j * cf;
    sm += cf;
  }
  elevated[0] = sm;
  const float down_factor = 1.0f / (D + 1), up_factor = static_cast<float>(D + 1);
  float rem0[D + 1];
  float fsum = 0.f;
#pragma unroll
  for (int i = 0; i <= D; ++i) {
    const float v = down_factor * elevated[i];
    const float up = ceilf(v) * up_factor, down = floorf(v) * up_factor;
    rem0[i] = (up - elevated[i] < elevated[i] - down) ? up : down;
    fsum += rem0[i];
  }
  const int sum = __float2int_rn(fsum * down_factor);
  int rank[D + 1];
#pragma unroll
  for (int i = 0; i <= D; ++i) rank[i] = 0;
#pragma unroll
  for (int i = 0; i < D; ++i) {
    const float di = elevated[i] - rem0[i];
#pragma unroll
    for (int j = i + 1; j <= D; ++j) {
      if (di < elevated[j] - rem0[j]) rank[i]++;
      else rank[j]++;
    }
  }
#pragma unroll
  for (int i = 0; i <= D; ++i) {
    rank[i] += sum;
    if (rank[i] < 0) {
      rank[i] += D + 1;
      rem0[i] += D + 1;
    } else if (rank[i] > D) {
      rank[i] -= D + 1;
      rem0[i] -= D + 1;
    }
  }
  float bary[D + 2];
#pragma unroll
  for (int i = 0; i <= D + 1; ++i) bary[i] = 0.f;
#pragma unroll
  for (int i = 0; i <= D; ++i) {
    const float v = (elevated[i] - rem0[i]) * down_factor;
    // bary[D - rank[i]] += v; bary[D - rank[i] + 1] -= v   (rank is a run-time index: select instead of indexing)
#pragma unroll
    for (int k = 0; k <= D + 1; ++k) {
      if (k == D - rank[i]) bary[k] += v;
      if (k == D - rank[i] + 1) bary[k] -= v;
    }
  }
  bary[0] += 1.0f + bary[D + 1];
  const long long bias = 1ll << (p.bits - 1);
  const long long mask = (1ll << p.bits) - 1;
#pragma unroll
  for (int r = 0; r <= D; ++r) {
    long long key = 0;
#pragma unroll
    for (int i = 0; i < D; ++i) {
      // canonical[r][rank[i]] = r if rank[i] <= D - r else r - (D + 1)
      const int canon = (rank[i] <= D - r) ? r : r - (D + 1);
      const long long kc = static_cast<long long>(rem0[i]) + canon;
      key = (key << p.bits) | ((kc + bias) & mask);
    }
    p.keys[pix * (D + 1) + r] = key;
    p.bary[pix * (D + 1) + r] = bary[r];
  }
}

// unary energies and the initial Q from class scores at full resolution: probs = softmax(logits[:, pix]);
// U = -log(clip(probs, 1e-5, 1)) (pydensecrf.utils.unary_from_softmax); Q0 = softmax(-U) (densecrf.cpp inference)
__global__ void __launch_bounds__(256)
crf_unary_kernel(const float* __restrict__ logits /* [C][N] */, float* __restrict__ unary, float* __restrict__ Q, long long N, int C) {
  const int lane = threadIdx.x & 31;
  const long long pix = (1ll * blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (pix >= N) return;
  const bool on = lane < C;
  const float z = on ? logits[1ll * lane * N + pix] : -INFINITY;
  const float mx = warp_max(z);
  const float e = on ? __expf(z - mx) : 0.f;
  const float pr = e / warp_sum(e);
  const float u = -__logf(fminf(fmaxf(pr, 1e-5f), 1.0f));
  const float t = on ? -u : -INFINITY;
  const float m2 = warp_max(t);
  const float e2 = on ? __expf(t - m2) : 0.f;
  const float q = e2 / warp_sum(e2);
  unary[pix * CRF_LD + lane] = on ? u : 0.f;
  Q[pix * CRF_LD + lane] = on ? q : 0.f;
}

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

// values[c][i][col] = sum over the slots s of point i, in CSR order: bary[s] * v(pixel(s)), v = norm * Q[col] (rows of
// W floats) or 1 (W = 1: the ones-splat of the normalisation)
template <int D, int W>
__global__ void __launch_bounds__(256)
crf_splat_kernel(GatherLattice L, int copies, const float* __restrict__ Q, float* __restrict__ values) {
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
    const float v = (W == 1) ? 1.0f : L.norm[pix] * Q[(pix0 + pix) * W + col];
    s += L.bary[slot] * v;
  }
  values[e] = s;
}

// one axis of the blur: values'[c][i] = values[c][i] + 0.5 (values[c][n1(i)] + values[c][n2(i)])
template <int W>
__global__ void __launch_bounds__(256)
crf_blur_kernel(const float* __restrict__ old_v, float* __restrict__ new_v, const int* __restrict__ n1,
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

// norm[pixel] = 1 / sqrt(alpha sum_r bary values[offset] + 1e-20) from the blurred ones-splat
template <int D>
__global__ void __launch_bounds__(256)
crf_norm_kernel(const int* __restrict__ offset, const float* __restrict__ bary, const float* __restrict__ values,
                float alpha, float* __restrict__ norm_out, long long N) {
  const long long pix = 1ll * blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= N) return;
  float s = 0.f;
#pragma unroll
  for (int r = 0; r <= D; ++r) s += bary[pix * (D + 1) + r] * values[offset[pix * (D + 1) + r]] * alpha;
  norm_out[pix] = 1.0f / sqrtf(s + 1e-20f);  // pairwise.cpp NORMALIZE_SYMMETRIC
}

struct UpdateParams {
  const float* unary;  // [B*N][32 * probes]
  float* Q;            // [B*N][32 * probes], in / out
  GatherLattice g;     // position lattice: n_pix = N, copies = B
  GatherLattice b;     // concatenated bilateral lattices: n_pix = B*N, one copy
  const float* val_g;  // blurred values [B*Mg][32 * probes]
  const float* val_b;  // blurred values [Mb][32 * probes]
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

// Q <- softmax(-U + w_g n_g K_g + w_b n_b K_b) for NP probes (rows of 32 * NP floats: the linear probe, or the class
// scores of dense_crf, in [0, 32), the cluster probe in [32, 64)).  Warp per pixel, lane = class, grid-stride (so the
// last iteration flushes its per-CTA confusion counts once per CTA).
template <int NP, bool LAST>
__global__ void __launch_bounds__(256)
crf_update_kernel(UpdateParams p) {
  constexpr int LD = 32 * NP;
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
    float sg[NP], sb[NP];
#pragma unroll
    for (int k = 0; k < NP; ++k) sg[k] = sb[k] = 0.f;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const float w = p.g.bary[pix * 3 + r];
      const float* v = p.val_g + (frame * p.g.M + p.g.offset[pix * 3 + r]) * LD;
#pragma unroll
      for (int k = 0; k < NP; ++k) sg[k] += w * v[32 * k + lane];
    }
#pragma unroll
    for (int r = 0; r < 6; ++r) {
      const float w = p.b.bary[gp * 6 + r];
      const float* v = p.val_b + 1ll * p.b.offset[gp * 6 + r] * LD;
#pragma unroll
      for (int k = 0; k < NP; ++k) sb[k] += w * v[32 * k + lane];
    }
    const float ng = p.g.norm[pix], nb = p.b.norm[gp];
    const float* u = p.unary + gp * LD;
    float t[NP], q[NP];
    bool on[NP];
#pragma unroll
    for (int k = 0; k < NP; ++k)
      t[k] = -u[32 * k + lane] + p.w_g * (sg[k] * alpha_g * ng) + p.w_b * (sb[k] * alpha_b * nb);
#pragma unroll
    for (int k = 0; k < NP; ++k) {
      on[k] = lane < (k ? p.n_clu : p.n_lin);
      q[k] = warp_softmax(t[k], on[k]);
    }
    if (!LAST) {
#pragma unroll
      for (int k = 0; k < NP; ++k) p.Q[gp * LD + 32 * k + lane] = q[k];
      continue;
    }
    if (p.lin_q && on[0]) p.lin_q[(frame * p.n_lin + lane) * p.N + pix] = q[0];
    const int a0 = warp_argmax(on[0] ? q[0] : -INFINITY);
    int a1 = -1;  // one probe: no cluster prediction, nothing counted for it
    if constexpr (NP == 2) {
      if (p.clu_q && on[1]) p.clu_q[(frame * p.n_clu + lane) * p.N + pix] = q[1];
      a1 = warp_argmax(on[1] ? q[1] : -INFINITY);
    }
    if (lane == 0) {
      if (p.lin_pred) p.lin_pred[gp] = static_cast<unsigned char>(a0);
      if (NP == 2 && p.clu_pred) p.clu_pred[gp] = static_cast<unsigned char>(a1);
      if (want_conf) conf_hist_add(hist, read_label(p.label, p.label_bytes, gp), p.n_cls, a0, a1);
    }
  }
  if (want_conf) conf_hist_flush(hist, p.lin_conf, p.clu_conf, p.n_lin, p.n_clu, p.n_cls);
}

static unsigned blocks_for(long long threads) { return (unsigned)((threads + 255) / 256); }

// splat (gather) + the d+1 blur passes of one lattice (W floats per row); the blurred values end in values_tmp for
// d = 2 (three passes) and back in values for d = 5 (six passes)
template <int D, int W>
static int crf_filter(const GatherLattice& L, int copies, const float* Q, float* values, float* values_tmp,
                      cudaStream_t stream) {
  const long long n = 1ll * copies * L.M * W;
  crf_splat_kernel<D, W><<<blocks_for(n), 256, 0, stream>>>(L, copies, Q, values);
  STEGO_CHECK_LAUNCH("crf_splat_kernel");
  float* a = values;
  float* b = values_tmp;
  for (int j = 0; j <= D; ++j) {
    crf_blur_kernel<W><<<blocks_for(n), 256, 0, stream>>>(a, b, L.n1 + 1ll * j * L.M, L.n2 + 1ll * j * L.M, L.M, copies);
    STEGO_CHECK_LAUNCH("crf_blur_kernel");
    float* t = a; a = b; b = t;
  }
  return STEGO_OK;
}

// n_iter iterations of splat + blur of both lattices and the update, NP probes per row
template <int NP>
static int crf_mean_field(UpdateParams p, int n_iter, float* Q, float* val_g, float* tmp_g, float* val_b, float* tmp_b,
                          cudaStream_t stream) {
  p.val_g = tmp_g;  // three blur passes: the blurred position values end in tmp_g
  p.val_b = val_b;  // six passes: back in val_b
  const long long warps = 1ll * p.B * p.N;
  const long long cap = 8ll * num_sms();
  const long long grid = (warps + 7) / 8 < cap ? (warps + 7) / 8 : cap;
  for (int it = 0; it < n_iter; ++it) {
    int rc;
    if ((rc = crf_filter<2, 32 * NP>(p.g, p.B, Q, val_g, tmp_g, stream)) != STEGO_OK) return rc;
    if ((rc = crf_filter<5, 32 * NP>(p.b, 1, Q, val_b, tmp_b, stream)) != STEGO_OK) return rc;
    if (it + 1 < n_iter) {
      crf_update_kernel<NP, false><<<(unsigned)grid, 256, 0, stream>>>(p);
    } else {
      crf_update_kernel<NP, true><<<(unsigned)grid, 256, 0, stream>>>(p);
    }
    STEGO_CHECK_LAUNCH("crf_update_kernel");
  }
  return STEGO_OK;
}

}  // namespace stego

using namespace stego;

// Lattice embedding of every pixel.  image: [H][W][3] uint8 (only for d == 5).  keys: [N][d+1] int64, bary: [N][d+1] fp32.
extern "C" int stego_crf_lattice(int H, int W, int d, float sxy, float srgb, const unsigned char* image, long long* keys,
                                 float* bary, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(H > 0 && W > 0 && keys && bary, "stego_crf_lattice: bad args");
  STEGO_CHECK_ARG(d == 2 || (d == 5 && image), "stego_crf_lattice: d must be 2 (position) or 5 (position + colour, needs the image)");
  STEGO_CHECK_ARG(sxy > 0 && (d == 2 || srgb > 0), "stego_crf_lattice: standard deviations must be positive");
  LatticeParams p;
  p.H = H; p.W = W; p.d = d; p.inv_sxy = 1.0f / sxy; p.inv_srgb = d == 5 ? 1.0f / srgb : 0.f; p.image = image;
  p.keys = keys; p.bary = bary;
  p.bits = 60 / d;  // 30 bits per coordinate for d = 2, 12 for d = 5
  // coordinate magnitude bound: |elevated| <= (d+1) * sqrt(2/3) * sum |f| (scale factors <= (d+1) sqrt(2/3) / sqrt 2)
  const double fmax = (double)(W > H ? W : H) / sxy * 2 + (d == 5 ? 3 * 255.0 / srgb : 0.0);
  const double bound = (d + 1) * 0.8165 * fmax + 2 * (d + 1);
  STEGO_CHECK_ARG(bound < (double)(1ll << (p.bits - 1)), "stego_crf_lattice: lattice coordinates up to %.0f do not fit %d-bit keys "
                  "(image %dx%d, sxy %.2f, srgb %.2f)", bound, p.bits, H, W, sxy, srgb);
  const long long N = 1ll * H * W;
  const unsigned blocks = (unsigned)((N + 255) / 256);
  if (d == 2) crf_lattice_kernel<2><<<blocks, 256, 0, stream>>>(p);
  else crf_lattice_kernel<5><<<blocks, 256, 0, stream>>>(p);
  STEGO_CHECK_LAUNCH("crf_lattice_kernel");
  return STEGO_OK;
}

// logits [C][N] (full resolution class scores) -> unary [N][32], Q0 [N][32].
extern "C" int stego_crf_unary(const float* logits, float* unary, float* Q, long long N, int C, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(logits && unary && Q && N > 0 && C > 0 && C <= CRF_LD, "stego_crf_unary: bad args");
  crf_unary_kernel<<<(unsigned)((N * 32 + 255) / 256), 256, 0, stream>>>(logits, unary, Q, N, C);
  STEGO_CHECK_LAUNCH("crf_unary_kernel");
  return STEGO_OK;
}

static GatherLattice make_lattice(const int* offset, const float* bary, const int* rowptr, const int* slots, const int* n1,
                                  const int* n2, const float* norm, long long n_pix, int M) {
  GatherLattice L;
  L.offset = offset; L.bary = bary; L.rowptr = rowptr; L.slots = slots; L.n1 = n1; L.n2 = n2; L.norm = norm;
  L.n_pix = n_pix; L.M = M;
  return L;
}

// NORMALIZE_SYMMETRIC factor of a lattice by gathers: norm[pixel] = 1 / sqrt(K 1 + 1e-20).  values, values_tmp: [M] fp32
// scratch.  (rowptr, slots): the CSR list of the (pixel, vertex) slots of every point.
extern "C" int stego_crf_norm(int d, long long N, int M, const int* offset, const float* bary, const int* rowptr,
                              const int* slots, const int* n1, const int* n2, float* values, float* values_tmp,
                              float* norm_out, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG((d == 2 || d == 5) && N > 0 && M > 0 && offset && bary && rowptr && slots && n1 && n2 && values &&
                  values_tmp && norm_out, "stego_crf_norm: bad args");
  STEGO_CHECK_ARG(N * (d + 1) < (1ll << 31), "stego_crf_norm: %lld pixels exceed the int32 slot ids", N);
  const GatherLattice L = make_lattice(offset, bary, rowptr, slots, n1, n2, nullptr, N, M);
  int rc = d == 2 ? crf_filter<2, 1>(L, 1, nullptr, values, values_tmp, stream)
                  : crf_filter<5, 1>(L, 1, nullptr, values, values_tmp, stream);
  if (rc != STEGO_OK) return rc;
  const float* blurred = d == 2 ? values_tmp : values;
  const float alpha = 1.0f / (1.0f + exp2f(-(float)d));
  if (d == 2) crf_norm_kernel<2><<<blocks_for(N), 256, 0, stream>>>(offset, bary, blurred, alpha, norm_out, N);
  else crf_norm_kernel<5><<<blocks_for(N), 256, 0, stream>>>(offset, bary, blurred, alpha, norm_out, N);
  STEGO_CHECK_LAUNCH("crf_norm_kernel");
  return STEGO_OK;
}

// n_iter mean-field iterations of B frames of N pixels, one probe (n_clu = 0: rows of 32 floats) or two (rows of 64).
// unary, Q: [B*N][32 or 64] (stego_crf_unary / stego_eval_crf_unary; Q is overwritten).  Position lattice (*_g): one
// frame, Mg points, shared by the B frames.  Bilateral lattice (*_b): the frames' lattices concatenated, Mb points over
// B*N pixels.  Scratch: val_g, tmp_g [B*Mg][row], val_b, tmp_b [Mb][row].  Outputs of the last iteration, each optional:
// marginals lin_q [B][n_lin][N], clu_q [B][n_clu][N]; argmax maps lin_pred, clu_pred [B][N] uint8; with label [B][N]
// (label_bytes 8 / 4 / 1) the confusion counts lin_conf [n_lin][n_label_classes], clu_conf [n_clu][n_label_classes] are
// incremented at [pred][actual] for every pixel with 0 <= label < n_label_classes and pred < n_label_classes.
extern "C" int stego_crf_mean_field(int B, long long N, int n_lin, int n_clu, int n_iter, const float* unary, float* Q,
                                    const int* off_g, const float* bary_g, const int* rowptr_g, const int* slots_g,
                                    const int* n1_g, const int* n2_g, const float* norm_g, int Mg,
                                    const int* off_b, const float* bary_b, const int* rowptr_b, const int* slots_b,
                                    const int* n1_b, const int* n2_b, const float* norm_b, int Mb, float w_g,
                                    float w_b, float* val_g, float* tmp_g, float* val_b, float* tmp_b, float* lin_q,
                                    float* clu_q, unsigned char* lin_pred, unsigned char* clu_pred,
                                    const void* label, int label_bytes, int n_label_classes, long long* lin_conf,
                                    long long* clu_conf, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(B > 0 && N > 0 && n_iter > 0 && Mg > 0 && Mb > 0 && n_lin > 0 && n_lin <= 32 && n_clu >= 0 &&
                  n_clu <= 32, "stego_crf_mean_field: B=%d N=%lld n_lin=%d n_clu=%d n_iter=%d Mg=%d Mb=%d unsupported "
                  "(classes <= 32, at least one iteration)", B, N, n_lin, n_clu, n_iter, Mg, Mb);
  STEGO_CHECK_ARG(unary && Q && off_g && bary_g && rowptr_g && slots_g && n1_g && n2_g && norm_g && off_b && bary_b &&
                  rowptr_b && slots_b && n1_b && n2_b && norm_b && val_g && tmp_g && val_b && tmp_b,
                  "stego_crf_mean_field: null pointer");
  STEGO_CHECK_ARG(1ll * B * N * 6 < (1ll << 31) && 1ll * B * Mg < (1ll << 31),
                  "stego_crf_mean_field: %d x %lld pixels exceed the int32 slot ids", B, N);
  STEGO_CHECK_ARG(!label || ((label_bytes == 8 || label_bytes == 4 || label_bytes == 1) && n_label_classes > 0 &&
                             n_label_classes <= 32 && (lin_conf || clu_conf)),
                  "stego_crf_mean_field: confusion counts need label_bytes in {8,4,1}, n_label_classes <= 32 and an "
                  "output");
  UpdateParams p;
  p.unary = unary; p.Q = Q;
  p.g = make_lattice(off_g, bary_g, rowptr_g, slots_g, n1_g, n2_g, norm_g, N, Mg);
  p.b = make_lattice(off_b, bary_b, rowptr_b, slots_b, n1_b, n2_b, norm_b, 1ll * B * N, Mb);
  p.w_g = w_g; p.w_b = w_b; p.N = N; p.B = B; p.n_lin = n_lin; p.n_clu = n_clu;
  p.lin_q = lin_q; p.clu_q = clu_q; p.lin_pred = lin_pred; p.clu_pred = clu_pred;
  p.label = label; p.label_bytes = label_bytes; p.n_cls = n_label_classes;
  p.lin_conf = reinterpret_cast<unsigned long long*>(lin_conf);
  p.clu_conf = reinterpret_cast<unsigned long long*>(clu_conf);
  return n_clu == 0 ? crf_mean_field<1>(p, n_iter, Q, val_g, tmp_g, val_b, tmp_b, stream)
                    : crf_mean_field<2>(p, n_iter, Q, val_g, tmp_g, val_b, tmp_b, stream);
}

