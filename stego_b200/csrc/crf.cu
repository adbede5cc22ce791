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
// Pieces (all HBM / L2-bound gather-scatter work, no tensor cores — lanes = classes, one warp per pixel or lattice point):
//   crf_lattice_kernel   per pixel: embed the feature (x/sxy, y/sxy[, c0..c2/srgb]) in the permutohedral lattice, find
//                        the enclosing simplex, its d+1 vertices as packed 64-bit keys and the barycentric weights
//   (host)               unique keys -> lattice point ids, neighbour tables along the d+1 axes (torch.unique / searchsorted:
//                        construction, once per image)
//   crf_splat_kernel     values[point] += bary * norm[pixel] * Q[pixel]        (vector reductions, 128 B per warp)
//   crf_blur_kernel      values'[p] = values[p] + 0.5 (values[n1(p)] + values[n2(p)])   along one axis
//   crf_update_kernel    slice both kernels, tmp = -U + w_g K_g(Q) + w_b K_b(Q), Q <- softmax(tmp); last iteration also
//                        writes Q as [C][H][W] and the argmax map
#include "common.cuh"
#include "host_util.h"

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

// values[(offset+1)][c] += bary * scale[pixel] * in[pixel][c]; warp per pixel, lanes = classes
template <int D>
__global__ void __launch_bounds__(256)
crf_splat_kernel(const int* __restrict__ offset, const float* __restrict__ bary, const float* __restrict__ scale,
                 const float* __restrict__ in, int in_is_one, float* __restrict__ values, long long N, int C) {
  const int lane = threadIdx.x & 31;
  const long long pix = (1ll * blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (pix >= N || lane >= C) return;
  const float v = (in_is_one ? 1.0f : in[pix * CRF_LD + lane]) * (scale ? scale[pix] : 1.0f);
#pragma unroll
  for (int r = 0; r <= D; ++r) {
    const int o = offset[pix * (D + 1) + r] + 1;
    atomicAdd(values + 1ll * o * CRF_LD + lane, bary[pix * (D + 1) + r] * v);
  }
}

// one axis of the blur; row 0 is the "missing neighbour" row (zeros); warp per lattice point
__global__ void __launch_bounds__(256)
crf_blur_kernel(const float* __restrict__ old_v, float* __restrict__ new_v, const int* __restrict__ n1, const int* __restrict__ n2,
                int M, int C) {
  const int lane = threadIdx.x & 31;
  const long long i = (1ll * blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (i >= M || lane >= C) return;
  const long long a = n1[i] + 1, b = n2[i] + 1;
  new_v[(i + 1) * CRF_LD + lane] = old_v[(i + 1) * CRF_LD + lane] + 0.5f * (old_v[a * CRF_LD + lane] + old_v[b * CRF_LD + lane]);
}

// slice of a value_size-1 filter: out[pixel] = alpha * sum_r bary * values[offset+1][0]; thread per pixel
template <int D>
__global__ void __launch_bounds__(256)
crf_slice1_kernel(const int* __restrict__ offset, const float* __restrict__ bary, const float* __restrict__ values, float alpha,
                  float* __restrict__ norm_out, long long N) {
  const long long pix = 1ll * blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= N) return;
  float s = 0.f;
#pragma unroll
  for (int r = 0; r <= D; ++r) s += bary[pix * (D + 1) + r] * values[1ll * (offset[pix * (D + 1) + r] + 1) * CRF_LD] * alpha;
  norm_out[pix] = 1.0f / sqrtf(s + 1e-20f);  // pairwise.cpp NORMALIZE_SYMMETRIC
}

struct UpdateParams {
  const float* unary;  // [N][CRF_LD] energies (-log p)
  const int* off_g;    // Gaussian kernel: [N][3]
  const float* bary_g;
  const float* val_g;  // blurred lattice values [(Mg+1)][CRF_LD]
  const float* norm_g;
  const int* off_b;    // bilateral kernel: [N][6]
  const float* bary_b;
  const float* val_b;
  const float* norm_b;
  float w_g, w_b;      // Potts weights (compat)
  float* Q;            // [N][CRF_LD], in/out
  float* q_out;        // [C][N] or null (last iteration)
  unsigned char* arg_out;  // [N] or null
  long long N;
  int C;
};

// Q <- softmax(-U + w_g n_g K_g(n_g Q) + w_b n_b K_b(n_b Q)): slice both lattices, warp per pixel, lanes = classes
__global__ void __launch_bounds__(256)
crf_update_kernel(UpdateParams p) {
  const int lane = threadIdx.x & 31;
  const long long pix = (1ll * blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (pix >= p.N) return;
  const bool on = lane < p.C;
  float t = -INFINITY;
  if (on) {
    float sg = 0.f, sb = 0.f;
#pragma unroll
    for (int r = 0; r < 3; ++r)
      sg += p.bary_g[pix * 3 + r] * p.val_g[1ll * (p.off_g[pix * 3 + r] + 1) * CRF_LD + lane];
#pragma unroll
    for (int r = 0; r < 6; ++r)
      sb += p.bary_b[pix * 6 + r] * p.val_b[1ll * (p.off_b[pix * 6 + r] + 1) * CRF_LD + lane];
    const float alpha_g = 1.0f / (1.0f + 0.25f), alpha_b = 1.0f / (1.0f + 0.03125f);  // 1 / (1 + 2^-d), d = 2, 5
    t = -p.unary[pix * CRF_LD + lane] + p.w_g * (sg * alpha_g * p.norm_g[pix]) + p.w_b * (sb * alpha_b * p.norm_b[pix]);
  }
  const float mx = warp_max(t);
  const float e = on ? __expf(t - mx) : 0.f;
  const float q = e / warp_sum(e);
  if (on) {
    p.Q[pix * CRF_LD + lane] = q;
    if (p.q_out) p.q_out[1ll * lane * p.N + pix] = q;
  }
  if (p.arg_out) {
    // argmax with the lowest index on ties (np.argmax / torch.argmax convention)
    float best = on ? q : -1.f;
    int idx = lane;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
      if (ob > best || (ob == best && oi < idx)) { best = ob; idx = oi; }
    }
    if (lane == 0) p.arg_out[pix] = static_cast<unsigned char>(idx);
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

// One application of a lattice filter, without the slice: values (zeroed by the caller, [(M+1)][32]) <- splat of
// scale[pixel] * in[pixel][:C] (in == null: ones), then the d+1 blur passes (ping-pong with values_tmp; neighbours
// n1 / n2: [d+1][M], -1 = missing).  The blurred values end up in values_tmp for d = 2 (three passes) and back in
// values for d = 5 (six passes).
extern "C" int stego_crf_splat_blur(int d, long long N, int M, int C, const int* offset, const float* bary, const float* scale,
                                    const float* in, const int* n1, const int* n2, float* values, float* values_tmp,
                                    void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG((d == 2 || d == 5) && N > 0 && M > 0 && C > 0 && C <= CRF_LD && offset && bary && n1 && n2 && values &&
                  values_tmp, "stego_crf_splat_blur: bad args");
  const unsigned pb = (unsigned)((N * 32 + 255) / 256);
  if (d == 2) crf_splat_kernel<2><<<pb, 256, 0, stream>>>(offset, bary, scale, in, in == nullptr, values, N, C);
  else crf_splat_kernel<5><<<pb, 256, 0, stream>>>(offset, bary, scale, in, in == nullptr, values, N, C);
  STEGO_CHECK_LAUNCH("crf_splat_kernel");
  float* a = values;
  float* b = values_tmp;
  const unsigned mb = (unsigned)((1ll * M * 32 + 255) / 256);
  for (int j = 0; j <= d; ++j) {
    crf_blur_kernel<<<mb, 256, 0, stream>>>(a, b, n1 + 1ll * j * M, n2 + 1ll * j * M, M, C);
    STEGO_CHECK_LAUNCH("crf_blur_kernel");
    float* t = a; a = b; b = t;
  }
  return STEGO_OK;
}

// norm[pixel] = 1 / sqrt(K 1 + 1e-20) from the blurred values of a ones-splat (C = 1).
extern "C" int stego_crf_norm(int d, long long N, const int* offset, const float* bary, const float* values, float* norm_out,
                              void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG((d == 2 || d == 5) && N > 0 && offset && bary && values && norm_out, "stego_crf_norm: bad args");
  const unsigned blocks = (unsigned)((N + 255) / 256);
  const float alpha = 1.0f / (1.0f + exp2f(-(float)d));
  if (d == 2) crf_slice1_kernel<2><<<blocks, 256, 0, stream>>>(offset, bary, values, alpha, norm_out, N);
  else crf_slice1_kernel<5><<<blocks, 256, 0, stream>>>(offset, bary, values, alpha, norm_out, N);
  STEGO_CHECK_LAUNCH("crf_slice1_kernel");
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

// One mean-field update from the blurred lattice values of both kernels (see UpdateParams).
extern "C" int stego_crf_update(const float* unary, const int* off_g, const float* bary_g, const float* val_g, const float* norm_g,
                                const int* off_b, const float* bary_b, const float* val_b, const float* norm_b, float w_g,
                                float w_b, float* Q, float* q_out, unsigned char* argmax_out, long long N, int C, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(unary && off_g && bary_g && val_g && norm_g && off_b && bary_b && val_b && norm_b && Q && N > 0 && C > 0 &&
                  C <= CRF_LD, "stego_crf_update: bad args");
  UpdateParams p;
  p.unary = unary; p.off_g = off_g; p.bary_g = bary_g; p.val_g = val_g; p.norm_g = norm_g;
  p.off_b = off_b; p.bary_b = bary_b; p.val_b = val_b; p.norm_b = norm_b; p.w_g = w_g; p.w_b = w_b;
  p.Q = Q; p.q_out = q_out; p.arg_out = argmax_out; p.N = N; p.C = C;
  crf_update_kernel<<<(unsigned)((N * 32 + 255) / 256), 256, 0, stream>>>(p);
  STEGO_CHECK_LAUNCH("crf_update_kernel");
  return STEGO_OK;
}
