// Contrastive CRF loss (optional training term, SURVEY.md §8 row f4): src/modules.py:437-469
//     coords        = randint(h) x randint(w), n_samples points shared by the whole batch
//     sim_kernel    = w1 exp(-|dp|^2 / 2 alpha - |dI|^2 / 2 beta) + w2 exp(-|dp|^2 / 2 gamma) - shift      [B, n, n]
//     cluster_sims  = einsum("nka,nkb->nab", clusters[..., coords], clusters[..., coords])                 [B, n, n]
//     return -(cluster_sims * sim_kernel)
// The reference materialises coord_diff, guidance_diff ([B, 3, n, n]), two exponentials, the Gram matrix and the product
// as separate [B, n, n] tensors (n = 1000: 4 MB each per image).  Here: one gather kernel that lays the selected code
// vectors out k-major ([B][C][n], n contiguous), then one tile kernel that computes the 64 x 64 Gram tile with fp32 FMAs
// out of shared memory (fp32 parity with the reference; 4.5 GFLOP per step at B = 32 — not worth a tensor-core path),
// evaluates the pairwise kernel in registers and writes the product once.  The backward recomputes the (symmetric)
// pairwise kernel instead of saving it:  d sel[a] = sum_b -(g[a,b] + g[b,a]) sim[a,b] sel[b],  scattered back to the
// code gradient with atomics (coords may repeat).
//
// The training step's term, crf_loss_fn(resize(img, 56), normalize(resize(code, 56))).mean() (train_segmentation.py:
// 201-208), has entry points of its own (stego_crf_guidance / _mean_fwd / _mean_loss / _mean_bwd): the loss reads only
// the n sampled points, so neither 56 x 56 map is built.  The gathers take the bilinear taps of F.interpolate(...,
// align_corners=False) at the samples (resize.cuh: bit-equal to torch's resized maps there) and normalise the code over
// its channels; the tile kernel's MEAN mode writes one fixed-order fp64 partial per tile instead of [B, n, n], and the
// backward's UNIFORM mode takes the mean's scalar gradient in place of grad_out.  d sel goes back through the norm and
// the taps into the code gradient with atomics.
#include "common.cuh"
#include "host_util.h"
#include "resize.cuh"

namespace stego {

constexpr int CL_T = 64;   // output tile edge
constexpr int CL_WS = 65;  // row stride of the transposed weight tile (conflict-free both ways)

struct CrfLossParams {
  const float* sel;      // [B][C][NP] gathered code vectors, k-major, zero padded to NP = round_up(n, 64)
  const float4* gsel;    // [B][NP] gathered guidance (up to 3 channels + 0)
  const int2* pos;       // [NP] (y, x) of every sample
  int B, C, n, NP;
  float inv2a, inv2b, inv2g, w1, w2, shift;
  float* out;            // fwd: [B][n][n]
  double* tile_sum;      // fwd, MEAN: [B][NP/64][NP/64] sum of each tile's outputs
  const float* gout;     // bwd: [B][n][n] upstream gradient
  const float* gscalar;  // bwd, UNIFORM: [1] the upstream gradient of every output
  float* dsel;           // bwd: [B][C][NP]
};

__device__ __forceinline__ float crf_pair_kernel(const CrfLossParams& p, int2 pa, int2 pb, float4 ga, float4 gb) {
  const int dy = pa.x - pb.x, dx = pa.y - pb.y;
  const float cd = static_cast<float>(dy * dy + dx * dx);
  const float d0 = ga.x - gb.x, d1 = ga.y - gb.y, d2 = ga.z - gb.z;
  const float gd = d0 * d0 + d1 * d1 + d2 * d2;
  return p.w1 * expf(-cd * p.inv2a - gd * p.inv2b) + p.w2 * expf(-cd * p.inv2g) - p.shift;
}

// gather: one thread per (image, channel-or-guidance, sample)
struct CrfGatherParams {
  const float* clusters; long long c_sb, c_sc, c_sy, c_sx;   // element strides of [B, C, H, W]
  const float* guidance; long long g_sb, g_sc, g_sy, g_sx;   // [B, Cg, H, W]
  const long long* coords;                                    // [2][n]: row 0 indexes H, row 1 indexes W
  int B, C, Cg, n, NP, H, W;
  float* sel; float4* gsel; int2* pos;
};

__global__ void __launch_bounds__(256) crf_loss_gather_kernel(CrfGatherParams p) {
  const int a = blockIdx.x * 256 + threadIdx.x;
  const int k = blockIdx.y, b = blockIdx.z;
  if (a >= p.NP) return;
  const bool real = a < p.n;
  int y = 0, x = 0;
  if (real) {
    y = static_cast<int>(p.coords[a]);
    x = static_cast<int>(p.coords[p.n + a]);
  }
  if (k < p.C) {
    p.sel[(1ll * b * p.C + k) * p.NP + a] = real ? p.clusters[b * p.c_sb + k * p.c_sc + y * p.c_sy + x * p.c_sx] : 0.f;
  } else {  // k == C: guidance + positions
    float g[3] = {0.f, 0.f, 0.f};
    if (real)
      for (int c = 0; c < p.Cg; ++c) g[c] = p.guidance[b * p.g_sb + c * p.g_sc + y * p.g_sy + x * p.g_sx];
    p.gsel[1ll * b * p.NP + a] = make_float4(g[0], g[1], g[2], 0.f);
    if (b == 0) p.pos[a] = make_int2(y, x);
  }
}

// forward: grid (NP/64, NP/64, B), 256 threads as 16 x 16, 4 x 4 outputs each.  MEAN: the tile's sum instead of the tile
template <bool MEAN>
__global__ void __launch_bounds__(256) crf_loss_fwd_kernel(CrfLossParams p) {
  extern __shared__ __align__(16) float sm[];
  float* As = sm;                  // [C][64]
  float* Bs = sm + p.C * CL_T;     // [C][64]
  __shared__ float4 ga_s[CL_T], gb_s[CL_T];
  __shared__ int2 pa_s[CL_T], pb_s[CL_T];
  const int b = blockIdx.z, a0 = blockIdx.y * CL_T, b0 = blockIdx.x * CL_T;
  const float* sel = p.sel + 1ll * b * p.C * p.NP;
  for (int i = threadIdx.x; i < p.C * (CL_T / 4); i += 256) {
    const int k = i / (CL_T / 4), q = i % (CL_T / 4);
    reinterpret_cast<float4*>(As)[i] = *reinterpret_cast<const float4*>(sel + 1ll * k * p.NP + a0 + 4 * q);
    reinterpret_cast<float4*>(Bs)[i] = *reinterpret_cast<const float4*>(sel + 1ll * k * p.NP + b0 + 4 * q);
  }
  if (threadIdx.x < CL_T) {
    ga_s[threadIdx.x] = p.gsel[1ll * b * p.NP + a0 + threadIdx.x];
    pa_s[threadIdx.x] = p.pos[a0 + threadIdx.x];
  } else if (threadIdx.x < 2 * CL_T) {
    const int t = threadIdx.x - CL_T;
    gb_s[t] = p.gsel[1ll * b * p.NP + b0 + t];
    pb_s[t] = p.pos[b0 + t];
  }
  __syncthreads();
  const int ty = threadIdx.x >> 4, tx = threadIdx.x & 15;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int k = 0; k < p.C; ++k) {
    const float4 av = *reinterpret_cast<const float4*>(As + k * CL_T + 4 * ty);
    const float4 bv = *reinterpret_cast<const float4*>(Bs + k * CL_T + 4 * tx);
    const float ar[4] = {av.x, av.y, av.z, av.w}, br[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(ar[i], br[j], acc[i][j]);
  }
  if constexpr (MEAN) {
    // the thread's outputs in row order, then a fixed tree over the CTA: the sum repeats bit for bit
    __shared__ double part[256];
    double t = 0.0;
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (a0 + 4 * ty + i < p.n && b0 + 4 * tx + j < p.n)
          t += static_cast<double>(
              -(acc[i][j] * crf_pair_kernel(p, pa_s[4 * ty + i], pb_s[4 * tx + j], ga_s[4 * ty + i], gb_s[4 * tx + j])));
    part[threadIdx.x] = t;
    __syncthreads();
    for (int w = 128; w > 0; w >>= 1) {
      if (threadIdx.x < w) part[threadIdx.x] += part[threadIdx.x + w];
      __syncthreads();
    }
    if (threadIdx.x == 0) p.tile_sum[(1ll * b * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x] = part[0];
    return;
  }
  const bool vec = (p.n & 3) == 0;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int a = a0 + 4 * ty + i;
    if (a >= p.n) continue;
    float o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j)
      o[j] = -(acc[i][j] * crf_pair_kernel(p, pa_s[4 * ty + i], pb_s[4 * tx + j], ga_s[4 * ty + i], gb_s[4 * tx + j]));
    float* dst = p.out + (1ll * b * p.n + a) * p.n + b0 + 4 * tx;
    if (vec && b0 + 4 * tx + 3 < p.n) {
      *reinterpret_cast<float4*>(dst) = make_float4(o[0], o[1], o[2], o[3]);
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (b0 + 4 * tx + j < p.n) dst[j] = o[j];
    }
  }
}

// backward: grid (NP/64, B); the CTA owns 64 samples a and walks all b tiles.  UNIFORM: every upstream gradient is
// *gscalar (the mean's), read once instead of from [B][n][n]
constexpr int CL_KMAX = 20;  // channels per thread group (C <= 80)
template <bool UNIFORM>
__global__ void __launch_bounds__(256) crf_loss_bwd_kernel(CrfLossParams p) {
  extern __shared__ __align__(16) float sm[];
  float* Bs = sm;                    // [C][64]   sel of the current b tile
  float* Wt = sm + p.C * CL_T;       // [64 b][64 a]  -(g[a,b] + g[b,a]) sim[a,b]
  __shared__ float4 ga_s[CL_T], gb_s[CL_T];
  __shared__ int2 pa_s[CL_T], pb_s[CL_T];
  const int b = blockIdx.y, a0 = blockIdx.x * CL_T;
  const float* sel = p.sel + 1ll * b * p.C * p.NP;
  const float* g = UNIFORM ? nullptr : p.gout + 1ll * b * p.n * p.n;
  const float gs = UNIFORM ? p.gscalar[0] : 0.f;
  if (threadIdx.x < CL_T) {
    ga_s[threadIdx.x] = p.gsel[1ll * b * p.NP + a0 + threadIdx.x];
    pa_s[threadIdx.x] = p.pos[a0 + threadIdx.x];
  }
  const int a = threadIdx.x & 63, kq = threadIdx.x >> 6;
  const int kper = (p.C + 3) / 4, kbeg = kq * kper;
  float acc[CL_KMAX];
#pragma unroll
  for (int i = 0; i < CL_KMAX; ++i) acc[i] = 0.f;
  for (int b0 = 0; b0 < p.NP; b0 += CL_T) {
    __syncthreads();  // previous tile consumed (and ga_s / pa_s visible on the first pass)
    for (int i = threadIdx.x; i < p.C * (CL_T / 4); i += 256) {
      const int k = i / (CL_T / 4), q = i % (CL_T / 4);
      reinterpret_cast<float4*>(Bs)[i] = *reinterpret_cast<const float4*>(sel + 1ll * k * p.NP + b0 + 4 * q);
    }
    if (threadIdx.x < CL_T) {
      gb_s[threadIdx.x] = p.gsel[1ll * b * p.NP + b0 + threadIdx.x];
      pb_s[threadIdx.x] = p.pos[b0 + threadIdx.x];
    }
    // g[a0 + r][b0 + c] read row-wise (coalesced) into Wt[c][r]; g[b0 + r][a0 + c] read row-wise and added at Wt[r][c]
    for (int i = threadIdx.x; i < CL_T * CL_T; i += 256) {
      const int r = i >> 6, c = i & 63;
      const int ga = a0 + r, gb = b0 + c;
      Wt[c * CL_WS + r] = (ga < p.n && gb < p.n) ? (UNIFORM ? gs : g[1ll * ga * p.n + gb]) : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < CL_T * CL_T; i += 256) {
      const int r = i >> 6, c = i & 63;  // r: b index, c: a index
      const int gb = b0 + r, ga = a0 + c;
      const float gt = (ga < p.n && gb < p.n) ? (UNIFORM ? gs : g[1ll * gb * p.n + ga]) : 0.f;
      const float s = crf_pair_kernel(p, pa_s[c], pb_s[r], ga_s[c], gb_s[r]);
      Wt[r * CL_WS + c] = -(Wt[r * CL_WS + c] + gt) * s;
    }
    __syncthreads();
#pragma unroll 1
    for (int b4 = 0; b4 < CL_T / 4; ++b4) {
      const float w0 = Wt[(4 * b4 + 0) * CL_WS + a], w1 = Wt[(4 * b4 + 1) * CL_WS + a];
      const float w2 = Wt[(4 * b4 + 2) * CL_WS + a], w3 = Wt[(4 * b4 + 3) * CL_WS + a];
#pragma unroll
      for (int kk = 0; kk < CL_KMAX; ++kk) {
        if (kk < kper && kbeg + kk < p.C) {
          const float4 v = *reinterpret_cast<const float4*>(Bs + (kbeg + kk) * CL_T + 4 * b4);
          acc[kk] = fmaf(w0, v.x, fmaf(w1, v.y, fmaf(w2, v.z, fmaf(w3, v.w, acc[kk]))));
        }
      }
    }
  }
#pragma unroll
  for (int kk = 0; kk < CL_KMAX; ++kk)
    if (kk < kper && kbeg + kk < p.C) p.dsel[(1ll * b * p.C + kbeg + kk) * p.NP + a0 + a] = acc[kk];
}

struct CrfScatterParams {
  const float* dsel; const long long* coords; int B, C, n, NP;
  float* dclusters; long long sb, sc, sy, sx;
};
__global__ void __launch_bounds__(256) crf_loss_scatter_kernel(CrfScatterParams p) {
  const int a = blockIdx.x * 256 + threadIdx.x;
  const int k = blockIdx.y, b = blockIdx.z;
  if (a >= p.n) return;
  const long long y = p.coords[a], x = p.coords[p.n + a];
  atomicAdd(p.dclusters + b * p.sb + k * p.sc + y * p.sy + x * p.sx, p.dsel[(1ll * b * p.C + k) * p.NP + a]);
}

// ---- the training step's term: samples at S x S (56) positions of the bilinearly resized code and image
struct CrfStepParams {
  const float* src; long long sb, sc, sy, sx;   // code [B][C][h][w] (guidance: the image [B][Cg][h][w]), any strides
  const long long* coords;                      // [2][n]: rows, then columns, of the S x S map
  int B, C, n, NP, h, w;
  float scale_h, scale_w;                       // ATen's (float)h / S, (float)w / S
  float* raw; float* sel; float* nrm;           // [B][C][NP] samples and normalised samples (k-major), [B][NP] norms
  float4* gsel; int2* pos;                      // guidance: [B][NP], [NP]
  const float* dsel;                            // bwd: [B][C][NP]
};

__device__ __forceinline__ ResizeTaps crf_sample_taps(const CrfStepParams& p, int a) {
  return resize_taps(static_cast<int>(p.coords[a]), static_cast<int>(p.coords[p.n + a]), p.scale_h, p.scale_w, p.h, p.w);
}

// one thread per (image, sample): the resized image channels at the sample (and the positions, once)
__global__ void __launch_bounds__(256) crf_guidance_kernel(CrfStepParams p) {
  const int a = blockIdx.x * 256 + threadIdx.x, b = blockIdx.y;
  if (a >= p.NP) return;
  float g[3] = {0.f, 0.f, 0.f};
  int2 yx = make_int2(0, 0);
  if (a < p.n) {
    const ResizeTaps t = crf_sample_taps(p, a);
    const float* base = p.src + b * p.sb;
    for (int c = 0; c < p.C; ++c)
      g[c] = resize_at(t, [&](int y, int x) { return base[c * p.sc + y * p.sy + x * p.sx]; });
    yx = make_int2(static_cast<int>(p.coords[a]), static_cast<int>(p.coords[p.n + a]));
  }
  p.gsel[1ll * b * p.NP + a] = make_float4(g[0], g[1], g[2], 0.f);
  if (b == 0) p.pos[a] = yx;
}

// one warp per (image, sample), lanes over channels (C <= 80 < 96): the resized code at the sample, then F.normalize
// (x / max(|x|, eps)) over the channels; padding samples are zero.  NHWC: the arithmetic of ATen's channels-last kernel,
// which F.interpolate runs for a channels-last code of >= 16 channels (the head's output is one)
template <bool NHWC>
__global__ void __launch_bounds__(256) crf_code_gather_kernel(CrfStepParams p) {
  const long long wid = (1ll * blockIdx.x * 256 + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (wid >= 1ll * p.B * p.NP) return;
  const int b = static_cast<int>(wid / p.NP), a = static_cast<int>(wid % p.NP);
  float v[3] = {0.f, 0.f, 0.f};
  float ss = 0.f;
  if (a < p.n) {
    const ResizeTaps t = crf_sample_taps(p, a);
    const float* base = p.src + b * p.sb;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      const int c = lane + 32 * j;
      if (c < p.C) {
        const auto at = [&](int y, int x) { return base[c * p.sc + y * p.sy + x * p.sx]; };
        v[j] = NHWC ? resize_at_nhwc(t, at) : resize_at(t, at);
        ss = fmaf(v[j], v[j], ss);
      }
    }
  }
  const float nv = sqrtf(warp_sum(ss)), den = fmaxf(nv, 1e-10f);
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const int c = lane + 32 * j;
    if (c < p.C) {
      p.raw[(1ll * b * p.C + c) * p.NP + a] = v[j];
      p.sel[(1ll * b * p.C + c) * p.NP + a] = v[j] / den;
    }
  }
  if (lane == 0) p.nrm[1ll * b * p.NP + a] = nv;
}

// one warp per (image, sample): d x = (d sel - [|x| >= eps] sel <sel, d sel>) / max(|x|, eps) (F.normalize's backward),
// then d code += the four tap weights x d x, by atomics (samples repeat and taps of different samples coincide)
__global__ void __launch_bounds__(256) crf_code_scatter_kernel(CrfStepParams p, float* dcode) {
  const long long wid = (1ll * blockIdx.x * 256 + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (wid >= 1ll * p.B * p.n) return;
  const int b = static_cast<int>(wid / p.n), a = static_cast<int>(wid % p.n);
  float y[3], dy[3], dot = 0.f;
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const int c = lane + 32 * j;
    const long long o = (1ll * b * p.C + c) * p.NP + a;
    y[j] = c < p.C ? p.sel[o] : 0.f;
    dy[j] = c < p.C ? p.dsel[o] : 0.f;
    dot = fmaf(y[j], dy[j], dot);
  }
  dot = warp_sum(dot);
  const float nv = p.nrm[1ll * b * p.NP + a], den = fmaxf(nv, 1e-10f), k = nv >= 1e-10f ? dot : 0.f;
  const ResizeTaps t = crf_sample_taps(p, a);
  const float h1l = t.ly, h0l = 1.f - t.ly, w1l = t.lx, w0l = 1.f - t.lx;
  const float wt[4] = {h0l * w0l, h0l * w1l, h1l * w0l, h1l * w1l};
  const long long off[4] = {t.y0 * p.sy + t.x0 * p.sx, t.y0 * p.sy + t.x1 * p.sx, t.y1 * p.sy + t.x0 * p.sx,
                            t.y1 * p.sy + t.x1 * p.sx};
  float* base = dcode + b * p.sb;
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const int c = lane + 32 * j;
    if (c >= p.C) continue;
    const float dx = (dy[j] - k * y[j]) / den;
#pragma unroll
    for (int q = 0; q < 4; ++q)
      if (wt[q] != 0.f) atomicAdd(base + c * p.sc + off[q], wt[q] * dx);
  }
}

// loss[0] = (sum of the tile sums) / count, in fp64 in a fixed order by one CTA; total[0] += weight * loss[0] (if given)
constexpr int kMeanThreads = 1024;
__global__ void __launch_bounds__(kMeanThreads) crf_mean_loss_kernel(const double* tile_sum, long long cnt, double count,
                                                                    float weight, float* loss, float* total) {
  __shared__ double part[kMeanThreads];
  double s = 0.0;
  for (long long i = threadIdx.x; i < cnt; i += kMeanThreads) s += tile_sum[i];
  part[threadIdx.x] = s;
  __syncthreads();
  for (int w = kMeanThreads / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) part[threadIdx.x] += part[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const float l = static_cast<float>(part[0] / count);
    loss[0] = l;
    if (total) total[0] = __fadd_rn(total[0], __fmul_rn(weight, l));
  }
}

static int crf_loss_check(int B, int C, int Cg, int n, int H, int W) {
  STEGO_CHECK_ARG(B > 0 && C > 0 && C <= 80 && Cg > 0 && Cg <= 3 && n > 0 && H > 0 && W > 0,
                  "stego_crf_loss: B=%d C=%d Cg=%d n=%d unsupported (C <= 80, guidance channels <= 3)", B, C, Cg, n);
  return STEGO_OK;
}

}  // namespace stego

using namespace stego;

// Workspace (caller-allocated): sel [B][C][NP] floats, gsel [B][NP] float4, pos [NP] int2, NP = round_up(n, 64).
// Strides are in elements; coords is the reference's [2][n] int64 tensor (row 0 indexes H, row 1 indexes W).
extern "C" int stego_crf_loss_fwd(const float* guidance, long long g_sb, long long g_sc, long long g_sy, long long g_sx, int Cg,
                                  const float* clusters, long long c_sb, long long c_sc, long long c_sy, long long c_sx, int C,
                                  const long long* coords, int B, int n, int H, int W, float alpha, float beta, float gamma,
                                  float w1, float w2, float shift, float* sel, float* gsel, int* pos, float* out,
                                  void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(guidance && clusters && coords && sel && gsel && pos && out, "stego_crf_loss_fwd: null pointer");
  if (int rc = crf_loss_check(B, C, Cg, n, H, W)) return rc;
  const int NP = (n + CL_T - 1) / CL_T * CL_T;
  CrfGatherParams gp;
  gp.clusters = clusters; gp.c_sb = c_sb; gp.c_sc = c_sc; gp.c_sy = c_sy; gp.c_sx = c_sx;
  gp.guidance = guidance; gp.g_sb = g_sb; gp.g_sc = g_sc; gp.g_sy = g_sy; gp.g_sx = g_sx;
  gp.coords = coords; gp.B = B; gp.C = C; gp.Cg = Cg; gp.n = n; gp.NP = NP; gp.H = H; gp.W = W;
  gp.sel = sel; gp.gsel = reinterpret_cast<float4*>(gsel); gp.pos = reinterpret_cast<int2*>(pos);
  crf_loss_gather_kernel<<<dim3((NP + 255) / 256, C + 1, B), 256, 0, stream>>>(gp);
  STEGO_CHECK_LAUNCH("crf_loss_gather_kernel");
  CrfLossParams p;
  p.sel = sel; p.gsel = reinterpret_cast<const float4*>(gsel); p.pos = reinterpret_cast<const int2*>(pos);
  p.B = B; p.C = C; p.n = n; p.NP = NP;
  p.inv2a = 1.0f / (2.0f * alpha); p.inv2b = 1.0f / (2.0f * beta); p.inv2g = 1.0f / (2.0f * gamma);
  p.w1 = w1; p.w2 = w2; p.shift = shift; p.out = out; p.tile_sum = nullptr; p.gout = nullptr; p.gscalar = nullptr;
  p.dsel = nullptr;
  crf_loss_fwd_kernel<false><<<dim3(NP / CL_T, NP / CL_T, B), 256, (size_t)2 * C * CL_T * sizeof(float), stream>>>(p);
  STEGO_CHECK_LAUNCH("crf_loss_fwd_kernel");
  return STEGO_OK;
}

// Backward with the workspace the forward filled (sel, gsel, pos).  grad_out [B][n][n] contiguous; dsel [B][C][NP] scratch;
// dclusters (same strides as clusters) is ACCUMULATED into: the caller zero-fills it.
extern "C" int stego_crf_loss_bwd(const float* grad_out, const float* sel, const float* gsel, const int* pos,
                                  const long long* coords, int B, int C, int n, float alpha, float beta, float gamma, float w1,
                                  float w2, float shift, float* dsel, float* dclusters, long long c_sb, long long c_sc,
                                  long long c_sy, long long c_sx, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(grad_out && sel && gsel && pos && coords && dsel && dclusters, "stego_crf_loss_bwd: null pointer");
  if (int rc = crf_loss_check(B, C, 1, n, 1, 1)) return rc;
  const int NP = (n + CL_T - 1) / CL_T * CL_T;
  CrfLossParams p;
  p.sel = sel; p.gsel = reinterpret_cast<const float4*>(gsel); p.pos = reinterpret_cast<const int2*>(pos);
  p.B = B; p.C = C; p.n = n; p.NP = NP;
  p.inv2a = 1.0f / (2.0f * alpha); p.inv2b = 1.0f / (2.0f * beta); p.inv2g = 1.0f / (2.0f * gamma);
  p.w1 = w1; p.w2 = w2; p.shift = shift; p.out = nullptr; p.tile_sum = nullptr; p.gout = grad_out; p.gscalar = nullptr;
  p.dsel = dsel;
  const size_t smem = ((size_t)C * CL_T + CL_T * CL_WS) * sizeof(float);
  crf_loss_bwd_kernel<false><<<dim3(NP / CL_T, B), 256, smem, stream>>>(p);
  STEGO_CHECK_LAUNCH("crf_loss_bwd_kernel");
  CrfScatterParams sp;
  sp.dsel = dsel; sp.coords = coords; sp.B = B; sp.C = C; sp.n = n; sp.NP = NP;
  sp.dclusters = dclusters; sp.sb = c_sb; sp.sc = c_sc; sp.sy = c_sy; sp.sx = c_sx;
  crf_loss_scatter_kernel<<<dim3((n + 255) / 256, C, B), 256, 0, stream>>>(sp);
  STEGO_CHECK_LAUNCH("crf_loss_scatter_kernel");
  return STEGO_OK;
}

// ---- the training step's term (see the head of this file).  S: the side of the resized maps (56); coords [2][n] index
// them.  Workspace: gsel [B][NP] float4, pos [NP] int2, sel / dsel [B][C][NP], nrm [B][NP], tile_sum [B][NP/64][NP/64]
// doubles, NP = round_up(n, 64).

static int crf_step_check(int B, int C, int n, int h, int w, int S, const char* who) {
  STEGO_CHECK_ARG(B > 0 && C > 0 && C <= 80 && n > 0 && h > 0 && w > 0 && S > 0,
                  "%s: B=%d C=%d n=%d h=%d w=%d S=%d unsupported (C <= 80)", who, B, C, n, h, w, S);
  return STEGO_OK;
}

static CrfStepParams crf_step_params(const float* src, long long sb, long long sc, long long sy, long long sx,
                                     const long long* coords, int B, int C, int n, int h, int w, int S) {
  CrfStepParams p{};
  p.src = src; p.sb = sb; p.sc = sc; p.sy = sy; p.sx = sx; p.coords = coords;
  p.B = B; p.C = C; p.n = n; p.NP = (n + CL_T - 1) / CL_T * CL_T; p.h = h; p.w = w;
  p.scale_h = static_cast<float>(h) / static_cast<float>(S);
  p.scale_w = static_cast<float>(w) / static_cast<float>(S);
  return p;
}

static CrfLossParams crf_tile_params(int B, int C, int n, float alpha, float beta, float gamma, float w1, float w2,
                                     float shift, const float* sel, const float* gsel, const int* pos) {
  CrfLossParams p{};
  p.sel = sel; p.gsel = reinterpret_cast<const float4*>(gsel); p.pos = reinterpret_cast<const int2*>(pos);
  p.B = B; p.C = C; p.n = n; p.NP = (n + CL_T - 1) / CL_T * CL_T;
  p.inv2a = 1.0f / (2.0f * alpha); p.inv2b = 1.0f / (2.0f * beta); p.inv2g = 1.0f / (2.0f * gamma);
  p.w1 = w1; p.w2 = w2; p.shift = shift;
  return p;
}

// gsel / pos from the image (fp32 [B][Cg][H][W], any strides, Cg <= 3) resized to S x S, at the samples
extern "C" int stego_crf_guidance(const float* img, long long sb, long long sc, long long sy, long long sx, int Cg,
                                  int H, int W, const long long* coords, int B, int n, int S, float* gsel, int* pos,
                                  void* stream_) {
  STEGO_CHECK_ARG(img && coords && gsel && pos, "stego_crf_guidance: null pointer");
  STEGO_CHECK_ARG(Cg >= 1 && Cg <= 3, "stego_crf_guidance: %d guidance channels (<= 3)", Cg);
  if (int rc = crf_step_check(B, 1, n, H, W, S, "stego_crf_guidance")) return rc;
  CrfStepParams p = crf_step_params(img, sb, sc, sy, sx, coords, B, Cg, n, H, W, S);
  p.gsel = reinterpret_cast<float4*>(gsel); p.pos = reinterpret_cast<int2*>(pos);
  crf_guidance_kernel<<<dim3((p.NP + 255) / 256, B), 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(p);
  STEGO_CHECK_LAUNCH("crf_guidance_kernel");
  return STEGO_OK;
}

// raw / sel / nrm from the code (fp32 [B][C][h][w], any strides), then the tile sums of -(Gram x pairwise kernel)
extern "C" int stego_crf_mean_fwd(const float* code, long long sb, long long sc, long long sy, long long sx, int C, int h,
                                  int w, const long long* coords, int B, int n, int S, float alpha, float beta,
                                  float gamma, float w1, float w2, float shift, const float* gsel, const int* pos,
                                  float* raw, float* sel, float* nrm, double* tile_sum, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(code && coords && gsel && pos && raw && sel && nrm && tile_sum, "stego_crf_mean_fwd: null pointer");
  if (int rc = crf_step_check(B, C, n, h, w, S, "stego_crf_mean_fwd")) return rc;
  CrfStepParams g = crf_step_params(code, sb, sc, sy, sx, coords, B, C, n, h, w, S);
  g.raw = raw; g.sel = sel; g.nrm = nrm;
  const long long threads = 32ll * B * g.NP;
  if (C >= 16 && aten_channels_last(B, C, h, w, sb, sc, sy, sx))
    crf_code_gather_kernel<true><<<(unsigned)((threads + 255) / 256), 256, 0, stream>>>(g);
  else
    crf_code_gather_kernel<false><<<(unsigned)((threads + 255) / 256), 256, 0, stream>>>(g);
  STEGO_CHECK_LAUNCH("crf_code_gather_kernel");
  CrfLossParams p = crf_tile_params(B, C, n, alpha, beta, gamma, w1, w2, shift, sel, gsel, pos);
  p.tile_sum = tile_sum;
  crf_loss_fwd_kernel<true><<<dim3(g.NP / CL_T, g.NP / CL_T, B), 256, (size_t)2 * C * CL_T * sizeof(float), stream>>>(p);
  STEGO_CHECK_LAUNCH("crf_loss_fwd_kernel");
  return STEGO_OK;
}

// loss[0] = mean of the B n^2 outputs from the tile sums; total[0] += weight * loss[0] when total is given
extern "C" int stego_crf_mean_loss(const double* tile_sum, int B, int n, float weight, float* loss, float* total,
                                   void* stream_) {
  STEGO_CHECK_ARG(tile_sum && loss && B > 0 && n > 0, "stego_crf_mean_loss: null pointer or B=%d n=%d", B, n);
  const long long nt = (n + CL_T - 1) / CL_T;
  crf_mean_loss_kernel<<<1, kMeanThreads, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      tile_sum, B * nt * nt, static_cast<double>(B) * n * n, weight, loss, total);
  STEGO_CHECK_LAUNCH("crf_mean_loss_kernel");
  return STEGO_OK;
}

// d code (the forward's code strides) += the gradient of the mean with upstream gradient gscalar[0] (fl(weight / B n^2)),
// by atomics; dsel is scratch
extern "C" int stego_crf_mean_bwd(const float* gscalar, const float* sel, const float* nrm, const float* gsel,
                                  const int* pos, const long long* coords, int B, int C, int n, int h, int w, int S,
                                  float alpha, float beta, float gamma, float w1, float w2, float shift, float* dsel,
                                  float* dcode, long long sb, long long sc, long long sy, long long sx, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(gscalar && sel && nrm && gsel && pos && coords && dsel && dcode, "stego_crf_mean_bwd: null pointer");
  if (int rc = crf_step_check(B, C, n, h, w, S, "stego_crf_mean_bwd")) return rc;
  CrfLossParams p = crf_tile_params(B, C, n, alpha, beta, gamma, w1, w2, shift, sel, gsel, pos);
  p.gscalar = gscalar; p.dsel = dsel;
  const size_t smem = ((size_t)C * CL_T + CL_T * CL_WS) * sizeof(float);
  crf_loss_bwd_kernel<true><<<dim3(p.NP / CL_T, B), 256, smem, stream>>>(p);
  STEGO_CHECK_LAUNCH("crf_loss_bwd_kernel");
  CrfStepParams g = crf_step_params(nullptr, sb, sc, sy, sx, coords, B, C, n, h, w, S);
  g.sel = const_cast<float*>(sel); g.nrm = const_cast<float*>(nrm); g.dsel = dsel;
  const long long threads = 32ll * B * n;
  crf_code_scatter_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, stream>>>(g, dcode);
  STEGO_CHECK_LAUNCH("crf_code_scatter_kernel");
  return STEGO_OK;
}
