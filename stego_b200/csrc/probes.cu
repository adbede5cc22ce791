// Probe heads of the STEGO training / eval step (sm_90a; HBM-bound, fp32 arithmetic):
//
//   ClusterLookup            src/modules.py:134-161   cosine similarity to n_classes centroids,
//                                                     argmax one-hot / softmax(alpha.) / log_softmax(alpha.), loss
//   linear probe + CE        src/train_segmentation.py:210-219
//                                                     1x1 conv -> bilinear upsample (align_corners=False) -> masked CE
//
// Both are evaluated per pixel in registers; nothing of size [B, n_classes, H, W] is materialised unless the
// caller asks for the probabilities.  Dot products are sequential fp32 FMAs in channel order, so the
// argmax is deterministic; centroids are normalised once per CTA into shared memory.
#include <algorithm>

#include "host_util.h"
#include "probe_common.cuh"

namespace stego {

constexpr int PR_MAX_CLASSES = 64;
constexpr int PR_MAX_DIM = 96;
constexpr int PR_THREADS = 128;

struct ClusterParams {
  const float* x;            // features, element strides below
  long long sb, sc, sp;      // batch / channel / pixel strides (pixel index = y*W + x must be affine: sp)
  const float* clusters;     // [n][C]
  int B, C, n;
  long long npix;            // pixels per image (H*W)
  int mode;                  // 0: alpha=None (argmax one-hot), 1: softmax(alpha * ip)
  float alpha;
  long long* assign;         // optional [B][npix] argmax
  float* probs;              // optional [B][n][npix] (one-hot or softmax)
  float* logp;               // optional [B][n][npix] log_softmax(alpha * ip)
  float* loss_partials;      // [gridDim.x] sum over pixels of sum_k probs_k * ip_k
  // backward
  const float* grad_loss;    // device scalar: upstream gradient of the loss
  float grad_scale;          // -1 / (B*npix)
  float* dnc;                // [n][C] gradient wrt the NORMALISED centroids (atomically accumulated)
};

template <bool kBackward>
__global__ void __launch_bounds__(PR_THREADS)
cluster_lookup_kernel(ClusterParams p) {
  extern __shared__ float sm[];
  float* snc = sm;                         // [n][C]
  float* sacc = sm + p.n * p.C;            // backward: [n][C] block accumulator
  float* sred = sacc + (kBackward ? p.n * p.C : 0);  // [4]
  normalize_centroids(p.clusters, p.n, p.C, blockDim.x >> 5, snc, p.C, 1);
  __syncthreads();
  if (kBackward) p.grad_scale *= p.grad_loss[0];
  if (kBackward) {
    for (int i = threadIdx.x; i < p.n * p.C; i += blockDim.x) sacc[i] = 0.f;
    __syncthreads();
  }
  const long long total = 1ll * p.B * p.npix;
  float loss_acc = 0.f;
  for (long long pix = 1ll * blockIdx.x * blockDim.x + threadIdx.x; pix < total; pix += 1ll * gridDim.x * blockDim.x) {
    const int b = static_cast<int>(pix / p.npix);
    const long long q = pix % p.npix;
    const float* xp = p.x + b * p.sb + q * p.sp;
    float xv[PR_MAX_DIM];
    float ss = 0.f;
#pragma unroll 8
    for (int c = 0; c < p.C; ++c) { xv[c] = xp[c * p.sc]; ss += xv[c] * xv[c]; }
    const float inv = 1.0f / fmaxf(sqrtf(ss), 1e-12f);
    float ip[PR_MAX_CLASSES];
    float best = -INFINITY;
    int arg = 0;
    for (int k = 0; k < p.n; ++k) {
      float d = 0.f;
      const float* ck = snc + k * p.C;
#pragma unroll 8
      for (int c = 0; c < p.C; ++c) d = fmaf(xv[c] * inv, ck[c], d);
      ip[k] = d;
      if (d > best) { best = d; arg = k; }  // first maximum wins, like torch.argmax
    }
    if (p.mode == 0) {
      loss_acc += best;
      if (!kBackward) {
        if (p.assign) p.assign[pix] = arg;
        if (p.probs)
          for (int k = 0; k < p.n; ++k) p.probs[(1ll * b * p.n + k) * p.npix + q] = (k == arg) ? 1.f : 0.f;
      } else {
        for (int c = 0; c < p.C; ++c) atomicAdd(&sacc[arg * p.C + c], p.grad_scale * xv[c] * inv);
      }
    } else {
      float mx = -INFINITY;
      for (int k = 0; k < p.n; ++k) mx = fmaxf(mx, ip[k] * p.alpha);
      float se = 0.f;
      for (int k = 0; k < p.n; ++k) se += expf(ip[k] * p.alpha - mx);
      const float lse = mx + logf(se);
      float dotp = 0.f;
      for (int k = 0; k < p.n; ++k) dotp += expf(ip[k] * p.alpha - lse) * ip[k];
      loss_acc += dotp;
      if (!kBackward) {
        if (p.assign) p.assign[pix] = arg;
        for (int k = 0; k < p.n; ++k) {
          const float lp = ip[k] * p.alpha - lse;
          if (p.probs) p.probs[(1ll * b * p.n + k) * p.npix + q] = expf(lp);
          if (p.logp) p.logp[(1ll * b * p.n + k) * p.npix + q] = lp;
        }
      } else {
        for (int k = 0; k < p.n; ++k) {
          const float pk = expf(ip[k] * p.alpha - lse);
          const float dip = p.grad_scale * (pk + p.alpha * pk * (ip[k] - dotp));
          for (int c = 0; c < p.C; ++c) atomicAdd(&sacc[k * p.C + c], dip * xv[c] * inv);
        }
      }
    }
  }
  if (!kBackward) {
    loss_acc = warp_sum(loss_acc);
    if ((threadIdx.x & 31) == 0) sred[threadIdx.x >> 5] = loss_acc;
    __syncthreads();
    if (threadIdx.x == 0) {
      float t = 0.f;
      for (int w = 0; w < (blockDim.x >> 5); ++w) t += sred[w];
      p.loss_partials[blockIdx.x] = t;
    }
  } else {
    __syncthreads();
    for (int i = threadIdx.x; i < p.n * p.C; i += blockDim.x)
      if (sacc[i] != 0.f) atomicAdd(p.dnc + i, sacc[i]);
  }
}

// Channels-last variant (channel stride 1; the layout of the training step): one WARP per pixel, lanes = classes.
// The pixel's channels sit in 3 registers per lane and are broadcast with shuffles; each lane accumulates the dot
// product with "its" centroid in the same ascending-channel FMA order as the per-thread kernel above, so both
// kernels produce identical inner products.  Handles alpha=None forward/backward and the softmax forward.
template <bool kBackward>
__global__ void __launch_bounds__(256)
cluster_lookup_cl_kernel(ClusterParams p) {
  extern __shared__ float sm[];
  float* sncT = sm;                        // [C][32] transposed normalised centroids (lanes >= n read 0)
  float* sacc = sm + p.C * 32;             // backward: [n][C]
  __shared__ float sred[8];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < p.C * 32; i += blockDim.x) sncT[i] = 0.f;
  if (kBackward)
    for (int i = threadIdx.x; i < p.n * p.C; i += blockDim.x) sacc[i] = 0.f;
  __syncthreads();
  normalize_centroids(p.clusters, p.n, p.C, 8, sncT, 1, 32);
  __syncthreads();
  const float gs = kBackward ? p.grad_scale * p.grad_loss[0] : 0.f;
  const long long total = 1ll * p.B * p.npix;
  float loss_acc = 0.f;
  for (long long pix = 1ll * blockIdx.x * 8 + warp; pix < total; pix += 1ll * gridDim.x * 8) {
    const int b = static_cast<int>(pix / p.npix);
    const long long q = pix % p.npix;
    const float* xp = p.x + b * p.sb + q * p.sp;
    float xr[3];
    load_channels(xp, p.C, lane, xr);
    // same summation order as the per-thread kernel is not required for the norm (it only scales all classes)
    const float ss = warp_sum(xr[0] * xr[0] + xr[1] * xr[1] + xr[2] * xr[2]);
    const float inv = 1.0f / fmaxf(sqrtf(ss), 1e-12f);
    float d = 0.f;
    for_each_channel(xr, p.C, [&](int c, float xc) { d = fmaf(xc * inv, sncT[c * 32 + lane], d); });
    const float ip = (lane < p.n) ? d : -INFINITY;
    const float best = warp_max(ip);
    const int arg = __ffs(__ballot_sync(0xffffffffu, ip == best)) - 1;  // first maximum, like torch.argmax
    if (p.mode == 0) {
      if (lane == 0) loss_acc += best;
      if (!kBackward) {
        if (p.assign && lane == 0) p.assign[pix] = arg;
        if (p.probs && lane < p.n) p.probs[(1ll * b * p.n + lane) * p.npix + q] = (lane == arg) ? 1.f : 0.f;
      } else {
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const int c = lane + 32 * k;
          if (c < p.C) atomicAdd(&sacc[arg * p.C + c], gs * xr[k] * inv);
        }
      }
    } else {
      const float sc = ip * p.alpha;
      const float mx = warp_max(lane < p.n ? sc : -INFINITY);
      const float e = (lane < p.n) ? expf(sc - mx) : 0.f;
      const float lse = mx + logf(warp_sum(e));
      const float lp = sc - lse;
      const float pk = (lane < p.n) ? expf(lp) : 0.f;
      const float dotp = warp_sum((lane < p.n) ? pk * ip : 0.f);
      if (lane == 0) loss_acc += dotp;
      if (p.assign && lane == 0) p.assign[pix] = arg;
      if (lane < p.n) {
        if (p.probs) p.probs[(1ll * b * p.n + lane) * p.npix + q] = pk;
        if (p.logp) p.logp[(1ll * b * p.n + lane) * p.npix + q] = lp;
      }
    }
  }
  if (!kBackward) {
    if (lane == 0) sred[warp] = loss_acc;
    __syncthreads();
    if (threadIdx.x == 0) {
      float t = 0.f;
      for (int w = 0; w < 8; ++w) t += sred[w];
      p.loss_partials[blockIdx.x] = t;
    }
  } else {
    __syncthreads();
    for (int i = threadIdx.x; i < p.n * p.C; i += blockDim.x)
      if (sacc[i] != 0.f) atomicAdd(p.dnc + i, sacc[i]);
  }
}

// d clusters from d normalised clusters: row-wise normalize backward
__global__ void cluster_norm_bwd_kernel(const float* __restrict__ clusters, const float* __restrict__ dnc,
                                        float* __restrict__ dclusters, int n, int C) {
  const int k = blockIdx.x;
  const int lane = threadIdx.x;
  float ss = 0.f, dot = 0.f;
  for (int c = lane; c < C; c += 32) { const float v = clusters[k * C + c]; ss += v * v; dot += v * dnc[k * C + c]; }
  ss = warp_sum(ss);
  dot = warp_sum(dot);
  const float nrm = sqrtf(ss);
  for (int c = lane; c < C; c += 32) {
    float g;
    if (nrm > 1e-12f) g = (dnc[k * C + c] - clusters[k * C + c] * dot / ss) / nrm;
    else g = dnc[k * C + c] / 1e-12f;
    dclusters[k * C + c] += g;
  }
}

// out[0] = scale * sum(partials[0..n))   (deterministic, single block)
__global__ void sum_partials_kernel(const float* __restrict__ partials, int n, float scale, float* __restrict__ out) {
  __shared__ double sh[256];
  double acc = 0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) acc += static_cast<double>(partials[i]);
  sh[threadIdx.x] = acc;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) out[0] = static_cast<float>(sh[0] * scale);
}

// ---------------------------------------------------------------------------------------------
// linear probe: low-res logits, then per hi-res pixel: bilinear interpolation + masked CE fwd/bwd
// ---------------------------------------------------------------------------------------------
constexpr int LP_LD = 32;  // row stride of the low-res logit / grad buffers (n_classes <= 32)

// one warp per low-res pixel, lanes = classes: channels are broadcast with shuffles, W^T sits in smem as [C][32]
__global__ void __launch_bounds__(256)
linear_logits_kernel(const float* __restrict__ code, long long ld_code, int C, const float* __restrict__ W,
                     const float* __restrict__ bias, int n, float* __restrict__ logits, long long rows) {
  extern __shared__ float sw[];  // [C][32]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < C * 32; i += blockDim.x) {
    const int c = i >> 5, k = i & 31;
    sw[i] = (k < n) ? W[k * C + c] : 0.f;
  }
  __syncthreads();
  const float bk = (lane < n) ? bias[lane] : 0.f;
  for (long long r = 1ll * blockIdx.x * 8 + warp; r < rows; r += 1ll * gridDim.x * 8) {
    float xr[3];
    load_channels(code + r * ld_code, C, lane, xr);
    float d = bk;
    for_each_channel(xr, C, [&](int c, float xc) { d = fmaf(xc, sw[c * 32 + lane], d); });
    logits[r * LP_LD + lane] = (lane < n) ? d : 0.f;
  }
}

struct LinearCEParams {
  const float* logits;   // [B*h*w][LP_LD]
  const void* label;     // [B][H][W] int64 / int32 / uint8 (label_bytes = 8 / 4 / 1; uint8: 255 = ignore)
  int label_bytes;
  int B, h, w, H, W, n;
  float* dlogits;        // [B*h*w][LP_LD] unnormalised gradient (atomics), or null (loss only)
  unsigned long long* dfix;  // linear_ce_kernel<true>: the gradient as int64 fixed point (LCE_FIX_SCALE) instead
  double* acc;           // [2]: loss sum, valid count (zeroed before the launch)
  int tiles_y, tiles_x, box_h, box_w;
};

constexpr int LCE_TILE = 16;  // hi-res pixels per tile side (256 threads = one per pixel)

// One CTA per 16x16 tile of output pixels, three phases, no per-pixel atomics:
//   1. thread = pixel: the low-res logits the tile can touch (its "box") are staged in shared memory; bilinear
//      upsample + softmax + CE in registers; the per-pixel logit gradient g[pixel][k] goes to shared memory.
//   2. the bilinear transpose is separable: T[Y][cx][k] = sum_X wx[X][cx] g[Y][X][k], then
//      G[cy][cx][k] = sum_Y wy[Y][cy] T[Y][cx][k], each a conflict-free shared-memory reduction.
//   3. one global atomic per (box cell, class) of the tile.
constexpr int LCE_SLD = 33;  // smem stride of one box cell (odd: lanes reading different cells hit different banks)
// kFixed: the tiles' contributions to a cell are added as int64 multiples of 2^-40 (every contribution is at most the
// tile's 256 pixel gradients in [-1, 1], far inside the range), and integer adds do not depend on their order: the
// gradient is the same bit for bit from run to run, where float atomics are not
constexpr double LCE_FIX_SCALE = 1099511627776.0;  // 2^40

template <bool kFixed>
__global__ void __launch_bounds__(256)
linear_ce_kernel(LinearCEParams p) {
  extern __shared__ float sm[];
  const int bhm = p.box_h, bwm = p.box_w, n = p.n;
  float* slog = sm;                                   // [box_h*box_w][LCE_SLD]
  float* sg = slog + bhm * bwm * LCE_SLD;             // [256][n]   (odd stride n=27: conflict-free)
  float* sT = sg + 256 * n;                           // [16][box_w][n]  (phase 2)
  float* sX = sT;                                     // [16][box_h][LCE_SLD] (phase 1: logits interpolated along x) — same region
  const int region = max(LCE_TILE * bwm * n, LCE_TILE * bhm * LCE_SLD);
  float* swx = sT + region;                           // [16][box_w]
  float* swy = swx + LCE_TILE * bwm;                  // [16][box_h]
  __shared__ float sred[2][8];
  const int tile = blockIdx.x;
  const int tx = tile % p.tiles_x;
  const int ty = (tile / p.tiles_x) % p.tiles_y;
  const int b = tile / (p.tiles_x * p.tiles_y);
  const int Y0 = ty * LCE_TILE, X0 = tx * LCE_TILE;
  const int Yl = min(Y0 + LCE_TILE - 1, p.H - 1), Xl = min(X0 + LCE_TILE - 1, p.W - 1);
  const float sy = static_cast<float>(p.h) / p.H, sx = static_cast<float>(p.w) / p.W;
  int by0, bh, bx0, bw;  // bh <= box_h, bw <= box_w by construction on the host
  src_span(Y0, Yl, sy, p.h, by0, bh);
  src_span(X0, Xl, sx, p.w, bx0, bw);
  const long long base = 1ll * b * p.h * p.w;
  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  // box load: one warp per cell, lanes = classes (no integer division in the loop)
  for (int cell = warp; cell < bh * bw; cell += 8) {
    const int r = cell / bw, c = cell - r * bw;
    slog[cell * LCE_SLD + lane] = (lane < n) ? p.logits[(base + 1ll * (by0 + r) * p.w + bx0 + c) * LP_LD + lane] : 0.f;
  }
  for (int idx = tid; idx < LCE_TILE * bwm; idx += 256) swx[idx] = 0.f;
  for (int idx = tid; idx < LCE_TILE * bhm; idx += 256) swy[idx] = 0.f;
  __syncthreads();
  // interpolation weights of the tile's rows / columns towards the box cells
  if (tid < LCE_TILE) {
    const int X = min(X0 + tid, p.W - 1);
    int x0, x1; float lx;
    src_index(X, sx, p.w, x0, x1, lx);
    swx[tid * bwm + (x0 - bx0)] += 1.f - lx;
    swx[tid * bwm + (x1 - bx0)] += lx;
  } else if (tid < 2 * LCE_TILE) {
    const int t = tid - LCE_TILE;
    const int Y = min(Y0 + t, p.H - 1);
    int y0, y1; float ly;
    src_index(Y, sy, p.h, y0, y1, ly);
    swy[t * bhm + (y0 - by0)] += 1.f - ly;
    swy[t * bhm + (y1 - by0)] += ly;
  }
  // ---- phase 0: interpolate the box along x once per tile column (shared by the 16 pixels of that column):
  //      sX[x][row][k] = (1 - lx) * L[row][x0][k] + lx * L[row][x1][k]; warps take columns, lanes = classes
  for (int xc = warp; xc < LCE_TILE; xc += 8) {
    int x0, x1; float lx;
    src_index(min(X0 + xc, p.W - 1), sx, p.w, x0, x1, lx);
    const float* c0 = slog + (x0 - bx0) * LCE_SLD + lane;
    const float* c1 = slog + (x1 - bx0) * LCE_SLD + lane;
    for (int row = 0; row < bh; ++row)
      sX[(xc * bhm + row) * LCE_SLD + lane] = (1.f - lx) * c0[row * bw * LCE_SLD] + lx * c1[row * bw * LCE_SLD];
  }
  __syncthreads();
  // ---- phase 1: thread = pixel
  const int py = tid / LCE_TILE, px = tid % LCE_TILE;
  const int Y = Y0 + py, X = X0 + px;
  const bool inb = (Y < p.H) && (X < p.W);
  const long long lab = inb ? read_label(p.label, p.label_bytes, (1ll * b * p.H + Y) * p.W + X) : -1;
  const bool valid = inb && lab >= 0 && lab < n;
  float lsum = 0.f, cnt = 0.f;
  {
    int y0, y1;
    float ly;
    src_index(min(Y, p.H - 1), sy, p.h, y0, y1, ly);
    const float wy0 = 1.f - ly;
    const float* r0 = sX + (px * bhm + (y0 - by0)) * LCE_SLD;
    const float* r1 = sX + (px * bhm + (y1 - by0)) * LCE_SLD;
    float z[LP_LD];
    float mx = -INFINITY;
#pragma unroll
    for (int k = 0; k < LP_LD; ++k) {
      if (k < n) {
        z[k] = fmaf(ly, r1[k], wy0 * r0[k]);
        mx = fmaxf(mx, z[k]);
      }
    }
    float se = 0.f;
#pragma unroll
    for (int k = 0; k < LP_LD; ++k)
      if (k < n) { z[k] = __expf(z[k] - mx); se += z[k]; }   // z now holds exp(z - max)  (ex2.approx: 2 ulp)
    const float inv = 1.0f / se;
    if (valid) {
      const int li = static_cast<int>(lab);
      const float zl = fmaf(ly, r1[li], wy0 * r0[li]);  // dynamic smem index
      lsum = __logf(se) - (zl - mx);  // lse - z_lab
      cnt = 1.f;
    }
    if (p.dlogits) {
      float* gp = sg + tid * n;
      if (valid) {
#pragma unroll
        for (int k = 0; k < LP_LD; ++k)
          if (k < n) gp[k] = z[k] * inv;
        gp[static_cast<int>(lab)] -= 1.f;
      } else {
#pragma unroll
        for (int k = 0; k < LP_LD; ++k)
          if (k < n) gp[k] = 0.f;
      }
    }
  }
  lsum = warp_sum(lsum);
  cnt = warp_sum(cnt);
  if (lane == 0) { sred[0][warp] = lsum; sred[1][warp] = cnt; }
  __syncthreads();
  if (tid == 0) {
    double a = 0, c = 0;
    for (int w = 0; w < 8; ++w) { a += sred[0][w]; c += sred[1][w]; }
    if (c > 0) { atomicAdd(p.acc, a); atomicAdd(p.acc + 1, c); }
  }
  if (!p.dlogits) return;
  // ---- phase 2a: reduce over the tile's columns.  pair = (box column, class); each thread keeps ONE pair for all
  //      the rows it handles, so the only integer division happens once per thread.
  const int pairs = bw * n;                 // <= 160 for the shipped shapes
  const int reps = max(1, 256 / pairs);     // row interleave factor
  const int pair = tid % pairs, rep = tid / pairs;
  const int pcx = pair / n, pk = pair - pcx * n;
  if (rep < reps) {
    for (int pr = pair; pr < pairs; pr += 256) {  // pairs > 256 only for very small upsampling ratios
      const int cx = (pr == pair) ? pcx : pr / n, k = (pr == pair) ? pk : pr % n;
      for (int yy = rep; yy < LCE_TILE; yy += reps) {
        float acc = 0.f;
#pragma unroll
        for (int xx = 0; xx < LCE_TILE; ++xx) acc = fmaf(swx[xx * bwm + cx], sg[(yy * LCE_TILE + xx) * n + k], acc);
        sT[(yy * bwm + cx) * n + k] = acc;
      }
    }
  }
  __syncthreads();
  // ---- phase 2b + 3: reduce over the rows, one atomic per (cell, class)
  for (int cy = rep; cy < bh; cy += reps) {
    if (rep >= reps) break;
    for (int pr = pair; pr < pairs; pr += 256) {
      const int cx = (pr == pair) ? pcx : pr / n, k = (pr == pair) ? pk : pr % n;
      float acc = 0.f;
#pragma unroll
      for (int yy = 0; yy < LCE_TILE; ++yy) acc = fmaf(swy[yy * bhm + cy], sT[(yy * bwm + cx) * n + k], acc);
      if (acc == 0.f) continue;
      const long long idx = (base + 1ll * (by0 + cy) * p.w + bx0 + cx) * LP_LD + k;
      if (kFixed) atomicAdd(p.dfix + idx, static_cast<unsigned long long>(__double2ll_rn(acc * LCE_FIX_SCALE)));
      else atomicAdd(p.dlogits + idx, acc);
    }
  }
}

// dlogits[i] = dfix[i] * 2^-40 (linear_ce_kernel<true>'s fixed-point gradient)
__global__ void fixed_to_float_kernel(const unsigned long long* __restrict__ dfix, float* __restrict__ out, long long n) {
  for (long long i = 1ll * blockIdx.x * blockDim.x + threadIdx.x; i < n; i += 1ll * gridDim.x * blockDim.x)
    out[i] = static_cast<float>(static_cast<double>(static_cast<long long>(dfix[i])) * (1.0 / LCE_FIX_SCALE));
}

// out[0] = loss_sum / count ; out[1] = count
__global__ void linear_ce_finish_kernel(const double* __restrict__ acc, float* __restrict__ out) {
  out[0] = static_cast<float>(acc[0] / acc[1]);
  out[1] = static_cast<float>(acc[1]);
}

// dW[k][c] += (gscale/count) * sum_r dlogits[r][k] code[r][c];  db[k] += (gscale/count) * sum_r dlogits[r][k]
// (count = 0 adds nothing: with every label ignored dlogits is all zero, and the reference's gradient is zero too)
// One CTA per 128-row chunk: both operand tiles are staged in shared memory, every thread owns ~8 of the
// n*C outputs and walks the 128 rows; one atomic per (CTA, output).
constexpr int LW_ROWS = 128;
__global__ void __launch_bounds__(256)
linear_wgrad_kernel(const float* __restrict__ dlogits, const float* __restrict__ code, long long ld_code, int C, int n,
                    long long rows, const float* __restrict__ loss_out, float gscale, float* __restrict__ dW,
                    float* __restrict__ db) {
  extern __shared__ float sm[];
  float* sdl = sm;                    // [128][32]
  float* scode = sm + LW_ROWS * 32;   // [128][C]
  const long long r0 = 1ll * blockIdx.x * LW_ROWS;
  const int nr = static_cast<int>((rows - r0 < LW_ROWS) ? rows - r0 : LW_ROWS);
  for (int i = threadIdx.x; i < LW_ROWS * 32; i += blockDim.x) {
    const int r = i >> 5;
    sdl[i] = (r < nr) ? dlogits[(r0 + r) * LP_LD + (i & 31)] : 0.f;
  }
  for (int i = threadIdx.x; i < LW_ROWS * C; i += blockDim.x) {
    const int r = i / C, c = i % C;
    scode[i] = (r < nr) ? code[(r0 + r) * ld_code + c] : 0.f;
  }
  __syncthreads();
  // no valid label pixel: the loss is NaN (0 / 0, as in the reference) but the gradient is zero, not 0 * inf
  const float cnt = loss_out[1];
  const float s = cnt > 0.f ? gscale / cnt : 0.f;
  for (int o = threadIdx.x; o < n * C; o += blockDim.x) {
    const int k = o / C, c = o % C;
    float acc = 0.f;
#pragma unroll 8
    for (int r = 0; r < LW_ROWS; ++r) acc = fmaf(sdl[r * 32 + k], scode[r * C + c], acc);
    atomicAdd(dW + o, acc * s);
  }
  if (threadIdx.x < n) {
    float acc = 0.f;
    for (int r = 0; r < LW_ROWS; ++r) acc += sdl[r * 32 + threadIdx.x];
    atomicAdd(db + threadIdx.x, acc * s);
  }
}

// ---------------------------------------------------------------------------------------------
// wide codes: the backbone's 384 / 768 channels (projection_type None, the DINO baseline)
// ---------------------------------------------------------------------------------------------
// The kernels above keep a pixel's channels in registers (<= 96).  At the backbone's widths the dots run as K tiles
// (wide_tile_dots), and every reduction over rows (dW, db, d clusters) is one CTA per output tile walking all rows in a
// fixed order: no atomics, so two identical steps are bit-identical.
static bool wide_dim(int C) { return C == 384 || C == 768; }

// logits[r][k] = bias[k] + code[r] . W[k]  (k < n <= 32; zeros up to LP_LD), as linear_logits_kernel
__global__ void __launch_bounds__(256, 2)
linear_logits_wide_kernel(const float* __restrict__ code, long long ld_code, int C, const float* __restrict__ W,
                          const float* __restrict__ bias, int n, float* __restrict__ logits, long long rows) {
  __shared__ __align__(16) float sX[PW_ROWS * PW_SX];
  __shared__ float sT[PW_KC * 64];
  const int o = threadIdx.x & 63, rg = threadIdx.x >> 6;
  for (long long r0 = 1ll * blockIdx.x * PW_ROWS; r0 < rows; r0 += 1ll * gridDim.x * PW_ROWS) {
    float acc[16], ss = 0.f;
    const float b0 = (o < n) ? bias[o] : 0.f;
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[i] = b0;
    wide_tile_dots<false>([&](long long r, int c) { return code[r * ld_code + c]; }, rows, r0, C,
                   [&](int c, int k) { return k < n ? W[1ll * k * C + c] : 0.f; }, sX, sT, acc, ss);
    if (o < LP_LD) {
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const long long r = r0 + rg * 16 + i;
        if (r < rows) logits[r * LP_LD + o] = acc[i];
      }
    }
  }
}

// ClusterLookup with alpha None on wide rows: ip[r][k] = <x_r / |x_r|, c_k / |c_k|>, assign[r] = first argmax,
// inv[r] = 1 / max(|x_r|, 1e-12), loss_partials[cta] = sum of the CTA's max ip (the loss is minus their mean)
__global__ void __launch_bounds__(256, 2)
cluster_wide_fwd_kernel(const float* __restrict__ x, long long ld, long long rows, int C,
                        const float* __restrict__ clusters, int n, int* __restrict__ assign, float* __restrict__ inv,
                        float* __restrict__ loss_partials) {
  __shared__ __align__(16) float sX[PW_ROWS * PW_SX];
  __shared__ float sT[PW_KC * 64];
  __shared__ float sD[PW_ROWS * 65];
  __shared__ float sinv[64], sss[PW_ROWS], sred[8];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int o = threadIdx.x & 63, rg = threadIdx.x >> 6;
  centroid_inv_norms(clusters, n, C, sinv);
  __syncthreads();
  float loss_acc = 0.f;
  for (long long r0 = 1ll * blockIdx.x * PW_ROWS; r0 < rows; r0 += 1ll * gridDim.x * PW_ROWS) {
    float acc[16], ss = 0.f;
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[i] = 0.f;
    wide_tile_dots<true>([&](long long r, int c) { return x[r * ld + c]; }, rows, r0, C,
                   [&](int c, int k) { return k < n ? clusters[1ll * k * C + c] * sinv[k] : 0.f; }, sX, sT, acc, ss);
#pragma unroll
    for (int i = 0; i < 16; ++i) sD[(rg * 16 + i) * 65 + o] = acc[i];
    if (threadIdx.x < PW_ROWS) sss[threadIdx.x] = ss;
    __syncthreads();
    for (int rr = warp; rr < PW_ROWS; rr += 8) {
      const long long r = r0 + rr;
      if (r >= rows) break;
      const float iv = 1.0f / fmaxf(sqrtf(sss[rr]), 1e-12f);
      const float ip0 = (lane < n) ? sD[rr * 65 + lane] * iv : -INFINITY;
      const float ip1 = (lane + 32 < n) ? sD[rr * 65 + lane + 32] * iv : -INFINITY;
      const float best = warp_max(fmaxf(ip0, ip1));
      const unsigned lo = __ballot_sync(0xffffffffu, ip0 == best), hi = __ballot_sync(0xffffffffu, ip1 == best);
      const int arg = lo ? __ffs(lo) - 1 : 32 + __ffs(hi) - 1;  // first maximum, like torch.argmax
      if (lane == 0) {
        loss_acc += best;
        assign[r] = arg;
        inv[r] = iv;
      }
    }
  }
  if (lane == 0) sred[warp] = loss_acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < 8; ++w) t += sred[w];
    loss_partials[blockIdx.x] = t;
  }
}

// out[k][c] += s * sum_r coef(r, k) x[r][c] for the CTA's 32 rows k = 32 blockIdx.y + kk (< n) and 4 channels
// c = 4 blockIdx.x + cc; the CTA with blockIdx.x == C / 4 takes the constant channel 1 instead and adds into
// out_sum[k].  coef: G[r][k] (row stride 32: the linear probe's dlogits) or, with assign, inv[r] where assign[r] == k (the
// one-hot gradient of ClusterLookup's alpha None loss).  s = scale / count[0] (0 when count[0] == 0: no valid label, a
// zero gradient) or, without count, scale.  Rows in a fixed order: thread row group rg takes rows rg, rg + 64, ... of
// each 256-row tile, and the 64 groups' sums are added in order at the end.  Narrow channel blocks give the
// C / 4 + 1 CTAs that keep the walk over every row short.
struct WideWgradParams {
  const float* x;
  long long ld, rows;
  int C, n;
  const float* G;
  const int* assign;
  const float* inv;
  const float* count;
  float scale;
  float* out;      // [n][C]
  float* out_sum;  // [n] or null
};

constexpr int PWG_ROWS = 256, PWG_C = 4, PWG_SG = 36;  // rows per tile, channels per CTA, sG row stride

__global__ void __launch_bounds__(256)
wide_wgrad_kernel(WideWgradParams p) {
  __shared__ __align__(16) float sG[PWG_ROWS * PWG_SG];
  __shared__ float sXc[PWG_ROWS * PWG_C];
  __shared__ float sRed[32 * PWG_C];
  const int cc = threadIdx.x & (PWG_C - 1), rg = threadIdx.x / PWG_C;  // channel of the CTA's 4, row group of 64
  const bool ones = blockIdx.x * PWG_C >= p.C;
  const int k0 = blockIdx.y * 32;
  float acc[32];
#pragma unroll
  for (int k = 0; k < 32; ++k) acc[k] = 0.f;
  for (long long r0 = 0; r0 < p.rows; r0 += PWG_ROWS) {
    // the tile's loads are all issued before the first shared store (a load per iteration would wait on each)
    float gv[PWG_ROWS * 32 / 256], xs[PWG_ROWS * PWG_C / 256];
#pragma unroll
    for (int j = 0; j < PWG_ROWS * 32 / 256; ++j) {
      const int i = threadIdx.x + 256 * j, rr = i >> 5, k = i & 31;
      const long long r = r0 + rr;
      gv[j] = 0.f;
      if (r < p.rows && k0 + k < p.n) {
        if (p.assign) gv[j] = (p.assign[r] == k0 + k) ? p.inv[r] : 0.f;
        else gv[j] = p.G[r * LP_LD + k0 + k];
      }
    }
#pragma unroll
    for (int j = 0; j < PWG_ROWS * PWG_C / 256; ++j) {
      const int i = threadIdx.x + 256 * j, rr = i / PWG_C, ci = i % PWG_C;
      const long long r = r0 + rr;
      xs[j] = 0.f;
      if (r < p.rows) xs[j] = ones ? (ci == 0 ? 1.f : 0.f) : p.x[r * p.ld + blockIdx.x * PWG_C + ci];
    }
    __syncthreads();  // the previous tile has been read
#pragma unroll
    for (int j = 0; j < PWG_ROWS * 32 / 256; ++j) {
      const int i = threadIdx.x + 256 * j;
      sG[(i >> 5) * PWG_SG + (i & 31)] = gv[j];
    }
#pragma unroll
    for (int j = 0; j < PWG_ROWS * PWG_C / 256; ++j) sXc[threadIdx.x + 256 * j] = xs[j];
    __syncthreads();
#pragma unroll
    for (int j = 0; j < PWG_ROWS / 64; ++j) {
      const int rr = rg + 64 * j;
      const float xv = sXc[rr * PWG_C + cc];
#pragma unroll
      for (int k = 0; k < 32; k += 4) {
        const float4 g = *reinterpret_cast<const float4*>(&sG[rr * PWG_SG + k]);
        acc[k] = fmaf(g.x, xv, acc[k]);
        acc[k + 1] = fmaf(g.y, xv, acc[k + 1]);
        acc[k + 2] = fmaf(g.z, xv, acc[k + 2]);
        acc[k + 3] = fmaf(g.w, xv, acc[k + 3]);
      }
    }
  }
  for (int g = 0; g < 64; ++g) {  // the row groups' partial sums, in order
    __syncthreads();
    if (rg == g)
#pragma unroll
      for (int k = 0; k < 32; ++k) sRed[k * PWG_C + cc] = (g == 0) ? acc[k] : sRed[k * PWG_C + cc] + acc[k];
  }
  __syncthreads();
  float s = p.scale;
  if (p.count) s = p.count[0] > 0.f ? p.scale / p.count[0] : 0.f;
  if (threadIdx.x < 32 * PWG_C) {
    const int k = threadIdx.x / PWG_C, ci = threadIdx.x % PWG_C;
    if (k0 + k < p.n) {
      if (!ones) p.out[1ll * (k0 + k) * p.C + blockIdx.x * PWG_C + ci] += s * sRed[threadIdx.x];
      else if (ci == 0 && p.out_sum) p.out_sum[k0 + k] += s * sRed[threadIdx.x];
    }
  }
}

static int launch_wide_wgrad(const WideWgradParams& p, cudaStream_t stream) {
  const dim3 grid(p.C / PWG_C + (p.out_sum ? 1 : 0), (p.n + 31) / 32);
  wide_wgrad_kernel<<<grid, 256, 0, stream>>>(p);
  STEGO_CHECK_LAUNCH("wide_wgrad_kernel");
  return STEGO_OK;
}

static unsigned wide_row_grid(long long rows) {
  const long long tiles = (rows + PW_ROWS - 1) / PW_ROWS;
  const long long cap = 2ll * num_sms();
  return (unsigned)(tiles < cap ? tiles : cap);
}

}  // namespace stego

using namespace stego;

static int fill_cluster(ClusterParams& p, const float* x, long long sb, long long sc, long long sp,
                        const float* clusters, int B, int C, int n, long long npix, int use_alpha, float alpha) {
  STEGO_CHECK_ARG(x && clusters && B > 0 && npix > 0, "cluster_lookup: bad args");
  STEGO_CHECK_ARG(C > 0 && C <= PR_MAX_DIM, "cluster_lookup: dim %d unsupported (<= %d)", C, PR_MAX_DIM);
  STEGO_CHECK_ARG(n > 0 && n <= PR_MAX_CLASSES, "cluster_lookup: n_classes %d unsupported (<= %d)", n, PR_MAX_CLASSES);
  p.x = x; p.sb = sb; p.sc = sc; p.sp = sp; p.clusters = clusters;
  p.B = B; p.C = C; p.n = n; p.npix = npix; p.mode = use_alpha ? 1 : 0; p.alpha = alpha;
  p.assign = nullptr; p.probs = nullptr; p.logp = nullptr; p.loss_partials = nullptr; p.grad_loss = nullptr;
  p.grad_scale = 0.f; p.dnc = nullptr;
  return STEGO_OK;
}

static int cluster_grid(long long total) {
  long long g = (total + PR_THREADS - 1) / PR_THREADS;
  const long long cap = 8ll * num_sms();
  return (int)(g < cap ? g : cap);
}

// x: features with element strides (batch, channel, pixel); pixel index = y*W + x must be a single stride.
// loss_out[0] = -(sum_k probs_k ip_k).mean(); scratch: at least 16*SMs floats.
extern "C" int stego_cluster_lookup_fwd(const float* x, long long stride_b, long long stride_c, long long stride_pix,
                                        const float* clusters, int B, int C, int n_classes, long long npix,
                                        int use_alpha, float alpha, long long* assign, float* probs, float* log_probs,
                                        float* loss_out, float* scratch, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ClusterParams p;
  int rc = fill_cluster(p, x, stride_b, stride_c, stride_pix, clusters, B, C, n_classes, npix, use_alpha, alpha);
  if (rc != STEGO_OK) return rc;
  STEGO_CHECK_ARG(loss_out && scratch, "stego_cluster_lookup_fwd: null loss_out/scratch");
  STEGO_CHECK_ARG(!log_probs || use_alpha, "stego_cluster_lookup_fwd: log_probs needs alpha");
  p.assign = assign; p.probs = probs; p.logp = log_probs; p.loss_partials = scratch;
  const long long total = 1ll * B * npix;
  int grid;
  if (stride_c == 1 && n_classes <= 32) {
    long long g = (total + 7) / 8;
    const long long cap = 16ll * num_sms();  // (2 CTAs/SM measured slower: 51 vs 47 us — the pixel loop needs the parallelism)
    grid = (int)(g < cap ? g : cap);
    cluster_lookup_cl_kernel<false><<<grid, 256, (size_t)C * 32 * sizeof(float), stream>>>(p);
    STEGO_CHECK_LAUNCH("cluster_lookup_cl_kernel<fwd>");
  } else {
    grid = cluster_grid(total);
    const size_t smem = (size_t)(n_classes * C + 8) * sizeof(float);
    cluster_lookup_kernel<false><<<grid, PR_THREADS, smem, stream>>>(p);
    STEGO_CHECK_LAUNCH("cluster_lookup_kernel<fwd>");
  }
  sum_partials_kernel<<<1, 256, 0, stream>>>(scratch, grid, (float)(-1.0 / (double)total), loss_out);
  STEGO_CHECK_LAUNCH("sum_partials_kernel");
  return STEGO_OK;
}

// dclusters [n][C] += grad_loss_dev[0] * d(loss)/d(clusters) (upstream scalar read on the device: no host sync). dnc_scratch: [n][C] floats, zeroed by the caller.
extern "C" int stego_cluster_lookup_bwd(const float* x, long long stride_b, long long stride_c, long long stride_pix,
                                        const float* clusters, int B, int C, int n_classes, long long npix,
                                        int use_alpha, float alpha, const float* grad_loss_dev,
                                        float* dnc_scratch, float* dclusters, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ClusterParams p;
  int rc = fill_cluster(p, x, stride_b, stride_c, stride_pix, clusters, B, C, n_classes, npix, use_alpha, alpha);
  if (rc != STEGO_OK) return rc;
  STEGO_CHECK_ARG(dnc_scratch && dclusters && grad_loss_dev, "stego_cluster_lookup_bwd: null pointer");
  const long long total = 1ll * B * npix;
  p.grad_scale = (float)(-1.0 / (double)total);
  p.grad_loss = grad_loss_dev;
  p.dnc = dnc_scratch;
  if (stride_c == 1 && n_classes <= 32 && !use_alpha) {
    long long g = (total + 7) / 8;
    const long long cap = 4ll * num_sms();
    const int grid = (int)(g < cap ? g : cap);
    cluster_lookup_cl_kernel<true><<<grid, 256, (size_t)(C * 32 + n_classes * C) * sizeof(float), stream>>>(p);
    STEGO_CHECK_LAUNCH("cluster_lookup_cl_kernel<bwd>");
  } else {
    const int grid = cluster_grid(total);
    const size_t smem = (size_t)(2 * n_classes * C + 8) * sizeof(float);  // 48 KB and more from n * C > 6140
    if ((rc = opt_in_smem<cluster_lookup_kernel<true>>(smem, "cluster_lookup_kernel<bwd>")) != STEGO_OK) return rc;
    cluster_lookup_kernel<true><<<grid, PR_THREADS, smem, stream>>>(p);
    STEGO_CHECK_LAUNCH("cluster_lookup_kernel<bwd>");
  }
  cluster_norm_bwd_kernel<<<n_classes, 32, 0, stream>>>(clusters, dnc_scratch, dclusters, n_classes, C);
  STEGO_CHECK_LAUNCH("cluster_norm_bwd_kernel");
  return STEGO_OK;
}

// Linear probe + bilinear upsample + masked cross entropy, forward and (optionally) backward in one call.
//   code [B*h*w][ld_code] fp32 tokens-major (detached), W [n][C], bias [n], label [B][H][W] int64 / int32 / uint8
//   (label_bytes = 8 / 4 / 1; a label outside [0, n) is ignored: -1 for the signed types, 255 for uint8)
//   loss_out[0] = CE mean over valid pixels, loss_out[1] = number of valid pixels
//   logits_scratch / dlogits_scratch: [B*h*w][32] floats (dlogits zeroed by the caller; null = forward only)
//   dW / db: accumulated (+=) with grad_loss * d(loss)/d(.)
// The linear probe step of stego_linear_probe_ce (C <= 96; dfix null) and stego_linear_probe_ce_wide (C = 384 / 768;
// the gradient accumulated in the int64 fixed point of dfix, so that dW / db are the same bit for bit run to run)
static int linear_probe_ce(const char* who, const float* code, long long ld_code, int C, const float* W,
                           const float* bias, int n_classes, const void* label, int label_bytes, int B, int h, int w,
                           int H, int Wimg, float* logits_scratch, float* dlogits_scratch,
                           unsigned long long* dfix_scratch, float* partials_scratch, float* loss_out, float grad_loss,
                           float* dW, float* db, cudaStream_t stream) {
  const bool wide = wide_dim(C);
  STEGO_CHECK_ARG(code && W && bias && label && logits_scratch && partials_scratch && loss_out, "%s: null pointer", who);
  STEGO_CHECK_ARG(n_classes > 0 && n_classes <= LP_LD, "%s: C=%d n=%d unsupported (n <= %d)", who, C, n_classes, LP_LD);
  STEGO_CHECK_ARG(label_bytes == 8 || label_bytes == 4 || label_bytes == 1, "%s: label_bytes=%d (8, 4 or 1)", who,
                  label_bytes);
  STEGO_CHECK_ARG(!dlogits_scratch || (dW && db), "%s: backward needs dW and db", who);
  STEGO_CHECK_ARG(!wide || !dlogits_scratch || dfix_scratch, "%s: the backward needs dfix_scratch", who);
  const long long rows = 1ll * B * h * w;
  if (wide) {
    linear_logits_wide_kernel<<<wide_row_grid(rows), 256, 0, stream>>>(code, ld_code, C, W, bias, n_classes,
                                                                       logits_scratch, rows);
    STEGO_CHECK_LAUNCH("linear_logits_wide_kernel");
  } else {
    long long g = (rows + 7) / 8;
    const long long capg = 16ll * num_sms();
    linear_logits_kernel<<<(unsigned)(g < capg ? g : capg), 256, (size_t)C * 32 * sizeof(float), stream>>>(
        code, ld_code, C, W, bias, n_classes, logits_scratch, rows);
    STEGO_CHECK_LAUNCH("linear_logits_kernel");
  }
  LinearCEParams p;
  p.logits = logits_scratch; p.label = label; p.label_bytes = label_bytes; p.B = B; p.h = h; p.w = w; p.H = H; p.W = Wimg; p.n = n_classes;
  p.dlogits = dlogits_scratch;
  p.dfix = wide ? dfix_scratch : nullptr;
  STEGO_CHECK_ARG((reinterpret_cast<uintptr_t>(partials_scratch) & 7u) == 0, "%s: scratch not 8-byte aligned", who);
  p.acc = reinterpret_cast<double*>(partials_scratch);
  p.tiles_y = (H + LCE_TILE - 1) / LCE_TILE;
  p.tiles_x = (Wimg + LCE_TILE - 1) / LCE_TILE;
  p.box_h = src_span_max(LCE_TILE, h, H);
  p.box_w = src_span_max(LCE_TILE, w, Wimg);
  const size_t region = std::max((size_t)LCE_TILE * p.box_w * n_classes, (size_t)LCE_TILE * p.box_h * LCE_SLD);
  const size_t ce_smem = ((size_t)p.box_h * p.box_w * LCE_SLD + 256 * (size_t)n_classes + region +
                          (size_t)LCE_TILE * (p.box_w + p.box_h)) * sizeof(float);
  STEGO_CHECK_ARG(ce_smem <= 200 * 1024, "%s: upsample ratio %dx%d -> %dx%d needs %zu B of smem", who, h, w, H, Wimg, ce_smem);
  int rc = wide ? opt_in_smem<linear_ce_kernel<true>>(ce_smem, "linear_ce_kernel")
                : opt_in_smem<linear_ce_kernel<false>>(ce_smem, "linear_ce_kernel");
  if (rc != STEGO_OK) return rc;
  {
    cudaError_t e = cudaMemsetAsync(partials_scratch, 0, 2 * sizeof(double), stream);
    if (e != cudaSuccess) return cuda_fail(e, "cudaMemsetAsync(linear_ce acc)");
  }
  const int grid = B * p.tiles_y * p.tiles_x;
  if (wide && dlogits_scratch) linear_ce_kernel<true><<<grid, 256, ce_smem, stream>>>(p);
  else linear_ce_kernel<false><<<grid, 256, ce_smem, stream>>>(p);
  STEGO_CHECK_LAUNCH("linear_ce_kernel");
  linear_ce_finish_kernel<<<1, 1, 0, stream>>>(p.acc, loss_out);
  STEGO_CHECK_LAUNCH("linear_ce_finish_kernel");
  if (dlogits_scratch && wide) {
    const long long n = rows * LP_LD;
    const long long cap = 8ll * num_sms();
    const long long g = (n + 255) / 256;
    fixed_to_float_kernel<<<(unsigned)(g < cap ? g : cap), 256, 0, stream>>>(dfix_scratch, dlogits_scratch, n);
    STEGO_CHECK_LAUNCH("fixed_to_float_kernel");
    WideWgradParams wg{code, ld_code, rows, C, n_classes, dlogits_scratch, nullptr, nullptr, loss_out + 1, grad_loss, dW, db};
    return launch_wide_wgrad(wg, stream);
  }
  if (dlogits_scratch) {
    const unsigned blocks = (unsigned)((rows + LW_ROWS - 1) / LW_ROWS);
    const size_t wsmem = (size_t)(LW_ROWS * 32 + LW_ROWS * C) * sizeof(float);
    if ((rc = opt_in_smem<linear_wgrad_kernel>(wsmem, "linear_wgrad_kernel")) != STEGO_OK) return rc;
    linear_wgrad_kernel<<<blocks, 256, wsmem, stream>>>(dlogits_scratch, code, ld_code, C, n_classes, rows, loss_out,
                                                        grad_loss, dW, db);
    STEGO_CHECK_LAUNCH("linear_wgrad_kernel");
  }
  return STEGO_OK;
}

extern "C" int stego_linear_probe_ce(const float* code, long long ld_code, int C, const float* W, const float* bias,
                                     int n_classes, const void* label, int label_bytes, int B, int h, int w, int H,
                                     int Wimg, float* logits_scratch, float* dlogits_scratch, float* partials_scratch,
                                     float* loss_out, float grad_loss, float* dW, float* db, void* stream_) {
  STEGO_CHECK_ARG(C > 0 && C <= PR_MAX_DIM && n_classes > 0 && n_classes <= LP_LD,
                  "stego_linear_probe_ce: C=%d n=%d unsupported", C, n_classes);
  return linear_probe_ce("stego_linear_probe_ce", code, ld_code, C, W, bias, n_classes, label, label_bytes, B, h, w, H,
                         Wimg, logits_scratch, dlogits_scratch, nullptr, partials_scratch, loss_out, grad_loss, dW, db,
                         reinterpret_cast<cudaStream_t>(stream_));
}

// stego_linear_probe_ce for a wide code (C = 384 / 768: projection_type None); dfix_scratch: int64 [B*h*w][32], zeroed by
// the caller, needed with dlogits_scratch.  Every reduction has a fixed order or is exact: bit-identical run to run.
extern "C" int stego_linear_probe_ce_wide(const float* code, long long ld_code, int C, const float* W, const float* bias,
                                          int n_classes, const void* label, int label_bytes, int B, int h, int w, int H,
                                          int Wimg, float* logits_scratch, float* dlogits_scratch, long long* dfix_scratch,
                                          float* partials_scratch, float* loss_out, float grad_loss, float* dW, float* db,
                                          void* stream_) {
  STEGO_CHECK_ARG(wide_dim(C), "stego_linear_probe_ce_wide: C=%d unsupported (384 or 768)", C);
  return linear_probe_ce("stego_linear_probe_ce_wide", code, ld_code, C, W, bias, n_classes, label, label_bytes, B, h, w,
                         H, Wimg, logits_scratch, dlogits_scratch, reinterpret_cast<unsigned long long*>(dfix_scratch),
                         partials_scratch, loss_out, grad_loss, dW, db, reinterpret_cast<cudaStream_t>(stream_));
}

// ClusterLookup's alpha None loss (the training step's cluster probe, train_segmentation.py:221-223) and, optionally,
// its gradient in one call for a wide code (C = 384 or 768: projection_type None).  x [rows][ld_x] fp32 tokens-major;
// clusters [n][C], n <= 64.  loss_out[0] = -mean_r max_k <x_r / |x_r|, c_k / |c_k|>.  Scratch: assign_scratch int32 and
// inv_scratch fp32, [rows] each; partials_scratch: 16 * SMs floats.  With dclusters: dclusters [n][C] += d loss_out[0] /
// d clusters, through dnc_scratch [n][C] (zeroed by the caller).  Deterministic: no atomics.
extern "C" int stego_cluster_lookup_wide(const float* x, long long ld_x, long long rows, int C, const float* clusters,
                                         int n_classes, int* assign_scratch, float* inv_scratch,
                                         float* partials_scratch, float* loss_out, float* dnc_scratch,
                                         float* dclusters, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(x && clusters && assign_scratch && inv_scratch && partials_scratch && loss_out && rows > 0,
                  "stego_cluster_lookup_wide: bad args");
  STEGO_CHECK_ARG(wide_dim(C) && ld_x >= C, "stego_cluster_lookup_wide: C=%d (384 or 768), ld_x=%lld", C, ld_x);
  STEGO_CHECK_ARG(n_classes > 0 && n_classes <= PR_MAX_CLASSES, "stego_cluster_lookup_wide: n_classes %d unsupported (<= %d)",
                  n_classes, PR_MAX_CLASSES);
  STEGO_CHECK_ARG(!dclusters || dnc_scratch, "stego_cluster_lookup_wide: the gradient needs dnc_scratch");
  const unsigned grid = wide_row_grid(rows);
  cluster_wide_fwd_kernel<<<grid, 256, 0, stream>>>(x, ld_x, rows, C, clusters, n_classes, assign_scratch, inv_scratch,
                                                    partials_scratch);
  STEGO_CHECK_LAUNCH("cluster_wide_fwd_kernel");
  sum_partials_kernel<<<1, 256, 0, stream>>>(partials_scratch, (int)grid, (float)(-1.0 / (double)rows), loss_out);
  STEGO_CHECK_LAUNCH("sum_partials_kernel");
  if (!dclusters) return STEGO_OK;
  WideWgradParams g{x, ld_x, rows, C, n_classes, nullptr, assign_scratch, inv_scratch, nullptr,
                    (float)(-1.0 / (double)rows), dnc_scratch, nullptr};
  int rc;
  if ((rc = launch_wide_wgrad(g, stream)) != STEGO_OK) return rc;
  cluster_norm_bwd_kernel<<<n_classes, 32, 0, stream>>>(clusters, dnc_scratch, dclusters, n_classes, C);
  STEGO_CHECK_LAUNCH("cluster_norm_bwd_kernel");
  return STEGO_OK;
}
