// Fused evaluation probes (BASELINE.json configs[4]: 1024 x 2048 frames): the reference's eval loop
// (src/eval_segmentation.py:128-131) does
//     code = F.interpolate(code, label.shape[-2:], mode='bilinear', align_corners=False)   # [B,70,H,W]: 587 MB/img
//     linear_probs  = torch.log_softmax(model.linear_probe(code), dim=1)                   # [B,27,H,W]
//     cluster_probs = model.cluster_probe(code, 2, log_probs=True)                          # [B,27,H,W]
// Here the upsampled code is never materialised.  Both probes are evaluated per output pixel from a few
// low-resolution quantities, using the linearity of bilinear interpolation:
//   * linear probe:  conv1x1(interp(code)) == interp(conv1x1(code))  -> interpolate the 27 low-res logits;
//   * cluster probe: <interp(code), c_k> == interp(<code, c_k>)      -> interpolate the low-res dot products with the
//     normalised centroids; ||interp(code)||^2 = sum_{t,t'} w_t w_t' <code_t, code_t'> needs only the Gram
//     entries between neighbouring low-res pixels (self, right, down, down-right, down-left).  Those entries and their
//     combination are fp64: where neighbouring codes nearly cancel (a class edge where the code flips direction) the
//     norm is a small difference of large terms, and in fp32 its error would grow with the square of
//     sum_t w_t |code_t| / ||interp(code)|| instead of linearly, as it does when the code is upsampled first.
// Two kernels: a per-low-res-pixel preparation (warp per pixel) and the per-output-pixel evaluation, which is
// bound by writing the two [B,n,H,W] fp32 log-probability maps (HBM): 453 MB per 1024x2048 image.
// Also fused here (src/eval_segmentation.py:124-126, 138-139; src/utils.py:219-229):
//   * flip test-time augmentation  code = (code(img) + code(img.flip(3)).flip(3)) / 2  — averaged on the low-res code
//     inside the preparation kernel (interpolation is linear, and the reference averages before it as well);
//   * UnsupervisedMetrics.update for both probes: the [pred][actual] confusion counts are accumulated per CTA in shared
//     memory from the argmax the kernel already has, one 64-bit atomic per non-zero cell per CTA.
#include "host_util.h"
#include "probe_common.cuh"

namespace stego {

constexpr int EV_LD = 80;  // floats per low-res pixel: [0,32) linear logits, [32,64) centroid dots, [64,74) Gram entries
constexpr int EV_G = 64;   // the five fp64 Gram entries (self, right, down, down-right, down-left) start at this float
constexpr int EV_SS = 0, EV_R = 1, EV_D = 2, EV_DR = 3, EV_DL = 4;  // their index among those doubles

__device__ __forceinline__ double warp_sum_f64(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ const double* ev_grams(const float* cell) {
  return reinterpret_cast<const double*>(cell + EV_G);
}

struct EvalPrepParams {
  const float* code;   // [B*h*w][ld] tokens-major
  const float* code_flip;  // code of the horizontally flipped image (same layout) or null: flip-TTA average
  long long ld;
  int B, h, w, C;
  const float* W;      // [n_lin][C]
  const float* bias;   // [n_lin]
  int n_lin;
  const float* clusters;  // [n_clu][C]
  int n_clu;
  float* lr;           // [B*h*w][EV_LD]
};

// one warp per low-res pixel; lanes = classes for the dot products, lanes = channels for the Gram entries
__global__ void __launch_bounds__(256)
eval_prep_kernel(EvalPrepParams p) {
  extern __shared__ float sm[];
  float* swT = sm;                 // [C][32] linear weights transposed
  float* scT = sm + p.C * 32;      // [C][32] normalised centroids transposed
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < p.C * 32; i += blockDim.x) {
    const int c = i >> 5, k = i & 31;
    swT[i] = (k < p.n_lin) ? p.W[k * p.C + c] : 0.f;
    scT[i] = 0.f;
  }
  __syncthreads();
  normalize_centroids(p.clusters, p.n_clu, p.C, 8, scT, 1, 32);
  __syncthreads();
  const float bk = (lane < p.n_lin) ? p.bias[lane] : 0.f;
  const long long rows = 1ll * p.B * p.h * p.w;
  for (long long r = 1ll * blockIdx.x * 8 + warp; r < rows; r += 1ll * gridDim.x * 8) {
    const int x = static_cast<int>(r % p.w);
    const int y = static_cast<int>((r / p.w) % p.h);
    const float* cp = p.code + r * p.ld;
    // flipped image: its column w-1-x holds this pixel; moving right here is moving left there
    const float* fp = p.code_flip ? p.code_flip + (r - x + (p.w - 1 - x)) * p.ld : nullptr;
    float xr[3], nr[3], nd[3], ndr[3], ndl[3];
    const bool hr = x + 1 < p.w, hd = y + 1 < p.h, hl = x > 0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const int c = lane + 32 * k;
      const bool ok = c < p.C;
      xr[k] = ok ? cp[c] : 0.f;
      nr[k] = (ok && hr) ? cp[p.ld + c] : 0.f;
      nd[k] = (ok && hd) ? cp[p.w * p.ld + c] : 0.f;
      ndr[k] = (ok && hd && hr) ? cp[(p.w + 1) * p.ld + c] : 0.f;
      ndl[k] = (ok && hd && hl) ? cp[(p.w - 1) * p.ld + c] : 0.f;
      if (fp) {
        xr[k] = 0.5f * (xr[k] + (ok ? fp[c] : 0.f));
        nr[k] = 0.5f * (nr[k] + ((ok && hr) ? fp[c - p.ld] : 0.f));
        nd[k] = 0.5f * (nd[k] + ((ok && hd) ? fp[p.w * p.ld + c] : 0.f));
        ndr[k] = 0.5f * (ndr[k] + ((ok && hd && hr) ? fp[(p.w - 1) * p.ld + c] : 0.f));
        ndl[k] = 0.5f * (ndl[k] + ((ok && hd && hl) ? fp[(p.w + 1) * p.ld + c] : 0.f));
      }
    }
    double g0 = 0.0, g1 = 0.0, g2 = 0.0, g3 = 0.0, g4 = 0.0;  // products of fp32 values are exact in fp64
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const double x = xr[k];
      g0 = fma(x, x, g0);
      g1 = fma(x, (double)nr[k], g1);
      g2 = fma(x, (double)nd[k], g2);
      g3 = fma(x, (double)ndr[k], g3);
      g4 = fma(x, (double)ndl[k], g4);
    }
    g0 = warp_sum_f64(g0); g1 = warp_sum_f64(g1); g2 = warp_sum_f64(g2); g3 = warp_sum_f64(g3); g4 = warp_sum_f64(g4);
    float dl = bk, dc = 0.f;
    for_each_channel(xr, p.C, [&](int c, float xc) {
      dl = fmaf(xc, swT[c * 32 + lane], dl);
      dc = fmaf(xc, scT[c * 32 + lane], dc);
    });
    float* o = p.lr + r * EV_LD;
    o[lane] = dl;
    o[32 + lane] = dc;
    if (lane == 0) {
      double* og = reinterpret_cast<double*>(o + EV_G);
      og[EV_SS] = g0; og[EV_R] = g1; og[EV_D] = g2; og[EV_DR] = g3; og[EV_DL] = g4;
    }
  }
}

struct EvalProbeParams {
  const float* lr;   // [B*h*w][EV_LD]
  int B, h, w, H, W, n_lin, n_clu;
  float alpha;
  float* lin_logp;   // [B][n_lin][H][W] or null
  float* clu_logp;   // [B][n_clu][H][W] or null
  unsigned char* lin_arg;  // [B][H][W] or null
  unsigned char* clu_arg;  // [B][H][W] or null
  int box_h, box_w;
  const void* label;       // [B][H][W] int64 / int32 / uint8 (label_bytes 8 / 4 / 1) or null
  int label_bytes;
  int n_cls;               // label classes: a pixel counts when 0 <= label < n_cls and pred < n_cls (utils.py:222)
  unsigned long long* lin_conf;  // [n_lin][n_cls] += counts of (pred, actual), or null
  unsigned long long* clu_conf;  // [n_clu][n_cls]
};

// Output tile of a CTA: 64 x 4 pixels, thread = pixel, x fastest (coalesced plane writes).  (Measured and rejected in
// round 2: 64 x 16 tiles in four passes under a 120-register cap, two CTAs per SM: 1.35 ms instead of 1.00 ms per 4 frames.)
constexpr int EVT_W = 64, EVT_H = 4;

// Gram entry <code_p, code_q> (fp64) for box-relative low-res pixels p, q that are equal or 8-neighbours
__device__ __forceinline__ double ev_gram(const float* slr, int bw, int py, int px, int qy, int qx) {
  int dy = qy - py, dx = qx - px;
  if (dy < 0 || (dy == 0 && dx < 0)) {  // look the pair up from the upper / left pixel
    const int ty = py, tx = px;
    py = qy; px = qx; qy = ty; qx = tx;
    dy = -dy; dx = -dx;
  }
  const double* e = ev_grams(slr + (py * bw + px) * EV_LD);
  if (dy == 0) return dx == 0 ? e[EV_SS] : e[EV_R];
  return dx == 0 ? e[EV_D] : (dx > 0 ? e[EV_DR] : e[EV_DL]);
}

// The output tile of CTA blockIdx.x (tile_w x tile_h pixels of image b, tiles row-major per image) and the low-res
// box [by0, by0 + bh) x [bx0, bx0 + bw) its pixels interpolate from, copied from the preparation table lr into
// shared memory slr [bh*bw][EV_LD].  Shared by eval_probe_kernel and eval_crf_unary_kernel; the caller synchronises.
struct EvTile {
  int b, X0, Y0, by0, bh, bx0, bw;
  float sy, sx;
};

__device__ __forceinline__ EvTile ev_tile_load(const float* lr, float* slr, int h, int w, int H, int W, int tile_w,
                                               int tile_h) {
  EvTile t;
  const int tiles_x = (W + tile_w - 1) / tile_w, tiles_y = (H + tile_h - 1) / tile_h;
  const int tile = blockIdx.x;
  const int tx = tile % tiles_x, ty = (tile / tiles_x) % tiles_y;
  t.b = tile / (tiles_x * tiles_y);
  t.X0 = tx * tile_w;
  t.Y0 = ty * tile_h;
  const int Xl = min(t.X0 + tile_w - 1, W - 1), Yl = min(t.Y0 + tile_h - 1, H - 1);
  t.sy = static_cast<float>(h) / H;
  t.sx = static_cast<float>(w) / W;
  src_span(t.Y0, Yl, t.sy, h, t.by0, t.bh);
  src_span(t.X0, Xl, t.sx, w, t.bx0, t.bw);
  const long long base = 1ll * t.b * h * w;
  for (int i = threadIdx.x; i < t.bh * t.bw * EV_LD; i += blockDim.x) {
    const int cell = i / EV_LD, k = i % EV_LD;
    const int r = cell / t.bw, c = cell % t.bw;
    slr[i] = lr[(base + 1ll * (t.by0 + r) * w + t.bx0 + c) * EV_LD + k];
  }
  return t;
}

// The four box-relative corners of output pixel (Y, X) and their bilinear weights
struct EvCorners {
  const float *ea, *eb, *ec, *ed;
  float wa, wb, wc, wd;
  int y0, y1, x0, x1;
};

__device__ __forceinline__ EvCorners ev_corners(const float* slr, const EvTile& t, int h, int w, int Y, int X) {
  EvCorners e;
  float ly, lx;
  src_index(Y, t.sy, h, e.y0, e.y1, ly);
  src_index(X, t.sx, w, e.x0, e.x1, lx);
  e.y0 -= t.by0; e.y1 -= t.by0; e.x0 -= t.bx0; e.x1 -= t.bx0;
  e.wa = (1.f - ly) * (1.f - lx); e.wb = (1.f - ly) * lx; e.wc = ly * (1.f - lx); e.wd = ly * lx;
  e.ea = slr + (e.y0 * t.bw + e.x0) * EV_LD;
  e.eb = slr + (e.y0 * t.bw + e.x1) * EV_LD;
  e.ec = slr + (e.y1 * t.bw + e.x0) * EV_LD;
  e.ed = slr + (e.y1 * t.bw + e.x1) * EV_LD;
  return e;
}

// Linear probe: the interpolated logits z[k < n], their maximum and first argmax
__device__ __forceinline__ void ev_linear(const EvCorners& e, int n, float (&z)[32], float& mx, int& arg) {
  mx = -INFINITY;
  arg = 0;
#pragma unroll
  for (int k = 0; k < 32; ++k) {
    if (k < n) {
      z[k] = e.wa * e.ea[k] + e.wb * e.eb[k] + e.wc * e.ec[k] + e.wd * e.ed[k];
      if (z[k] > mx) { mx = z[k]; arg = k; }
    }
  }
}

// Cluster probe: cosine similarities z[k < n] of the interpolated code with the normalised centroids, their maximum and
// first argmax.  The squared norm of the interpolated code comes from the fp32 weights and the fp64 Gram entries,
// combined in fp64 (their products are exact there).
__device__ __forceinline__ void ev_cluster(const float* slr, int bw, const EvCorners& e, int n, float (&z)[32],
                                           float& mx, int& arg) {
  const double da = e.wa, db = e.wb, dc = e.wc, dd = e.wd;
  double n2 = da * da * ev_grams(e.ea)[EV_SS] + db * db * ev_grams(e.eb)[EV_SS] + dc * dc * ev_grams(e.ec)[EV_SS] +
              dd * dd * ev_grams(e.ed)[EV_SS];
  n2 += 2.0 * (da * db * ev_gram(slr, bw, e.y0, e.x0, e.y0, e.x1) + da * dc * ev_gram(slr, bw, e.y0, e.x0, e.y1, e.x0) +
               da * dd * ev_gram(slr, bw, e.y0, e.x0, e.y1, e.x1) + db * dc * ev_gram(slr, bw, e.y0, e.x1, e.y1, e.x0) +
               db * dd * ev_gram(slr, bw, e.y0, e.x1, e.y1, e.x1) + dc * dd * ev_gram(slr, bw, e.y1, e.x0, e.y1, e.x1));
  const float inv = 1.0f / fmaxf(sqrtf(fmaxf(static_cast<float>(n2), 0.f)), 1e-12f);
  mx = -INFINITY;
  arg = 0;
#pragma unroll
  for (int k = 0; k < 32; ++k) {
    if (k < n) {
      z[k] = (e.wa * e.ea[32 + k] + e.wb * e.eb[32 + k] + e.wc * e.ec[32 + k] + e.wd * e.ed[32 + k]) * inv;
      if (z[k] > mx) { mx = z[k]; arg = k; }
    }
  }
}

__global__ void __launch_bounds__(EVT_W* EVT_H)
eval_probe_kernel(EvalProbeParams p) {
  extern __shared__ float slr[];  // [box_h*box_w][EV_LD]
  __shared__ ConfHist hist;
  const bool want_conf = p.label != nullptr;
  if (want_conf)
    for (int i = threadIdx.x; i < 2 * 32 * 32; i += blockDim.x) (&hist[0][0])[i] = 0u;
  const EvTile t = ev_tile_load(p.lr, slr, p.h, p.w, p.H, p.W, EVT_W, EVT_H);
  const int b = t.b;
  __syncthreads();
  const int X = t.X0 + (threadIdx.x % EVT_W), Y = t.Y0 + (threadIdx.x / EVT_W);
  const bool active = X < p.W && Y < p.H;
  int lin_pred = -1, clu_pred = -1;
  if (active) {
    const EvCorners e = ev_corners(slr, t, p.h, p.w, Y, X);
    const long long plane = 1ll * p.H * p.W;
    const long long pix = 1ll * Y * p.W + X;
    // ---- linear probe: log_softmax of the interpolated logits
    if (p.lin_logp || p.lin_arg) {
      float z[32];
      float mx;
      int arg;
      ev_linear(e, p.n_lin, z, mx, arg);
      lin_pred = arg;
      if (p.lin_arg) p.lin_arg[b * plane + pix] = static_cast<unsigned char>(arg);
      if (p.lin_logp) {
        float se = 0.f;
#pragma unroll
        for (int k = 0; k < 32; ++k)
          if (k < p.n_lin) se += __expf(z[k] - mx);
        const float lse = mx + __logf(se);
        float* o = p.lin_logp + (1ll * b * p.n_lin) * plane + pix;
#pragma unroll
        for (int k = 0; k < 32; ++k)
          if (k < p.n_lin) o[k * plane] = z[k] - lse;
      }
    }
    // ---- cluster probe: cosine similarity of the interpolated code with the centroids, log_softmax(alpha * .)
    if (p.clu_logp || p.clu_arg) {
      float z[32];
      float mx;
      int arg;
      ev_cluster(slr, t.bw, e, p.n_clu, z, mx, arg);
      clu_pred = arg;
      if (p.clu_arg) p.clu_arg[b * plane + pix] = static_cast<unsigned char>(arg);
      if (p.clu_logp) {
        float m2 = -INFINITY;
#pragma unroll
        for (int k = 0; k < 32; ++k)
          if (k < p.n_clu) m2 = fmaxf(m2, z[k] * p.alpha);
        float se = 0.f;
#pragma unroll
        for (int k = 0; k < 32; ++k)
          if (k < p.n_clu) se += __expf(z[k] * p.alpha - m2);
        const float lse = m2 + __logf(se);
        float* o = p.clu_logp + (1ll * b * p.n_clu) * plane + pix;
#pragma unroll
        for (int k = 0; k < 32; ++k)
          if (k < p.n_clu) o[k * plane] = z[k] * p.alpha - lse;
      }
    }
  }
  if (want_conf) {
    if (active)
      conf_hist_add(hist, read_label(p.label, p.label_bytes, 1ll * b * p.H * p.W + 1ll * Y * p.W + X), p.n_cls,
                    lin_pred, clu_pred);
    conf_hist_flush(hist, p.lin_conf, p.clu_conf, p.n_lin, p.n_clu, p.n_cls);
  }
}

// ---- dense-CRF unaries straight from the preparation table (stego_eval_crf_unary) -------------------------------------
// The CRF-refined evaluation (src/eval_segmentation.py:133-135 -> src/crf.py:22-45) runs the dense CRF on each probe's
// log-probabilities.  This kernel evaluates both probes per output pixel exactly as eval_probe_kernel does and writes,
// instead of the [B,n,H,W] log-probability planes, one 64-float row per pixel of the CRF's unary table
// U = -log(clip(softmax, 1e-5, 1)) (pydensecrf.utils.unary_from_softmax) and one of the initial Q = softmax(-U)
// (densecrf.cpp inference): linear probe in [0, 32), cluster probe in [32, 64), zeros beyond each probe's class count.
constexpr int EVC_LD = 64;

// One probe's unary and initial-Q half rows from its scores s[k < n] (softmax(s) = the probe's probabilities)
__device__ __forceinline__ void ev_crf_half_rows(const float (&s)[32], int n, float* u_row, float* q_row) {
  float mx = -INFINITY;
#pragma unroll
  for (int k = 0; k < 32; ++k)
    if (k < n) mx = fmaxf(mx, s[k]);
  float se = 0.f;
#pragma unroll
  for (int k = 0; k < 32; ++k)
    if (k < n) se += __expf(s[k] - mx);
  float u[32];
  float m2 = -INFINITY;
#pragma unroll
  for (int k = 0; k < 32; ++k) {
    u[k] = 0.f;
    if (k < n) {
      u[k] = -__logf(fminf(fmaxf(__expf(s[k] - mx) / se, 1e-5f), 1.0f));
      m2 = fmaxf(m2, -u[k]);
    }
  }
  float s2 = 0.f;
#pragma unroll
  for (int k = 0; k < 32; ++k)
    if (k < n) s2 += __expf(-u[k] - m2);
#pragma unroll
  for (int k = 0; k < 32; k += 4) {
    float4 uv, qv;
    uv.x = u[k]; uv.y = u[k + 1]; uv.z = u[k + 2]; uv.w = u[k + 3];
    qv.x = (k < n) ? __expf(-u[k] - m2) / s2 : 0.f;
    qv.y = (k + 1 < n) ? __expf(-u[k + 1] - m2) / s2 : 0.f;
    qv.z = (k + 2 < n) ? __expf(-u[k + 2] - m2) / s2 : 0.f;
    qv.w = (k + 3 < n) ? __expf(-u[k + 3] - m2) / s2 : 0.f;
    *reinterpret_cast<float4*>(u_row + k) = uv;
    *reinterpret_cast<float4*>(q_row + k) = qv;
  }
}

struct EvalCrfUnaryParams {
  const float* lr;  // [B*h*w][EV_LD]
  int B, h, w, H, W, n_lin, n_clu;
  float alpha;
  float* unary;     // [B*H*W][EVC_LD]
  float* Q;         // [B*H*W][EVC_LD]
};

__global__ void __launch_bounds__(EVT_W* EVT_H)
eval_crf_unary_kernel(EvalCrfUnaryParams p) {
  extern __shared__ float slr[];  // [box_h*box_w][EV_LD]
  const EvTile t = ev_tile_load(p.lr, slr, p.h, p.w, p.H, p.W, EVT_W, EVT_H);
  __syncthreads();
  const int X = t.X0 + (threadIdx.x % EVT_W), Y = t.Y0 + (threadIdx.x / EVT_W);
  if (X >= p.W || Y >= p.H) return;
  const EvCorners e = ev_corners(slr, t, p.h, p.w, Y, X);
  const long long row = (1ll * t.b * p.H + Y) * p.W + X;
  float* u_row = p.unary + row * EVC_LD;
  float* q_row = p.Q + row * EVC_LD;
  float z[32];
  float mx;
  int arg;
  ev_linear(e, p.n_lin, z, mx, arg);
  ev_crf_half_rows(z, p.n_lin, u_row, q_row);
  ev_cluster(slr, t.bw, e, p.n_clu, z, mx, arg);
#pragma unroll
  for (int k = 0; k < 32; ++k) z[k] *= p.alpha;
  ev_crf_half_rows(z, p.n_clu, u_row + 32, q_row + 32);
}


// ---- four pixels per thread (round 2) --------------------------------------------------------------------------------
// The pixel-per-thread kernel above is issue-bound, not HBM-bound (ncu: 70 % issue-active, 2900 warp instructions per
// 32 pixels, 20 % of the DRAM throughput): every class costs four scalar shared-memory loads, four FMAs and a strided
// 4-byte store per pixel.  When the horizontal upsampling factor is a multiple of 8, four x-adjacent output pixels
// (X = 4t .. 4t+3) always interpolate between the same two low-res columns, so a thread that owns all four
//   * loads the four corner rows once, as float4 (LDS.128, same address across most of the warp = broadcast),
//   * interpolates vertically once:  L[k] = a + ly (c - a),  R[k] = b + ly (d - b),  D[k] = R[k] - L[k],
//   * evaluates each pixel as z_j[k] = L[k] + lx_j D[k]  (one FMA per class), recomputing it in the three passes
//     (max/argmax, sum of exponentials, output) instead of keeping 4 x 27 logits in registers,
//   * writes one float4 per class plane (a warp covers 512 contiguous bytes of a plane row).
// Class counts are template parameters (27/27 = both shipped label sets); any other shape takes the generic kernel.
constexpr int EV4_TW = 64, EV4_ROWS = 4, EV4_W = 4 * EV4_TW;  // CTA tile: 256 x 4 pixels, 256 threads

template <int N, bool SCALED>
__device__ __forceinline__ void ev4_probe(const float* ea, const float* eb, const float* ec, const float* ed, float ly,
                                          const float (&lx)[4], const float (&scale)[4], float* out, long long plane,
                                          int (&pred)[4]) {
  constexpr int Q = (N + 3) / 4;
  float L[4 * Q], D[4 * Q];
#pragma unroll
  for (int q = 0; q < Q; ++q) {
    const float4 a = reinterpret_cast<const float4*>(ea)[q], b = reinterpret_cast<const float4*>(eb)[q];
    const float4 c = reinterpret_cast<const float4*>(ec)[q], d = reinterpret_cast<const float4*>(ed)[q];
    const float l0 = fmaf(ly, c.x - a.x, a.x), l1 = fmaf(ly, c.y - a.y, a.y), l2 = fmaf(ly, c.z - a.z, a.z),
                l3 = fmaf(ly, c.w - a.w, a.w);
    L[4 * q] = l0; L[4 * q + 1] = l1; L[4 * q + 2] = l2; L[4 * q + 3] = l3;
    D[4 * q] = fmaf(ly, d.x - b.x, b.x) - l0;
    D[4 * q + 1] = fmaf(ly, d.y - b.y, b.y) - l1;
    D[4 * q + 2] = fmaf(ly, d.z - b.z, b.z) - l2;
    D[4 * q + 3] = fmaf(ly, d.w - b.w, b.w) - l3;
  }
  float lse[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float mx = -INFINITY;
    int arg = 0;
#pragma unroll
    for (int k = 0; k < N; ++k) {
      float z = fmaf(lx[j], D[k], L[k]);
      if (SCALED) z *= scale[j];
      if (z > mx) { mx = z; arg = k; }
    }
    pred[j] = arg;
    float se = 0.f;
    if (out) {
      const float nmx = -mx * 1.4426950408889634f;
#pragma unroll
      for (int k = 0; k < N; ++k) {
        float z = fmaf(lx[j], D[k], L[k]);
        if (SCALED) z *= scale[j];
        se += ex2_approx(fmaf(z, 1.4426950408889634f, nmx));
      }
    }
    lse[j] = mx + __logf(se);
  }
  if (out) {
#pragma unroll
    for (int k = 0; k < N; ++k) {
      float4 o;
      o.x = fmaf(lx[0], D[k], L[k]); o.y = fmaf(lx[1], D[k], L[k]); o.z = fmaf(lx[2], D[k], L[k]); o.w = fmaf(lx[3], D[k], L[k]);
      if (SCALED) { o.x *= scale[0]; o.y *= scale[1]; o.z *= scale[2]; o.w *= scale[3]; }
      o.x -= lse[0]; o.y -= lse[1]; o.z -= lse[2]; o.w -= lse[3];
      *reinterpret_cast<float4*>(out + k * plane) = o;
    }
  }
}

template <int NL, int NC>
__global__ void __launch_bounds__(EV4_TW* EV4_ROWS, 2)
eval_probe_vec4_kernel(EvalProbeParams p) {
  extern __shared__ __align__(16) float slr[];  // [box_h*box_w][EV_LD]
  __shared__ ConfHist hist;
  const bool want_conf = p.label != nullptr;
  if (want_conf)
    for (int i = threadIdx.x; i < 2 * 32 * 32; i += blockDim.x) (&hist[0][0])[i] = 0u;
  const int tiles_x = (p.W + EV4_W - 1) / EV4_W, tiles_y = (p.H + EV4_ROWS - 1) / EV4_ROWS;
  const int tile = blockIdx.x;
  const int tx = tile % tiles_x, ty = (tile / tiles_x) % tiles_y, b = tile / (tiles_x * tiles_y);
  const int X0 = tx * EV4_W, Y0 = ty * EV4_ROWS;
  const int Xl = min(X0 + EV4_W - 1, p.W - 1), Yl = min(Y0 + EV4_ROWS - 1, p.H - 1);
  const float sy = static_cast<float>(p.h) / p.H, sx = static_cast<float>(p.w) / p.W;
  int by0, bh, bx0, bw;
  src_span(Y0, Yl, sy, p.h, by0, bh);
  src_span(X0, Xl, sx, p.w, bx0, bw);
  const long long base = 1ll * b * p.h * p.w;
  {
    constexpr int LD4 = EV_LD / 4;
    float4* s4 = reinterpret_cast<float4*>(slr);
    const float4* g4 = reinterpret_cast<const float4*>(p.lr);
    for (int i = threadIdx.x; i < bh * bw * LD4; i += blockDim.x) {
      const int cell = i / LD4, k = i % LD4;
      const int r = cell / bw, c = cell % bw;
      s4[i] = g4[(base + 1ll * (by0 + r) * p.w + bx0 + c) * LD4 + k];
    }
  }
  __syncthreads();
  const int X = X0 + 4 * (threadIdx.x % EV4_TW), Y = Y0 + threadIdx.x / EV4_TW;
  const bool active = X < p.W && Y < p.H;  // W % 4 == 0: a group is entirely inside or outside
  if (active) {
    int y0, y1, x0, x1;
    float ly, lx[4];
    src_index(Y, sy, p.h, y0, y1, ly);
    src_index(X, sx, p.w, x0, x1, lx[0]);
#pragma unroll
    for (int j = 1; j < 4; ++j) {  // same two columns for the whole group (host checks the upsampling factor)
      int t0, t1;
      src_index(X + j, sx, p.w, t0, t1, lx[j]);
    }
    y0 -= by0; y1 -= by0; x0 -= bx0; x1 -= bx0;
    const float* ea = slr + (y0 * bw + x0) * EV_LD;
    const float* eb = slr + (y0 * bw + x1) * EV_LD;
    const float* ec = slr + (y1 * bw + x0) * EV_LD;
    const float* ed = slr + (y1 * bw + x1) * EV_LD;
    const long long plane = 1ll * p.H * p.W;
    const long long pix = 1ll * Y * p.W + X;
    int lin_pred[4] = {-1, -1, -1, -1}, clu_pred[4] = {-1, -1, -1, -1};
    float one[4] = {1.f, 1.f, 1.f, 1.f};
    if (p.lin_logp || p.lin_arg) {
      ev4_probe<NL, false>(ea, eb, ec, ed, ly, lx, one, p.lin_logp ? p.lin_logp + (1ll * b * NL) * plane + pix : nullptr,
                           plane, lin_pred);
      if (p.lin_arg)
        *reinterpret_cast<uchar4*>(p.lin_arg + b * plane + pix) =
            make_uchar4((unsigned char)lin_pred[0], (unsigned char)lin_pred[1], (unsigned char)lin_pred[2], (unsigned char)lin_pred[3]);
    }
    if (p.clu_logp || p.clu_arg) {
      const double gaa = ev_grams(ea)[EV_SS], gbb = ev_grams(eb)[EV_SS], gcc = ev_grams(ec)[EV_SS], gdd = ev_grams(ed)[EV_SS];
      const double gab = ev_gram(slr, bw, y0, x0, y0, x1), gac = ev_gram(slr, bw, y0, x0, y1, x0);
      const double gad = ev_gram(slr, bw, y0, x0, y1, x1), gbc = ev_gram(slr, bw, y0, x1, y1, x0);
      const double gbd = ev_gram(slr, bw, y0, x1, y1, x1), gcd = ev_gram(slr, bw, y1, x0, y1, x1);
      // in fp64, once per thread: the vertically interpolated left / right codes l = (1-ly) a + ly c, r = (1-ly) b + ly d
      // give |l|^2, <l, r>, |r|^2, and each pixel's |(1-lx) l + lx r|^2 is a quadratic in its lx
      const double wy = ly, wy0 = 1.0 - wy;
      const double ll = wy0 * (wy0 * gaa + 2.0 * wy * gac) + wy * wy * gcc;
      const double rr = wy0 * (wy0 * gbb + 2.0 * wy * gbd) + wy * wy * gdd;
      const double lr = wy0 * (wy0 * gab + wy * (gad + gbc)) + wy * wy * gcd;
      float scale[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const double wx = lx[j], wx0 = 1.0 - wx;
        const double n2 = wx0 * (wx0 * ll + 2.0 * wx * lr) + wx * wx * rr;
        scale[j] = p.alpha / fmaxf(sqrtf(fmaxf(static_cast<float>(n2), 0.f)), 1e-12f);
      }
      ev4_probe<NC, true>(ea + 32, eb + 32, ec + 32, ed + 32, ly, lx, scale,
                          p.clu_logp ? p.clu_logp + (1ll * b * NC) * plane + pix : nullptr, plane, clu_pred);
      if (p.clu_arg)
        *reinterpret_cast<uchar4*>(p.clu_arg + b * plane + pix) =
            make_uchar4((unsigned char)clu_pred[0], (unsigned char)clu_pred[1], (unsigned char)clu_pred[2], (unsigned char)clu_pred[3]);
    }
    if (want_conf) {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        conf_hist_add(hist, read_label(p.label, p.label_bytes, b * plane + pix + j), p.n_cls, lin_pred[j], clu_pred[j]);
    }
  }
  if (want_conf) conf_hist_flush(hist, p.lin_conf, p.clu_conf, NL, NC, p.n_cls);
}

}  // namespace stego

using namespace stego;

// eval_prep_kernel over the B*h*w low-res pixels (arguments checked by the caller)
static int launch_eval_prep(const float* code, const float* code_flip, long long ld_code, int C, int B, int h, int w,
                            const float* lin_weight, const float* lin_bias, int n_lin, const float* clusters, int n_clu,
                            float* lr_scratch, cudaStream_t stream) {
  EvalPrepParams q;
  q.code = code; q.code_flip = code_flip; q.ld = ld_code; q.B = B; q.h = h; q.w = w; q.C = C; q.W = lin_weight; q.bias = lin_bias;
  q.n_lin = n_lin; q.clusters = clusters; q.n_clu = n_clu; q.lr = lr_scratch;
  const long long rows = 1ll * B * h * w;
  long long g = (rows + 7) / 8;
  const long long cap = 16ll * num_sms();
  eval_prep_kernel<<<(unsigned)(g < cap ? g : cap), 256, (size_t)C * 64 * sizeof(float), stream>>>(q);
  STEGO_CHECK_LAUNCH("eval_prep_kernel");
  return STEGO_OK;
}

// code: tokens-major low-res code [B*h*w][ld_code] fp32 (what DinoFeaturizer produces); outputs at [H][W].
// code_flip: the code of the horizontally flipped images (flip-TTA) or null.  lr_scratch: [B*h*w][80] floats, 16-byte aligned.
// label + confusion outputs (int64, accumulated): optional.  Any output pointer may be null.
extern "C" int stego_eval_probes(const float* code, const float* code_flip, long long ld_code, int C, int B, int h, int w,
                                 int H, int W, const float* lin_weight, const float* lin_bias, int n_lin,
                                 const float* clusters, int n_clu, float alpha, float* lr_scratch, float* lin_log_probs,
                                 float* clu_log_probs, unsigned char* lin_argmax, unsigned char* clu_argmax,
                                 const void* label, int label_bytes, int n_label_classes, long long* lin_confusion,
                                 long long* clu_confusion, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(code && lin_weight && lin_bias && clusters && lr_scratch, "stego_eval_probes: null pointer");
  STEGO_CHECK_ARG((reinterpret_cast<uintptr_t>(lr_scratch) & 7u) == 0, "stego_eval_probes: lr_scratch not 8-byte aligned");
  STEGO_CHECK_ARG(C > 0 && C <= 96 && n_lin > 0 && n_lin <= 32 && n_clu > 0 && n_clu <= 32,
                  "stego_eval_probes: C=%d n_lin=%d n_clu=%d unsupported (C <= 96, classes <= 32)", C, n_lin, n_clu);
  STEGO_CHECK_ARG(B > 0 && h > 0 && w > 0 && H >= h && W >= w, "stego_eval_probes: bad sizes (upsampling only)");
  STEGO_CHECK_ARG(!label || ((label_bytes == 8 || label_bytes == 4 || label_bytes == 1) && n_label_classes > 0 &&
                             n_label_classes <= 32 && (lin_confusion || clu_confusion)),
                  "stego_eval_probes: confusion counts need label_bytes in {8,4,1}, n_label_classes <= 32 and an output");
  int rc;
  if ((rc = launch_eval_prep(code, code_flip, ld_code, C, B, h, w, lin_weight, lin_bias, n_lin, clusters, n_clu,
                             lr_scratch, stream)) != STEGO_OK)
    return rc;
  EvalProbeParams p;
  p.lr = lr_scratch; p.B = B; p.h = h; p.w = w; p.H = H; p.W = W; p.n_lin = n_lin; p.n_clu = n_clu; p.alpha = alpha;
  p.lin_logp = lin_log_probs; p.clu_logp = clu_log_probs; p.lin_arg = lin_argmax; p.clu_arg = clu_argmax;
  p.label = label; p.label_bytes = label_bytes; p.n_cls = n_label_classes;
  p.lin_conf = reinterpret_cast<unsigned long long*>(lin_confusion);
  p.clu_conf = reinterpret_cast<unsigned long long*>(clu_confusion);
  // four pixels per thread when a group of four x-adjacent pixels always shares its two source columns: integer
  // horizontal factor that is a multiple of 8 (every patch-8 / patch-16 model evaluated at the label resolution)
  const bool vec4 = n_lin == 27 && n_clu == 27 && W % w == 0 && (W / w) % 8 == 0 &&
                    (!lin_log_probs || (reinterpret_cast<uintptr_t>(lin_log_probs) & 15) == 0) &&
                    (!clu_log_probs || (reinterpret_cast<uintptr_t>(clu_log_probs) & 15) == 0) &&
                    (!lin_argmax || (reinterpret_cast<uintptr_t>(lin_argmax) & 3) == 0) &&
                    (!clu_argmax || (reinterpret_cast<uintptr_t>(clu_argmax) & 3) == 0) &&
                    (reinterpret_cast<uintptr_t>(lr_scratch) & 15) == 0;
  const int tile_h = vec4 ? EV4_ROWS : EVT_H, tile_w = vec4 ? EV4_W : EVT_W;
  p.box_h = src_span_max(tile_h, h, H);
  p.box_w = src_span_max(tile_w, w, W);
  const size_t smem = (size_t)p.box_h * p.box_w * EV_LD * sizeof(float);
  STEGO_CHECK_ARG(smem <= 200 * 1024, "stego_eval_probes: upsample ratio needs %zu B of shared memory", smem);
  const long long tiles = 1ll * B * ((H + tile_h - 1) / tile_h) * ((W + tile_w - 1) / tile_w);
  STEGO_CHECK_ARG(tiles < (1ll << 31), "stego_eval_probes: too many tiles");
  if (vec4) {
    if ((rc = opt_in_smem<eval_probe_vec4_kernel<27, 27>>(smem, "eval_probe_vec4_kernel")) != STEGO_OK) return rc;
    eval_probe_vec4_kernel<27, 27><<<(unsigned)tiles, EV4_TW * EV4_ROWS, smem, stream>>>(p);
    STEGO_CHECK_LAUNCH("eval_probe_vec4_kernel");
    return STEGO_OK;
  }
  if ((rc = opt_in_smem<eval_probe_kernel>(smem, "eval_probe_kernel")) != STEGO_OK) return rc;
  eval_probe_kernel<<<(unsigned)tiles, EVT_W * EVT_H, smem, stream>>>(p);
  STEGO_CHECK_LAUNCH("eval_probe_kernel");
  return STEGO_OK;
}

// The dense-CRF unaries of both probes at [H][W] (see eval_crf_unary_kernel): the same inputs as stego_eval_probes;
// unary and Q: [B*H*W][64] fp32, 16-byte aligned (linear probe in floats [0, 32), cluster probe in [32, 64)).
extern "C" int stego_eval_crf_unary(const float* code, const float* code_flip, long long ld_code, int C, int B, int h, int w,
                                    int H, int W, const float* lin_weight, const float* lin_bias, int n_lin,
                                    const float* clusters, int n_clu, float alpha, float* lr_scratch, float* unary, float* Q,
                                    void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(code && lin_weight && lin_bias && clusters && lr_scratch && unary && Q, "stego_eval_crf_unary: null pointer");
  STEGO_CHECK_ARG((reinterpret_cast<uintptr_t>(lr_scratch) & 7u) == 0 && (reinterpret_cast<uintptr_t>(unary) & 15u) == 0 &&
                  (reinterpret_cast<uintptr_t>(Q) & 15u) == 0,
                  "stego_eval_crf_unary: lr_scratch must be 8-byte aligned, unary and Q 16-byte aligned");
  STEGO_CHECK_ARG(C > 0 && C <= 96 && n_lin > 0 && n_lin <= 32 && n_clu > 0 && n_clu <= 32,
                  "stego_eval_crf_unary: C=%d n_lin=%d n_clu=%d unsupported (C <= 96, classes <= 32)", C, n_lin, n_clu);
  STEGO_CHECK_ARG(B > 0 && h > 0 && w > 0 && H >= h && W >= w, "stego_eval_crf_unary: bad sizes (upsampling only)");
  const int box_h = src_span_max(EVT_H, h, H), box_w = src_span_max(EVT_W, w, W);
  const size_t smem = (size_t)box_h * box_w * EV_LD * sizeof(float);
  STEGO_CHECK_ARG(smem <= 200 * 1024, "stego_eval_crf_unary: upsample ratio needs %zu B of shared memory", smem);
  const long long tiles = 1ll * B * ((H + EVT_H - 1) / EVT_H) * ((W + EVT_W - 1) / EVT_W);
  STEGO_CHECK_ARG(tiles < (1ll << 31), "stego_eval_crf_unary: too many tiles");
  int rc;
  if ((rc = launch_eval_prep(code, code_flip, ld_code, C, B, h, w, lin_weight, lin_bias, n_lin, clusters, n_clu,
                             lr_scratch, stream)) != STEGO_OK)
    return rc;
  if ((rc = opt_in_smem<eval_crf_unary_kernel>(smem, "eval_crf_unary_kernel")) != STEGO_OK) return rc;
  EvalCrfUnaryParams p;
  p.lr = lr_scratch; p.B = B; p.h = h; p.w = w; p.H = H; p.W = W; p.n_lin = n_lin; p.n_clu = n_clu; p.alpha = alpha;
  p.unary = unary; p.Q = Q;
  eval_crf_unary_kernel<<<(unsigned)tiles, EVT_W * EVT_H, smem, stream>>>(p);
  STEGO_CHECK_LAUNCH("eval_crf_unary_kernel");
  return STEGO_OK;
}
