// The aug-alignment views of the reference's training data (src/data.py:527-563 with the transforms of
// src/train_segmentation.py:408-416), for a batch in two launches:
//
//     img_aug   = RandomApply([GaussianBlur((5, 5))]) . RandomGrayscale(.2) . ColorJitter(.3, .3, .3, .1)
//                 . RandomResizedCrop(size, scale=(.8, 1)) . RandomHorizontalFlip()  (img)
//     coord_aug = RandomResizedCrop . RandomHorizontalFlip (coord), coord = meshgrid(linspace(-1, 1, H), linspace(-1, 1, W))
//
// with torchvision's tensor arithmetic (transforms/_functional_tensor.py) on the normalised fp32 frames.  The host draws
// every random parameter (stego_b200/augment.py) and uploads one record of AUG_WORDS words per sample.
//
// aug_geometry_kernel: one thread per output pixel.  hflip, crop and interpolate(bilinear, align_corners=False,
//   antialias=True) as ATen's separable antialiased filter: per axis scale = crop / size, support = max(scale, 1),
//   taps [lo, lo + n) around centre = scale (o + .5), triangle weights at (k - centre + .5) / max(scale, 1) divided by
//   their sum; each row is summed over the x taps, then the rows over the y taps.  Applies the colour-jitter ops that
//   precede contrast, writes the three channels to scratch (`mid`) and coord_aug to its output, and leaves one fp64
//   partial sum of rgb_to_grayscale per CTA for contrast's mean.
// aug_photometric_kernel: one CTA per 32 x 8 output tile of an image.  Sums the image's partials in a fixed order (the
//   outputs are bit-reproducible), runs contrast and the ops after it, grayscale, on the tile and a 2-pixel reflected
//   halo held in shared memory, and applies the 5 x 5 blur there (each CTA recomputes its halo instead of a third pass).
//
// Every fp32 operation is rounded as torch rounds it (no contraction into FMA), including on inputs outside [0, 1]:
// hue before the first clamp sees negative values, and its `maxc == 0` pixels give torch's NaN.
#include "common.cuh"
#include "host_util.h"

namespace stego {

constexpr int AUG_TX = 32, AUG_TY = 8, AUG_THREADS = AUG_TX * AUG_TY, AUG_HALO = 2;
constexpr int AUG_WORDS = 48;
// record layout (int32 words; factors and weights are fp32 bit patterns)
enum : int {
  A_FLIP = 0, A_TOP, A_LEFT, A_CROP_H, A_CROP_W,
  A_ORDER = 5,              // 4 words: ColorJitter's fn_idx (0 brightness, 1 contrast, 2 saturation, 3 hue)
  A_GRAY = 9, A_BLUR,
  A_BRIGHT = 11, A_BRIGHT1, // factor, fl(1 - factor): _blend's two ratios
  A_CONTRAST, A_CONTRAST1, A_SAT, A_SAT1, A_HUE,
  A_KERNEL = 18,            // 25 words: the 5 x 5 Gaussian weights, row-major
};

struct AugParams {
  const float* img;
  long long sb, sc, sy, sx;
  const int* rec;     // [B][AUG_WORDS]
  double* partials;   // [B][tiles]
  float* mid;         // [B][3][size][size]
  float* img_aug;     // [B][3][size][size]
  float* coord_aug;   // [B][size][size][2]
  int B, H, W, size, tiles_x, tiles;
};

__device__ __forceinline__ float recf(const int* r, int k) { return __int_as_float(r[k]); }

__device__ __forceinline__ float clamp01(float v) { return v < 0.0f ? 0.0f : (v > 1.0f ? 1.0f : v); }  // NaN stays

__device__ __forceinline__ float gray_of(float r, float g, float b) {
  return __fadd_rn(__fadd_rn(__fmul_rn(0.2989f, r), __fmul_rn(0.587f, g)), __fmul_rn(0.114f, b));
}

// _blend(img1, img2, ratio) = (ratio img1 + (1 - ratio) img2).clamp(0, 1)
__device__ __forceinline__ float blend(float a, float b, float ratio, float ratio1) {
  return clamp01(__fadd_rn(__fmul_rn(ratio, a), __fmul_rn(ratio1, b)));
}

// adjust_hue: _rgb2hsv, h = (h + factor) % 1.0 (torch.remainder), _hsv2rgb
__device__ __forceinline__ void hue(float& r, float& g, float& b, float factor) {
  const float maxc = fmaxf(r, fmaxf(g, b)), minc = fminf(r, fminf(g, b));
  const bool eqc = maxc == minc;
  const float cr = __fsub_rn(maxc, minc);
  const float s = __fdiv_rn(cr, eqc ? 1.0f : maxc);
  const float crd = eqc ? 1.0f : cr;
  const float rc = __fdiv_rn(__fsub_rn(maxc, r), crd), gc = __fdiv_rn(__fsub_rn(maxc, g), crd);
  const float bc = __fdiv_rn(__fsub_rn(maxc, b), crd);
  const float hr = maxc == r ? __fsub_rn(bc, gc) : 0.0f;
  const float hg = (maxc == g && maxc != r) ? __fsub_rn(__fadd_rn(2.0f, rc), bc) : 0.0f;
  const float hb = (maxc != g && maxc != r) ? __fsub_rn(__fadd_rn(4.0f, gc), rc) : 0.0f;
  float h = fmodf(__fadd_rn(__fdiv_rn(__fadd_rn(__fadd_rn(hr, hg), hb), 6.0f), 1.0f), 1.0f);
  h = fmodf(__fadd_rn(h, factor), 1.0f);
  if (h != 0.0f && h < 0.0f) h = __fadd_rn(h, 1.0f);
  const float h6 = __fmul_rn(h, 6.0f), fl = floorf(h6);
  const float f = __fsub_rn(h6, fl);
  const int i = static_cast<int>(fl) % 6;
  const float v = maxc;
  const float p = clamp01(__fmul_rn(v, __fsub_rn(1.0f, s)));
  const float q = clamp01(__fmul_rn(v, __fsub_rn(1.0f, __fmul_rn(s, f))));
  const float t = clamp01(__fmul_rn(v, __fsub_rn(1.0f, __fmul_rn(s, __fsub_rn(1.0f, f)))));
  if (isnan(p) || isnan(q) || isnan(t)) {  // the einsum multiplies every candidate by its 0 / 1 mask
    r = g = b = __int_as_float(0x7fffffff);
    return;
  }
  switch (i) {
    case 0: r = v; g = t; b = p; break;
    case 1: r = q; g = v; b = p; break;
    case 2: r = p; g = v; b = t; break;
    case 3: r = p; g = q; b = v; break;
    case 4: r = t; g = p; b = v; break;
    default: r = v; g = p; b = q; break;
  }
}

// the jitter ops at positions [from, to) of the record's order; contrast (id 1) uses `mean`
__device__ __forceinline__ void jitter(const int* rec, int from, int to, float mean, float& r, float& g, float& b) {
  for (int k = from; k < to; ++k) {
    const int op = rec[A_ORDER + k];
    if (op == 0) {
      const float f = recf(rec, A_BRIGHT), f1 = recf(rec, A_BRIGHT1);
      r = blend(r, 0.0f, f, f1); g = blend(g, 0.0f, f, f1); b = blend(b, 0.0f, f, f1);
    } else if (op == 1) {
      const float f = recf(rec, A_CONTRAST), f1 = recf(rec, A_CONTRAST1);
      r = blend(r, mean, f, f1); g = blend(g, mean, f, f1); b = blend(b, mean, f, f1);
    } else if (op == 2) {
      const float f = recf(rec, A_SAT), f1 = recf(rec, A_SAT1), l = gray_of(r, g, b);
      r = blend(r, l, f, f1); g = blend(g, l, f, f1); b = blend(b, l, f, f1);
    } else {
      hue(r, g, b, recf(rec, A_HUE));
    }
  }
}

__device__ __forceinline__ int contrast_pos(const int* rec) {
  int k = 0;
  while (k < 3 && rec[A_ORDER + k] != 1) ++k;
  return k;
}

// one axis of ATen's antialiased bilinear resize (align_corners=False) of `in_size` samples to `out_size`
struct AaAxis {
  float center, invscale, total;
  int lo, n;
};

__device__ __forceinline__ float tri(float x) {
  x = fabsf(x);
  return x < 1.0f ? __fsub_rn(1.0f, x) : 0.0f;
}

__device__ __forceinline__ AaAxis aa_axis(int o, int in_size, int out_size) {
  AaAxis a;
  const float scale = __fdiv_rn(static_cast<float>(in_size), static_cast<float>(out_size));
  const float support = scale >= 1.0f ? scale : 1.0f;
  a.invscale = scale >= 1.0f ? __fdiv_rn(1.0f, scale) : 1.0f;
  a.center = __fmul_rn(scale, __fadd_rn(static_cast<float>(o), 0.5f));
  a.lo = max(static_cast<int>(__fadd_rn(__fsub_rn(a.center, support), 0.5f)), 0);
  a.n = min(static_cast<int>(__fadd_rn(__fadd_rn(a.center, support), 0.5f)), in_size) - a.lo;
  a.total = 0.0f;
  for (int k = 0; k < a.n; ++k) a.total = __fadd_rn(a.total, tri(__fmul_rn(__fadd_rn(__fsub_rn(
      static_cast<float>(k + a.lo), a.center), 0.5f), a.invscale)));
  return a;
}

__device__ __forceinline__ float aa_weight(const AaAxis& a, int k) {
  const float w = tri(__fmul_rn(__fadd_rn(__fsub_rn(static_cast<float>(k + a.lo), a.center), 0.5f), a.invscale));
  return a.total != 0.0f ? __fdiv_rn(w, a.total) : w;
}

// torch.linspace(-1, 1, n)[k] in fp32: start + step k on the first half, end - step (n - 1 - k) on the second
__device__ __forceinline__ float linspace_pm1(int k, int n) {
  if (n == 1) return -1.0f;
  const float step = __fdiv_rn(2.0f, static_cast<float>(n - 1));
  return k < n / 2 ? __fadd_rn(-1.0f, __fmul_rn(step, static_cast<float>(k)))
                   : __fsub_rn(1.0f, __fmul_rn(step, static_cast<float>(n - 1 - k)));
}

__global__ void __launch_bounds__(AUG_THREADS) aug_geometry_kernel(AugParams p) {
  __shared__ double warp_sums[AUG_THREADS / 32];
  const int b = blockIdx.y, tile = blockIdx.x;
  const int ox = (tile % p.tiles_x) * AUG_TX + (threadIdx.x & (AUG_TX - 1));
  const int oy = (tile / p.tiles_x) * AUG_TY + threadIdx.x / AUG_TX;
  const int* rec = p.rec + static_cast<size_t>(b) * AUG_WORDS;
  double gsum = 0.0;
  if (ox < p.size && oy < p.size) {
    const int flip = rec[A_FLIP], top = rec[A_TOP], left = rec[A_LEFT];
    const AaAxis ay = aa_axis(oy, rec[A_CROP_H], p.size), ax = aa_axis(ox, rec[A_CROP_W], p.size);
    const float* src = p.img + static_cast<size_t>(b) * p.sb;
    float acc[5] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
    for (int j = 0; j < ay.n; ++j) {
      const int y = min(max(top + ay.lo + j, 0), p.H - 1);
      const float ly = linspace_pm1(y, p.H);
      float row[5] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
      for (int i = 0; i < ax.n; ++i) {
        const int xf = min(max(left + ax.lo + i, 0), p.W - 1);  // column of the flipped frame
        const int x = flip ? p.W - 1 - xf : xf;
        const float w = aa_weight(ax, i);
        const float* s = src + y * p.sy + x * p.sx;
        row[0] = __fadd_rn(row[0], __fmul_rn(w, s[0]));
        row[1] = __fadd_rn(row[1], __fmul_rn(w, s[p.sc]));
        row[2] = __fadd_rn(row[2], __fmul_rn(w, s[2 * p.sc]));
        row[3] = __fadd_rn(row[3], __fmul_rn(w, ly));
        row[4] = __fadd_rn(row[4], __fmul_rn(w, linspace_pm1(x, p.W)));
      }
      const float w = aa_weight(ay, j);
#pragma unroll
      for (int c = 0; c < 5; ++c) acc[c] = __fadd_rn(acc[c], __fmul_rn(w, row[c]));
    }
    float r = acc[0], g = acc[1], bl = acc[2];
    jitter(rec, 0, contrast_pos(rec), 0.0f, r, g, bl);
    const size_t plane = static_cast<size_t>(p.size) * p.size, pix = static_cast<size_t>(oy) * p.size + ox;
    float* mid = p.mid + static_cast<size_t>(b) * 3 * plane + pix;
    mid[0] = r; mid[plane] = g; mid[2 * plane] = bl;
    float* co = p.coord_aug + (static_cast<size_t>(b) * plane + pix) * 2;
    co[0] = acc[3]; co[1] = acc[4];
    gsum = static_cast<double>(gray_of(r, g, bl));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) gsum += __shfl_xor_sync(0xffffffffu, gsum, o);
  if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = gsum;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int k = 0; k < AUG_THREADS / 32; ++k) t += warp_sums[k];
    p.partials[static_cast<size_t>(b) * p.tiles + tile] = t;
  }
}

__device__ __forceinline__ int reflect_index(int k, int n) {
  k = k < 0 ? -k : (k >= n ? 2 * n - 2 - k : k);
  return min(max(k, 0), n - 1);  // positions only tile padding reaches
}

__global__ void __launch_bounds__(AUG_THREADS) aug_photometric_kernel(AugParams p) {
  constexpr int HX = AUG_TX + 2 * AUG_HALO, HY = AUG_TY + 2 * AUG_HALO;
  __shared__ float px[3][HY][HX];
  __shared__ float mean_s;
  const int b = blockIdx.y, tile = blockIdx.x;
  const int x0 = (tile % p.tiles_x) * AUG_TX, y0 = (tile / p.tiles_x) * AUG_TY;
  const int* rec = p.rec + static_cast<size_t>(b) * AUG_WORDS;
  if (threadIdx.x < 32) {  // contrast's mean: the image's partials in a fixed order
    const double* part = p.partials + static_cast<size_t>(b) * p.tiles;
    double t = 0.0;
    for (int k = threadIdx.x; k < p.tiles; k += 32) t += part[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if (threadIdx.x == 0) mean_s = static_cast<float>(t / (static_cast<double>(p.size) * p.size));
  }
  __syncthreads();
  const float mean = mean_s;
  const int from = contrast_pos(rec), gray = rec[A_GRAY], blur = rec[A_BLUR];
  const size_t plane = static_cast<size_t>(p.size) * p.size;
  const float* mid = p.mid + static_cast<size_t>(b) * 3 * plane;
  for (int e = threadIdx.x; e < HX * HY; e += AUG_THREADS) {
    const int hy = e / HX, hx = e - hy * HX;
    const size_t pix = static_cast<size_t>(reflect_index(y0 - AUG_HALO + hy, p.size)) * p.size +
                       reflect_index(x0 - AUG_HALO + hx, p.size);
    float r = mid[pix], g = mid[plane + pix], bl = mid[2 * plane + pix];
    jitter(rec, from, 4, mean, r, g, bl);
    if (gray) r = g = bl = gray_of(r, g, bl);
    px[0][hy][hx] = r; px[1][hy][hx] = g; px[2][hy][hx] = bl;
  }
  __syncthreads();
  const int tx = threadIdx.x & (AUG_TX - 1), ty = threadIdx.x / AUG_TX;
  const int ox = x0 + tx, oy = y0 + ty;
  if (ox >= p.size || oy >= p.size) return;
  float* out = p.img_aug + static_cast<size_t>(b) * 3 * plane + static_cast<size_t>(oy) * p.size + ox;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float v;
    if (blur) {
      v = 0.0f;
#pragma unroll
      for (int ky = 0; ky < 5; ++ky)
#pragma unroll
        for (int kx = 0; kx < 5; ++kx) v = __fmaf_rn(recf(rec, A_KERNEL + ky * 5 + kx), px[c][ty + ky][tx + kx], v);
    } else {
      v = px[c][ty + AUG_HALO][tx + AUG_HALO];
    }
    out[c * plane] = v;
  }
}

static int aug_tiles(int size) { return ((size + AUG_TX - 1) / AUG_TX) * ((size + AUG_TY - 1) / AUG_TY); }

static long long aug_mid_offset(int B, int size) {  // fp64 partials first, then the fp32 intermediate
  return (8ll * B * aug_tiles(size) + 255) / 256 * 256;
}

}  // namespace stego

using namespace stego;

// C-ABI: see include/stego_b200.h for the contract.
extern "C" int stego_aug_record_words(void) { return AUG_WORDS; }

extern "C" long long stego_aug_scratch_bytes(int B, int size) {
  if (B < 1 || size < 1) return 0;
  return aug_mid_offset(B, size) + 12ll * B * size * size;
}

extern "C" int stego_aug_views(const float* img, long long stride_b, long long stride_c, long long stride_y,
                               long long stride_x, int B, int H, int W, int size, const int* records, void* scratch,
                               float* img_aug, float* coord_aug, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(img && records && scratch && img_aug && coord_aug, "stego_aug_views: null pointer");
  STEGO_CHECK_ARG(B >= 1 && B <= 65535, "stego_aug_views: B=%d (1..65535)", B);
  STEGO_CHECK_ARG(H >= 1 && W >= 1, "stego_aug_views: H=%d W=%d must be >= 1", H, W);
  STEGO_CHECK_ARG(size >= 3 && size <= 8192, "stego_aug_views: size=%d (3..8192: the blur's reflect padding needs 3)",
                  size);
  STEGO_CHECK_ARG(reinterpret_cast<uintptr_t>(scratch) % 8 == 0, "stego_aug_views: scratch must be 8-byte aligned");
  AugParams p;
  p.img = img; p.sb = stride_b; p.sc = stride_c; p.sy = stride_y; p.sx = stride_x;
  p.rec = records;
  p.partials = static_cast<double*>(scratch);
  p.mid = reinterpret_cast<float*>(static_cast<char*>(scratch) + aug_mid_offset(B, size));
  p.img_aug = img_aug; p.coord_aug = coord_aug;
  p.B = B; p.H = H; p.W = W; p.size = size;
  p.tiles_x = (size + AUG_TX - 1) / AUG_TX;
  p.tiles = aug_tiles(size);
  const dim3 grid(p.tiles, B);
  aug_geometry_kernel<<<grid, AUG_THREADS, 0, stream>>>(p);
  STEGO_CHECK_LAUNCH("aug_geometry_kernel launch");
  aug_photometric_kernel<<<grid, AUG_THREADS, 0, stream>>>(p);
  STEGO_CHECK_LAUNCH("aug_photometric_kernel launch");
  return STEGO_OK;
}
