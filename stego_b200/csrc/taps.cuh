// Bilinear source taps of F.grid_sample(mode='bilinear', padding_mode='border', align_corners=True), shared by the
// correspondence-loss samplers (corr_loss.cu: make_taps) and the heatmap query sampler (heatmap.cu).
#pragma once
#include <cuda_runtime.h>

namespace stego {

struct Taps {
  int i00, i01, i10, i11;      // pixel offsets (y*W + x), clamped in-bounds
  float w00, w01, w10, w11;    // nw, ne, sw, se weights (0 for out-of-bounds taps)
};

// Taps of the grid point (gx, gy) in [-1, 1] (values beyond are clamped to the border) on an H x W map, with ATen's
// fp32 arithmetic: source coordinate ((g + 1) / 2) * (size - 1), clipped to [0, size - 1].
__device__ __forceinline__ Taps grid_taps(float gx, float gy, int H, int W) {
  float x = ((gx + 1.f) / 2.f) * (W - 1);
  float y = ((gy + 1.f) / 2.f) * (H - 1);
  x = fminf(fmaxf(x, 0.f), static_cast<float>(W - 1));
  y = fminf(fmaxf(y, 0.f), static_cast<float>(H - 1));
  const float x0 = floorf(x), y0 = floorf(y);
  const float x1 = x0 + 1.f, y1 = y0 + 1.f;
  Taps t;
  t.w00 = (x1 - x) * (y1 - y);
  t.w01 = (x - x0) * (y1 - y);
  t.w10 = (x1 - x) * (y - y0);
  t.w11 = (x - x0) * (y - y0);
  const int ix0 = static_cast<int>(x0), iy0 = static_cast<int>(y0);
  int ix1 = ix0 + 1, iy1 = iy0 + 1;
  if (ix1 > W - 1) { ix1 = W - 1; t.w01 = 0.f; t.w11 = 0.f; }
  if (iy1 > H - 1) { iy1 = H - 1; t.w10 = 0.f; t.w11 = 0.f; }
  t.i00 = iy0 * W + ix0;
  t.i01 = iy0 * W + ix1;
  t.i10 = iy1 * W + ix0;
  t.i11 = iy1 * W + ix1;
  return t;
}

}  // namespace stego
