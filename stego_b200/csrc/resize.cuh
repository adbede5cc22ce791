// F.interpolate(mode="bilinear", align_corners=False) evaluated at single output points, with ATen's
// upsample_bilinear2d arithmetic: the source indices and lambdas of src_index (probe_common.cuh) and the tap expression
// of upsample_bilinear2d_out_frame, so a value computed here is bit-equal to torch's resized map at that point.  Shared by
// the aug-alignment coordinate resize (aug_align.cu) and the CRF term's sampled code and guidance (crf_loss.cu).
#pragma once
#include "probe_common.cuh"

namespace stego {

struct ResizeTaps {
  int y0, y1, x0, x1;
  float ly, lx;  // weights of the y1 / x1 taps
};

// Taps of output point (i, j) of an in_h x in_w map resized with scales (float)in / out (ATen's, no scale factor given)
__device__ __forceinline__ ResizeTaps resize_taps(int i, int j, float scale_h, float scale_w, int in_h, int in_w) {
  ResizeTaps t;
  src_index(i, scale_h, in_h, t.y0, t.y1, t.ly);
  src_index(j, scale_w, in_w, t.x0, t.x1, t.lx);
  return t;
}

// h0l * (w0l * at(y0, x0) + w1l * at(y0, x1)) + h1l * (w0l * at(y1, x0) + w1l * at(y1, x1)), ATen's expression as
// upsample_bilinear2d_out_frame evaluates it (the NCHW kernel)
template <class At>
__device__ __forceinline__ float resize_at(const ResizeTaps& t, At at) {
  const float h1l = t.ly, h0l = 1.f - t.ly, w1l = t.lx, w0l = 1.f - t.lx;
  return h0l * (w0l * at(t.y0, t.x0) + w1l * at(t.y0, t.x1)) + h1l * (w0l * at(t.y1, t.x0) + w1l * at(t.y1, t.x1));
}

// The same expression as upsample_bilinear2d_nhwc_out_frame evaluates it: the kernel ATen runs for channels-last inputs
// with at least 16 channels, whose compiled form fuses other products into the sums (read from its sm_90 SASS):
// top = w1l at(y0, x1) + fl(w0l at(y0, x0)), bottom = w0l at(y1, x0) + fl(w1l at(y1, x1)), h0l top + fl(h1l bottom)
template <class At>
__device__ __forceinline__ float resize_at_nhwc(const ResizeTaps& t, At at) {
  const float h1l = t.ly, h0l = 1.f - t.ly, w1l = t.lx, w0l = 1.f - t.lx;
  const float top = __fmaf_rn(w1l, at(t.y0, t.x1), __fmul_rn(w0l, at(t.y0, t.x0)));
  const float bot = __fmaf_rn(w0l, at(t.y1, t.x0), __fmul_rn(w1l, at(t.y1, t.x1)));
  return __fmaf_rn(h0l, top, __fmul_rn(h1l, bot));
}

// at::TensorImpl's channels-last test (is_channels_last_strides_2d_s4) for sizes (B, C, H, W) and element strides: the
// layout F.interpolate reads a tensor as
inline bool aten_channels_last(long long B, long long C, long long H, long long W, long long sb, long long sc, long long sy,
                               long long sx) {
  const long long sizes[4] = {B, C, H, W}, strides[4] = {sb, sc, sy, sx};
  if (strides[1] == 0) return false;
  long long min = 0;
  for (int d : {1, 3, 2, 0}) {
    if (sizes[d] == 0 || strides[d] < min) return false;
    if (d == 0 && min == strides[1]) return false;
    min = strides[d];
    if (sizes[d] > 1) min *= sizes[d];
  }
  return true;
}

}  // namespace stego
