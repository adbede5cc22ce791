// The sampling half of the aug-alignment term (src/train_segmentation.py:189-199, src/utils.py:61-62,
// src/modules.py:287-288):
//     coord = F.interpolate(coord_aug.permute(0, 3, 1, 2), h, mode="bilinear", align_corners=False).permute(0, 2, 3, 1)
//     sampled = F.grid_sample(code, coord.permute(0, 2, 1, 3), padding_mode="border", align_corners=True)
//     aug_alignment = -cosine(sampled, code_aug).mean()
// The resize of the two coordinate channels is evaluated only at the h x h points grid_sample reads, with ATen's
// upsample_bilinear2d arithmetic (resize.cuh); the taps are grid_sample's (grid_taps of taps.cuh),
// accumulated in ATen's order, so both match torch's CUDA results bit for bit.  Output pixel (p, q) reads grid point
// (q, p): the permute(0, 2, 1, 3).
// The cosine and its gradients are stego_cosine_fwd / _bwd; the backward here scatters d(sampled) into d(code) with
// the same taps, and stego_aug_align_loss is the fixed-order mean (the logged term repeats bit for bit).
#include "resize.cuh"
#include "taps.cuh"
#include "host_util.h"

namespace stego {

struct AugAlignParams {
  const float* coord_aug;  // [B][S][S][2] contiguous
  int S;
  float scale;             // ATen's (float)S / h
  const float* code; long long sb, sc, sy, sx;  // [B][C][h][h], any strides (fwd: read, bwd: accumulated into)
  int B, C, h;
  float* grid;             // [B][h][h][2]: `coord` above (fwd: written, bwd: read)
  float* sampled;          // [B][C][h][h] contiguous (fwd: written; bwd: d(sampled), read)
};

// One thread per output pixel (b, p, q); consecutive threads take consecutive q, so the NCHW stores coalesce.
__global__ void __launch_bounds__(256) aug_align_fwd_kernel(AugAlignParams p) {
  const long long npix = 1ll * p.B * p.h * p.h;
  const long long pix = 1ll * blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= npix) return;
  const int q = static_cast<int>(pix % p.h), pp = static_cast<int>((pix / p.h) % p.h), b = static_cast<int>(pix / (1ll * p.h * p.h));
  // this thread writes grid point (i, j) = (pp, q) and samples with grid point (q, pp)
  const float* cb = p.coord_aug + static_cast<long long>(b) * p.S * p.S * 2;
  // grid[b][i][j][c] = channel c of the resized coordinates at (i, j)
  auto chan = [&](int c) { return [=](int y, int x) { return cb[(static_cast<long long>(y) * p.S + x) * 2 + c]; }; };
  ResizeTaps rt = resize_taps(pp, q, p.scale, p.scale, p.S, p.S);
  float* gw = p.grid + ((static_cast<long long>(b) * p.h + pp) * p.h + q) * 2;
  gw[0] = resize_at(rt, chan(0));
  gw[1] = resize_at(rt, chan(1));
  rt = resize_taps(q, pp, p.scale, p.scale, p.S, p.S);
  const float gx = resize_at(rt, chan(0)), gy = resize_at(rt, chan(1));
  const Taps t = grid_taps(gx, gy, p.h, p.h);
  auto off = [&](int i) { return static_cast<long long>(i / p.h) * p.sy + static_cast<long long>(i % p.h) * p.sx; };
  const float* base = p.code + static_cast<long long>(b) * p.sb;
  const long long o00 = off(t.i00), o01 = off(t.i01), o10 = off(t.i10), o11 = off(t.i11);
  float* out = p.sampled + static_cast<long long>(b) * p.C * p.h * p.h + static_cast<long long>(pp) * p.h + q;
  for (int c = 0; c < p.C; ++c) {
    const float* cp = base + c * p.sc;
    // ATen's grid_sampler_2d_kernel: out_acc = 0, then out_acc += tap * weight for nw, ne, sw, se, each fused onto the
    // running sum (the first is a plain rounded product).  Written with intrinsics so that nvcc cannot pick another
    // product to fuse.  A zero-weight tap (the border clamp) adds exactly nothing, as ATen's skipped branch does.
    float v = __fmul_rn(cp[o00], t.w00);
    v = __fmaf_rn(cp[o01], t.w01, v);
    v = __fmaf_rn(cp[o10], t.w10, v);
    v = __fmaf_rn(cp[o11], t.w11, v);
    out[static_cast<long long>(c) * p.h * p.h] = v;
  }
}

// d(code) += the four tap weights x d(sampled), by atomics (taps of different pixels coincide).  A zero-weight tap
// (the border clamp, or a grid point on an integer tap) adds nothing and is skipped.
__global__ void __launch_bounds__(256) aug_align_bwd_kernel(AugAlignParams p) {
  const long long npix = 1ll * p.B * p.h * p.h;
  const long long pix = 1ll * blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= npix) return;
  const int q = static_cast<int>(pix % p.h), pp = static_cast<int>((pix / p.h) % p.h), b = static_cast<int>(pix / (1ll * p.h * p.h));
  const float* g = p.grid + ((static_cast<long long>(b) * p.h + q) * p.h + pp) * 2;
  const Taps t = grid_taps(g[0], g[1], p.h, p.h);
  auto off = [&](int i) { return static_cast<long long>(i / p.h) * p.sy + static_cast<long long>(i % p.h) * p.sx; };
  float* base = const_cast<float*>(p.code) + static_cast<long long>(b) * p.sb;
  const long long o[4] = {off(t.i00), off(t.i01), off(t.i10), off(t.i11)};
  const float w[4] = {t.w00, t.w01, t.w10, t.w11};
  const float* d = p.sampled + static_cast<long long>(b) * p.C * p.h * p.h + static_cast<long long>(pp) * p.h + q;
  for (int c = 0; c < p.C; ++c) {
    const float dv = d[static_cast<long long>(c) * p.h * p.h];
    float* cp = base + c * p.sc;
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (w[k] != 0.f) atomicAdd(cp + o[k], w[k] * dv);
  }
}

// loss[0] = -(sum of cosv) / n, summed in fp64 in a fixed order by one CTA; total[0] += weight * loss[0] (if given).
constexpr int kLossThreads = 1024;
__global__ void __launch_bounds__(kLossThreads) aug_align_loss_kernel(const float* cosv, long long n, float weight,
                                                                     float* loss, float* total) {
  __shared__ double part[kLossThreads];
  double s = 0.0;
  for (long long i = threadIdx.x; i < n; i += kLossThreads) s += static_cast<double>(cosv[i]);
  part[threadIdx.x] = s;
  __syncthreads();
  for (int w = kLossThreads / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) part[threadIdx.x] += part[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const float l = static_cast<float>(-(part[0] / static_cast<double>(n)));
    loss[0] = l;
    if (total) total[0] = __fadd_rn(total[0], __fmul_rn(weight, l));
  }
}

inline int check_common(const float* code, int B, int C, int h, const float* grid, const float* sampled, const char* who) {
  STEGO_CHECK_ARG(code && grid && sampled, "%s: null pointer", who);
  STEGO_CHECK_ARG(B >= 1 && C >= 1 && h >= 1 && 1ll * B * h * h <= (1ll << 31), "%s: B=%d C=%d h=%d", who, B, C, h);
  return STEGO_OK;
}

}  // namespace stego

using namespace stego;

extern "C" int stego_aug_align_fwd(const float* coord_aug, int S, const float* code, long long sb, long long sc,
                                   long long sy, long long sx, int B, int C, int h, float* grid, float* sampled,
                                   void* stream_) {
  if (int rc = check_common(code, B, C, h, grid, sampled, "stego_aug_align_fwd")) return rc;
  STEGO_CHECK_ARG(coord_aug && S >= 1, "stego_aug_align_fwd: coord_aug null or S=%d", S);
  AugAlignParams p{coord_aug, S, static_cast<float>(S) / static_cast<float>(h), code, sb, sc, sy, sx, B, C, h, grid,
                   sampled};
  const long long npix = 1ll * B * h * h;
  aug_align_fwd_kernel<<<(unsigned)((npix + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(p);
  STEGO_CHECK_LAUNCH("aug_align_fwd_kernel");
  return STEGO_OK;
}

extern "C" int stego_aug_align_bwd(const float* grid, const float* dsampled, int B, int C, int h, float* dcode,
                                   long long sb, long long sc, long long sy, long long sx, void* stream_) {
  if (int rc = check_common(dcode, B, C, h, grid, dsampled, "stego_aug_align_bwd")) return rc;
  AugAlignParams p{nullptr, 0, 0.f, dcode, sb, sc, sy, sx, B, C, h, const_cast<float*>(grid), const_cast<float*>(dsampled)};
  const long long npix = 1ll * B * h * h;
  aug_align_bwd_kernel<<<(unsigned)((npix + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(p);
  STEGO_CHECK_LAUNCH("aug_align_bwd_kernel");
  return STEGO_OK;
}

extern "C" int stego_aug_align_loss(const float* cosv, long long n, float weight, float* loss, float* total,
                                    void* stream_) {
  STEGO_CHECK_ARG(cosv && loss && n >= 1, "stego_aug_align_loss: null pointer or n=%lld", n);
  aug_align_loss_kernel<<<1, kLossThreads, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(cosv, n, weight, loss, total);
  STEGO_CHECK_LAUNCH("aug_align_loss_kernel");
  return STEGO_OK;
}
