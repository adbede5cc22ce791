// Per-pixel cosine similarity of two feature maps and its backward: the arithmetic of the reference's two optional
// alignment terms (SURVEY.md §8 row f4),
//     rec_loss      = -(norm(decoder(code)) * norm(feats)).sum(1).mean()                         train_segmentation.py:183-187
//     aug_alignment = -einsum("bkhw,bkhw->bhw", norm(sample(code, coord)), norm(code_aug)).mean() train_segmentation.py:189-199
// with norm = F.normalize(t, dim=1, eps=1e-10) (src/modules.py:275-276).  The reference runs two normalisations (four
// passes each), a product and a channel reduction over [B, C, h, w] tensors; here each input is read once in the forward
// and once in the backward.  Inputs are fp32 with arbitrary element strides: channels-last views (what DinoFeaturizer
// returns, channel stride 1) take the warp-per-pixel path, anything else the thread-per-pixel path.
#include "common.cuh"
#include "cosine.cuh"
#include "host_util.h"

namespace stego {

struct CosParams {
  const float* a; long long a_sb, a_sc, a_sy, a_sx;
  const float* b; long long b_sb, b_sc, b_sy, b_sx;
  int B, C, H, W;
  float eps;
  float* cosv;   // [B*H*W]
  float* norma;  // [B*H*W] |a| in fp32, unclamped: the backward needs |a| >= eps, which 1 / max(|a|, eps) cannot tell
  float* normb;
  const float* g;   // bwd: [B*H*W] upstream gradient of cosv
  float* da; float* db;  // bwd: same strides as a / b
};

template <bool WARP>
__global__ void __launch_bounds__(256) cosine_fwd_kernel(CosParams p) {
  const long long npix = 1ll * p.B * p.H * p.W;
  const int lane = threadIdx.x & 31;
  const long long pix = WARP ? (1ll * blockIdx.x * 8 + (threadIdx.x >> 5)) : (1ll * blockIdx.x * 256 + threadIdx.x);
  if (pix >= npix) return;
  const int x = static_cast<int>(pix % p.W), y = static_cast<int>((pix / p.W) % p.H), b = static_cast<int>(pix / (1ll * p.W * p.H));
  const float* pa = p.a + b * p.a_sb + y * p.a_sy + x * p.a_sx;
  const float* pb = p.b + b * p.b_sb + y * p.b_sy + x * p.b_sx;
  float saa = 0.f, sbb = 0.f, sab = 0.f;
  for (int c = WARP ? lane : 0; c < p.C; c += WARP ? 32 : 1) {
    const float va = pa[c * p.a_sc], vb = pb[c * p.b_sc];
    saa = fmaf(va, va, saa);
    sbb = fmaf(vb, vb, sbb);
    sab = fmaf(va, vb, sab);
  }
  if (WARP) { saa = warp_sum(saa); sbb = warp_sum(sbb); sab = warp_sum(sab); }
  const float na = sqrtf(saa), nb = sqrtf(sbb);
  const float ia = 1.0f / fmaxf(na, p.eps), ib = 1.0f / fmaxf(nb, p.eps);
  if (!WARP || lane == 0) {
    p.cosv[pix] = sab * ia * ib;
    p.norma[pix] = na;
    p.normb[pix] = nb;
  }
}

// the gradient formulas are CosineGrad's (cosine.cuh)
template <bool WARP>
__global__ void __launch_bounds__(256) cosine_bwd_kernel(CosParams p) {
  const long long npix = 1ll * p.B * p.H * p.W;
  const int lane = threadIdx.x & 31;
  const long long pix = WARP ? (1ll * blockIdx.x * 8 + (threadIdx.x >> 5)) : (1ll * blockIdx.x * 256 + threadIdx.x);
  if (pix >= npix) return;
  const int x = static_cast<int>(pix % p.W), y = static_cast<int>((pix / p.W) % p.H), b = static_cast<int>(pix / (1ll * p.W * p.H));
  const long long oa = b * p.a_sb + y * p.a_sy + x * p.a_sx, ob = b * p.b_sb + y * p.b_sy + x * p.b_sx;
  const float g = p.g[pix], cs = p.cosv[pix], na = p.norma[pix], nb = p.normb[pix];
  const CosineGrad cg(cs, na, nb, p.eps);
  for (int c = WARP ? lane : 0; c < p.C; c += WARP ? 32 : 1) {
    const float va = p.a[oa + c * p.a_sc], vb = p.b[ob + c * p.b_sc];
    if (p.da) p.da[oa + c * p.a_sc] = cg.da(g, va, vb);
    if (p.db) p.db[ob + c * p.b_sc] = cg.db(g, va, vb);
  }
}

}  // namespace stego

using namespace stego;

// cosv / norma / normb: [B*H*W] floats each (cosv is the result, the unclamped fp32 norms are saved for the backward).
extern "C" int stego_cosine_fwd(const float* a, long long a_sb, long long a_sc, long long a_sy, long long a_sx, const float* b,
                                long long b_sb, long long b_sc, long long b_sy, long long b_sx, int B, int C, int H, int W,
                                float eps, float* cosv, float* norma, float* normb, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(a && b && cosv && norma && normb, "stego_cosine_fwd: null pointer");
  STEGO_CHECK_ARG(B > 0 && C > 0 && H > 0 && W > 0 && eps > 0.f, "stego_cosine_fwd: bad sizes");
  CosParams p;
  p.a = a; p.a_sb = a_sb; p.a_sc = a_sc; p.a_sy = a_sy; p.a_sx = a_sx;
  p.b = b; p.b_sb = b_sb; p.b_sc = b_sc; p.b_sy = b_sy; p.b_sx = b_sx;
  p.B = B; p.C = C; p.H = H; p.W = W; p.eps = eps; p.cosv = cosv; p.norma = norma; p.normb = normb;
  p.g = nullptr; p.da = nullptr; p.db = nullptr;
  const long long npix = 1ll * B * H * W;
  if (a_sc == 1 && b_sc == 1) {
    cosine_fwd_kernel<true><<<(unsigned)((npix + 7) / 8), 256, 0, stream>>>(p);
  } else {
    cosine_fwd_kernel<false><<<(unsigned)((npix + 255) / 256), 256, 0, stream>>>(p);
  }
  STEGO_CHECK_LAUNCH("cosine_fwd_kernel");
  return STEGO_OK;
}

// grad_cos [B*H*W]; da / db (either may be null) are written with the strides of a / b.
extern "C" int stego_cosine_bwd(const float* a, long long a_sb, long long a_sc, long long a_sy, long long a_sx, const float* b,
                                long long b_sb, long long b_sc, long long b_sy, long long b_sx, int B, int C, int H, int W,
                                float eps, const float* cosv, const float* norma, const float* normb, const float* grad_cos,
                                float* da, float* db, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(a && b && cosv && norma && normb && grad_cos && (da || db), "stego_cosine_bwd: null pointer");
  STEGO_CHECK_ARG(B > 0 && C > 0 && H > 0 && W > 0 && eps > 0.f, "stego_cosine_bwd: bad sizes");
  CosParams p;
  p.a = a; p.a_sb = a_sb; p.a_sc = a_sc; p.a_sy = a_sy; p.a_sx = a_sx;
  p.b = b; p.b_sb = b_sb; p.b_sc = b_sc; p.b_sy = b_sy; p.b_sx = b_sx;
  p.B = B; p.C = C; p.H = H; p.W = W; p.eps = eps;
  p.cosv = const_cast<float*>(cosv); p.norma = const_cast<float*>(norma); p.normb = const_cast<float*>(normb);
  p.g = grad_cos; p.da = da; p.db = db;
  const long long npix = 1ll * B * H * W;
  if (a_sc == 1 && b_sc == 1) {
    cosine_bwd_kernel<true><<<(unsigned)((npix + 7) / 8), 256, 0, stream>>>(p);
  } else {
    cosine_bwd_kernel<false><<<(unsigned)((npix + 255) / 256), 256, 0, stream>>>(p);
  }
  STEGO_CHECK_LAUNCH("cosine_bwd_kernel");
  return STEGO_OK;
}
