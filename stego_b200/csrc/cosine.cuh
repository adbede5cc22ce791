// The gradient of cos = <normalize(a), normalize(b)> (F.normalize, eps clamp) from the forward's saved cosine and
// unclamped norms.  Shared by the per-pixel cosine backward (cosine_loss.cu) and the reconstruction term's backward
// (rec_loss.cu), which recomputes `a` (the decoder output) instead of reading it.
#pragma once
#include <cuda_runtime.h>

namespace stego {

// d cos / d a = ib * (ia * b - [|a| >= eps] * cos * ia^2 * a) ... written with the saved norms, ia = 1 / max(|a|, eps)
// recomputed from them (the forward's bits):
//   a_hat = a * ia, b_hat = b * ib, cos = <a_hat, b_hat>
//   |a| >= eps:  d cos / d a = ia * (b_hat - cos * a_hat)        |a| < eps (ia = 1/eps constant):  d cos / d a = ia * b_hat
// F.normalize's clamp_min passes the gradient at |a| == eps too, which the inverse alone cannot tell from |a| < eps.
struct CosineGrad {
  float ia, ib, ka, kb;
  __device__ __forceinline__ CosineGrad(float cs, float na, float nb, float eps)
      : ia(1.0f / fmaxf(na, eps)), ib(1.0f / fmaxf(nb, eps)), ka((na >= eps) ? cs : 0.f), kb((nb >= eps) ? cs : 0.f) {}
  // g x d cos / d a and g x d cos / d b for one channel with values a, b
  __device__ __forceinline__ float da(float g, float a, float b) const {
    const float ah = a * ia, bh = b * ib;
    return g * ia * (bh - ka * ah);
  }
  __device__ __forceinline__ float db(float g, float a, float b) const {
    const float ah = a * ia, bh = b * ib;
    return g * ib * (ah - kb * bh);
  }
};

}  // namespace stego
