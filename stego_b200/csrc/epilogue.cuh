// Activation helpers shared by the GEMM epilogues (gemm.cu).
#pragma once
#include "common.cuh"

namespace stego {

// Exact (erf) GELU, nn.GELU default.  erf by Abramowitz-Stegun 7.1.26 (|abs err| < 1.5e-7): one rcp + one ex2 on
// the MUFU pipe and ~10 FMAs instead of the ~25-instruction erff — the fc1 epilogue is issue-bound otherwise.
__device__ __forceinline__ float gelu_erf(float x) {
  const float z = fabsf(x) * 0.70710678118654752f;
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;\n" : "=f"(t) : "f"(fmaf(0.3275911f, z, 1.0f)));  // MUFU.RCP, no Newton fix-up
  float poly = fmaf(t, 1.061405429f, -1.453152027f);
  poly = fmaf(poly, t, 1.421413741f);
  poly = fmaf(poly, t, -0.284496736f);
  poly = fmaf(poly, t, 0.254829592f);
  poly *= t;
  const float erf_abs = fmaf(-poly, ex2_approx(-1.4426950408889634f * z * z), 1.0f);
  return 0.5f * x * (1.0f + copysignf(erf_abs, x));
}

// bf16-output GELU, MUFU-free (the fc1 epilogue applies GELU to 77 M elements per layer; two MUFU ops per element
// made it MUFU-bound), eight elements in lock-step as four fp32 pairs, ~9 instructions per element instead of 13:
//   erf(|x|/sqrt2) ~ e = min(xc * Q(xc^2), 1), xc = min(|x|, 3.2*sqrt2), Q of degree 8 (minimax fit, |abs err| <
//   4.3e-5 in fp32 evaluation), and gelu(x) = 0.5 x (1 + sign(x) erf(|x|/sqrt2)) = h + |h| * e with h = x/2.
// The error on GELU is |h| times the erf error: at most ~1e-4 (near |x| = 4.5), an absolute error that does not grow
// with |x|.  The cap matters: at the clamp xc * Q(xc^2) is 1 + 2.7e-5, which without it made every x below -4.19
// positive, by an amount growing linearly in |x|.  With it, x below the clamp gives exactly 0 and x above exactly x.
__device__ __forceinline__ void gelu_erf_poly8(float* x) {
  uint64_t xc[4], u[4], q[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    xc[j] = pack_f32x2(fminf(fabsf(x[2 * j]), 4.525483399593904f), fminf(fabsf(x[2 * j + 1]), 4.525483399593904f));
    u[j] = mul_f32x2(xc[j], xc[j]);
    q[j] = fma_f32x2(u[j], pack_f32x2(7.28493733954992e-11f, 7.28493733954992e-11f),
                     pack_f32x2(-7.739619932988917e-09f, -7.739619932988917e-09f));
  }
#define STEGO_POLY_STEP(C) \
  _Pragma("unroll") for (int j = 0; j < 4; ++j) q[j] = fma_f32x2(q[j], u[j], pack_f32x2(C, C));
  STEGO_POLY_STEP(3.6041332307651457e-07f)
  STEGO_POLY_STEP(-9.764514095986007e-06f)
  STEGO_POLY_STEP(0.0001730121070631224f)
  STEGO_POLY_STEP(-0.0021448454598048446f)
  STEGO_POLY_STEP(0.01943352726774955f)
  STEGO_POLY_STEP(-0.13244709440462024f)
  STEGO_POLY_STEP(0.7977185244870058f)
#undef STEGO_POLY_STEP
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float e0, e1;
    unpack_f32x2(mul_f32x2(q[j], xc[j]), e0, e1);
    const uint64_t e = pack_f32x2(fminf(e0, 1.0f), fminf(e1, 1.0f));
    const float h0 = 0.5f * x[2 * j], h1 = 0.5f * x[2 * j + 1];
    const uint64_t r = fma_f32x2(pack_f32x2(fabsf(h0), fabsf(h1)), e, pack_f32x2(h0, h1));
    unpack_f32x2(r, x[2 * j], x[2 * j + 1]);
  }
}

}  // namespace stego
