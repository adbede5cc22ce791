// Bandwidth-bound pieces of the frozen DINO ViT forward (reference: src/dino/vision_transformer.py):
//   patchify      : NCHW fp32 image -> im2col rows [B*hw][3*P*P] bf16  (PatchEmbed conv, :127-131, as a GEMM operand),
//                   optionally followed by the rows of the mirrored images (flip-TTA)
//   cls rows      : x[b,0,:] = cls_token + pos_embed[0]                 (prepare_tokens, :203-207)
//   layernorm     : fp32 residual stream -> bf16 GEMM operand            (Block norm1/norm2 :107,111; final norm :234)
// The residual stream is kept in fp32 (the reference computes in fp32); GEMM operands are bf16.
// All kernels are HBM-bound: 16-byte vector accesses, one warp per row, no shared memory needed.
#include "common.cuh"
#include "host_util.h"

namespace stego {

// ---------------------------------------------------------------------------------------------
// patchify: one thread per (patch, channel, ky): reads P contiguous pixels, writes P bf16.
// column order c*P*P + ky*P + kx == flattening of the conv weight [E][3][P][P].
// MIRROR: the rows of 2B images are written, images B..2B-1 being img.flip(3) (the flip-TTA frames of
// eval_segmentation.py:125): patch column px reads source patch fw-1-px with its P pixels in reverse order, so the
// mirrored batch is never materialised.  The values are the same bits as patchify of the flipped image.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t swap_bf16x2(uint32_t v) { return __byte_perm(v, 0, 0x1032); }

template <int P, typename T, bool MIRROR>
__global__ void patchify_kernel(const T* __restrict__ img, bf16* __restrict__ out, int B, int H, int W) {
  const int fh = H / P, fw = W / P;
  const long long total = 1ll * (MIRROR ? 2 * B : B) * fh * fw * 3 * P;
  const long long idx = 1ll * blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int ky = idx % P;
  const int c = (idx / P) % 3;
  const long long patch = idx / (3 * P);
  const int px = patch % fw;
  const int py = (patch / fw) % fh;
  const int b = patch / (1ll * fw * fh);
  const bool flip = MIRROR && b >= B;
  const int sb = flip ? b - B : b, sx = flip ? fw - 1 - px : px;
  const T* src = img + ((1ll * sb * 3 + c) * H + (py * P + ky)) * W + sx * P;
  bf16* dst = out + patch * (3 * P * P) + c * P * P + ky * P;
  static_assert(P == 8 || P == 16, "patch size");
#pragma unroll
  for (int v = 0; v < P / 8; ++v) {
    const int sv = flip ? P / 8 - 1 - v : v;  // 8-pixel group of the source; reversed inside below when flipped
    uint4 w;
    if constexpr (sizeof(T) == 2) {
      // bf16 image (already the precision the GEMM operand has): a straight 16-byte copy
      w = *reinterpret_cast<const uint4*>(src + sv * 8);
    } else {
      const float4 a = *reinterpret_cast<const float4*>(src + sv * 8);
      const float4 b4 = *reinterpret_cast<const float4*>(src + sv * 8 + 4);
      w.x = pack_bf16x2(a.x, a.y);
      w.y = pack_bf16x2(a.z, a.w);
      w.z = pack_bf16x2(b4.x, b4.y);
      w.w = pack_bf16x2(b4.z, b4.w);
    }
    if (flip) w = make_uint4(swap_bf16x2(w.w), swap_bf16x2(w.z), swap_bf16x2(w.y), swap_bf16x2(w.x));
    *reinterpret_cast<uint4*>(dst + v * 8) = w;
  }
}

__global__ void cls_rows_kernel(float* __restrict__ x, const float* __restrict__ cls, const float* __restrict__ pos,
                                int B, int ntok, int E) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * E) return;
  const int b = i / E, e = i % E;
  x[(1ll * b * ntok) * E + e] = cls[e] + pos[e];
}

// ---------------------------------------------------------------------------------------------
// LayerNorm: one warp per row, row held in registers (E = 128*V4 floats), two-pass statistics.
// drop_cls > 0: rows are tokens of images with `drop_cls` tokens each; token 0 (cls) is skipped and
// the output is packed tokens-major [B][ntok-1][E] (modules.py:97 drops the cls token).
// ---------------------------------------------------------------------------------------------
template <int V4>
__global__ void __launch_bounds__(256)
layernorm_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                 bf16* __restrict__ out, int rows, float eps, int drop_cls) {
  constexpr int E = V4 * 128;
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  long long orow = row;
  if (drop_cls > 0) {
    const int t = row % drop_cls;
    if (t == 0) return;
    orow = 1ll * (row / drop_cls) * (drop_cls - 1) + (t - 1);
  }
  const float4* xr = reinterpret_cast<const float4*>(x + 1ll * row * E);
  float4 v[V4];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < V4; ++i) {
    v[i] = xr[lane + 32 * i];
    s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
  }
  // __fmul_rn: the mean is rounded once and every `x - mean` subtracts that value.  A plain `sum * (1/E)` is contracted
  // into each `x - mean` as fma(sum, -1/E, x), which keeps the error of the inexact 1/E (E = 384, 768) unrounded, so a
  // constant row did not centre to exactly 0 and came out as beta - 1e-4 gamma instead of beta.
  const float mean = __fmul_rn(warp_sum(s), 1.0f / E);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < V4; ++i) {
    const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
    q += (a * a + b * b) + (c * c + d * d);
  }
  const float rstd = rsqrtf(warp_sum(q) * (1.0f / E) + eps);
  const float4* g4 = reinterpret_cast<const float4*>(gamma);
  const float4* b4 = reinterpret_cast<const float4*>(beta);
  uint2* o = reinterpret_cast<uint2*>(out + orow * E);
#pragma unroll
  for (int i = 0; i < V4; ++i) {
    const float4 g = __ldg(g4 + lane + 32 * i);
    const float4 bb = __ldg(b4 + lane + 32 * i);
    uint2 w;
    w.x = pack_bf16x2((v[i].x - mean) * rstd * g.x + bb.x, (v[i].y - mean) * rstd * g.y + bb.y);
    w.y = pack_bf16x2((v[i].z - mean) * rstd * g.z + bb.z, (v[i].w - mean) * rstd * g.w + bb.w);
    o[lane + 32 * i] = w;
  }
}

// ---------------------------------------------------------------------------------------------
// Final LayerNorm fused with the global average pool of src/precompute_knns.py:19
//     feats = model(img).mean([2, 3])          (model(img) = norm(x)[:, 1:] viewed as [B, E, h, w], src/modules.py:97)
// One CTA of 8 warps per (image, chunk of patch tokens): every warp normalises its rows (cls token skipped) and keeps
// per-channel running sums in registers; the CTA reduces them through shared memory and adds sum / (ntok - 1) to
// out[b][E] with one atomic per channel.  The [B, hw, E] feature map is never written.
// ---------------------------------------------------------------------------------------------
template <int V4>
__global__ void __launch_bounds__(256)
layernorm_gap_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                     float* __restrict__ out, int ntok, float eps, int rows_per_cta) {
  constexpr int E = V4 * 128;
  __shared__ float4 red[8][V4 * 32];
  const int b = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int t0 = 1 + blockIdx.x * rows_per_cta;  // token 0 is the cls token
  const int t1 = min(ntok, t0 + rows_per_cta);
  const float4* g4 = reinterpret_cast<const float4*>(gamma);
  float4 g[V4], acc[V4];
#pragma unroll
  for (int i = 0; i < V4; ++i) {
    g[i] = __ldg(g4 + lane + 32 * i);
    acc[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  int nrows = 0;
  for (int t = t0 + warp; t < t1; t += 8) {
    const float4* xr = reinterpret_cast<const float4*>(x + (1ll * b * ntok + t) * E);
    float4 v[V4];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < V4; ++i) {
      v[i] = xr[lane + 32 * i];
      s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    }
    const float mean = __fmul_rn(warp_sum(s), 1.0f / E);  // rounded once, as in layernorm_kernel
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < V4; ++i) {
      const float a = v[i].x - mean, bq = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
      q += (a * a + bq * bq) + (c * c + d * d);
    }
    const float rstd = rsqrtf(warp_sum(q) * (1.0f / E) + eps);
#pragma unroll
    for (int i = 0; i < V4; ++i) {  // beta is added once per row at the end (rows counted in nrows)
      acc[i].x += (v[i].x - mean) * rstd * g[i].x;
      acc[i].y += (v[i].y - mean) * rstd * g[i].y;
      acc[i].z += (v[i].z - mean) * rstd * g[i].z;
      acc[i].w += (v[i].w - mean) * rstd * g[i].w;
    }
    ++nrows;
  }
#pragma unroll
  for (int i = 0; i < V4; ++i) red[warp][lane + 32 * i] = acc[i];
  __shared__ int cnt[8];
  if (lane == 0) cnt[warp] = nrows;
  __syncthreads();
  const float inv = 1.0f / (ntok - 1);
  int total = 0;
#pragma unroll
  for (int w = 0; w < 8; ++w) total += cnt[w];
  for (int c4 = threadIdx.x; c4 < V4 * 32; c4 += blockDim.x) {
    float4 sum = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int w = 0; w < 8; ++w) {
      const float4 r = red[w][c4];
      sum.x += r.x; sum.y += r.y; sum.z += r.z; sum.w += r.w;
    }
    const float4 bb = __ldg(reinterpret_cast<const float4*>(beta) + c4);
    float* o = out + 1ll * b * E + 4 * c4;
    atomicAdd(o + 0, (sum.x + total * bb.x) * inv);
    atomicAdd(o + 1, (sum.y + total * bb.y) * inv);
    atomicAdd(o + 2, (sum.z + total * bb.z) * inv);
    atomicAdd(o + 3, (sum.w + total * bb.w) * inv);
  }
}

// ---------------------------------------------------------------------------------------------
// out[b][n] = x[b] . w[n] + bias[n]: fp32 rows against bf16 weight rows, one warp per output element, 16-byte loads of
// 8 weights (and the 8 matching fp32 inputs) per lane, fp32 accumulation.  Used for the "KK" kNN descriptors: the mean
// of the last block's keys is the key projection of the mean of its LN1 outputs (the projection is linear), so the
// [B, hw, E] key map is never written.  Tiny (B x E x E): latency-bound, no shared memory.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
linear_rows_f32_kernel(const float* __restrict__ x, const bf16* __restrict__ w, int ldw, const float* __restrict__ bias,
                       float* __restrict__ out, int B, int N, int K) {
  const long long o = 1ll * blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (o >= 1ll * B * N) return;
  const int lane = threadIdx.x & 31;
  const int b = static_cast<int>(o / N), n = static_cast<int>(o % N);
  const float4* xr = reinterpret_cast<const float4*>(x + 1ll * b * K);
  const uint4* wr = reinterpret_cast<const uint4*>(w + 1ll * n * ldw);
  float acc = 0.f;
  for (int c = lane; c < K / 8; c += 32) {
    const uint4 wv = __ldg(wr + c);
    const float4 x0 = __ldg(xr + 2 * c), x1 = __ldg(xr + 2 * c + 1);
    const bf16* wb = reinterpret_cast<const bf16*>(&wv);
    acc = fmaf(x0.x, __bfloat162float(wb[0]), acc);
    acc = fmaf(x0.y, __bfloat162float(wb[1]), acc);
    acc = fmaf(x0.z, __bfloat162float(wb[2]), acc);
    acc = fmaf(x0.w, __bfloat162float(wb[3]), acc);
    acc = fmaf(x1.x, __bfloat162float(wb[4]), acc);
    acc = fmaf(x1.y, __bfloat162float(wb[5]), acc);
    acc = fmaf(x1.z, __bfloat162float(wb[6]), acc);
    acc = fmaf(x1.w, __bfloat162float(wb[7]), acc);
  }
  acc = warp_sum(acc);
  if (lane == 0) out[o] = acc + (bias ? bias[n] : 0.f);
}

}  // namespace stego

using namespace stego;

template <bool MIRROR>
static int launch_patchify(const void* img, int img_is_bf16, void* out_bf16, int B, int H, int W, int patch,
                           cudaStream_t stream) {
  const char* name = MIRROR ? "stego_vit_patchify_tta" : "stego_vit_patchify";
  STEGO_CHECK_ARG(img && out_bf16, "%s: null pointer", name);
  STEGO_CHECK_ARG(patch == 8 || patch == 16, "%s: patch size %d unsupported (8 or 16)", name, patch);
  STEGO_CHECK_ARG(B > 0 && H % patch == 0 && W % patch == 0 && W % 8 == 0, "%s: bad image %dx%dx%d", name, B, H, W);
  STEGO_CHECK_ARG((reinterpret_cast<uintptr_t>(img) & 15u) == 0, "%s: image not 16-byte aligned", name);
  const long long total = 1ll * (MIRROR ? 2 * B : B) * (H / patch) * (W / patch) * 3 * patch;
  const int threads = 256;
  const int blocks = (int)((total + threads - 1) / threads);
  bf16* out = reinterpret_cast<bf16*>(out_bf16);
  if (img_is_bf16) {
    const bf16* im = reinterpret_cast<const bf16*>(img);
    if (patch == 8) patchify_kernel<8, bf16, MIRROR><<<blocks, threads, 0, stream>>>(im, out, B, H, W);
    else patchify_kernel<16, bf16, MIRROR><<<blocks, threads, 0, stream>>>(im, out, B, H, W);
  } else {
    const float* im = reinterpret_cast<const float*>(img);
    if (patch == 8) patchify_kernel<8, float, MIRROR><<<blocks, threads, 0, stream>>>(im, out, B, H, W);
    else patchify_kernel<16, float, MIRROR><<<blocks, threads, 0, stream>>>(im, out, B, H, W);
  }
  STEGO_CHECK_LAUNCH("patchify_kernel");
  return STEGO_OK;
}

extern "C" int stego_vit_patchify(const float* img, void* out_bf16, int B, int H, int W, int patch, void* stream_) {
  return launch_patchify<false>(img, 0, out_bf16, B, H, W, patch, reinterpret_cast<cudaStream_t>(stream_));
}

// Same im2col for an image batch that is already bf16 (the GEMM operand precision): results are bit-identical to
// feeding the fp32 image whenever the fp32 image holds bf16-representable values, and the H2D copy is half the size.
extern "C" int stego_vit_patchify_bf16(const void* img_bf16, void* out_bf16, int B, int H, int W, int patch,
                                       void* stream_) {
  return launch_patchify<false>(img_bf16, 1, out_bf16, B, H, W, patch, reinterpret_cast<cudaStream_t>(stream_));
}

// The rows of the 2B images [img ; img.flip(3)] from the B images of img (fp32, or bf16 with img_is_bf16 = 1).
extern "C" int stego_vit_patchify_tta(const void* img, int img_is_bf16, void* out_bf16, int B, int H, int W, int patch,
                                      void* stream_) {
  return launch_patchify<true>(img, img_is_bf16, out_bf16, B, H, W, patch, reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int stego_vit_cls_rows(float* x, const float* cls_token, const float* pos_embed, int B, int ntok, int E,
                                  void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(x && cls_token && pos_embed && B > 0 && ntok > 0 && E > 0, "stego_vit_cls_rows: bad args");
  cls_rows_kernel<<<(B * E + 255) / 256, 256, 0, stream>>>(x, cls_token, pos_embed, B, ntok, E);
  STEGO_CHECK_LAUNCH("cls_rows_kernel");
  return STEGO_OK;
}

extern "C" int stego_layernorm_bf16(const float* x, const float* gamma, const float* beta, void* out_bf16, int rows,
                                    int E, float eps, int drop_cls_ntok, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(x && gamma && beta && out_bf16 && rows > 0, "stego_layernorm_bf16: bad args");
  STEGO_CHECK_ARG(drop_cls_ntok == 0 || rows % drop_cls_ntok == 0, "stego_layernorm_bf16: rows %% ntok != 0");
  const int warps = 8;
  const int blocks = (rows + warps - 1) / warps;
  bf16* o = reinterpret_cast<bf16*>(out_bf16);
  switch (E) {
    case 384: layernorm_kernel<3><<<blocks, warps * 32, 0, stream>>>(x, gamma, beta, o, rows, eps, drop_cls_ntok); break;
    case 768: layernorm_kernel<6><<<blocks, warps * 32, 0, stream>>>(x, gamma, beta, o, rows, eps, drop_cls_ntok); break;
    case 128: layernorm_kernel<1><<<blocks, warps * 32, 0, stream>>>(x, gamma, beta, o, rows, eps, drop_cls_ntok); break;
    case 192: /* vit_tiny: 1.5 x 128 — not a multiple */
    default:
      set_error("stego_layernorm_bf16: embed dim %d unsupported (128, 384, 768)", E);
      return STEGO_ERR_UNSUPPORTED;
  }
  STEGO_CHECK_LAUNCH("layernorm_kernel");
  return STEGO_OK;
}

// Final norm + GAP over the patch tokens (cls dropped): x fp32 [B][ntok][E] -> out fp32 [B][E] (zeroed by the caller).
extern "C" int stego_layernorm_gap(const float* x, const float* gamma, const float* beta, float* out, int B, int ntok,
                                   int E, float eps, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(x && gamma && beta && out && B > 0 && ntok > 1, "stego_layernorm_gap: bad args");
  const int rows_per_cta = 64;
  dim3 grid((ntok - 1 + rows_per_cta - 1) / rows_per_cta, B);
  switch (E) {
    case 384: layernorm_gap_kernel<3><<<grid, 256, 0, stream>>>(x, gamma, beta, out, ntok, eps, rows_per_cta); break;
    case 768: layernorm_gap_kernel<6><<<grid, 256, 0, stream>>>(x, gamma, beta, out, ntok, eps, rows_per_cta); break;
    case 128: layernorm_gap_kernel<1><<<grid, 256, 0, stream>>>(x, gamma, beta, out, ntok, eps, rows_per_cta); break;
    default:
      set_error("stego_layernorm_gap: embed dim %d unsupported (128, 384, 768)", E);
      return STEGO_ERR_UNSUPPORTED;
  }
  STEGO_CHECK_LAUNCH("layernorm_gap_kernel");
  return STEGO_OK;
}

// out fp32 [B][N] = x fp32 [B][K] . w bf16 [N][ldw]^T (+ bias fp32 [N]).
extern "C" int stego_linear_rows_f32(const float* x, const void* w_bf16, int ldw, const float* bias, float* out, int B,
                                     int N, int K, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(x && w_bf16 && out, "stego_linear_rows_f32: null pointer");
  STEGO_CHECK_ARG(B > 0 && N > 0 && K > 0 && K % 8 == 0, "stego_linear_rows_f32: bad sizes B=%d N=%d K=%d (K a multiple of 8)",
                  B, N, K);
  STEGO_CHECK_ARG(ldw >= K && ldw % 8 == 0, "stego_linear_rows_f32: ldw=%d (>= K, a multiple of 8)", ldw);
  STEGO_CHECK_ARG((reinterpret_cast<uintptr_t>(x) & 15u) == 0 && (reinterpret_cast<uintptr_t>(w_bf16) & 15u) == 0,
                  "stego_linear_rows_f32: x and w must be 16-byte aligned");
  const long long outputs = 1ll * B * N;
  const int warps = 8;
  const long long blocks = (outputs + warps - 1) / warps;
  STEGO_CHECK_ARG(blocks <= 0x7fffffffll, "stego_linear_rows_f32: B*N=%lld too large", outputs);
  linear_rows_f32_kernel<<<static_cast<unsigned>(blocks), warps * 32, 0, stream>>>(
      x, reinterpret_cast<const bf16*>(w_bf16), ldw, bias, out, B, N, K);
  STEGO_CHECK_LAUNCH("linear_rows_f32_kernel");
  return STEGO_OK;
}
