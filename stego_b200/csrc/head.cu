// Elementwise / reduction helpers around the segmentation-head GEMMs (sm_90a, HBM-bound).
//
// Reference: src/modules.py:108-118 (DinoFeaturizer.forward tail):
//     code = cluster1(dropout(f)) + cluster2(dropout(f));  return dropout(f), code
// The three Dropout2d calls each draw an independent [B,C,1,1] Bernoulli noise; here one pass over the
// frozen features applies all three masks (the reference re-reads the feature map three times).
// The 1x1 convs themselves run on the wgmma GEMM (gemm.cu); this file supplies what sits between
// GEMMs in forward and backward: mask application, fp32->bf16 operand packing, ReLU backward and the
// bias-gradient column sums, and the fused Adam update (torch.optim.Adam semantics,
// src/train_segmentation.py:373-383).
#include "common.cuh"
#include "host_util.h"

namespace stego {

// feat [B*hw][E] bf16 (tokens-major); masks [B][E] fp32 or null; outs [B*hw][E] bf16 or null.
__global__ void __launch_bounds__(256)
dropout3_kernel(const bf16* __restrict__ feat, const float* __restrict__ m1, const float* __restrict__ m2,
                const float* __restrict__ m3, bf16* __restrict__ o1, bf16* __restrict__ o2, bf16* __restrict__ o3,
                long long rows, int hw, int E) {
  const int vec_per_row = E / 8;
  const long long idx = 1ll * blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * vec_per_row) return;
  const long long row = idx / vec_per_row;
  const int c0 = static_cast<int>(idx % vec_per_row) * 8;
  const int b = static_cast<int>(row / hw);
  const uint4 raw = *reinterpret_cast<const uint4*>(feat + row * E + c0);
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&raw);
  float x[8];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 f = __bfloat1622float2(h[i]);
    x[2 * i] = f.x;
    x[2 * i + 1] = f.y;
  }
  auto emit = [&](const float* m, bf16* o) {
    if (!o) return;
    const float4 ma = *reinterpret_cast<const float4*>(m + 1ll * b * E + c0);
    const float4 mb = *reinterpret_cast<const float4*>(m + 1ll * b * E + c0 + 4);
    uint4 w;
    w.x = pack_bf16x2(x[0] * ma.x, x[1] * ma.y);
    w.y = pack_bf16x2(x[2] * ma.z, x[3] * ma.w);
    w.z = pack_bf16x2(x[4] * mb.x, x[5] * mb.y);
    w.w = pack_bf16x2(x[6] * mb.z, x[7] * mb.w);
    *reinterpret_cast<uint4*>(o + row * E + c0) = w;
  };
  emit(m1, o1);
  emit(m2, o2);
  emit(m3, o3);
}

// fp32 [rows][ld_in] (first C columns) -> bf16 [rows][ld_out], zero padded to ld_out columns.
__global__ void __launch_bounds__(256)
cast_pad_kernel(const float* __restrict__ in, int ld_in, int C, bf16* __restrict__ out, int ld_out, long long rows) {
  const long long idx = 1ll * blockIdx.x * blockDim.x + threadIdx.x;
  const int pairs = ld_out / 2;
  if (idx >= rows * pairs) return;
  const long long row = idx / pairs;
  const int c = static_cast<int>(idx % pairs) * 2;
  const float a = (c < C) ? in[row * ld_in + c] : 0.f;
  const float b = (c + 1 < C) ? in[row * ld_in + c + 1] : 0.f;
  *reinterpret_cast<uint32_t*>(out + row * ld_out + c) = pack_bf16x2(a, b);
}

// dh_out = bf16( dh_in * (h > 0) ), all [rows][E]
__global__ void __launch_bounds__(256)
relu_bwd_kernel(const float* __restrict__ dh, const bf16* __restrict__ h, bf16* __restrict__ out, long long n4) {
  const long long idx = 1ll * blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n4) return;
  const float4 g = reinterpret_cast<const float4*>(dh)[idx];
  const uint2 hv = reinterpret_cast<const uint2*>(h)[idx];
  const __nv_bfloat162* hp = reinterpret_cast<const __nv_bfloat162*>(&hv);
  const float2 h0 = __bfloat1622float2(hp[0]), h1 = __bfloat1622float2(hp[1]);
  uint2 w;
  w.x = pack_bf16x2(h0.x > 0.f ? g.x : 0.f, h0.y > 0.f ? g.y : 0.f);
  w.y = pack_bf16x2(h1.x > 0.f ? g.z : 0.f, h1.y > 0.f ? g.w : 0.f);
  reinterpret_cast<uint2*>(out)[idx] = w;
}

// out[c] += sum over rows of in[row][c].  One warp per 32-row chunk; each lane owns 16-byte column groups
// (8 bf16 / 4 fp32) so a row is read with full-width coalesced loads; block-level combine in shared memory, one
// atomic per (block, column).  Requires ld * sizeof(T) % 16 == 0 and a 16-byte aligned base (checked on the host).
template <typename T, int NG>  // NG = ceil(C / (32 * V)), V = 16 / sizeof(T)
__global__ void __launch_bounds__(256)
colsum_kernel(const T* __restrict__ in, int ld, int C, long long rows, float* __restrict__ out) {
  constexpr int V = 16 / sizeof(T);
  __shared__ float part[8][NG * 32 * V];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long r0 = (1ll * blockIdx.x * 8 + warp) * 32;
  float acc[NG][V];
#pragma unroll
  for (int g = 0; g < NG; ++g)
#pragma unroll
    for (int v = 0; v < V; ++v) acc[g][v] = 0.f;
  for (long long r = r0; r < r0 + 32 && r < rows; ++r) {
#pragma unroll
    for (int g = 0; g < NG; ++g) {
      const int c = (lane + 32 * g) * V;
      if (c < C) {  // C % V == 0 is guaranteed by the host for this path
        const uint4 raw = *reinterpret_cast<const uint4*>(in + r * ld + c);
        if constexpr (sizeof(T) == 2) {
          const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&raw);
#pragma unroll
          for (int v = 0; v < 4; ++v) {
            const float2 f = __bfloat1622float2(h[v]);
            acc[g][2 * v] += f.x;
            acc[g][2 * v + 1] += f.y;
          }
        } else {
          const float* f = reinterpret_cast<const float*>(&raw);
#pragma unroll
          for (int v = 0; v < 4; ++v) acc[g][v] += f[v];
        }
      }
    }
  }
#pragma unroll
  for (int g = 0; g < NG; ++g)
#pragma unroll
    for (int v = 0; v < V; ++v) part[warp][(lane + 32 * g) * V + v] = acc[g][v];
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += part[w][c];
    atomicAdd(out + c, t);
  }
}

// scalar fallback (any C / alignment): one thread per column, row chunk per blockIdx.y
template <typename T>
__global__ void __launch_bounds__(128)
colsum_scalar_kernel(const T* __restrict__ in, int ld, int C, long long rows, int rows_per_block, float* __restrict__ out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const long long r0 = 1ll * blockIdx.y * rows_per_block;
  const long long r1 = (r0 + rows_per_block < rows) ? r0 + rows_per_block : rows;
  float acc = 0.f;
  for (long long r = r0; r < r1; ++r) {
    if constexpr (sizeof(T) == 2) acc += __bfloat162float(in[r * ld + c]);
    else acc += in[r * ld + c];
  }
  atomicAdd(out + c, acc);
}

// torch.optim.Adam (amsgrad=False, weight_decay=0, maximize=False): step is 1-based.
__global__ void __launch_bounds__(256)
adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
            long long n, float lr, float b1, float b2, float eps, float bc1, float sqrt_bc2, float grad_scale) {
  const long long i = 1ll * blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float gi = g[i] * grad_scale;
  const float mi = m[i] * b1 + (1.f - b1) * gi;
  const float vi = v[i] * b2 + (1.f - b2) * gi * gi;
  m[i] = mi;
  v[i] = vi;
  const float denom = sqrtf(vi) / sqrt_bc2 + eps;
  p[i] -= (lr / bc1) * (mi / denom);
}

}  // namespace stego

using namespace stego;

extern "C" int stego_head_dropout3(const void* feat_bf16, const float* mask1, const float* mask2, const float* mask3,
                                   void* out1, void* out2, void* out3, int B, int hw, int E, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(feat_bf16 && B > 0 && hw > 0 && E % 8 == 0, "stego_head_dropout3: bad args");
  STEGO_CHECK_ARG((!out1 || mask1) && (!out2 || mask2) && (!out3 || mask3), "stego_head_dropout3: output without mask");
  const long long rows = 1ll * B * hw;
  const long long n = rows * (E / 8);
  dropout3_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(
      reinterpret_cast<const bf16*>(feat_bf16), mask1, mask2, mask3, reinterpret_cast<bf16*>(out1),
      reinterpret_cast<bf16*>(out2), reinterpret_cast<bf16*>(out3), rows, hw, E);
  STEGO_CHECK_LAUNCH("dropout3_kernel");
  return STEGO_OK;
}

extern "C" int stego_cast_pad_bf16(const float* in, int ld_in, int C, void* out_bf16, int ld_out, long long rows,
                                   void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(in && out_bf16 && C > 0 && C <= ld_in && C <= ld_out && ld_out % 2 == 0 && rows > 0,
                  "stego_cast_pad_bf16: bad args");
  const long long n = rows * (ld_out / 2);
  cast_pad_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(in, ld_in, C, reinterpret_cast<bf16*>(out_bf16),
                                                                   ld_out, rows);
  STEGO_CHECK_LAUNCH("cast_pad_kernel");
  return STEGO_OK;
}

extern "C" int stego_relu_bwd_bf16(const float* dh, const void* h_bf16, void* out_bf16, long long n, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(dh && h_bf16 && out_bf16 && n > 0 && n % 4 == 0, "stego_relu_bwd_bf16: bad args");
  const long long n4 = n / 4;
  relu_bwd_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, stream>>>(dh, reinterpret_cast<const bf16*>(h_bf16),
                                                                    reinterpret_cast<bf16*>(out_bf16), n4);
  STEGO_CHECK_LAUNCH("relu_bwd_kernel");
  return STEGO_OK;
}

// out[C] (fp32) += column sums of in [rows][ld]; in_is_bf16 selects the element type.
extern "C" int stego_colsum(const void* in, int in_is_bf16, int ld, int C, long long rows, float* out, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(in && out && C > 0 && C <= ld && rows > 0, "stego_colsum: bad args");
  const size_t esz = in_is_bf16 ? 2 : 4;
  const int V = (int)(16 / esz);
  const bool vec_ok = (reinterpret_cast<uintptr_t>(in) & 15u) == 0 && (size_t(ld) * esz) % 16 == 0 && C % V == 0 &&
                      C <= (in_is_bf16 ? 768 : 384);
  if (vec_ok) {
    const unsigned blocks = (unsigned)((rows + 255) / 256);
    const int ng = (C + 32 * V - 1) / (32 * V);
    if (in_is_bf16) {
      const bf16* p = reinterpret_cast<const bf16*>(in);
      if (ng <= 1) colsum_kernel<bf16, 1><<<blocks, 256, 0, stream>>>(p, ld, C, rows, out);
      else if (ng <= 2) colsum_kernel<bf16, 2><<<blocks, 256, 0, stream>>>(p, ld, C, rows, out);
      else colsum_kernel<bf16, 3><<<blocks, 256, 0, stream>>>(p, ld, C, rows, out);
    } else {
      const float* p = reinterpret_cast<const float*>(in);
      if (ng <= 1) colsum_kernel<float, 1><<<blocks, 256, 0, stream>>>(p, ld, C, rows, out);
      else if (ng <= 2) colsum_kernel<float, 2><<<blocks, 256, 0, stream>>>(p, ld, C, rows, out);
      else colsum_kernel<float, 3><<<blocks, 256, 0, stream>>>(p, ld, C, rows, out);
    }
  } else {
    const int rpb = 512;
    dim3 grid((C + 127) / 128, (unsigned)((rows + rpb - 1) / rpb));
    if (in_is_bf16)
      colsum_scalar_kernel<bf16><<<grid, 128, 0, stream>>>(reinterpret_cast<const bf16*>(in), ld, C, rows, rpb, out);
    else
      colsum_scalar_kernel<float><<<grid, 128, 0, stream>>>(reinterpret_cast<const float*>(in), ld, C, rows, rpb, out);
  }
  STEGO_CHECK_LAUNCH("colsum_kernel");
  return STEGO_OK;
}

namespace stego {
struct StepLossParams {
  const float* stats;  // [ncalls][4] from stego_corr_loss_fwd
  int ncalls;
  float w[16];         // weight of each call's mean loss in the total
  const float* extra0; // optional device scalars added to the total (linear / cluster probe losses)
  const float* extra1;
  float* out;          // [4]: total, weighted correspondence term, mean loss of calls 2.., mean cd of calls 2..
};
__global__ void step_losses_kernel(StepLossParams p) {
  if (threadIdx.x != 0) return;
  float corr = 0.f, neg = 0.f, negcd = 0.f;
  for (int c = 0; c < p.ncalls; ++c) {
    corr += p.w[c] * p.stats[c * 4];
    if (c >= 2) { neg += p.stats[c * 4]; negcd += p.stats[c * 4 + 1]; }
  }
  const int nn = p.ncalls > 2 ? p.ncalls - 2 : 1;
  float total = corr;
  if (p.extra0) total += p.extra0[0];
  if (p.extra1) total += p.extra1[0];
  p.out[0] = total; p.out[1] = corr; p.out[2] = neg / nn; p.out[3] = negcd / nn;
}
}  // namespace stego

extern "C" int stego_step_losses(const float* corr_stats, int ncalls, const float* call_weights_host,
                                 const float* extra0, const float* extra1, float* out4, void* stream_) {
  STEGO_CHECK_ARG(corr_stats && call_weights_host && out4, "stego_step_losses: null pointer");
  STEGO_CHECK_ARG(ncalls >= 1 && ncalls <= 16, "stego_step_losses: ncalls=%d (1..16)", ncalls);
  stego::StepLossParams p;
  p.stats = corr_stats; p.ncalls = ncalls; p.extra0 = extra0; p.extra1 = extra1; p.out = out4;
  for (int c = 0; c < 16; ++c) p.w[c] = c < ncalls ? call_weights_host[c] : 0.f;
  stego::step_losses_kernel<<<1, 32, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(p);
  STEGO_CHECK_LAUNCH("step_losses_kernel launch");
  return stego::STEGO_OK;
}

extern "C" int stego_adam_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, long long n,
                               float lr, float beta1, float beta2, float eps, int step, float grad_scale,
                               void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(param && grad && exp_avg && exp_avg_sq && n > 0 && step >= 1, "stego_adam_step: bad args");
  const double bc1 = 1.0 - pow((double)beta1, (double)step);
  const double bc2 = 1.0 - pow((double)beta2, (double)step);
  adam_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(param, grad, exp_avg, exp_avg_sq, n, lr, beta1, beta2,
                                                               eps, (float)bc1, (float)sqrt(bc2), grad_scale);
  STEGO_CHECK_LAUNCH("adam_kernel");
  return STEGO_OK;
}
