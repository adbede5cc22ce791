// The reconstruction term of the training step (src/train_segmentation.py:183-187), fused:
//     r        = decoder(code)                          1x1 conv D -> E, fp32
//     f        = feats * m3                             the step's returned-feature dropout (modules.py:116)
//     rec_loss = -(normalize(r) * normalize(f)).sum(1).mean()      F.normalize eps 1e-10
// The forward never writes r: each CTA takes 32 pixel rows, streams the decoder weight through shared memory 64 output
// channels at a time, and keeps sum r^2, sum r f and sum f^2 per row in registers; it writes the cosine and the two norms
// per pixel (the mean is stego_aug_align_loss, a fixed-order fp64 sum).  The backward recomputes r chunk by chunk with the
// same arithmetic, forms d r with F.normalize's clamp rule (CosineGrad, cosine.cuh), adds d r . W to the code gradient
// (each row block has one owner CTA, so no atomics) and keeps per-CTA partials of dW / db that a second launch sums in a
// fixed order: the decoder gradient repeats bit for bit.  fp32 FMAs, not tensor cores: ~5 GFLOP per step at B = 32,
// ViT-S/8 224^2, and the decoder stays at the fp32 bars of the autograd path (the same choice as crf_loss.cu).
#include <cuda_bf16.h>

#include "common.cuh"
#include "cosine.cuh"
#include "host_util.h"

namespace stego {

constexpr int RL_ROWS = 32;  // pixel rows per block
constexpr int RL_EC = 64;    // decoder output channels per chunk
constexpr int RL_DMAX = 96;
constexpr int RL_WLD = 68;   // stride of the [D][64] weight tile and the [32][64] d r tile: 16-byte rows for the
                             // backward's float4 reads, conflict-free row-wise and in 8-lane float4 phases
constexpr int RL_CLD = 36;   // stride of the [D][32] code tile (16-byte aligned rows for the float4 reads)
constexpr float RL_EPS = 1e-10f;

struct RecParams {
  const float* code; long long ldc;           // [M][ldc] fp32, first D columns
  const __nv_bfloat16* feat; long long ldf;   // [M][ldf] bf16, first E columns
  const float* m3;                            // [M / hw][E] or null
  int hw;
  const float* weight; const float* bias;     // [E][D], [E]
  long long M; int E, D;
  float* cosv; float* nr; float* nf;          // [M]
  const float* dcos;                          // bwd: [1] d loss / d cos
  float* dcode; long long ldd;                // bwd: [M][ldd], accumulated into
  float* part;                                // bwd: [gridDim.x][E * D + E]
};

// floats of the code tile, which the backward reuses as the [32][D + 1] d code tile
__host__ __device__ constexpr int rec_code_tile_floats(int D) {
  return D * RL_CLD > RL_ROWS * (D + 1) ? D * RL_CLD : RL_ROWS * (D + 1);
}

// shared-memory floats of either kernel for code width D
__host__ __device__ constexpr int rec_smem_floats(int D) {
  return D * RL_WLD + rec_code_tile_floats(D) + RL_ROWS * RL_WLD + RL_EC + 3 * RL_ROWS;
}

struct RecSmem {
  float* Cs;   // [D][RL_CLD]   code rows, transposed, at offset 0 for the float4 reads (the backward reuses it as the
               //               [32][D + 1] d code tile)
  float* Ws;   // [D][RL_WLD]   weight chunk, transposed
  float* DRs;  // [32][RL_WLD]  d r of the chunk (backward)
  float* bs;   // [64]          bias chunk
  float* rs;   // [3][32]       per-row cos, |r|, |f| (backward)
  __device__ explicit RecSmem(float* sm, int D)
      : Cs(sm), Ws(sm + rec_code_tile_floats(D)), DRs(Ws + D * RL_WLD), bs(DRs + RL_ROWS * RL_WLD), rs(bs + RL_EC) {}
};

__device__ __forceinline__ void rec_load_weight_chunk(const RecParams& p, const RecSmem& s, int e0) {
  for (int i = threadIdx.x; i < RL_EC * p.D; i += blockDim.x) {
    const int e = i / p.D, d = i % p.D;
    s.Ws[d * RL_WLD + e] = (e0 + e < p.E) ? p.weight[1ll * (e0 + e) * p.D + d] : 0.f;
  }
  for (int e = threadIdx.x; e < RL_EC; e += blockDim.x) s.bs[e] = (e0 + e < p.E) ? p.bias[e0 + e] : 0.f;
}

__device__ __forceinline__ void rec_load_code(const RecParams& p, const RecSmem& s, long long row0) {
  for (int i = threadIdx.x; i < RL_ROWS * p.D; i += blockDim.x) {
    const int r = i / p.D, d = i % p.D;
    s.Cs[d * RL_CLD + r] = (row0 + r < p.M) ? p.code[(row0 + r) * p.ldc + d] : 0.f;
  }
}

// acc[i] = sum_d W[e0 + tx][d] code[row ty * 8 + i][d]: the thread's column of the chunk for its 8 rows.  Forward and
// backward run this same loop, so the recomputed r is the forward's r bit for bit.
__device__ __forceinline__ void rec_chunk_dot(const RecParams& p, const RecSmem& s, int tx, int ty, float (&acc)[8]) {
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  for (int d = 0; d < p.D; ++d) {
    const float w = s.Ws[d * RL_WLD + tx];
    const float4 c0 = *reinterpret_cast<const float4*>(s.Cs + d * RL_CLD + ty * 8);
    const float4 c1 = *reinterpret_cast<const float4*>(s.Cs + d * RL_CLD + ty * 8 + 4);
    const float c[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = fmaf(c[i], w, acc[i]);
  }
}

// f = feat * m3 at (row, e), as the reference's feats.float() * m3
__device__ __forceinline__ float rec_feature(const RecParams& p, int row, int e) {
  float f = __bfloat162float(p.feat[row * p.ldf + e]);
  if (p.m3) f = f * p.m3[1ll * (row / p.hw) * p.E + e];
  return f;
}

// grid: one CTA per 32 rows; 256 threads as 64 columns x 4 row groups of 8
__global__ void __launch_bounds__(256) rec_fwd_kernel(RecParams p) {
  extern __shared__ __align__(16) float sm[];
  const RecSmem s(sm, p.D);
  const int tx = threadIdx.x & 63, ty = threadIdx.x >> 6;
  const long long row0 = 1ll * blockIdx.x * RL_ROWS;
  rec_load_code(p, s, row0);
  float srr[8], srf[8], sff[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) srr[i] = srf[i] = sff[i] = 0.f;
  for (int e0 = 0; e0 < p.E; e0 += RL_EC) {
    __syncthreads();  // previous chunk consumed (and the code tile visible on the first pass)
    rec_load_weight_chunk(p, s, e0);
    __syncthreads();
    float acc[8];
    rec_chunk_dot(p, s, tx, ty, acc);
    if (e0 + tx < p.E) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const long long row = row0 + ty * 8 + i;
        if (row < p.M) {
          const float r = acc[i] + s.bs[tx], f = rec_feature(p, static_cast<int>(row), e0 + tx);
          srr[i] = fmaf(r, r, srr[i]);
          srf[i] = fmaf(r, f, srf[i]);
          sff[i] = fmaf(f, f, sff[i]);
        }
      }
    }
  }
  // rows ty * 8 + i: the two warps of a row group each hold 32 columns' sums; combined in a fixed order
  __shared__ float red[2][RL_ROWS][3];
  const int half = tx >> 5;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float a = warp_sum(srr[i]), b = warp_sum(srf[i]), c = warp_sum(sff[i]);
    if ((tx & 31) == 0) {
      red[half][ty * 8 + i][0] = a;
      red[half][ty * 8 + i][1] = b;
      red[half][ty * 8 + i][2] = c;
    }
  }
  __syncthreads();
  if (threadIdx.x < RL_ROWS && row0 + threadIdx.x < p.M) {
    const int r = threadIdx.x;
    const float rr = red[0][r][0] + red[1][r][0], rf = red[0][r][1] + red[1][r][1], ff = red[0][r][2] + red[1][r][2];
    const float na = sqrtf(rr), nb = sqrtf(ff);
    const float ia = 1.0f / fmaxf(na, RL_EPS), ib = 1.0f / fmaxf(nb, RL_EPS);
    p.cosv[row0 + r] = rf * ia * ib;
    p.nr[row0 + r] = na;
    p.nf[row0 + r] = nb;
  }
}

// grid: G CTAs; CTA g takes row blocks g, g + G, ... for every chunk of 64 decoder channels in turn.  Per chunk it keeps
// its dW / db partial in registers (thread: channel tx, code columns ty + 4k) and writes it to part[g] at the chunk's end.
__global__ void __launch_bounds__(256) rec_bwd_kernel(RecParams p) {
  extern __shared__ __align__(16) float sm[];
  const RecSmem s(sm, p.D);
  const int tx = threadIdx.x & 63, ty = threadIdx.x >> 6;
  const long long nblk = (p.M + RL_ROWS - 1) / RL_ROWS;
  const float g = p.dcos[0];
  constexpr int KW = RL_DMAX / 4, KC = RL_DMAX / 8;
  float* part = p.part + 1ll * blockIdx.x * (1ll * p.E * p.D + p.E);
  for (int e0 = 0; e0 < p.E; e0 += RL_EC) {
    float dw[KW], db = 0.f;
#pragma unroll
    for (int k = 0; k < KW; ++k) dw[k] = 0.f;
    __syncthreads();  // the previous chunk's tiles consumed
    rec_load_weight_chunk(p, s, e0);
    for (long long blk = blockIdx.x; blk < nblk; blk += gridDim.x) {
      const long long row0 = blk * RL_ROWS;
      rec_load_code(p, s, row0);
      if (threadIdx.x < RL_ROWS) {
        const long long row = row0 + threadIdx.x;
        const bool in = row < p.M;
        s.rs[threadIdx.x] = in ? p.cosv[row] : 0.f;
        s.rs[RL_ROWS + threadIdx.x] = in ? p.nr[row] : 0.f;
        s.rs[2 * RL_ROWS + threadIdx.x] = in ? p.nf[row] : 0.f;
      }
      __syncthreads();
      // d r of the chunk -> DRs
      float acc[8];
      rec_chunk_dot(p, s, tx, ty, acc);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int r = ty * 8 + i;
        const long long row = row0 + r;
        float dr = 0.f;
        if (row < p.M && e0 + tx < p.E) {
          const CosineGrad cg(s.rs[r], s.rs[RL_ROWS + r], s.rs[2 * RL_ROWS + r], RL_EPS);
          dr = cg.da(g, acc[i] + s.bs[tx], rec_feature(p, static_cast<int>(row), e0 + tx));
        }
        s.DRs[r * RL_WLD + tx] = dr;
      }
      __syncthreads();
      // dW[e][d] += sum_r dr[r][e] code[r][d];  db[e] += sum_r dr[r][e]
      for (int r = 0; r < RL_ROWS; r += 4) {
        const float d0 = s.DRs[r * RL_WLD + tx], d1 = s.DRs[(r + 1) * RL_WLD + tx];
        const float d2 = s.DRs[(r + 2) * RL_WLD + tx], d3 = s.DRs[(r + 3) * RL_WLD + tx];
#pragma unroll
        for (int k = 0; k < KW; ++k) {
          const int d = ty + 4 * k;
          if (d < p.D) {
            const float4 c = *reinterpret_cast<const float4*>(s.Cs + d * RL_CLD + r);
            dw[k] = fmaf(d3, c.w, fmaf(d2, c.z, fmaf(d1, c.y, fmaf(d0, c.x, dw[k]))));
          }
        }
      }
      if (ty == 0)
        for (int r = 0; r < RL_ROWS; ++r) db += s.DRs[r * RL_WLD + tx];
      // d code[r][d] = sum_e dr[r][e] W[e][d] over the chunk (thread: row lane, code columns warp + 8k)
      const int lr = threadIdx.x & 31, wd = threadIdx.x >> 5;
      float dc[KC];
#pragma unroll
      for (int k = 0; k < KC; ++k) dc[k] = 0.f;
      for (int e = 0; e < RL_EC; e += 4) {
        const float4 g4 = *reinterpret_cast<const float4*>(s.DRs + lr * RL_WLD + e);
#pragma unroll
        for (int k = 0; k < KC; ++k) {
          const int d = wd + 8 * k;
          if (d < p.D) {
            const float4 w4 = *reinterpret_cast<const float4*>(s.Ws + d * RL_WLD + e);
            dc[k] = fmaf(g4.w, w4.w, fmaf(g4.z, w4.z, fmaf(g4.y, w4.y, fmaf(g4.x, w4.x, dc[k]))));
          }
        }
      }
      __syncthreads();  // the code tile is consumed: it becomes the d code tile
      float* Dc = s.Cs;
#pragma unroll
      for (int k = 0; k < KC; ++k) {
        const int d = wd + 8 * k;
        if (d < p.D) Dc[lr * (p.D + 1) + d] = dc[k];
      }
      __syncthreads();
      for (int i = threadIdx.x; i < RL_ROWS * p.D; i += blockDim.x) {
        const int r = i / p.D, d = i % p.D;
        if (row0 + r < p.M) p.dcode[(row0 + r) * p.ldd + d] += Dc[r * (p.D + 1) + d];
      }
      __syncthreads();  // Dc / DRs consumed before the next block
    }
    if (e0 + tx < p.E) {
#pragma unroll
      for (int k = 0; k < KW; ++k) {
        const int d = ty + 4 * k;
        if (d < p.D) part[1ll * (e0 + tx) * p.D + d] = dw[k];
      }
      if (ty == 0) part[1ll * p.E * p.D + e0 + tx] = db;
    }
  }
}

// out[i] = sum over g = 0 .. G-1 of part[g][i], in that order: dW (E * D values), then db (E values)
__global__ void __launch_bounds__(256) rec_reduce_kernel(const float* part, int G, int E, int D, float* dweight,
                                                         float* dbias) {
  const long long n = 1ll * E * D + E, i = 1ll * blockIdx.x * 256 + threadIdx.x;
  if (i >= n) return;
  float s = 0.f;
  for (int g = 0; g < G; ++g) s += part[1ll * g * n + i];
  if (i < 1ll * E * D) dweight[i] = s;
  else dbias[i - 1ll * E * D] = s;
}

static int rec_bwd_grid(long long M) {
  const long long nblk = (M + RL_ROWS - 1) / RL_ROWS;
  const long long g = 2ll * num_sms();
  return static_cast<int>(nblk < g ? nblk : g);
}

static int rec_check(const float* code, long long ldc, const void* feat, long long ldf, int hw, const float* weight,
                     const float* bias, long long M, int E, int D, const char* who) {
  STEGO_CHECK_ARG(code && feat && weight && bias, "%s: null pointer", who);
  STEGO_CHECK_ARG(M >= 1 && E >= 1 && D >= 1 && D <= RL_DMAX && hw >= 1 && ldc >= D && ldf >= E && M < (1ll << 31),
                  "%s: M=%lld E=%d D=%d hw=%d ldc=%lld ldf=%lld unsupported (D <= 96)", who, M, E, D, hw, ldc, ldf);
  return STEGO_OK;
}

static RecParams rec_params(const float* code, long long ldc, const void* feat, long long ldf, const float* m3, int hw,
                            const float* weight, const float* bias, long long M, int E, int D, const float* cosv,
                            const float* nr, const float* nf) {
  RecParams p{};
  p.code = code; p.ldc = ldc; p.feat = reinterpret_cast<const __nv_bfloat16*>(feat); p.ldf = ldf; p.m3 = m3; p.hw = hw;
  p.weight = weight; p.bias = bias; p.M = M; p.E = E; p.D = D;
  p.cosv = const_cast<float*>(cosv); p.nr = const_cast<float*>(nr); p.nf = const_cast<float*>(nf);
  return p;
}

}  // namespace stego

using namespace stego;

// code: fp32 rows [M][ldc] (first D columns); feat: bf16 rows [M][ldf] (first E columns); m3: fp32 [M / hw][E] or null;
// weight [E][D], bias [E] fp32.  Writes cosv, nr = |r|, nf = |f| ([M] each; the norms unclamped, for the backward).
extern "C" int stego_rec_fwd(const float* code, long long ldc, const void* feat, long long ldf, const float* m3, int hw,
                             const float* weight, const float* bias, long long M, int E, int D, float* cosv, float* nr,
                             float* nf, void* stream_) {
  if (int rc = rec_check(code, ldc, feat, ldf, hw, weight, bias, M, E, D, "stego_rec_fwd")) return rc;
  STEGO_CHECK_ARG(cosv && nr && nf, "stego_rec_fwd: null pointer");
  const RecParams p = rec_params(code, ldc, feat, ldf, m3, hw, weight, bias, M, E, D, cosv, nr, nf);
  const size_t smem = rec_smem_floats(D) * sizeof(float);
  if (int rc = opt_in_smem<rec_fwd_kernel>(smem, "rec_fwd_kernel smem")) return rc;
  rec_fwd_kernel<<<(unsigned)((M + RL_ROWS - 1) / RL_ROWS), 256, smem, reinterpret_cast<cudaStream_t>(stream_)>>>(p);
  STEGO_CHECK_LAUNCH("rec_fwd_kernel");
  return STEGO_OK;
}

// Bytes of the per-CTA dW / db partials stego_rec_bwd needs on the current device (its grid is min(blocks, 2 x SMs)).
extern "C" long long stego_rec_scratch_bytes(long long M, int E, int D) {
  if (M < 1 || E < 1 || D < 1) return 0;
  return 1ll * rec_bwd_grid(M) * (1ll * E * D + E) * static_cast<long long>(sizeof(float));
}

// The forward's inputs and outputs, plus dcos ([1]: d loss / d cos, the same for every pixel).  dcode [M][ldd] (first D
// columns) is ACCUMULATED into; dweight [E][D] and dbias [E] are written, summed over the rows in a fixed order.
extern "C" int stego_rec_bwd(const float* code, long long ldc, const void* feat, long long ldf, const float* m3, int hw,
                             const float* weight, const float* bias, long long M, int E, int D, const float* cosv,
                             const float* nr, const float* nf, const float* dcos, float* dcode, long long ldd,
                             float* scratch, long long scratch_bytes, float* dweight, float* dbias, void* stream_) {
  if (int rc = rec_check(code, ldc, feat, ldf, hw, weight, bias, M, E, D, "stego_rec_bwd")) return rc;
  STEGO_CHECK_ARG(cosv && nr && nf && dcos && dcode && scratch && dweight && dbias, "stego_rec_bwd: null pointer");
  STEGO_CHECK_ARG(ldd >= D, "stego_rec_bwd: ldd=%lld < D=%d", ldd, D);
  const long long need = stego_rec_scratch_bytes(M, E, D);
  STEGO_CHECK_ARG(scratch_bytes >= need, "stego_rec_bwd: scratch of %lld bytes, %lld needed", scratch_bytes, need);
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  RecParams p = rec_params(code, ldc, feat, ldf, m3, hw, weight, bias, M, E, D, cosv, nr, nf);
  p.dcos = dcos; p.dcode = dcode; p.ldd = ldd; p.part = scratch;
  const int G = rec_bwd_grid(M);
  const size_t smem = rec_smem_floats(D) * sizeof(float);
  if (int rc = opt_in_smem<rec_bwd_kernel>(smem, "rec_bwd_kernel smem")) return rc;
  rec_bwd_kernel<<<G, 256, smem, stream>>>(p);
  STEGO_CHECK_LAUNCH("rec_bwd_kernel");
  const long long n = 1ll * E * D + E;
  rec_reduce_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(scratch, G, E, D, dweight, dbias);
  STEGO_CHECK_LAUNCH("rec_reduce_kernel");
  return STEGO_OK;
}
