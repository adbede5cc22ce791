// Fused multi-head self-attention forward for the frozen DINO ViT (sm_90a, wgmma + TMA + mbarrier).
//
// Reference: src/dino/vision_transformer.py:78-90 (Attention.forward):
//     attn = softmax(q k^T * head_dim^-0.5);  x = attn v
// The reference materialises the [B, heads, N, N] fp32 score tensor three times per layer; here it
// never leaves the SM: S = Q K^T accumulates in registers (wgmma, both operands in shared memory), the online
// softmax runs on those registers, and P (bf16) feeds the P V wgmma straight from registers (no shared-memory round
// trip: the accumulator fragment of S is the A-operand fragment of P V).
//
// One CTA per (128-query tile, head, image), head_dim = 64, 288 threads:
//   warps 0..3  MMA/softmax warpgroup 0 (query rows 0..63 of the tile)
//   warps 4..7  MMA/softmax warpgroup 1 (query rows 64..127)
//   warp 8      TMA producer: the Q tile, then a 4-stage ring of 64-key (K, V) tiles shared by both warpgroups
// Each warpgroup keeps its rows' running max / sum and O (64 x 64 fp32) in registers; the [64 x 64] output tile is
// staged in the warpgroup's (then idle) half of the Q tile and leaves as one TMA bulk store.
// Two CTAs per SM (80 KB of shared memory each).
// Input is the packed qkv GEMM output [B, N, 3E] bf16 (q | k | v, head-major inside each), read through
// ONE 3-D tensor map; rows past N (ragged last tile: N = hw + 1 is never a multiple of 128) are
// zero-filled by TMA, masked to -inf in the softmax and clipped from the output store.
#include <stdlib.h>

#include "common.cuh"
#include "host_util.h"

namespace stego {

constexpr int ATT_BQ = 128;
constexpr int ATT_BKV = 64;   // 64-key tiles: 6 % padding waste at N = 785 (128-key tiles waste 14 %), half the smem
constexpr int ATT_D = 64;
constexpr int ATT_STAGES = 4;
constexpr int ATT_THREADS = 288;

constexpr uint32_t ATT_Q_BYTES = 128 * 64 * 2;   // 16 KB [128 q][64 d]
constexpr uint32_t ATT_KV_BYTES = 64 * 64 * 2;   // 8 KB  [64 kv][64 d]
constexpr uint32_t ATT_SMEM_Q = 0;
constexpr uint32_t ATT_SMEM_KV = ATT_Q_BYTES;                                   // stages x (K,V)
constexpr uint32_t ATT_SMEM_BAR = ATT_SMEM_KV + ATT_STAGES * 2 * ATT_KV_BYTES;
constexpr uint32_t ATT_SMEM_TOTAL = ATT_SMEM_BAR + 128;

struct AttnParams {
  int N;       // tokens per image
  int E;       // embed dim = heads * 64
  float scale_log2e;  // head_dim^-0.5 * log2(e)
};

__global__ void __launch_bounds__(ATT_THREADS, 2)
attention_fwd_kernel(const __grid_constant__ CUtensorMap tmQKV, const __grid_constant__ CUtensorMap tmOut, AttnParams p) {
  // no static shared memory in this kernel: the dynamic window starts at offset 0 of the CTA's allocation and the
  // __align__(1024) below is honoured (128B-swizzled tiles need 1024-byte alignment); checked at run time.
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0u) __trap();
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + ATT_SMEM_BAR);
  uint64_t* q_full = bars;                        // [1]
  uint64_t* kv_full = bars + 1;                   // [STAGES]
  uint64_t* kv_empty = kv_full + ATT_STAGES;      // [STAGES]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * ATT_BQ;
  const int head = blockIdx.y;
  const int img = blockIdx.z;
  const int nkv = (p.N + ATT_BKV - 1) / ATT_BKV;

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int s = 0; s < ATT_STAGES; ++s) {
      mbar_init(&kv_full[s], 1);
      mbar_init(&kv_empty[s], 2);  // one arrive per warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 8) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      tma_prefetch_desc(&tmQKV);
      tma_prefetch_desc(&tmOut);
      mbar_arrive_expect_tx(q_full, ATT_Q_BYTES);
      tma_load_3d(smem + ATT_SMEM_Q, &tmQKV, q_full, head * ATT_D, q0, img);
      tma_load_3d(smem + ATT_SMEM_Q + ATT_Q_BYTES / 2, &tmQKV, q_full, head * ATT_D, q0 + 64, img);
      uint32_t stage = 0, phase = 0;
      for (int j = 0; j < nkv; ++j) {
        mbar_wait(&kv_empty[stage], phase ^ 1u);
        uint8_t* sk = smem + ATT_SMEM_KV + stage * 2 * ATT_KV_BYTES;
        mbar_arrive_expect_tx(&kv_full[stage], 2 * ATT_KV_BYTES);
        tma_load_3d(sk, &tmQKV, &kv_full[stage], p.E + head * ATT_D, j * ATT_BKV, img);
        tma_load_3d(sk + ATT_KV_BYTES, &tmQKV, &kv_full[stage], 2 * p.E + head * ATT_D, j * ATT_BKV, img);
        if (++stage == ATT_STAGES) { stage = 0; phase ^= 1u; }
      }
    }
    return;
  }

  // ===================== MMA / softmax warpgroups =====================
  const int wg = warp >> 2;
  const int wq = warp & 3;
  const bool leader = (threadIdx.x & 127) == 0;
  const float c = p.scale_log2e;
  constexpr uint32_t DESC_HI = smem_desc_hi_sw128(1024);
  uint8_t* sq = smem + ATT_SMEM_Q + wg * (ATT_Q_BYTES / 2);  // this warpgroup's 64 query rows
  const uint32_t q_lo = smem_desc_lo(smem_u32(sq), 16);
  const uint32_t k_lo0 = smem_desc_lo(smem_u32(smem + ATT_SMEM_KV), 16);
  const uint32_t v_lo0 = smem_desc_lo(smem_u32(smem + ATT_SMEM_KV + ATT_KV_BYTES), 8192);
  // accumulator fragment: rows wq*16 + lane/4 (+8 for h = 1), columns 8 i + 2 (lane % 4) + {0, 1}
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};  // l_run: this thread's partial row sums
  mbar_wait(q_full, 0);
  uint32_t stage = 0, phase = 0;
  for (int j = 0; j < nkv; ++j) {
    mbar_wait(&kv_full[stage], phase);
    const uint32_t k_lo = k_lo0 + stage * ((2 * ATT_KV_BYTES) >> 4);
    const uint32_t v_lo = v_lo0 + stage * ((2 * ATT_KV_BYTES) >> 4);
    float s[32];
    wgmma_fence();
#pragma unroll
    for (uint32_t k = 0; k < ATT_D / 16; ++k)
      wgmma_ss<64, 0, 0>(s, smem_desc_join(q_lo + k * 2, DESC_HI), smem_desc_join(k_lo + k * 2, DESC_HI), k > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    fence_operands(s);
    const int valid = p.N - j * ATT_BKV;  // number of real keys in this tile (>= 1)
    if (valid < ATT_BKV) {
#pragma unroll
      for (int i = 0; i < 32; ++i)
        if (8 * (i >> 2) + 2 * (lane & 3) + (i & 1) >= valid) s[i] = -INFINITY;
    }
    float alpha[2], mc[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = -INFINITY;
#pragma unroll
      for (int i = 0; i < 8; ++i) mx = fmaxf(mx, fmaxf(s[4 * i + 2 * h], s[4 * i + 2 * h + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[h], mx);
      alpha[h] = ex2_approx((m_run[h] - m_new) * c);  // 0 on the first tile (m_run = -inf)
      m_run[h] = m_new;
      mc[h] = m_new * c;
    }
    // P = exp2(s c - m c) packed to bf16 in the A-operand fragment of the P V wgmma: k16 slice kk of P is
    // accumulator columns 16 kk .. 16 kk + 15, i.e. n8 groups 2 kk (regs 0, 1) and 2 kk + 1 (regs 2, 3)
    uint32_t a[4][4];
    float rs[2] = {0.f, 0.f};
#pragma unroll
    for (int i = 0; i < 8; ++i) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float e0 = ex2_approx(fmaf(s[4 * i + 2 * h], c, -mc[h]));
        const float e1 = ex2_approx(fmaf(s[4 * i + 2 * h + 1], c, -mc[h]));
        rs[h] += e0 + e1;
        a[i >> 1][(i & 1) * 2 + h] = pack_bf16x2(e0, e1);
      }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) l_run[h] = l_run[h] * alpha[h] + rs[h];
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] *= alpha[(i >> 1) & 1];
    wgmma_fence();
#pragma unroll
    for (uint32_t kk = 0; kk < ATT_BKV / 16; ++kk)
      wgmma_rs_n64<1>(o, a[kk], smem_desc_join(v_lo + kk * (2048u >> 4), DESC_HI), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    fence_operands(o);
    if (leader) mbar_arrive(&kv_empty[stage]);  // K_j and V_j are no longer needed by this warpgroup
    if (++stage == ATT_STAGES) { stage = 0; phase ^= 1u; }
  }
  // normalise and stage the [64 q][64 d] bf16 tile in this warpgroup's half of the Q tile (its last reader, the final
  // S wgmma, has retired), 128B-swizzled like the output tensor map; rows >= N are clipped by the map
  float inv[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float l = l_run[h];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    inv[h] = __fdividef(1.0f, l);
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const uint32_t r = static_cast<uint32_t>(wq * 16 + (lane >> 2) + 8 * h);
      const uint32_t off = sw128_offset(r, static_cast<uint32_t>(i)) + 4u * static_cast<uint32_t>(lane & 3);
      *reinterpret_cast<uint32_t*>(sq + off) = pack_bf16x2(o[4 * i + 2 * h] * inv[h], o[4 * i + 2 * h + 1] * inv[h]);
    }
  }
  fence_proxy_async_smem();
  asm volatile("bar.sync %0, 128;\n" ::"r"(wg + 1) : "memory");  // this warpgroup's tile is staged
  if (leader) {
    tma_store_3d(sq, &tmOut, head * ATT_D, q0 + wg * 64, img);
    tma_commit_group();
    tma_wait_group_read<0>();  // the staging tile must outlive the bulk store
  }
}

}  // namespace stego

using namespace stego;

// qkv: [B][N][3E] bf16 packed (q|k|v), out: [B][N][E] bf16.
extern "C" int stego_attention_fwd(const void* qkv, void* out, int B, int N, int E, int heads, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(qkv && out, "stego_attention_fwd: null pointer");
  STEGO_CHECK_ARG(B > 0 && N > 0 && heads > 0, "stego_attention_fwd: bad sizes");
  STEGO_CHECK_ARG(E == heads * ATT_D, "stego_attention_fwd: head_dim must be 64 (E=%d heads=%d)", E, heads);
  STEGO_CHECK_ARG((reinterpret_cast<uintptr_t>(out) & 15u) == 0, "stego_attention_fwd: out not 16-byte aligned");
  CUtensorMap tm;
  uint64_t dims[3] = {(uint64_t)3 * E, (uint64_t)N, (uint64_t)B};
  uint64_t str[2] = {(uint64_t)3 * E * 2, (uint64_t)N * 3 * E * 2};
  uint32_t box[3] = {64, 64, 1};  // one 64-row box serves K, V (one load) and Q (two loads)
  int rc = make_tmap_bf16(&tm, qkv, 3, dims, str, box);
  if (rc != STEGO_OK) return rc;
  CUtensorMap tmo;  // output [B][N][E]: per-image row clipping for the ragged last query tile
  uint64_t odims[3] = {(uint64_t)E, (uint64_t)N, (uint64_t)B};
  uint64_t ostr[2] = {(uint64_t)E * 2, (uint64_t)N * E * 2};
  if ((rc = make_tmap_bf16(&tmo, out, 3, odims, ostr, box)) != STEGO_OK) return rc;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(attention_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)ATT_SMEM_TOTAL);
    if (e != cudaSuccess) return cuda_fail(e, "cudaFuncSetAttribute(attention)");
    configured = true;
  }
  AttnParams p;
  p.N = N;
  p.E = E;
  p.scale_log2e = 0.125f * 1.4426950408889634f;
  dim3 grid((N + ATT_BQ - 1) / ATT_BQ, heads, B);
  attention_fwd_kernel<<<grid, ATT_THREADS, ATT_SMEM_TOTAL, stream>>>(tm, tmo, p);
  STEGO_CHECK_LAUNCH("attention_fwd_kernel");
  return STEGO_OK;
}
