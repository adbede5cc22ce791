// wgmma / TMA / mbarrier GEMM for the STEGO hot path (sm_90a).
//
//   out[M,N] = act(A[M,K] . B[N,K]^T + bias[N]) + residual[M,N]
//
// used for every dense contraction on the path that is a plain GEMM:
//   * DINO ViT linears  (reference: src/dino/vision_transformer.py:58-62 Mlp, :80,:88 Attention qkv/proj,
//                        :127-131 PatchEmbed as an im2col GEMM)
//   * segmentation head (reference: src/modules.py:73-81 cluster1/cluster2 1x1 convs) forward,
//     dgrad (B operand MN-major) and wgrad (both operands MN-major, split-K + fp32 atomics).
//
// Structure: persistent CTAs (one per SM), 384 threads = three warpgroups:
//   warpgroup 0     TMA producer (one thread: cp.async.bulk.tensor -> 128B-swizzled smem ring, mbarrier expect_tx)
//   warpgroups 1,2  MMA + epilogue, rows 0..63 and 64..127 of the 128 x BN tile: wgmma with both operands in shared
//                   memory, fp32 accumulators in registers (BN / 2 per thread), then bias / GELU / ReLU / residual and
//                   the stores straight from the accumulator registers.
// Operand tiles are 128 x 64 (A) and BN x 64 (B) bf16; accumulation fp32.
#include <stdlib.h>

#include "common.cuh"
#include "epilogue.cuh"
#include "host_util.h"

namespace stego {

constexpr int GEMM_BM = 128;
constexpr int GEMM_BK = 64;
constexpr int GEMM_THREADS = 384;

struct GemmParams {
  int M, N, K;        // logical GEMM sizes; K is the reduction length
  int splits;         // split-K factor (>=1); every split owns >= 1 k-block
  int kb_per_split;   // k-blocks per split
  void* out;          // [M or remapped rows][ldo]
  int ldo;
  int out_bf16;       // 1: bf16 output, 0: fp32 output
  const float* bias;  // [N] or null
  int act;            // 0 none, 1 GELU(erf), 2 ReLU
  const float* residual;  // fp32 [rows][ldr] or null (may alias out)
  int ldr;
  int row_div;        // >0: patch-embed mode: out_row = r + r/row_div + 1, residual row = r % row_div + 1
  int atomic;         // 1: fp32 atomicAdd into out (split-K)
  int vec_ok;         // host-verified alignment for paired (8-byte fp32 / 4-byte bf16) accesses of out / residual / bias
  int batch;          // independent GEMMs of the same shape (third tensor-map dimension); 1 = plain GEMM
  long long out_bs;   // element stride between the outputs / residuals of consecutive batch entries
  long long res_bs;
};

// Epilogue of one warpgroup's 64 x BN accumulator, straight from the wgmma fragment: each thread holds rows
// row_top and row_top + 8, and column pairs 8 c + 2 (lane % 4) + {0, 1}.
template <int BN>
__device__ __forceinline__ void gemm_epilogue(float (&acc)[BN / 2], const GemmParams& p, int row_top, int col_base,
                                              int tb) {
  void* const outp = p.out_bf16 ? static_cast<void*>(reinterpret_cast<bf16*>(p.out) + tb * p.out_bs)
                                : static_cast<void*>(reinterpret_cast<float*>(p.out) + tb * p.out_bs);
  const float* const resp = p.residual ? p.residual + tb * p.res_bs : nullptr;
  if (p.bias != nullptr) {
#pragma unroll
    for (int c = 0; c < BN / 8; ++c) {
      const int col = col_base + 8 * c;
      float b0 = 0.f, b1 = 0.f;
      if (col + 1 < p.N && p.vec_ok) {
        const float2 b2 = __ldg(reinterpret_cast<const float2*>(p.bias + col));
        b0 = b2.x; b1 = b2.y;
      } else {
        if (col < p.N) b0 = __ldg(p.bias + col);
        if (col + 1 < p.N) b1 = __ldg(p.bias + col + 1);
      }
      acc[4 * c + 0] += b0; acc[4 * c + 1] += b1;
      acc[4 * c + 2] += b0; acc[4 * c + 3] += b1;
    }
  }
  if (p.act == 1) {
    // bf16 outputs take the MUFU-free polynomial (error far below the bf16 rounding), fp32 outputs the A-S erf
    if (p.out_bf16) {
#pragma unroll
      for (int j = 0; j < BN / 2; j += 8) gelu_erf_poly8(acc + j);
    } else {
#pragma unroll
      for (int j = 0; j < BN / 2; ++j) acc[j] = gelu_erf(acc[j]);
    }
  } else if (p.act == 2) {
#pragma unroll
    for (int j = 0; j < BN / 2; ++j) acc[j] = fmaxf(acc[j], 0.0f);
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = row_top + 8 * h;
    if (row >= p.M) continue;
    int out_row = row, res_row = row;
    if (p.row_div > 0) {
      out_row = row + row / p.row_div + 1;
      res_row = row % p.row_div + 1;
    }
    const size_t obase = static_cast<size_t>(out_row) * p.ldo;
    const size_t rbase = static_cast<size_t>(res_row) * p.ldr;
#pragma unroll
    for (int c = 0; c < BN / 8; ++c) {
      const int col = col_base + 8 * c;
      if (col >= p.N) break;
      const bool two = col + 1 < p.N;
      float x0 = acc[4 * c + 2 * h], x1 = acc[4 * c + 2 * h + 1];
      if (p.atomic) {
        float* o = reinterpret_cast<float*>(outp) + obase + col;
        atomicAdd(o, x0);
        if (two) atomicAdd(o + 1, x1);
        continue;
      }
      const bool vec = two && p.vec_ok;
      if (resp != nullptr) {
        if (vec) {
          const float2 r = *reinterpret_cast<const float2*>(resp + rbase + col);
          x0 += r.x; x1 += r.y;
        } else {
          x0 += resp[rbase + col];
          if (two) x1 += resp[rbase + col + 1];
        }
      }
      if (p.out_bf16) {
        bf16* o = reinterpret_cast<bf16*>(outp) + obase + col;
        if (vec) {
          *reinterpret_cast<uint32_t*>(o) = pack_bf16x2(x0, x1);
        } else {
          o[0] = __float2bfloat16_rn(x0);
          if (two) o[1] = __float2bfloat16_rn(x1);
        }
      } else {
        float* o = reinterpret_cast<float*>(outp) + obase + col;
        if (vec) {
          *reinterpret_cast<float2*>(o) = make_float2(x0, x1);
        } else {
          o[0] = x0;
          if (two) o[1] = x1;
        }
      }
    }
  }
}

template <int BN, int kStages, bool A_MN, bool B_MN>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, GemmParams p) {
  constexpr uint32_t A_BYTES = GEMM_BM * GEMM_BK * 2;  // 16 KB
  constexpr uint32_t B_BYTES = BN * GEMM_BK * 2;
  constexpr uint32_t STAGE_BYTES = A_BYTES + B_BYTES;
  static_assert(BN == 128 || BN == 256, "BN must be 128 or 256");
  static_assert(BN == 128 || (!A_MN && !B_MN), "256-wide tiles are K-major only");
  constexpr int kBBox = 128;  // K-major B box rows

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kStages * STAGE_BYTES);
  uint64_t* empty_bar = full_bar + kStages;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = warp >> 2;  // 0 producer, 1..2 MMA warpgroups

  const int tiles_m = (p.M + GEMM_BM - 1) / GEMM_BM;
  const int tiles_n = (p.N + BN - 1) / BN;
  const int num_kb = (p.K + GEMM_BK - 1) / GEMM_BK;  // K tail: TMA zero-fills out-of-bounds
  const int tiles_per_batch = tiles_m * tiles_n * p.splits;
  const int total_tiles = tiles_per_batch * p.batch;
  const int sched_start = static_cast<int>(blockIdx.x);
  const int sched_step = static_cast<int>(gridDim.x);

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);  // one arrive per MMA warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ===================== TMA producer =====================
    warpgroup_reg_dealloc<40>();
    if (threadIdx.x == 0) {
      uint32_t stage = 0, phase = 0;
      for (int t = sched_start; t < total_tiles; t += sched_step) {
        const int tb = t / tiles_per_batch, tl = t % tiles_per_batch;
        const int split = tl % p.splits;
        const int tn = (tl / p.splits) % tiles_n;
        const int tm = tl / (p.splits * tiles_n);
        const int kb0 = split * p.kb_per_split;
        const int kb1 = min(num_kb, kb0 + p.kb_per_split);
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1u);
          uint8_t* sa = smem + stage * STAGE_BYTES;
          uint8_t* sb = sa + A_BYTES;
          mbar_arrive_expect_tx(&full_bar[stage], STAGE_BYTES);
          if (!A_MN) {
            tma_load_3d(sa, &tmA, &full_bar[stage], kb * GEMM_BK, tm * GEMM_BM, tb);
          } else {
#pragma unroll
            for (int blk = 0; blk < GEMM_BM / 64; ++blk)
              tma_load_3d(sa + blk * 8192, &tmA, &full_bar[stage], tm * GEMM_BM + blk * 64, kb * GEMM_BK, tb);
          }
          if (!B_MN) {
#pragma unroll
            for (int blk = 0; blk < BN / kBBox; ++blk)  // tensor-map box = kBBox rows
              tma_load_3d(sb + blk * (kBBox * 128), &tmB, &full_bar[stage], kb * GEMM_BK, tn * BN + blk * kBBox, tb);
          } else {
#pragma unroll
            for (int blk = 0; blk < BN / 64; ++blk)
              tma_load_3d(sb + blk * 8192, &tmB, &full_bar[stage], tn * BN + blk * 64, kb * GEMM_BK, tb);
          }
          if (++stage == kStages) { stage = 0; phase ^= 1u; }
        }
      }
    }
  } else {
    // ===================== MMA warpgroups =====================
    warpgroup_reg_alloc<232>();
    const int mwg = wg - 1;  // rows 64 * mwg .. of every tile
    // K-major A: rows 64.. start 64 x 128 B further; MN-major A: the second 64-wide M block, also 8 KB further
    constexpr uint32_t DESC_HI = smem_desc_hi_sw128(1024);
    constexpr uint32_t A_KSTEP = A_MN ? (2048u >> 4) : (32u >> 4);  // low-word step per k16 slice
    constexpr uint32_t B_KSTEP = B_MN ? (2048u >> 4) : (32u >> 4);
    const uint32_t a_lo0 = smem_desc_lo(smem_u32(smem) + mwg * 8192u, 8192u);
    const uint32_t b_lo0 = smem_desc_lo(smem_u32(smem) + A_BYTES, 8192u);
    const bool leader = (threadIdx.x & 127) == 0;
    uint32_t stage = 0, phase = 0;
    float acc[BN / 2];
    for (int t = sched_start; t < total_tiles; t += sched_step) {
      const int tb = t / tiles_per_batch, tl = t % tiles_per_batch;
      const int split = tl % p.splits;
      const int tn = (tl / p.splits) % tiles_n;
      const int tm = tl / (p.splits * tiles_n);
      const int kb0 = split * p.kb_per_split;
      const int kb1 = min(num_kb, kb0 + p.kb_per_split);
#pragma unroll
      for (int j = 0; j < BN / 2; ++j) acc[j] = 0.f;
      uint32_t prev_stage = 0;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t a_lo = a_lo0 + stage * (STAGE_BYTES >> 4);
        const uint32_t b_lo = b_lo0 + stage * (STAGE_BYTES >> 4);
        fence_operands(acc);
        wgmma_fence();
#pragma unroll
        for (uint32_t k = 0; k < GEMM_BK / 16; ++k)
          wgmma_ss<BN, A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, smem_desc_join(a_lo + k * A_KSTEP, DESC_HI),
                                                  smem_desc_join(b_lo + k * B_KSTEP, DESC_HI), 1u);
        wgmma_commit();
        wgmma_wait<1>();  // the previous k-block's MMAs have retired: its smem slot is reusable
        if (kb > kb0 && leader) mbar_arrive(&empty_bar[prev_stage]);
        prev_stage = stage;
        if (++stage == kStages) { stage = 0; phase ^= 1u; }
      }
      wgmma_wait<0>();
      fence_operands(acc);
      if (kb1 > kb0 && leader) mbar_arrive(&empty_bar[prev_stage]);
      const int wq = (threadIdx.x >> 5) & 3;
      gemm_epilogue<BN>(acc, p, tm * GEMM_BM + mwg * 64 + wq * 16 + (lane >> 2), tn * BN + 2 * (lane & 3), tb);
    }
  }
}

template <int BN, int kStages, bool A_MN, bool B_MN>
static int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParams& p, cudaStream_t stream) {
  constexpr size_t smem = size_t(kStages) * (GEMM_BM * GEMM_BK * 2 + BN * GEMM_BK * 2) + 1024 + 256;
  static_assert(smem <= 232448, "exceeds the 227 KB of shared memory a CTA can opt into");
  auto kern = gemm_bf16_kernel<BN, kStages, A_MN, B_MN>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return cuda_fail(e, "cudaFuncSetAttribute(gemm)");
    configured = true;
  }
  const int tiles_m = (p.M + GEMM_BM - 1) / GEMM_BM;
  const int tiles_n = (p.N + BN - 1) / BN;
  const int tiles = tiles_m * tiles_n * p.splits * p.batch;
  const int grid = tiles < num_sms() ? tiles : num_sms();
  kern<<<grid, GEMM_THREADS, smem, stream>>>(tmA, tmB, p);
  STEGO_CHECK_LAUNCH("gemm_bf16_kernel launch");
  return STEGO_OK;
}

}  // namespace stego

using namespace stego;

// Shared implementation of stego_gemm_bf16 (batch = 1) and stego_gemm_bf16_batched: `batch` independent GEMMs of one
// shape, entry b reading A + b * a_bs, B + b * b_bs and writing out + b * out_bs (element strides); every tensor map
// is 3-D with the batch as its outermost dimension, so rows past M / N of an entry are out of bounds for TMA (zero
// fill on loads, clipped on stores) instead of running into the next entry.
static int gemm_impl(const void* A, int lda, long long a_bs, int a_mn_major, const void* B, int ldb, long long b_bs,
                     int b_mn_major, int batch, int M, int N, int K, void* out, int ldo, long long out_bs, int out_bf16,
                     const float* bias, int act, const float* residual, int ldr, long long res_bs, int row_div, int splits,
                     int atomic_out, cudaStream_t stream) {
  STEGO_CHECK_ARG(A && B && out, "stego_gemm_bf16: null pointer");
  STEGO_CHECK_ARG(M > 0 && N > 0 && K > 0 && batch > 0, "stego_gemm_bf16: bad sizes M=%d N=%d K=%d batch=%d", M, N, K, batch);
  STEGO_CHECK_ARG(lda % 8 == 0 && ldb % 8 == 0, "stego_gemm_bf16: lda/ldb must be multiples of 8 elements");
  STEGO_CHECK_ARG(batch == 1 || (a_bs % 8 == 0 && b_bs % 8 == 0 && row_div == 0),
                  "stego_gemm_bf16_batched: operand batch strides must be multiples of 8 elements");
  STEGO_CHECK_ARG(act >= 0 && act <= 2, "stego_gemm_bf16: act=%d", act);
  STEGO_CHECK_ARG(!(atomic_out && out_bf16), "stego_gemm_bf16: atomic output must be fp32");
  STEGO_CHECK_ARG(splits >= 1, "stego_gemm_bf16: splits=%d", splits);
  STEGO_CHECK_ARG(splits == 1 || atomic_out, "stego_gemm_bf16: split-K requires atomic_out");
  if (batch == 1) {  // any 16-byte-compatible value: the third coordinate is always 0
    a_bs = static_cast<long long>(a_mn_major ? K : M) * lda;
    b_bs = static_cast<long long>(b_mn_major ? K : N) * ldb;
    out_bs = static_cast<long long>(M) * ldo;
    res_bs = 0;
  }

  GemmParams p;
  p.M = M; p.N = N; p.K = K;
  const int num_kb = (K + GEMM_BK - 1) / GEMM_BK;
  if (splits > num_kb) splits = num_kb;
  p.kb_per_split = (num_kb + splits - 1) / splits;
  p.splits = (num_kb + p.kb_per_split - 1) / p.kb_per_split;
  p.out = out; p.ldo = ldo; p.out_bf16 = out_bf16;
  p.bias = bias; p.act = act;
  p.residual = residual; p.ldr = ldr;
  p.row_div = row_div; p.atomic = atomic_out;
  p.batch = batch; p.out_bs = out_bs; p.res_bs = res_bs;
  const size_t esz = out_bf16 ? 2 : 4;
  const size_t pair = 2 * esz;  // paired accesses: two consecutive elements
  p.vec_ok = ((reinterpret_cast<uintptr_t>(out) % pair) == 0) && (ldo % 2 == 0) && (out_bs % 2 == 0) &&
             (residual == nullptr || ((reinterpret_cast<uintptr_t>(residual) % 8) == 0 && ldr % 2 == 0 && res_bs % 2 == 0)) &&
             (bias == nullptr || (reinterpret_cast<uintptr_t>(bias) % 8) == 0);
  // Tile shape: 128 x 256 for wide-N K-major linears (qkv: N = 3E, fc1: N = 4E; halves the A re-reads from L2),
  // 128 x 128 for everything else (incl. MN-major operands and split-K).
  const bool wide = !a_mn_major && !b_mn_major && splits == 1 && N >= 1024;

  CUtensorMap tmA, tmB;
  int rc;
  {
    // K-major: tensor is [batch][M][K] (inner = K). MN-major: tensor is [batch][K][M] (inner = M).
    uint64_t dims[3] = {a_mn_major ? (uint64_t)M : (uint64_t)K, a_mn_major ? (uint64_t)K : (uint64_t)M, (uint64_t)batch};
    uint64_t str[2] = {(uint64_t)lda * 2, (uint64_t)a_bs * 2};
    uint32_t box[3] = {64, a_mn_major ? 64u : (uint32_t)GEMM_BM, 1};
    if ((rc = make_tmap_bf16(&tmA, A, 3, dims, str, box)) != STEGO_OK) return rc;
  }
  {
    uint64_t dims[3] = {b_mn_major ? (uint64_t)N : (uint64_t)K, b_mn_major ? (uint64_t)K : (uint64_t)N, (uint64_t)batch};
    uint64_t str[2] = {(uint64_t)ldb * 2, (uint64_t)b_bs * 2};
    uint32_t box[3] = {64, b_mn_major ? 64u : 128u, 1};  // rows per B box: must match the kernel's kBBox
    if ((rc = make_tmap_bf16(&tmB, B, 3, dims, str, box)) != STEGO_OK) return rc;
  }
  if (wide) return launch_gemm<256, 4, false, false>(tmA, tmB, p, stream);
  if (!a_mn_major && !b_mn_major) return launch_gemm<128, 6, false, false>(tmA, tmB, p, stream);
  if (!a_mn_major && b_mn_major) return launch_gemm<128, 6, false, true>(tmA, tmB, p, stream);
  if (a_mn_major && b_mn_major) return launch_gemm<128, 6, true, true>(tmA, tmB, p, stream);
  return launch_gemm<128, 6, true, false>(tmA, tmB, p, stream);
}

// C-ABI: see include/stego_b200.h for the contract.
extern "C" int stego_gemm_bf16(const void* A, int lda, int a_mn_major, const void* B, int ldb, int b_mn_major, int M,
                               int N, int K, void* out, int ldo, int out_bf16, const float* bias, int act,
                               const float* residual, int ldr, int row_div, int splits, int atomic_out,
                               void* stream_) {
  return gemm_impl(A, lda, 0, a_mn_major, B, ldb, 0, b_mn_major, 1, M, N, K, out, ldo, 0, out_bf16, bias, act, residual, ldr, 0,
                   row_div, splits, atomic_out, reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int stego_gemm_bf16_batched(const void* A, int lda, long long a_batch_stride, int a_mn_major, const void* B,
                                       int ldb, long long b_batch_stride, int b_mn_major, int batch, int M, int N, int K,
                                       void* out, int ldo, long long out_batch_stride, int out_bf16, const float* bias,
                                       int act, void* stream_) {
  return gemm_impl(A, lda, a_batch_stride, a_mn_major, B, ldb, b_batch_stride, b_mn_major, batch, M, N, K, out, ldo,
                   out_batch_stride, out_bf16, bias, act, nullptr, 0, 0, 0, 1, 0, reinterpret_cast<cudaStream_t>(stream_));
}
