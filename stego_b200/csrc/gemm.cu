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
// Structure: persistent CTAs (one per SM), 384 threads = three warpgroups, ping-pong schedule:
//   warpgroup 0     TMA producer (one thread: cp.async.bulk.tensor -> 128B-swizzled smem ring, mbarrier expect_tx),
//                   loading the CTA's tiles in order
//   warpgroups 1,2  MMA + epilogue.  The CTA's i-th tile belongs to MMA warpgroup i % 2, which computes the whole
//                   128 x 128 tile (two m64n128 wgmmas per k16 slice, 128 fp32 accumulators per thread).  The two take
//                   turns on the tensor cores (an mbarrier hand-over after each mainloop), so one runs its mainloop
//                   while the other runs its epilogue.
// Epilogues: bias / GELU / ReLU in registers, then either
//   * TMA: the tile is staged in 128B-swizzled shared memory in 16 KB column chunks and leaves by TMA bulk stores, or
//     by TMA fp32 reduce-adds when the residual is the output itself (x += ...); no global loads; or
//   * registers: paired stores straight from the accumulator fragments, for what TMA cannot express: split-K atomics,
//     the patch-embed row remap, a residual other than the output, outputs (or rows of N outputs) not 16-byte aligned.
// Operand tiles are 128 x 64 bf16 (A and B); accumulation fp32.
// Large GEMMs with K <= 384 (the ViT-S qkv, proj, fc1) run gemm_bf16_resident_kernel instead, which keeps each CTA's
// 128-column block of B in shared memory and streams only A.
#include <stdlib.h>
#include <string.h>

#include "common.cuh"
#include "epilogue.cuh"
#include "host_util.h"

namespace stego {

constexpr int GEMM_BM = 128;
constexpr int GEMM_BN = 128;
constexpr int GEMM_BK = 64;
constexpr int GEMM_THREADS = 384;
constexpr uint32_t GEMM_STAGE_BYTES = (GEMM_BM + GEMM_BN) * GEMM_BK * 2;  // 32 KB
constexpr uint32_t GEMM_CHUNK_BYTES = GEMM_BM * 128;                        // one [128 rows][128 B] staging chunk

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
  int reduce_add;     // TMA epilogue: 1 = out += tile (residual is out), 0 = out = tile
  int batch;          // independent GEMMs of the same shape (third tensor-map dimension); 1 = plain GEMM
  long long out_bs;   // element stride between the outputs / residuals of consecutive batch entries
  long long res_bs;
};

// Bias and activation on one 64 x BN accumulator fragment: each thread holds column pairs 8 c + 2 (lane % 4) + {0, 1}
// of rows row_top and row_top + 8.
template <int BN>
__device__ __forceinline__ void gemm_bias_act(float (&acc)[BN / 2], const GemmParams& p, int col_base) {
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
    // bf16 outputs take the MUFU-free polynomial (absolute error ~1e-4), fp32 outputs the A-S erf (~5e-7)
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
}

// Register epilogue of one 64 x BN accumulator fragment (after gemm_bias_act): residual, then paired stores or
// atomics straight from the fragment, rows row_top and row_top + 8.
template <int BN>
__device__ __forceinline__ void gemm_store_regs(const float (&acc)[BN / 2], const GemmParams& p, int row_top,
                                                int col_base, int tb) {
  void* const outp = p.out_bf16 ? static_cast<void*>(reinterpret_cast<bf16*>(p.out) + tb * p.out_bs)
                                : static_cast<void*>(reinterpret_cast<float*>(p.out) + tb * p.out_bs);
  const float* const resp = p.residual ? p.residual + tb * p.res_bs : nullptr;
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

// TMA epilogue of one warpgroup's 128 x 128 tile (after gemm_bias_act).  The tile leaves in column chunks of 128 B per
// row (64 bf16 or 32 fp32 columns), each staged as a [128 rows][128 B] SWIZZLE_128B box — the layout the output tensor
// map describes — in one of the warpgroup's two 16 KB buffers, alternating, so writing chunk c overlaps the store of
// chunk c - 1.  Every chunk is its own bulk group: before buffer reuse the issuing thread waits only until the store
// two chunks back has READ its buffer.  Rows past M and columns past N are clipped by TMA.  The named barrier (one
// per warpgroup, 128 threads) only orders the warpgroup's own staging writes against its issuing thread.
template <bool kBf16, int kBufs = 2>
__device__ __forceinline__ void gemm_store_tma(const float (&acc)[2][GEMM_BN / 2], const GemmParams& p,
                                               const CUtensorMap* tm_out, uint32_t stage, int bar_id, bool issuer,
                                               int m0, int n0, int tb) {
  constexpr int kCols = kBf16 ? 64 : 32;  // columns per chunk
  const int lane = threadIdx.x & 31;
  const int wq = (threadIdx.x >> 5) & 3;
  const uint32_t q = lane & 3;
  const uint32_t swz = (lane >> 2) & 7;  // row & 7 of every row this thread holds
#pragma unroll
  for (int ch = 0; ch < GEMM_BN / kCols; ++ch) {
    const uint32_t buf = stage + (ch % kBufs) * GEMM_CHUNK_BYTES;
    if (issuer) tma_wait_group_read<kBufs - 1>();
    named_bar_sync(bar_id, 128);
    // this thread's rows are 16 wq + lane / 4 + {0, 8, 64, 72}, all with the same row & 7
    const uint32_t rbase = buf + (16 * wq + (lane >> 2)) * 128u;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
      for (int e2 = 0; e2 < 2; ++e2) {
        const uint32_t rp = rbase + (64 * h + 8 * e2) * 128u;
        if constexpr (kBf16) {
          // 64 columns: 8-column group j is 16-byte unit j of the row; this thread's pair sits at byte 4 q of it
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const int c = 8 * ch + j;
            st_shared_b32(rp + (((uint32_t)j ^ swz) << 4) + 4 * q,
                          pack_bf16x2(acc[h][4 * c + 2 * e2], acc[h][4 * c + 2 * e2 + 1]));
          }
        } else {
          // 32 columns: 8-column group j covers 16-byte units 2 j and 2 j + 1; the pair sits at byte 8 q of the two
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int c = 4 * ch + j;
            const uint32_t unit = 2 * j + (q >> 1);
            st_shared_v2_f32(rp + ((unit ^ swz) << 4) + 8 * (q & 1), acc[h][4 * c + 2 * e2],
                             acc[h][4 * c + 2 * e2 + 1]);
          }
        }
      }
    }
    fence_proxy_async_smem();  // generic-proxy smem writes -> visible to the TMA (async proxy) read
    named_bar_sync(bar_id, 128);
    if (issuer) {
      const int col = n0 + ch * kCols;
      if (p.reduce_add) tma_reduce_add_3d(buf, tm_out, col, m0, tb);
      else tma_store_3d(buf, tm_out, col, m0, tb);
      tma_commit_group();
    }
  }
}

// Advance a ring position by n stages.
template <int kStages>
__device__ __forceinline__ void ring_advance(uint32_t& stage, uint32_t& phase, int n) {
  stage += n;
  while (stage >= kStages) { stage -= kStages; phase ^= 1u; }
}

template <int kStages, bool A_MN, bool B_MN, bool kTmaEpi>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const __grid_constant__ CUtensorMap tmOut, GemmParams p) {
  constexpr uint32_t A_BYTES = GEMM_BM * GEMM_BK * 2;  // 16 KB
  constexpr uint32_t STAGE_BYTES = GEMM_STAGE_BYTES;

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* staging = smem + kStages * STAGE_BYTES;  // kTmaEpi: two 16 KB chunk buffers per MMA warpgroup
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(staging + (kTmaEpi ? 4 * GEMM_CHUNK_BYTES : 0));
  uint64_t* empty_bar = full_bar + kStages;
  uint64_t* turn_bar = empty_bar + kStages;  // turn_bar[w]: MMA warpgroup w may start its next mainloop

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = warp >> 2;  // 0 producer, 1..2 MMA warpgroups

  const int tiles_m = (p.M + GEMM_BM - 1) / GEMM_BM;
  const int tiles_n = (p.N + GEMM_BN - 1) / GEMM_BN;
  const int num_kb = (p.K + GEMM_BK - 1) / GEMM_BK;  // K tail: TMA zero-fills out-of-bounds
  const int tiles_per_batch = tiles_m * tiles_n * p.splits;
  const int total_tiles = tiles_per_batch * p.batch;
  const int sched_start = static_cast<int>(blockIdx.x);
  const int sched_step = static_cast<int>(gridDim.x);

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if (kTmaEpi) tma_prefetch_desc(&tmOut);
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 1);  // every stage is consumed by exactly one MMA warpgroup
    }
    mbar_init(&turn_bar[0], 1);
    mbar_init(&turn_bar[1], 1);
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
            tma_load_3d(sb, &tmB, &full_bar[stage], kb * GEMM_BK, tn * GEMM_BN, tb);
          } else {
#pragma unroll
            for (int blk = 0; blk < GEMM_BN / 64; ++blk)
              tma_load_3d(sb + blk * 8192, &tmB, &full_bar[stage], tn * GEMM_BN + blk * 64, kb * GEMM_BK, tb);
          }
          if (++stage == kStages) { stage = 0; phase ^= 1u; }
        }
      }
    }
  } else {
    // ===================== MMA warpgroups =====================
    warpgroup_reg_alloc<232>();
    const int mwg = wg - 1;  // owns the CTA's tiles i with i % 2 == mwg
    // rows 64.. of the A tile start 8 KB further in both layouts (K-major: 64 rows x 128 B; MN-major: the second
    // 64-wide M block)
    constexpr uint32_t DESC_HI = smem_desc_hi_sw128(1024);
    constexpr uint32_t A_KSTEP = A_MN ? (2048u >> 4) : (32u >> 4);  // low-word step per k16 slice
    constexpr uint32_t B_KSTEP = B_MN ? (2048u >> 4) : (32u >> 4);
    constexpr uint32_t A_HALF = 8192u >> 4;
    const uint32_t a_lo0 = smem_desc_lo(smem_u32(smem), 8192u);
    const uint32_t b_lo0 = smem_desc_lo(smem_u32(smem) + A_BYTES, 8192u);
    const bool leader = (threadIdx.x & 127) == 0;
    const int wq = (threadIdx.x >> 5) & 3;
    uint32_t stage = 0, phase = 0;
    float acc[2][GEMM_BN / 2];
    int i = 0;
    for (int t = sched_start; t < total_tiles; t += sched_step, ++i) {
      const int tb = t / tiles_per_batch, tl = t % tiles_per_batch;
      const int split = tl % p.splits;
      const int tn = (tl / p.splits) % tiles_n;
      const int tm = tl / (p.splits * tiles_n);
      const int kb0 = split * p.kb_per_split;
      const int kb1 = min(num_kb, kb0 + p.kb_per_split);
      if ((i & 1) != mwg) {  // the partner's tile: its k-blocks pass through the ring in between
        ring_advance<kStages>(stage, phase, kb1 - kb0);
        continue;
      }
      // Wait for the turn: the partner has issued all MMAs of the tile before this one.  Tile i - 1 always exists,
      // so a warpgroup never waits on a partner that has run out of tiles; the hand-over after the CTA's last tile
      // completes a phase nobody waits for.
      if (i > 0) mbar_wait(&turn_bar[mwg], ((i - 1) >> 1) & 1);
#pragma unroll
      for (int j = 0; j < GEMM_BN / 2; ++j) { acc[0][j] = 0.f; acc[1][j] = 0.f; }
      uint32_t prev_stage = 0;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t a_lo = a_lo0 + stage * (STAGE_BYTES >> 4);
        const uint32_t b_lo = b_lo0 + stage * (STAGE_BYTES >> 4);
        fence_operands(acc[0]);
        fence_operands(acc[1]);
        wgmma_fence();
#pragma unroll
        for (uint32_t k = 0; k < GEMM_BK / 16; ++k) {
          const uint64_t db = smem_desc_join(b_lo + k * B_KSTEP, DESC_HI);
#pragma unroll
          for (uint32_t h = 0; h < 2; ++h)
            wgmma_ss<GEMM_BN, A_MN ? 1 : 0, B_MN ? 1 : 0>(
                acc[h], smem_desc_join(a_lo + h * A_HALF + k * A_KSTEP, DESC_HI), db, 1u);
        }
        wgmma_commit();
        wgmma_wait<1>();  // the previous k-block's MMAs have retired: its smem slot is reusable
        if (kb > kb0 && leader) mbar_arrive(&empty_bar[prev_stage]);
        prev_stage = stage;
        if (++stage == kStages) { stage = 0; phase ^= 1u; }
      }
      if (leader) mbar_arrive(&turn_bar[mwg ^ 1]);  // hand the tensor cores to the partner
      wgmma_wait<0>();
      fence_operands(acc[0]);
      fence_operands(acc[1]);
      if (kb1 > kb0 && leader) mbar_arrive(&empty_bar[prev_stage]);
      const int col_base = tn * GEMM_BN + 2 * (lane & 3);
      gemm_bias_act<GEMM_BN>(acc[0], p, col_base);
      gemm_bias_act<GEMM_BN>(acc[1], p, col_base);
      if constexpr (kTmaEpi) {
        const uint32_t st = smem_u32(staging) + mwg * 2 * GEMM_CHUNK_BYTES;
        if (p.out_bf16) gemm_store_tma<true>(acc, p, &tmOut, st, 1 + mwg, leader, tm * GEMM_BM, tn * GEMM_BN, tb);
        else gemm_store_tma<false>(acc, p, &tmOut, st, 1 + mwg, leader, tm * GEMM_BM, tn * GEMM_BN, tb);
      } else {
        const int row_top = tm * GEMM_BM + wq * 16 + (lane >> 2);
        gemm_store_regs<GEMM_BN>(acc[0], p, row_top, col_base, tb);
        gemm_store_regs<GEMM_BN>(acc[1], p, row_top + 64, col_base, tb);
      }
    }
    if (kTmaEpi && leader) tma_wait_group<0>();  // every store has completed before the CTA (and its smem) goes away
  }
}

template <int kStages, bool A_MN, bool B_MN, bool kTmaEpi>
static int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmOut, const GemmParams& p,
                       cudaStream_t stream) {
  constexpr size_t smem = size_t(kStages) * GEMM_STAGE_BYTES + (kTmaEpi ? 4 * GEMM_CHUNK_BYTES : 0) + 1024 + 256;
  static_assert(smem <= 232448, "exceeds the 227 KB of shared memory a CTA can opt into");
  constexpr auto kern = gemm_bf16_kernel<kStages, A_MN, B_MN, kTmaEpi>;
  if (const int rc = opt_in_smem<kern>(smem, "gemm_bf16_kernel"); rc != STEGO_OK) return rc;
  const int tiles_m = (p.M + GEMM_BM - 1) / GEMM_BM;
  const int tiles_n = (p.N + GEMM_BN - 1) / GEMM_BN;
  const int tiles = tiles_m * tiles_n * p.splits * p.batch;
  const int grid = tiles < num_sms() ? tiles : num_sms();
  kern<<<grid, GEMM_THREADS, smem, stream>>>(tmA, tmB, tmOut, p);
  STEGO_CHECK_LAUNCH("gemm_bf16_kernel launch");
  return STEGO_OK;
}

// Ring depth: 6 x 32 KB stages, or 5 when the TMA epilogue's 64 KB of staging buffers share the CTA's shared memory.
template <bool A_MN, bool B_MN>
static int launch_gemm_epi(bool tma_epi, const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmOut,
                           const GemmParams& p, cudaStream_t stream) {
  if (tma_epi) return launch_gemm<5, A_MN, B_MN, true>(tmA, tmB, tmOut, p, stream);
  return launch_gemm<6, A_MN, B_MN, false>(tmA, tmB, tmOut, p, stream);
}

// Resident-weight variant for K <= GEMM_RES_MAX_K, both operands K-major, batch 1, TMA epilogue.  Every tile of
// gemm_bf16_kernel streams a 128 x 64 A box and a 128 x 64 B box per k-block; here each CTA owns one 128-column block
// tn of the output, loads B[tn] ([128 cols][K], ceil(K / 64) SWIZZLE_128B boxes) into shared memory once, and the
// ring carries only A boxes: half the L2-to-SM bytes per tile.  The CTAs sharing column tn walk the row tiles
// tm = blockIdx.x / tiles_n, strided by their count, so the CTAs of all columns advance through A together and A's
// re-reads (once per column) hit L2.  Warp roles, the ping-pong hand-over and the epilogue are gemm_bf16_kernel's; each
// output element sees the same k16 wgmma sequence, so the results are bit-identical to it.
constexpr int GEMM_RES_MAX_K = 384;
constexpr uint32_t GEMM_RES_BOX_BYTES = GEMM_BM * GEMM_BK * 2;  // one 128 x 64 bf16 box, A or B: 16 KB
constexpr uint32_t GEMM_RES_B_BYTES = (GEMM_RES_MAX_K / GEMM_BK) * GEMM_RES_BOX_BYTES;

//
// Shared memory: 96 KB of B, then either 4 A stages and two 16 KB staging buffers per MMA warpgroup (kBufs = 2), or 6
// A stages and one buffer per warpgroup (kBufs = 1).  At the c1 shapes on an H100 the deeper ring made the GELU / ReLU
// GEMMs 4-7 % faster and the plain bf16 / fp32 x += ones slower (their stores serialise on the single buffer).
template <int kStages, int kBufs>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_resident_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                          const __grid_constant__ CUtensorMap tmOut, GemmParams p) {
  constexpr uint32_t BOX = GEMM_RES_BOX_BYTES;

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sb = smem;                                  // B column block: box kb at kb * 16 KB
  uint8_t* sa = smem + GEMM_RES_B_BYTES;               // A ring
  uint8_t* staging = sa + kStages * BOX;               // kBufs 16 KB chunk buffers per MMA warpgroup
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(staging + 2 * kBufs * GEMM_CHUNK_BYTES);
  uint64_t* empty_bar = full_bar + kStages;
  uint64_t* turn_bar = empty_bar + kStages;  // turn_bar[w]: MMA warpgroup w may start its next mainloop
  uint64_t* b_bar = turn_bar + 2;            // the B column block has landed

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = warp >> 2;  // 0 producer, 1..2 MMA warpgroups

  const int tiles_m = (p.M + GEMM_BM - 1) / GEMM_BM;
  const int tiles_n = (p.N + GEMM_BN - 1) / GEMM_BN;
  const int num_kb = (p.K + GEMM_BK - 1) / GEMM_BK;  // K tail: TMA zero-fills out-of-bounds
  // the host launches at least tiles_n CTAs, so every column block has one
  const int tn = static_cast<int>(blockIdx.x) % tiles_n;
  const int tm_start = static_cast<int>(blockIdx.x) / tiles_n;
  const int tm_step = (static_cast<int>(gridDim.x) - tn + tiles_n - 1) / tiles_n;  // CTAs that own column tn

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    tma_prefetch_desc(&tmOut);
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 1);  // every stage is consumed by exactly one MMA warpgroup
    }
    mbar_init(&turn_bar[0], 1);
    mbar_init(&turn_bar[1], 1);
    mbar_init(b_bar, 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ===================== TMA producer =====================
    warpgroup_reg_dealloc<40>();
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(b_bar, num_kb * BOX);
      for (int kb = 0; kb < num_kb; ++kb) tma_load_3d(sb + kb * BOX, &tmB, b_bar, kb * GEMM_BK, tn * GEMM_BN, 0);
      uint32_t stage = 0, phase = 0;
      for (int tm = tm_start; tm < tiles_m; tm += tm_step) {
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1u);
          mbar_arrive_expect_tx(&full_bar[stage], BOX);
          tma_load_3d(sa + stage * BOX, &tmA, &full_bar[stage], kb * GEMM_BK, tm * GEMM_BM, 0);
          if (++stage == kStages) { stage = 0; phase ^= 1u; }
        }
      }
    }
  } else {
    // ===================== MMA warpgroups =====================
    warpgroup_reg_alloc<232>();
    const int mwg = wg - 1;  // owns the CTA's tiles i with i % 2 == mwg
    constexpr uint32_t DESC_HI = smem_desc_hi_sw128(1024);
    constexpr uint32_t KSTEP = 32u >> 4;     // low-word step per k16 slice (K-major)
    constexpr uint32_t A_HALF = 8192u >> 4;  // rows 64.. of the A tile
    const uint32_t a_lo0 = smem_desc_lo(smem_u32(sa), 8192u);
    const uint32_t b_lo0 = smem_desc_lo(smem_u32(sb), 8192u);
    const bool leader = (threadIdx.x & 127) == 0;
    uint32_t stage = 0, phase = 0;
    float acc[2][GEMM_BN / 2];
    mbar_wait(b_bar, 0);
    int i = 0;
    for (int tm = tm_start; tm < tiles_m; tm += tm_step, ++i) {
      if ((i & 1) != mwg) {  // the partner's tile: its k-blocks pass through the ring in between
        ring_advance<kStages>(stage, phase, num_kb);
        continue;
      }
      if (i > 0) mbar_wait(&turn_bar[mwg], ((i - 1) >> 1) & 1);  // as in gemm_bf16_kernel
#pragma unroll
      for (int j = 0; j < GEMM_BN / 2; ++j) { acc[0][j] = 0.f; acc[1][j] = 0.f; }
      uint32_t prev_stage = 0;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t a_lo = a_lo0 + stage * (BOX >> 4);
        const uint32_t b_lo = b_lo0 + kb * (BOX >> 4);
        fence_operands(acc[0]);
        fence_operands(acc[1]);
        wgmma_fence();
#pragma unroll
        for (uint32_t k = 0; k < GEMM_BK / 16; ++k) {
          const uint64_t db = smem_desc_join(b_lo + k * KSTEP, DESC_HI);
#pragma unroll
          for (uint32_t h = 0; h < 2; ++h)
            wgmma_ss<GEMM_BN, 0, 0>(acc[h], smem_desc_join(a_lo + h * A_HALF + k * KSTEP, DESC_HI), db, 1u);
        }
        wgmma_commit();
        wgmma_wait<1>();  // the previous k-block's MMAs have retired: its A slot is reusable
        if (kb > 0 && leader) mbar_arrive(&empty_bar[prev_stage]);
        prev_stage = stage;
        if (++stage == kStages) { stage = 0; phase ^= 1u; }
      }
      if (leader) mbar_arrive(&turn_bar[mwg ^ 1]);  // hand the tensor cores to the partner
      wgmma_wait<0>();
      fence_operands(acc[0]);
      fence_operands(acc[1]);
      if (leader) mbar_arrive(&empty_bar[prev_stage]);
      const int col_base = tn * GEMM_BN + 2 * (lane & 3);
      gemm_bias_act<GEMM_BN>(acc[0], p, col_base);
      gemm_bias_act<GEMM_BN>(acc[1], p, col_base);
      const uint32_t st = smem_u32(staging) + mwg * kBufs * GEMM_CHUNK_BYTES;
      if (p.out_bf16) gemm_store_tma<true, kBufs>(acc, p, &tmOut, st, 1 + mwg, leader, tm * GEMM_BM, tn * GEMM_BN, 0);
      else gemm_store_tma<false, kBufs>(acc, p, &tmOut, st, 1 + mwg, leader, tm * GEMM_BM, tn * GEMM_BN, 0);
    }
    if (leader) tma_wait_group<0>();  // every store has completed before the CTA (and its smem) goes away
  }
}

template <int kStages, int kBufs>
static int launch_gemm_resident_kernel(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmOut,
                                       const GemmParams& p, int grid, cudaStream_t stream) {
  constexpr size_t smem = GEMM_RES_B_BYTES + kStages * GEMM_RES_BOX_BYTES + 2 * kBufs * GEMM_CHUNK_BYTES + 1024 + 256;
  static_assert(smem <= 232448, "exceeds the 227 KB of shared memory a CTA can opt into");
  constexpr auto kern = gemm_bf16_resident_kernel<kStages, kBufs>;
  if (const int rc = opt_in_smem<kern>(smem, "gemm_bf16_resident_kernel"); rc != STEGO_OK) return rc;
  kern<<<grid, GEMM_THREADS, smem, stream>>>(tmA, tmB, tmOut, p);
  STEGO_CHECK_LAUNCH("gemm_bf16_resident_kernel launch");
  return STEGO_OK;
}

static int launch_gemm_resident(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmOut,
                                const GemmParams& p, int grid, cudaStream_t stream) {
  if (p.act != 0) return launch_gemm_resident_kernel<6, 1>(tmA, tmB, tmOut, p, grid, stream);
  return launch_gemm_resident_kernel<4, 2>(tmA, tmB, tmOut, p, grid, stream);
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
  // every split adds its partial sum into out: a bias would be added `splits` times, an activation would act on the
  // partial sums, and the register epilogue's atomics have no residual term
  STEGO_CHECK_ARG(!atomic_out || (bias == nullptr && act == 0 && residual == nullptr),
                  "stego_gemm_bf16: atomic_out takes no bias, act or residual (bias=%p act=%d residual=%p)",
                  (const void*)bias, act, (const void*)residual);
  STEGO_CHECK_ARG(lda >= (a_mn_major ? M : K) && ldb >= (b_mn_major ? N : K),
                  "stego_gemm_bf16: lda=%d / ldb=%d shorter than a row (M=%d N=%d K=%d, a_mn_major=%d b_mn_major=%d)",
                  lda, ldb, M, N, K, a_mn_major, b_mn_major);
  STEGO_CHECK_ARG(ldo >= N && (residual == nullptr || ldr >= N),
                  "stego_gemm_bf16: ldo=%d / ldr=%d shorter than a row of N=%d", ldo, ldr, N);
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
  // Epilogue: TMA stores (or fp32 TMA reduce-adds for out += ..., the residual being the output itself) whenever a
  // tensor map can describe the output: no split-K atomics, no row remap, 16-byte aligned base and strides, and rows
  // of whole 16-byte units — with N * size not a multiple of 16 B, the store's last 16-byte unit of a row wrote the
  // padding columns after N (zeros) on the H100, and callers keep data there (the head's [M][72] code rows, N = 70).
  const bool in_place = residual != nullptr && residual == out && ldr == ldo && !out_bf16;
  const bool tma_epi = !atomic_out && row_div == 0 && (residual == nullptr || in_place) &&
                       (reinterpret_cast<uintptr_t>(out) % 16) == 0 && (static_cast<size_t>(ldo) * esz) % 16 == 0 &&
                       (static_cast<size_t>(out_bs) * esz) % 16 == 0 && (static_cast<size_t>(N) * esz) % 16 == 0;
  p.reduce_add = tma_epi && in_place;

  CUtensorMap tmA, tmB, tmOut;
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
    uint32_t box[3] = {64, b_mn_major ? 64u : (uint32_t)GEMM_BN, 1};
    if ((rc = make_tmap_bf16(&tmB, B, 3, dims, str, box)) != STEGO_OK) return rc;
  }
  if (tma_epi) {
    // exactly [batch][M][N]: TMA clips the stores of ragged tiles at M and N, never touching padding columns
    uint64_t dims[3] = {(uint64_t)N, (uint64_t)M, (uint64_t)batch};
    uint64_t str[2] = {(uint64_t)ldo * esz, (uint64_t)out_bs * esz};
    uint32_t box[3] = {(uint32_t)(128 / esz), (uint32_t)GEMM_BM, 1};  // one staging chunk: [128 rows][128 B]
    rc = out_bf16 ? make_tmap_bf16(&tmOut, out, 3, dims, str, box) : make_tmap_f32(&tmOut, out, 3, dims, str, box);
    if (rc != STEGO_OK) return rc;
  } else {
    memset(&tmOut, 0, sizeof(tmOut));  // unused by the register epilogue
  }
  // The resident-weight kernel needs its B column block to fit in shared memory (K <= 384) and enough tiles per CTA
  // (>= 4 per SM) to amortise loading it; one CTA per SM, at least one per column block.
  const int tiles_n = (N + GEMM_BN - 1) / GEMM_BN;
  const long long tiles = static_cast<long long>((M + GEMM_BM - 1) / GEMM_BM) * tiles_n;
  const int sms = num_sms();
  if (batch == 1 && !a_mn_major && !b_mn_major && tma_epi && K <= GEMM_RES_MAX_K && tiles >= 4LL * sms &&
      tiles_n <= sms)
    return launch_gemm_resident(tmA, tmB, tmOut, p, sms, stream);
  if (!a_mn_major && !b_mn_major) return launch_gemm_epi<false, false>(tma_epi, tmA, tmB, tmOut, p, stream);
  if (!a_mn_major && b_mn_major) return launch_gemm_epi<false, true>(tma_epi, tmA, tmB, tmOut, p, stream);
  if (a_mn_major && b_mn_major) return launch_gemm_epi<true, true>(tma_epi, tmA, tmB, tmOut, p, stream);
  return launch_gemm_epi<true, false>(tma_epi, tmA, tmB, tmOut, p, stream);
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
