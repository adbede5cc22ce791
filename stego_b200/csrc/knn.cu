// Fused k-nearest-neighbour search over L2-normalised image descriptors (SURVEY.md §8(f) rank 1, the step that
// PRODUCES img_pos for the training path).
//
// Reference: src/precompute_knns.py:15-21 (get_feats: F.normalize(model(img).mean([2, 3]), dim=1)) and :83-96
//     pairwise_sims = torch.einsum("nf,mf->nm", batch_feats, normed_feats);  all_nns.append(torch.topk(pairwise_sims, 30)[1])
// The reference materialises an [n/16, n] fp32 similarity slab per batch on the host (n = 118 K for COCO: 3.5 GB per
// slab, 14 G similarities in total).  Here the similarity tile never leaves the SM: S = F F^T accumulates in registers
// (bf16 hi/lo split, three wgmma passes = ~2^-16 relative accuracy, enough to rank neighbours), is staged transposed in
// shared memory, and two scan threads per query row (one per half of the key tile) keep a running top-k in a sorted
// private list, compared against a register threshold (an insert happens ~k ln(n/k) times per row, everything else
// is one FSETP per similarity).  The two lists of a row are merged once per row block.
//
//   knn_prep_kernel   : fp32 [n][E] -> L2-normalise (eps 1e-12 like F.normalize) -> bf16 hi / lo planes [2][n][E]
//   knn_topk_kernel   : persistent CTAs, one 128-row query block at a time against all 128-column key tiles
//       warpgroups 0,1  wgmma for query rows 0..63 / 64..127: 3 passes (hi.hi, hi.lo, lo.hi) x E/64 k-blocks per tile,
//                       then the scan of those rows; after the last tile the row's k indices (descending similarity,
//                       ties -> lower index first) are written as int64
//       warpgroup 2     TMA producer (A = query rows, B = key rows, both from the same planes tensor, 3-stage ring)
#include "common.cuh"
#include "host_util.h"

namespace stego {

constexpr int KNN_BM = 128, KNN_BN = 128, KNN_BK = 64, KNN_STAGES = 3, KNN_THREADS = 384, KNN_MAXK = 32;
constexpr uint32_t KNN_A_BYTES = KNN_BM * KNN_BK * 2;   // 16 KB
constexpr uint32_t KNN_B_BYTES = KNN_BN * KNN_BK * 2;   // 16 KB
constexpr uint32_t KNN_STAGE_BYTES = KNN_A_BYTES + KNN_B_BYTES;
constexpr int KNN_ST_LD = KNN_BM + 4;                   // transposed score tile [key col][query row], padded
constexpr uint32_t KNN_ST_BYTES = KNN_BN * KNN_ST_LD * 4;
constexpr uint32_t KNN_MERGE_BYTES = KNN_BM * KNN_MAXK * 8;  // second-half lists: [row][k] value + index
constexpr size_t KNN_SMEM = size_t(KNN_STAGES) * KNN_STAGE_BYTES + KNN_ST_BYTES + KNN_MERGE_BYTES + 1024 + 256;

struct KnnParams {
  int n, E, k;
  long long* idx_out;  // [n][k]
  float* val_out;      // [n][k] or null
};

__global__ void knn_prep_kernel(const float* __restrict__ x, bf16* __restrict__ planes, int n, int E) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= n) return;
  const float* xr = x + static_cast<size_t>(row) * E;
  float ss = 0.f;
  for (int c = lane; c < E; c += 32) ss = fmaf(xr[c], xr[c], ss);
  ss = warp_sum(ss);
  const float inv = 1.0f / fmaxf(sqrtf(ss), 1e-12f);
  bf16* hi = planes + static_cast<size_t>(row) * E;
  bf16* lo = planes + (static_cast<size_t>(n) + row) * E;
  for (int c = lane; c < E; c += 32) {
    const float v = xr[c] * inv;
    const bf16 h = __float2bfloat16_rn(v);
    hi[c] = h;
    lo[c] = __float2bfloat16_rn(v - __bfloat162float(h));
  }
}

__global__ void __launch_bounds__(KNN_THREADS, 1)
knn_topk_kernel(const __grid_constant__ CUtensorMap tmF, KnnParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  float* st = reinterpret_cast<float*>(smem + KNN_STAGES * KNN_STAGE_BYTES);
  float* merge_v = reinterpret_cast<float*>(smem + KNN_STAGES * KNN_STAGE_BYTES + KNN_ST_BYTES);
  int* merge_i = reinterpret_cast<int*>(merge_v + KNN_BM * KNN_MAXK);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + KNN_STAGES * KNN_STAGE_BYTES + KNN_ST_BYTES + KNN_MERGE_BYTES);
  uint64_t* empty_bar = full_bar + KNN_STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int row_blocks = (p.n + KNN_BM - 1) / KNN_BM;
  const int col_tiles = (p.n + KNN_BN - 1) / KNN_BN;
  const int nkb = p.E / KNN_BK;
  const int ksteps = 3 * nkb;  // pass 0: A hi x B hi, pass 1: A hi x B lo, pass 2: A lo x B hi

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmF);
    for (int s = 0; s < KNN_STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);  // one arrive per MMA warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= 8) {
    // ===================== TMA producer =====================
    warpgroup_reg_dealloc<40>();
    if (warp == 8 && lane == 0) {
      uint32_t stage = 0, phase = 0;
      for (int rb = blockIdx.x; rb < row_blocks; rb += gridDim.x) {
        for (int ct = 0; ct < col_tiles; ++ct) {
          for (int ks = 0; ks < ksteps; ++ks) {
            const int pass = ks / nkb, kb = ks - pass * nkb;
            const int pa = (pass == 2) ? 1 : 0, pb = (pass == 1) ? 1 : 0;
            mbar_wait(&empty_bar[stage], phase ^ 1u);
            uint8_t* sa = smem + stage * KNN_STAGE_BYTES;
            uint8_t* sb = sa + KNN_A_BYTES;
            mbar_arrive_expect_tx(&full_bar[stage], KNN_STAGE_BYTES);
            tma_load_3d(sa, &tmF, &full_bar[stage], kb * KNN_BK, rb * KNN_BM, pa);
            tma_load_3d(sb, &tmF, &full_bar[stage], kb * KNN_BK, ct * KNN_BN, pb);
            if (++stage == KNN_STAGES) { stage = 0; phase ^= 1u; }
          }
        }
      }
    }
    return;
  }

  // ===================== MMA + scan warpgroups =====================
  warpgroup_reg_alloc<232>();
  const int mwg = warp >> 2;
  const int t128 = threadIdx.x & 127;
  const bool leader = t128 == 0;
  const int wq = warp & 3;
  constexpr uint32_t DESC_HI = smem_desc_hi_sw128(1024);
  const uint32_t a_lo0 = smem_desc_lo(smem_u32(smem) + mwg * (KNN_A_BYTES / 2), 16);
  const uint32_t b_lo0 = smem_desc_lo(smem_u32(smem) + KNN_A_BYTES, 16);
  // scan role: query row `srow` of the tile, key columns [64 half, 64 half + 64) of every key tile
  const int srow = mwg * 64 + (t128 & 63);
  const int half = t128 >> 6;
  const int k = p.k;
  uint32_t stage = 0, phase = 0;
  float tv[KNN_MAXK];  // sorted descending; dynamic indexing -> local memory (touched only on inserts)
  int ti[KNN_MAXK];
  float acc[KNN_BN / 2];
  for (int rb = blockIdx.x; rb < row_blocks; rb += gridDim.x) {
#pragma unroll 1
    for (int i = 0; i < KNN_MAXK; ++i) { tv[i] = -INFINITY; ti[i] = -1; }
    float thr = -INFINITY;  // similarity of the current k-th neighbour
    for (int ct = 0; ct < col_tiles; ++ct) {
#pragma unroll
      for (int j = 0; j < KNN_BN / 2; ++j) acc[j] = 0.f;
      uint32_t prev = 0;
      for (int ks = 0; ks < ksteps; ++ks) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t a_lo = a_lo0 + stage * (KNN_STAGE_BYTES >> 4);
        const uint32_t b_lo = b_lo0 + stage * (KNN_STAGE_BYTES >> 4);
        fence_operands(acc);
        wgmma_fence();
#pragma unroll
        for (uint32_t kk = 0; kk < KNN_BK / 16; ++kk)
          wgmma_ss<KNN_BN, 0, 0>(acc, smem_desc_join(a_lo + 2 * kk, DESC_HI), smem_desc_join(b_lo + 2 * kk, DESC_HI), 1u);
        wgmma_commit();
        wgmma_wait<1>();
        if (ks > 0 && leader) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == KNN_STAGES) { stage = 0; phase ^= 1u; }
      }
      wgmma_wait<0>();
      fence_operands(acc);
      if (leader) mbar_arrive(&empty_bar[prev]);
      // stage the tile transposed (bank-conflict-free both ways); this warpgroup's previous scan must be over
      asm volatile("bar.sync %0, 128;\n" ::"r"(1 + mwg) : "memory");
#pragma unroll
      for (int t = 0; t < KNN_BN / 2; ++t) {
        const int r = mwg * 64 + wq * 16 + (lane >> 2) + 8 * ((t >> 1) & 1);
        const int col = 8 * (t >> 2) + 2 * (lane & 3) + (t & 1);
        st[col * KNN_ST_LD + r] = acc[t];
      }
      asm volatile("bar.sync %0, 128;\n" ::"r"(1 + mwg) : "memory");
      const int col0 = ct * KNN_BN + half * 64;
#pragma unroll 1
      for (int c = 0; c < 64; c += 32) {
        if (col0 + c >= p.n) break;  // warp-uniform: key rows past n are zero-filled padding
        float v[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] = st[(half * 64 + c + j) * KNN_ST_LD + srow];
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          const float s = v[j];
          const int col = col0 + c + j;
          if (s > thr && col < p.n) {
            int pos = k - 1;
            while (pos > 0 && tv[pos - 1] < s) {  // strict: earlier (lower) columns stay ahead on ties
              tv[pos] = tv[pos - 1];
              ti[pos] = ti[pos - 1];
              --pos;
            }
            tv[pos] = s;
            ti[pos] = col;
            thr = tv[k - 1];
          }
        }
      }
    }
    // merge the two half lists of every row: (value desc, index asc), the order a single scan would produce
    if (half == 1) {
      for (int i = 0; i < k; ++i) {
        merge_v[srow * KNN_MAXK + i] = tv[i];
        merge_i[srow * KNN_MAXK + i] = ti[i];
      }
    }
    asm volatile("bar.sync %0, 128;\n" ::"r"(1 + mwg) : "memory");
    const int row = rb * KNN_BM + srow;
    if (half == 0 && row < p.n) {
      int ia = 0, ib = 0;
      for (int i = 0; i < k; ++i) {
        const float vb = merge_v[srow * KNN_MAXK + ib];
        const int xb = merge_i[srow * KNN_MAXK + ib];
        const bool take_a = tv[ia] > vb || (tv[ia] == vb && ti[ia] >= 0 && (xb < 0 || ti[ia] < xb));
        const float v = take_a ? tv[ia] : vb;
        const int x = take_a ? ti[ia] : xb;
        if (take_a) ++ia; else ++ib;
        p.idx_out[static_cast<size_t>(row) * k + i] = x;
        if (p.val_out) p.val_out[static_cast<size_t>(row) * k + i] = v;
      }
    }
    asm volatile("bar.sync %0, 128;\n" ::"r"(1 + mwg) : "memory");  // merge buffer free for the next row block
  }
}

}  // namespace stego

using namespace stego;

// C-ABI: see include/stego_b200.h for the contract.
extern "C" int stego_knn_topk(const float* feats, int n, int E, int k, void* planes_scratch, long long* idx_out,
                              float* val_out, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(feats && planes_scratch && idx_out, "stego_knn_topk: null pointer");
  STEGO_CHECK_ARG(n > 0 && E > 0 && E % KNN_BK == 0, "stego_knn_topk: E=%d must be a positive multiple of 64", E);
  STEGO_CHECK_ARG(k >= 1 && k <= KNN_MAXK && k <= n, "stego_knn_topk: k=%d (1..%d, <= n)", k, KNN_MAXK);
  STEGO_CHECK_ARG((reinterpret_cast<uintptr_t>(planes_scratch) & 15u) == 0, "stego_knn_topk: planes_scratch not 16-byte aligned");
  knn_prep_kernel<<<(n + 7) / 8, 256, 0, stream>>>(feats, reinterpret_cast<bf16*>(planes_scratch), n, E);
  STEGO_CHECK_LAUNCH("knn_prep_kernel launch");
  CUtensorMap tm;
  uint64_t dims[3] = {(uint64_t)E, (uint64_t)n, 2};
  uint64_t str[2] = {(uint64_t)E * 2, (uint64_t)n * E * 2};
  uint32_t box[3] = {64, 128, 1};  // KNN_BM = KNN_BN = 128 rows
  int rc = make_tmap_bf16(&tm, planes_scratch, 3, dims, str, box);
  if (rc != STEGO_OK) return rc;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(knn_topk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)KNN_SMEM);
    if (e != cudaSuccess) return cuda_fail(e, "cudaFuncSetAttribute(knn_topk)");
    configured = true;
  }
  KnnParams p;
  p.n = n; p.E = E; p.k = k; p.idx_out = idx_out; p.val_out = val_out;
  const int row_blocks = (n + KNN_BM - 1) / KNN_BM;
  const int grid = row_blocks < num_sms() ? row_blocks : num_sms();
  knn_topk_kernel<<<grid, KNN_THREADS, KNN_SMEM, stream>>>(tm, p);
  STEGO_CHECK_LAUNCH("knn_topk_kernel launch");
  return STEGO_OK;
}
