// Salient sampling locations of the correspondence loss with use_salience (reference src/modules.py:298-311, 357-364):
//
//     nz   = sample_nonzero_locations(salience, [B, fs, fs, 2])       one torch.randint per image, for both maps
//     reg  = torch.rand([B, fs, fs, 2]) * 2 - 1
//     keep = (torch.rand([B, fs, fs]) > .1).float()
//     coords = nz * keep + reg * (1 - keep)
//
// The reference finds each image's nonzeros with torch.nonzero and a boolean index, which makes the host wait for the
// device once per image.  Here one CTA per (map, image) unit builds the image's bitmap as 32-pixel ballot words with an
// exclusive popcount prefix (shared memory, or caller scratch for large maps), and every sample is located by a binary
// search over the prefix and __fns inside the word.
//
// Which generator a unit draws from depends on its count.  An image with nonzeros draws
// torch.randint(count, (n,)) without a device argument: on the CPU generator, so the caller needs the counts
// (salience_counts_kernel, one small copy to the host) and passes the n draws in.  An image without nonzeros draws
// randint(H, (n, 2)) on the CUDA generator: y from element 2 s, x from element 2 s + 1.  torch's CUDA randint (ATen
// random_from_to_kernel, range < 2^28) gives element li the value curand4(state).x % H with
// state = curand_init(seed, li, offset): Philox4x32-10 on the counter (offset / 4, li, 0) under the key seed, and each
// call advances the generator's offset by 4; the caller assigns each empty unit its offset.
//
// Coordinates: float(index) * fl(1 / H) * 2 - 1 for both components (the reference divides by t.shape[1] = H, and
// torch's CUDA division by a host scalar multiplies by its fp32 reciprocal), (x, y) order, every step rounded once.
#include <curand_philox4x32_x.h>

#include "common.cuh"
#include "host_util.h"

namespace stego {

constexpr int SAL_THREADS = 512, SAL_WARPS = SAL_THREADS / 32;
constexpr long long SAL_SMEM_WORDS = 12288;  // bitmap words a CTA keeps in shared memory: words + prefix = 96 KB
constexpr long long SAL_MAX_PIXELS = 1ll << 28;

struct SalParams {
  const void* mask[2];      // [B][H][W] contiguous, mask_bytes per element
  const float* ureg[2];     // [B][fs][fs][2] uniforms of the two reg draws
  const float* ukeep;       // [B][fs][fs] uniforms of the keep draw
  float* out[2];            // [B][fs][fs][2] coords1 / coords2 (may alias ureg)
  const uint32_t* draws;    // [2B][2 fs^2] draws: the CPU randint values, and the empty units' values without offsets
  const long long* offsets; // [2B] Philox offset of each empty unit, or null
  uint32_t* scratch;        // [2B][2 nwords] when the bitmap does not fit in shared memory, else null
  unsigned long long seed;
  float inv_h;
  int mask_bytes, B, H, W, fs, nwords;
};

__device__ __forceinline__ bool salient(const char* m, int bytes, long long i) {
  if (bytes == 4) return reinterpret_cast<const float*>(m)[i] != 0.0f;  // NaN counts, -0 does not
  return reinterpret_cast<const unsigned char*>(m)[i] != 0;
}

__device__ __forceinline__ uint32_t given_draw(const SalParams& p, int unit, uint32_t li) {
  return p.draws[static_cast<size_t>(unit) * 2 * p.fs * p.fs + li];
}

__device__ __forceinline__ uint32_t empty_draw(const SalParams& p, int unit, uint32_t li, uint2 key) {
  if (!p.offsets) return given_draw(p, unit, li);
  const unsigned long long q = static_cast<unsigned long long>(p.offsets[unit]) >> 2;
  return curand_Philox4x32_10(make_uint4(static_cast<uint32_t>(q), static_cast<uint32_t>(q >> 32), li, 0u), key).x;
}

__device__ __forceinline__ float unit_coord(int v, float inv_h) {
  return __fsub_rn(__fmul_rn(__fmul_rn(__int2float_rn(v), inv_h), 2.0f), 1.0f);
}

__global__ void __launch_bounds__(SAL_THREADS) salience_coords_kernel(SalParams p) {
  extern __shared__ uint32_t sal_smem[];
  __shared__ uint32_t warp_total[SAL_WARPS];
  const int unit = blockIdx.x, map = unit / p.B, b = unit - map * p.B;
  const int nw = p.nwords, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint32_t* words = p.scratch ? p.scratch + static_cast<size_t>(unit) * 2 * nw : sal_smem;
  uint32_t* prefix = words + nw;
  const long long hw = static_cast<long long>(p.H) * p.W;
  const char* m = static_cast<const char*>(p.mask[map]) + static_cast<size_t>(b) * hw * p.mask_bytes;

  // bitmap: warp k owns words [w0, w1); per pass lane j keeps the ballot of word base + j, then a warp scan of the
  // popcounts gives the warp-local exclusive prefix
  const int chunk = (nw + SAL_WARPS - 1) / SAL_WARPS;
  const int w0 = min(nw, warp * chunk), w1 = min(nw, w0 + chunk);
  uint32_t run = 0;
  for (int base = w0; base < w1; base += 32) {
    const int cnt = min(32, w1 - base);
    uint32_t mine = 0;
    for (int j = 0; j < cnt; ++j) {
      const long long px = static_cast<long long>(base + j) * 32 + lane;
      const uint32_t bal = __ballot_sync(0xffffffffu, px < hw && salient(m, p.mask_bytes, px));
      if (lane == j) mine = bal;
    }
    const uint32_t c = __popc(mine);
    uint32_t incl = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += v;
    }
    if (lane < cnt) {
      words[base + lane] = mine;
      prefix[base + lane] = run + incl - c;
    }
    run += __shfl_sync(0xffffffffu, incl, 31);
  }
  if (lane == 0) warp_total[warp] = run;
  __syncthreads();
  uint32_t offset = 0, total = 0;
  for (int k = 0; k < SAL_WARPS; ++k) {
    if (k < warp) offset += warp_total[k];
    total += warp_total[k];
  }
  if (offset)
    for (int w = w0 + lane; w < w1; w += 32) prefix[w] += offset;
  __syncthreads();

  const int n = p.fs * p.fs;
  const uint2 key = make_uint2(static_cast<uint32_t>(p.seed), static_cast<uint32_t>(p.seed >> 32));
  const float* ureg = p.ureg[map];
  float* out = p.out[map];
  for (int s = threadIdx.x; s < n; s += SAL_THREADS) {
    int y, x;
    if (total > 0) {
      const uint32_t r = given_draw(p, unit, s) % total;
      int lo = 0, hi = nw - 1;  // the last word whose exclusive prefix is <= r holds the r-th nonzero
      while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (prefix[mid] <= r) lo = mid; else hi = mid - 1;
      }
      const long long px = static_cast<long long>(lo) * 32 + __fns(words[lo], 0, static_cast<int>(r - prefix[lo]) + 1);
      y = static_cast<int>(px / p.W);
      x = static_cast<int>(px - static_cast<long long>(y) * p.W);
    } else {
      y = static_cast<int>(empty_draw(p, unit, 2 * s, key) % static_cast<uint32_t>(p.H));
      x = static_cast<int>(empty_draw(p, unit, 2 * s + 1, key) % static_cast<uint32_t>(p.H));
    }
    const size_t e = static_cast<size_t>(b) * n + s;
    const float keep = p.ukeep[e] > 0.1f ? 1.0f : 0.0f;  // fp32 comparison: u == 0.1f is not kept
    const float drop = __fsub_rn(1.0f, keep);
    const float nzx = unit_coord(x, p.inv_h), nzy = unit_coord(y, p.inv_h);
    const float rx = __fsub_rn(__fmul_rn(ureg[2 * e], 2.0f), 1.0f);
    const float ry = __fsub_rn(__fmul_rn(ureg[2 * e + 1], 2.0f), 1.0f);
    out[2 * e] = __fadd_rn(__fmul_rn(nzx, keep), __fmul_rn(rx, drop));
    out[2 * e + 1] = __fadd_rn(__fmul_rn(nzy, keep), __fmul_rn(ry, drop));
  }
}

// counts[u] = nonzeros of unit u's mask, one CTA per unit
__global__ void __launch_bounds__(SAL_THREADS) salience_counts_kernel(const void* m0, const void* m1, int mask_bytes,
                                                                     int B, long long hw, int* counts) {
  __shared__ uint32_t warp_total[SAL_WARPS];
  const int unit = blockIdx.x, map = unit / B, b = unit - map * B;
  const char* m = static_cast<const char*>(map ? m1 : m0) + static_cast<size_t>(b) * hw * mask_bytes;
  uint32_t c = 0;
  for (long long i = threadIdx.x; i < hw; i += SAL_THREADS) c += salient(m, mask_bytes, i);
#pragma unroll
  for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0) warp_total[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t t = 0;
    for (int k = 0; k < SAL_WARPS; ++k) t += warp_total[k];
    counts[unit] = static_cast<int>(t);
  }
}

static long long sal_words(int H, int W) { return (static_cast<long long>(H) * W + 31) / 32; }

}  // namespace stego

using namespace stego;

// C-ABI: see include/stego_b200.h for the contract.
extern "C" long long stego_salience_scratch_bytes(int B, int H, int W) {
  if (B < 1 || H < 1 || W < 1) return 0;
  const long long nw = sal_words(H, W);
  return nw <= SAL_SMEM_WORDS ? 0 : 2ll * B * 2 * nw * 4;
}

extern "C" int stego_salience_counts(const void* salience, const void* salience_pos, int mask_bytes, int B, int H,
                                     int W, int* counts, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(salience && salience_pos && counts, "stego_salience_counts: null pointer");
  STEGO_CHECK_ARG(mask_bytes == 1 || mask_bytes == 4, "stego_salience_counts: mask_bytes=%d (1 or 4)", mask_bytes);
  STEGO_CHECK_ARG(B >= 1 && H >= 1 && W >= 1, "stego_salience_counts: B=%d H=%d W=%d must be >= 1", B, H, W);
  STEGO_CHECK_ARG(static_cast<long long>(H) * W < SAL_MAX_PIXELS, "stego_salience_counts: H*W=%lld must be < 2^28",
                  static_cast<long long>(H) * W);
  salience_counts_kernel<<<2 * B, SAL_THREADS, 0, stream>>>(salience, salience_pos, mask_bytes, B,
                                                            static_cast<long long>(H) * W, counts);
  STEGO_CHECK_LAUNCH("salience_counts_kernel launch");
  return STEGO_OK;
}

extern "C" int stego_salience_coords(const void* salience, const void* salience_pos, int mask_bytes, int B, int H,
                                     int W, int feature_samples, long long seed, const long long* offsets,
                                     const void* draws_u32, const float* u_reg1, const float* u_reg2,
                                     const float* u_keep, float* coords1, float* coords2, void* scratch,
                                     void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(salience && salience_pos && draws_u32 && u_reg1 && u_reg2 && u_keep && coords1 && coords2,
                  "stego_salience_coords: null pointer");
  STEGO_CHECK_ARG(mask_bytes == 1 || mask_bytes == 4, "stego_salience_coords: mask_bytes=%d (1 or 4)", mask_bytes);
  STEGO_CHECK_ARG(B >= 1 && H >= 1 && W >= 1, "stego_salience_coords: B=%d H=%d W=%d must be >= 1", B, H, W);
  STEGO_CHECK_ARG(static_cast<long long>(H) * W < SAL_MAX_PIXELS, "stego_salience_coords: H*W=%lld must be < 2^28",
                  static_cast<long long>(H) * W);
  STEGO_CHECK_ARG(feature_samples >= 1 && feature_samples <= 64, "stego_salience_coords: feature_samples=%d (1..64)",
                  feature_samples);
  const long long nw = sal_words(H, W);
  const bool in_smem = nw <= SAL_SMEM_WORDS;
  STEGO_CHECK_ARG(in_smem || scratch, "stego_salience_coords: H*W=%lld needs scratch of "
                  "stego_salience_scratch_bytes bytes", static_cast<long long>(H) * W);
  SalParams p;
  p.mask[0] = salience; p.mask[1] = salience_pos;
  p.ureg[0] = u_reg1; p.ureg[1] = u_reg2; p.ukeep = u_keep;
  p.out[0] = coords1; p.out[1] = coords2;
  p.draws = static_cast<const uint32_t*>(draws_u32);
  p.offsets = offsets;
  p.scratch = in_smem ? nullptr : static_cast<uint32_t*>(scratch);
  p.seed = static_cast<unsigned long long>(seed);
  p.inv_h = 1.0f / static_cast<float>(H);
  p.mask_bytes = mask_bytes; p.B = B; p.H = H; p.W = W; p.fs = feature_samples; p.nwords = static_cast<int>(nw);
  const size_t smem = in_smem ? static_cast<size_t>(nw) * 8 : 0;
  int rc = opt_in_smem<salience_coords_kernel>(static_cast<size_t>(SAL_SMEM_WORDS) * 8, "salience_coords_kernel");
  if (rc != STEGO_OK) return rc;
  salience_coords_kernel<<<2 * B, SAL_THREADS, smem, stream>>>(p);
  STEGO_CHECK_LAUNCH("salience_coords_kernel launch");
  return STEGO_OK;
}
