// Fused feature-correspondence loss for STEGO (sm_90a): sampling + L2-norm, the tensor_correlation
// einsum on wgmma, the centre/shift/clamp/product reduction, and the full backward.
//
// Reference: src/modules.py
//   :275-276 norm, :283-284 tensor_correlation (einsum nchw,ncij->nhwij), :287-288 sample (grid_sample),
//   :325-347 ContrastiveCorrelationLoss.helper, :349-398 ContrastiveCorrelationLoss.forward.
//
// Pipeline (K = 2 + neg_samples helper "calls", S = feature_samples^2 sampled points per image, padded to R = whole
// 128-row tiles):
//   1. sample_norm_*  : bilinear 4-tap gather (border, align_corners=True) of S points per image for every
//                       distinct operand ("slot": 0 = img@coords1, 1 = pos@coords2, 2.. = img[perm_i]@coords2),
//                       L2-normalise over channels in fp32, write [R][C] operand tiles as a bf16 hi/lo SPLIT
//                       (x = hi + lo).  The einsum is then three bf16 tensor-core passes
//                       hi.hi + lo.hi + hi.lo, i.e. ~2^-16 relative accuracy with fp32 accumulation.
//   2. corr_kernel    : TMA-staged tiles -> wgmma -> fd and cd accumulators of one 128x128 block in the registers of
//                       two warpgroups (64 rows each); epilogue straight on the accumulator fragments.  For S <= 128
//                       one CTA per (image, call) holds whole rows: row means (pointwise centring), clamp, shift,
//                       product, five partial sums per CTA.  For larger S, per-row partials per block (see section 2).
//   3. corr_finish    : per call: old_mean, loss mean, cd mean (corr_tiled_finish: also the row means, fp64).
//   4. corr_kernel    : backward phases: recompute fd, cd, form G = dL/dfd, run dA = G . Bc and dB = G^T . Ac on the
//                       tensor cores and accumulate into per-slot gradient tiles.
//   5. sample_norm_bwd: normalisation backward + grid_sample backward (per-pixel gather of the 4-tap contributions
//                       into d_code, fixed order, no atomics).
#include "common.cuh"
#include "host_util.h"
#include "probe_common.cuh"
#include "taps.cuh"
#include "tb_hist.cuh"

namespace stego {

constexpr int CL_ROWS = 128;     // rows of one operand tile
constexpr int CL_CODE_PAD = 128; // code channels padded to 2 k-blocks
constexpr int CL_MAX_CALLS = 16;
constexpr int CL_DT_LD = 96;     // row stride (floats) of the per-slot gradient tiles: every code channel (D <= 96)
constexpr int CT_MAX_FS = 64;    // largest feature_samples (S = 4096 points per image)
constexpr int CL_PR_BINS = 4096; // score bins of the precision-recall counts (STEGO_PR_BINS)

// ---------------------------------------------------------------------------------------------
// 1. sampling + normalisation
// ---------------------------------------------------------------------------------------------
struct SampleParams {
  const void* src;      // slot 0 and slots >= 2 (through perm)
  const void* src_pos;  // slot 1
  int src_bf16;         // element type of both sources
  int label_bytes;      // label source (sample_labels_kernel): width of one label, 8 / 4 / 1
  long long sb, sc, sy, sx;  // element strides (batch, channel, y, x) — shared by src and src_pos
  const float* chan_scale;      // optional [B][C] per-(image,channel) multiplier (Dropout2d noise), slot 0/2+
  const float* chan_scale_pos;  // same for src_pos
  const float* coords1;  // [B][fs][fs][2]
  const float* coords2;
  const long long* perms;  // [nslots-2][B]
  int perms_raw;           // 1: perms are raw randperm draws; apply super_perm's fix-up (p == b -> (p+1) % B) here
  bf16* tiles;             // [2 planes][nslots][B][R][Cpad]
  int B, C, Cpad, H, W, fs, S, nslots;
  int R;                   // rows per (plane, slot, image) of the operand and gradient tiles: S rounded up to 128s
  float eps;
};

// grid_sample(bilinear, padding_mode='border', align_corners=True) source taps (taps.cuh) for sample index
// s = i*fs + j, which reads coords[b][j][i] because `sample` permutes the grid (modules.py:288).
__device__ __forceinline__ Taps make_taps(const float* coords, int b, int s, int fs, int H, int W) {
  const int i = s / fs, j = s % fs;
  const float* cp = coords + ((static_cast<long long>(b) * fs + j) * fs + i) * 2;
  return grid_taps(cp[0], cp[1], H, W);
}

__device__ __forceinline__ void slot_source(const SampleParams& p, int slot, int b, const void*& src,
                                            const float*& cscale, const float*& coords, int& img) {
  if (slot == 0) { src = p.src; cscale = p.chan_scale; coords = p.coords1; img = b; }
  else if (slot == 1) { src = p.src_pos; cscale = p.chan_scale_pos; coords = p.coords2; img = b; }
  else {
    src = p.src; cscale = p.chan_scale; coords = p.coords2;
    img = static_cast<int>(p.perms[(slot - 2) * p.B + b]);
    if (p.perms_raw && img == b) img = (img + 1) % p.B;  // modules.py:291-295
  }
}

// One warp per tile row: row s of (slot, image b) in block (s / 8, slot * B + b).  Generic strides / dtypes; each
// lane owns channels lane, lane+32, ...
// kLabels: the source is a label map [B][H][W] (strides sb, sy, sx; sc unused) read as the C = n_classes + 1 channel
// map one_hot_feats(label + 1, C) of train_segmentation.py:135-137 (utils.py:65-66) without materialising it: channel c
// of a tap is 1 when the tap's class is c, else 0.  A label outside 0 .. n_classes - 1 (-1, uint8 255, any other value)
// is class 0, where F.one_hot would raise on values >= n_classes or < -1.  The products and sums below are then the
// ones the feature path computes on the materialised fp32 one-hot map (times 0 or 1 and adding 0 are exact): the tiles
// are bit-identical.  One body, two kernels: sample_norm_kernel (features) and sample_labels_kernel (labels).
template <int NV, bool kLabels>  // NV = Cpad / 32
__device__ __forceinline__ void sample_norm_row(const SampleParams& p) {
  const int R = p.R;
  const int s = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);  // grid (R / 8, nslots * B)
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.y % p.B;
  const int slot = blockIdx.y / p.B;
  const size_t plane = static_cast<size_t>(p.nslots) * p.B * R * p.Cpad;
  bf16* hi = p.tiles + (static_cast<size_t>(slot) * p.B + b) * R * p.Cpad + static_cast<size_t>(s) * p.Cpad;
  bf16* lo = hi + plane;
  float v[NV];
  if (s >= p.S) {
#pragma unroll
    for (int k = 0; k < NV; ++k) { hi[lane + 32 * k] = __float2bfloat16_rn(0.f); lo[lane + 32 * k] = __float2bfloat16_rn(0.f); }
    return;
  }
  const void* src; const float* cscale; const float* coords; int img;
  slot_source(p, slot, b, src, cscale, coords, img);
  const Taps t = make_taps(coords, b, s, p.fs, p.H, p.W);
  // pixel offset -> element offset
  auto off = [&](int pix) { return static_cast<long long>(pix / p.W) * p.sy + static_cast<long long>(pix % p.W) * p.sx; };
  const long long o00 = off(t.i00), o01 = off(t.i01), o10 = off(t.i10), o11 = off(t.i11);
  const long long base = static_cast<long long>(img) * p.sb;
  int k00 = 0, k01 = 0, k10 = 0, k11 = 0;  // classes of the four taps (label source)
  if constexpr (kLabels) {
    auto cls = [&](long long o) {
      const long long l = read_label(src, p.label_bytes, base + o);
      return (l >= 0 && l < p.C - 1) ? static_cast<int>(l) + 1 : 0;
    };
    k00 = cls(o00); k01 = cls(o01); k10 = cls(o10); k11 = cls(o11);
  }
  float ss = 0.f;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    const int c = lane + 32 * k;
    float val = 0.f;
    if (c < p.C) {
      const long long cb = base + static_cast<long long>(c) * p.sc;
      float a00, a01, a10, a11;
      if constexpr (kLabels) {
        a00 = k00 == c ? 1.f : 0.f; a01 = k01 == c ? 1.f : 0.f;
        a10 = k10 == c ? 1.f : 0.f; a11 = k11 == c ? 1.f : 0.f;
      } else if (p.src_bf16) {
        const bf16* q = reinterpret_cast<const bf16*>(src) + cb;
        a00 = __bfloat162float(q[o00]); a01 = __bfloat162float(q[o01]);
        a10 = __bfloat162float(q[o10]); a11 = __bfloat162float(q[o11]);
      } else {
        const float* q = reinterpret_cast<const float*>(src) + cb;
        a00 = q[o00]; a01 = q[o01]; a10 = q[o10]; a11 = q[o11];
      }
      // same accumulation order as ATen's grid_sampler_2d: nw, ne, sw, se
      val = a00 * t.w00;
      val += a01 * t.w01;
      val += a10 * t.w10;
      val += a11 * t.w11;
      if (cscale) val *= cscale[static_cast<long long>(img) * p.C + c];
    }
    v[k] = val;
    ss += val * val;
  }
  ss = warp_sum(ss);
  const float inv = 1.0f / fmaxf(sqrtf(ss), p.eps);
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    const float n = v[k] * inv;
    const bf16 h = __float2bfloat16_rn(n);
    hi[lane + 32 * k] = h;
    lo[lane + 32 * k] = __float2bfloat16_rn(n - __bfloat162float(h));
  }
}

template <int NV>
__global__ void __launch_bounds__(256) sample_norm_kernel(SampleParams p) { sample_norm_row<NV, false>(p); }

template <int NV>
__global__ void __launch_bounds__(256) sample_labels_kernel(SampleParams p) { sample_norm_row<NV, true>(p); }

// Pure class id of each sample point, for the precision-recall counts (CP_PR): ids[slot][b][s] = c when every tap of
// make_taps with a non-zero weight has class c, else -1 ("mixed").  A tap's class is sample_labels_kernel's: label + 1
// for 0 <= label < n_classes, else 0.  Slot 0 samples image b at coords1, slot 1 the same image at coords2.  In fp32 a
// tap weight is zero exactly when its exact value is, so "pure" is exactly "the sampled one-hot vector is e_c".  One
// thread per sample; rows S .. R - 1 of ids are not written (CP_PR never reads them).
__global__ void __launch_bounds__(256)
sample_label_ids_kernel(const void* label, int label_bytes, const float* coords1, const float* coords2, int* ids, int B,
                        int n_classes, int H, int W, int fs, int R) {
  const int S = fs * fs;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= 2ll * B * S) return;
  const int s = static_cast<int>(idx % S);
  const int sb = static_cast<int>(idx / S);  // slot * B + b
  const int b = sb % B;
  const Taps t = make_taps(sb >= B ? coords2 : coords1, b, s, fs, H, W);
  const long long base = static_cast<long long>(b) * H * W;
  int c = -1;
  bool mixed = false;
  auto visit = [&](float w, int pix) {
    if (w == 0.f) return;
    const long long l = read_label(label, label_bytes, base + pix);
    const int k = (l >= 0 && l < n_classes) ? static_cast<int>(l) + 1 : 0;
    if (c < 0) c = k;
    else if (k != c) mixed = true;
  };
  visit(t.w00, t.i00);
  visit(t.w01, t.i01);
  visit(t.w10, t.i10);
  visit(t.w11, t.i11);
  ids[static_cast<size_t>(sb) * R + s] = mixed ? -1 : c;
}

// Vectorised variant for the layout the training step uses: bf16 source, channel stride 1 (tokens-major),
// C % 8 == 0, Cpad == C.  Each lane owns 8 consecutive channels per step: four 16-byte tap loads, two 16-byte tile
// stores (hi, lo) — 8x fewer memory instructions than the generic kernel.
template <int NI>  // NI = ceil(C / 256)
__global__ void __launch_bounds__(256)
sample_norm_vec8_kernel(SampleParams p) {
  const int R = p.R;
  const int s = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);  // grid (R / 8, nslots * B)
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.y % p.B;
  const int slot = blockIdx.y / p.B;
  const size_t plane = static_cast<size_t>(p.nslots) * p.B * R * p.Cpad;
  bf16* hi = p.tiles + (static_cast<size_t>(slot) * p.B + b) * R * p.Cpad + static_cast<size_t>(s) * p.Cpad;
  bf16* lo = hi + plane;
  if (s >= p.S) {
#pragma unroll
    for (int i = 0; i < NI; ++i) {
      const int c = (lane + 32 * i) * 8;
      if (c < p.C) {
        *reinterpret_cast<uint4*>(hi + c) = make_uint4(0, 0, 0, 0);
        *reinterpret_cast<uint4*>(lo + c) = make_uint4(0, 0, 0, 0);
      }
    }
    return;
  }
  const void* src; const float* cscale; const float* coords; int img;
  slot_source(p, slot, b, src, cscale, coords, img);
  const Taps t = make_taps(coords, b, s, p.fs, p.H, p.W);
  auto off = [&](int pix) { return static_cast<long long>(pix / p.W) * p.sy + static_cast<long long>(pix % p.W) * p.sx; };
  const bf16* q = reinterpret_cast<const bf16*>(src) + static_cast<long long>(img) * p.sb;
  const bf16* q00 = q + off(t.i00);
  const bf16* q01 = q + off(t.i01);
  const bf16* q10 = q + off(t.i10);
  const bf16* q11 = q + off(t.i11);
  float v[NI][8];
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < NI; ++i) {
    const int c = (lane + 32 * i) * 8;
    if (c < p.C) {
      const uint4 a00 = *reinterpret_cast<const uint4*>(q00 + c), a01 = *reinterpret_cast<const uint4*>(q01 + c);
      const uint4 a10 = *reinterpret_cast<const uint4*>(q10 + c), a11 = *reinterpret_cast<const uint4*>(q11 + c);
      const __nv_bfloat162* h00 = reinterpret_cast<const __nv_bfloat162*>(&a00);
      const __nv_bfloat162* h01 = reinterpret_cast<const __nv_bfloat162*>(&a01);
      const __nv_bfloat162* h10 = reinterpret_cast<const __nv_bfloat162*>(&a10);
      const __nv_bfloat162* h11 = reinterpret_cast<const __nv_bfloat162*>(&a11);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 f00 = __bfloat1622float2(h00[k]), f01 = __bfloat1622float2(h01[k]);
        const float2 f10 = __bfloat1622float2(h10[k]), f11 = __bfloat1622float2(h11[k]);
        float x = f00.x * t.w00; x += f01.x * t.w01; x += f10.x * t.w10; x += f11.x * t.w11;
        float y = f00.y * t.w00; y += f01.y * t.w01; y += f10.y * t.w10; y += f11.y * t.w11;
        if (cscale) {
          x *= cscale[static_cast<long long>(img) * p.C + c + 2 * k];
          y *= cscale[static_cast<long long>(img) * p.C + c + 2 * k + 1];
        }
        v[i][2 * k] = x;
        v[i][2 * k + 1] = y;
        ss += x * x + y * y;
      }
    } else {
#pragma unroll
      for (int k = 0; k < 8; ++k) v[i][k] = 0.f;
    }
  }
  ss = warp_sum(ss);
  const float inv = 1.0f / fmaxf(sqrtf(ss), p.eps);
#pragma unroll
  for (int i = 0; i < NI; ++i) {
    const int c = (lane + 32 * i) * 8;
    if (c < p.C) {
      uint32_t wh[4], wl[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float n0 = v[i][2 * k] * inv, n1 = v[i][2 * k + 1] * inv;
        const float h0 = __bfloat162float(__float2bfloat16_rn(n0)), h1 = __bfloat162float(__float2bfloat16_rn(n1));
        wh[k] = pack_bf16x2(h0, h1);
        wl[k] = pack_bf16x2(n0 - h0, n1 - h1);
      }
      *reinterpret_cast<uint4*>(hi + c) = make_uint4(wh[0], wh[1], wh[2], wh[3]);
      *reinterpret_cast<uint4*>(lo + c) = make_uint4(wl[0], wl[1], wl[2], wl[3]);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// 2./4. correlation + loss forward / backward
//
// The operand tiles hold R rows per (plane, slot, image), i.e. nT = R / 128 row tiles.  A work unit is one 128x128
// (row tile rt, column tile ct) block of fd / cd for one (image, call).  Two schedules share one kernel body:
//   whole row  (S <= 128, R = 128, nT = 1): the unit holds entire rows of fd, so the forward takes the row means in
//              registers and reduces the loss to five partial sums per CTA (no atomics, deterministic); the batch-global
//              `old_mean` enters the loss linearly, so corr_finish_kernel applies it.  The backward is one CTA per image
//              walking the calls in order and computes dA and dB from one recompute of fd / cd.
//   multi-tile (S up to CT_MAX_FS^2): the loss is linear in the row mean m_i of fd,
//                sum_j cl_ij (fd_ij - m_i - shift) = sum_j cl_ij fd_ij - (m_i + shift) sum_j cl_ij,
//              so each forward unit emits per-row partials over its columns (sum fd, sum cl fd, sum cl, sum cd) without
//              knowing m_i; corr_tiled_finish_kernel reduces them over the column tiles in a fixed order (fp64) into the
//              row means and the per-call stats.  dA = G . Bc sums over column tiles and dB = G^T . Ac over row tiles,
//              so the backward runs one pass for each, in which ONE CTA owns the output rows and walks the units in a
//              fixed order.
// The backward recomputes fd, cd (cheaper than stashing them), forms G = dL/dfd in registers, writes it as a swizzled
// bf16 hi/lo tile to smem and runs the backward GEMMs on the tensor cores from that smem image: dA = G . Bc (G as
// K-major A) and dB = G^T . Ac (G as MN-major A); the code tiles Ac/Bc stay resident in smem from the recompute and are
// reused as MN-major B operands.  Every gradient element has one writer, which adds in a fixed order: the gradient
// tiles are bit-reproducible run to run.
// ---------------------------------------------------------------------------------------------
struct CorrParams {
  int B, S, R, nT, E, D, nslots, ncalls;
  int slot_of_call[CL_MAX_CALLS];   // B-operand slot per call (A operand is always slot 0)
  float shift[CL_MAX_CALLS];
  int pointwise;
  float clamp_lo;    // 0 (zero_clamp) or -9999
  float clamp_hi;    // 0.8 (stabalize) or +inf
  // forward outputs
  float* partials;   // whole row: [ncalls][B][8]: P1..P5 (see the epilogue)
  float* rowpart;    // multi-tile: [ncalls][B][nT (column tile)][R][4]: sum fd, sum cl*fd, sum cl, sum cd over its columns
  float* cd_out;     // optional [ncalls][B][S][S]
  float* fd_out;     // optional [ncalls][B][S][S]: whole row: row-centred fd; multi-tile: raw fd, centred in place by
                     // corr_tiled_elems_kernel
  // backward inputs
  const float* stats;    // [ncalls][4]: loss_mean, cd_mean, old_mean, mean_c
  const float* rowmean;  // multi-tile: [ncalls][B][R], the pointwise row means of fd (0 when !pointwise)
  const float* gscale;   // [ncalls] upstream grad of each call's mean loss
  const float* gelem;    // optional [ncalls][B][S][S] upstream grad of unreduced loss elements
  const float* gcd;      // optional [ncalls][B][S][S] upstream grad of cd elements
  float* dtiles;         // [nslots][B][R][CL_DT_LD] fp32, zero-initialised by the caller
  // histogram variants (kVariant | CP_HIST) only: TensorBoard histograms of cd per group (call 0, call 1, calls 2..)
  const float* hist_thr;             // [TB_THR] fp32 bucket thresholds (tb_hist.cuh)
  unsigned long long* hist_counts;   // [3][TB_BINS], zeroed by the caller, added to with integer atomics
  double* hist_part;                 // [ncalls][B][CTAs per (image, call)][4]: min, max, sum, sum of squares
  // precision-recall phase (CP_PR) only
  const int* pr_ids;                 // [2][B][R]: pure class id of each sample of slot 0 / slot 1, -1 if mixed
  unsigned long long* pr_counts;     // [2 (fd, cd)][2 (negative, positive)][CL_PR_BINS], added to
};

constexpr int CL_THREADS = 384;  // two MMA warpgroups (rows 0..63 / 64..127 of the tile) + the TMA producer warpgroup
constexpr uint32_t CL_TILE = 128 * 64 * 2;  // 16 KB

// Phases of corr_kernel: which units a CTA walks, and what it does with each block of fd / cd.
constexpr int CP_FWD = 0;          // whole row, grid (B, ncalls): row means in registers, five partial sums
constexpr int CP_FWD_ROWPART = 1;  // multi-tile, grid (B, ncalls, nT^2): per-row partials over the unit's columns
constexpr int CP_BWD = 2;          // whole row, grid (B): the calls in order, dA -> slot 0 and dB -> the call's slot
constexpr int CP_BWD_DB = 3;       // multi-tile, grid (B, nT): CTA per (image, ct) walking (call, rt) -> dB rows ct
constexpr int CP_BWD_DA = 4;       // multi-tile, grid (B, nT): CTA per (image, rt) walking (call, ct) -> dA rows rt
constexpr int CP_HIST = 8;         // flag on CP_FWD / CP_FWD_ROWPART: also bin cd into TensorBoard histograms
constexpr int CP_PR = 16;          // grid (B, 1, nT^2) like CP_FWD_ROWPART, one call (slot 0 vs slot 1): bin raw fd and
                                   // cd by label agreement into precision-recall counts; no loss, fd or cd output

// unit u of this CTA -> (call, row tile, column tile)
template <int kPhase>
__device__ __forceinline__ void corr_unit(const CorrParams& p, int u, int& call, int& rt, int& ct) {
  if constexpr (kPhase == CP_FWD) {
    call = blockIdx.y; rt = 0; ct = 0;
  } else if constexpr (kPhase == CP_FWD_ROWPART || kPhase == CP_PR) {
    call = blockIdx.y; rt = blockIdx.z / p.nT; ct = blockIdx.z % p.nT;
  } else if constexpr (kPhase == CP_BWD) {
    call = u; rt = 0; ct = 0;
  } else if constexpr (kPhase == CP_BWD_DB) {
    call = u / p.nT; rt = u % p.nT; ct = blockIdx.y;
  } else {
    call = u / p.nT; ct = u % p.nT; rt = blockIdx.y;
  }
}

// first operand-tile row of 128-row tile `tile` of (plane, slot, image b)
__device__ __forceinline__ uint32_t tile_row(const CorrParams& p, int plane, int slot, int b, int tile) {
  return static_cast<uint32_t>(((plane * p.nslots + slot) * p.B + b) * p.R + tile * CL_ROWS);
}

// shared by forward and backward: issue order of the (A plane, B plane) split passes
__device__ __forceinline__ void split_pass(int pass, int& pa, int& pb) {
  pa = (pass == 1) ? 1 : 0;  // (hi,hi), (lo,hi), (hi,lo)
  pb = (pass == 2) ? 1 : 0;
}

// Histogram epilogue of the forward variants: bins this CTA's cd block into the TensorBoard histogram of the call's
// group (0: call 0, 1: call 1, 2: the negatives, which the reference concatenates) and writes the CTA's min / max / sum
// / sum-of-squares partial.  Only elements with row and column < S are values of the reference's cd tensors: the
// padding rows / columns of the 128-row tiles hold cd = 0 and are skipped.  Run by the 256 MMA threads after a
// bar.sync that both warpgroups reach past their wgmma_wait<0>.  The bins live in the operand ring, which is free then:
// a forward CTA runs one unit, its producer issues no load after the unit's last stage, every stage's full barrier has
// been waited on (so each TMA write into the ring has landed), and no wgmma reads the ring any more.
__device__ __forceinline__ void corr_hist_epilogue(const CorrParams& p, const float (&cd)[64], int i0, int j0, int call,
                                                   int b, uint8_t* smem, int warp, int lane) {
  float* thr = reinterpret_cast<float*>(smem);
  uint32_t* bins = reinterpret_cast<uint32_t*>(smem + 6208);             // after TB_THR floats, 16-byte aligned
  TbStats* wred = reinterpret_cast<TbStats*>(smem + 6208 + 4 * TB_BINS);  // [8 warps]
  const int tid = threadIdx.x;  // 0 .. 255: the MMA warpgroups
  for (int k = tid; k < TB_THR; k += 256) thr[k] = p.hist_thr[k];
  for (int k = tid; k < TB_BINS; k += 256) bins[k] = 0;
  asm volatile("bar.sync 1, 256;\n" ::: "memory");
  const int S = p.S;
  TbStats st;
  st.init();
#pragma unroll
  for (int t = 0; t < 64; ++t) {
    const int i = i0 + 8 * ((t >> 1) & 1);
    const int j = j0 + 8 * (t >> 2) + (t & 1);
    if (i < S && j < S) {
      const int k = tb_bucket(cd[t], thr);
      if (k >= 0) atomicAdd(&bins[k], 1u);
      st.add(cd[t]);
    }
  }
  st.warp_reduce();
  if (lane == 0) wred[warp] = st;
  asm volatile("bar.sync 1, 256;\n" ::: "memory");
  unsigned long long* counts = p.hist_counts + static_cast<size_t>(min(call, 2)) * TB_BINS;
  for (int k = tid; k < TB_BINS; k += 256)
    if (bins[k]) atomicAdd(&counts[k], static_cast<unsigned long long>(bins[k]));
  if (tid == 0) {
    TbStats c = wred[0];
    for (int w = 1; w < 8; ++w) {
      c.mn = fminf(c.mn, wred[w].mn);
      c.mx = fmaxf(c.mx, wred[w].mx);
      c.s += wred[w].s;
      c.s2 += wred[w].s2;
    }
    double* o = p.hist_part + ((static_cast<size_t>(call) * p.B + b) * gridDim.z + blockIdx.z) * 4;
    o[0] = c.mn; o[1] = c.mx; o[2] = c.s; o[3] = c.s2;
  }
}

// Score bin of the precision-recall counts: clamp(floor((score + 1) * CL_PR_BINS / 2), 0, CL_PR_BINS - 1) in fp32.  The
// scale is a power of two, so the only rounding is score + 1, and the bin is non-decreasing in the score.
__device__ __forceinline__ int pr_bin(float score) {
  const int k = static_cast<int>(floorf((score + 1.f) * static_cast<float>(CL_PR_BINS / 2)));
  return min(max(k, 0), CL_PR_BINS - 1);
}

// Precision-recall epilogue (CP_PR): bins the raw fd and cd of every element with row and column < S by score
// (pr_bin) and by label agreement — positive when row sample i (slot 0) and column sample j (slot 1) are both pure with
// the same class (sample_label_ids_kernel).  The per-CTA uint32 bins [2 (fd, cd)][2 (negative, positive)][CL_PR_BINS]
// (64 KB) and the unit's 128 row and 128 column ids live in the operand ring, free here for the reasons
// corr_hist_epilogue gives; the caller's bar.sync has put both warpgroups past their wgmma_wait<0>.  The non-empty bins
// are then added to the global counts with one integer atomic each, so the counts are exact and run-to-run identical.
__device__ __forceinline__ void corr_pr_epilogue(const CorrParams& p, const float (&fd)[64], const float (&cd)[64],
                                                 int i_loc, int j_base, int rt, int ct, int b, uint8_t* smem) {
  uint32_t* bins = reinterpret_cast<uint32_t*>(smem);
  int* rid = reinterpret_cast<int*>(smem + 4 * 4 * CL_PR_BINS);  // [128] ids of the unit's rows
  int* cid = rid + CL_ROWS;                                      // [128] ids of the unit's columns
  const int tid = threadIdx.x;  // 0 .. 255: the MMA warpgroups
  const int S = p.S;
  for (int k = tid; k < CL_PR_BINS; k += 256) reinterpret_cast<uint4*>(bins)[k] = make_uint4(0, 0, 0, 0);
  if (tid < CL_ROWS) {
    const int i = rt * CL_ROWS + tid;
    rid[tid] = i < S ? p.pr_ids[static_cast<size_t>(b) * p.R + i] : -1;
  } else {
    const int j = ct * CL_ROWS + tid - CL_ROWS;
    cid[tid - CL_ROWS] = j < S ? p.pr_ids[(static_cast<size_t>(p.B) + b) * p.R + j] : -1;
  }
  asm volatile("bar.sync 1, 256;\n" ::: "memory");
  const int r0 = rid[i_loc], r1 = rid[i_loc + 8];
#pragma unroll
  for (int t = 0; t < 64; ++t) {
    const int h = (t >> 1) & 1;
    const int jl = 8 * (t >> 2) + j_base + (t & 1);
    if (rt * CL_ROWS + i_loc + 8 * h < S && ct * CL_ROWS + jl < S) {
      const int ri = h ? r1 : r0;
      const int pos = (ri >= 0 && ri == cid[jl]) ? CL_PR_BINS : 0;
      atomicAdd(&bins[pos + pr_bin(fd[t])], 1u);
      atomicAdd(&bins[2 * CL_PR_BINS + pos + pr_bin(cd[t])], 1u);
    }
  }
  asm volatile("bar.sync 1, 256;\n" ::: "memory");
  for (int k = tid; k < 4 * CL_PR_BINS; k += 256)
    if (bins[k]) atomicAdd(&p.pr_counts[k], static_cast<unsigned long long>(bins[k]));
}

template <int kVariant>
__global__ void __launch_bounds__(CL_THREADS, 1)
corr_kernel(const __grid_constant__ CUtensorMap tmF, const __grid_constant__ CUtensorMap tmC, CorrParams p) {
  constexpr int kPhase = kVariant & ~CP_HIST;
  constexpr bool kHist = (kVariant & CP_HIST) != 0;
  static_assert(!kHist || kPhase <= CP_FWD_ROWPART, "histograms are a forward epilogue");
  constexpr bool kPR = kPhase == CP_PR;
  constexpr bool kBackward = kPhase >= CP_BWD && !kPR;
  constexpr bool kDA = kPhase == CP_BWD || kPhase == CP_BWD_DA;
  constexpr bool kDB = kPhase == CP_BWD || kPhase == CP_BWD_DB;
  // smem: ring of kRing stages x (A 16K + B 16K) for the feature GEMM, then the resident code tiles.
  constexpr int kRing = kBackward ? 2 : 3;
  constexpr uint32_t RING_BYTES = kRing * 2 * CL_TILE;
  constexpr uint32_t CODE_BYTES = 8 * CL_TILE;  // Ac: [plane][kb] 4 tiles, Bc: 4 tiles
  constexpr uint32_t OFF_CODE = RING_BYTES;
  constexpr uint32_t OFF_BAR = OFF_CODE + CODE_BYTES;
  static_assert(!kPR || RING_BYTES >= 4 * 4 * CL_PR_BINS + 2 * 4 * CL_ROWS, "the PR bins live in the operand ring");

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + OFF_BAR);
  uint64_t* full_bar = bars;                // [kRing]
  uint64_t* empty_bar = bars + kRing;       // [kRing]
  uint64_t* code_full = empty_bar + kRing;  // [1]
  uint64_t* unit_done = code_full + 1;      // [1] backward: ring (G) and code tiles of the unit are no longer read
  float* red = reinterpret_cast<float*>(unit_done + 1);  // [8 warps][8]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.x;
  const int nunits = kPhase == CP_BWD ? p.ncalls : kBackward ? p.ncalls * p.nT : 1;
  const int nkb_f = p.E / 64;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmF);
    tma_prefetch_desc(&tmC);
    for (int s = 0; s < kRing; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 2); }
    mbar_init(code_full, 1);
    mbar_init(unit_done, 2);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= 8) {
    warpgroup_reg_dealloc<40>();
    if (warp == 8 && lane == 0) {
      uint32_t stage = 0, phase = 0;
      for (int u = 0; u < nunits; ++u) {
        int call, rt, ct;
        corr_unit<kPhase>(p, u, call, rt, ct);
        const int slotB = p.slot_of_call[call];
        if (u > 0) mbar_wait(unit_done, static_cast<uint32_t>(u - 1) & 1u);
        // code tiles first (small, resident): Ac planes then Bc planes, 2 k-blocks each
        mbar_arrive_expect_tx(code_full, CODE_BYTES);
        for (int pl = 0; pl < 2; ++pl)
          for (int kb = 0; kb < 2; ++kb) {
            tma_load_2d(smem + OFF_CODE + (pl * 2 + kb) * CL_TILE, &tmC, code_full, kb * 64, tile_row(p, pl, 0, b, rt));
            tma_load_2d(smem + OFF_CODE + (4 + pl * 2 + kb) * CL_TILE, &tmC, code_full, kb * 64,
                        tile_row(p, pl, slotB, b, ct));
          }
        for (int pass = 0; pass < 3; ++pass) {
          int pa, pb;
          split_pass(pass, pa, pb);
          for (int kb = 0; kb < nkb_f; ++kb) {
            mbar_wait(&empty_bar[stage], phase ^ 1u);
            uint8_t* sa = smem + stage * 2 * CL_TILE;
            mbar_arrive_expect_tx(&full_bar[stage], 2 * CL_TILE);
            tma_load_2d(sa, &tmF, &full_bar[stage], kb * 64, tile_row(p, pa, 0, b, rt));
            tma_load_2d(sa + CL_TILE, &tmF, &full_bar[stage], kb * 64, tile_row(p, pb, slotB, b, ct));
            if (++stage == kRing) { stage = 0; phase ^= 1u; }
          }
        }
      }
    }
    return;
  }

  // ===================== MMA warpgroups: rows 64 mwg .. 64 mwg + 63 of the unit's fd / cd block =====================
  warpgroup_reg_alloc<232>();
  const int mwg = warp >> 2;
  const int wq = warp & 3;
  const bool leader = (threadIdx.x & 127) == 0;
  constexpr uint32_t DESC_HI = smem_desc_hi_sw128(1024);
  constexpr uint32_t TILE16 = CL_TILE >> 4;
  constexpr uint32_t HALF16 = (CL_TILE / 2) >> 4;  // rows 64.. of a [128][64] K-major tile
  const uint32_t ring_lo = smem_desc_lo(smem_u32(smem), 16);
  const uint32_t code_lo = smem_desc_lo(smem_u32(smem + OFF_CODE), 16);
  // this thread's accumulator fragment: tile-local rows i_loc (h = 0) and i_loc + 8 (h = 1), tile-local columns
  // 8 n + j_base + {0, 1}
  const int S = p.S;
  const int i_loc = mwg * 64 + wq * 16 + (lane >> 2);
  const int j_base = 2 * (lane & 3);
  uint32_t stage = 0, phase = 0;
  for (int u = 0; u < nunits; ++u) {
    int call, rt, ct;
    corr_unit<kPhase>(p, u, call, rt, ct);
    const int slotB = p.slot_of_call[call];
    float fd[64], cd[64];
#pragma unroll
    for (int t = 0; t < 64; ++t) { fd[t] = 0.f; cd[t] = 0.f; }
    {
      // fd = An_f . Bn_f^T  (3 split passes over E)
      uint32_t prev = 0;
      for (int ks = 0; ks < 3 * nkb_f; ++ks) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t a_lo = ring_lo + stage * 2 * TILE16;
        fence_operands(fd);
        wgmma_fence();
#pragma unroll
        for (uint32_t k = 0; k < 4; ++k)
          wgmma_ss<128, 0, 0>(fd, smem_desc_join(a_lo + mwg * HALF16 + 2 * k, DESC_HI),
                              smem_desc_join(a_lo + TILE16 + 2 * k, DESC_HI), 1u);
        wgmma_commit();
        wgmma_wait<1>();
        if (ks > 0 && leader) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == kRing) { stage = 0; phase ^= 1u; }
      }
      // cd = An_c . Bn_c^T from the resident code tiles
      mbar_wait(code_full, static_cast<uint32_t>(u) & 1u);
      wgmma_fence();
#pragma unroll
      for (int pass = 0; pass < 3; ++pass) {
        int pa, pb;
        split_pass(pass, pa, pb);
#pragma unroll
        for (int kb = 0; kb < 2; ++kb) {
          const uint32_t a_lo = code_lo + (pa * 2 + kb) * TILE16 + mwg * HALF16;
          const uint32_t b_lo = code_lo + (4 + pb * 2 + kb) * TILE16;
#pragma unroll
          for (uint32_t k = 0; k < 4; ++k)
            wgmma_ss<128, 0, 0>(cd, smem_desc_join(a_lo + 2 * k, DESC_HI), smem_desc_join(b_lo + 2 * k, DESC_HI), 1u);
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      fence_operands(fd);
      fence_operands(cd);
      if (leader) mbar_arrive(&empty_bar[prev]);
    }

    if constexpr (kPR) {
      asm volatile("bar.sync 1, 256;\n" ::: "memory");
      corr_pr_epilogue(p, fd, cd, i_loc, j_base, rt, ct, b, smem);
      return;
    }
    // ===================== epilogue on the accumulator fragments =====================
    const int i0 = rt * CL_ROWS + i_loc;  // rows of fragment halves 0 / 1: i0, i0 + 8
    const int j0 = ct * CL_ROWS + j_base;
    const size_t e_row0 = (static_cast<size_t>(call) * p.B + b) * S;  // [ncalls][B][S][S] outputs: row 0 of the unit
    if constexpr (kPhase == CP_FWD_ROWPART) {
      // per-row partials over this tile's valid columns; the four lanes of a quad hold disjoint columns of a row
      float r_fd[2] = {0.f, 0.f}, r_clfd[2] = {0.f, 0.f}, r_cl[2] = {0.f, 0.f}, r_cd[2] = {0.f, 0.f};
#pragma unroll
      for (int t = 0; t < 64; ++t) {
        const int h = (t >> 1) & 1;
        const int i = i0 + 8 * h;
        const int j = j0 + 8 * (t >> 2) + (t & 1);
        if (i < S && j < S) {
          const float cl = fminf(fmaxf(cd[t], p.clamp_lo), p.clamp_hi);
          r_fd[h] += fd[t];
          r_clfd[h] += cl * fd[t];
          r_cl[h] += cl;
          r_cd[h] += cd[t];
          const size_t e = (e_row0 + i) * S + j;
          if (p.cd_out) p.cd_out[e] = cd[t];
          if (p.fd_out) p.fd_out[e] = fd[t];
        }
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int o = 1; o <= 2; o <<= 1) {
          r_fd[h] += __shfl_xor_sync(0xffffffffu, r_fd[h], o);
          r_clfd[h] += __shfl_xor_sync(0xffffffffu, r_clfd[h], o);
          r_cl[h] += __shfl_xor_sync(0xffffffffu, r_cl[h], o);
          r_cd[h] += __shfl_xor_sync(0xffffffffu, r_cd[h], o);
        }
        const int i = i0 + 8 * h;
        if ((lane & 3) == 0 && i < S)
          *reinterpret_cast<float4*>(p.rowpart + (((static_cast<size_t>(call) * p.B + b) * p.nT + ct) * p.R + i) * 4) =
              make_float4(r_fd[h], r_clfd[h], r_cl[h], r_cd[h]);
      }
      if constexpr (kHist) {
        asm volatile("bar.sync 1, 256;\n" ::: "memory");
        corr_hist_epilogue(p, cd, i0, j0, call, b, smem, warp, lane);
      }
      return;
    }
    // the row means of fd for fragment halves 0 / 1: from the row sums over the valid columns of the whole-row unit
    // (the four lanes of a row hold disjoint columns), or from the multi-tile forward's finish
    float rsum[2] = {0.f, 0.f}, rmean[2];
    if constexpr (kPhase == CP_FWD || kPhase == CP_BWD) {
#pragma unroll
      for (int t = 0; t < 64; ++t)
        if (j0 + 8 * (t >> 2) + (t & 1) < S) rsum[(t >> 1) & 1] += fd[t];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        rsum[h] += __shfl_xor_sync(0xffffffffu, rsum[h], 1);
        rsum[h] += __shfl_xor_sync(0xffffffffu, rsum[h], 2);
        rmean[h] = p.pointwise ? rsum[h] / static_cast<float>(S) : 0.f;
      }
    } else {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int i = i0 + 8 * h;
        rmean[h] = i < S ? p.rowmean[(static_cast<size_t>(call) * p.B + b) * p.R + i] : 0.f;
      }
    }
    const float shift = p.shift[call];
    if constexpr (kPhase == CP_FWD) {
      float P1 = 0.f, P2 = 0.f, P3 = 0.f, P4 = 0.f, P5 = 0.f;
      if ((lane & 3) == 0) {  // each row's sum once
        if (i0 < S) P3 += rsum[0];
        if (i0 + 8 < S) P3 += rsum[1];
      }
#pragma unroll
      for (int t = 0; t < 64; ++t) {
        const int h = (t >> 1) & 1;
        const int i = i0 + 8 * h;
        const int j = j0 + 8 * (t >> 2) + (t & 1);
        if (i < S && j < S) {
          const float fdc = fd[t] - rmean[h];
          const float cl = fminf(fmaxf(cd[t], p.clamp_lo), p.clamp_hi);
          P1 += cl * (fdc - shift);
          P2 += cl;
          P4 += fdc;
          P5 += cd[t];
          const size_t e = (e_row0 + i) * S + j;
          if (p.cd_out) p.cd_out[e] = cd[t];
          if (p.fd_out) p.fd_out[e] = fdc;
        }
      }
      // deterministic block reduction of the five partial sums
      P1 = warp_sum(P1); P2 = warp_sum(P2); P3 = warp_sum(P3); P4 = warp_sum(P4); P5 = warp_sum(P5);
      if (lane == 0) {
        float* r = red + warp * 8;
        r[0] = P1; r[1] = P2; r[2] = P3; r[3] = P4; r[4] = P5;
      }
      asm volatile("bar.sync 1, 256;\n" ::: "memory");
      if (warp == 0 && lane < 5) {
        float tot = 0.f;
#pragma unroll
        for (int w = 0; w < 8; ++w) tot += red[w * 8 + lane];
        p.partials[(static_cast<size_t>(call) * p.B + b) * 8 + lane] = tot;
      }
      if constexpr (kHist) corr_hist_epilogue(p, cd, i0, j0, call, b, smem, warp, lane);
      return;
    }
    {
      // ---- backward: G = dL/dfd in place of fd
      const float* st = p.stats + call * 4;
      const float offset = p.pointwise ? (st[2] - st[3]) : 0.f;  // old_mean - mean(centred fd)
      const float gs = p.gscale[call] / (static_cast<float>(p.B) * S * S);
#pragma unroll
      for (int t = 0; t < 64; ++t) {
        const int h = (t >> 1) & 1;
        const int i = i0 + 8 * h;
        const int j = j0 + 8 * (t >> 2) + (t & 1);
        float gv = 0.f;
        if (i < S && j < S) {
          const size_t e = (e_row0 + i) * S + j;
          const float cdv = cd[t];
          float up = gs;
          if (p.gelem) up += p.gelem[e];
          const bool pass_grad = (cdv >= p.clamp_lo) && (cdv <= p.clamp_hi);
          gv = pass_grad ? -up * (fd[t] - rmean[h] + offset - shift) : 0.f;
          if (p.gcd) gv += p.gcd[e];
        }
        fd[t] = gv;
      }
    }
    // ---- G[i][j] as a bf16 hi/lo split into the ring area ([j block][i][64 j], 128B-swizzled K-major image, hi plane
    //      at +0, lo plane at +2 tiles).  Both warpgroups' feature MMAs must have retired first.
    asm volatile("bar.sync 1, 256;\n" ::: "memory");
#pragma unroll
    for (int t = 0; t < 64; t += 2) {
      const int i = i_loc + 8 * ((t >> 1) & 1);
      const int j = 8 * (t >> 2) + j_base;
      const float h0 = __bfloat162float(__float2bfloat16_rn(fd[t]));
      const float h1 = __bfloat162float(__float2bfloat16_rn(fd[t + 1]));
      const uint32_t o = (j >> 6) * CL_TILE + sw128_offset(i, (j & 63) >> 3) + (j & 7) * 2;
      *reinterpret_cast<uint32_t*>(smem + o) = pack_bf16x2(h0, h1);
      *reinterpret_cast<uint32_t*>(smem + 2 * CL_TILE + o) = pack_bf16x2(fd[t] - h0, fd[t + 1] - h1);
    }
    fence_proxy_async_smem();  // generic-proxy smem writes -> visible to the tensor cores
    asm volatile("bar.sync 1, 256;\n" ::: "memory");
    // dA accumulates in cd; dB in fd when the whole-row backward computes both, in cd when it is the only GEMM
    float (&dacc)[64] = kDA ? fd : cd;
    {
      // dA[i][c] += sum_j G[i][j] Bc[j][c]: A = G K-major (k = j), B = Bc MN-major (n = c contiguous), rows i of this
      // warpgroup.  dB[j][c] += sum_i G[i][j] Ac[i][c]: A = G^T MN-major (m = j: the j block of this warpgroup, k = i).
      // MN-major operands: LBO = CL_TILE (64-wide blocks 16 KB apart).
      const uint32_t g_k_lo = ring_lo + mwg * HALF16;
      const uint32_t g_mn_lo = smem_desc_lo(smem_u32(smem), CL_TILE) + mwg * TILE16;
      const uint32_t code_mn_lo = smem_desc_lo(smem_u32(smem + OFF_CODE), CL_TILE);
#pragma unroll
      for (int t = 0; t < 64; ++t) {
        if constexpr (kDA) cd[t] = 0.f;
        if constexpr (kDB) dacc[t] = 0.f;
      }
      wgmma_fence();
#pragma unroll
      for (int pass = 0; pass < 3; ++pass) {
        int pg, pc;
        split_pass(pass, pg, pc);
        const uint32_t g_off = pg * 2 * TILE16;
        const uint32_t bc_lo = code_mn_lo + (4 + pc * 2) * TILE16;  // Bc plane: c-blocks 16 KB apart, rows = j
        const uint32_t ac_lo = code_mn_lo + (pc * 2) * TILE16;      // Ac plane: rows = i
        if constexpr (kDA) {
#pragma unroll
          for (uint32_t kk = 0; kk < 8; ++kk)
            wgmma_ss<128, 0, 1>(cd, smem_desc_join(g_k_lo + g_off + (kk >> 2) * TILE16 + (kk & 3) * 2, DESC_HI),
                                smem_desc_join(bc_lo + kk * (2048u >> 4), DESC_HI), 1u);
        }
        if constexpr (kDB) {
#pragma unroll
          for (uint32_t kk = 0; kk < 8; ++kk)
            wgmma_ss<128, 1, 1>(dacc, smem_desc_join(g_mn_lo + g_off + kk * (2048u >> 4), DESC_HI),
                                smem_desc_join(ac_lo + kk * (2048u >> 4), DESC_HI), 1u);
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      if constexpr (kDA) fence_operands(cd);
      if constexpr (kDB) fence_operands(dacc);
    }
    if (leader) mbar_arrive(unit_done);  // the producer may refill the ring and the code tiles
    // dA -> rows of row tile rt of slot 0, dB -> rows of column tile ct of the call's slot (slot 0 again for the intra
    // call: code is on both GEMM sides).  Each gradient row has one owner CTA, which adds its units in a fixed order:
    // plain read-modify-write.  Rows >= S carry zero gradients and are skipped.
    float* dA = p.dtiles + static_cast<size_t>(b) * p.R * CL_DT_LD;
    float* dB = p.dtiles + (static_cast<size_t>(slotB) * p.B + b) * p.R * CL_DT_LD;
#pragma unroll
    for (int t = 0; t < 64; ++t) {
      const int r = i_loc + 8 * ((t >> 1) & 1);
      const int c = 8 * (t >> 2) + j_base + (t & 1);
      const int ra = rt * CL_ROWS + r, rb = ct * CL_ROWS + r;
      if constexpr (kDA) if (ra < S && c < p.D) dA[static_cast<size_t>(ra) * CL_DT_LD + c] += cd[t];
      if constexpr (kDB) if (rb < S && c < p.D) dB[static_cast<size_t>(rb) * CL_DT_LD + c] += dacc[t];
    }
  }
}

// ---------------------------------------------------------------------------------------------
// 3. finish: per call statistics.  stats[call] = {loss_mean, cd_mean, old_mean, mean_c}
// ---------------------------------------------------------------------------------------------
__global__ void corr_finish_kernel(const float* __restrict__ partials, float* __restrict__ stats, int ncalls, int B,
                                   int S, int pointwise) {
  const int call = blockIdx.x;
  const int lane = threadIdx.x;  // 32 threads
  double acc[5] = {0, 0, 0, 0, 0};
  for (int b = lane; b < B; b += 32) {
    const float* r = partials + (static_cast<size_t>(call) * B + b) * 8;
    for (int k = 0; k < 5; ++k) acc[k] += static_cast<double>(r[k]);
  }
  for (int k = 0; k < 5; ++k)
    for (int o = 16; o > 0; o >>= 1) acc[k] += __shfl_xor_sync(0xffffffffu, acc[k], o);
  if (lane == 0) {
    const double n = static_cast<double>(B) * S * S;
    const double old_mean = acc[2] / n;
    const double mean_c = acc[3] / n;
    const double offset = pointwise ? (old_mean - mean_c) : 0.0;
    stats[call * 4 + 0] = static_cast<float>(-(acc[0] + offset * acc[1]) / n);
    stats[call * 4 + 1] = static_cast<float>(acc[4] / n);
    stats[call * 4 + 2] = static_cast<float>(old_mean);
    stats[call * 4 + 3] = static_cast<float>(mean_c);
  }
}

// unreduced loss elements for API compatibility (modules.py:337-345 returns them for the negatives)
__global__ void corr_loss_elems_kernel(const float* __restrict__ cd, const float* __restrict__ fdc,
                                       const float* __restrict__ stats, float* __restrict__ loss, long long per_call,
                                       CorrParams p) {
  const long long idx = 1ll * blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= per_call * p.ncalls) return;
  const int call = static_cast<int>(idx / per_call);
  const float offset = p.pointwise ? (stats[call * 4 + 2] - stats[call * 4 + 3]) : 0.f;
  const float cl = fminf(fmaxf(cd[idx], p.clamp_lo), p.clamp_hi);
  loss[idx] = -cl * (fdc[idx] + offset - p.shift[call]);
}

// Multi-tile finish, per call: row means and stats from the per-row partials, fp64, every sum in a fixed order.
constexpr int CT_FINISH_THREADS = 256;
__global__ void __launch_bounds__(CT_FINISH_THREADS)
corr_tiled_finish_kernel(CorrParams p, float* __restrict__ rowmean, float* __restrict__ stats) {
  const int call = blockIdx.x;
  const int S = p.S;
  const double shift = p.shift[call];
  // acc: 0 sum cl (fd - m - shift), 1 sum cl, 2 sum fd, 3 sum (fd - m), 4 sum cd
  double acc[5] = {0, 0, 0, 0, 0};
  for (int r = threadIdx.x; r < p.B * S; r += CT_FINISH_THREADS) {
    const int b = r / S, i = r % S;
    double s_fd = 0, s_clfd = 0, s_cl = 0, s_cd = 0;
    const float* rp = p.rowpart + ((static_cast<size_t>(call) * p.B + b) * p.nT * p.R + i) * 4;
    for (int ct = 0; ct < p.nT; ++ct) {
      const float4 v = *reinterpret_cast<const float4*>(rp + static_cast<size_t>(ct) * p.R * 4);
      s_fd += v.x; s_clfd += v.y; s_cl += v.z; s_cd += v.w;
    }
    const float m = p.pointwise ? static_cast<float>(s_fd / S) : 0.f;
    rowmean[(static_cast<size_t>(call) * p.B + b) * p.R + i] = m;
    acc[0] += s_clfd - (static_cast<double>(m) + shift) * s_cl;
    acc[1] += s_cl;
    acc[2] += s_fd;
    acc[3] += s_fd - static_cast<double>(S) * m;
    acc[4] += s_cd;
  }
  __shared__ double red[5][CT_FINISH_THREADS];
#pragma unroll
  for (int k = 0; k < 5; ++k) red[k][threadIdx.x] = acc[k];
  __syncthreads();
  for (int w = CT_FINISH_THREADS / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w)
#pragma unroll
      for (int k = 0; k < 5; ++k) red[k][threadIdx.x] += red[k][threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const double n = static_cast<double>(p.B) * S * S;
    const double old_mean = red[2][0] / n;
    const double mean_c = red[3][0] / n;
    const double offset = p.pointwise ? (old_mean - mean_c) : 0.0;
    stats[call * 4 + 0] = static_cast<float>(-(red[0][0] + offset * red[1][0]) / n);
    stats[call * 4 + 1] = static_cast<float>(red[4][0] / n);
    stats[call * 4 + 2] = static_cast<float>(old_mean);
    stats[call * 4 + 3] = static_cast<float>(mean_c);
  }
}

// centres fd_out in place with the row means and writes the unreduced loss elements
__global__ void corr_tiled_elems_kernel(const float* __restrict__ cd, float* __restrict__ fdc,
                                        const float* __restrict__ rowmean, const float* __restrict__ stats,
                                        float* __restrict__ loss, CorrParams p) {
  const long long per_call = 1ll * p.B * p.S * p.S;
  const long long idx = 1ll * blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= per_call * p.ncalls) return;
  const int call = static_cast<int>(idx / per_call);
  const long long row = idx / p.S;  // (call * B + b) * S + i
  const int i = static_cast<int>(row % p.S);
  const long long cb = row / p.S;   // call * B + b
  const float v = fdc[idx] - rowmean[cb * p.R + i];
  fdc[idx] = v;
  if (loss) {
    const float offset = p.pointwise ? (stats[call * 4 + 2] - stats[call * 4 + 3]) : 0.f;
    const float cl = fminf(fmaxf(cd[idx], p.clamp_lo), p.clamp_hi);
    loss[idx] = -cl * (v + offset - p.shift[call]);
  }
}

// ---------------------------------------------------------------------------------------------
// 5. normalisation + grid_sample backward, as a gather: one warp per destination pixel (of code or code_pos) visits
//    every (slot, image, sample) whose bilinear taps reach that pixel, in a fixed order, and writes its channels once —
//    no atomics, so the code gradient is bit-reproducible run to run.
// ---------------------------------------------------------------------------------------------
struct SampleBwdParams {
  SampleParams f;        // forward description of the code sampling (src = code, src_pos = code_pos)
  const float* dtiles;   // [nslots][B][R][CL_DT_LD]
  float* dsrc;           // gradient wrt src, same strides as src, fp32, zero-initialised / accumulated into
  float* dsrc_pos;
};

// d/dv of the normalised sample v/||v|| for (slot, b, s), lane-owned channels lane + 32 k
template <int NV>
__device__ __forceinline__ void sample_dv(const SampleBwdParams& q, int slot, int b, int s, const Taps& t,
                                          const float* src, int img, int lane, float (&dv)[NV]) {
  const SampleParams& p = q.f;
  auto off = [&](int pix) { return static_cast<long long>(pix / p.W) * p.sy + static_cast<long long>(pix % p.W) * p.sx; };
  const long long o00 = off(t.i00), o01 = off(t.i01), o10 = off(t.i10), o11 = off(t.i11);
  const long long base = static_cast<long long>(img) * p.sb;
  const float* g = q.dtiles + ((static_cast<size_t>(slot) * p.B + b) * p.R + s) * CL_DT_LD;
  float v[NV], gr[NV];
  float ss = 0.f, dot = 0.f;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    const int c = lane + 32 * k;
    float val = 0.f, gg = 0.f;
    if (c < p.C) {
      const float* qf = src + base + static_cast<long long>(c) * p.sc;
      val = qf[o00] * t.w00;
      val += qf[o01] * t.w01;
      val += qf[o10] * t.w10;
      val += qf[o11] * t.w11;
      gg = g[c];
    }
    v[k] = val; gr[k] = gg;
    ss += val * val;
    dot += val * gg;
  }
  ss = warp_sum(ss);
  dot = warp_sum(dot);
  const float nrm = sqrtf(ss);
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    if (nrm > p.eps) {
      const float inv = 1.0f / nrm;
      dv[k] = (gr[k] - v[k] * (dot * inv * inv)) * inv;  // d/dv of v/||v||
    } else {
      dv[k] = gr[k] / p.eps;
    }
  }
}

template <int NV>
__global__ void __launch_bounds__(256)
sample_norm_bwd_kernel(SampleBwdParams q) {
  const SampleParams& p = q.f;
  const int warp_global = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const int HW = p.H * p.W;
  if (warp_global >= 2 * p.B * HW) return;
  const bool pos = warp_global >= p.B * HW;  // destination: code_pos (slot 1 only) or code (slot 0 and slots >= 2)
  const int dst_img = (warp_global % (p.B * HW)) / HW;
  const int pix = warp_global % HW;
  float acc[NV];
#pragma unroll
  for (int k = 0; k < NV; ++k) acc[k] = 0.f;
  for (int slot = 0; slot < p.nslots; ++slot) {
    if ((slot == 1) != pos) continue;
    for (int b0 = 0; b0 < p.B; b0 += 32) {
      // the images (slot, b0 + lane) sample from, tested 32 at a time; then the hits in ascending b
      int lane_img = -1;
      if (b0 + lane < p.B) {
        const void* src_l; const float* cscale_l; const float* coords_l;
        slot_source(p, slot, b0 + lane, src_l, cscale_l, coords_l, lane_img);
      }
      uint32_t bhits = __ballot_sync(0xffffffffu, lane_img == dst_img);
      while (bhits) {
        const int b = b0 + __ffs(bhits) - 1;
        bhits &= bhits - 1;
        const void* src; const float* cscale; const float* coords; int img;
        slot_source(p, slot, b, src, cscale, coords, img);
        for (int s0 = 0; s0 < p.S; s0 += 32) {
          const int s = s0 + lane;
          float w = 0.f;
          Taps t;
          if (s < p.S) {
            t = make_taps(coords, b, s, p.fs, p.H, p.W);
            // at most one tap with a non-zero weight lands on a given pixel (a clamped duplicate tap has weight 0)
            w = (t.i00 == pix && t.w00 != 0.f) ? t.w00 : (t.i01 == pix && t.w01 != 0.f) ? t.w01
              : (t.i10 == pix && t.w10 != 0.f) ? t.w10 : (t.i11 == pix && t.w11 != 0.f) ? t.w11 : 0.f;
          }
          uint32_t hits = __ballot_sync(0xffffffffu, w != 0.f);
          while (hits) {  // samples in ascending order
            const int src_lane = __ffs(hits) - 1;
            hits &= hits - 1;
            const float wm = __shfl_sync(0xffffffffu, w, src_lane);
            const Taps tm = make_taps(coords, b, s0 + src_lane, p.fs, p.H, p.W);
            float dv[NV];
            sample_dv<NV>(q, slot, b, s0 + src_lane, tm, reinterpret_cast<const float*>(src), img, lane, dv);
#pragma unroll
            for (int k = 0; k < NV; ++k) acc[k] += dv[k] * wm;
          }
        }
      }
    }
  }
  float* d = (pos ? q.dsrc_pos : q.dsrc) + static_cast<long long>(dst_img) * p.sb +
             static_cast<long long>(pix / p.W) * p.sy + static_cast<long long>(pix % p.W) * p.sx;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    const int c = lane + 32 * k;
    if (c < p.C) d[static_cast<long long>(c) * p.sc] += acc[k];
  }
}

static int encode_tile_maps(const void* ftiles, const void* ctiles, const CorrParams& p, CUtensorMap* tmF,
                            CUtensorMap* tmC) {
  int rc;
  const uint64_t rows = (uint64_t)2 * p.nslots * p.B * p.R;
  {
    uint64_t dims[2] = {(uint64_t)p.E, rows};
    uint64_t str[1] = {(uint64_t)p.E * 2};
    uint32_t box[2] = {64, 128};
    if ((rc = make_tmap_bf16(tmF, ftiles, 2, dims, str, box)) != STEGO_OK) return rc;
  }
  {
    uint64_t dims[2] = {(uint64_t)CL_CODE_PAD, rows};
    uint64_t str[1] = {(uint64_t)CL_CODE_PAD * 2};
    uint32_t box[2] = {64, 128};
    if ((rc = make_tmap_bf16(tmC, ctiles, 2, dims, str, box)) != STEGO_OK) return rc;
  }
  return STEGO_OK;
}

static int fill_sample_params(SampleParams& sp, const void* src, const void* src_pos, int src_bf16, long long sb,
                              long long sc, long long sy, long long sx, const float* chan_scale,
                              const float* chan_scale_pos, const float* coords1, const float* coords2,
                              const long long* perms, void* tiles, int B, int C, int Cpad, int H, int W, int fs,
                              int nslots) {
  STEGO_CHECK_ARG(src && src_pos && coords1 && coords2, "sample_norm: null pointer");
  STEGO_CHECK_ARG(nslots >= 2 && (nslots == 2 || perms), "sample_norm: nslots=%d needs perms", nslots);
  STEGO_CHECK_ARG(fs >= 1 && fs <= CT_MAX_FS, "sample_norm: feature_samples=%d outside 1..%d", fs, CT_MAX_FS);
  STEGO_CHECK_ARG(C > 0 && C <= Cpad && Cpad % 64 == 0 && Cpad <= 768, "sample_norm: C=%d Cpad=%d", C, Cpad);
  STEGO_CHECK_ARG(B > 0 && H > 1 && W > 1, "sample_norm: B=%d H=%d W=%d", B, H, W);
  sp.src = src; sp.src_pos = src_pos; sp.src_bf16 = src_bf16; sp.label_bytes = 0;
  sp.sb = sb; sp.sc = sc; sp.sy = sy; sp.sx = sx;
  sp.chan_scale = chan_scale; sp.chan_scale_pos = chan_scale_pos;
  sp.coords1 = coords1; sp.coords2 = coords2; sp.perms = perms; sp.perms_raw = 0;
  sp.tiles = reinterpret_cast<bf16*>(tiles);
  sp.B = B; sp.C = C; sp.Cpad = Cpad; sp.H = H; sp.W = W; sp.fs = fs; sp.S = fs * fs; sp.nslots = nslots;
  sp.R = (sp.S + CL_ROWS - 1) / CL_ROWS * CL_ROWS;
  sp.eps = 1e-10f;
  return STEGO_OK;
}

// The generic sampler for sp.Cpad: 64 .. 256 channels for both sources, 384 and 768 for features only.
template <int NV, bool kLabels>
static void launch_sampler(const SampleParams& sp, dim3 blocks, cudaStream_t stream) {
  if constexpr (kLabels) sample_labels_kernel<NV><<<blocks, 256, 0, stream>>>(sp);
  else sample_norm_kernel<NV><<<blocks, 256, 0, stream>>>(sp);
}

template <bool kLabels>
static int launch_sample_norm(const SampleParams& sp, cudaStream_t stream, const char* who) {
  const dim3 blocks(sp.R / 8, sp.nslots * sp.B);  // 8 warps per block, one per tile row
  switch (sp.Cpad / 32) {
    case 2: launch_sampler<2, kLabels>(sp, blocks, stream); break;
    case 4: launch_sampler<4, kLabels>(sp, blocks, stream); break;
    case 6: launch_sampler<6, kLabels>(sp, blocks, stream); break;
    case 8: launch_sampler<8, kLabels>(sp, blocks, stream); break;
    default:
      if constexpr (!kLabels) {
        if (sp.Cpad == 384) { launch_sampler<12, false>(sp, blocks, stream); break; }
        if (sp.Cpad == 768) { launch_sampler<24, false>(sp, blocks, stream); break; }
      }
      set_error("%s: Cpad=%d unsupported (%s)", who, sp.Cpad, kLabels ? "64,128,192,256" : "64,128,192,256,384,768");
      return STEGO_ERR_UNSUPPORTED;
  }
  STEGO_CHECK_LAUNCH(kLabels ? "sample_labels_kernel" : "sample_norm_kernel");
  return STEGO_OK;
}

}  // namespace stego

using namespace stego;

extern "C" int stego_sample_norm_fwd(const void* src, const void* src_pos, int src_is_bf16, long long stride_b,
                                     long long stride_c, long long stride_y, long long stride_x,
                                     const float* chan_scale, const float* chan_scale_pos, const float* coords1,
                                     const float* coords2, const long long* perms, void* tiles, int B, int C,
                                     int Cpad, int H, int W, int feature_samples, int nslots, int perms_are_raw_randperm,
                                     void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SampleParams sp;
  int rc = fill_sample_params(sp, src, src_pos, src_is_bf16, stride_b, stride_c, stride_y, stride_x, chan_scale,
                              chan_scale_pos, coords1, coords2, perms, tiles, B, C, Cpad, H, W, feature_samples, nslots);
  if (rc != STEGO_OK) return rc;
  sp.perms_raw = perms_are_raw_randperm;
  STEGO_CHECK_ARG(tiles, "stego_sample_norm_fwd: null tiles");
  STEGO_CHECK_ARG(nslots * B <= 65535, "stego_sample_norm_fwd: nslots * B = %d exceeds 65535", nslots * B);
  const dim3 blocks(sp.R / 8, nslots * B);  // 8 warps per block, one per tile row
  const bool aligned = ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(src_pos) |
                         reinterpret_cast<uintptr_t>(tiles)) & 15u) == 0 &&
                       stride_b % 8 == 0 && stride_y % 8 == 0 && stride_x % 8 == 0;
  if (src_is_bf16 && stride_c == 1 && C % 8 == 0 && Cpad == C && aligned && C <= 768) {
    const int ni = (C + 255) / 256;
    if (ni == 1) sample_norm_vec8_kernel<1><<<blocks, 256, 0, stream>>>(sp);
    else if (ni == 2) sample_norm_vec8_kernel<2><<<blocks, 256, 0, stream>>>(sp);
    else sample_norm_vec8_kernel<3><<<blocks, 256, 0, stream>>>(sp);
    STEGO_CHECK_LAUNCH("sample_norm_vec8_kernel");
    return STEGO_OK;
  }
  return launch_sample_norm<false>(sp, stream, "stego_sample_norm_fwd");
}

extern "C" int stego_sample_labels_fwd(const void* label, const void* label_pos, int label_bytes,
                                       const float* coords1, const float* coords2, const long long* perms, void* tiles,
                                       int B, int n_classes, int Cpad, int H, int W, int feature_samples, int nslots,
                                       int perms_are_raw_randperm, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(label_bytes == 8 || label_bytes == 4 || label_bytes == 1,
                  "stego_sample_labels_fwd: label_bytes=%d (8, 4 or 1)", label_bytes);
  STEGO_CHECK_ARG(n_classes >= 1 && n_classes + 1 <= 256, "stego_sample_labels_fwd: n_classes=%d outside 1..255",
                  n_classes);
  STEGO_CHECK_ARG(Cpad <= 256, "stego_sample_labels_fwd: Cpad=%d exceeds 256", Cpad);
  SampleParams sp;
  int rc = fill_sample_params(sp, label, label_pos, 0, static_cast<long long>(H) * W, 0, W, 1, nullptr, nullptr,
                              coords1, coords2, perms, tiles, B, n_classes + 1, Cpad, H, W, feature_samples, nslots);
  if (rc != STEGO_OK) return rc;
  sp.label_bytes = label_bytes;
  sp.perms_raw = perms_are_raw_randperm;
  STEGO_CHECK_ARG(tiles, "stego_sample_labels_fwd: null tiles");
  STEGO_CHECK_ARG(nslots * B <= 65535, "stego_sample_labels_fwd: nslots * B = %d exceeds 65535", nslots * B);
  return launch_sample_norm<true>(sp, stream, "stego_sample_labels_fwd");
}

extern "C" int stego_sample_norm_bwd(const float* code, const float* code_pos, long long stride_b, long long stride_c,
                                     long long stride_y, long long stride_x, const float* coords1,
                                     const float* coords2, const long long* perms, const float* dtiles, float* dcode,
                                     float* dcode_pos, int B, int C, int H, int W, int feature_samples, int nslots,
                                     int perms_are_raw_randperm, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(dtiles && dcode && dcode_pos, "stego_sample_norm_bwd: null pointer");
  STEGO_CHECK_ARG(C <= 96, "stego_sample_norm_bwd: C=%d unsupported (<= 96)", C);
  SampleBwdParams q;
  int rc = fill_sample_params(q.f, code, code_pos, 0, stride_b, stride_c, stride_y, stride_x, nullptr, nullptr,
                              coords1, coords2, perms, nullptr, B, C, CL_CODE_PAD, H, W, feature_samples, nslots);
  if (rc != STEGO_OK) return rc;
  q.f.perms_raw = perms_are_raw_randperm;
  q.dtiles = dtiles; q.dsrc = dcode; q.dsrc_pos = dcode_pos;
  const int warps = 2 * B * H * W;
  sample_norm_bwd_kernel<3><<<(warps + 7) / 8, 256, 0, stream>>>(q);
  STEGO_CHECK_LAUNCH("sample_norm_bwd_kernel");
  return STEGO_OK;
}

// The whole-row kernels take feature_samples^2 <= 128 in one 128-row tile; the multi-tile ones any feature_samples up
// to CT_MAX_FS, in R = ceil(S / 128) * 128 rows.
static int fill_corr_params(CorrParams& p, bool tiled, int B, int fs, int E, int D, int nslots, int ncalls,
                            const int* slot_of_call, const float* shifts, int pointwise, int zero_clamp,
                            int stabilize) {
  const char* who = tiled ? "corr_tiled" : "corr";
  if (!tiled) {
    STEGO_CHECK_ARG(B > 0 && fs * fs <= CL_ROWS && E % 64 == 0 && E >= 64, "corr: B=%d fs=%d E=%d", B, fs, E);
  } else {
    STEGO_CHECK_ARG(B > 0 && fs >= 1 && E % 64 == 0 && E >= 64 && E <= 768, "corr_tiled: B=%d fs=%d E=%d", B, fs, E);
    STEGO_CHECK_ARG(fs <= CT_MAX_FS, "corr_tiled: feature_samples=%d exceeds the supported maximum %d", fs, CT_MAX_FS);
  }
  STEGO_CHECK_ARG(D > 0 && D <= 96, "%s: code dim %d unsupported (<= 96)", who, D);
  STEGO_CHECK_ARG(ncalls > 0 && ncalls <= CL_MAX_CALLS && nslots >= 2, "%s: ncalls=%d nslots=%d", who, ncalls, nslots);
  p.B = B; p.S = fs * fs; p.R = tiled ? (p.S + CL_ROWS - 1) / CL_ROWS * CL_ROWS : CL_ROWS; p.nT = p.R / CL_ROWS;
  p.E = E; p.D = D; p.nslots = nslots; p.ncalls = ncalls;
  for (int k = 0; k < ncalls; ++k) {
    STEGO_CHECK_ARG(slot_of_call[k] >= 0 && slot_of_call[k] < nslots, "%s: slot_of_call[%d]=%d", who, k,
                    slot_of_call[k]);
    p.slot_of_call[k] = slot_of_call[k];
    p.shift[k] = shifts[k];
  }
  p.pointwise = pointwise;
  p.clamp_lo = zero_clamp ? 0.0f : -9999.0f;
  p.clamp_hi = stabilize ? 0.8f : INFINITY;
  p.partials = nullptr; p.rowpart = nullptr; p.cd_out = nullptr; p.fd_out = nullptr;
  p.stats = nullptr; p.rowmean = nullptr; p.gscale = nullptr; p.gelem = nullptr; p.gcd = nullptr; p.dtiles = nullptr;
  p.hist_thr = nullptr; p.hist_counts = nullptr; p.hist_part = nullptr;
  p.pr_ids = nullptr; p.pr_counts = nullptr;
  return STEGO_OK;
}

template <int kVariant>
static int launch_corr(const CUtensorMap& tmF, const CUtensorMap& tmC, const CorrParams& p, cudaStream_t stream) {
  constexpr int kPhase = kVariant & ~CP_HIST;
  constexpr int kRing = (kPhase >= CP_BWD && kPhase <= CP_BWD_DA) ? 2 : 3;
  constexpr size_t smem = size_t(kRing) * 2 * CL_TILE + 8 * CL_TILE + 512 + 1024;
  static_assert(smem <= 232448, "exceeds the 227 KB of shared memory a CTA can opt into");
  constexpr auto kern = corr_kernel<kVariant>;
  if (const int rc = opt_in_smem<kern>(smem, "corr_kernel"); rc != STEGO_OK) return rc;
  const dim3 grid = kPhase == CP_FWD ? dim3(p.B, p.ncalls)
                  : (kPhase == CP_FWD_ROWPART || kPhase == CP_PR) ? dim3(p.B, p.ncalls, p.nT * p.nT)
                  : kPhase == CP_BWD ? dim3(p.B) : dim3(p.B, p.nT);
  kern<<<grid, CL_THREADS, smem, stream>>>(tmF, tmC, p);
  STEGO_CHECK_LAUNCH("corr_kernel");
  return STEGO_OK;
}

// Histogram outputs of the *_fwd_hist entry points (null: the plain forward).
struct HistOut {
  const float* thresholds;  // [TB_THR]
  long long* counts;        // [3][TB_BINS], overwritten
  double* cta_partials;     // scratch [ncalls][B][CTAs per (image, call)][4]
  double* stats;            // [3][4]: min, max, sum, sum of squares per group
};

// Zeroes the counts and points the kernel at the histogram outputs.
static int hist_prepare(CorrParams& p, const HistOut& h, cudaStream_t stream, const char* who) {
  STEGO_CHECK_ARG(h.thresholds && h.counts && h.cta_partials && h.stats, "%s: null histogram pointer", who);
  cudaError_t e = cudaMemsetAsync(h.counts, 0, sizeof(long long) * TB_GROUPS_MAX * TB_BINS, stream);
  if (e != cudaSuccess) return cuda_fail(e, who);
  p.hist_thr = h.thresholds;
  p.hist_counts = reinterpret_cast<unsigned long long*>(h.counts);
  p.hist_part = h.cta_partials;
  return STEGO_OK;
}

// min / max / sums per group from the per-CTA partials: group 0 = call 0, 1 = call 1, 2 = calls 2..
static int hist_finish(const CorrParams& p, const HistOut& h, int ctas_per_call, cudaStream_t stream) {
  const int per_call = p.B * ctas_per_call;
  int first[TB_GROUPS_MAX + 1] = {0, per_call, 2 * per_call, p.ncalls * per_call};
  const int ngroups = p.ncalls < TB_GROUPS_MAX ? p.ncalls : TB_GROUPS_MAX;
  first[ngroups] = p.ncalls * per_call;
  return tb_launch_finish(h.cta_partials, first, ngroups, h.stats, stream);
}

static int corr_fwd(const void* feat_tiles, const void* code_tiles, int B, int feature_samples, int E, int D,
                    int nslots, int ncalls, const int* slot_of_call_host, const float* shifts_host, int pointwise,
                    int zero_clamp, int stabilize, float* partials, float* stats, float* cd_out, float* fdc_out,
                    float* loss_out, const HistOut* hist, cudaStream_t stream) {
  STEGO_CHECK_ARG(feat_tiles && code_tiles && partials && stats && slot_of_call_host && shifts_host,
                  "stego_corr_loss_fwd: null pointer");
  STEGO_CHECK_ARG(!loss_out || (cd_out && fdc_out), "stego_corr_loss_fwd: loss_out needs cd_out and fdc_out");
  CorrParams p;
  int rc = fill_corr_params(p, false, B, feature_samples, E, D, nslots, ncalls, slot_of_call_host, shifts_host,
                            pointwise, zero_clamp, stabilize);
  if (rc != STEGO_OK) return rc;
  p.partials = partials; p.cd_out = cd_out; p.fd_out = fdc_out;
  CUtensorMap tmF, tmC;
  if ((rc = encode_tile_maps(feat_tiles, code_tiles, p, &tmF, &tmC)) != STEGO_OK) return rc;
  if (hist) {
    if ((rc = hist_prepare(p, *hist, stream, "stego_corr_loss_fwd_hist")) != STEGO_OK) return rc;
    if ((rc = launch_corr<CP_FWD | CP_HIST>(tmF, tmC, p, stream)) != STEGO_OK) return rc;
    if ((rc = hist_finish(p, *hist, 1, stream)) != STEGO_OK) return rc;
  } else if ((rc = launch_corr<CP_FWD>(tmF, tmC, p, stream)) != STEGO_OK) {
    return rc;
  }
  corr_finish_kernel<<<ncalls, 32, 0, stream>>>(partials, stats, ncalls, B, p.S, pointwise);
  STEGO_CHECK_LAUNCH("corr_finish_kernel");
  if (loss_out) {
    const long long per_call = 1ll * B * p.S * p.S;
    const long long n = per_call * ncalls;
    corr_loss_elems_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(cd_out, fdc_out, stats, loss_out, per_call, p);
    STEGO_CHECK_LAUNCH("corr_loss_elems_kernel");
  }
  return STEGO_OK;
}

// host arrays (slot_of_call, shifts) are plain host pointers: they are copied into kernel parameters.
extern "C" int stego_corr_loss_fwd(const void* feat_tiles, const void* code_tiles, int B, int feature_samples, int E,
                                   int D, int nslots, int ncalls, const int* slot_of_call_host,
                                   const float* shifts_host, int pointwise, int zero_clamp, int stabilize,
                                   float* partials, float* stats, float* cd_out, float* fdc_out, float* loss_out,
                                   void* stream_) {
  return corr_fwd(feat_tiles, code_tiles, B, feature_samples, E, D, nslots, ncalls, slot_of_call_host, shifts_host,
                  pointwise, zero_clamp, stabilize, partials, stats, cd_out, fdc_out, loss_out, nullptr,
                  reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int stego_corr_loss_fwd_hist(const void* feat_tiles, const void* code_tiles, int B, int feature_samples,
                                        int E, int D, int nslots, int ncalls, const int* slot_of_call_host,
                                        const float* shifts_host, int pointwise, int zero_clamp, int stabilize,
                                        float* partials, float* stats, float* cd_out, float* fdc_out, float* loss_out,
                                        const float* thresholds, long long* hist_counts, double* hist_cta_partials,
                                        double* hist_stats, void* stream_) {
  const HistOut h{thresholds, hist_counts, hist_cta_partials, hist_stats};
  return corr_fwd(feat_tiles, code_tiles, B, feature_samples, E, D, nslots, ncalls, slot_of_call_host, shifts_host,
                  pointwise, zero_clamp, stabilize, partials, stats, cd_out, fdc_out, loss_out, &h,
                  reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int stego_corr_loss_bwd(const void* feat_tiles, const void* code_tiles, int B, int feature_samples, int E,
                                   int D, int nslots, int ncalls, const int* slot_of_call_host,
                                   const float* shifts_host, int pointwise, int zero_clamp, int stabilize,
                                   const float* stats, const float* gscale, const float* gelem, const float* gcd,
                                   float* dtiles, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(feat_tiles && code_tiles && stats && gscale && dtiles && slot_of_call_host && shifts_host,
                  "stego_corr_loss_bwd: null pointer");
  CorrParams p;
  int rc = fill_corr_params(p, false, B, feature_samples, E, D, nslots, ncalls, slot_of_call_host, shifts_host,
                            pointwise, zero_clamp, stabilize);
  if (rc != STEGO_OK) return rc;
  p.stats = stats; p.gscale = gscale; p.gelem = gelem; p.gcd = gcd; p.dtiles = dtiles;
  CUtensorMap tmF, tmC;
  if ((rc = encode_tile_maps(feat_tiles, code_tiles, p, &tmF, &tmC)) != STEGO_OK) return rc;
  return launch_corr<CP_BWD>(tmF, tmC, p, stream);
}

static int corr_tiled_fwd(const void* feat_tiles, const void* code_tiles, int B, int feature_samples, int E, int D,
                          int nslots, int ncalls, const int* slot_of_call_host, const float* shifts_host, int pointwise,
                          int zero_clamp, int stabilize, float* row_partials, float* row_means, float* stats,
                          float* cd_out, float* fdc_out, float* loss_out, const HistOut* hist, cudaStream_t stream) {
  STEGO_CHECK_ARG(feat_tiles && code_tiles && row_partials && row_means && stats && slot_of_call_host && shifts_host,
                  "stego_corr_loss_tiled_fwd: null pointer");
  STEGO_CHECK_ARG(!loss_out || (cd_out && fdc_out), "stego_corr_loss_tiled_fwd: loss_out needs cd_out and fdc_out");
  CorrParams p;
  int rc = fill_corr_params(p, true, B, feature_samples, E, D, nslots, ncalls, slot_of_call_host, shifts_host,
                            pointwise, zero_clamp, stabilize);
  if (rc != STEGO_OK) return rc;
  p.rowpart = row_partials; p.cd_out = cd_out; p.fd_out = fdc_out;
  CUtensorMap tmF, tmC;
  if ((rc = encode_tile_maps(feat_tiles, code_tiles, p, &tmF, &tmC)) != STEGO_OK) return rc;
  if (hist) {
    if ((rc = hist_prepare(p, *hist, stream, "stego_corr_loss_tiled_fwd_hist")) != STEGO_OK) return rc;
    if ((rc = launch_corr<CP_FWD_ROWPART | CP_HIST>(tmF, tmC, p, stream)) != STEGO_OK) return rc;
    if ((rc = hist_finish(p, *hist, p.nT * p.nT, stream)) != STEGO_OK) return rc;
  } else if ((rc = launch_corr<CP_FWD_ROWPART>(tmF, tmC, p, stream)) != STEGO_OK) {
    return rc;
  }
  corr_tiled_finish_kernel<<<ncalls, CT_FINISH_THREADS, 0, stream>>>(p, row_means, stats);
  STEGO_CHECK_LAUNCH("corr_tiled_finish_kernel");
  if (fdc_out) {
    const long long n = 1ll * ncalls * B * p.S * p.S;
    corr_tiled_elems_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(cd_out, fdc_out, row_means, stats,
                                                                              loss_out, p);
    STEGO_CHECK_LAUNCH("corr_tiled_elems_kernel");
  }
  return STEGO_OK;
}

extern "C" int stego_corr_loss_tiled_fwd(const void* feat_tiles, const void* code_tiles, int B, int feature_samples,
                                         int E, int D, int nslots, int ncalls, const int* slot_of_call_host,
                                         const float* shifts_host, int pointwise, int zero_clamp, int stabilize,
                                         float* row_partials, float* row_means, float* stats, float* cd_out,
                                         float* fdc_out, float* loss_out, void* stream_) {
  return corr_tiled_fwd(feat_tiles, code_tiles, B, feature_samples, E, D, nslots, ncalls, slot_of_call_host,
                        shifts_host, pointwise, zero_clamp, stabilize, row_partials, row_means, stats, cd_out, fdc_out,
                        loss_out, nullptr, reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int stego_corr_loss_tiled_fwd_hist(const void* feat_tiles, const void* code_tiles, int B,
                                              int feature_samples, int E, int D, int nslots, int ncalls,
                                              const int* slot_of_call_host, const float* shifts_host, int pointwise,
                                              int zero_clamp, int stabilize, float* row_partials, float* row_means,
                                              float* stats, float* cd_out, float* fdc_out, float* loss_out,
                                              const float* thresholds, long long* hist_counts,
                                              double* hist_cta_partials, double* hist_stats, void* stream_) {
  const HistOut h{thresholds, hist_counts, hist_cta_partials, hist_stats};
  return corr_tiled_fwd(feat_tiles, code_tiles, B, feature_samples, E, D, nslots, ncalls, slot_of_call_host,
                        shifts_host, pointwise, zero_clamp, stabilize, row_partials, row_means, stats, cd_out, fdc_out,
                        loss_out, &h, reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int stego_corr_loss_tiled_bwd(const void* feat_tiles, const void* code_tiles, int B, int feature_samples,
                                         int E, int D, int nslots, int ncalls, const int* slot_of_call_host,
                                         const float* shifts_host, int pointwise, int zero_clamp, int stabilize,
                                         const float* stats, const float* row_means, const float* gscale,
                                         const float* gelem, const float* gcd, float* dtiles, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(feat_tiles && code_tiles && stats && row_means && gscale && dtiles && slot_of_call_host &&
                  shifts_host, "stego_corr_loss_tiled_bwd: null pointer");
  CorrParams p;
  int rc = fill_corr_params(p, true, B, feature_samples, E, D, nslots, ncalls, slot_of_call_host, shifts_host,
                            pointwise, zero_clamp, stabilize);
  if (rc != STEGO_OK) return rc;
  p.stats = stats; p.rowmean = row_means; p.gscale = gscale; p.gelem = gelem; p.gcd = gcd; p.dtiles = dtiles;
  CUtensorMap tmF, tmC;
  if ((rc = encode_tile_maps(feat_tiles, code_tiles, p, &tmF, &tmC)) != STEGO_OK) return rc;
  // dB (every slot, slot 0 included for the intra call) then dA (slot 0): stream order fixes the summation order
  if ((rc = launch_corr<CP_BWD_DB>(tmF, tmC, p, stream)) != STEGO_OK) return rc;
  return launch_corr<CP_BWD_DA>(tmF, tmC, p, stream);
}

extern "C" int stego_sample_label_ids(const void* label, int label_bytes, const float* coords1, const float* coords2,
                                      int* ids, int B, int n_classes, int H, int W, int feature_samples, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(label && coords1 && coords2 && ids, "stego_sample_label_ids: null pointer");
  STEGO_CHECK_ARG(label_bytes == 8 || label_bytes == 4 || label_bytes == 1,
                  "stego_sample_label_ids: label_bytes=%d (8, 4 or 1)", label_bytes);
  STEGO_CHECK_ARG(n_classes >= 1 && n_classes <= 255, "stego_sample_label_ids: n_classes=%d outside 1..255", n_classes);
  STEGO_CHECK_ARG(feature_samples >= 1 && feature_samples <= CT_MAX_FS,
                  "stego_sample_label_ids: feature_samples=%d outside 1..%d", feature_samples, CT_MAX_FS);
  STEGO_CHECK_ARG(B > 0 && H > 1 && W > 1, "stego_sample_label_ids: B=%d H=%d W=%d", B, H, W);
  const int S = feature_samples * feature_samples;
  const int R = (S + CL_ROWS - 1) / CL_ROWS * CL_ROWS;
  const long long n = 2ll * B * S;
  sample_label_ids_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, stream>>>(
      label, label_bytes, coords1, coords2, ids, B, n_classes, H, W, feature_samples, R);
  STEGO_CHECK_LAUNCH("sample_label_ids_kernel");
  return STEGO_OK;
}

extern "C" int stego_corr_pr(const void* feat_tiles, const void* code_tiles, const int* ids, long long* counts, int B,
                             int feature_samples, int E, int D, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(feat_tiles && code_tiles && ids && counts, "stego_corr_pr: null pointer");
  STEGO_CHECK_ARG(feature_samples >= 1 && feature_samples <= CT_MAX_FS,
                  "stego_corr_pr: feature_samples=%d outside 1..%d", feature_samples, CT_MAX_FS);
  const int slot_of_call[1] = {1};
  const float shifts[1] = {0.f};
  CorrParams p;
  int rc = fill_corr_params(p, true, B, feature_samples, E, D, 2, 1, slot_of_call, shifts, 0, 0, 0);
  if (rc != STEGO_OK) return rc;
  p.pr_ids = ids;
  p.pr_counts = reinterpret_cast<unsigned long long*>(counts);
  CUtensorMap tmF, tmC;
  if ((rc = encode_tile_maps(feat_tiles, code_tiles, p, &tmF, &tmC)) != STEGO_OK) return rc;
  return launch_corr<CP_PR>(tmF, tmC, p, stream);
}
