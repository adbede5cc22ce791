/*
 * stego_b200 — C-ABI of the H100-native STEGO correspondence-distillation hot path.
 *
 * This header is the drop-in boundary.  The reference (mhamilton723/STEGO) has no FFI layer: its
 * hot path is Python over torch ops in src/modules.py / src/dino/vision_transformer.py /
 * src/train_segmentation.py.  Each entry point below replaces the torch-op sequence cited next to
 * it (reference file:line) with hand-written sm_90a kernels; stego_b200/modules.py binds them with
 * ctypes behind the reference's own class / function names (see INTEGRATION.md).
 *
 * Conventions
 *   - every pointer is a borrowed DEVICE pointer into caller-owned (PyTorch-owned) memory; the
 *     library allocates nothing and keeps no pointer after the call returns;
 *   - `stream` is a cudaStream_t passed as void*; all work is enqueued on it, nothing synchronises;
 *   - return value: 0 = ok, -1 = bad argument, -2 = unsupported, -3 = CUDA error;
 *     stego_last_error() returns a thread-local message for the last non-zero status;
 *   - bf16 tensors are raw __nv_bfloat16 (uint16) storage; "tokens-major" means [.., HW, C] with the
 *     channel dimension contiguous (PyTorch channels_last for an NCHW view).
 */
#ifndef STEGO_B200_H_
#define STEGO_B200_H_

#ifdef __cplusplus
extern "C" {
#endif

#define STEGO_API

/* ------------------------------------------------------------------------------------------------
 * Library
 * ---------------------------------------------------------------------------------------------- */
STEGO_API int stego_version(void);
STEGO_API const char* stego_last_error(void);
/* number of CUDA kernels this library has launched in this process (bench.py's gpu_launches) */
STEGO_API long long stego_launch_count(void);

/* ------------------------------------------------------------------------------------------------
 * Dense contraction (wgmma + TMA + mbarrier):
 *     out[M,N] = act(A . B^T + bias[N]) + residual
 * replaces nn.Linear / 1x1 Conv2d calls of the path:
 *   src/dino/vision_transformer.py:80,88 (qkv, proj), :58-62 (fc1+GELU, fc2), :127-131 (patch embed),
 *   src/modules.py:73-81 (cluster1 / cluster2 heads) and their autograd backward (dgrad, wgrad).
 *   a_mn_major = 0: A is [M][lda] (K contiguous);   1: A is stored transposed, [K][lda] (M contiguous)
 *   b_mn_major = 0: B is [N][ldb] (K contiguous);   1: B is [K][ldb] (N contiguous)
 *   lda/ldb multiples of 8 elements (16-byte rows for TMA); a K tail (K % 64 != 0) is zero-filled by TMA.
 *   act: 0 none, 1 GELU(erf) (nn.GELU default), 2 ReLU.
 *   residual: fp32 [M][ldr] added after the activation (may alias out for an in-place update).
 *   row_div > 0 (patch-embed mode): output row r goes to r + r/row_div + 1 (skips the cls slot of
 *     each image) and the residual row is r % row_div + 1 (positional embedding broadcast).
 *   splits > 1 requires atomic_out = 1: split-K partial sums are atomically added into fp32 `out`.
 *   atomic_out = 1 computes out += A . B^T only: a bias, act != 0 or a residual is refused.
 *   Every leading dimension holds a whole row: lda >= K (a_mn_major: >= M), ldb >= K (b_mn_major: >= N),
 *   ldo >= N and, with a residual, ldr >= N; a shorter one is refused.
 *   A refused call returns a non-zero status before anything is launched and leaves `out` untouched.
 * ---------------------------------------------------------------------------------------------- */
STEGO_API int stego_gemm_bf16(const void* A, int lda, int a_mn_major, const void* B, int ldb, int b_mn_major,
                              int M, int N, int K, void* out, int ldo, int out_bf16, const float* bias, int act,
                              const float* residual, int ldr, int row_div, int splits, int atomic_out,
                              void* stream);

/* `batch` independent GEMMs of one shape in ONE launch: entry b reads A + b * a_batch_stride, B + b * b_batch_stride and
 * writes out + b * out_batch_stride (strides in elements; operand strides multiples of 8).  Rows past M / N of an entry
 * are zero-filled / clipped by TMA, so M and N need not be tile multiples; the leading dimensions follow the rules of
 * stego_gemm_bf16.  This is `tensor_correlation`
 * (src/modules.py:283-284: einsum nchw,ncij->nhwij = one [hw, C] x [C, ij] GEMM per image) for ANY h w, i j — the dense
 * S = h w case of SURVEY.md 8(d) included — with the bf16 hi/lo split folded into K ([hi | lo | hi] . [hi | hi | lo]). */
STEGO_API int stego_gemm_bf16_batched(const void* A, int lda, long long a_batch_stride, int a_mn_major, const void* B,
                                      int ldb, long long b_batch_stride, int b_mn_major, int batch, int M, int N, int K,
                                      void* out, int ldo, long long out_batch_stride, int out_bf16, const float* bias,
                                      int act, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Frozen DINO ViT forward pieces (reference: src/dino/vision_transformer.py)
 * ---------------------------------------------------------------------------------------------- */
/* PatchEmbed conv (:127-131) as im2col: img [B][3][H][W] fp32 -> rows [B*(H/p)*(W/p)][3*p*p] bf16,
 * column order = flattening of the conv weight [E][3][p][p]. */
STEGO_API int stego_vit_patchify(const float* img, void* out_bf16, int B, int H, int W, int patch, void* stream);
/* Same, for an image batch already held in bf16 (the precision the fp32 variant rounds to): half the input bytes. */
STEGO_API int stego_vit_patchify_bf16(const void* img_bf16, void* out_bf16, int B, int H, int W, int patch,
                                      void* stream);
/* Flip-TTA im2col (eval_segmentation.py:124-125): the rows of 2B images from img [B][3][H][W] (fp32, or bf16 with
 * img_is_bf16 = 1) -> rows [2B*(H/p)*(W/p)][3*p*p] bf16.  Images 0..B-1 are img, images B..2B-1 are img.flip(3): their
 * patch column px reads source patch W/p-1-px with its pixel columns reversed.  Bit-identical to stego_vit_patchify of
 * the two batches; same argument rules (p = 8 or 16, W % 8 == 0, 16-byte aligned img). */
STEGO_API int stego_vit_patchify_tta(const void* img, int img_is_bf16, void* out_bf16, int B, int H, int W, int patch,
                                     void* stream);
/* prepare_tokens (:203-207): x[b][0][:] = cls_token + pos_embed[0] (fp32 residual stream [B][ntok][E]). */
STEGO_API int stego_vit_cls_rows(float* x, const float* cls_token, const float* pos_embed, int B, int ntok, int E,
                                 void* stream);
/* nn.LayerNorm (:107,111,234): fp32 rows [rows][E] -> bf16. drop_cls_ntok > 0: rows are tokens of images with
 * that many tokens each; the cls token (token 0) is dropped and the output packed [B][ntok-1][E]
 * (src/modules.py:97). E in {128, 384, 768}. */
STEGO_API int stego_layernorm_bf16(const float* x, const float* gamma, const float* beta, void* out_bf16, int rows,
                                   int E, float eps, int drop_cls_ntok, void* stream);
/* Final norm fused with the global average pool of src/precompute_knns.py:19 (`model(img).mean([2, 3])`): x fp32
 * [B][ntok][E] residual stream -> out fp32 [B][E] (+=; zero it first) = mean over the ntok-1 patch tokens of LayerNorm(x). */
STEGO_API int stego_layernorm_gap(const float* x, const float* gamma, const float* beta, float* out, int B, int ntok,
                                  int E, float eps, void* stream);
/* out fp32 [B][N] = x fp32 [B][K] . w^T + bias, w bf16 rows [N] at stride ldw (>= K, a multiple of 8), bias fp32 [N]
 * or null; K a multiple of 8, x and w 16-byte aligned.  The key projection of the pooled LN1 outputs of the last block:
 * the "KK" kNN descriptors (mean over patches of the keys, src/modules.py:98-101 + src/precompute_knns.py:19). */
STEGO_API int stego_linear_rows_f32(const float* x, const void* w_bf16, int ldw, const float* bias, float* out, int B,
                                    int N, int K, void* stream);
/* Attention.forward (:78-90) without the projections: softmax(q k^T / sqrt(64)) v, fused (flash-style) on
 * wgmma; qkv [B][N][3E] bf16 packed q|k|v with heads contiguous inside each third, out [B][N][E] bf16. */
STEGO_API int stego_attention_fwd(const void* qkv, void* out, int B, int N, int E, int heads, void* stream);
/* The attention matrix of the same Attention.forward (:83-84): probs [B][heads][N][N] fp32 row-major =
 * softmax(q k^T / sqrt(64)) of the packed bf16 qkv above.  probs must be 4-byte aligned; B, heads <= 65535. */
STEGO_API int stego_attention_probs(const void* qkv, float* probs, int B, int N, int E, int heads, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Correspondence loss (reference: src/modules.py:275-295, 325-398)
 *
 * "slot" = one distinct sampled operand: 0 = (src, coords1), 1 = (src_pos, coords2),
 * 2+i = (src[perm_i], coords2).  "call" = one ContrastiveCorrelationLoss.helper invocation; its A
 * operand is always slot 0 and its B operand is slot_of_call[call].
 * Operand tiles: bf16 [2 planes (hi, lo)][nslots][B][R][Cpad] with R = ceil(feature_samples^2 / 128) * 128 rows
 * per (plane, slot, image), i.e. R = 128 for feature_samples <= 11; rows >= feature_samples^2 are zero.  Gradient
 * tiles: fp32 [nslots][B][R][96] (one row holds all D <= 96 code channels).
 * ---------------------------------------------------------------------------------------------- */
/* sample (:287-288) + norm (:275-276): bilinear border/align_corners=True gather at the coords, optional
 * per-(image,channel) scale (the Dropout2d noise of modules.py:116), L2 normalise (eps 1e-10), write
 * the hi/lo split tiles.  src strides are in elements; coords are [B][fs][fs][2] fp32;
 * perms [nslots-2][B] int64: super_perm results (:291-295), or — perms_are_raw_randperm = 1 — the raw randperm
 * draws, in which case the kernel applies super_perm's fix-up (p == b -> (p + 1) % B) itself.
 * feature_samples 1..64.  This call and stego_sample_norm_bwd serve both loss kernel pairs below; they replace
 * stego_sample_norm_tiled_fwd / _bwd, which had the same signatures. */
STEGO_API int stego_sample_norm_fwd(const void* src, const void* src_pos, int src_is_bf16, long long stride_b,
                                    long long stride_c, long long stride_y, long long stride_x,
                                    const float* chan_scale, const float* chan_scale_pos, const float* coords1,
                                    const float* coords2, const long long* perms, void* tiles, int B, int C,
                                    int Cpad, int H, int W, int feature_samples, int nslots, int perms_are_raw_randperm,
                                    void* stream);
/* The same tiles for the ground-truth teacher signal of cfg.use_true_labels (train_segmentation.py:135-137):
 * one_hot_feats(label + 1, n_classes + 1) (utils.py:65-66) sampled and normalised without materialising it.  label /
 * label_pos: contiguous [B][H][W] of label_bytes = 8 (int64), 4 (int32) or 1 (uint8) per element.  Class 0 is
 * "unlabelled": a label outside 0 .. n_classes - 1 (-1, uint8 255 or any other value) maps to it, where F.one_hot
 * would raise.  n_classes + 1 <= Cpad <= 256, Cpad a multiple of 64, H and W >= 2; coords, perms, slots and rows as
 * above.  On the same coordinates the tiles are bit-identical to stego_sample_norm_fwd's on the fp32 one-hot map. */
STEGO_API int stego_sample_labels_fwd(const void* label, const void* label_pos, int label_bytes, const float* coords1,
                                      const float* coords2, const long long* perms, void* tiles, int B, int n_classes,
                                      int Cpad, int H, int W, int feature_samples, int nslots,
                                      int perms_are_raw_randperm, void* stream);
/* helper (:325-347) for all calls at once, feature_samples <= 11 (R = 128): fd and cd einsums on wgmma (bf16 hi/lo
 * split, fp32 accumulate), pointwise centring, clamp, shift, product and reduction.  slot_of_call / shifts are HOST arrays.
 * partials: scratch [ncalls][B][8]; stats: out [ncalls][4] = {mean loss, mean cd, old_mean, mean of centred fd}.
 * Optional (may be null): cd_out / fdc_out / loss_out [ncalls][B][S][S] (loss_out needs the other two). */
STEGO_API int stego_corr_loss_fwd(const void* feat_tiles, const void* code_tiles, int B, int feature_samples, int E,
                                  int D, int nslots, int ncalls, const int* slot_of_call_host,
                                  const float* shifts_host, int pointwise, int zero_clamp, int stabilize,
                                  float* partials, float* stats, float* cd_out, float* fdc_out, float* loss_out,
                                  void* stream);
/* Backward of the above wrt the normalised code tiles.  gscale [ncalls] = upstream gradient of each call's mean
 * loss; gelem / gcd (optional) = upstream gradients of the unreduced loss / cd elements [ncalls][B][S][S].
 * dtiles: fp32 [nslots][B][128][96], must be zero on entry, receives d(loss)/d(normalised sampled code). */
STEGO_API int stego_corr_loss_bwd(const void* feat_tiles, const void* code_tiles, int B, int feature_samples, int E,
                                  int D, int nslots, int ncalls, const int* slot_of_call_host,
                                  const float* shifts_host, int pointwise, int zero_clamp, int stabilize,
                                  const float* stats, const float* gscale, const float* gelem, const float* gcd,
                                  float* dtiles, void* stream);
/* Backward of norm + sample for the code tensors: adds into dcode / dcode_pos (same strides as code); every element is
 * written once, in a fixed order (no atomics). */
STEGO_API int stego_sample_norm_bwd(const float* code, const float* code_pos, long long stride_b, long long stride_c,
                                    long long stride_y, long long stride_x, const float* coords1,
                                    const float* coords2, const long long* perms, const float* dtiles, float* dcode,
                                    float* dcode_pos, int B, int C, int H, int W, int feature_samples, int nslots,
                                    int perms_are_raw_randperm, void* stream);

/* Multi-tile counterparts of the two loss calls above for feature_samples 1..64 (S = fs^2 up to 4096 points; the
 * training path uses them for fs >= 12, where S exceeds one 128-row tile).  They take the tiles of
 * stego_sample_norm_fwd and return gradient tiles for stego_sample_norm_bwd.  The fd / cd einsums run per 128x128
 * (row tile, column tile) block on wgmma, with the same bf16 hi/lo split and fp32 accumulation; every reduction runs
 * in a fixed order (no atomics), so results are bit-reproducible run to run. */
/* row_partials: scratch [ncalls][B][R / 128][R][4] (per-row, per-column-tile sums of fd, clamp(cd) * fd, clamp(cd),
 * cd); row_means: out [ncalls][B][R], the pointwise row means of fd (0 when !pointwise), needed by the backward;
 * stats / cd_out / fdc_out / loss_out as for stego_corr_loss_fwd (fdc_out is centred with the row means). */
STEGO_API int stego_corr_loss_tiled_fwd(const void* feat_tiles, const void* code_tiles, int B, int feature_samples,
                                        int E, int D, int nslots, int ncalls, const int* slot_of_call_host,
                                        const float* shifts_host, int pointwise, int zero_clamp, int stabilize,
                                        float* row_partials, float* row_means, float* stats, float* cd_out,
                                        float* fdc_out, float* loss_out, void* stream);
/* dtiles: fp32 [nslots][B][R][96], zero on entry.  Two passes recompute fd / cd per block: dB (all slots) then dA
 * (slot 0), each with one CTA owning its output rows. */
STEGO_API int stego_corr_loss_tiled_bwd(const void* feat_tiles, const void* code_tiles, int B, int feature_samples,
                                        int E, int D, int nslots, int ncalls, const int* slot_of_call_host,
                                        const float* shifts_host, int pointwise, int zero_clamp, int stabilize,
                                        const float* stats, const float* row_means, const float* gscale,
                                        const float* gelem, const float* gcd, float* dtiles, void* stream);

/* Salient sampling locations (cfg.use_salience; src/modules.py:298-311, 357-364, fed from train_segmentation.py:147-152)
 * for both maps of a batch, in two launches.  salience / salience_pos: contiguous [B][H][W] masks of mask_bytes = 4
 * (fp32, a pixel is salient when != 0: NaN is, -0 is not) or 1 (bool / uint8, != 0).  Unit u = map * B + b (map 0 =
 * salience, 1 = salience_pos) is the u-th torch.randint call of the reference.  Which generator that call uses
 * depends on the image: randint(count, (fs^2,)) runs on the CPU generator (the reference passes no device), and an
 * image without nonzeros draws randint(H, (fs^2, 2)) on the CUDA generator.  So the caller reads the counts first.
 * stego_salience_counts: counts [2B] int32 = the nonzeros of each unit's mask. */
STEGO_API int stego_salience_counts(const void* salience, const void* salience_pos, int mask_bytes, int B, int H, int W,
                                    int* counts, void* stream);
/* stego_salience_coords: coords1 / coords2 [B][fs][fs][2] (may alias u_reg1 / u_reg2) = nz * keep + reg * (1 - keep)
 * with nz = (x, y) * fl(1 / H) * 2 - 1 of the picked pixel, reg = u_reg * 2 - 1, keep = u_keep > 0.1f, each operation
 * rounded once in fp32.  u_reg1 / u_reg2 [B][fs][fs][2] and u_keep [B][fs][fs]: the uniforms of the three torch.rand
 * draws that follow the randint calls.
 * draws_u32 [2B][2 fs^2] (element li of unit u at u * 2 fs^2 + li): for a unit with nonzeros, elements 0 .. fs^2 - 1
 * pick the (draw % count)-th nonzero in row-major order (the CPU randint's values).  For an empty unit y, x = draw % H
 * from elements 2 s, 2 s + 1, where the draws are Philox4x32-10 at (seed, offsets[u]), as torch's CUDA randint makes
 * them (offsets: device int64 [2B], each a multiple of 4), or, with offsets null, the given elements (tests).
 * scratch: stego_salience_scratch_bytes(B, H, W) bytes, 4-byte aligned (null when that is 0).
 * Limits: B, H, W >= 1, H * W < 2^28 (torch's randint switches to 64-bit draws there), fs 1..64. */
STEGO_API int stego_salience_coords(const void* salience, const void* salience_pos, int mask_bytes, int B, int H, int W,
                                    int feature_samples, long long seed, const long long* offsets,
                                    const void* draws_u32, const float* u_reg1, const float* u_reg2,
                                    const float* u_keep, float* coords1, float* coords2, void* scratch, void* stream);
/* Scratch bytes stego_salience_coords needs: 0 while an image's bitmap (ceil(H W / 32) words and their prefix) fits in
 * the 96 KB of shared memory a CTA uses (H W <= 393 216), else 16 B ceil(H W / 32).  No CUDA call. */
STEGO_API long long stego_salience_scratch_bytes(int B, int H, int W);

/* ------------------------------------------------------------------------------------------------
 * Aug-alignment views (src/data.py:527-563 with the transforms of src/train_segmentation.py:408-416): img_aug and
 * coord_aug of a batch, with torchvision's tensor arithmetic, in two launches.
 * ---------------------------------------------------------------------------------------------- */
/* Words per sample in the records of stego_aug_views (48).  No CUDA call. */
STEGO_API int stego_aug_record_words(void);
/* Scratch bytes stego_aug_views needs for B samples at output size `size`: fp64 partial sums of contrast's mean and an
 * fp32 [B][3][size][size] intermediate.  No CUDA call. */
STEGO_API long long stego_aug_scratch_bytes(int B, int size);
/* img fp32 [B][3][H][W] at element strides (batch, channel, y, x), the normalised frames.  records: device int32
 * [B][48], one per sample, drawn by the host (stego_b200/augment.py): word 0 flip, 1-4 the crop box (top, left, height,
 * width) on the flipped frame, inside it; 5-8 ColorJitter's fn_idx; 9 grayscale; 10 blur; as fp32 bits: 11-12 the
 * brightness factor b and fl(1 - b), 13-14 contrast, 15-16 saturation, 17 the hue factor, 18-42 the 5x5 Gaussian
 * weights (row-major).  Outputs: img_aug fp32 [B][3][size][size] = flip, crop, antialiased bilinear resize
 * (align_corners=False), the four jitter ops in fn_idx order (contrast blends with the mean of rgb_to_grayscale at that
 * point of the chain), grayscale, 5x5 blur with reflect padding; coord_aug fp32 [B][size][size][2] = the same flip,
 * crop and resize of meshgrid(linspace(-1, 1, H), linspace(-1, 1, W)) ("ij": element 0 varies along rows).
 * scratch: stego_aug_scratch_bytes(B, size) bytes, 8-byte aligned.  B 1..65535, H, W >= 1, size 3..8192.  The means are
 * summed in a fixed order: repeated calls return identical bits. */
STEGO_API int stego_aug_views(const float* img, long long stride_b, long long stride_c, long long stride_y,
                              long long stride_x, int B, int H, int W, int size, const int* records, void* scratch,
                              float* img_aug, float* coord_aug, void* stream);

/* ------------------------------------------------------------------------------------------------
 * TensorBoard histograms (SummaryWriter.add_histogram with its default bins="tensorflow")
 * ---------------------------------------------------------------------------------------------- */
/* The 1549 float64 bucket edges of torch's SummaryWriter.default_bins (edges, may be null) and the 1550 fp32
 * thresholds the kernels compare against (thresholds, may be null): the smallest float >= each edge, then the largest
 * float <= the last edge.  Host arrays; no CUDA call. */
STEGO_API int stego_tb_tables(double* edges, float* thresholds);
/* np.histogram(values.astype(float64), default_bins) of n fp32 device values: counts [1548] int64 (overwritten; bucket
 * k is [e_k, e_k+1), the last one closed, values outside [e_0, e_1548] not counted) and stats [4] float64 = min, max,
 * sum, sum of squares.  thresholds: device copy of stego_tb_tables' table; cta_partials: scratch [264][4] float64.
 * Counts are exact; the sums are reduced in a fixed order (bit-reproducible). */
STEGO_API int stego_tb_histogram(const float* values, long long n, const float* thresholds, long long* counts,
                                 double* cta_partials, double* stats, void* stream);
/* stego_corr_loss_fwd / stego_corr_loss_tiled_fwd that also bin cd (the values cd_out would hold, padding excluded)
 * into three histograms: group 0 = call 0, 1 = call 1, 2 = calls 2.. (the negatives).  Every other output is
 * bit-identical to the plain call.  hist_counts [3][1548] int64 (overwritten); hist_stats [3][4] float64 as for
 * stego_tb_histogram; hist_cta_partials: scratch [ncalls][B][4] float64 (tiled: [ncalls][B][(R/128)^2][4]). */
STEGO_API int stego_corr_loss_fwd_hist(const void* feat_tiles, const void* code_tiles, int B, int feature_samples,
                                       int E, int D, int nslots, int ncalls, const int* slot_of_call_host,
                                       const float* shifts_host, int pointwise, int zero_clamp, int stabilize,
                                       float* partials, float* stats, float* cd_out, float* fdc_out, float* loss_out,
                                       const float* thresholds, long long* hist_counts, double* hist_cta_partials,
                                       double* hist_stats, void* stream);
STEGO_API int stego_corr_loss_tiled_fwd_hist(const void* feat_tiles, const void* code_tiles, int B,
                                             int feature_samples, int E, int D, int nslots, int ncalls,
                                             const int* slot_of_call_host, const float* shifts_host, int pointwise,
                                             int zero_clamp, int stabilize, float* row_partials, float* row_means,
                                             float* stats, float* cd_out, float* fdc_out, float* loss_out,
                                             const float* thresholds, long long* hist_counts,
                                             double* hist_cta_partials, double* hist_stats, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Correspondence precision-recall (plot_pr_curves.py:108-167): do feature / code correlations predict label agreement?
 * ---------------------------------------------------------------------------------------------- */
#define STEGO_PR_BINS 4096
/* ids: out int32 [2][B][R] (R = ceil(fs^2 / 128) * 128; rows fs^2 .. R - 1 are not written): for slot 0 (coords1) and
 * slot 1 (coords2) of image b, the class of sample s when every bilinear tap with a non-zero weight has that class,
 * else -1.  A tap's class is label + 1 for 0 <= label < n_classes, else 0 ("unlabelled").  label: contiguous
 * [B][H][W] of label_bytes = 8 / 4 / 1; coords as for stego_sample_norm_fwd.  n_classes 1..255, fs 1..64. */
STEGO_API int stego_sample_label_ids(const void* label, int label_bytes, const float* coords1, const float* coords2,
                                     int* ids, int B, int n_classes, int H, int W, int feature_samples, void* stream);
/* Adds the precision-recall counts of one batch to counts, int64 [2][2][STEGO_PR_BINS]: [0 = fd (features), 1 = cd
 * (code)][0 = negative, 1 = positive pair][bin].  Tiles: stego_sample_norm_fwd's with nslots = 2 of the same image
 * (slot 0 at coords1, slot 1 at coords2), features E wide (a multiple of 64, <= 768), code padded to 128 (D <= 96).
 * Every pair (i, j) of samples of one image is scored by its raw cosine, binned at
 * clamp(floor((score + 1) * STEGO_PR_BINS / 2), 0, STEGO_PR_BINS - 1) in fp32, and is positive when ids of both
 * samples are the same class (>= 0).  Integer atomics: the counts are exact and reproducible. */
STEGO_API int stego_corr_pr(const void* feat_tiles, const void* code_tiles, const int* ids, long long* counts, int B,
                            int feature_samples, int E, int D, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Dense correspondence heatmaps (plot_dino_correspondence.py:39-58, get_heatmaps), in four steps around one
 * stego_gemm_bf16_batched call raw[b] = q_ops[b] . t_ops[b]^T (M = P, N = h w, K = nseg * Epad, fp32 [B][P][h w]).
 * Feature maps have element strides (batch, channel, y, x), fp32 or bf16 (is_bf16); 1 <= E <= 768, Epad a multiple of 8
 * >= E (<= 768); nseg = 2 for a bf16 target, 3 for an fp32 one.
 * ---------------------------------------------------------------------------------------------- */
/* Target map [B][E][h][w] -> ops bf16 [B][h w][nseg * Epad] (K-major; bf16: [t | t], fp32: [hi | hi | lo] with
 * t = hi + lo; zeros past E in each segment) and inv_norm fp32 [B][h w] = 1 / max(||t||, 1e-12). */
STEGO_API int stego_heatmap_prep_target(const void* target, int target_is_bf16, long long stride_b, long long stride_c,
                                        long long stride_y, long long stride_x, int B, int E, int h, int w, int Epad,
                                        void* ops, float* inv_norm, void* stream);
/* grid_sample (bilinear, border, align_corners=True) of feats [B][E][h][w] at points fp32 [B][P][2] = (x, y), L2
 * normalised in fp32 (eps 1e-12) and split n = hi + lo -> ops bf16 [B][P][nseg * Epad]: [hi | lo] (nseg 2) or
 * [hi | lo | hi] (nseg 3), the counterpart of the target's operand. */
STEGO_API int stego_heatmap_sample_queries(const void* feats, int feats_is_bf16, long long stride_b, long long stride_c,
                                           long long stride_y, long long stride_x, const float* points, int B, int P,
                                           int E, int h, int w, int Epad, int nseg, void* ops, void* stream);
/* In place on corr fp32 [B][P][hw] (the GEMM's raw dots): c = raw * inv_norm[b], then max(c - mean_j c, 0) per row;
 * the row mean is reduced in a fixed order (bit-reproducible). */
STEGO_API int stego_heatmap_finish(float* corr, const float* inv_norm, int B, int P, int hw, void* stream);
/* F.interpolate(in, (H, W), mode="bilinear", align_corners=True): in fp32 [n][h][w] -> out fp32 [n][H][W] (64-bit
 * offsets, H <= 65535), with the arithmetic of ATen's CUDA upsample_bilinear2d; 16-byte streaming stores when W % 4 == 0
 * and out is 16-byte aligned. */
STEGO_API int stego_heatmap_upsample(const float* in, float* out, long long n, int h, int w, int H, int W, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Segmentation head glue (reference: src/modules.py:73-81, 108-118) and optimiser
 * ---------------------------------------------------------------------------------------------- */
/* Apply the three Dropout2d noises of DinoFeaturizer.forward (:109,:111,:116) in one pass:
 * out_i[b][p][c] = feat[b][p][c] * mask_i[b][c]; feat/out tokens-major bf16 [B*hw][E]; mask fp32 [B][E].
 * Any (mask_i, out_i) pair may be null. */
STEGO_API int stego_head_dropout3(const void* feat_bf16, const float* mask1, const float* mask2, const float* mask3,
                                  void* out1, void* out2, void* out3, int B, int hw, int E, void* stream);
/* fp32 [rows][ld_in] (first C columns) -> bf16 [rows][ld_out] zero-padded: packs d(code) as a GEMM operand. */
STEGO_API int stego_cast_pad_bf16(const float* in, int ld_in, int C, void* out_bf16, int ld_out, long long rows,
                                  void* stream);
/* ReLU backward between the two cluster2 convs: out = bf16(dh * (h > 0)), n elements (multiple of 4). */
STEGO_API int stego_relu_bwd_bf16(const float* dh, const void* h_bf16, void* out_bf16, long long n, void* stream);
/* Bias gradients: out[C] += column sums of in [rows][ld] (fp32 or bf16). */
STEGO_API int stego_colsum(const void* in, int in_is_bf16, int ld, int C, long long rows, float* out, void* stream);
/* torch.optim.Adam step (src/train_segmentation.py:379-381; amsgrad off, weight_decay 0) on a flat fp32 buffer;
 * `step` is 1-based; grad is multiplied by grad_scale first (1/world_size after a sum-allreduce).  The coefficients
 * 1 - beta1, 1 - beta2, lr / (1 - beta1^step) and sqrt(1 - beta2^step) are formed in double from the double
 * hyper-parameters and rounded to fp32 once each. */
STEGO_API int stego_adam_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, long long n,
                              double lr, double beta1, double beta2, double eps, int step, float grad_scale,
                              void* stream);

/* The scalar arithmetic at the end of training_step (src/train_segmentation.py:196-201, 219-225) in one launch:
 * out4[0] = sum_c call_weights_host[c] * corr_stats[c][0] + extra0[0] + extra1[0]   (total loss)
 * out4[1] = the weighted correspondence term alone, out4[2] / out4[3] = mean loss / mean cd of calls 2.. (negatives).
 * corr_stats is stego_corr_loss_fwd's `stats`; extra0/extra1 are device scalars or null; ncalls <= 16. */
STEGO_API int stego_step_losses(const float* corr_stats, int ncalls, const float* call_weights_host,
                                const float* extra0, const float* extra1, float* out4, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Probes
 * ---------------------------------------------------------------------------------------------- */
/* ClusterLookup.forward (src/modules.py:146-161). x has element strides (batch, channel, pixel) with
 * pixel = y*W + x; clusters [n][C].  use_alpha = 0 is `alpha is None` (one-hot argmax).
 * loss_out[0] = -(probs * inner_products).sum(1).mean().  Optional outputs (may be null): assign [B][npix]
 * int64 argmax, probs [B][n][npix], log_probs [B][n][npix] (needs alpha).  scratch: >= 16*SMs floats. */
STEGO_API int stego_cluster_lookup_fwd(const float* x, long long stride_b, long long stride_c, long long stride_pix,
                                       const float* clusters, int B, int C, int n_classes, long long npix,
                                       int use_alpha, float alpha, long long* assign, float* probs, float* log_probs,
                                       float* loss_out, float* scratch, void* stream);
/* Gradient of the ClusterLookup loss wrt the centroids: dclusters += grad_loss_dev[0] * dloss/dclusters
 * (the upstream scalar is a DEVICE pointer so autograd never synchronises). dnc_scratch [n][C] zero on entry. */
STEGO_API int stego_cluster_lookup_bwd(const float* x, long long stride_b, long long stride_c, long long stride_pix,
                                       const float* clusters, int B, int C, int n_classes, long long npix,
                                       int use_alpha, float alpha, const float* grad_loss_dev,
                                       float* dnc_scratch, float* dclusters, void* stream);
/* Linear probe step (src/train_segmentation.py:213-218): 1x1 conv on tokens-major code [B*h*w][ld_code],
 * bilinear upsample to [H][W] (align_corners=False), CrossEntropyLoss over pixels with 0 <= label < n.
 * label [B][H][W]: int64 (the reference's dtype), int32 or uint8 — label_bytes = 8 / 4 / 1; labels outside [0, n)
 * are ignored (-1 in the signed types, 255 in uint8: the same mask as src/train_segmentation.py:211).
 * loss_out[0] = mean CE, loss_out[1] = valid pixel count.  If dlogits_scratch is non-null (zeroed by the
 * caller) the backward also runs: dW [n][C] and db [n] += grad_loss * gradient.
 * logits_scratch / dlogits_scratch: [B*h*w][32] floats; partials_scratch: >= 16*SMs floats. */
STEGO_API int stego_linear_probe_ce(const float* code, long long ld_code, int C, const float* W, const float* bias,
                                    int n_classes, const void* label, int label_bytes, int B, int h, int w, int H,
                                    int Wimg, float* logits_scratch, float* dlogits_scratch, float* partials_scratch,
                                    float* loss_out, float grad_loss, float* dW, float* db, void* stream);
/* stego_linear_probe_ce for a wide code: the backbone's C = 384 / 768 channels (projection_type None).  Same arguments
 * plus dfix_scratch, int64 [B*h*w][32] zeroed by the caller (needed with dlogits_scratch): the logit gradient is
 * accumulated there as exact fixed-point integers, and dW / db are reduced over the rows in a fixed order, so two
 * identical calls give bit-identical results. */
STEGO_API int stego_linear_probe_ce_wide(const float* code, long long ld_code, int C, const float* W, const float* bias,
                                         int n_classes, const void* label, int label_bytes, int B, int h, int w, int H,
                                         int Wimg, float* logits_scratch, float* dlogits_scratch,
                                         long long* dfix_scratch, float* partials_scratch, float* loss_out,
                                         float grad_loss, float* dW, float* db, void* stream);
/* The training step's ClusterLookup (alpha None, src/train_segmentation.py:221-223) on a wide code: the backbone's
 * C = 384 / 768 channels (projection_type None), x [rows][ld_x] fp32 tokens-major, clusters [n][C] with n <= 64.
 * loss_out[0] = -mean_r max_k <x_r / |x_r|, c_k / |c_k|>; with dclusters (and dnc_scratch [n][C], zeroed by the
 * caller) also dclusters += d loss_out[0] / d clusters.  Scratch: assign_scratch int32 [rows], inv_scratch fp32
 * [rows], partials_scratch >= 16*SMs floats.  Every reduction over rows has a fixed order (no atomics). */
STEGO_API int stego_cluster_lookup_wide(const float* x, long long ld_x, long long rows, int C, const float* clusters,
                                        int n_classes, int* assign_scratch, float* inv_scratch, float* partials_scratch,
                                        float* loss_out, float* dnc_scratch, float* dclusters, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Fused evaluation probes (src/eval_segmentation.py:128-131, BASELINE.json configs[4]):
 *   code_up = F.interpolate(code, (H, W), mode="bilinear", align_corners=False)
 *   lin_log_probs = log_softmax(linear_probe(code_up), 1);  clu_log_probs = cluster_probe(code_up, alpha, log_probs=True)
 * evaluated per output pixel from the LOW-RES code (the [B,C,H,W] upsampled tensor is never materialised).
 *   code: tokens-major low-res code [B*h*w][ld_code] fp32; lin_weight [n_lin][C], lin_bias [n_lin], clusters [n_clu][C];
 *   lr_scratch: [B*h*w][80] floats, 8-byte aligned (low-res logits, centroid dots, fp64 Gram entries).  Outputs (each may be null): log-probabilities [B][n][H][W] fp32 and
 *   per-pixel argmax maps [B][H][W] uint8.  C <= 96, n_lin, n_clu <= 32, H >= h, W >= w.
 * Optional, fused (src/eval_segmentation.py:124-126,138-139; src/utils.py:219-229):
 *   code_flip  the code of the horizontally flipped images: the kernel evaluates (code + flip(code_flip)) / 2 (flip-TTA);
 *   label      [B][H][W] int64 / int32 / uint8 (label_bytes 8 / 4 / 1): UnsupervisedMetrics.update — the int64
 *              confusion counts lin_confusion [n_lin][n_label_classes], clu_confusion [n_clu][n_label_classes] are
 *              incremented at [pred][actual] for every pixel with 0 <= label < n_label_classes and pred < n_label_classes.
 * ---------------------------------------------------------------------------------------------- */
STEGO_API int stego_eval_probes(const float* code, const float* code_flip, long long ld_code, int C, int B, int h, int w,
                                int H, int W, const float* lin_weight, const float* lin_bias, int n_lin,
                                const float* clusters, int n_clu, float alpha, float* lr_scratch, float* lin_log_probs,
                                float* clu_log_probs, unsigned char* lin_argmax, unsigned char* clu_argmax,
                                const void* label, int label_bytes, int n_label_classes, long long* lin_confusion,
                                long long* clu_confusion, void* stream);
/* stego_eval_probes with its outputs placed in a mosaic of tiles (plot_potsdam.py:65-81): frame b is tile tile0 + b of a
 * tile_rows x tiles_per_row grid, in row-major tile order, and its pixel (y, x) goes to row
 * ((tile0 + b) / tiles_per_row) * H + y, column ((tile0 + b) % tiles_per_row) * W + x of a plane of row pitch `pitch`
 * (>= tiles_per_row * W): argmax maps [tile_rows*H][pitch] uint8, log-probabilities [n][tile_rows*H][pitch] fp32.
 * label stays [B][H][W] (the B tiles' own labels); the confusion counts are those of stego_eval_probes. */
STEGO_API int stego_eval_probes_mosaic(const float* code, const float* code_flip, long long ld_code, int C, int B, int h,
                                       int w, int H, int W, const float* lin_weight, const float* lin_bias, int n_lin,
                                       const float* clusters, int n_clu, float alpha, float* lr_scratch,
                                       float* lin_log_probs, float* clu_log_probs, unsigned char* lin_argmax,
                                       unsigned char* clu_argmax, const void* label, int label_bytes,
                                       int n_label_classes, long long* lin_confusion, long long* clu_confusion,
                                       int tile0, int tile_rows, int tiles_per_row, long long pitch, void* stream);

/* ------------------------------------------------------------------------------------------------
 * k-nearest-neighbour descriptors (SURVEY.md 8(f) rank 1; src/precompute_knns.py:15-21, 83-96):
 *   normed = F.normalize(feats, dim=1);  sims = einsum("nf,mf->nm", normed, normed);  idx = topk(sims, k)[1]
 * fused: the [n][n] similarity matrix is never materialised (wgmma tiles in registers, bf16 hi/lo split = 3 passes,
 * per-row running top-k in the epilogue).  feats: fp32 [n][E] (un-normalised, e.g. GAP-pooled ViT features),
 * E a multiple of 64, 1 <= k <= min(32, n).  planes_scratch: 2*n*E bf16 (16-byte aligned).  idx_out: int64 [n][k]:
 * column 0 is the row's own index, always (the reference's loader, src/data.py:524, draws from columns 1..k as "not the
 * image itself"; the similarity alone would not guarantee it: an exact duplicate ties with the row and a near duplicate's
 * computed similarity can exceed the row's own 1 - O(2^-17); an all-zero row ties with everything at 0); columns 1..k-1
 * are the other rows by (similarity descending, index ascending).
 * val_out: optional fp32 [n][k] computed similarities of those indices (column 0: the row with itself, so columns
 * 1..k-1 are non-increasing and column 1 may exceed column 0 by rounding).
 * ---------------------------------------------------------------------------------------------- */
STEGO_API int stego_knn_topk(const float* feats, int n, int E, int k, void* planes_scratch, long long* idx_out,
                             float* val_out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Dense CRF post-processing (BASELINE.json configs[4]; src/crf.py:22-45 -> pydensecrf, third-party, parity UNPINNED:
 * the kernels follow the published densecrf / permutohedral-lattice algorithm as restated by oracle/crf_oracle.py).
 * Rows of Q / unary / lattice values are 32 floats per probe (classes padded to a warp); C <= 32.
 * ---------------------------------------------------------------------------------------------- */
/* Permutohedral embedding of every pixel of an [H][W] frame: features (x/sxy, y/sxy) for d = 2, plus the three
 * image channels / srgb for d = 5 (image [H][W][3] uint8).  keys [N][d+1] int64 (packed lattice vertex coordinates),
 * bary [N][d+1] fp32 barycentric weights. */
STEGO_API int stego_crf_lattice(int H, int W, int d, float sxy, float srgb, const unsigned char* image, long long* keys,
                                float* bary, void* stream);
/* Class scores [C][N] at full resolution -> unary energies -log(clip(softmax, 1e-5, 1)) [N][32] and Q_0 = softmax(-U). */
STEGO_API int stego_crf_unary(const float* logits, float* unary, float* Q, long long N, int C, void* stream);
/* NORMALIZE_SYMMETRIC factor norm [N] = 1 / sqrt(K 1 + 1e-20) of a lattice (offset, bary [N][d+1]; CSR rowptr [M+1]
 * and slots [N*(d+1)] = pixel*(d+1)+vertex sorted by point; n1 / n2 [d+1][M], -1 = missing); values, values_tmp [M]
 * scratch. */
STEGO_API int stego_crf_norm(int d, long long N, int M, const int* offset, const float* bary, const int* rowptr,
                             const int* slots, const int* n1, const int* n2, float* values, float* values_tmp,
                             float* norm_out, void* stream);
/* n_iter >= 1 mean-field iterations Q <- softmax(-U + w_g n_g K_g(n_g Q) + w_b n_b K_b(n_b Q)) of B frames of N pixels,
 * deterministic (gather splats, no float atomics).  One probe (n_clu = 0): rows of 32 floats per pixel and lattice
 * point, classes n_lin (unary and Q from stego_crf_unary).  Two probes: rows of 64 floats, the linear probe in
 * [0, 32) and the cluster probe in [32, 64) (stego_eval_crf_unary).  Position lattice (*_g, Mg points): one frame's,
 * shared by the B frames.  Bilateral lattice (*_b, Mb points): the frames' lattices concatenated over B*N pixels.
 * Scratch val_g, tmp_g [B*Mg][row], val_b, tmp_b [Mb][row].  Last-iteration outputs, each optional: marginals
 * lin_q [B][n_lin][N], clu_q [B][n_clu][N]; argmax maps lin_pred, clu_pred [B][N] uint8 (lowest index on ties); with
 * label [B][N] (label_bytes 8 / 4 / 1) the int64 confusion counts lin_conf [n_lin][n_label_classes],
 * clu_conf [n_clu][n_label_classes] are incremented at [pred][actual] for every pixel with
 * 0 <= label < n_label_classes and pred < n_label_classes. */
STEGO_API int stego_crf_mean_field(int B, long long N, int n_lin, int n_clu, int n_iter, const float* unary, float* Q,
                                   const int* off_g, const float* bary_g, const int* rowptr_g, const int* slots_g,
                                   const int* n1_g, const int* n2_g, const float* norm_g, int Mg,
                                   const int* off_b, const float* bary_b, const int* rowptr_b, const int* slots_b,
                                   const int* n1_b, const int* n2_b, const float* norm_b, int Mb, float w_g,
                                   float w_b, float* val_g, float* tmp_g, float* val_b, float* tmp_b, float* lin_q,
                                   float* clu_q, unsigned char* lin_pred, unsigned char* clu_pred,
                                   const void* label, int label_bytes, int n_label_classes, long long* lin_conf,
                                   long long* clu_conf, void* stream);

/* ---- CRF-refined evaluation (src/eval_segmentation.py:124-141 with run_crf=True): both probes' dense CRFs for a batch
 * of frames through stego_crf_mean_field with two probes per row.
 * stego_eval_crf_unary: the inputs of stego_eval_probes (lr_scratch [B*h*w][80] floats) -> unary energies
 *   -log(clip(softmax(probe), 1e-5, 1)) and the initial Q = softmax(-U), both [B*H*W][64] fp32, 16-byte aligned. */
STEGO_API int stego_eval_crf_unary(const float* code, const float* code_flip, long long ld_code, int C, int B, int h, int w,
                                   int H, int W, const float* lin_weight, const float* lin_bias, int n_lin,
                                   const float* clusters, int n_clu, float alpha, float* lr_scratch, float* unary, float* Q,
                                   void* stream);
/* stego_eval_crf_unary with the rows placed in a mosaic (the addressing of stego_eval_probes_mosaic: pixel (y, x) of
 * frame b is row ((tile0 + b) / tiles_per_row * H + y) * pitch + (tile0 + b) % tiles_per_row * W + x).  probes = 3:
 * rows of both probes (64 floats); 1 or 2: rows of 32 floats of the linear or the cluster probe alone
 * (stego_crf_mean_field's one-probe rows). */
STEGO_API int stego_eval_crf_unary_mosaic(const float* code, const float* code_flip, long long ld_code, int C, int B,
                                          int h, int w, int H, int W, const float* lin_weight, const float* lin_bias,
                                          int n_lin, const float* clusters, int n_clu, float alpha, float* lr_scratch,
                                          float* unary, float* Q, int probes, int tile0, int tile_rows,
                                          int tiles_per_row, long long pitch, void* stream);

/* ---- wide codes (projection_type None, the DINO baseline: the probes on the backbone's features) ---------------------
 * The four eval entries above also take C = 384 or 768 (fp32 code).  The _bf16 entries below are the same four with
 * a bf16 code and code_flip, C = 384 or 768 only: the backbone's tokens read in place, e.g. the two halves of the
 * [2B, h*w, E] mirrored tokens.  Every other width is refused. */
STEGO_API int stego_eval_probes_bf16(const void* code, const void* code_flip, long long ld_code, int C, int B, int h,
                                     int w, int H, int W, const float* lin_weight, const float* lin_bias, int n_lin,
                                     const float* clusters, int n_clu, float alpha, float* lr_scratch,
                                     float* lin_log_probs, float* clu_log_probs, unsigned char* lin_argmax,
                                     unsigned char* clu_argmax, const void* label, int label_bytes,
                                     int n_label_classes, long long* lin_confusion, long long* clu_confusion,
                                     void* stream);
STEGO_API int stego_eval_probes_mosaic_bf16(const void* code, const void* code_flip, long long ld_code, int C, int B,
                                            int h, int w, int H, int W, const float* lin_weight, const float* lin_bias,
                                            int n_lin, const float* clusters, int n_clu, float alpha,
                                            float* lr_scratch, float* lin_log_probs, float* clu_log_probs,
                                            unsigned char* lin_argmax, unsigned char* clu_argmax, const void* label,
                                            int label_bytes, int n_label_classes, long long* lin_confusion,
                                            long long* clu_confusion, int tile0, int tile_rows, int tiles_per_row,
                                            long long pitch, void* stream);
STEGO_API int stego_eval_crf_unary_bf16(const void* code, const void* code_flip, long long ld_code, int C, int B, int h,
                                        int w, int H, int W, const float* lin_weight, const float* lin_bias, int n_lin,
                                        const float* clusters, int n_clu, float alpha, float* lr_scratch, float* unary,
                                        float* Q, void* stream);
STEGO_API int stego_eval_crf_unary_mosaic_bf16(const void* code, const void* code_flip, long long ld_code, int C, int B,
                                               int h, int w, int H, int W, const float* lin_weight,
                                               const float* lin_bias, int n_lin, const float* clusters, int n_clu,
                                               float alpha, float* lr_scratch, float* unary, float* Q, int probes,
                                               int tile0, int tile_rows, int tiles_per_row, long long pitch,
                                               void* stream);

/* ---- contrastive CRF loss (optional training term; replaces ContrastiveCRFLoss.forward, src/modules.py:449-469, and its
 * autograd backward).  guidance [B, Cg <= 3, H, W] and clusters [B, C <= 80, H, W] are fp32 with arbitrary element strides;
 * coords is the reference's int64 [2][n] tensor (row 0 indexes H, row 1 indexes W; shared by the batch).
 * Workspace, caller-allocated, NP = round_up(n, 64): sel [B][C][NP] floats, gsel [B][NP][4] floats, pos [NP][2] ints.
 * out [B][n][n] = -(<sel_a, sel_b> * (w1 exp(-|dp|^2/2alpha - |dI|^2/2beta) + w2 exp(-|dp|^2/2gamma) - shift)). */
STEGO_API int stego_crf_loss_fwd(const float* guidance, long long g_sb, long long g_sc, long long g_sy, long long g_sx, int Cg,
                                 const float* clusters, long long c_sb, long long c_sc, long long c_sy, long long c_sx, int C,
                                 const long long* coords, int B, int n, int H, int W, float alpha, float beta, float gamma,
                                 float w1, float w2, float shift, float* sel, float* gsel, int* pos, float* out, void* stream);
/* Backward over the workspace the forward filled: grad_out [B][n][n] contiguous, dsel [B][C][NP] scratch; the gradient is
 * ACCUMULATED into dclusters (element strides given; zero-fill it first) with atomics (coords may repeat). */
STEGO_API int stego_crf_loss_bwd(const float* grad_out, const float* sel, const float* gsel, const int* pos,
                                 const long long* coords, int B, int C, int n, float alpha, float beta, float gamma, float w1,
                                 float w2, float shift, float* dsel, float* dclusters, long long c_sb, long long c_sc,
                                 long long c_sy, long long c_sx, void* stream);

/* ---- per-pixel cosine similarity <normalize(a), normalize(b)> over the channel axis and its backward: the arithmetic of the
 * optional reconstruction and augmentation-alignment terms (src/train_segmentation.py:183-199; F.normalize eps semantics of
 * src/modules.py:275-276).  a, b: fp32 [B, C, H, W] with arbitrary element strides; cosv / norma / normb: [B*H*W] floats,
 * the cosine and the unclamped fp32 norms |a|, |b| the backward reads (it needs |a| >= eps, F.normalize's rule). */
STEGO_API int stego_cosine_fwd(const float* a, long long a_sb, long long a_sc, long long a_sy, long long a_sx, const float* b,
                               long long b_sb, long long b_sc, long long b_sy, long long b_sx, int B, int C, int H, int W,
                               float eps, float* cosv, float* norma, float* normb, void* stream);
/* grad_cos [B*H*W]; da / db (either may be null) are written with the strides of a / b. */
STEGO_API int stego_cosine_bwd(const float* a, long long a_sb, long long a_sc, long long a_sy, long long a_sx, const float* b,
                               long long b_sb, long long b_sc, long long b_sy, long long b_sx, int B, int C, int H, int W,
                               float eps, const float* cosv, const float* norma, const float* normb, const float* grad_cos,
                               float* da, float* db, void* stream);

/* ---- sampling half of the aug-alignment term (src/train_segmentation.py:189-199, src/modules.py:287-288): the code of
 * img read at the view's coordinates, ahead of the cosine above.  coord_aug: fp32 [B][S][S][2] contiguous; code: fp32
 * [B][C][h][h] with element strides (sb, sc, sy, sx).  grid [B][h][h][2] = F.interpolate(coord_aug.permute(0, 3, 1, 2), h,
 * mode="bilinear", align_corners=False).permute(0, 2, 3, 1), ATen's arithmetic; sampled [B][C][h][h] contiguous =
 * F.grid_sample(code, grid.permute(0, 2, 1, 3), padding_mode="border", align_corners=True), ATen's arithmetic. */
STEGO_API int stego_aug_align_fwd(const float* coord_aug, int S, const float* code, long long sb, long long sc,
                                  long long sy, long long sx, int B, int C, int h, float* grid, float* sampled,
                                  void* stream);
/* d(code) += the grid_sample backward of dsampled [B][C][h][h] contiguous at the forward's grid, by fp32 atomics
 * (dcode strides as the forward's code). */
STEGO_API int stego_aug_align_bwd(const float* grid, const float* dsampled, int B, int C, int h, float* dcode,
                                  long long sb, long long sc, long long sy, long long sx, void* stream);
/* loss[0] = -mean(cosv[0 .. n)) summed in fp64 in a fixed order (bit-reproducible); total[0] += weight * loss[0] when
 * total is not null. */
STEGO_API int stego_aug_align_loss(const float* cosv, long long n, float weight, float* loss, float* total, void* stream);

/* ---- reconstruction term of the training step (src/train_segmentation.py:183-187): cos = <normalize(decoder(code)),
 * normalize(feat * m3)> per pixel, the decoder a 1x1 conv D -> E in fp32, never written out.  code: fp32 rows [M][ldc]
 * (first D <= 96 columns); feat: bf16 rows [M][ldf] (first E columns); m3: fp32 [M / hw][E] per-image channel scale, or
 * null; weight [E][D], bias [E] fp32.  cosv / nr / nf: [M] floats, the cosine and the unclamped norms |r|, |f|. */
STEGO_API int stego_rec_fwd(const float* code, long long ldc, const void* feat, long long ldf, const float* m3, int hw,
                            const float* weight, const float* bias, long long M, int E, int D, float* cosv, float* nr,
                            float* nf, void* stream);
/* Bytes of the scratch stego_rec_bwd needs on the current device (per-CTA dW / db partials; 0 for bad sizes). */
STEGO_API long long stego_rec_scratch_bytes(long long M, int E, int D);
/* Backward with the forward's inputs and outputs; dcos [1] is d loss / d cos of every pixel.  dcode [M][ldd] (first D
 * columns) is ACCUMULATED into (each row by one CTA, no atomics); dweight [E][D] and dbias [E] are WRITTEN, the rows
 * summed in a fixed order (bit-reproducible). */
STEGO_API int stego_rec_bwd(const float* code, long long ldc, const void* feat, long long ldf, const float* m3, int hw,
                            const float* weight, const float* bias, long long M, int E, int D, const float* cosv,
                            const float* nr, const float* nf, const float* dcos, float* dcode, long long ldd,
                            float* scratch, long long scratch_bytes, float* dweight, float* dbias, void* stream);

/* ---- contrastive CRF term of the training step (src/train_segmentation.py:201-208):
 * crf_loss_fn(resize(img, S), normalize(resize(code, S))).mean() with resize = F.interpolate(bilinear,
 * align_corners=False), evaluated at the n sampled points of the S x S maps only (coords [2][n] int64: rows, then
 * columns).  The taps follow ATen's arithmetic, so the resized values are bit-equal to torch's at those points.
 * Workspace, NP = round_up(n, 64): gsel [B][NP][4] and sel / dsel [B][C][NP] floats, pos [NP][2] ints, nrm [B][NP]
 * floats, tile_sum [B][NP/64][NP/64] doubles.
 * Guidance: img fp32 [B][Cg <= 3][H][W] (element strides) -> gsel, pos. */
STEGO_API int stego_crf_guidance(const float* img, long long sb, long long sc, long long sy, long long sx, int Cg, int H,
                                 int W, const long long* coords, int B, int n, int S, float* gsel, int* pos, void* stream);
/* code fp32 [B][C <= 80][h][w] (element strides) -> raw (the resized code at the samples, [B][C][NP]), sel (raw
 * normalised over the channels), nrm (the unclamped norms), and the fixed-order
 * fp64 sum of every 64 x 64 tile of -(Gram x pairwise kernel) in tile_sum (no [B][n][n] output). */
STEGO_API int stego_crf_mean_fwd(const float* code, long long sb, long long sc, long long sy, long long sx, int C, int h,
                                 int w, const long long* coords, int B, int n, int S, float alpha, float beta, float gamma,
                                 float w1, float w2, float shift, const float* gsel, const int* pos, float* raw,
                                 float* sel, float* nrm, double* tile_sum, void* stream);
/* loss[0] = the mean of the B n^2 outputs, from tile_sum in a fixed order; total[0] += weight * loss[0] when total is
 * not null. */
STEGO_API int stego_crf_mean_loss(const double* tile_sum, int B, int n, float weight, float* loss, float* total,
                                  void* stream);
/* d code (strides as given) += the mean's gradient for the upstream gradient gscalar[0] of every output, through the
 * Gram x kernel product, F.normalize and the bilinear taps, by fp32 atomics; dsel is scratch. */
STEGO_API int stego_crf_mean_bwd(const float* gscalar, const float* sel, const float* nrm, const float* gsel,
                                 const int* pos, const long long* coords, int B, int C, int n, int h, int w, int S,
                                 float alpha, float beta, float gamma, float w1, float w2, float shift, float* dsel,
                                 float* dcode, long long sb, long long sc, long long sy, long long sx, void* stream);

/* ---- data-parallel exchange over NVLink peer memory: gradient all-reduce fused into the Adam update (replaces the DDP
 * all-reduce behind manual_backward + the three optimizer.step() calls, src/train_segmentation.py:227-230, 476).
 * Every rank allocates one peer-visible block [export 2 x n_pad floats | flags world x uint32], exchanges the 64-byte CUDA
 * IPC handles out of band (the host does it over torch.distributed) and opens the other ranks' blocks. */
STEGO_API int stego_p2p_alloc(long long bytes, long long* ptr_out, unsigned char* handle_out);
STEGO_API int stego_p2p_open(const unsigned char* handle, long long* ptr_out);
STEGO_API int stego_p2p_close(long long ptr);
STEGO_API int stego_p2p_free(long long ptr);
/* Copy the local flat gradient into export_slot (= this rank's export[epoch & 1]), store `epoch` into flags[rank] of every
 * rank's block (peer_flags: host array of `world` addresses) and wait until every rank has published `epoch`.  The wait is
 * one 32-thread CTA without shared memory.  status (device int) is set to 1 on time-out. */
STEGO_API int stego_p2p_publish(const float* grad, long long n, float* export_slot, const long long* peer_flags, int rank,
                                int world, int epoch, int* status, int timeout_ms, void* stream);
/* grad[i] = sum over ranks r = 0..world-1 (fixed order) of peer_exports[r][i], read from peer memory; then torch.optim.Adam
 * (amsgrad off, weight decay 0) with grad * grad_scale on every group.  group_desc: ngroups x 7 doubles
 * (start, numel, lr, beta1, beta2, eps, 1-based step). */
STEGO_API int stego_p2p_adam(const long long* peer_exports, int world, float* param, float* grad, float* exp_avg,
                             float* exp_avg_sq, long long n, const double* group_desc, int ngroups, float grad_scale,
                             void* stream);

#ifdef __cplusplus
}
#endif
#endif /* STEGO_B200_H_ */
