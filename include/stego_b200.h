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
 * ---------------------------------------------------------------------------------------------- */
STEGO_API int stego_gemm_bf16(const void* A, int lda, int a_mn_major, const void* B, int ldb, int b_mn_major,
                              int M, int N, int K, void* out, int ldo, int out_bf16, const float* bias, int act,
                              const float* residual, int ldr, int row_div, int splits, int atomic_out,
                              void* stream);

/* `batch` independent GEMMs of one shape in ONE launch: entry b reads A + b * a_batch_stride, B + b * b_batch_stride and
 * writes out + b * out_batch_stride (strides in elements; operand strides multiples of 8).  Rows past M / N of an entry
 * are zero-filled / clipped by TMA, so M and N need not be tile multiples.  This is `tensor_correlation`
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
 * tiles: fp32 [nslots][B][R][72].
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
 * dtiles: fp32 [nslots][B][128][72], must be zero on entry, receives d(loss)/d(normalised sampled code). */
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
/* dtiles: fp32 [nslots][B][R][72], zero on entry.  Two passes recompute fd / cd per block: dB (all slots) then dA
 * (slot 0), each with one CTA owning its output rows. */
STEGO_API int stego_corr_loss_tiled_bwd(const void* feat_tiles, const void* code_tiles, int B, int feature_samples,
                                        int E, int D, int nslots, int ncalls, const int* slot_of_call_host,
                                        const float* shifts_host, int pointwise, int zero_clamp, int stabilize,
                                        const float* stats, const float* row_means, const float* gscale,
                                        const float* gelem, const float* gcd, float* dtiles, void* stream);

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
 * `step` is 1-based; grad is multiplied by grad_scale first (1/world_size after a sum-allreduce). */
STEGO_API int stego_adam_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, long long n,
                              float lr, float beta1, float beta2, float eps, int step, float grad_scale,
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

/* ------------------------------------------------------------------------------------------------
 * k-nearest-neighbour descriptors (SURVEY.md 8(f) rank 1; src/precompute_knns.py:15-21, 83-96):
 *   normed = F.normalize(feats, dim=1);  sims = einsum("nf,mf->nm", normed, normed);  idx = topk(sims, k)[1]
 * fused: the [n][n] similarity matrix is never materialised (wgmma tiles in registers, bf16 hi/lo split = 3 passes,
 * per-row running top-k in the epilogue).  feats: fp32 [n][E] (un-normalised, e.g. GAP-pooled ViT features),
 * E a multiple of 64, 1 <= k <= 32.  planes_scratch: 2*n*E bf16 (16-byte aligned).  idx_out: int64 [n][k], sorted by
 * descending similarity (ties: lower index first; a row is its own nearest neighbour, as in the reference);
 * val_out: optional fp32 [n][k] similarities.
 * ---------------------------------------------------------------------------------------------- */
STEGO_API int stego_knn_topk(const float* feats, int n, int E, int k, void* planes_scratch, long long* idx_out,
                             float* val_out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Dense CRF post-processing (BASELINE.json configs[4]; src/crf.py:22-45 -> pydensecrf, third-party, parity UNPINNED:
 * the kernels follow the published densecrf / permutohedral-lattice algorithm as restated by oracle/crf_oracle.py).
 * Rows of Q / unary / lattice values are 32 floats (classes padded to a warp); C <= 32.
 * ---------------------------------------------------------------------------------------------- */
/* Permutohedral embedding of every pixel of an [H][W] frame: features (x/sxy, y/sxy) for d = 2, plus the three
 * image channels / srgb for d = 5 (image [H][W][3] uint8).  keys [N][d+1] int64 (packed lattice vertex coordinates),
 * bary [N][d+1] fp32 barycentric weights. */
STEGO_API int stego_crf_lattice(int H, int W, int d, float sxy, float srgb, const unsigned char* image, long long* keys,
                                float* bary, void* stream);
/* Splat scale[pixel] * in[pixel][:C] (in null: ones; scale null: 1) onto the lattice (values: [(M+1)][32], zeroed by the
 * caller; row 0 = missing neighbour) and blur along the d+1 axes (n1 / n2: [d+1][M] neighbour ids, -1 = missing).
 * Result in values_tmp for d = 2, in values for d = 5. */
STEGO_API int stego_crf_splat_blur(int d, long long N, int M, int C, const int* offset, const float* bary, const float* scale,
                                   const float* in, const int* n1, const int* n2, float* values, float* values_tmp,
                                   void* stream);
/* NORMALIZE_SYMMETRIC factor of a kernel from the blurred ones-splat: norm[pixel] = 1 / sqrt(K 1 + 1e-20). */
STEGO_API int stego_crf_norm(int d, long long N, const int* offset, const float* bary, const float* values, float* norm_out,
                             void* stream);
/* Class scores [C][N] at full resolution -> unary energies -log(clip(softmax, 1e-5, 1)) [N][32] and Q_0 = softmax(-U). */
STEGO_API int stego_crf_unary(const float* logits, float* unary, float* Q, long long N, int C, void* stream);
/* One mean-field update Q <- softmax(-U + w_g n_g K_g(n_g Q) + w_b n_b K_b(n_b Q)) from the blurred lattice values of the
 * Gaussian (d = 2) and bilateral (d = 5) kernels; q_out [C][N] and argmax_out [N] are optional (last iteration). */
STEGO_API int stego_crf_update(const float* unary, const int* off_g, const float* bary_g, const float* val_g, const float* norm_g,
                               const int* off_b, const float* bary_b, const float* val_b, const float* norm_b, float w_g,
                               float w_b, float* Q, float* q_out, unsigned char* argmax_out, long long N, int C, void* stream);

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
 * src/modules.py:275-276).  a, b: fp32 [B, C, H, W] with arbitrary element strides; cosv / inva / invb: [B*H*W] floats. */
STEGO_API int stego_cosine_fwd(const float* a, long long a_sb, long long a_sc, long long a_sy, long long a_sx, const float* b,
                               long long b_sb, long long b_sc, long long b_sy, long long b_sx, int B, int C, int H, int W,
                               float eps, float* cosv, float* inva, float* invb, void* stream);
/* grad_cos [B*H*W]; da / db (either may be null) are written with the strides of a / b. */
STEGO_API int stego_cosine_bwd(const float* a, long long a_sb, long long a_sc, long long a_sy, long long a_sx, const float* b,
                               long long b_sb, long long b_sc, long long b_sy, long long b_sx, int B, int C, int H, int W,
                               float eps, const float* cosv, const float* inva, const float* invb, const float* grad_cos,
                               float* da, float* db, void* stream);

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
