"""The training-step configurations the hand-scheduled step accepts beyond the shipped one (ROWS) and its optional modes
alone and crossed with them (MODE_ROWS), both with the reconstruction and CRF terms (REC_CRF_ROWS), their model and
batch builders, and the float64 composition of one training
step from the existing references, shared by tests/test_step_configs_fp64_gpu.py, tests/test_step_modes_fp64_gpu.py,
tests/test_step_rec_crf_fp64_gpu.py and tests/test_step_fp64_reference.py.

The composition chains the stage references: _head_fp64.head_forward (cluster1 + cluster2, or cluster1 alone for the
linear head), _corr_fp64.CorrRef (the correspondence loss on the returned features, Dropout2d-scaled by the third noise
when cfg.dropout), _probes_fp64.linear_ce_ref and cluster_ref on the detached code of img, and _head_fp64.head_backward
of the correspondence loss's d(code).  The modes: any feature_samples (CorrRef's call count and S follow the
coordinates); use_true_labels (the teacher is one_hot_feats(label + 1, n + 1) at label resolution, not Dropout2d-scaled;
train_segmentation.py:135-137); the aug-alignment term (train_segmentation.py:189-199: its cosine's d(code) joins the
correspondence loss's, and the head runs over 3B rows); the cd histograms (the fp64 cd of each loss group binned into
hist.default_bins()).  use_salience and dino_feat_type "KK" change only the inputs (coordinates, tokens).  Plain torch
and device-agnostic: the GPU test feeds it the step's own tensors,
the CPU test pins it to float64 autograd through a restatement of DinoFeaturizer.forward and training_step.
"""
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _corr_fp64 as RC  # noqa: E402
import _head_fp64 as RH  # noqa: E402
import _probes_fp64 as RP  # noqa: E402
import stego_oracle as O  # noqa: E402  (oracle/ is on sys.path through _head_fp64)

# name -> (arch, patch, (H, W) of the frames, (LH, LW) of the labels or None for the frame size, B, n_classes,
#          cfg overrides).  Unless a row says otherwise: ViT-S/8 at 224^2, B = 8, 27 classes, the shipped settings.
BASE = dict(arch="vit_small", patch=8, frame=(224, 224), label=None, B=8, n_classes=27, cfg={})
ROWS = {
    "potsdam_discrete": dict(n_classes=3, cfg=dict(continuous=False)),          # D = 3
    "coco_discrete": dict(cfg=dict(continuous=False)),                          # D = 27
    "dim1": dict(cfg=dict(dim=1)),
    "dim64": dict(cfg=dict(dim=64)),   # the code tiles' second 64-wide k-block is padding only
    "dim65": dict(cfg=dict(dim=65)),   # one real channel in it
    "dim96": dict(cfg=dict(dim=96)),   # the largest code width
    "linear_head": dict(cfg=dict(projection_type="linear")),
    "no_dropout": dict(cfg=dict(dropout=False)),
    "linear_no_dropout": dict(cfg=dict(projection_type="linear", dropout=False)),
    "extra5": dict(cfg=dict(extra_clusters=5)),    # 32 cluster rows: the channels-last cluster kernels
    "extra6": dict(cfg=dict(extra_clusters=6)),    # 33 rows: the generic per-thread cluster kernels
    "classes32_extra32": dict(n_classes=32, cfg=dict(extra_clusters=32)),  # 32 linear classes, 64 cluster rows
    "patch16_s": dict(patch=16),                                             # hw = 196
    "patch16_b": dict(arch="vit_base", patch=16, frame=(320, 320)),          # hw = 400
    "B1": dict(B=1),   # super_perm's negatives are the image itself
    "B3": dict(B=3),
    "nonsquare": dict(frame=(224, 320)),                                     # 28 x 40 features
    "nonsquare_labels": dict(frame=(224, 320), label=(112, 150)),            # 4x and 3.75x label upsampling
    "neg1": dict(cfg=dict(neg_samples=1)),
    "neg_max": dict(cfg=dict(neg_samples=14)),     # 16 loss calls, the most the loss kernels take
    "no_pointwise": dict(cfg=dict(pointwise=False)),
    "stabalize": dict(cfg=dict(zero_clamp=False, stabalize=True)),
}
CONFIGS = {name: {**BASE, **row} for name, row in ROWS.items()}

# The optional modes, alone and crossed with ROWS' configurations.  Extra keys: labels (the dtype of label and
# label_pos), masks (use_salience: "fp32" random masks, or "uint8_empty_full" with an all-zero mask on image 0 and an
# all-ones mask on image 1), hist (a logger and hist_freq = 1: the compared step replays the histogram graph).  The aug
# rows train on square frames at cfg.res (make_model sets it).
TL, SAL, KK, AUG = dict(use_true_labels=True), dict(use_salience=True), dict(dino_feat_type="KK"), \
    dict(aug_alignment_weight=0.6)
MODE_ROWS = {
    "fs12": dict(cfg=dict(feature_samples=12)),         # S = 144: two 128-row tiles
    "fs16": dict(cfg=dict(feature_samples=16)),
    "fs28": dict(cfg=dict(feature_samples=28)),         # seven tiles
    "fs64_B2": dict(B=2, cfg=dict(feature_samples=64)),  # S = 4096, the most the multi-tile kernels take
    "fs16_dim96": dict(cfg=dict(feature_samples=16, dim=96)),  # the multi-tile backward's last column tile
    "fs28_neg14": dict(cfg=dict(feature_samples=28, neg_samples=14)),
    "tl": dict(cfg=TL),
    "tl_potsdam": dict(n_classes=3, labels="uint8", cfg=dict(TL, continuous=False)),
    "tl_classes32_extra32": dict(n_classes=32, labels="int32", cfg=dict(TL, extra_clusters=32)),  # 33-class teacher
    "tl_fs28": dict(cfg=dict(TL, feature_samples=28)),
    "tl_nonsquare_labels": dict(frame=(224, 320), label=(112, 150), cfg=TL),
    "tl_B1": dict(B=1, cfg=TL),
    "sal": dict(masks="fp32", cfg=SAL),
    "sal_uint8_empty_full": dict(masks="uint8_empty_full", cfg=SAL),
    "sal_fs64_B2": dict(B=2, masks="fp32", cfg=dict(SAL, feature_samples=64)),
    "sal_nonsquare": dict(frame=(224, 320), masks="fp32", cfg=SAL),
    "sal_B1": dict(B=1, masks="fp32", cfg=SAL),
    "kk": dict(cfg=KK),
    "kk_patch16_b": dict(arch="vit_base", patch=16, frame=(320, 320), cfg=KK),
    "aug": dict(cfg=AUG),
    "aug_patch16": dict(patch=16, cfg=AUG),                                  # h = 14
    "aug_vitb320": dict(arch="vit_base", frame=(320, 320), cfg=AUG),         # h = 40
    "aug_dim1": dict(cfg=dict(AUG, dim=1)),     # ws.code pitch 8
    "aug_dim27": dict(cfg=dict(AUG, dim=27)),   # pitch 32
    "aug_dim96": dict(cfg=dict(AUG, dim=96)),
    "aug_linear_no_dropout": dict(cfg=dict(AUG, projection_type="linear", dropout=False)),  # no M2 / M3
    "aug_B1": dict(B=1, cfg=AUG),
    "aug_neg14": dict(cfg=dict(AUG, neg_samples=14)),
    "hist": dict(hist=True, cfg={}),
    "hist_fs28_neg14": dict(hist=True, cfg=dict(feature_samples=28, neg_samples=14)),  # 16 calls, 49 CTAs per call
    "hist_tl": dict(hist=True, cfg=TL),
    "everything": dict(B=3, masks="fp32", hist=True, cfg=dict(KK, **TL, **SAL, **AUG, feature_samples=16, dim=27,
                                                              projection_type="linear")),
}
MODE_CONFIGS = {name: {**BASE, "labels": "int64", "masks": None, "hist": False, **row} for name, row in MODE_ROWS.items()}

# The reconstruction and CRF terms (cfg.fused_rec_crf) on ROWS' configurations and the modes: each base row with the
# reconstruction term alone ("rec"), the CRF term alone ("crf") and both ("both"); the CRF term only where its kernels
# take the code (at most 80 channels), and crf_samples rows only with it.
REC, CRF = dict(rec_weight=0.7, fused_rec_crf=True), dict(crf_weight=0.5, fused_rec_crf=True)
_REC_CRF_BASE = {
    "plain": {},
    "no_dropout": dict(cfg=dict(dropout=False)),          # m3 = None in the reconstruction kernels
    "linear_no_dropout": dict(cfg=dict(projection_type="linear", dropout=False)),
    "linear_head": dict(cfg=dict(projection_type="linear")),
    "dim1": dict(cfg=dict(dim=1)),
    "dim27": dict(cfg=dict(dim=27)),
    "dim65": dict(cfg=dict(dim=65)),
    "dim80": dict(cfg=dict(dim=80)),                      # the most channels the CRF kernels take
    "dim96": dict(cfg=dict(dim=96)),                      # reconstruction only
    "patch16_s": dict(patch=16),                          # 14 x 14 code: the CRF resize upsamples 4x
    "patch16_b": dict(arch="vit_base", patch=16, frame=(320, 320)),
    "vitb8_320": dict(arch="vit_base", frame=(320, 320)),  # 40 x 40 code, E = 768
    "nonsquare": dict(frame=(224, 320)),                  # 28 x 40 code: scale_h != scale_w
    "nonsquare_labels": dict(frame=(224, 320), label=(112, 150)),
    "B1": dict(B=1),
    "B3": dict(B=3),
    "neg_max": dict(cfg=dict(neg_samples=14)),
    "extra6": dict(cfg=dict(extra_clusters=6)),
    "classes32_extra32": dict(n_classes=32, cfg=dict(extra_clusters=32)),
    "fs16": dict(cfg=dict(feature_samples=16)),
    "fs28_neg14": dict(cfg=dict(feature_samples=28, neg_samples=14)),
    "tl": dict(cfg=TL),
    "sal": dict(masks="fp32", cfg=SAL),
    "kk": dict(cfg=KK),
    "aug": dict(cfg=AUG),                                 # the aug scatter shares the img rows' accumulators
    "hist": dict(hist=True, cfg={}),                      # the histogram graph replays with the terms
    "crf_samples1": dict(cfg=dict(crf_samples=1)),
    "crf_samples64": dict(cfg=dict(crf_samples=64)),      # one full 64-sample tile
    "crf_samples65": dict(cfg=dict(crf_samples=65)),      # a second tile with one sample
    "everything": dict(B=3, masks="fp32", hist=True, terms=("both",),
                       cfg=dict(KK, **TL, **SAL, **AUG, feature_samples=16, dim=27)),
}


def _rec_crf_rows():
    rows = {}
    for name, row in _REC_CRF_BASE.items():
        row = dict(row)
        cfg, only = row.pop("cfg", {}), row.pop("terms", None)
        for terms, over in (("rec", REC), ("crf", CRF), ("both", dict(REC, **CRF))):
            if only is not None and terms not in only:
                continue
            if "crf_weight" in over and cfg.get("dim", 70) > 80:
                continue
            if "crf_weight" not in over and "crf_samples" in cfg:
                continue
            rows[f"{name}_{terms}"] = dict(row, cfg=dict(cfg, **over))
    return rows


REC_CRF_ROWS = _rec_crf_rows()
REC_CRF_CONFIGS = {name: {**BASE, "labels": "int64", "masks": None, "hist": False, **row}
                   for name, row in REC_CRF_ROWS.items()}

HEAD =["net.cluster1.0.weight", "net.cluster1.0.bias", "net.cluster2.0.weight", "net.cluster2.0.bias",
        "net.cluster2.2.weight", "net.cluster2.2.bias"]
PROBES = ["linear_probe.weight", "linear_probe.bias", "cluster_probe.clusters"]
DECODER = ["decoder.weight", "decoder.bias"]


def make_model(row, dev, fused=True, seed=0):
    from _parity_util import make_model as mk
    cfg = dict(row["cfg"])
    if cfg.get("aug_alignment_weight", 0) > 0:
        cfg["res"] = row["frame"][0]
    if row.get("hist"):
        cfg["hist_freq"] = 1
    model, _ = mk(row["arch"], dev, fused=fused, seed=seed, n_classes=row["n_classes"], patch=row["patch"], **cfg)
    return model


def make_batch(row, dev, seed=1):
    """img, img_pos (img + 0.3 noise) and labels in [-1, n_classes] (both ends ignored) at the row's sizes; with the
    modes: label_pos (use_true_labels; uint8 labels hold 255 for -1), mask / mask_pos at frame size (use_salience) and
    per-sample seeds (the aug-alignment term)"""
    B, (H, W), n, cfg = row["B"], row["frame"], row["n_classes"], row["cfg"]
    LH, LW = row["label"] or row["frame"]
    g = torch.Generator().manual_seed(seed)
    img = torch.randn(B, 3, H, W, generator=g)
    img_pos = img + 0.3 * torch.randn(B, 3, H, W, generator=g)
    label = torch.randint(-1, n + 1, (B, LH, LW), generator=g)
    out = dict(img=img.to(dev), img_pos=img_pos.to(dev), label=label)
    if cfg.get("use_true_labels"):
        out["label_pos"] = torch.randint(-1, n + 1, (B, LH, LW), generator=g)
    dt = getattr(torch, row.get("labels", "int64"))
    for k in ("label", "label_pos"):
        if k in out:
            lab = torch.where(out[k] < 0, 255, out[k]) if dt == torch.uint8 else out[k]
            out[k] = lab.to(dt).to(dev)
    kind = row.get("masks")
    if kind == "fp32":
        out["mask"], out["mask_pos"] = ((torch.rand(B, 1, H, W, generator=g) > t).float().to(dev) for t in (0.6, 0.3))
    elif kind == "uint8_empty_full":
        m = (torch.rand(2, B, H, W, generator=g) > 0.5).to(torch.uint8)
        m[0, 0] = 0   # no salient pixel: the draw falls back to the CUDA generator (Philox)
        m[0, 1] = 1   # every pixel salient
        out["mask"], out["mask_pos"] = m[0].to(dev), m[1].to(dev)
    if cfg.get("aug_alignment_weight", 0) > 0:
        out["seed"] = [1000 * seed + i for i in range(B)]
    return out


def names_of(model):
    """the trainable parameters of the step, in NAMES order (the linear head has no cluster2), then the decoder when
    the reconstruction term trains it"""
    have = dict(model.named_parameters())
    return [k for k in HEAD + PROBES if k in have] + (DECODER if model.cfg.rec_weight > 0 else [])


def loss_cfg(cfg):
    """the loss settings of a model config as the references take them"""
    return O.LossCfg(pointwise=cfg.pointwise, zero_clamp=cfg.zero_clamp, stabalize=cfg.stabalize,
                     feature_samples=cfg.feature_samples, neg_samples=cfg.neg_samples,
                     pos_intra_shift=cfg.pos_intra_shift, pos_inter_shift=cfg.pos_inter_shift,
                     neg_inter_shift=cfg.neg_inter_shift, pos_intra_weight=cfg.pos_intra_weight,
                     pos_inter_weight=cfg.pos_inter_weight, neg_inter_weight=cfg.neg_inter_weight)


def call_weights(cfg):
    """d(total) / d(call mean loss) per loss call: intra, inter, then each negative (train_segmentation.py:169-181)"""
    cw, n = float(cfg.correspondence_weight), int(cfg.neg_samples)
    return [cfg.pos_intra_weight * cw, cfg.pos_inter_weight * cw] + [cfg.neg_inter_weight * cw / n] * n


def one_hot_teacher(label, n_classes, width):
    """one_hot_feats(label + 1, n_classes + 1) (train_segmentation.py:135-137) as a float64 [B, width, LH, LW] map,
    zero-padded to the teacher tile width; a label outside [0, n_classes) is class 0 (build_label_tiles' rule)"""
    lab = label.reshape(label.shape[0], *label.shape[-2:]).long()
    cls = torch.where((lab >= 0) & (lab < n_classes), lab + 1, torch.zeros_like(lab))
    return F.one_hot(cls, width).permute(0, 3, 1, 2).double()


def aug_term(code_img, code_aug, coord_aug, weight, grid=None, dsampled=None):
    """The aug-alignment term (train_segmentation.py:189-199) in float64: grid = interpolate(coord_aug, h, bilinear,
    align_corners=False); sampled = grid_sample(code of img, grid^T, border, align_corners=True); cos = <normalize
    (sampled), normalize(code_aug)>; loss = -mean(cos); and d(w loss) into both codes.  grid / dsampled: the kernels'
    own grid and d(sampled) (stage-wise; None: the reference's).  Also returns the grid_sample backward of |d(sampled)|
    (A, what the scatter's fp32 atomics round against)."""
    B, D, fh, fw = code_img.shape
    g64 = F.interpolate(coord_aug.double().permute(0, 3, 1, 2), (fh, fw), mode="bilinear",
                        align_corners=False).permute(0, 2, 3, 1)
    g = g64 if grid is None else grid.double()
    ci = code_img.detach().double().requires_grad_(True)
    ca = code_aug.detach().double().requires_grad_(True)
    sampled = F.grid_sample(ci, g.permute(0, 2, 1, 3), padding_mode="border", align_corners=True)
    sd = sampled.detach().requires_grad_(True)
    cos = (F.normalize(sd, dim=1, eps=RC.EPS) * F.normalize(ca, dim=1, eps=RC.EPS)).sum(1)
    loss = -cos.mean()
    ds, dca = torch.autograd.grad(weight * loss, (sd, ca))
    up = ds if dsampled is None else dsampled.double()
    dci, = torch.autograd.grad(sampled, ci, up)
    ca2 = code_img.detach().double().requires_grad_(True)
    A, = torch.autograd.grad(F.grid_sample(ca2, g.permute(0, 2, 1, 3), padding_mode="border", align_corners=True), ca2,
                             up.abs())
    return dict(grid=g64, sampled=sampled.detach(), cos=cos.detach(), loss=loss.item(), dsampled=ds, dcode_img=dci,
                dcode_aug=dca, A=A)


def aug_grid_bar(coord_aug):
    """|grid - fp64 resize| of stego_aug_align_fwd: ATen's lambdas are exact (an integer scale), so each value is four
    products and three sums of numbers of magnitude <= m = max|coord_aug|: 6 u m (derivation: test_aug_step_gpu.py)"""
    return 6 * RC.U * coord_aug.abs().max().item()


def aug_sampled_bar(code_img, h):
    """|sampled - fp64 grid_sample at the kernel's grid|: the source position ((g + 1) / 2) (h - 1) is formed with three
    roundings (|dx| <= 3 u h), the weights move by <= 2 (3 u h) + 3 u, the sum of four products adds 4 u; c = max|code|"""
    U = RC.U
    return code_img.abs().max().item() * (4 * (6 * U * h + 3 * U) + 4 * U)


def tap_counts(grid, h):
    """[B, 1, h, h]: how many non-zero-weight taps of the grid land on each code element (the scatter's atomics)"""
    g = grid.double().permute(0, 2, 1, 3)  # the point output (p, q) reads
    x = (((g[..., 0] + 1) / 2) * (h - 1)).clamp(0, h - 1)
    y = (((g[..., 1] + 1) / 2) * (h - 1)).clamp(0, h - 1)
    x0, y0 = x.floor(), y.floor()
    B = grid.shape[0]
    cnt = torch.zeros(B, h * h, dtype=torch.float64, device=grid.device)
    for dy in (0, 1):
        for dx in (0, 1):
            wx = (x - x0) if dx else (x0 + 1 - x)
            wy = (y - y0) if dy else (y0 + 1 - y)
            xi, yi = (x0 + dx).clamp(max=h - 1).long(), (y0 + dy).clamp(max=h - 1).long()
            live = ((wx * wy) != 0) & (x0 + dx <= h - 1) & (y0 + dy <= h - 1)
            cnt.scatter_add_(1, (yi * h + xi).reshape(B, -1), live.double().reshape(B, -1))
    return cnt.view(B, 1, h, h)


def aug_scatter_bar(grid, A, dsampled, h):
    """|d(code) - fp64| of the scatter of d(sampled) at the kernel's grid: each element sums k contributions w g in any
    order ((k + 1) u A, A the fp64 grid_sample backward of |g|), with weights formed in fp32 from the fp32 position (each
    product off by <= (6 h + 8) u absolute): + k (6 h + 8) u max|g|"""
    U = RC.U
    k = tap_counts(grid, h)
    return (k + 1) * U * A + k * (6 * h + 8) * U * dsampled.abs().max().item() + 1e-30


def cd_histograms(corr, edges):
    """The cd histograms of the step (intra_cd: call 0, inter_cd: call 1, neg_cd: the negatives' calls stacked) from
    CorrRef's fp64 cd, binned by np.histogram's rule into the float64 `edges` (hist.default_bins()), with the bins of
    cd -+ E_cd: the kernel's fp32 cd may land anywhere between them.  Per group: counts [bins] of the fp64 cd, lo / hi
    [bins] the counts of the lowest / highest bin each element may land in, ambiguous (lo != hi), and min, max, sum,
    sum of squares with their bars."""
    nb = edges.numel() - 1
    out = [dict(counts=0, lo=0, hi=0, ambiguous=0, min=float("inf"), max=-float("inf"), E_minmax=0.0, sum=0.0,
                E_sum=0.0, sumsq=0.0, E_sumsq=0.0, abs_sum=0.0, num=0) for _ in range(min(corr.ncalls, 3))]

    def binof(x):
        return (torch.searchsorted(edges, x.contiguous(), right=True) - 1).clamp(0, nb - 1).reshape(-1)

    def visit(k, b, x):
        h = out[min(k, 2)]
        cd, E = x["cd"], x["Ecd"]
        lo, mid, hi = binof(cd - E), binof(cd), binof(cd + E)
        for key, ix in (("counts", mid), ("lo", lo), ("hi", hi)):
            h[key] = h[key] + torch.bincount(ix, minlength=nb)
        h["ambiguous"] += int((lo != hi).sum())
        mn, mx = cd.min().item(), cd.max().item()
        if mn < h["min"]:
            h["min"] = mn
        if mx > h["max"]:
            h["max"] = mx
        h["E_minmax"] = max(h["E_minmax"], E.max().item())  # min and max are 1-Lipschitz in the sup norm
        h["sum"] += cd.sum().item()
        h["E_sum"] += E.sum().item()
        h["sumsq"] += (cd * cd).sum().item()
        h["E_sumsq"] += (E * (2 * cd.abs() + E)).sum().item()
        h["abs_sum"] += cd.abs().sum().item()
        h["num"] += cd.numel()
    return out, visit


def compose(tok, B, fh, fw, M1, M2, M3, coords1, coords2, perms, params, label, cfg, n_classes, rnd=True, hid=None,
            code=None, hi=RC.HI, vec8=True, label_pos=None, aug=None, hist_edges=None):
    """One training step in float64 from its inputs.
    tok [nB*hw, E]: backbone tokens of img then img_pos (then img_aug: n = 3 with aug, else 2); M1 / M2 / M3 [nB, E]:
    the Dropout2d noises of the cluster1 input, the cluster2 input (None: linear head) and the returned features (None:
    cfg.dropout off; only its first 2B rows scale anything); coords [B, fs, fs, 2] (any fs) and perms [n_neg, B] (raw
    randperm draws); params: name -> tensor for names_of(model); label [B, LH, LW].
    label_pos: use_true_labels, the teacher is one_hot_teacher of label / label_pos at label resolution.
    aug: dict(coord=coord_aug [B, H, W, 2], w=aug_alignment_weight, grid=, dsampled= (optional, the kernels' own)).
    hist_edges: bin the cd histograms into these edges (cd_histograms).
    rnd: round where the kernels store bf16 (the exact step with rnd=False).  hid / code: the kernel's own hidden
    activation / code storage [nB*hw, >= D] (stage-wise: everything downstream then starts from what the step computed);
    None: the reference's own.  Returns head (head_forward), corr (CorrRef after forward and backward, glosses the call
    weights), dcode [nB*hw, D] and the correspondence loss's bar on it (zero on the img_aug rows), lin (linear_ce_ref), clu (cluster_ref), hb (head_backward of dcode), aug
    (aug_term), hist (cd_histograms), losses (the logged terms and the total) and grads (name -> gradient in the
    parameter's shape)."""
    E = tok.shape[1]
    hw = fh * fw
    nI = 3 if aug is not None else 2
    nonlinear = M2 is not None or "net.cluster2.0.weight" in params
    p = {k: v for k, v in params.items()}
    w = [p.get(k) for k in HEAD]
    head = RH.head_forward(tok, M1, M2 if nonlinear else None, nI * B, *w, rnd=rnd, hid=hid if nonlinear else None)
    D = w[0].shape[0]
    cst = head["code"] if code is None else code[:, :D].double()
    nchw = lambda t, C: t.reshape(nI * B, fh, fw, C).permute(0, 3, 1, 2)
    feats, code4 = nchw(tok, E), nchw(cst, D)
    lc = loss_cfg(cfg)
    if label_pos is not None:  # the one-hot teacher, not Dropout2d-scaled (its M3 is drawn and scales nothing)
        from stego_b200.corr import teacher_width
        wt = teacher_width(n_classes + 1)
        t1, t2 = one_hot_teacher(label, n_classes, wt), one_hot_teacher(label_pos, n_classes, wt)
        corr = RC.CorrRef(t1.to(tok.device), t2.to(tok.device), code4[:B], code4[B:2 * B], coords1, coords2, perms, lc,
                          raw_perms=True, vec8=False, hi=hi)
    else:
        m3 = (M3[:B], M3[B:2 * B]) if M3 is not None else (None, None)
        corr = RC.CorrRef(feats[:B], feats[B:2 * B], code4[:B], code4[B:2 * B], coords1, coords2, perms, lc, m3[0],
                          m3[1], raw_perms=True, vec8=vec8, hi=hi)
    stats = corr.forward()
    cw = call_weights(cfg)
    hist, visit = None, None
    if hist_edges is not None:
        hist, visit = cd_histograms(corr, hist_edges.to(tok.device))
    (dc, Edc), (dcp, Edcp) = corr.backward(cw, visit=visit)
    parts, bars = [dc, dcp], [Edc, Edcp]
    a = None
    if aug is not None:
        a = aug_term(code4[:B], code4[2 * B:], aug["coord"], float(aug["w"]), aug.get("grid"), aug.get("dsampled"))
        parts = [dc + a["dcode_img"], dcp, a["dcode_aug"]]
        bars.append(torch.zeros_like(a["dcode_aug"]))
    dcode = torch.cat(parts).permute(0, 2, 3, 1).reshape(nI * B * hw, D)
    # the bf16 operand copies of the weights the kernels read (the exact weights with rnd=False)
    wb = None
    if nonlinear:
        wb = p["net.cluster2.2.weight"].detach().double().reshape(D, E)
        wb = RH.bf16(wb) if rnd else wb
    hb = RH.head_backward(dcode, head["x1"], head.get("x2"), head.get("hid"), wb, d=D, rnd=rnd)
    x = code4[:B]
    lin = RP.linear_ce_ref(x, p["linear_probe.weight"], p["linear_probe.bias"], label, n_classes)
    clu = RP.cluster_ref(x.reshape(B, D, hw), p["cluster_probe.clusters"], None)
    n_neg = len(stats) - 2
    losses = dict(pos_intra=stats[0]["loss"], pos_inter=stats[1]["loss"],
                  neg_inter=sum(s["loss"] for s in stats[2:]) / n_neg, cd_intra=stats[0]["cd_mean"],
                  cd_inter=stats[1]["cd_mean"], cd_neg=sum(s["cd_mean"] for s in stats[2:]) / n_neg,
                  linear=float(lin["loss"]), cluster=float(clu["loss"]))
    losses["corr"] = sum(c * s["loss"] for c, s in zip(cw, stats))
    losses["total"] = losses["corr"] + losses["linear"] + losses["cluster"]
    if a is not None:
        losses["aug_alignment"] = a["loss"]
        losses["total"] += float(aug["w"]) * a["loss"]
    shape = lambda k: params[k].shape
    grads = {"net.cluster1.0.weight": hb["dw1"].reshape(shape("net.cluster1.0.weight")),
             "net.cluster1.0.bias": hb["db"][:D],
             "linear_probe.weight": lin["dW"].reshape(shape("linear_probe.weight")), "linear_probe.bias": lin["db"],
             "cluster_probe.clusters": clu["dcl"]}
    if nonlinear:
        grads.update({"net.cluster2.0.weight": hb["dwa"].reshape(shape("net.cluster2.0.weight")),
                      "net.cluster2.0.bias": hb["dba"],
                      "net.cluster2.2.weight": hb["dwb"].reshape(shape("net.cluster2.2.weight")),
                      "net.cluster2.2.bias": hb["db"][:D]})
    return dict(head=head, corr=corr, stats=stats, dcode=dcode, dcode_bar=torch.cat(bars).permute(0, 2, 3, 1)
                .reshape(nI * B * hw, D), lin=lin, clu=clu, hb=hb, aug=a, hist=hist, losses=losses, grads=grads, D=D)
