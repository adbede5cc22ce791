"""The training-step configurations the hand-scheduled step accepts beyond the shipped one, their model and batch
builders, and the float64 composition of one training step from the existing references, shared by
tests/test_step_configs_fp64_gpu.py and tests/test_step_fp64_reference.py.

The composition chains the stage references: _head_fp64.head_forward (cluster1 + cluster2, or cluster1 alone for the
linear head), _corr_fp64.CorrRef (the correspondence loss on the returned features, Dropout2d-scaled by the third noise
when cfg.dropout), _probes_fp64.linear_ce_ref and cluster_ref on the detached code of img, and _head_fp64.head_backward
of the correspondence loss's d(code).  Plain torch and device-agnostic: the GPU test feeds it the step's own tensors,
the CPU test pins it to float64 autograd through a restatement of DinoFeaturizer.forward and training_step.
"""
import os
import sys

import torch

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

HEAD = ["net.cluster1.0.weight", "net.cluster1.0.bias", "net.cluster2.0.weight", "net.cluster2.0.bias",
        "net.cluster2.2.weight", "net.cluster2.2.bias"]
PROBES = ["linear_probe.weight", "linear_probe.bias", "cluster_probe.clusters"]


def make_model(row, dev, fused=True, seed=0):
    from _parity_util import make_model as mk
    model, _ = mk(row["arch"], dev, fused=fused, seed=seed, n_classes=row["n_classes"], patch=row["patch"],
                  **row["cfg"])
    return model


def make_batch(row, dev, seed=1):
    """img, img_pos (img + 0.3 noise) and labels in [-1, n_classes] (both ends ignored) at the row's sizes"""
    B, (H, W), n = row["B"], row["frame"], row["n_classes"]
    LH, LW = row["label"] or row["frame"]
    g = torch.Generator().manual_seed(seed)
    img = torch.randn(B, 3, H, W, generator=g)
    img_pos = img + 0.3 * torch.randn(B, 3, H, W, generator=g)
    label = torch.randint(-1, n + 1, (B, LH, LW), generator=g)
    return dict(img=img.to(dev), img_pos=img_pos.to(dev), label=label.to(dev))


def names_of(model):
    """the trainable parameters of the step, in NAMES order (the linear head has no cluster2)"""
    have = dict(model.named_parameters())
    return [k for k in HEAD + PROBES if k in have]


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


def compose(tok, B, fh, fw, M1, M2, M3, coords1, coords2, perms, params, label, cfg, n_classes, rnd=True, hid=None,
            code=None, hi=RC.HI, vec8=True):
    """One training step in float64 from its inputs.
    tok [2B*hw, E]: backbone tokens of img then img_pos; M1 / M2 / M3 [2B, E]: the Dropout2d noises of the cluster1
    input, the cluster2 input (None: linear head) and the returned features (None: cfg.dropout off); coords [B, fs, fs,
    2] and perms [n_neg, B] (raw randperm draws); params: name -> tensor for names_of(model); label [B, LH, LW].
    rnd: round where the kernels store bf16 (the exact step with rnd=False).  hid / code: the kernel's own hidden
    activation / code storage [2B*hw, >= D] (stage-wise: everything downstream then starts from what the step computed);
    None: the reference's own.  Returns head (head_forward), corr (CorrRef after forward and backward, glosses the call
    weights), dcode [2B*hw, D], lin (linear_ce_ref), clu (cluster_ref), hb (head_backward of dcode), losses (the logged
    terms and the total) and grads (name -> gradient in the parameter's shape)."""
    E = tok.shape[1]
    hw = fh * fw
    nonlinear = M2 is not None or "net.cluster2.0.weight" in params
    p = {k: v for k, v in params.items()}
    w = [p.get(k) for k in HEAD]
    head = RH.head_forward(tok, M1, M2 if nonlinear else None, 2 * B, *w, rnd=rnd, hid=hid if nonlinear else None)
    D = w[0].shape[0]
    cst = head["code"] if code is None else code[:, :D].double()
    nchw = lambda t, C: t.reshape(2 * B, fh, fw, C).permute(0, 3, 1, 2)
    feats, code4 = nchw(tok, E), nchw(cst, D)
    lc = loss_cfg(cfg)
    m3 = (M3[:B], M3[B:]) if M3 is not None else (None, None)
    corr = RC.CorrRef(feats[:B], feats[B:], code4[:B], code4[B:], coords1, coords2, perms, lc, m3[0], m3[1],
                      raw_perms=True, vec8=vec8, hi=hi)
    stats = corr.forward()
    cw = call_weights(cfg)
    (dc, Edc), (dcp, Edcp) = corr.backward(cw)
    dcode = torch.cat([dc, dcp]).permute(0, 2, 3, 1).reshape(2 * B * hw, D)
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
    return dict(head=head, corr=corr, stats=stats, dcode=dcode, dcode_bar=torch.cat([Edc, Edcp]).permute(0, 2, 3, 1)
                .reshape(2 * B * hw, D), lin=lin, clu=clu, hb=hb, losses=losses, grads=grads, D=D)
