"""The float64 training-step composition of tests/_step_fp64.py, pinned on the CPU to float64 autograd through a plain
restatement of the reference's DinoFeaturizer.forward (src/modules.py:108-118: cluster1 on Dropout2d(image_feat), plus
cluster2 on a second Dropout2d(image_feat) for the nonlinear head; the returned features Dropout2d-ed only when
cfg.dropout) and of the loss assembly of training_step (train_segmentation.py:130-225, the oracle's
correlation_loss / linear_probe_loss / cluster_lookup), for the linear head, dropout off, continuous=False (D =
n_classes), extra clusters and feature_samples 16 / 28, and through oracle/true_labels_oracle.py (use_true_labels), a
restatement of the aug-alignment term (train_segmentation.py:189-199) and np.histogram of the oracle's cd (the cd
histograms).  Exact arithmetic on both sides (rnd=False, the clamp bound 0.8 in float64, dyadic
coordinates so that the kernels' fp32 tap arithmetic is exact): losses and every gradient agree to 1e-9 relative."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _step_fp64 as S  # noqa: E402
import stego_oracle as O  # noqa: E402

# (n_classes, dim or None for continuous=False, nonlinear, dropout, extra_clusters, cfg overrides)
CASES = {
    "shipped": (27, 70, True, True, 0, {}),
    "linear_head": (27, 70, False, True, 0, {}),
    "no_dropout": (27, 70, True, False, 0, {}),
    "linear_no_dropout": (5, 9, False, False, 0, {}),
    "potsdam_discrete": (3, None, True, True, 0, {}),
    "extra_clusters": (6, 11, True, True, 5, {}),
    "stabalize_no_pointwise": (4, 7, True, True, 2, dict(zero_clamp=False, stabalize=True, pointwise=False)),
    "fs16": (27, 70, True, True, 0, dict(feature_samples=16)),        # S = 256: the multi-tile layout
    "fs28": (5, 9, False, False, 0, dict(feature_samples=28, neg_samples=2)),
}


def featurizer(f, params, m1, m2, m3, nonlinear, dropout):
    """DinoFeaturizer.forward after the backbone (modules.py:108-118) with the Dropout2d noises given"""
    code = F.conv2d(f * m1, params["net.cluster1.0.weight"], params["net.cluster1.0.bias"])
    if nonlinear:
        h = torch.relu(F.conv2d(f * m2, params["net.cluster2.0.weight"], params["net.cluster2.0.bias"]))
        code = code + F.conv2d(h, params["net.cluster2.2.weight"], params["net.cluster2.2.bias"])
    return (f * m3 if dropout else f), code


def reference_step(f, f_pos, params, masks, masks_pos, c1, c2, perms, label, cfg, n_classes, nonlinear, dropout):
    """training_step's loss assembly (train_segmentation.py:130-225) on the restated featurizer"""
    feats, code = featurizer(f, params, *masks, nonlinear, dropout)
    feats_pos, code_pos = featurizer(f_pos, params, *masks_pos, nonlinear, dropout)
    lc = S.loss_cfg(cfg)
    intra, cd_i, inter, cd_p, neg, cd_n = O.correlation_loss(feats, feats_pos, code, code_pos, c1, c2, perms, lc)
    corr = (cfg.pos_inter_weight * inter + cfg.pos_intra_weight * intra + cfg.neg_inter_weight * neg.mean()) * \
        cfg.correspondence_weight
    detached = code.detach().clone()
    lin = O.linear_probe_loss(detached, params["linear_probe.weight"], params["linear_probe.bias"], label, n_classes)
    clu, _ = O.cluster_lookup(detached, params["cluster_probe.clusters"], None)
    return dict(total=corr + lin + clu, corr=corr, linear=lin, cluster=clu, pos_intra=intra, pos_inter=inter,
                neg_inter=neg.mean(), cd_intra=cd_i.mean(), cd_inter=cd_p.mean(), cd_neg=cd_n.mean(), code=code,
                cds=(cd_i, cd_p, cd_n))


def _params(n_classes, D, E, nonlinear, n_clu, g):
    u = lambda *s: (torch.rand(*s, generator=g, dtype=torch.float64) * 2 - 1) / E ** 0.5
    p = {"net.cluster1.0.weight": u(D, E, 1, 1), "net.cluster1.0.bias": u(D)}
    if nonlinear:
        p.update({"net.cluster2.0.weight": u(E, E, 1, 1), "net.cluster2.0.bias": u(E),
                  "net.cluster2.2.weight": u(D, E, 1, 1), "net.cluster2.2.bias": u(D)})
    p.update({"linear_probe.weight": u(n_classes, D, 1, 1) * 8, "linear_probe.bias": u(n_classes),
              "cluster_probe.clusters": torch.randn(n_clu, D, generator=g, dtype=torch.float64)})
    return p


@pytest.mark.parametrize("case", list(CASES))
def test_composition_matches_fp64_autograd(case):
    from stego_b200.config import make_cfg
    n, dim, nonlinear, dropout, extra, over = CASES[case]
    cfg = make_cfg(continuous=dim is not None, dim=dim or 70, dropout=dropout, extra_clusters=extra,
                   projection_type="nonlinear" if nonlinear else "linear", **dict(dict(feature_samples=4, neg_samples=3),
                                                                                   **over))
    D = dim if dim is not None else n
    B, E, fh, fw, LH, LW = 3, 64, 5, 6, 9, 13
    g = torch.Generator().manual_seed(len(case))
    params = _params(n, D, E, nonlinear, n + extra, g)
    tok = torch.randn(2 * B * fh * fw, E, generator=g, dtype=torch.float64)
    keep = lambda: (torch.rand(2 * B, E, generator=g) > 0.1).double() / 0.9
    M1, M2, M3 = keep(), keep() if nonlinear else None, keep() if dropout else None
    fs = cfg.feature_samples
    coords = [torch.randint(-20, 21, (B, fs, fs, 2), generator=g).double() / 16 for _ in range(2)]
    perms = torch.stack([torch.randperm(B, generator=g) for _ in range(cfg.neg_samples)])
    perms[0] = torch.arange(B)  # fixed points: super_perm's fix-up
    label = torch.randint(-1, n + 1, (B, LH, LW), generator=g)

    got = S.compose(tok, B, fh, fw, M1, M2, M3, coords[0], coords[1], perms, params, label, cfg, n, rnd=False, hi=0.8,
                    vec8=False)
    leaves = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    nchw = tok.view(2 * B, fh, fw, E).permute(0, 3, 1, 2)
    m4 = lambda m, sl: m[sl].view(B, E, 1, 1) if m is not None else 1.0
    half = (slice(0, B), slice(B, 2 * B))
    masks = [tuple(m4(m, sl) for m in (M1, M2, M3)) for sl in half]
    resolved = [O.super_perm_from_randperm(p) for p in perms]
    want = reference_step(nchw[:B], nchw[B:], leaves, masks[0], masks[1], coords[0], coords[1], resolved, label, cfg, n,
                          nonlinear, dropout)
    want["total"].backward()
    for k in ("pos_intra", "pos_inter", "neg_inter", "cd_intra", "cd_inter", "cd_neg", "linear", "cluster", "total"):
        w = want[k].item()
        assert abs(got["losses"][k] - w) <= 1e-9 * abs(w) + 1e-15, (case, k, got["losses"][k], w)
    assert set(got["grads"]) == set(params)
    for k, v in leaves.items():
        gr = got["grads"][k]
        assert gr.shape == v.shape, (case, k)
        scale = v.grad.abs().max().item()
        assert scale > 0, (case, k)
        assert (gr - v.grad).abs().max().item() <= 1e-9 * scale, (case, k, (gr - v.grad).abs().max().item(), scale)
    assert got["D"] == D


def test_rows_name_what_they_change():
    """every row builds a configuration the step accepts: code width, classes and cluster rows inside the limits"""
    for name, row in S.CONFIGS.items():
        c = row["cfg"]
        D = row["n_classes"] if c.get("continuous", True) is False else c.get("dim", 70)
        assert 1 <= D <= 96 and row["n_classes"] <= 32 and row["n_classes"] + c.get("extra_clusters", 0) <= 64, name
        assert 1 <= c.get("neg_samples", 5) <= 14, name
        assert row["frame"][0] % row["patch"] == 0 and row["frame"][1] % row["patch"] == 0, name
    assert S.CONFIGS["extra5"]["n_classes"] + 5 == 32 and S.CONFIGS["extra6"]["n_classes"] + 6 == 33
    for name, row in S.MODE_CONFIGS.items():
        c = row["cfg"]
        D = row["n_classes"] if c.get("continuous", True) is False else c.get("dim", 70)
        assert 1 <= D <= 96 and row["n_classes"] <= 32 and 1 <= c.get("neg_samples", 5) <= 14, name
        assert 1 <= c.get("feature_samples", 11) <= 64, name
        assert (row["masks"] is not None) == bool(c.get("use_salience")), name
        if c.get("aug_alignment_weight", 0) > 0:  # the step builds the views of square frames at cfg.res
            assert row["frame"][0] == row["frame"][1], name
    every = S.MODE_CONFIGS["everything"]
    assert every["hist"] and every["cfg"]["feature_samples"] == 16 and all(
        every["cfg"].get(k) for k in ("use_true_labels", "use_salience", "aug_alignment_weight"))


@pytest.mark.parametrize("over,n_classes,limit", [(dict(dim=97), 27, "96"), ({}, 33, "32"), (dict(continuous=False), 33, "32"),
                                                  (dict(extra_clusters=38), 27, "64"), (dict(neg_samples=15), 27, "14"),
                                                  (dict(dim=0), 27, "96")])
def test_limits_refused_at_construction(over, n_classes, limit):
    """Configurations just outside what the kernels take fail when the model is built, naming the limit, before the
    construction draws anything from the generators (so nothing of a training step has run either)."""
    from stego_b200.config import make_cfg
    from stego_b200.segmenter import LitUnsupervisedSegmenter
    cfg = make_cfg(random_backbone_init=True, **over)
    st = torch.get_rng_state()
    with pytest.raises(RuntimeError, match=limit):
        LitUnsupervisedSegmenter(n_classes, cfg)
    assert torch.equal(torch.get_rng_state(), st)


def _inputs(n, D, nonlinear, dropout, extra, cfg, seed, n_img=2, LH=9, LW=13, label_hi=None):
    """the inputs of one small step: B = 3, E = 64, 5 x 6 features (n_img images of each), dyadic coordinates"""
    B, E, fh, fw = 3, 64, 5, 6
    g = torch.Generator().manual_seed(seed)
    params = _params(n, D, E, nonlinear, n + extra, g)
    tok = torch.randn(n_img * B * fh * fw, E, generator=g, dtype=torch.float64)
    keep = lambda: (torch.rand(n_img * B, E, generator=g) > 0.1).double() / 0.9
    M1, M2, M3 = keep(), keep() if nonlinear else None, keep() if dropout else None
    fs = cfg.feature_samples
    coords = [torch.randint(-20, 21, (B, fs, fs, 2), generator=g).double() / 16 for _ in range(2)]
    perms = torch.stack([torch.randperm(B, generator=g) for _ in range(cfg.neg_samples)])
    perms[0] = torch.arange(B)
    label = torch.randint(-1, n + 1 if label_hi is None else label_hi, (B, LH, LW), generator=g)
    return dict(B=B, E=E, fh=fh, fw=fw, g=g, params=params, tok=tok, M=(M1, M2, M3), coords=coords, perms=perms,
                label=label)


def _masks4(x, B, E, n_img):
    m4 = lambda m, sl: m[sl].view(B, E, 1, 1) if m is not None else 1.0
    return [tuple(m4(m, slice(i * B, (i + 1) * B)) for m in x["M"]) for i in range(n_img)]


def _agree(case, got, want, leaves, keys):
    for k in keys:
        w = want[k].item()
        assert abs(got["losses"][k] - w) <= 1e-9 * abs(w) + 1e-15, (case, k, got["losses"][k], w)
    assert set(got["grads"]) == set(leaves)
    for k, v in leaves.items():
        gr = got["grads"][k]
        assert gr.shape == v.shape, (case, k)
        scale = v.grad.abs().max().item()
        assert scale > 0, (case, k)
        assert (gr - v.grad).abs().max().item() <= 1e-9 * scale, (case, k, (gr - v.grad).abs().max().item(), scale)


LOSS_KEYS = ("pos_intra", "pos_inter", "neg_inter", "cd_intra", "cd_inter", "cd_neg", "linear", "cluster", "total")


@pytest.mark.parametrize("fs", [4, 12])
def test_true_labels_composition_matches_oracle(fs, monkeypatch):
    """use_true_labels: the teacher is one_hot_feats(label + 1, n + 1) at label resolution (9 x 13 labels on 5 x 6
    features), not Dropout2d-scaled; against oracle/true_labels_oracle.training_losses in float64."""
    import true_labels_oracle as TL
    from stego_b200.config import make_cfg
    n, D = 6, 10
    cfg = make_cfg(dim=D, use_true_labels=True, feature_samples=fs, neg_samples=3)
    x = _inputs(n, D, True, True, 0, cfg, seed=11 + fs, label_hi=n)  # F.one_hot raises on n
    B, E, fh, fw = x["B"], x["E"], x["fh"], x["fw"]
    label_pos = torch.randint(-1, n, (B, 9, 13), generator=x["g"])
    got = S.compose(x["tok"], B, fh, fw, *x["M"], *x["coords"], x["perms"], x["params"], x["label"], cfg, n,
                    rnd=False, hi=0.8, vec8=False, label_pos=label_pos)
    orig = TL.one_hot_feats
    monkeypatch.setattr(TL, "one_hot_feats", lambda lab, c: orig(lab, c).double())
    leaves = {k: v.clone().requires_grad_(True) for k, v in x["params"].items()}
    hp = {k[len("net."):]: v for k, v in leaves.items() if k.startswith("net.")}
    probes = {k: v for k, v in leaves.items() if not k.startswith("net.")}
    nchw = x["tok"].view(2 * B, fh, fw, E).permute(0, 3, 1, 2)
    masks = _masks4(x, B, E, 2)
    resolved = [O.super_perm_from_randperm(p) for p in x["perms"]]
    want = TL.training_losses(nchw[:B], nchw[B:], hp, probes, x["label"], label_pos, masks[0], masks[1], *x["coords"],
                              resolved, S.loss_cfg(cfg), n)
    want["total"].backward()
    _agree(f"tl_fs{fs}", got, want, leaves, LOSS_KEYS)
    # the teacher: n + 1 classes zero-padded to the tile width; out-of-range labels (n, 255, -7) are class 0
    lab = torch.tensor([[[-1, 0, n - 1, n, 255, -7]]])
    oh = S.one_hot_teacher(lab, n, 64)
    assert oh.shape == (1, 64, 1, 6) and oh[:, n + 1:].abs().sum() == 0
    assert oh[0, :, 0].argmax(0).tolist() == [0, 1, n, 0, 0, 0]


@pytest.mark.parametrize("case", ["shipped", "linear_no_dropout"])
def test_aug_composition_matches_restatement(case):
    """The aug-alignment term (train_segmentation.py:189-199) on the restated featurizer of net(img_aug): the head over
    3B rows (the img_aug rows use their M1 / M2, not M3), the cosine's d(code) into the img rows through grid_sample and
    into the img_aug rows, loss/total with w * aug."""
    from stego_b200.config import make_cfg
    n, D, nonlinear, dropout = 5, 9, case == "shipped", case == "shipped"
    cfg = make_cfg(dim=D, dropout=dropout, projection_type="nonlinear" if nonlinear else "linear",
                   aug_alignment_weight=0.6, feature_samples=4, neg_samples=3)
    x = _inputs(n, D, nonlinear, dropout, 0, cfg, seed=23, n_img=3)
    B, E, fh, fw = x["B"], x["E"], x["fh"], x["fw"]
    fw = fh  # square frames
    x["tok"] = x["tok"].view(3 * B, 5, 6, E)[:, :, :5].reshape(-1, E).contiguous()
    res = 20
    coord = (torch.randint(-24, 25, (B, res, res, 2), generator=x["g"]).double() / 16)
    got = S.compose(x["tok"], B, fh, fw, *x["M"], *x["coords"], x["perms"], x["params"], x["label"][..., :7, :7], cfg,
                    n, rnd=False, hi=0.8, vec8=False, aug=dict(coord=coord, w=0.6))
    leaves = {k: v.clone().requires_grad_(True) for k, v in x["params"].items()}
    nchw = x["tok"].view(3 * B, fh, fw, E).permute(0, 3, 1, 2)
    masks = _masks4(x, B, E, 3)
    resolved = [O.super_perm_from_randperm(p) for p in x["perms"]]
    want = reference_step(nchw[:B], nchw[B:2 * B], leaves, masks[0], masks[1], *x["coords"], resolved,
                          x["label"][..., :7, :7], cfg, n, nonlinear, dropout)
    _, code_aug = featurizer(nchw[2 * B:], leaves, *masks[2], nonlinear, dropout)
    down = F.interpolate(coord.permute(0, 3, 1, 2), code_aug.shape[2], mode="bilinear",
                         align_corners=False).permute(0, 2, 3, 1)
    sampled = F.grid_sample(want["code"], down.permute(0, 2, 1, 3), padding_mode="border", align_corners=True)
    norm = lambda t: F.normalize(t, dim=1, eps=1e-10)
    aug = -torch.einsum("bkhw,bkhw->bhw", norm(sampled), norm(code_aug)).mean()
    want["aug_alignment"] = aug
    want["total"] = want["total"] + 0.6 * aug
    want["total"].backward()
    _agree(f"aug_{case}", got, want, leaves, LOSS_KEYS + ("aug_alignment",))
    a = got["aug"]
    assert (a["grid"] - down).abs().max().item() == 0.0
    assert (a["sampled"] - sampled.detach()).abs().max().item() <= 1e-12 * sampled.abs().max().item()


def test_cd_histograms_of_an_exact_case():
    """compose's cd histograms (hist.default_bins(), np.histogram's bucket rule) equal np.histogram of the oracle's cd
    for each loss group, and its bin brackets hold them."""
    from stego_b200 import hist
    from stego_b200.config import make_cfg
    n, D = 5, 9
    cfg = make_cfg(dim=D, feature_samples=6, neg_samples=3)
    x = _inputs(n, D, True, True, 0, cfg, seed=31)
    B, E, fh, fw = x["B"], x["E"], x["fh"], x["fw"]
    edges = torch.from_numpy(hist.default_bins().copy())
    got = S.compose(x["tok"], B, fh, fw, *x["M"], *x["coords"], x["perms"], x["params"], x["label"], cfg, n,
                    rnd=False, hi=0.8, vec8=False, hist_edges=edges)
    nchw = x["tok"].view(2 * B, fh, fw, E).permute(0, 3, 1, 2)
    masks = _masks4(x, B, E, 2)
    resolved = [O.super_perm_from_randperm(p) for p in x["perms"]]
    want = reference_step(nchw[:B], nchw[B:], x["params"], masks[0], masks[1], *x["coords"], resolved, x["label"], cfg,
                          n, True, True)
    assert len(got["hist"]) == 3
    for h, cd in zip(got["hist"], want["cds"]):
        v = cd.detach().reshape(-1).numpy()
        counts, _ = np.histogram(v, bins=hist.default_bins())
        assert np.array_equal(h["counts"].numpy(), counts)
        assert h["num"] == v.size and int(h["counts"].sum()) == v.size
        cum = np.cumsum(counts)
        assert (np.cumsum(h["hi"].numpy()) <= cum).all() and (cum <= np.cumsum(h["lo"].numpy())).all()
        assert abs(h["min"] - v.min()) <= 1e-12 and abs(h["max"] - v.max()) <= 1e-12
        assert abs(h["sum"] - v.sum()) <= 1e-12 * np.abs(v).sum()
        assert abs(h["sumsq"] - v.dot(v)) <= 1e-12 * v.dot(v)
    assert sum(int(c.sum()) for c in (h["counts"] for h in got["hist"])) == (2 + cfg.neg_samples) * B * 36 ** 2
