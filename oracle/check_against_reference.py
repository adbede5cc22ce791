"""Pin the oracle: compare oracle/stego_oracle.py function-by-function with the REAL reference code.

    STEGO_REFERENCE_SRC=<reference checkout>/src python oracle/check_against_reference.py

Exit status 0 iff every check passes.  `reference_outputs()` runs the reference on seeded inputs and
`oracle_outputs()` runs the oracle on the same inputs; oracle/make_golden.py stores a fixed sample of the reference
side in tests/golden/reference_pins.pt, so tests/test_oracle_golden.py runs the same comparison without the reference.
"""
from __future__ import annotations

import os
import sys
import types

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import stego_oracle as O  # noqa: E402

LOSS_CFGS = [(True, True, False), (False, True, False), (True, False, True)]
VIT_CASES = [("vit_small", 224), ("vit_small", 96), ("vit_base", 64)]
LOSS_NAMES = ["intra", "intra_cd", "inter", "inter_cd", "neg", "neg_cd"]


def _cfg_ns(cfg: O.LossCfg):
    return types.SimpleNamespace(**cfg.__dict__)


# ---- seeded inputs shared by both sides --------------------------------------------------------------
def _sample_inputs():
    torch.manual_seed(0)
    t = torch.randn(3, 20, 9, 13)
    coords = torch.rand(3, 5, 7, 2) * 2.4 - 1.2  # includes out-of-range coords (border clamp)
    a, b = torch.randn(2, 16, 5, 5), torch.randn(2, 16, 4, 6)
    corner = torch.tensor([[[[-1., -1.], [1., -1.]], [[-1., 1.], [1., 1.]]]]).repeat(3, 1, 1, 1)
    return t, coords, a, b, corner


def _loss_inputs():
    torch.manual_seed(7)
    B, E, D, h = 3, 48, 70, 14
    feats, feats_pos = torch.randn(B, E, h, h), torch.randn(B, E, h, h)
    code = torch.randn(B, D, h, h, requires_grad=True)
    code_pos = torch.randn(B, D, h, h, requires_grad=True)
    return feats, feats_pos, code, code_pos


def _head_inputs():
    torch.manual_seed(5)
    E, D, B, h = 384, 70, 2, 6
    return O.head_random_state(E, D, seed=4), torch.randn(B, E, h, h)


def _crf_inputs():
    torch.manual_seed(31)
    gd = torch.rand(2, 3, 20, 24)
    cl = torch.nn.functional.normalize(torch.randn(2, 70, 20, 24), dim=1).requires_grad_(True)
    return gd, cl


def reference_outputs(ref, vits) -> dict:
    """Every value the checks compare, computed by the reference (`ref` = src/modules.py, `vits` =
    src/dino/vision_transformer.py)."""
    out = {}
    t, coords, a, b, corner = _sample_inputs()
    out["norm"] = ref.norm(t)
    out["tensor_correlation"] = ref.tensor_correlation(a, b)
    out["sample"] = ref.sample(t, coords)
    out["sample_corners"] = ref.sample(t, corner)
    for size in (1, 2, 5, 32):
        torch.manual_seed(123 + size)
        out[f"super_perm_{size}"] = torch.stack([ref.super_perm(size, torch.device("cpu")) for _ in range(4)])
    for pointwise, zero_clamp, stab in LOSS_CFGS:
        cfg = O.LossCfg(pointwise=pointwise, zero_clamp=zero_clamp, stabalize=stab)
        feats, feats_pos, code, code_pos = _loss_inputs()
        torch.manual_seed(99)
        want = ref.ContrastiveCorrelationLoss(_cfg_ns(cfg))(feats, feats_pos, None, None, code, code_pos)
        gw = torch.autograd.grad(O.weighted_correspondence_loss(want, cfg), [code, code_pos])
        tag = f"loss[pw={pointwise},zc={zero_clamp},st={stab}]"
        for i, name in enumerate(LOSS_NAMES):
            out[f"{tag}.{name}"] = want[i].detach()
        out[f"{tag}.dcode"], out[f"{tag}.dcode_pos"] = gw
    torch.manual_seed(7)
    cl = ref.ClusterLookup(70, 27)
    x = torch.randn(2, 70, 28, 28)
    out["ClusterLookup.clusters"] = cl.clusters.detach().clone()
    loss, probs = cl(x, None)
    out["ClusterLookup.loss"] = loss.detach()
    out["ClusterLookup.argmax"] = probs.argmax(1)
    out["ClusterLookup.log_probs(alpha=2)"] = cl(x, 2.0, log_probs=True).detach()
    out["ClusterLookup.softmax(alpha=3)"] = cl(x, 3.0)[1].detach()
    for arch, res in VIT_CASES:
        sd = O.perturb_vit_state(O.vit_random_state(arch, 8, seed=3))
        model = vits.__dict__[arch](patch_size=8, num_classes=0)
        model.load_state_dict(sd, strict=True)
        model.eval()
        torch.manual_seed(11)
        img = torch.randn(1, 3, res, res)
        with torch.no_grad():
            feat, _, _ = model.get_intermediate_feat(img, n=1)
        out[f"ViT {arch}/8 @{res} tokens"] = feat[0]
    # head (DinoFeaturizer.forward tail) with the dropout masks drawn from the same seed
    hp, f = _head_inputs()
    E, D = f.shape[1], 70
    c1 = torch.nn.Sequential(torch.nn.Conv2d(E, D, (1, 1)))
    c2 = torch.nn.Sequential(torch.nn.Conv2d(E, E, (1, 1)), torch.nn.ReLU(), torch.nn.Conv2d(E, D, (1, 1)))
    c1.load_state_dict({k[len("cluster1."):]: v for k, v in hp.items() if k.startswith("cluster1.")})
    c2.load_state_dict({k[len("cluster2."):]: v for k, v in hp.items() if k.startswith("cluster2.")})
    drop = torch.nn.Dropout2d(p=.1)
    torch.manual_seed(21)
    code = c1(drop(f))  # modules.py:109
    code = code + c2(drop(f))  # modules.py:111
    out["head code (dropout masks replayed)"] = code.detach()
    out["head returned feats"] = drop(f)  # modules.py:116
    # ContrastiveCRFLoss (modules.py:437-469), train_config.yml:131-137 parameters
    gd, cl_ = _crf_inputs()
    crf = ref.ContrastiveCRFLoss(200, .5, .15, .05, 10.0, 3.0, 0.00)
    torch.manual_seed(32)
    want = crf(gd, cl_)
    out["ContrastiveCRFLoss d/dclusters"], = torch.autograd.grad(want.mean(), cl_)
    out["ContrastiveCRFLoss"] = want.detach()
    return out


def oracle_outputs(clusters: torch.Tensor) -> dict:
    """The oracle's values for every entry of reference_outputs(); `clusters` are the reference ClusterLookup's
    parameters (its initialisation is the reference's own)."""
    out = {}
    t, coords, a, b, corner = _sample_inputs()
    out["norm"] = O.l2_normalize(t)
    out["tensor_correlation"] = O.correlation(a, b)
    out["sample"] = O.bilinear_sample(t, coords)
    out["sample_corners"] = O.bilinear_sample(t, corner)
    for size in (1, 2, 5, 32):
        torch.manual_seed(123 + size)
        out[f"super_perm_{size}"] = torch.stack([O.super_perm_from_randperm(torch.randperm(size, dtype=torch.long))
                                                 for _ in range(4)])
    for pointwise, zero_clamp, stab in LOSS_CFGS:
        cfg = O.LossCfg(pointwise=pointwise, zero_clamp=zero_clamp, stabalize=stab)
        feats, feats_pos, code, code_pos = _loss_inputs()
        torch.manual_seed(99)
        c1, c2, perms = O.draw_loss_randomness(feats.shape[0], cfg)
        got = O.correlation_loss(feats, feats_pos, code, code_pos, c1, c2, perms, cfg)
        gg = torch.autograd.grad(O.weighted_correspondence_loss(got, cfg), [code, code_pos])
        tag = f"loss[pw={pointwise},zc={zero_clamp},st={stab}]"
        for i, name in enumerate(LOSS_NAMES):
            out[f"{tag}.{name}"] = got[i].detach()
        out[f"{tag}.dcode"], out[f"{tag}.dcode_pos"] = gg
    torch.manual_seed(7)
    torch.randn(27, 70)  # the draw ClusterLookup's constructor makes: x below comes from the same stream position
    x = torch.randn(2, 70, 28, 28)
    loss, probs = O.cluster_lookup(x, clusters, None)
    out["ClusterLookup.loss"] = loss
    out["ClusterLookup.argmax"] = probs.argmax(1)
    out["ClusterLookup.log_probs(alpha=2)"] = O.cluster_lookup(x, clusters, 2.0, log_probs=True)
    out["ClusterLookup.softmax(alpha=3)"] = O.cluster_lookup(x, clusters, 3.0)[1]
    for arch, res in VIT_CASES:
        sd = O.perturb_vit_state(O.vit_random_state(arch, 8, seed=3))
        torch.manual_seed(11)
        img = torch.randn(1, 3, res, res)
        with torch.no_grad():
            out[f"ViT {arch}/8 @{res} tokens"] = O.vit_forward(sd, img, arch, 8)
    hp, f = _head_inputs()
    torch.manual_seed(21)
    masks = [O.draw_dropout2d_mask(f.shape[0], f.shape[1]) for _ in range(3)]
    feat, code = O.head_forward(f, hp, masks)
    out["head code (dropout masks replayed)"] = code.detach()
    out["head returned feats"] = feat.detach()
    gd, cl_ = _crf_inputs()
    torch.manual_seed(32)
    coords = torch.cat([torch.randint(0, 20, size=[1, 200]), torch.randint(0, 24, size=[1, 200])], 0)
    got = O.contrastive_crf_loss(gd, cl_, coords, .5, .15, .05, 10.0, 3.0, 0.00)
    out["ContrastiveCRFLoss d/dclusters"], = torch.autograd.grad(got.mean(), cl_)
    out["ContrastiveCRFLoss"] = got.detach()
    return out


# max|oracle - reference| <= tol * max(max|reference|, 1); None: bit-exact
TOLS = {"norm": 1e-6, "tensor_correlation": 1e-5, "sample": 1e-5, "sample_corners": 1e-6,
        "ClusterLookup.loss": 1e-6, "ClusterLookup.argmax": None, "ClusterLookup.log_probs(alpha=2)": 1e-5,
        "ClusterLookup.softmax(alpha=3)": 1e-6, "head code (dropout masks replayed)": 1e-5, "head returned feats": 1e-6,
        "ContrastiveCRFLoss": 1e-6, "ContrastiveCRFLoss d/dclusters": 1e-6}
TOLS.update({f"super_perm_{s}": None for s in (1, 2, 5, 32)})
for _pw, _zc, _st in LOSS_CFGS:
    _tag = f"loss[pw={_pw},zc={_zc},st={_st}]"
    TOLS.update({f"{_tag}.{n}": 2e-6 for n in LOSS_NAMES})
    TOLS.update({f"{_tag}.dcode": 1e-5, f"{_tag}.dcode_pos": 1e-5})
TOLS.update({f"ViT {a}/8 @{r} tokens": 2e-5 for a, r in VIT_CASES})


def sample_outputs(want: dict, n: int = 2048, seed: int = 0) -> dict:
    """A fixed, seeded sample of every reference value (all of it when small, and always all of the ClusterLookup
    parameters the oracle side needs) with its full-tensor scale."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for k, v in want.items():
        flat = v.detach().reshape(-1)
        idx = torch.arange(flat.numel()) if flat.numel() <= n or k == "ClusterLookup.clusters" else torch.randperm(flat.numel(), generator=g)[:n].sort().values
        scale = flat.abs().max().item() if flat.is_floating_point() else 0.0
        out[k] = dict(shape=tuple(v.shape), idx=idx.to(torch.int32), values=flat[idx].clone(), scale=scale)
    return out


def run_checks(samples: dict) -> bool:
    """Compare the oracle with the (sampled) reference values from sample_outputs()."""
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    got = oracle_outputs(samples["ClusterLookup.clusters"]["values"].reshape(samples["ClusterLookup.clusters"]["shape"]))
    ok = True
    for k, tol in TOLS.items():
        s = samples[k]
        g = got[k].detach()
        good = tuple(g.shape) == tuple(s["shape"])
        if good:
            gs = g.reshape(-1)[s["idx"].long()]
            if tol is None:
                good = torch.equal(gs, s["values"])
                msg = "bit-exact"
            else:
                err = (gs - s["values"]).abs().max().item()
                good = err <= tol * max(s["scale"], 1.0)
                msg = f"max|diff|={err:.3e} (scale {s['scale']:.3e})"
        else:
            msg = f"shape {tuple(g.shape)} != {tuple(s['shape'])}"
        print(f"  {'ok ' if good else 'BAD'} {k}: {msg}")
        ok &= good
    print("ORACLE PINNED AGAINST REFERENCE" if ok else "ORACLE MISMATCH")
    return bool(ok)


if __name__ == "__main__":
    import reference_shim
    ref_, vits_ = reference_shim.import_reference()
    sys.exit(0 if run_checks(sample_outputs(reference_outputs(ref_, vits_), n=1 << 62)) else 1)
