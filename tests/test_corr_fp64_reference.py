"""The fp64 correspondence-loss references of tests/_corr_fp64.py, pinned on the CPU: to the oracle
(oracle/stego_oracle.py: bilinear_sample, corr_helper, correlation_loss) within 1e-12 with fp64 inputs and dyadic
coordinates (where fp32 and fp64 coordinate arithmetic agree exactly), the analytic backward to fp64 autograd through
the oracle in every cfg branch and with upstream weights on the loss elements and on cd, and every input builder to
what it claims to make."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _corr_fp64 as R  # noqa: E402
import stego_oracle as O  # noqa: E402  (oracle/ is on sys.path through _corr_fp64)

BRANCHES = {"default": {}, "no_pointwise": dict(pointwise=False), "no_zero_clamp_stabalize": dict(zero_clamp=False,
            stabalize=True), "stabalize": dict(stabalize=True)}


def _inputs(B, E, D, H, W, fs, n_neg, seed):
    g = torch.Generator().manual_seed(seed)
    d = R.make_inputs("corr", B, E, D, H, W, fs, n_neg, seed=seed)
    for k in ("coords1", "coords2"):  # dyadic, some beyond +-1
        d[k] = torch.randint(-20, 21, d[k].shape, generator=g).float() / 16
    return d


def _oracle_calls(d, cfg, raw):
    """per call (loss elements, cd) of the oracle in fp64, chan_scale applied to the features before sampling"""
    f64 = lambda t: t.double()
    feats, feats_pos = f64(d["feats"]), f64(d["feats_pos"])
    if d["chan_scale"] is not None:
        feats = feats * f64(d["chan_scale"])[:, :, None, None]
        feats_pos = feats_pos * f64(d["chan_scale_pos"])[:, :, None, None]
    c1, c2 = f64(d["coords1"]), f64(d["coords2"])
    code, code_pos = d["code64"], d["code_pos64"]
    f, c = O.bilinear_sample(feats, c1), O.bilinear_sample(code, c1)
    fp, cp = O.bilinear_sample(feats_pos, c2), O.bilinear_sample(code_pos, c2)
    out = [O.corr_helper(f, f, c, c, cfg.pos_intra_shift, cfg), O.corr_helper(f, fp, c, cp, cfg.pos_inter_shift, cfg)]
    if cfg.neg_samples:
        perms = R.resolve_perms(d["perms"], feats.shape[0], raw)
        for p in perms:
            out.append(O.corr_helper(f, O.bilinear_sample(feats[p], c2), c, O.bilinear_sample(code[p], c2),
                                     cfg.neg_inter_shift, cfg))
    return out


@pytest.mark.parametrize("branch", list(BRANCHES))
@pytest.mark.parametrize("fs,n_neg,raw", [(3, 2, False), (4, 0, False), (3, 3, True)])
def test_reference_matches_oracle_and_autograd(branch, fs, n_neg, raw):
    B, E, D, H, W = 3, 64, 7, 5, 9
    cfg = O.LossCfg(feature_samples=fs, neg_samples=n_neg, **BRANCHES[branch])
    d = _inputs(B, E, D, H, W, fs, n_neg, seed=fs * 10 + n_neg)
    if raw:
        d["perms"][0] = torch.arange(B)  # fixed points
    d["code64"] = d["code"].double().requires_grad_(True)
    d["code_pos64"] = d["code_pos"].double().requires_grad_(True)
    calls = _oracle_calls(d, cfg, raw)
    ref = R.CorrRef(d["feats"].double(), d["feats_pos"].double(), d["code"].double(), d["code_pos"].double(),
                    d["coords1"], d["coords2"], d["perms"], cfg, d["chan_scale"], d["chan_scale_pos"], raw_perms=raw,
                    hi=0.8)
    stats = ref.forward()
    S, nc = fs * fs, 2 + n_neg
    g = torch.Generator().manual_seed(7)
    gl = torch.randn(nc, generator=g, dtype=torch.float64)
    gelem = torch.randn(nc, B, S, S, generator=g, dtype=torch.float64)
    gcd = torch.randn(nc, B, S, S, generator=g, dtype=torch.float64) * 0.1
    for k, (el, cd) in enumerate(calls):
        assert abs(stats[k]["loss"] - el.mean().item()) < 1e-12
        assert abs(stats[k]["cd_mean"] - cd.mean().item()) < 1e-12

    def visit(k, b, x):
        el, cd = calls[k]
        assert (x["cd"] - cd[b].detach().reshape(S, S)).abs().max() < 1e-12
        assert (x["elem"] - el[b].detach().reshape(S, S)).abs().max() < 1e-12

    (dc, _), (dcp, _) = ref.backward(gl, gelem, gcd, visit=visit)
    obj = sum(gl[k] * el.mean() + (gelem[k] * el.reshape(B, S, S)).sum() + (gcd[k] * cd.reshape(B, S, S)).sum()
              for k, (el, cd) in enumerate(calls))
    ga, gpa = torch.autograd.grad(obj, [d["code64"], d["code_pos64"]])
    scale = max(ga.abs().max().item(), gpa.abs().max().item())
    assert (dc - ga).abs().max().item() < 1e-12 * scale
    assert (dcp - gpa).abs().max().item() < 1e-12 * scale


def test_oracle_pin_of_the_sampler():
    """taps + gather at dyadic coordinates, including beyond +-1 and exactly on the last row / column"""
    g = torch.Generator().manual_seed(3)
    src = torch.randn(2, 5, 4, 7, generator=g, dtype=torch.float64)
    coords = torch.randint(-20, 21, (2, 6, 6, 2), generator=g).double() / 16
    coords[:, 0, :, :] = 1.0
    idx, w = R.taps(coords, 4, 7)
    v, _ = R.gather_sample(src, torch.arange(2), idx, w)
    want = O.bilinear_sample(src, coords).reshape(2, 5, 36).transpose(1, 2)
    assert (v - want).abs().max() < 1e-12


def test_builders_make_what_they_claim():
    B, E, D, H, W, fs = 3, 64, 70, 9, 13, 6
    cfg = O.LossCfg(feature_samples=fs, neg_samples=2, stabalize=True)

    def ref_of(d, raw=False):
        return R.CorrRef(d["feats"].double(), d["feats_pos"].double(), d["code"].double(), d["code_pos"].double(),
                         d["coords1"], d["coords2"], d["perms"], cfg, d["chan_scale"], d["chan_scale_pos"], raw_perms=raw)

    # flat: centred fd at most 1e-3 of fd, and fd ~ 1
    d = R.make_inputs("flat", B, E, D, H, W, fs, 2, seed=1)
    r = ref_of(d)
    for k in range(r.ncalls):
        x = r.block(k, 0)
        assert x["fdc"].abs().max() <= 1e-3 * x["fd"].abs().min() and x["fd"].min() > 0.9
    # kinks: bilinear weights all 0 / 1, cd exactly 0 and exactly 1, and within fp32 rounding of 0.8
    d = R.make_inputs("kinks", B, E, D, H, W, fs, 2, seed=2)
    for c in (d["coords1"], d["coords2"]):
        _, w = R.taps(c, H, W)
        assert ((w == 0) | (w == 1)).all()
    r = ref_of(d)
    cds = torch.cat([r.block(k, b)["cd"].reshape(-1) for k in range(r.ncalls) for b in range(B)])
    assert (cds == 0).sum() > 100 and (cds == 1).sum() > 100
    assert ((cds - R.HI).abs() < 1e-7).sum() > 10
    for s in range(r.nslots):  # the normalised codes are bf16-exact: hi carries them, lo is zero
        n = r.cn[s]
        assert torch.equal(n.float().bfloat16().double(), n) or ((n - R.HI).abs() < 1e-7).any()
    # border: clamped taps exist, and their weight is exactly 0 even before make_taps zeroes it (x = W - 1 there);
    # a quarter of an image's samples on one pixel
    d = R.make_inputs("border", B, E, D, H, W, fs, 2, seed=3)
    for c in (d["coords1"], d["coords2"]):
        cc = c.float().permute(0, 2, 1, 3).reshape(B, -1, 2)
        x = (((cc[..., 0] + 1.0) / 2.0) * float(W - 1)).clamp(0, W - 1)
        y = (((cc[..., 1] + 1.0) / 2.0) * float(H - 1)).clamp(0, H - 1)
        assert (x == W - 1).sum() > 5 and (y == H - 1).sum() > 5
        assert ((x - x.floor())[x == W - 1] == 0).all() and ((y - y.floor())[y == H - 1] == 0).all()
        assert (cc.abs() > 1).any() and (cc.abs() == 1).any()
    r = ref_of(d)
    gl = torch.ones(r.ncalls, dtype=torch.float64)
    r.forward()
    r.backward(gl)
    assert r.hits[0].max() >= fs * fs // 4
    # zeros: zero-norm code and feature samples; chan_scale zeroes every channel of image 0
    d = R.make_inputs("zeros", B, E, D, H, W, fs, 2, seed=4)
    r = ref_of(d)
    assert (r.cnrm[0] == 0).sum() > 3 and (r.cnrm[1] == 0).sum() > 3
    assert (r.fn[0][0] == 0).all()
    assert (r.fn[1][1].norm(dim=-1) == 0).any() or (r.fn[0][1].norm(dim=-1) == 0).any()
    # tagged: the raw draws of negative 0 are all fixed points; the fix-up picks image b + 1 mod B
    d = R.make_inputs("tagged", B, E, D, H, W, fs, 2, seed=5)
    assert torch.equal(R.resolve_perms(d["perms"], B, True)[0], (torch.arange(B) + 1) % B)
    for k in ("feats", "code"):
        assert (d[k].mean((2, 3))[0] - d[k].mean((2, 3))[1]).abs().mean() > 1.0
