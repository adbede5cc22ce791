"""CPU: the fp64 probe references of tests/_probes_fp64.py against the oracle and autograd, and the input builders
against what they claim to construct (the GPU tests' power rests on both)."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _probes_fp64 as R  # noqa: E402
import stego_oracle as O  # noqa: E402


@pytest.mark.parametrize("h,w,H,W", [(7, 9, 50, 61), (28, 28, 224, 224), (28, 28, 28, 28), (40, 8, 12, 64),
                                     (8, 40, 64, 12), (128, 256, 1024, 1536)])
def test_corners_equal_f_interpolate(h, w, H, W):
    torch.manual_seed(h + W)
    t = torch.randn(3, h, w, dtype=torch.float64)
    want = F.interpolate(t[None], (H, W), mode="bilinear", align_corners=False)[0]
    assert (R.upsample(t, H, W) - want).abs().max().item() <= 1e-12
    cr = R.Corners(h, w, H, W, "cpu", rows=(H // 3, H // 3 + 5))  # a band of rows alone
    assert (cr.interp(t.reshape(3, -1)).view(3, 5, W) - want[:, H // 3:H // 3 + 5]).abs().max().item() <= 1e-12
    # the adjoint is the transpose of the interpolation
    g = torch.randn(3, H * W, dtype=torch.float64)
    tt = t.clone().requires_grad_(True)
    (F.interpolate(tt[None], (H, W), mode="bilinear", align_corners=False)[0].reshape(3, -1) * g).sum().backward()
    adj = R.adjoint_into(torch.zeros(3, h * w, dtype=torch.float64), R.Corners(h, w, H, W, "cpu"), g)
    assert (adj - tt.grad.reshape(3, -1)).abs().max().item() <= 1e-12


def test_lambda_error_of_fp32_weights():
    """0 at power-of-two ratios (every c1-c4 shape); otherwise a few u times the source coordinate"""
    for n_in, n_out in ((28, 224), (40, 320), (56, 448), (128, 1024), (256, 2048), (28, 28)):
        assert R.axis(n_in, n_out)[3].max().item() == 0.0
    e = R.axis(7, 50)[3]
    assert 0 < e.max().item() < 3 * R.U * 7
    assert 0 < R.axis(256, 1536)[3].max().item() < 3 * R.U * 256


def _lookup_loss(x4, c, alpha):
    """src/modules.py:146-161 with F.normalize, whose gradient at an all-zero row is g / eps (the oracle's
    pow-sum-sqrt form is NaN there)"""
    nc, nx = F.normalize(c, dim=1), F.normalize(x4, dim=1)
    ip = torch.einsum("bchw,nc->bnhw", nx, nc)
    if alpha is None:
        probs = F.one_hot(ip.argmax(1), c.shape[0]).permute(0, 3, 1, 2).to(ip.dtype)
    else:
        probs = torch.softmax(alpha * ip, 1)
    return -(probs * ip).sum(1).mean()


@pytest.mark.parametrize("alpha", [None, 2.0, 50.0])
@pytest.mark.parametrize("regime", ["random", "ties", "zeros", "zerorow", "sharp"])
def test_cluster_ref_matches_oracle_and_autograd(regime, alpha):
    x, cl = R.cluster_inputs(regime, 2, 70, 36, 27, seed=3)
    x, cl = x.double(), cl.double()
    ref = R.cluster_ref(x, cl, alpha, grad=0.7)
    x4 = x.view(2, 70, 6, 6)
    loss, probs = O.cluster_lookup(x4, cl, alpha)
    c = cl.clone().requires_grad_(True)
    (0.7 * _lookup_loss(x4, c, alpha)).backward()
    assert abs(ref["loss"].item() - loss.item()) <= 1e-12
    assert (ref["probs"] - probs.double().reshape(2, 27, 36)).abs().max().item() <= 1e-12
    if alpha is not None:
        lp = O.cluster_lookup(x4, cl, alpha, log_probs=True)
        assert (ref["logp"] - lp.reshape(2, 27, 36)).abs().max().item() <= 1e-12
    scale = c.grad.abs().max().item()
    assert (ref["dcl"] - c.grad).abs().max().item() <= 1e-12 * max(scale, 1.0)
    assert (ref["S"] >= ref["ip"].abs() - 1e-15).all() and (ref["S"] <= 1 + 1e-12).all()


def test_cluster_builders():
    B, C, P, n = 2, 70, 64, 27
    x, cl = R.cluster_inputs("ties", B, C, P, n)
    assert torch.equal(cl[1], cl[0])
    assert torch.equal(cl[2, :10], cl[3, 10:20]) and (cl[2, 10:] == 0).all() and (cl[3, :10] == 0).all() \
        and (cl[3, 20:] == 0).all()
    assert (cl[2].double() ** 2).sum().item() == float((cl[2] ** 2).sum())  # the fp32 norm is exact: equal dots
    assert torch.equal(x[:, :10, P // 2:], x[:, 10:20, P // 2:])
    arg = R.cluster_ref(x, cl, None)["arg"]
    assert (arg[:, :P // 2] == 0).all() and (arg[:, P // 2:] == 2).all()  # the tied pair holds the maximum
    x, cl = R.cluster_inputs("sharp", B, C, P, n)
    p = R.cluster_ref(x, cl, 50.0)["probs"]
    assert (p.amax(1) > 0.99).float().mean() > 0.9
    x, _ = R.cluster_inputs("zeros", B, C, P, n)
    assert (x[:, :, ::7] == 0).all() and (x.abs().sum(1) > 0).sum() == B * (P - len(range(0, P, 7)))
    _, cl = R.cluster_inputs("zerorow", B, C, P, n)
    assert (cl[-1] == 0).all() and (cl[:-1].norm(dim=1) > 1).all()


@pytest.mark.parametrize("h,w,H,W,n", [(7, 9, 50, 61, 5), (4, 4, 32, 32, 27), (8, 40, 64, 12, 32)])
def test_linear_ce_ref_matches_oracle_and_autograd(h, w, H, W, n):
    code, Wt, b, label = R.linear_inputs(2, 70, h, w, H, W, n, seed=1)
    code, Wt, b = code.double(), Wt.double(), b.double()
    ref = R.linear_ce_ref(code, Wt, b, label, n, grad=0.37)
    Wp, bp = Wt.view(n, 70, 1, 1).clone().requires_grad_(True), b.clone().requires_grad_(True)
    loss = O.linear_probe_loss(code, Wp, bp, label, n)
    (0.37 * loss).backward()
    assert abs(ref["loss"].item() - loss.item()) <= 1e-12
    assert (ref["dW"] - Wp.grad.view(n, 70)).abs().max().item() <= 1e-12
    assert (ref["db"] - bp.grad).abs().max().item() <= 1e-12
    assert ref["count"] == int(((label >= 0) & (label < n)).sum())


def test_linear_ce_all_ignored_reference_semantics():
    """The reference's CrossEntropyLoss over an empty selection: NaN loss, zero (finite) gradients — and so the ref."""
    code, Wt, b, label = R.linear_inputs(2, 70, 4, 4, 32, 32, 27, ignore="all", seed=2)
    Wp, bp = Wt.view(27, 70, 1, 1).clone().requires_grad_(True), b.clone().requires_grad_(True)
    loss = O.linear_probe_loss(code, Wp, bp, label, 27)
    loss.backward()
    assert torch.isnan(loss)
    assert torch.equal(Wp.grad, torch.zeros_like(Wp.grad)) and torch.equal(bp.grad, torch.zeros_like(bp.grad))
    ref = R.linear_ce_ref(code, Wt, b, label, 27)
    assert ref["count"] == 0 and torch.isnan(ref["loss"])
    assert (ref["dW"] == 0).all() and (ref["db"] == 0).all()


@pytest.mark.parametrize("label_dtype", [torch.int64, torch.int32, torch.uint8])
def test_linear_builders(label_dtype):
    n = 27
    _, _, _, lab = R.linear_inputs(2, 70, 28, 28, 224, 224, n, label_dtype=label_dtype, seed=4)
    vals = set(lab.unique().tolist())
    assert {0, n - 1, n}.issubset(vals) and (255 in vals if label_dtype == torch.uint8 else -1 in vals)
    _, _, _, lab = R.linear_inputs(2, 70, 28, 28, 224, 224, n, label_dtype=label_dtype, ignore="tiles", seed=4)
    valid = ((lab.long() >= 0) & (lab.long() < n)).view(2, 14, 16, 14, 16).any(4).any(2)  # [B, tiles_y, tiles_x]
    assert (~valid).sum() >= 2 * 14 * 14 // 3 and valid.any()
    _, _, _, lab = R.linear_inputs(2, 70, 28, 28, 224, 224, n, label_dtype=label_dtype, ignore="image", seed=4)
    assert not ((lab[0].long() >= 0) & (lab[0].long() < n)).any() and ((lab[1].long() >= 0) & (lab[1].long() < n)).any()
    _, _, _, lab = R.linear_inputs(2, 70, 28, 28, 224, 224, n, label_dtype=label_dtype, ignore="all", seed=4)
    assert not ((lab.long() >= 0) & (lab.long() < n)).any()
    code, Wt, b, _ = R.linear_inputs(2, 70, 28, 28, 224, 224, n, spread=100.0, seed=4)
    lg = torch.einsum("kc,bchw->bkhw", Wt, code) + b.view(1, -1, 1, 1)
    assert 60 < lg.abs().max().item() < 250


@pytest.mark.parametrize("flip", [False, True])
def test_eval_band_matches_reference_sequence(flip):
    """TTA average -> F.interpolate -> conv / log_softmax and ClusterLookup log-probs (the oracle), in fp64, band by band."""
    torch.manual_seed(9)
    B, C, h, w, H, W = 1, 70, 6, 8, 48, 64
    code = torch.randn(B, C, h, w, dtype=torch.float64)
    code_f = torch.randn(B, C, h, w, dtype=torch.float64) if flip else None
    Wt, b, cl = torch.randn(27, C, dtype=torch.float64), torch.randn(27, dtype=torch.float64), torch.randn(30, C, dtype=torch.float64)
    x = (code + code_f.flip(3)) / 2 if flip else code
    up = F.interpolate(x, (H, W), mode="bilinear", align_corners=False)
    want_l = torch.log_softmax(F.conv2d(up, Wt.view(27, C, 1, 1), b), 1)[0]
    want_c = O.cluster_lookup(up, cl, 2.0, log_probs=True)[0]
    xbar = R.tta_code(code, code_f)[0]
    for rows in ((0, 16), (16, 48)):
        e = R.eval_band(xbar, Wt, b, cl, 2.0, H, W, rows)
        nr = rows[1] - rows[0]
        assert (e["lin_logp"].view(27, nr, W) - want_l[:, rows[0]:rows[1]]).abs().max().item() <= 1e-12
        assert (e["clu_logp"].view(30, nr, W) - want_c[:, rows[0]:rows[1]]).abs().max().item() <= 1e-12


def test_confusion_matches_unsupervised_metrics():
    """utils.py:219-229 semantics, extra clusters included (their rows stay 0: preds >= n_classes are masked)."""
    from stego_b200.eval import UnsupervisedMetrics
    torch.manual_seed(10)
    label = torch.randint(-1, 29, (2, 16, 16))
    pred = torch.randint(0, 30, (2, 16, 16))
    m = UnsupervisedMetrics("x/", 27, 3, True)
    m.update(pred, label)
    assert torch.equal(R.confusion(pred, label, 30, 27), m.stats)


@pytest.mark.parametrize("ratio", [1e-1, 1e-2, 1e-3])
def test_anticorrelated_builder(ratio):
    """At output columns 16 j + 7 of an 8x upsampling, |v| / sum_t w_t |x_t| is the requested ratio (to the vertical
    mix of two rows); elsewhere the conditioning stays moderate."""
    B, C, h, w = 1, 70, 8, 16
    x = R.anticorrelated_code(B, C, h, w, ratio, seed=1).double()[0]
    H, W = 8 * h, 8 * w
    cr = R.Corners(h, w, H, W, "cpu")
    v = cr.interp(x.reshape(C, -1)).norm(dim=0).view(H, W)
    den = cr.interp(x.reshape(C, -1).norm(dim=0, keepdim=True))[0].view(H, W)
    cond = v / den
    tgt = cond[:, 7::16]
    assert (tgt <= 1.05 * ratio).all() and (tgt.median() >= 0.5 * ratio)
    assert cond.median() > 0.05
