"""Fused correspondence loss (sample+norm tiles, wgmma einsum, loss reduction, backward) vs the oracle.

Tolerances: the CUDA path computes the einsum as a bf16 hi/lo split (~2^-16 relative) with fp32
accumulation, so losses / cd / gradients are compared at 1e-4 relative (well inside the 1e-3 bar of
BASELINE.json) against the fp32 oracle on IDENTICAL inputs, coords and perms.
"""
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.join(os.path.dirname(__file__), "..", "oracle"))


def _rel(x, y):
    return ((x.double().cpu() - y.double().cpu()).norm() / y.double().cpu().norm().clamp_min(1e-30)).item()


def _inputs(B, E, D, h, correlated, seed):
    g = torch.Generator().manual_seed(seed)
    if correlated:
        # low-rank mixtures so that fd spans a wide range and clamp / shift branches are all exercised
        basis_f = torch.randn(16, E, generator=g)
        basis_c = torch.randn(16, D, generator=g)
        def mk(C, basis):
            z = torch.randn(B, 16, h, h, generator=g)
            return torch.einsum("bkhw,kc->bchw", z, basis) + 0.1 * torch.randn(B, C, h, h, generator=g)
        z = torch.randn(B, 16, h, h, generator=g)
        feats = torch.einsum("bkhw,kc->bchw", z, basis_f) + 0.1 * torch.randn(B, E, h, h, generator=g)
        code = torch.einsum("bkhw,kc->bchw", z, basis_c) + 0.1 * torch.randn(B, D, h, h, generator=g)
        zp = z + 0.3 * torch.randn(B, 16, h, h, generator=g)
        feats_pos = torch.einsum("bkhw,kc->bchw", zp, basis_f) + 0.1 * torch.randn(B, E, h, h, generator=g)
        code_pos = torch.einsum("bkhw,kc->bchw", zp, basis_c) + 0.1 * torch.randn(B, D, h, h, generator=g)
    else:
        feats, feats_pos = torch.randn(B, E, h, h, generator=g), torch.randn(B, E, h, h, generator=g)
        code, code_pos = torch.randn(B, D, h, h, generator=g), torch.randn(B, D, h, h, generator=g)
    return feats, feats_pos, code, code_pos


@pytest.mark.parametrize("correlated", [False, True])
@pytest.mark.parametrize("B,E,h,pointwise,zero_clamp,stab", [
    (2, 384, 28, True, True, False),
    (5, 768, 20, True, True, False),
    (3, 384, 14, False, True, False),
    (3, 384, 14, True, False, True),
    (1, 64, 9, True, True, False),
])
def test_corr_loss_matches_oracle(cuda_dev, B, E, h, pointwise, zero_clamp, stab, correlated):
    import stego_oracle as O
    from stego_b200 import corr
    D = 70
    cfg = O.LossCfg(pointwise=pointwise, zero_clamp=zero_clamp, stabalize=stab)
    feats, feats_pos, code, code_pos = _inputs(B, E, D, h, correlated, seed=B * 100 + h)
    torch.manual_seed(99)
    c1, c2, perms = O.draw_loss_randomness(B, cfg)
    code.requires_grad_(True)
    code_pos.requires_grad_(True)
    want = O.correlation_loss(feats, feats_pos, code, code_pos, c1, c2, perms, cfg)
    wl = O.weighted_correspondence_loss(want, cfg)
    gw = torch.autograd.grad(wl, [code, code_pos])

    spec = corr.LossSpec(cfg)
    dc = lambda t: t.detach().to(cuda_dev)
    code_g = dc(code).requires_grad_(True)
    code_pos_g = dc(code_pos).requires_grad_(True)
    losses, cd_means, cd, elems = corr.corr_loss(dc(feats), dc(feats_pos), code_g, code_pos_g, dc(c1), dc(c2),
                                                  [dc(p) for p in perms], spec, want_elems=True)
    S = 121
    assert _rel(cd[0], want[1].reshape(B, S, S)) < 2e-5
    assert _rel(cd[1], want[3].reshape(B, S, S)) < 2e-5
    assert _rel(cd[2:], want[5].reshape(5, B, S, S)) < 2e-5
    assert _rel(elems[2:], want[4].reshape(5, B, S, S)) < 1e-4
    tot = cfg.pos_intra_weight * losses[0] + cfg.pos_inter_weight * losses[1] + cfg.neg_inter_weight * losses[2:].mean()
    # individual call means: absolute tolerance relative to the typical |loss element| (cancellation!)
    scale = want[4].abs().mean().item()
    assert abs(losses[0].item() - want[0].item()) < 1e-4 * scale + 1e-4 * abs(want[0].item())
    assert abs(losses[1].item() - want[2].item()) < 1e-4 * scale + 1e-4 * abs(want[2].item())
    assert abs(losses[2:].mean().item() - want[4].mean().item()) < 1e-4 * scale
    assert abs(tot.item() - wl.item()) < 1e-4 * scale + 1e-4 * abs(wl.item())
    gg = torch.autograd.grad(tot, [code_g, code_pos_g])
    assert _rel(gg[0], gw[0]) < 1e-4
    assert _rel(gg[1], gw[1]) < 1e-4


def test_corr_loss_elementwise_and_cd_grads(cuda_dev):
    """API path: gradients arriving through the unreduced negative loss and through the cd tensors."""
    import stego_oracle as O
    from stego_b200 import corr
    B, E, D, h = 3, 384, 70, 12
    cfg = O.LossCfg()
    feats, feats_pos, code, code_pos = _inputs(B, E, D, h, True, seed=5)
    torch.manual_seed(3)
    c1, c2, perms = O.draw_loss_randomness(B, cfg)
    wts = torch.randn(5 * B, 11, 11, 11, 11)
    code.requires_grad_(True)
    code_pos.requires_grad_(True)
    want = O.correlation_loss(feats, feats_pos, code, code_pos, c1, c2, perms, cfg)
    obj = (want[4] * wts).sum() / 1000 + want[0] + 0.01 * want[3].pow(2).sum()
    gw = torch.autograd.grad(obj, [code, code_pos])
    spec = corr.LossSpec(cfg)
    dc = lambda t: t.detach().to(cuda_dev)
    code_g, code_pos_g = dc(code).requires_grad_(True), dc(code_pos).requires_grad_(True)
    losses, _, cd, elems = corr.corr_loss(dc(feats), dc(feats_pos), code_g, code_pos_g, dc(c1), dc(c2),
                                          [dc(p) for p in perms], spec, want_elems=True)
    obj_g = (elems[2:].reshape(5 * B, 11, 11, 11, 11) * dc(wts)).sum() / 1000 + losses[0] + 0.01 * cd[1].pow(2).sum()
    gg = torch.autograd.grad(obj_g, [code_g, code_pos_g])
    assert _rel(gg[0], gw[0]) < 1e-4
    assert _rel(gg[1], gw[1]) < 1e-4


def test_corr_loss_bf16_channels_last_feats_and_padded_code(cuda_dev):
    """The layouts the fused training step actually uses: bf16 tokens-major feats, fp32 code padded to 72."""
    import stego_oracle as O
    from stego_b200 import corr
    B, E, D, h = 4, 384, 70, 28
    cfg = O.LossCfg()
    feats, feats_pos, code, code_pos = _inputs(B, E, D, h, True, seed=11)
    feats, feats_pos = feats.bfloat16().float(), feats_pos.bfloat16().float()
    torch.manual_seed(1)
    c1, c2, perms = O.draw_loss_randomness(B, cfg)
    code.requires_grad_(True)
    code_pos.requires_grad_(True)
    want = O.correlation_loss(feats, feats_pos, code, code_pos, c1, c2, perms, cfg)
    wl = O.weighted_correspondence_loss(want, cfg)
    gw = torch.autograd.grad(wl, [code, code_pos])
    spec = corr.LossSpec(cfg)
    dc = lambda t: t.detach().to(cuda_dev)
    f_cl = dc(feats).bfloat16().permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
    fp_cl = dc(feats_pos).bfloat16().permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)

    def padded(t):
        store = torch.zeros(B, h, h, 72, device=cuda_dev)
        store[..., :D] = dc(t).permute(0, 2, 3, 1)
        return store[..., :D].permute(0, 3, 1, 2).requires_grad_(True)

    cg, cpg = padded(code), padded(code_pos)
    losses, _, _, _ = corr.corr_loss(f_cl, fp_cl, cg, cpg, dc(c1), dc(c2), [dc(p) for p in perms], spec)
    tot = cfg.pos_intra_weight * losses[0] + cfg.pos_inter_weight * losses[1] + cfg.neg_inter_weight * losses[2:].mean()
    scale = want[4].abs().mean().item()
    assert abs(tot.item() - wl.item()) < 1e-4 * scale + 1e-4 * abs(wl.item())
    gg = torch.autograd.grad(tot, [cg, cpg])
    assert _rel(gg[0], gw[0]) < 1e-4
    assert _rel(gg[1], gw[1]) < 1e-4


@pytest.mark.parametrize("B,E,h,w,fs,neg", [(1, 384, 14, 14, 11, 5), (2, 128, 9, 13, 5, 2), (3, 64, 7, 5, 3, 0),
                                             (4, 384, 28, 20, 11, 1)])
def test_corr_loss_edge_shapes(cuda_dev, B, E, h, w, fs, neg):
    """Edge cases: batch of one (super_perm(1) == [0]: the negative of an image is itself), non-square maps,
    fewer sample points / negatives than the shipped config, no negatives at all."""
    import stego_oracle as O
    from stego_b200 import corr
    D = 70
    cfg = O.LossCfg(feature_samples=fs, neg_samples=neg)
    g = torch.Generator().manual_seed(B * 31 + h)
    feats, feats_pos = torch.randn(B, E, h, w, generator=g), torch.randn(B, E, h, w, generator=g)
    code = torch.randn(B, D, h, w, generator=g, requires_grad=True)
    code_pos = torch.randn(B, D, h, w, generator=g, requires_grad=True)
    torch.manual_seed(B)
    c1, c2, perms = O.draw_loss_randomness(B, cfg)
    c1 = c1 * 1.2  # some coordinates outside [-1, 1]: border clamping
    want = O.correlation_loss(feats, feats_pos, code, code_pos, c1, c2, perms, cfg) if neg > 0 else None
    if neg == 0:
        f, c = O.bilinear_sample(feats, c1), O.bilinear_sample(code, c1)
        fp, cp = O.bilinear_sample(feats_pos, c2), O.bilinear_sample(code_pos, c2)
        li, _ = O.corr_helper(f, f, c, c, cfg.pos_intra_shift, cfg)
        le, _ = O.corr_helper(f, fp, c, cp, cfg.pos_inter_shift, cfg)
        wl = 0.67 * li.mean() + 0.25 * le.mean()
        want_losses = [li.mean(), le.mean()]
    else:
        wl = O.weighted_correspondence_loss(want, cfg)
        want_losses = [want[0], want[2]] + [x.mean() for x in want[4].chunk(neg, 0)]
    gw = torch.autograd.grad(wl, [code, code_pos])
    spec = corr.LossSpec(cfg)
    dc = lambda t: t.detach().to(cuda_dev)
    cg, cpg = dc(code).requires_grad_(True), dc(code_pos).requires_grad_(True)
    losses, _, _, _ = corr.corr_loss(dc(feats), dc(feats_pos), cg, cpg, dc(c1), dc(c2), [dc(p) for p in perms], spec)
    assert losses.shape == (2 + neg,)
    for got, ref in zip(losses.tolist(), want_losses):
        assert abs(got - ref.item()) < 2e-5 + 1e-4 * abs(ref.item())
    tot = 0.67 * losses[0] + 0.25 * losses[1] + (0.63 * losses[2:].mean() if neg > 0 else 0.0)
    gg = torch.autograd.grad(tot, [cg, cpg])
    assert _rel(gg[0], gw[0]) < 2e-4
    assert _rel(gg[1], gw[1]) < 2e-4


def test_corr_loss_rejects_unsupported(cuda_dev):
    from stego_b200 import corr
    from stego_b200.config import make_cfg
    with pytest.raises(RuntimeError, match="feature_samples"):
        corr.LossSpec(make_cfg(feature_samples=12))
    spec = corr.LossSpec(make_cfg())
    f = torch.randn(2, 100, 8, 8, device=cuda_dev)  # channels not a multiple of 64
    c = torch.randn(2, 70, 8, 8, device=cuda_dev)
    z = torch.zeros(2, 11, 11, 2, device=cuda_dev)
    with pytest.raises(RuntimeError, match="unsupported"):
        corr.corr_loss(f, f, c, c, z, z, [torch.zeros(2, dtype=torch.long, device=cuda_dev)] * 5, spec)
