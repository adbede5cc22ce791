"""Multi-tile correspondence loss (feature_samples 12 .. 64, S = fs^2 > 128 sample points per image) against the oracle,
against the single-tile kernels where both apply, and through the training step (fused and autograd paths).

The tolerances are those of the single-tile tests: losses |d| < 2e-5 + 1e-4 |ref| and code gradients 2e-4 relative L2
(test_corr_gpu.py::test_corr_loss_edge_shapes), widened for clamp kinks as in test_boundary_gpu.py.
"""
import os
import sys

import pytest
import torch

from _parity_util import (NAMES, OracleStepper, feats_from_tokens, fp32_strict, grads_of, make_batch, make_model,
                          params_of, peek_draws, record, rel)

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.join(os.path.dirname(__file__), "..", "oracle"))


def _kink_tol(cds, base):
    """clamp(cd) makes dL/dcd jump at the clamp bounds: elements within fp32 noise of a bound can land on either side,
    and each moves a per-pixel code gradient by ~1/sqrt(active elements).  Widen the bar by the count of such elements."""
    edge = sum(int((c.abs() < 5e-6).sum()) + int(((c - 0.8).abs() < 5e-6).sum()) for c in cds)
    act = sum(int((c >= 0).sum()) for c in cds)
    return base + 3.0 * (edge / max(act, 1)) ** 0.5


def _maps(B, C, h, w, g, correlated):
    if not correlated:
        return torch.randn(B, C, h, w, generator=g)
    basis = torch.randn(16, C, generator=g)
    mix = torch.randn(B, h, w, 16, generator=g)
    return (mix @ basis + 0.1 * torch.randn(B, h, w, C, generator=g)).permute(0, 3, 1, 2).contiguous()


def _oracle(feats, feats_pos, code, code_pos, c1, c2, perms, cfg, neg):
    """Per-call mean losses, weighted total and the cd tensors of the oracle."""
    import stego_oracle as O
    if neg == 0:
        f, c = O.bilinear_sample(feats, c1), O.bilinear_sample(code, c1)
        fp, cp = O.bilinear_sample(feats_pos, c2), O.bilinear_sample(code_pos, c2)
        li, cdi = O.corr_helper(f, f, c, c, cfg.pos_intra_shift, cfg)
        le, cde = O.corr_helper(f, fp, c, cp, cfg.pos_inter_shift, cfg)
        return [li.mean(), le.mean()], 0.67 * li.mean() + 0.25 * le.mean(), [cdi, cde]
    want = O.correlation_loss(feats, feats_pos, code, code_pos, c1, c2, perms, cfg)
    losses = [want[0], want[2]] + [x.mean() for x in want[4].chunk(neg, 0)]
    return losses, O.weighted_correspondence_loss(want, cfg), [want[1], want[3], want[5]]


def _ours_total(losses, neg):
    return 0.67 * losses[0] + 0.25 * losses[1] + (0.63 * losses[2:].mean() if neg > 0 else 0.0)


def _run_vs_oracle(dev, B, E, h, w, fs, neg, cfg_over=None, bf16_feats=False, channels_last=False, correlated=False,
                   seed=0):
    import stego_oracle as O
    from stego_b200 import corr
    D = 70
    cfg = O.LossCfg(feature_samples=fs, neg_samples=neg, **(cfg_over or {}))
    g = torch.Generator().manual_seed(seed + B * 31 + h)
    feats, feats_pos = _maps(B, E, h, w, g, correlated), _maps(B, E, h, w, g, correlated)
    if bf16_feats:
        feats, feats_pos = feats.bfloat16().float(), feats_pos.bfloat16().float()
    code = _maps(B, D, h, w, g, correlated).requires_grad_(True)
    code_pos = _maps(B, D, h, w, g, correlated).requires_grad_(True)
    torch.manual_seed(B + fs)
    c1, c2, perms = O.draw_loss_randomness(B, cfg)
    c1 = c1 * 1.2  # some coordinates outside [-1, 1]: border clamping
    want_losses, wl, cds = _oracle(feats, feats_pos, code, code_pos, c1, c2, perms, cfg, neg)
    gw = torch.autograd.grad(wl, [code, code_pos])

    spec = corr.make_spec(cfg)
    assert isinstance(spec, corr.TiledLossSpec)

    dc = lambda t: t.detach().to(dev)
    f, fp = dc(feats), dc(feats_pos)
    if bf16_feats:
        f, fp = f.bfloat16(), fp.bfloat16()
    if channels_last:
        f = f.contiguous(memory_format=torch.channels_last)
        fp = fp.contiguous(memory_format=torch.channels_last)
    cg, cpg = dc(code).requires_grad_(True), dc(code_pos).requires_grad_(True)
    losses, _, _, _ = corr.corr_loss(f, fp, cg, cpg, dc(c1), dc(c2), [dc(p) for p in perms], spec)
    assert losses.shape == (2 + neg,)
    for got, ref in zip(losses.tolist(), want_losses):
        assert abs(got - ref.item()) < 2e-5 + 1e-4 * abs(ref.item()), (got, ref.item())
    gg = torch.autograd.grad(_ours_total(losses, neg), [cg, cpg])
    bar = _kink_tol(cds, 2e-4)
    assert rel(gg[0], gw[0]) < bar, (rel(gg[0], gw[0]), bar)
    assert rel(gg[1], gw[1]) < bar, (rel(gg[1], gw[1]), bar)


@pytest.mark.parametrize("B,E,h,w,fs,neg", [
    (2, 384, 28, 28, 12, 5),
    (3, 128, 9, 13, 16, 2),   # fs > h, non-square map
    (1, 64, 7, 5, 13, 0),     # batch of one, no negatives
    (2, 768, 20, 20, 24, 1),  # S = 576: not a multiple of 128
    (2, 384, 28, 28, 28, 5),
])
def test_tiled_loss_matches_oracle(cuda_dev, B, E, h, w, fs, neg):
    _run_vs_oracle(cuda_dev, B, E, h, w, fs, neg)


@pytest.mark.parametrize("over", [dict(pointwise=False), dict(zero_clamp=False, stabalize=True), dict(stabalize=True)],
                         ids=["no_pointwise", "no_zero_clamp_stabalize", "stabalize"])
def test_tiled_loss_branches(cuda_dev, over):
    _run_vs_oracle(cuda_dev, 2, 384, 20, 20, 14, 3, cfg_over=over, correlated=True)


@pytest.mark.parametrize("bf16_feats,channels_last", [(True, False), (False, True), (True, True)])
def test_tiled_loss_feature_layouts(cuda_dev, bf16_feats, channels_last):
    _run_vs_oracle(cuda_dev, 2, 384, 24, 24, 17, 2, bf16_feats=bf16_feats, channels_last=channels_last)


def test_tiled_contrastive_correlation_loss_6tuple(cuda_dev):
    """ContrastiveCorrelationLoss.forward at fs = 16: cd tensors, negative loss elements, and gradients arriving through
    them (random upstream weights) as well as through the call means."""
    import stego_oracle as O
    from stego_b200.config import make_cfg
    from stego_b200.modules import ContrastiveCorrelationLoss
    fs, B, E, D, h = 16, 2, 384, 70, 28
    cfg = make_cfg(feature_samples=fs)
    ocfg = O.LossCfg(feature_samples=fs)
    g = torch.Generator().manual_seed(17)
    feats, feats_pos = _maps(B, E, h, h, g, True), _maps(B, E, h, h, g, True)
    code, code_pos = _maps(B, D, h, h, g, True), _maps(B, D, h, h, g, True)
    dc = code.to(cuda_dev).requires_grad_(True)
    dcp = code_pos.to(cuda_dev).requires_grad_(True)
    torch.manual_seed(99)
    c1, c2, perms = O.draw_loss_randomness(B, ocfg, device=cuda_dev)  # the draws forward() is about to make
    torch.manual_seed(99)
    out = ContrastiveCorrelationLoss(cfg)(feats.to(cuda_dev), feats_pos.to(cuda_dev), None, None, dc, dcp)
    five = (fs, fs, fs, fs)
    assert len(out) == 6 and out[0].shape == () and out[2].shape == ()
    assert out[1].shape == (B, *five) and out[3].shape == (B, *five)
    assert out[4].shape == (5 * B, *five) and out[5].shape == (5 * B, *five)
    oc, ocp = code.clone().requires_grad_(True), code_pos.clone().requires_grad_(True)
    want = O.correlation_loss(feats, feats_pos, oc, ocp, c1.cpu(), c2.cpu(), [p.cpu() for p in perms], ocfg)
    scale = max(want[4].abs().max().item(), 1e-3)
    for i in (1, 3, 5):
        assert (out[i].cpu() - want[i]).abs().max().item() < 5e-5, i
    assert (out[4].cpu() - want[4]).abs().max().item() < 1e-4 * scale + 1e-5
    for i in (0, 2):
        assert abs(out[i].item() - want[i].item()) < 1e-3 * abs(want[i].item()) + 1e-4 * scale
    gen = torch.Generator().manual_seed(3)
    w_el = torch.randn(5 * B, *five, generator=gen)
    w_cd = torch.randn(B, *five, generator=gen)
    obj = lambda o, w1, w2: 0.67 * o[0] + 0.25 * o[2] + (o[4] * w1).sum() / 1000 + 0.01 * (o[3] * w2).sum()
    obj(out, w_el.to(cuda_dev), w_cd.to(cuda_dev)).backward()
    obj(want, w_el, w_cd).backward()
    bar = _kink_tol([want[1], want[3], want[5]], 1e-3)
    assert rel(dc.grad, oc.grad) < bar, rel(dc.grad, oc.grad)
    assert rel(dcp.grad, ocp.grad) < bar, rel(dcp.grad, ocp.grad)


@pytest.mark.parametrize("fs", [5, 11])
def test_tiled_agrees_with_single_tile(cuda_dev, fs):
    """Where both implementations apply (S <= 128), the multi-tile entry and the single-tile kernels agree to 1e-6."""
    import stego_oracle as O
    from stego_b200 import corr
    B, E, D, h, neg = 3, 384, 70, 20, 5
    cfg = O.LossCfg(feature_samples=fs, neg_samples=neg)
    g = torch.Generator().manual_seed(fs)
    feats, feats_pos = _maps(B, E, h, h, g, True).to(cuda_dev), _maps(B, E, h, h, g, True).to(cuda_dev)
    code, code_pos = _maps(B, D, h, h, g, True).to(cuda_dev), _maps(B, D, h, h, g, True).to(cuda_dev)
    torch.manual_seed(fs)
    c1, c2, perms = O.draw_loss_randomness(B, cfg, device=cuda_dev)
    wts = torch.randn(neg * B, fs * fs, fs * fs, device=cuda_dev)
    res = []
    for spec in (corr.LossSpec(cfg), corr.TiledLossSpec(cfg)):
        cg, cpg = code.clone().requires_grad_(True), code_pos.clone().requires_grad_(True)
        losses, cd_means, cd, elems = corr.corr_loss(feats, feats_pos, cg, cpg, c1, c2, perms, spec, want_elems=True)
        obj = _ours_total(losses, neg) + (elems[2:].reshape(neg * B, fs * fs, fs * fs) * wts).sum() / 1000
        gg = torch.autograd.grad(obj, [cg, cpg])
        res.append((losses.detach(), cd_means, cd, elems.detach(), gg))
    (l0, m0, cd0, e0, g0), (l1, m1, cd1, e1, g1) = res
    scale = e0.abs().mean().item()
    assert (l1 - l0).abs().max().item() < 1e-6 * (l0.abs().max().item() + scale)
    assert (m1 - m0).abs().max().item() < 1e-6 * m0.abs().max().item()
    assert torch.equal(cd1, cd0)  # same wgmma sequence on the same operand tiles
    assert rel(e1, e0) < 1e-6
    assert rel(g1[0], g0[0]) < 1e-6 and rel(g1[1], g0[1]) < 1e-6


def test_tiled_bit_reproducible(cuda_dev):
    from stego_b200 import corr
    from stego_b200.config import make_cfg
    import stego_oracle as O
    B, E, D, h, fs = 4, 384, 70, 28, 28
    cfg = make_cfg(feature_samples=fs)
    g = torch.Generator().manual_seed(1)
    feats, feats_pos = _maps(B, E, h, h, g, True).to(cuda_dev), _maps(B, E, h, h, g, True).to(cuda_dev)
    code, code_pos = _maps(B, D, h, h, g, True).to(cuda_dev), _maps(B, D, h, h, g, True).to(cuda_dev)
    torch.manual_seed(0)
    c1, c2, perms = O.draw_loss_randomness(B, O.LossCfg(feature_samples=fs), device=cuda_dev)
    spec = corr.make_spec(cfg)
    outs = []
    for _ in range(2):
        cg, cpg = code.clone().requires_grad_(True), code_pos.clone().requires_grad_(True)
        losses, _, _, _ = corr.corr_loss(feats, feats_pos, cg, cpg, c1, c2, perms, spec)
        gg = torch.autograd.grad(_ours_total(losses, 5), [cg, cpg])
        outs.append((losses.detach(), gg[0], gg[1]))
    for a, b in zip(*outs):
        assert torch.equal(a, b)


class _Stepper(OracleStepper):
    """OracleStepper with the loss configuration of the model (feature_samples != 11)."""

    def __init__(self, params0, odev, lcfg):
        super().__init__(params0, odev)
        self.lcfg = lcfg

    def losses(self, f_all, B, label, draws, round_bf16=True):
        import stego_oracle as O
        m, mp, c1, c2, perms = draws
        od = self.odev
        for t in self.p.values():
            t.grad = None
        hp = {k[len("net."):]: v for k, v in self.p.items() if k.startswith("net.")}
        probes = {k: v for k, v in self.p.items() if not k.startswith("net.")}
        to4 = lambda t: t.to(od).view(B, -1, 1, 1)
        out = O.training_losses(f_all[:B], f_all[B:], hp, probes, label.to(od), [to4(x) for x in m], [to4(x) for x in mp],
                                c1.to(od), c2.to(od), [p.to(od) for p in perms], self.lcfg, 27, round_bf16=round_bf16)
        out["total"].backward()
        return out


def _check_step_losses(model, loss, out, tol=1e-3):
    logged = {k: float(v) for k, v in model.logged.items()}
    elem_scale = 0.05
    for k_log, k_or in [("loss/pos_intra", "pos_intra"), ("loss/pos_inter", "pos_inter"), ("loss/neg_inter", "neg_inter")]:
        assert abs(logged[k_log] - out[k_or].item()) < tol * abs(out[k_or].item()) + tol * elem_scale, (k_log,)
    assert abs(float(loss) - out["total"].item()) < tol * abs(out["total"].item())


def test_tiled_training_steps_fused_vs_autograd_vs_oracle(cuda_dev):
    """fs = 16, ViT-S: eager step, graph capture, replays — the hand-scheduled step against the autograd path and the
    oracle stepping its own parameters (the bars of test_multistep_graph_replay_vs_autograd_vs_oracle)."""
    import stego_oracle as O
    from stego_b200 import corr
    fs, arch, res, B, nsteps = 16, "vit_small", 64, 4, 5
    fused, _ = make_model(arch, cuda_dev, fused=True, feature_samples=fs)
    twin, _ = make_model(arch, cuda_dev, fused=False, feature_samples=fs)
    assert isinstance(fused._spec, corr.TiledLossSpec)
    batches = [make_batch(B, res, cuda_dev, seed=1), make_batch(B, res, cuda_dev, seed=2)]
    orc = _Stepper(params_of(fused), "cpu", O.LossCfg(feature_samples=fs))
    h = res // 8
    torch.manual_seed(777)
    worst = dict(grad=0.0, param=0.0, twin_grad=0.0, twin_param=0.0)
    for s in range(nsteps):
        batch = batches[s % 2]
        draws = peek_draws(fused, B, cuda_dev)
        gpu_state, cpu_state = torch.cuda.get_rng_state(cuda_dev), torch.get_rng_state()
        p_before = params_of(fused)
        loss = fused.training_step(batch, s)
        g_f, p_f = grads_of(fused), params_of(fused)
        torch.cuda.set_rng_state(gpu_state, cuda_dev)
        torch.set_rng_state(cpu_state)
        loss_t = twin.training_step(batch, s)
        g_t, p_t = grads_of(twin), params_of(twin)
        assert fused._fused.step_idx == s + 1 and twin._fused is None
        if s >= 2:
            assert fused._fused.ws.graph is not None
        assert abs(float(loss) - float(loss_t.detach())) < 2e-5 * abs(float(loss_t.detach()))
        for k in NAMES:
            worst["twin_grad"] = max(worst["twin_grad"], rel(g_f[k], g_t[k]))
            assert rel(g_f[k], g_t[k]) < 3e-3, (s, k, rel(g_f[k], g_t[k]))
            worst["twin_param"] = max(worst["twin_param"], rel(p_f[k], p_t[k]))
            assert rel(p_f[k], p_t[k]) < 2e-4, (s, k, rel(p_f[k], p_t[k]))
        with torch.no_grad():
            tok = fused.net.backbone_tokens(torch.cat([batch["img"], batch["img_pos"]], 0)).float().cpu()
        out = orc.losses(feats_from_tokens(tok, 2 * B, h, h), B, batch["label"].cpu(), draws)
        _check_step_losses(fused, loss, out)
        g_o = orc.grads()
        for k in NAMES:
            worst["grad"] = max(worst["grad"], rel(g_f[k], g_o[k]))
            assert rel(g_f[k], g_o[k]) < 1e-3, (s, k, rel(g_f[k], g_o[k]))
        orc.adam(g_f)
        for k in NAMES:
            d_f = p_f[k].cpu() - p_before[k].cpu()
            d_o = orc.p[k].detach() - p_before[k].cpu()
            worst["param"] = max(worst["param"], rel(d_f, d_o))
            assert rel(d_f, d_o) < 1e-4, (s, k, rel(d_f, d_o))
            assert rel(p_f[k], orc.p[k]) < 1e-5, (s, k)
    record("tiled_multistep_fs16", dict(steps=nsteps, worst=worst))


def test_tiled_fullsize_c1_fs28_vs_gpu_fp32_oracle(cuda_dev):
    """c1 (ViT-S/8 224², B = 32) with feature_samples = 28 (S = 784): the graph-replayed step against the fp32 GPU
    oracle on identical backbone features, at the 1e-3 bar."""
    import stego_oracle as O
    fs, arch, res, B = 28, "vit_small", 224, 32
    fp32_strict()
    model, _ = make_model(arch, cuda_dev, fused=True, feature_samples=fs)
    batches = [make_batch(B, res, cuda_dev, seed=1), make_batch(B, res, cuda_dev, seed=2)]
    orc = _Stepper(params_of(model), "cuda", O.LossCfg(feature_samples=fs))
    h = res // 8
    torch.manual_seed(777)
    nsteps = 3
    for s in range(nsteps):
        batch = batches[s % 2]
        draws = peek_draws(model, B, cuda_dev)
        loss = model.training_step(batch, s)
        g = grads_of(model)
        if s < nsteps - 1:
            orc.adam(g)
            continue
        with torch.no_grad():
            tok = model.net.backbone_tokens(torch.cat([batch["img"], batch["img_pos"]], 0)).float()
        out = orc.losses(feats_from_tokens(tok, 2 * B, h, h), B, batch["label"], draws)
        _check_step_losses(model, loss, out)
        g_o = orc.grads()
        same = {k: rel(g[k], g_o[k]) for k in NAMES}
        record("tiled_fullsize_c1_fs28", dict(total_loss=float(loss), oracle_total=out["total"].item(),
                                               grad_rel_same_features=same))
        for k in NAMES:
            assert same[k] < 1e-3, (k, same[k])


def test_tiled_refusals(cuda_dev):
    from stego_b200 import corr
    from stego_b200.config import make_cfg
    from stego_b200.segmenter import LitUnsupervisedSegmenter
    with pytest.raises(RuntimeError, match="64"):
        corr.make_spec(make_cfg(feature_samples=65))
    with pytest.raises(RuntimeError, match="64"):
        LitUnsupervisedSegmenter(27, make_cfg(feature_samples=65, random_backbone_init=True))
    spec = corr.make_spec(make_cfg(feature_samples=16))
    f = torch.randn(2, 384, 8, 8)
    c = torch.randn(2, 70, 8, 8)
    z = torch.zeros(2, 16, 16, 2)
    with pytest.raises(RuntimeError, match="CUDA"):
        corr.corr_loss(f, f, c, c, z, z, [torch.zeros(2, dtype=torch.long)] * 5, spec)
