"""GPU: training with ground-truth label correspondences (cfg.use_true_labels, train_segmentation.py:135-140).

  * Tiles: stego_sample_labels_fwd (corr.build_label_tiles) writes, bit for bit, the tiles stego_sample_norm_fwd writes
    for the materialised fp32 map one_hot_feats(label + 1, n_classes + 1) on the same draws; and hi + lo sits within
    the split bound of the fp64 normalised interpolation.
  * The loss kernels at the narrow teacher widths the label tiles have (E = 64 .. 256), every stage against the fp64
    references of tests/_corr_fp64.py at the c1-c3 code shapes, with the bars of tests/test_corr_fp64_gpu.py.
  * The drop-in module on a one-hot signal at label resolution against the reference's 6-tuple, and the label-tile
    path against it bit for bit.
  * The training step: fused vs autograd bit-equal on the first step; six eager / capture / replay steps against the
    autograd twin and the oracle (oracle/true_labels_oracle.py); the shipped configuration unaffected.
"""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _corr_fp64 as R  # noqa: E402
import stego_oracle as O  # noqa: E402
import true_labels_oracle as TL  # noqa: E402
from _parity_util import (NAMES, OracleStepper, feats_from_tokens, grads_of, make_batch, make_model, params_of,  # noqa: E402
                          peek_draws, rel)
from test_corr_fp64_gpu import SHAPES, _case  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ================================================================================================
# label tiles
# ================================================================================================
def _labels(kind, B, H, W, n, dtype, g):
    """[2, B, H, W] label maps: `region` (piecewise constant 7x5 blocks, mostly pure one-hot samples), `random`
    (per-pixel), `unlabelled` (all -1 / 255), each with out-of-range values mixed in (-1, n, n + 5, and 255 for uint8,
    -7 and 2^40 for the signed types)."""
    if kind == "unlabelled":
        lab = torch.full((2, B, H, W), -1, dtype=torch.long)
    elif kind == "region":
        blocks = torch.randint(-1, n, (2, B, -(-H // 7), -(-W // 5)), generator=g)
        lab = blocks.repeat_interleave(7, -2).repeat_interleave(5, -1)[..., :H, :W].contiguous()
    else:
        lab = torch.randint(-1, n, (2, B, H, W), generator=g)
    if kind != "unlabelled":
        odd = torch.rand(2, B, H, W, generator=g) < 0.05
        bad = [n, n + 5] + ([255] if dtype == torch.uint8 else [-7, 2 ** 40 if dtype == torch.int64 else 2 ** 30])
        pick = torch.tensor(bad)[torch.randint(len(bad), (2, B, H, W), generator=g)]
        lab = torch.where(odd, pick, lab)
    if dtype == torch.uint8:
        lab = torch.where((lab < 0) | (lab > 255), torch.full_like(lab, 255), lab)
    return lab.to(dtype)


def _one_hot(lab, n):
    """the fp32 one_hot_feats(label + 1, n + 1) map, out-of-range labels as class 0 (build_label_tiles' rule)"""
    lab = lab.long()
    cls = torch.where((lab >= 0) & (lab < n), lab + 1, torch.zeros_like(lab))
    return F.one_hot(cls, n + 1).permute(0, 3, 1, 2).float().contiguous()


def _draws(B, fs, n_neg, g, dev):
    """coords in [-1.1, 1.1] (border clamping included), with the first row of coords1 on the corners; raw perms"""
    c1 = torch.rand(B, fs, fs, 2, generator=g) * 2.2 - 1.1
    c2 = torch.rand(B, fs, fs, 2, generator=g) * 2.2 - 1.1
    c1[:, 0, :4] = torch.tensor([[-1.0, -1.0], [1.0, -1.0], [-1.0, 1.0], [1.0, 1.0]])[: min(4, fs)]
    perms = torch.stack([torch.randperm(B, generator=g) for _ in range(n_neg)])
    return c1.to(dev), c2.to(dev), perms.to(dev)


TILE_CASES = {  # B, H, W (label map), fs, n_classes
    "B1_fs11_n27": (1, 37, 53, 11, 27),
    "B3_fs16_n63": (3, 90, 70, 16, 63),
    "B4_fs28_n100": (4, 226, 211, 28, 100),
}


@pytest.mark.parametrize("case", list(TILE_CASES))
@pytest.mark.parametrize("kind", ["region", "random", "unlabelled"])
@pytest.mark.parametrize("dtype", [torch.int64, torch.int32, torch.uint8], ids=["int64", "int32", "uint8"])
def test_label_tiles_bit_equal_to_materialised_one_hot(cuda_dev, case, kind, dtype):
    from stego_b200 import corr
    from stego_b200.config import make_cfg
    B, H, W, fs, n = TILE_CASES[case]
    g = torch.Generator().manual_seed(B * 100 + fs)
    lab = _labels(kind, B, H, W, n, dtype, g).to(cuda_dev)
    spec = corr.make_spec(make_cfg(feature_samples=fs))
    c1, c2, perms = _draws(B, fs, spec.n_neg, g, cuda_dev)
    for raw in (True, False):
        got = corr.build_label_tiles(lab[0], lab[1], c1, c2, perms, spec, n, raw_perms=raw)
        want = corr.build_tiles(_one_hot(lab[0], n), _one_hot(lab[1], n), c1, c2, perms, spec,
                                corr.teacher_width(n + 1), raw_perms=raw)
        assert got.shape == want.shape and got.shape[-1] == corr.teacher_width(n + 1)
        assert torch.equal(got.view(torch.int16), want.view(torch.int16)), (case, kind, dtype, raw)
    if kind == "unlabelled":  # every sample is the class-0 unit vector
        S = fs * fs
        assert torch.equal(got[0, :, :, :S, 0], torch.ones_like(got[0, :, :, :S, 0]))
        assert torch.count_nonzero(got[0, :, :, :S, 1:]) == 0 and torch.count_nonzero(got[1]) == 0


@pytest.mark.parametrize("case", list(TILE_CASES))
def test_label_tiles_within_split_bound_of_fp64(cuda_dev, case):
    """hi + lo against the fp64 normalised bilinear interpolation of the one-hot map (_corr_fp64.gather_sample /
    normalise, the bar test_corr_fp64_gpu.py uses for every operand tile).  Derivation for this source: each channel is
    sum_t w_t [class_t == c] in fp32; the products are exact, the <= 3 additions round against A = sum_t |w_t [...]|
    (within normalise's 5 u A), the sum of squares is a chain_norm(C)-term fp32 chain, then sqrt, reciprocal and the
    product round once each (normalise's E_n), and the bf16 split drops |x - hi - lo| <= 2^-16 |x|: bar
    E_n + 2^-16 (|n| + E_n).  Rows >= S and channels > n_classes are exactly zero."""
    from stego_b200 import corr
    from stego_b200.config import make_cfg
    B, H, W, fs, n = TILE_CASES[case]
    g = torch.Generator().manual_seed(7 + fs)
    lab = _labels("random", B, H, W, n, torch.int64, g).to(cuda_dev)
    spec = corr.make_spec(make_cfg(feature_samples=fs))
    c1, c2, perms = _draws(B, fs, spec.n_neg, g, cuda_dev)
    tiles = corr.build_label_tiles(lab[0], lab[1], c1, c2, perms, spec, n, raw_perms=True)
    S, C = fs * fs, n + 1
    assert torch.count_nonzero(tiles[:, :, :, S:]) == 0 and torch.count_nonzero(tiles[..., C:]) == 0
    hl = tiles.double()[0] + tiles.double()[1]
    pr = R.resolve_perms(perms, B, True)
    ar = torch.arange(B, device=cuda_dev)
    oh, oh_pos = _one_hot(lab[0], n), _one_hot(lab[1], n)
    slots = [(ar, c1, oh), (ar, c2, oh_pos)] + [(pr[k], c2, oh) for k in range(spec.n_neg)]
    worst = 0.0
    for s, (img, coords, src) in enumerate(slots):
        idx, w = R.taps(coords, H, W)
        v, A = R.gather_sample(src, img, idx, w)
        nv, En, _ = R.normalise(v, A, R.chain_norm(C))
        err = (hl[s, :, :S, :C] - nv).abs()
        bar = En + R.SPLIT * (nv.abs() + En)
        assert (err <= bar).all(), (case, s, float((err - bar).max()))
        worst = max(worst, float(torch.where(err == 0, torch.zeros_like(err), err / bar).max()))
    assert worst <= 1.0


# ================================================================================================
# the loss kernels at narrow teacher widths
# ================================================================================================
NARROW = [("c1", 11), ("c2", 11), ("c3", 11), ("c1", 16), ("c2", 16), ("c3", 28)]


@pytest.mark.parametrize("shape,fs", NARROW, ids=[f"{s}_fs{f}" for s, f in NARROW])
@pytest.mark.parametrize("E", [64, 128, 192, 256])
def test_loss_stages_at_narrow_teacher_width(cuda_dev, E, shape, fs):
    """Every stage (operand tiles, losses, cd means, cd / row means / loss elements, d code) against the fp64
    references at the c1-c3 code shapes with a teacher of E = 64 .. 256 channels: the widths of the label tiles.  fs 11
    runs the single-tile phases with the [ncalls, B, S, S] outputs and random upstream gradients, fs 16 / 28 the
    multi-tile phases (a 3-stage forward ring and a 2-stage backward ring over 3 E / 64 k-steps per unit, 3 at E = 64)."""
    B, h, _ = SHAPES[shape]
    _case(cuda_dev, f"narrow_E{E}_{shape}_fs{fs}", "corr", B, h, h, E, fs, want_elems=fs == 11, seed=E + fs)


# ================================================================================================
# the drop-in module on a one-hot signal at label resolution
# ================================================================================================
def _golden():
    return torch.load(os.path.join(ROOT, "tests", "golden", "true_labels_step.pt"))


def test_module_on_one_hot_signal_matches_reference(cuda_dev, monkeypatch):
    """ContrastiveCorrelationLoss (the drop-in) on one_hot_feats(label + 1, 28) [B, 28, 40, 40] with a [B, 70, 10, 10]
    code — 28 channels and a 4x finer grid than the code, as the reference's train_segmentation.py hands it — against
    the reference module's 6-tuple, with the reference's draws injected (bars of test_oracle_golden.py's corr_small
    check); then the label-tile path on the same draws gives the same losses bit for bit."""
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import make_golden_true_labels as MG
    from stego_b200 import corr, modules
    from stego_b200.config import make_cfg
    want = _golden()["module"]
    label, label_pos, code, code_pos = MG.module_inputs()
    sig, sig_pos = TL.label_signals(label, label_pos, MG.N_CLASSES)
    c1, c2, perms = (want[k].to(cuda_dev) for k in ("coords1", "coords2", "perms"))
    monkeypatch.setattr(modules.ContrastiveCorrelationLoss, "draw_coords", lambda self, *a: (c1, c2))
    queue = list(perms)
    monkeypatch.setattr(modules, "super_perm", lambda size, device: queue.pop(0))
    cfg = make_cfg()
    c = code.to(cuda_dev).requires_grad_(True)
    cp = code_pos.to(cuda_dev).requires_grad_(True)
    o = modules.ContrastiveCorrelationLoss(cfg)(sig.to(cuda_dev), sig_pos.to(cuda_dev), None, None, c, cp)
    assert not queue
    loss = .67 * o[0] + .25 * o[2] + .63 * o[4].mean()
    loss.backward()
    for got, ref in ((o[0], want["pos_intra_loss"]), (o[2], want["pos_inter_loss"]),
                     (o[4].mean(), want["neg_inter_loss_mean"]), (loss, want["total"])):
        assert abs(got.item() - ref.item()) < 2e-5 + 1e-4 * abs(ref.item()), (got.item(), ref.item())
    cdm = torch.stack([o[1].mean(), o[3].mean(), o[5].mean()]).cpu()
    assert (cdm - want["cd_means"]).abs().max() < 1e-4
    assert (o[3].detach().reshape(-1)[::53].cpu() - want["inter_cd_sub"]).abs().max() < 1e-4
    assert (o[4].detach().reshape(-1)[::53].cpu() - want["neg_loss_sub"]).abs().max() < 1e-4
    assert rel(c.grad, want["code_grad"]) < 2e-4 and rel(cp.grad, want["code_pos_grad"]) < 2e-4
    # the label-tile path on the same draws: the same tiles, so the same losses
    spec = corr.make_spec(cfg)
    ftiles = corr.build_label_tiles(label.to(cuda_dev), label_pos.to(cuda_dev), c1, c2, perms, spec, MG.N_CLASSES)
    losses, _, _, _ = corr.corr_loss(None, None, c.detach(), cp.detach(), c1, c2, perms, spec, ftiles=ftiles)
    mod = torch.stack([o[0], o[2]]).detach()
    assert torch.equal(losses[:2], mod), (losses[:2], mod)
    neg = torch.stack([o[4][k * 3:(k + 1) * 3].mean() for k in range(cfg.neg_samples)]).detach()
    assert (losses[2:] - neg).abs().max() <= 1e-5 * neg.abs().max() + 1e-7  # the module's elements, re-averaged


# ================================================================================================
# the training step
# ================================================================================================
def _true_batch(B, res, dev, seed):
    b = make_batch(B, res, dev, seed=seed)
    g = torch.Generator().manual_seed(seed + 50)
    b["label_pos"] = torch.randint(-1, 27, (B, res, res), generator=g).to(dev)
    return b


def test_batch_without_label_pos_is_refused(cuda_dev):
    model, _ = make_model("vit_small", cuda_dev, fused=True, use_true_labels=True)
    with pytest.raises(RuntimeError, match="label_pos"):
        model.training_step(make_batch(2, 64, cuda_dev), 0)


@pytest.mark.parametrize("ldt", [torch.int64, torch.int32, torch.uint8], ids=["int64", "int32", "uint8"])
def test_first_step_fused_and_autograd_bit_equal(cuda_dev, ldt):
    fused, _ = make_model("vit_small", cuda_dev, fused=True, use_true_labels=True)
    twin, _ = make_model("vit_small", cuda_dev, fused=False, use_true_labels=True)
    batch = _true_batch(4, 64, cuda_dev, seed=1)
    for k in ("label", "label_pos"):
        lab = batch[k]
        batch[k] = torch.where(lab < 0, torch.full_like(lab, 255), lab).to(ldt) if ldt == torch.uint8 else lab.to(ldt)
    torch.manual_seed(777)
    gpu_state, cpu_state = torch.cuda.get_rng_state(cuda_dev), torch.get_rng_state()
    fused.training_step(batch, 0)
    after = torch.cuda.get_rng_state(cuda_dev)
    torch.cuda.set_rng_state(gpu_state, cuda_dev)
    torch.set_rng_state(cpu_state)
    twin.training_step(batch, 0)
    assert fused._fused.step_idx == 1 and twin._fused is None
    assert torch.equal(torch.cuda.get_rng_state(cuda_dev), after)
    torch.cuda.synchronize()
    for key in ("loss/pos_intra", "loss/pos_inter", "cd/pos_intra", "cd/pos_inter", "loss/cluster"):
        assert torch.equal(fused.logged[key], twin.logged[key]), (key, fused.logged[key].item(),
                                                                  twin.logged[key].item())


def _check_losses(model, loss, out, tol=1e-3):
    logged = {k: float(v) for k, v in model.logged.items()}
    elem_scale = 0.05
    assert abs(logged["loss/linear"] - out["linear"].item()) < 1e-4 * abs(out["linear"].item()) + 1e-6
    assert abs(logged["loss/cluster"] - out["cluster"].item()) < 2e-4 * abs(out["cluster"].item()) + 1e-6
    for k_log, k_or in [("loss/pos_intra", "pos_intra"), ("loss/pos_inter", "pos_inter"), ("loss/neg_inter", "neg_inter")]:
        assert abs(logged[k_log] - out[k_or].item()) < tol * abs(out[k_or].item()) + tol * elem_scale, \
            (k_log, logged[k_log], out[k_or].item())
    assert abs(float(loss) - out["total"].item()) < tol * abs(out["total"].item())


class _TrueLabelStepper(OracleStepper):
    def losses_true(self, f_all, B, label, label_pos, draws):
        m, mp, c1, c2, perms = draws
        od = self.odev
        for t in self.p.values():
            t.grad = None
        hp = {k[len("net."):]: v for k, v in self.p.items() if k.startswith("net.")}
        probes = {k: v for k, v in self.p.items() if not k.startswith("net.")}
        to4 = lambda t: t.to(od).view(B, -1, 1, 1)
        out = TL.training_losses(f_all[:B], f_all[B:], hp, probes, label.to(od), label_pos.to(od),
                                 [to4(x) for x in m], [to4(x) for x in mp], c1.to(od), c2.to(od),
                                 [p.to(od) for p in perms], O.LossCfg(), 27, round_bf16=True)
        out["total"].backward()
        return out


@pytest.mark.parametrize("reset_at", [None, 2], ids=["plain", "reset_probe_steps=2"])
def test_multistep_graph_replay_vs_autograd_vs_oracle(cuda_dev, reset_at):
    """test_step_parity_gpu.py's six-step procedure (eager, capture, 4 replays; batches alternating) with
    use_true_labels, at that test's bars, against oracle/true_labels_oracle.py."""
    arch, res, B, nsteps = "vit_small", 64, 4, 6
    fused, _ = make_model(arch, cuda_dev, fused=True, reset_probe_steps=reset_at, use_true_labels=True)
    twin, _ = make_model(arch, cuda_dev, fused=False, reset_probe_steps=reset_at, use_true_labels=True)
    batches = [_true_batch(B, res, cuda_dev, seed=1), _true_batch(B, res, cuda_dev, seed=2)]
    orc = _TrueLabelStepper(params_of(fused), "cpu")
    h = res // 8
    torch.manual_seed(777)
    for s in range(nsteps):
        batch = batches[s % 2]
        draws = peek_draws(fused, B, cuda_dev)
        gpu_state, cpu_state = torch.cuda.get_rng_state(cuda_dev), torch.get_rng_state()
        p_before = params_of(fused)
        loss = fused.training_step(batch, s)
        g_f, p_f = grads_of(fused), params_of(fused)
        after_state = torch.cuda.get_rng_state(cuda_dev)
        torch.cuda.set_rng_state(gpu_state, cuda_dev)
        torch.set_rng_state(cpu_state)
        loss_t = twin.training_step(batch, s)
        g_t, p_t = grads_of(twin), params_of(twin)
        assert torch.equal(torch.cuda.get_rng_state(cuda_dev), after_state), f"step {s}: RNG consumption differs"
        assert fused._fused.step_idx == s + 1 and twin._fused is None
        if s >= 2:
            assert fused._fused.ws.graph is not None
        assert abs(float(loss) - float(loss_t)) < 2e-5 * abs(float(loss_t)), (s, float(loss), float(loss_t))
        for k in NAMES:
            assert rel(g_f[k], g_t[k]) < 3e-3, (s, k, rel(g_f[k], g_t[k]))
            assert rel(p_f[k], p_t[k]) < 2e-4, (s, k, rel(p_f[k], p_t[k]))
        with torch.no_grad():
            tok = fused.net.backbone_tokens(torch.cat([batch["img"], batch["img_pos"]], 0)).float().cpu()
        out = orc.losses_true(feats_from_tokens(tok, 2 * B, h, h), B, batch["label"].cpu(), batch["label_pos"].cpu(),
                              draws)
        _check_losses(fused, loss, out)
        g_o = orc.grads()
        for k in NAMES:
            assert rel(g_f[k], g_o[k]) < 1e-3, (s, k, rel(g_f[k], g_o[k]))
        orc.adam(g_f)
        resetting = reset_at is not None and s == reset_at
        if resetting:
            for k in ("linear_probe.weight", "linear_probe.bias", "cluster_probe.clusters"):
                assert torch.equal(p_f[k], p_t[k]), k
                orc.adopt(k, p_f[k])
        for k in NAMES:
            if resetting and not k.startswith("net."):
                continue
            d_f = p_f[k].cpu() - p_before[k].cpu()
            d_o = orc.p[k].detach() - p_before[k].cpu()
            assert rel(d_f, d_o) < 1e-4, (s, k, rel(d_f, d_o))
            assert rel(p_f[k], orc.p[k]) < 1e-5, (s, k)


def test_shipped_configuration_unchanged(cuda_dev):
    """use_true_labels=False: the step still samples the DINO features (the label tiles are never built) and a batch
    carrying label_pos computes what it computes without it, bit for bit."""
    from stego_b200 import corr
    calls = []
    orig = corr.build_label_tiles
    corr.build_label_tiles = lambda *a, **k: calls.append(1) or orig(*a, **k)
    try:
        a, _ = make_model("vit_small", cuda_dev, fused=True)
        b, _ = make_model("vit_small", cuda_dev, fused=True)
        batch = make_batch(4, 64, cuda_dev, seed=1)
        torch.manual_seed(777)
        a.training_step(batch, 0)
        torch.manual_seed(777)
        b.training_step(dict(batch, label_pos=batch["label"].flip(-1)), 0)
        torch.cuda.synchronize()
    finally:
        corr.build_label_tiles = orig
    assert not calls
    assert a._fused.ws.ftiles.shape[-1] == a.net.n_feats and a._fused.ws.label_pos is None
    for k in a.logged:
        assert torch.equal(a.logged[k], b.logged[k]), k
