"""GPU: the use_salience coordinate draws on the kernel (stego_salience_coords) against torch, bit for bit.

The twin is what the autograd training step runs: ContrastiveCorrelationLoss.draw_coords with use_salience, i.e.
modules.sample_nonzero_locations with real CUDA torch.randint calls plus the reference's mixing lines, on the masks as
train_segmentation.py:147-152 prepares them (`.to(torch.float32).squeeze(1)`).  Under one seed the kernel path must
return the same bits and leave the CUDA generator in the same state.  Injected raw draws and uniforms pin the edge
values against oracle/salience_oracle.py's expressions on the same values.  The fused training step with use_salience
is checked against the autograd step (first step bit for bit; six steps of eager / capture / replay at the bars of
test_true_labels_gpu.py) and the oracle.
"""
import os
import sys
from types import SimpleNamespace

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
import salience_oracle as SO  # noqa: E402
from _parity_util import (NAMES, OracleStepper, feats_from_tokens, grads_of, make_batch, make_model, params_of,  # noqa: E402
                          rel)

pytestmark = pytest.mark.gpu

KINDS = ("sparse", "empty", "single", "full", "nan")


def _bits(t):
    return t.contiguous().view(torch.int32)


def _masks(kind, B, H, W, g):
    """fp32 [B, H, W] masks; "mixed" cycles the other kinds over the images."""
    m = (torch.rand(B, H, W, generator=g) < 0.03).float() * torch.rand(B, H, W, generator=g).add(0.25)
    for i in range(B):
        k = KINDS[i % len(KINDS)] if kind == "mixed" else kind
        if k == "empty":
            m[i] = 0
            m[i].view(-1)[:: 7] = -0.0  # -0 is not salient
        elif k == "single":
            m[i] = 0
            m[i].view(-1)[int(torch.randint(H * W, (1,), generator=g))] = 3.0
        elif k == "full":
            m[i] = torch.rand(H, W, generator=g) + 0.5
        elif k == "nan":
            m[i].view(-1)[int(torch.randint(H * W, (1,), generator=g))] = float("nan")
    return m


def _twin(sal, sal_pos, fs):
    """The autograd step's draws (segmenter._training_step_autograd + ContrastiveCorrelationLoss.draw_coords)."""
    from stego_b200 import modules
    lossfn = modules.ContrastiveCorrelationLoss(SimpleNamespace(use_salience=True, feature_samples=fs))
    prep = lambda t: (t if t.dim() == 4 else t[:, None]).to(torch.float32).squeeze(1)
    return lossfn.draw_coords(torch.empty(sal.shape[0], 1, device=sal.device), prep(sal), prep(sal_pos))


def _compare(sal, sal_pos, fs, dev, seed=777):
    from stego_b200 import salience
    torch.manual_seed(seed)
    before, before_cpu = torch.cuda.get_rng_state(dev), torch.get_rng_state()
    got = salience.salience_coords(sal, sal_pos, fs)
    after, after_cpu = torch.cuda.get_rng_state(dev), torch.get_rng_state()
    torch.cuda.set_rng_state(before, dev)
    torch.set_rng_state(before_cpu)
    want = _twin(sal, sal_pos, fs)
    assert torch.equal(torch.cuda.get_rng_state(dev), after), "CUDA generator consumption differs"
    assert torch.equal(torch.get_rng_state(), after_cpu), "CPU generator consumption differs"
    for g, w in zip(got, want):
        assert g.shape == w.shape and g.dtype == torch.float32
        assert torch.equal(_bits(g), _bits(w)), int((_bits(g) != _bits(w)).sum())
    return got


# ================================================================================================
# torch internals the kernel relies on
# ================================================================================================
def test_torch_conventions(cuda_dev):
    """fp32 `> .1` compares against 0.1f (u == 0.1f is not kept) and CUDA division by a host scalar is a multiply by
    the fp32 reciprocal; randint of range < 2^28 moves the generator offset by 4 for any size up to 2 * 64^2; the
    reference's randint for an image with nonzeros (no device argument) draws from the CPU generator."""
    u = torch.tensor([0.1], dtype=torch.float32, device=cuda_dev)
    assert not bool((u > .1).item())
    assert bool((torch.nextafter(u, torch.ones_like(u)) > .1).item())
    idx = torch.arange(1 << 12, device=cuda_dev).float()
    for H in (7, 37, 53, 224, 320, 448, 1024, 3):
        inv = torch.tensor(1.0, dtype=torch.float32) / H
        assert torch.equal(idx / H, idx * inv.to(cuda_dev)), H
    gen = torch.cuda.default_generators[cuda_dev.index]
    for n in (1, 121, 8192):
        off = gen.get_offset()
        torch.randint((1 << 28) - 1, (n,), device=cuda_dev)
        assert gen.get_offset() == off + 4, n
    from stego_b200 import modules
    cpu_state, off = torch.get_rng_state(), gen.get_offset()
    modules.sample_nonzero_locations(torch.ones(1, 4, 4, device=cuda_dev), [1, 3, 3, 2])
    assert gen.get_offset() == off and not torch.equal(torch.get_rng_state(), cpu_state)
    off = gen.get_offset()
    modules.sample_nonzero_locations(torch.zeros(1, 4, 4, device=cuda_dev), [1, 3, 3, 2])
    assert gen.get_offset() == off + 4


# ================================================================================================
# kernel vs torch
# ================================================================================================
SHAPES = [(224, 224), (320, 320), (448, 448), (37, 53), (53, 37), (1, 1), (1024, 2048)]


@pytest.mark.parametrize("hw", SHAPES, ids=[f"{h}x{w}" for h, w in SHAPES])
@pytest.mark.parametrize("kind", KINDS + ("mixed",))
def test_maps_and_mask_kinds(cuda_dev, hw, kind):
    H, W = hw
    g = torch.Generator().manual_seed(H * 7 + W)
    B = 2 if H * W > 1 else 3
    sal, sal_pos = _masks(kind, B, H, W, g).to(cuda_dev), _masks("mixed", B, H, W, g).to(cuda_dev)
    _compare(sal, sal_pos, 11, cuda_dev)


@pytest.mark.parametrize("fs", [1, 11, 12, 28, 64])
@pytest.mark.parametrize("B", [1, 2, 32])
def test_batch_sizes_and_feature_samples(cuda_dev, B, fs):
    g = torch.Generator().manual_seed(100 * B + fs)
    sal, sal_pos = _masks("mixed", B, 224, 224, g).to(cuda_dev), _masks("sparse", B, 224, 224, g).to(cuda_dev)
    _compare(sal, sal_pos, fs, cuda_dev, seed=fs)


@pytest.mark.parametrize("dtype", [torch.float32, torch.uint8, torch.bool, torch.float16, torch.int64],
                         ids=["fp32", "uint8", "bool", "fp16", "int64"])
@pytest.mark.parametrize("layout", ["BHW", "B1HW"])
def test_mask_dtypes_and_views(cuda_dev, dtype, layout):
    g = torch.Generator().manual_seed(3)
    B, H, W = 4, 37, 53
    sal, sal_pos = _masks("mixed", B, H, W, g), _masks("sparse", B, H, W, g)
    if dtype != torch.float32:
        sal, sal_pos = torch.nan_to_num(sal, nan=1.0), torch.nan_to_num(sal_pos, nan=1.0)
        sal, sal_pos = (sal != 0).to(dtype), (sal_pos != 0).to(dtype)
    sal, sal_pos = sal.to(cuda_dev), sal_pos.to(cuda_dev)
    if layout == "B1HW":
        sal, sal_pos = sal[:, None], sal_pos[:, None]
    _compare(sal, sal_pos, 16, cuda_dev)
    # a [B, 1, H, W] view of a wider buffer (non-contiguous) gives the same answer
    wide = torch.zeros(B, 2, H, W, dtype=sal.dtype, device=cuda_dev)
    wide[:, 1] = sal.reshape(B, H, W)
    _compare(wide[:, 1:], sal_pos, 16, cuda_dev)


def test_mixed_mask_byte_widths(cuda_dev):
    g = torch.Generator().manual_seed(4)
    sal = _masks("mixed", 3, 20, 30, g).to(cuda_dev)
    _compare(sal, (_masks("sparse", 3, 20, 30, g) != 0).to(cuda_dev), 11, cuda_dev)


# ================================================================================================
# injected edge values
# ================================================================================================
def _prep(m):
    from stego_b200 import salience
    return salience.mask_view(m)


@pytest.mark.parametrize("hw", [(12, 12), (9, 17), (19, 7), (1, 1)], ids=["12x12", "9x17", "19x7", "1x1"])
def test_injected_draws_and_uniforms(cuda_dev, hw):
    """Raw draws 0, 2^32 - 1, multiples of the count and their neighbours; keep uniforms 0.1f and the floats around
    it, 0 and just below 1; reg uniforms 0.5 (reg = +0), 0, and values whose products are -0."""
    from stego_b200 import salience
    H, W = hw
    fs, B = 11, 4
    n = fs * fs
    g = torch.Generator().manual_seed(H + W)
    sal = _masks("mixed", B, H, W, g)
    sal_pos = _masks("sparse", B, H, W, g)
    sal_pos[1] = 1.0
    counts = [int((m[i] != 0).sum()) for m in (sal, sal_pos) for i in range(B)]
    draws = torch.randint(0, 1 << 32, (2 * B, 2 * n), generator=g, dtype=torch.int64)
    for u, c in enumerate(counts):
        mod = c if c > 0 else H
        edge = [0, (1 << 32) - 1, (1 << 32) - 2, mod, 2 * mod, mod - 1, mod + 1, ((1 << 32) // mod) * mod,
                ((1 << 32) // mod) * mod - 1, (1 << 31), (1 << 31) - 1]
        draws[u, :len(edge)] = torch.tensor(edge) % (1 << 32)
        draws[u, n:n + len(edge)] = torch.tensor(edge) % (1 << 32)
    f01 = torch.tensor(0.1, dtype=torch.float32)
    keep_vals = torch.stack([f01, torch.nextafter(f01, torch.tensor(0.0)), torch.nextafter(f01, torch.tensor(1.0)),
                             torch.tensor(0.0), torch.nextafter(torch.tensor(1.0), torch.tensor(0.0))])
    reg_vals = torch.tensor([0.5, 0.0, 0.25, 0.75, 0.49999997, 0.50000006, 0.9999999], dtype=torch.float32)
    ukeep = torch.rand(B, fs, fs, generator=g)
    ukeep.view(-1)[:len(keep_vals) * 9] = keep_vals.repeat(9)
    ureg1, ureg2 = torch.rand(B, fs, fs, 2, generator=g), torch.rand(B, fs, fs, 2, generator=g)
    ureg1.view(-1)[:70] = reg_vals.repeat(10)
    ureg2.view(-1)[-70:] = reg_vals.repeat(10)
    d = lambda t: t.to(cuda_dev)
    m1, nb = _prep(d(sal))
    m2, _ = _prep(d(sal_pos))
    out1, out2 = torch.full((B, fs, fs, 2), 7.0, device=cuda_dev), torch.full((B, fs, fs, 2), 7.0, device=cuda_dev)
    draws32 = d(torch.where(draws >= 1 << 31, draws - (1 << 32), draws).to(torch.int32))  # the uint32 bits
    salience.launch(m1, m2, nb, fs, 0, None, draws32, d(ureg1), d(ureg2), d(ukeep), out1, out2)
    nz1 = SO.nonzero_locations_from_draws(d(sal), fs, d(draws[:B]))
    nz2 = SO.nonzero_locations_from_draws(d(sal_pos), fs, d(draws[B:]))
    w1, w2 = SO.mix(nz1, nz2, d(ureg1), d(ureg2), d(ukeep))
    assert torch.equal(_bits(out1), _bits(w1)) and torch.equal(_bits(out2), _bits(w2))
    zeros = torch.cat([w1.reshape(-1), w2.reshape(-1)])
    zeros = zeros[zeros == 0]
    assert zeros.numel() > 0 and not bool(torch.signbit(zeros).any())  # mixing never leaves a -0 behind


# ================================================================================================
# other properties
# ================================================================================================
def test_reruns_bit_identical_and_one_host_wait(cuda_dev):
    """Same seed, same bits; the kernel path waits for the device once (the counts), the torch path 2B + 2 times."""
    import warnings
    from stego_b200 import salience
    g = torch.Generator().manual_seed(9)
    for H, W, B in ((224, 224, 32), (1024, 2048, 1)):
        sal, sal_pos = _masks("mixed", B, H, W, g).to(cuda_dev), _masks("sparse", B, H, W, g).to(cuda_dev)
        salience.salience_coords(sal, sal_pos, 11)  # first call: pinned host buffers are allocated
        torch.cuda.synchronize()
        outs, waits = [], []
        for fn in (lambda: salience.salience_coords(sal, sal_pos, 11), lambda: salience.salience_coords(sal, sal_pos, 11),
                   lambda: _twin(sal, sal_pos, 11)):
            torch.manual_seed(11)
            with warnings.catch_warnings(record=True) as rec:
                warnings.simplefilter("always")
                torch.cuda.set_sync_debug_mode("warn")
                try:
                    outs.append(fn())
                finally:
                    torch.cuda.set_sync_debug_mode(0)
            waits.append(sum("synchroniz" in str(w.message) for w in rec))
        for a, b in zip(*outs[:2]):
            assert torch.equal(_bits(a), _bits(b))
        # one wait for the counts; a call that grows the pinned host pool for its draw upload may add one
        assert min(waits[:2]) == 1 and max(waits[:2]) <= 2 and waits[2] >= 2 * B, waits


def test_sentinels_outside_outputs_survive(cuda_dev):
    from stego_b200 import salience
    g = torch.Generator().manual_seed(10)
    B, H, W, fs = 3, 1024, 2048, 11
    sal, sal_pos = _masks("mixed", B, H, W, g).to(cuda_dev), _masks("sparse", B, H, W, g).to(cuda_dev)
    m1, nb = _prep(sal)
    m2, _ = _prep(sal_pos)
    n = B * fs * fs * 2
    sentinel = -123.25
    buf = torch.full((3 * n + 64,), sentinel, device=cuda_dev)
    out1, out2 = buf[16:16 + n].view(B, fs, fs, 2), buf[32 + n:32 + 2 * n].view(B, fs, fs, 2)
    ur1, ur2, uk = torch.rand(B, fs, fs, 2, device=cuda_dev), torch.rand(B, fs, fs, 2, device=cuda_dev), \
        torch.rand(B, fs, fs, device=cuda_dev)
    scratch = salience.scratch_for(B, H, W, cuda_dev)
    assert scratch is not None
    big = torch.full((scratch.numel() + 128,), -7, dtype=torch.int32, device=cuda_dev)
    draws = torch.randint(0, 1 << 20, (2 * B, 2 * fs * fs), dtype=torch.int32, device=cuda_dev)
    offsets = torch.arange(0, 8 * B, 4, dtype=torch.int64, device=cuda_dev)
    salience.launch(m1, m2, nb, fs, 5, offsets, draws, ur1, ur2, uk, out1, out2, scratch=big[64:64 + scratch.numel()])
    torch.cuda.synchronize()
    keep = torch.ones_like(buf, dtype=torch.bool)
    keep[16:16 + n] = False
    keep[32 + n:32 + 2 * n] = False
    assert bool((buf[keep] == sentinel).all())
    assert bool((out1 != sentinel).all()) and bool((out2 != sentinel).all())
    assert bool((big[:64] == -7).all()) and bool((big[64 + scratch.numel():] == -7).all())


def test_wrapper_refuses_mismatched_masks(cuda_dev):
    from stego_b200 import salience
    a = torch.ones(2, 8, 8, device=cuda_dev)
    with pytest.raises(ValueError, match="expected 2 masks|differ"):
        salience.salience_coords(a, torch.ones(3, 8, 8, device=cuda_dev), 11)
    with pytest.raises(ValueError, match="differ"):
        salience.salience_coords(a, torch.ones(2, 8, 9, device=cuda_dev), 11)
    with pytest.raises(RuntimeError, match="CUDA"):
        salience.salience_coords(a, torch.ones(2, 8, 8), 11)


# ================================================================================================
# the fused training step
# ================================================================================================
def _sal_batch(B, res, dev, seed, dtype=torch.float32):
    b = make_batch(B, res, dev, seed=seed)
    g = torch.Generator().manual_seed(seed + 70)
    m, mp = _masks("mixed", B, res, res, g), _masks("sparse", B, res, res, g)
    if dtype != torch.float32:
        m, mp = (torch.nan_to_num(m, nan=1.0) != 0).to(dtype), (mp != 0).to(dtype)
    b["mask"], b["mask_pos"] = m[:, None].to(dev), mp[:, None].to(dev)
    b["label_pos"] = torch.randint(-1, 27, (B, res, res), generator=g).to(dev)
    return b


def _peek(model, batch, B, dev):
    """The next step's draws with use_salience: noises of net(img) and net(img_pos), the salience coordinates from
    the autograd step's own code, the raw permutations' fix-up (super_perm); both generators are put back."""
    from stego_b200.modules import super_perm
    st, st_cpu = torch.cuda.get_rng_state(dev), torch.get_rng_state()
    m, mp = model.net.draw_masks(B, dev), model.net.draw_masks(B, dev)
    c1, c2 = _twin(batch["mask"], batch["mask_pos"], model.cfg.feature_samples)
    perms = [super_perm(B, dev) for _ in range(model.cfg.neg_samples)]
    torch.cuda.set_rng_state(st, dev)
    torch.set_rng_state(st_cpu)
    return m, mp, c1, c2, perms


@pytest.mark.parametrize("variant", ["feat", "uint8_mask", "true_labels", "KK"])
def test_first_step_fused_and_autograd_bit_equal(cuda_dev, variant):
    over = dict(use_salience=True)
    if variant == "true_labels":
        over["use_true_labels"] = True
    if variant == "KK":
        over["dino_feat_type"] = "KK"
    fused, _ = make_model("vit_small", cuda_dev, fused=True, **over)
    twin, _ = make_model("vit_small", cuda_dev, fused=False, **over)
    batch = _sal_batch(4, 64, cuda_dev, seed=1, dtype=torch.uint8 if variant == "uint8_mask" else torch.float32)
    torch.manual_seed(777)
    _, _, c1, c2, _ = _peek(fused, batch, 4, cuda_dev)
    gpu_state, cpu_state = torch.cuda.get_rng_state(cuda_dev), torch.get_rng_state()
    fused.training_step(batch, 0)
    after, after_cpu = torch.cuda.get_rng_state(cuda_dev), torch.get_rng_state()
    torch.cuda.set_rng_state(gpu_state, cuda_dev)
    torch.set_rng_state(cpu_state)
    twin.training_step(batch, 0)
    assert fused._fused.step_idx == 1 and twin._fused is None
    assert torch.equal(torch.cuda.get_rng_state(cuda_dev), after) and torch.equal(torch.get_rng_state(), after_cpu)
    torch.cuda.synchronize()
    assert torch.equal(_bits(fused._fused.ws.c1), _bits(c1)) and torch.equal(_bits(fused._fused.ws.c2), _bits(c2))
    for key in ("loss/pos_intra", "loss/pos_inter", "cd/pos_intra", "cd/pos_inter", "loss/cluster"):
        assert torch.equal(fused.logged[key], twin.logged[key]), (key, fused.logged[key].item(),
                                                                  twin.logged[key].item())


def test_unsupported_masks_take_the_autograd_path(cuda_dev):
    from stego_b200.fused_step import FusedStep
    model, _ = make_model("vit_small", cuda_dev, fused=True, use_salience=True)
    fs = FusedStep(model)
    batch = _sal_batch(2, 64, cuda_dev, seed=1)
    assert fs.supported(batch)
    assert not fs.supported({k: v for k, v in batch.items() if k != "mask_pos"})
    assert not fs.supported(dict(batch, mask=batch["mask"].cpu()))
    assert not fs.supported(dict(batch, mask_pos=batch["mask_pos"][:, :, :32]))
    assert not fs.supported(dict(batch, mask=batch["mask"][:1], mask_pos=batch["mask_pos"][:1]))


def _check_losses(model, loss, out, tol=1e-3):
    logged = {k: float(v) for k, v in model.logged.items()}
    elem_scale = 0.05
    assert abs(logged["loss/linear"] - out["linear"].item()) < 1e-4 * abs(out["linear"].item()) + 1e-6
    assert abs(logged["loss/cluster"] - out["cluster"].item()) < 2e-4 * abs(out["cluster"].item()) + 1e-6
    for k_log, k_or in [("loss/pos_intra", "pos_intra"), ("loss/pos_inter", "pos_inter"), ("loss/neg_inter", "neg_inter")]:
        assert abs(logged[k_log] - out[k_or].item()) < tol * abs(out[k_or].item()) + tol * elem_scale, \
            (k_log, logged[k_log], out[k_or].item())
    assert abs(float(loss) - out["total"].item()) < tol * abs(out["total"].item())


@pytest.mark.parametrize("reset_at", [None, 2], ids=["plain", "reset_probe_steps=2"])
def test_multistep_graph_replay_vs_autograd_vs_oracle(cuda_dev, reset_at):
    """test_step_parity_gpu.py's six-step procedure (eager, capture, 4 replays; batches alternating) with
    use_salience, at test_true_labels_gpu.py's bars, against oracle/stego_oracle.py on the peeked draws."""
    arch, res, B, nsteps = "vit_small", 64, 4, 6
    fused, _ = make_model(arch, cuda_dev, fused=True, reset_probe_steps=reset_at, use_salience=True)
    twin, _ = make_model(arch, cuda_dev, fused=False, reset_probe_steps=reset_at, use_salience=True)
    batches = [_sal_batch(B, res, cuda_dev, seed=1), _sal_batch(B, res, cuda_dev, seed=2)]
    orc = OracleStepper(params_of(fused), "cpu")
    h = res // 8
    torch.manual_seed(777)
    for s in range(nsteps):
        batch = batches[s % 2]
        draws = _peek(fused, batch, B, cuda_dev)
        gpu_state, cpu_state = torch.cuda.get_rng_state(cuda_dev), torch.get_rng_state()
        p_before = params_of(fused)
        loss = fused.training_step(batch, s)
        g_f, p_f = grads_of(fused), params_of(fused)
        after_state, after_cpu = torch.cuda.get_rng_state(cuda_dev), torch.get_rng_state()
        assert torch.equal(_bits(fused._fused.ws.c1), _bits(draws[2])), s
        torch.cuda.set_rng_state(gpu_state, cuda_dev)
        torch.set_rng_state(cpu_state)
        loss_t = twin.training_step(batch, s)
        g_t, p_t = grads_of(twin), params_of(twin)
        assert torch.equal(torch.cuda.get_rng_state(cuda_dev), after_state), f"step {s}: RNG consumption differs"
        assert torch.equal(torch.get_rng_state(), after_cpu), f"step {s}: CPU RNG consumption differs"
        assert fused._fused.step_idx == s + 1 and twin._fused is None
        if s >= 2:
            assert fused._fused.ws.graph is not None
        assert abs(float(loss) - float(loss_t)) < 2e-5 * abs(float(loss_t)), (s, float(loss), float(loss_t))
        for k in NAMES:
            assert rel(g_f[k], g_t[k]) < 3e-3, (s, k, rel(g_f[k], g_t[k]))
            assert rel(p_f[k], p_t[k]) < 2e-4, (s, k, rel(p_f[k], p_t[k]))
        with torch.no_grad():
            tok = fused.net.backbone_tokens(torch.cat([batch["img"], batch["img_pos"]], 0)).float().cpu()
        out = orc.losses(feats_from_tokens(tok, 2 * B, h, h), B, batch["label"].cpu(), draws)
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


def test_histogram_step_with_salience(cuda_dev):
    """Histogram-logging steps (hist_freq) read the same coordinates: fused and autograd log equal losses."""
    models = []
    for fused in (True, False):
        m, _ = make_model("vit_small", cuda_dev, fused=fused, use_salience=True, hist_freq=1)
        m.logger = SimpleNamespace(experiment=SimpleNamespace(add_histogram_raw=lambda *a, **k: None))
        models.append(m)
    batch = _sal_batch(4, 64, cuda_dev, seed=3)
    torch.manual_seed(5)
    for s in range(2):  # step 1 logs histograms (global_step > 0)
        st, st_cpu = torch.cuda.get_rng_state(cuda_dev), torch.get_rng_state()
        models[0].training_step(batch, s)
        after = torch.cuda.get_rng_state(cuda_dev)
        torch.cuda.set_rng_state(st, cuda_dev)
        torch.set_rng_state(st_cpu)
        models[1].training_step(batch, s)
        assert torch.equal(torch.cuda.get_rng_state(cuda_dev), after)
        torch.cuda.synchronize()
        assert models[0]._fused.ws.hist is not None or s == 0
        for key in ("loss/pos_intra", "loss/pos_inter", "cd/pos_intra", "cd/pos_inter"):
            assert torch.equal(models[0].logged[key], models[1].logged[key]), (s, key)


def test_shipped_configuration_unchanged(cuda_dev):
    """use_salience=False: a batch carrying masks computes what it computes without them, bit for bit, and the
    salience kernel is never called."""
    from stego_b200 import salience
    calls = []
    orig = salience.launch
    salience.launch = lambda *a, **k: calls.append(1) or orig(*a, **k)
    try:
        a, _ = make_model("vit_small", cuda_dev, fused=True)
        b, _ = make_model("vit_small", cuda_dev, fused=True)
        batch = make_batch(4, 64, cuda_dev, seed=1)
        sb = _sal_batch(4, 64, cuda_dev, seed=1)
        torch.manual_seed(777)
        a.training_step(batch, 0)
        torch.manual_seed(777)
        b.training_step(dict(batch, mask=sb["mask"], mask_pos=sb["mask_pos"]), 0)
        torch.cuda.synchronize()
    finally:
        salience.launch = orig
    assert not calls
    assert a._fused.ws.keep is None and b._fused.ws.keep is None
    for k in a.logged:
        assert torch.equal(a.logged[k], b.logged[k]), k
