"""The cd histograms on the GPU: the generic TensorBoard histogram kernel against np.histogram on adversarial values,
the histogram variants of the correlation-loss forward against np.histogram of the cd the same launch writes, and the
training step's histogram logging (both paths), which must leave the step itself bit-for-bit unchanged."""
import types

import numpy as np
import pytest
import torch

from stego_b200 import corr, hist
from stego_b200.config import make_cfg

pytestmark = pytest.mark.gpu
SHAPES = {"c1": (32, 28, 384), "c2": (32, 40, 768), "c3": (16, 56, 768)}  # B, code side, feature channels


def _np_fields(values64: np.ndarray) -> dict:
    counts, _ = np.histogram(values64, bins=hist.default_bins())
    limits, kept = hist.trim(counts)
    return dict(min=values64.min(), max=values64.max(), num=values64.size, sum=values64.sum(),
                sum_squares=values64.dot(values64), bucket_limits=limits.tolist(), bucket_counts=kept.tolist(),
                counts=counts)


def _adversarial() -> np.ndarray:
    e = hist.default_bins()
    f = e.astype(np.float32)
    ru = np.where(f.astype(np.float64) < e, np.nextafter(f, np.float32(np.inf)), f)
    rd = np.where(f.astype(np.float64) > e, np.nextafter(f, np.float32(-np.inf)), f)
    around = np.concatenate([ru, rd, np.nextafter(ru, np.float32(-np.inf)), np.nextafter(rd, np.float32(np.inf))])
    tiny = np.float32(np.finfo(np.float32).smallest_subnormal)
    special = np.array([0.0, -0.0, tiny, -tiny, 1e-40, -1e-40, 1e-39, np.finfo(np.float32).tiny, 1e20, -1e20, 1.1e20,
                        -1.1e20, 3e38, -3e38, 1e-12, -1e-12], dtype=np.float32)
    rnd = np.random.default_rng(0).standard_normal(100_000).astype(np.float32) * 0.3
    return np.concatenate([around.astype(np.float32), special, rnd])


def test_generic_histogram_adversarial(cuda_dev):
    x = _adversarial()
    got = hist.tb_histogram(torch.from_numpy(x).to(cuda_dev))
    want = _np_fields(x.astype(np.float64))
    assert got["bucket_counts"] == want["bucket_counts"] and got["bucket_limits"] == want["bucket_limits"]
    assert got["min"] == want["min"] and got["max"] == want["max"] and got["num"] == want["num"]
    # the sum of +-3e38 and +-1e20 values cancels: its rounding error is relative to the sum of magnitudes
    x64 = x.astype(np.float64)
    assert abs(got["sum"] - want["sum"]) <= 1e-12 * np.abs(x64).sum(), (got["sum"], want["sum"])
    assert abs(got["sum_squares"] - want["sum_squares"]) <= 1e-12 * want["sum_squares"]
    # -0.0 sits with +0.0 in [0, 1e-12)
    z = hist.tb_histogram(torch.tensor([-0.0, 0.0], device=cuda_dev))
    assert z["bucket_counts"] == [0, 2] and z["bucket_limits"] == [0.0, 1e-12]


def test_generic_histogram_beyond_int32_elements(cuda_dev):
    n = (1 << 31) + 4096
    if torch.cuda.get_device_properties(cuda_dev).total_memory < 3 * n * 4:
        pytest.skip("needs ~26 GB of device memory")
    x = torch.full((n,), 0.25, device=cuda_dev)
    tail = torch.from_numpy(_adversarial()[:4096].copy())
    x[-4096:] = tail.to(cuda_dev)
    got = hist.tb_histogram(x)
    t64 = tail.numpy().astype(np.float64)
    counts, _ = np.histogram(t64, bins=hist.default_bins())
    counts[np.searchsorted(hist.default_bins(), 0.25, side="right") - 1] += n - 4096
    limits, kept = hist.trim(counts)
    assert got["bucket_counts"] == kept.tolist() and got["bucket_limits"] == limits.tolist()
    assert got["num"] == n and got["min"] == t64.min() and got["max"] == max(t64.max(), 0.25)
    s_want = t64.sum() + 0.25 * (n - 4096)
    assert abs(got["sum"] - s_want) <= 1e-12 * abs(s_want)
    del x


def _loss_inputs(B, h, E, fs, dev, seed=0, labels=False):
    cfg = make_cfg(feature_samples=fs)
    spec = corr.make_spec(cfg)
    g = torch.Generator().manual_seed(seed)
    code = torch.randn(B, 70, h, h, generator=g).to(dev)
    code_pos = (code.cpu() + 0.5 * torch.randn(B, 70, h, h, generator=g)).to(dev)
    c1 = (torch.rand(B, fs, fs, 2, generator=g) * 2 - 1).to(dev)
    c2 = (torch.rand(B, fs, fs, 2, generator=g) * 2 - 1).to(dev)
    perms = torch.stack([torch.randperm(B, generator=g) for _ in range(spec.n_neg)]).to(dev)
    if labels:
        lab = torch.randint(-1, 27, (B, 4 * h, 4 * h), generator=g).to(dev)
        lab_pos = torch.randint(-1, 27, (B, 4 * h, 4 * h), generator=g).to(dev)
        ftiles = corr.build_label_tiles(lab, lab_pos, c1, c2, perms, spec, 27, raw_perms=True)
    else:
        feats = torch.randn(B, E, h, h, generator=g).to(dev)
        feats_pos = (feats.cpu() + 0.3 * torch.randn(B, E, h, h, generator=g)).to(dev)
        ftiles = corr.build_tiles(feats, feats_pos, c1, c2, perms, spec, E, raw_perms=True)
    ctiles = corr.build_tiles(code, code_pos, c1, c2, perms, spec, corr.CODE_PAD, raw_perms=True)
    return spec, ftiles, ctiles


def _forward(spec, ftiles, ctiles, B, h_obj=None):
    dev = ftiles.device
    S = spec.fs * spec.fs
    partials, row_means = spec.scratch(B, dev)
    stats = torch.empty(spec.ncalls, 4, device=dev)
    cd = torch.empty(spec.ncalls, B, S, S, device=dev)
    fdc, elems = torch.empty_like(cd), torch.empty_like(cd)
    spec.forward(ftiles, ctiles, B, ftiles.shape[-1], 70, partials, row_means, stats, cd, fdc, elems, hist=h_obj)
    return stats, cd, fdc, elems


CASES = [("c1", 11, None, False), ("c2", 11, None, False), ("c3", 11, None, False), ("c1", 12, None, False),
         ("c1", 16, None, False), ("c3", 28, 4, False), ("c1", 64, 2, False), ("c1", 11, 1, False),
         ("c1", 28, 1, False), ("c1", 11, None, True), ("c1", 16, 8, True)]


@pytest.mark.parametrize("shape,fs,B_over,labels", CASES)
def test_loss_forward_histograms_match_cd(cuda_dev, shape, fs, B_over, labels):
    B, h, E = SHAPES[shape]
    B = B_over or B
    spec, ftiles, ctiles = _loss_inputs(B, h, E, fs, cuda_dev, labels=labels)
    plain = _forward(spec, ftiles, ctiles, B)
    hobj = hist.CdHistogram(spec, B, cuda_dev)
    with_h = _forward(spec, ftiles, ctiles, B, hobj)
    for a, b in zip(plain, with_h):
        assert torch.equal(a, b)
    torch.cuda.synchronize()
    cd = with_h[1]
    groups = [cd[0], cd[1], cd[2:]]
    counts, stats = hobj.counts.cpu().numpy(), hobj.stats.cpu().numpy()
    for g, vals in enumerate(groups):
        v = vals.reshape(-1).double().cpu().numpy()
        want = _np_fields(v)
        assert np.array_equal(counts[g], want["counts"]), (g, np.nonzero(counts[g] != want["counts"]))
        assert stats[g][0] == want["min"] and stats[g][1] == want["max"]
        assert abs(stats[g][2] - want["sum"]) <= 1e-9 * np.abs(v).sum()
        assert abs(stats[g][3] - want["sum_squares"]) <= 1e-12 * want["sum_squares"]
        assert hobj.num[g] == v.size


class _Recorder:
    def __init__(self):
        self.calls = []

    def add_histogram_raw(self, tag, **kw):
        self.calls.append((tag, kw))


def _run(fused, logger, steps, dev, hist_freq=2, sync_check_step=None):
    from _parity_util import make_batch, make_model
    model, _ = make_model("vit_small", dev, fused=fused, hist_freq=hist_freq)
    model.logger = logger
    batch = make_batch(4, 64, dev, seed=1)
    torch.manual_seed(777)
    losses = []
    for s in range(steps):
        if s == sync_check_step:
            torch.cuda.synchronize()
            torch.cuda.set_sync_debug_mode("error")
            try:
                loss = model.training_step(batch, s)
            finally:
                torch.cuda.set_sync_debug_mode(0)
        else:
            loss = model.training_step(batch, s)
        losses.append(loss.detach().clone())
    model.flush()
    rng = (torch.cuda.get_rng_state(dev).clone(), torch.get_rng_state().clone())
    params = {k: p.detach().clone() for k, p in model.named_parameters() if p.requires_grad}
    grads = {k: p.grad.detach().clone() for k, p in model.named_parameters() if p.grad is not None}
    return model, losses, params, grads, rng


@pytest.mark.parametrize("fused", [True, False])
def test_training_step_logs_histograms_without_changing_the_step(cuda_dev, fused):
    rec = _Recorder()
    model, losses, params, grads, rng = _run(fused, types.SimpleNamespace(experiment=rec), 6, cuda_dev,
                                             sync_check_step=4)
    _, losses0, params0, grads0, rng0 = _run(fused, None, 6, cuda_dev)
    assert all(torch.equal(a, b) for a, b in zip(losses, losses0))
    assert params.keys() == params0.keys() and grads.keys() == grads0.keys()
    # both probes reduce their gradients with atomics, so between any two runs their weights agree up to that order;
    # they read the detached code and feed nothing else
    for got, want in ((params, params0), (grads, grads0)):
        for k in got:
            if k.startswith(("linear_probe.", "cluster_probe.")):
                assert torch.allclose(got[k], want[k], rtol=1e-4, atol=1e-6), k
            else:
                assert torch.equal(got[k], want[k]), k
    assert torch.equal(rng[0], rng0[0]) and torch.equal(rng[1], rng0[1])
    B, S = 4, model.cfg.feature_samples ** 2
    n_neg = model.cfg.neg_samples
    assert [(t, kw["global_step"]) for t, kw in rec.calls] == [(t, s) for s in (2, 4) for t in hist.TAGS]
    nums = {"intra_cd": B * S * S, "inter_cd": B * S * S, "neg_cd": n_neg * B * S * S}
    for tag, kw in rec.calls:
        assert kw["num"] == nums[tag] and sum(kw["bucket_counts"]) == kw["num"]
    assert set(model.logged_histograms) == set(hist.TAGS)


def test_graph_capture_outlives_dead_graph_cycles(cuda_dev):
    """The test above builds two models per parameter: the previous models' graphs die in reference cycles (their
    captured closures hold the model).  If the garbage collector destroyed one while the next model captured, the
    capture would be invalidated.  _lib.Graph collects before capturing and holds automatic collection off until the
    capture ends, even when every allocation would otherwise trigger a pass."""
    import gc
    from stego_b200 import _lib
    x = torch.zeros(1024, device=cuda_dev)

    class Holder:
        pass

    for _ in range(3):
        h = Holder()
        h.self = h
        h.graph = _lib.Graph(lambda: x.add_(1.0))
        del h
    old = gc.get_threshold()
    gc.set_threshold(1, 1, 1)
    try:
        g = _lib.Graph(lambda: [x.add_(1.0) for _ in range(100)][-1])
    finally:
        gc.set_threshold(*old)
    assert gc.isenabled()
    g.replay()
    torch.cuda.synchronize()
    assert (x == 100).all()


def test_histograms_equal_the_steps_cd(cuda_dev):
    """The counts a hist step logs are np.histogram of that step's cd: recomputed by the autograd path's loss with
    want_elems on the same draws."""
    from _parity_util import make_batch, make_model
    rec = _Recorder()
    model, _ = make_model("vit_small", cuda_dev, fused=False, hist_freq=1)
    model.logger = types.SimpleNamespace(experiment=rec)
    batch = make_batch(4, 64, cuda_dev, seed=1)
    model.global_step = 1
    captured = {}
    orig = corr.corr_loss

    def spy(*a, **k):
        k2 = dict(k, want_elems=True, hist=None)
        state = (torch.cuda.get_rng_state(cuda_dev), torch.get_rng_state())
        out = orig(*a, **k)
        captured["cd"] = orig(*a, **k2)[2].detach().clone()
        torch.cuda.set_rng_state(state[0], cuda_dev)
        torch.set_rng_state(state[1])
        return out
    corr.corr_loss = spy
    try:
        torch.manual_seed(777)
        model.training_step(batch, 0)
    finally:
        corr.corr_loss = orig
    model.flush()
    cd = captured["cd"]
    for tag, vals in zip(hist.TAGS, [cd[0], cd[1], cd[2:]]):
        want = _np_fields(vals.reshape(-1).double().cpu().numpy())
        got = model.logged_histograms[tag]
        assert got["bucket_counts"] == want["bucket_counts"] and got["bucket_limits"] == want["bucket_limits"]
        assert got["min"] == want["min"] and got["max"] == want["max"]
