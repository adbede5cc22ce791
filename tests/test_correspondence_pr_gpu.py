"""Correspondence precision-recall on the GPU (stego_b200/correspondence.py, corr_loss.cu: sample_label_ids_kernel and
corr_kernel<CP_PR>).

  * label ids bit-equal to a torch restatement of the pure-class rule on make_taps' own fp32 taps;
  * pair counts against fp64 scores of the same samples (tests/_corr_fp64.py), binned by the same rule: totals exact,
    and at every bin edge the cumulative counts differ by at most the number of elements whose fp64 score lies within
    its bar (the fd / cd bars of tests/test_corr_fp64_gpu.py, plus the rounding of score + 1) of that edge;
  * streaming (two updates = one update of the concatenated batch), reset, run-to-run identical counts;
  * the exact-rule AP of the reference's fd (tests/golden/correspondence_pr.pt) inside the kernel's ap_bounds;
  * LitUnsupervisedSegmenter.correspondence_pr_step: the featurizer's outputs, the reference's two coordinate draws,
    and no effect on training.
"""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import _corr_fp64 as R  # noqa: E402
from _parity_util import make_batch, make_model  # noqa: E402

pytestmark = pytest.mark.gpu
NB = 4096
SHAPES = {"c1": (32, 28, 384), "c2": (32, 40, 768), "c3": (16, 56, 768)}
D = 70


def _metric(n, dev):
    from stego_b200.correspondence import CorrespondencePR
    return CorrespondencePR(n, dev)


# ---------------------------------------------------------------------------------------------------------------------
# label ids
# ---------------------------------------------------------------------------------------------------------------------
def ref_ids(label, n, coords):
    """[B, S] pure class of each sample (label + 1 for 0 <= label < n, else 0) or -1, on make_taps' fp32 taps."""
    B, H, W = label.shape
    idx, w = R.taps(coords, H, W)
    lab = label.reshape(B, -1).long()
    cls = torch.where((lab >= 0) & (lab < n), lab + 1, torch.zeros_like(lab))
    tc = cls.gather(1, idx.reshape(B, -1)).reshape(idx.shape)
    nz = w != 0
    mx = torch.where(nz, tc, torch.full_like(tc, -5)).max(-1).values
    mn = torch.where(nz, tc, torch.full_like(tc, 1 << 20)).min(-1).values
    return torch.where((mx == mn) & nz.any(-1), mx, torch.full_like(mx, -1))


def _kernel_ids(label, n, c1, c2, fs):
    from stego_b200 import _lib, ops
    B, H, W = label.shape
    S = fs * fs
    Rr = -(-S // 128) * 128
    lab, nbytes = ops.probe_label(label, B, H, W)
    ids = torch.full((2, B, Rr), -7, dtype=torch.int32, device=label.device)
    _lib.check(_lib.load().stego_sample_label_ids(_lib.ptr(lab), nbytes, _lib.ptr(c1), _lib.ptr(c2), _lib.ptr(ids), B,
                                                  n, H, W, fs, _lib.stream()), "stego_sample_label_ids")
    assert bool((ids[:, :, S:] == -7).all())  # rows >= S untouched
    return ids[:, :, :S]


def label_seed(dtype):
    return {torch.int64: 0, torch.int32: 100, torch.uint8: 200}[dtype]


def region_labels(B, H, W, n, g, lo=-1, cells=(5, 7)):
    small = torch.randint(lo, n, (B,) + cells, generator=g)
    ys = torch.arange(H) * cells[0] // H
    xs = torch.arange(W) * cells[1] // W
    return small[:, ys][:, :, xs].contiguous()


@pytest.mark.parametrize("fs", [1, 11, 12, 28, 64])
@pytest.mark.parametrize("dtype,kind", [(torch.int64, "region"), (torch.int32, "pixel"), (torch.uint8, "pixel"),
                                        (torch.int64, "grid")])
def test_label_ids_match_rule(cuda_dev, fs, dtype, kind):
    g = torch.Generator().manual_seed(fs * 7 + {"region": 1, "pixel": 2, "grid": 3}[kind] + label_seed(dtype))
    B, H, W, n = 3, 40, 56, 6
    if kind == "region":
        label = region_labels(B, H, W, n, g)
    else:
        label = torch.randint(-1, n + 3, (B, H, W), generator=g)
        if dtype == torch.uint8:
            label = torch.where(label < 0, torch.full_like(label, 255), label)
    label = label.to(dtype)
    if kind == "grid":
        c1, c2 = R.centre_grid(B, fs, H, W, g), R.centre_grid(B, fs, H, W, g, last=True)
        c2.view(B, -1, 2)[:, :1] = torch.tensor([-1.0, 1.0])  # an exact corner
    else:
        c1 = (torch.rand(B, fs, fs, 2, generator=g) * 2 - 1) * 1.2  # some beyond +-1
        c2 = (torch.rand(B, fs, fs, 2, generator=g) * 2 - 1) * 1.2
    label, c1, c2 = label.to(cuda_dev), c1.to(cuda_dev), c2.to(cuda_dev)
    got = _kernel_ids(label, n, c1, c2, fs)
    for slot, c in enumerate((c1, c2)):
        want = ref_ids(label, n, c).to(torch.int32)
        assert torch.equal(got[slot], want), (slot, int((got[slot] != want).sum()))
    if kind in ("region", "grid"):
        assert bool((got >= 0).any()) and (kind == "grid" or bool((got < 0).any()))


# ---------------------------------------------------------------------------------------------------------------------
# counts against fp64
# ---------------------------------------------------------------------------------------------------------------------
def _normed(src, coords, L):
    B, C, H, W = src.shape
    idx, w = R.taps(coords, H, W)
    v, A = R.gather_sample(src, torch.arange(B, device=src.device), idx, w)
    n, E, _ = R.normalise(v, A, L)
    return n, E


def fp64_check(feats, code, label, n_cls, c1, c2, counts):
    """Assert the kernel's counts [2][2][NB] against fp64 binning of the same pairs; returns the largest number of
    ambiguous elements at one edge (for the log)."""
    from stego_b200.corr import teacher_width
    B, fs = c1.shape[0], c1.shape[1]
    pos_all = []
    id1, id2 = ref_ids(label, n_cls, c1), ref_ids(label, n_cls, c2)
    worst = 0
    for m, src, K in ((0, feats, 3 * teacher_width(feats.shape[1])), (1, code, 3 * R.TILE)):
        C = src.shape[1]
        L = max(R.chain_norm(C), R.chain_norm(C, vec8=True))
        n1, E1 = _normed(src, c1, L)
        n2, E2 = _normed(src, c2, L)
        want = torch.zeros(2, NB, dtype=torch.int64, device=src.device)
        amb = torch.zeros(2, NB + 1, dtype=torch.int64, device=src.device)
        for b in range(B):
            a, bb = n1[b], n2[b]
            val = a @ bb.T
            bar = (E1[b] + R.SPLIT * a.abs()) @ bb.abs().T + a.abs() @ (E2[b] + R.SPLIT * bb.abs()).T + \
                (R.SPLIT + (K + 2) * R.U) * (a.abs() @ bb.abs().T) + 4 * R.U
            pos = ((id1[b][:, None] == id2[b][None, :]) & (id1[b][:, None] >= 0)).long().reshape(-1)
            k = torch.clamp(torch.floor((val + 1) * (NB // 2)), 0, NB - 1).long().reshape(-1)
            want.view(-1).index_add_(0, pos * NB + k, torch.ones_like(k))
            lo = torch.clamp(torch.ceil((val - bar + 1) * (NB // 2)), 1, NB).long().reshape(-1)
            hi = torch.clamp(torch.floor((val + bar + 1) * (NB // 2)), 0, NB - 1).long().reshape(-1)
            ok = lo <= hi
            one = torch.ones_like(lo[ok])
            amb.view(-1).index_add_(0, pos[ok] * (NB + 1) + lo[ok], one)
            amb.view(-1).index_add_(0, pos[ok] * (NB + 1) + hi[ok] + 1, -one)
            del val, bar
        amb = amb[:, :NB].cumsum(1)  # amb[:, e] = elements within their bar of edge e (between bins e - 1 and e)
        got = counts[m]
        assert torch.equal(got.sum(1), want.sum(1)), (m, got.sum(1).tolist(), want.sum(1).tolist())
        assert int(got.sum()) == B * fs ** 4
        cg = torch.cat([torch.zeros(2, 1, dtype=torch.int64, device=got.device), got.cumsum(1)[:, :-1]], 1)
        cw = torch.cat([torch.zeros(2, 1, dtype=torch.int64, device=got.device), want.cumsum(1)[:, :-1]], 1)
        bad = (cg - cw).abs() > amb
        assert not bool(bad.any()), (m, bad.nonzero()[:5].tolist())
        worst = max(worst, int(amb.max()))
        pos_all.append(int(want[1].sum()))
    assert pos_all[0] == pos_all[1]
    return worst


def _run_case(dev, feats, code, label, n, c1, c2):
    met = _metric(n, dev)
    met.update(feats, code, label, c1, c2)
    return fp64_check(feats.float(), code.float(), label, n, c1, c2, met.counts)


@pytest.mark.parametrize("shape", list(SHAPES))
def test_counts_fp64_production_shapes(cuda_dev, shape):
    B, h, E = SHAPES[shape]
    x = R.make_inputs("corr", B, E, D, h, h, 11, 0, seed=3)
    g = torch.Generator().manual_seed(4)
    label = region_labels(B, 8 * h, 8 * h, 27, g, cells=(6, 6)).to(cuda_dev)
    feats = x["feats"].to(cuda_dev).to(torch.bfloat16).permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
    w = _run_case(cuda_dev, feats, x["code"].to(cuda_dev), label, 27, x["coords1"].to(cuda_dev),
                  x["coords2"].to(cuda_dev))
    print(f"{shape}: most ambiguous elements at one edge {w}")


@pytest.mark.parametrize("fs,B", [(12, 4), (28, 3), (56, 2), (64, 2)])
def test_counts_fp64_multi_tile(cuda_dev, fs, B):
    x = R.make_inputs("corr", B, 384, D, 28, 28, fs, 0, seed=fs)
    g = torch.Generator().manual_seed(fs)
    label = region_labels(B, 224, 224, 27, g, cells=(4, 4)).to(cuda_dev)
    d = {k: (v.to(cuda_dev) if torch.is_tensor(v) else v) for k, v in x.items()}
    _run_case(cuda_dev, d["feats"], d["code"], label, 27, d["coords1"], d["coords2"])


@pytest.mark.parametrize("regime,fs,B", [("kinks", 11, 4), ("kinks", 28, 2), ("flat", 11, 4), ("zeros", 11, 4),
                                         ("zeros", 20, 2), ("corr", 11, 1), ("corr", 40, 1)])
def test_counts_fp64_regimes(cuda_dev, regime, fs, B):
    """kinks: one-hot codes at pixel centres (scores exactly 0 and 1: the top-bin clamp); flat: every feature one
    direction (fd ~ 1); zeros: zero code and feature vectors (score 0); B = 1."""
    x = R.make_inputs(regime, B, 128, D, 14, 14, fs, 0, seed=5)
    g = torch.Generator().manual_seed(6)
    label = region_labels(B, 14, 14, 4, g, cells=(3, 3)).to(cuda_dev)
    d = {k: (v.to(cuda_dev) if torch.is_tensor(v) else v) for k, v in x.items()}
    met = _metric(4, cuda_dev)
    met.update(d["feats"], d["code"], label, d["coords1"], d["coords2"])
    fp64_check(d["feats"], d["code"], label, 4, d["coords1"], d["coords2"], met.counts)
    if regime == "kinks":
        assert int(met.counts[1, :, NB - 1].sum()) > 0 and int(met.counts[1, :, NB // 2].sum()) > 0


@pytest.mark.parametrize("layout", ["fp32_nchw", "fp32_cl", "bf16_nchw", "bf16_cl"])
def test_counts_fp64_layouts(cuda_dev, layout):
    B, fs = 3, 16
    x = R.make_inputs("corr", B, 384, D, 20, 20, fs, 0, seed=8)
    feats = x["feats"].to(cuda_dev)
    code = x["code"].to(cuda_dev)
    if layout.startswith("bf16"):
        feats = feats.to(torch.bfloat16)
    if layout.endswith("_cl"):
        feats = feats.contiguous(memory_format=torch.channels_last)
        code = code.contiguous(memory_format=torch.channels_last)
    label = region_labels(B, 160, 160, 27, torch.Generator().manual_seed(9)).to(torch.int32).to(cuda_dev)
    _run_case(cuda_dev, feats, code, label, 27, x["coords1"].to(cuda_dev), x["coords2"].to(cuda_dev))


# ---------------------------------------------------------------------------------------------------------------------
# streaming, reset, reproducibility
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fs", [11, 28])
def test_streaming_reset_reproducible(cuda_dev, fs):
    B = 6
    x = R.make_inputs("corr", B, 384, D, 28, 28, fs, 0, seed=12)
    d = {k: (v.to(cuda_dev) if torch.is_tensor(v) else v) for k, v in x.items()}
    label = region_labels(B, 224, 224, 27, torch.Generator().manual_seed(13)).to(cuda_dev)
    args = (d["feats"], d["code"], label, d["coords1"], d["coords2"])
    whole = _metric(27, cuda_dev)
    whole.update(*args)
    parts = _metric(27, cuda_dev)
    parts.update(*(a[:2] for a in args))
    parts.update(*(a[2:] for a in args))
    assert torch.equal(whole.counts, parts.counts)
    again = _metric(27, cuda_dev)
    again.update(*args)
    assert torch.equal(whole.counts, again.counts)
    whole.reset()
    assert int(whole.counts.abs().sum()) == 0
    whole.update(*args)
    assert torch.equal(whole.counts, again.counts)
    r = again.compute()
    assert sorted(r) == ["code", "feats"]
    assert r["code"]["num_pairs"] == B * fs ** 4


# ---------------------------------------------------------------------------------------------------------------------
# golden fixture: the reference's fd, exact-rule AP
# ---------------------------------------------------------------------------------------------------------------------
def test_golden_ap_within_bounds(cuda_dev):
    sys.path.insert(0, os.path.join(os.path.dirname(HERE), "oracle"))
    import correspondence_oracle as CO
    g = CO.load_golden(os.path.join(HERE, "golden", "correspondence_pr.pt"))
    met = _metric(g["n_classes"], cuda_dev)
    met.update(*(g[k].to(cuda_dev) for k in ("feats", "code", "label", "coords1", "coords2")))
    r = met.compute()
    n_pos = int(CO.exact_targets(g["label"], g["n_classes"], g["coords1"], g["coords2"]).sum())
    for m in ("code", "feats"):
        lo, hi = r[m]["ap_bounds"]
        want = g["ap_exact"][m]
        dist = max(lo - want, want - hi, 0.0)
        print(f"{m}: exact-rule AP {want:.6f}, bounds [{lo:.6f}, {hi:.6f}], ap {r[m]['ap']:.6f}, outside by {dist:.2e}; "
              f"reference AP {g['ap_reference'][m]:.6f}")
        assert lo - 1e-4 <= want <= hi + 1e-4
        assert r[m]["num_pos"] == n_pos
        assert r[m]["num_pairs"] == g["label"].shape[0] * g["coords1"].shape[1] ** 4


# ---------------------------------------------------------------------------------------------------------------------
# LitUnsupervisedSegmenter.correspondence_pr_step
# ---------------------------------------------------------------------------------------------------------------------
def _train_state(model, dev):
    model.flush()
    torch.cuda.synchronize()
    f = model._flat
    return dict(param=f.param.clone(), grad=f.grad.clone(), exp_avg=f.exp_avg.clone(), exp_avg_sq=f.exp_avg_sq.clone(),
                cpu_rng=torch.get_rng_state(), cuda_rng=torch.cuda.get_rng_state(dev),
                adam_steps=torch.tensor([o.steps for o in f.optimizers]))


def test_correspondence_pr_step(cuda_dev):
    """ViT-S/8 at 224 px, B = 8: the counts equal `update` on the featurizer's own outputs with the coordinates of the
    reference's two torch.rand draws; the step consumes exactly those draws and changes nothing else of the training
    state; and a training step after it (from the same RNG state) matches one without it."""
    dev = cuda_dev
    steps = [make_batch(8, 224, dev, seed=20 + i) for i in range(2)]
    val = make_batch(8, 224, dev, seed=60)

    def run(with_pr):
        model, _ = make_model("vit_small", dev, fused=True, seed=0)
        torch.manual_seed(777)
        losses = [model.training_step(steps[0], 0).item()]
        if with_pr:
            fused = model._fused
            graph, key = fused.ws.graph, fused.key
            before = _train_state(model, dev)
            modes = [m.training for m in model.modules()]
            seen = []
            fwd = model.net.forward

            def rec(img, *a, **k):
                out = fwd(img, *a, **k)
                seen.append((out[0].detach().clone(), out[1].detach().clone()))
                return out
            model.net.forward = rec
            metric = _metric(27, dev)
            model.correspondence_pr_step(dict(img=val["img"], label=val["label"]), metric)
            model.net.forward = fwd
            after = _train_state(model, dev)
            assert [m.training for m in model.modules()] == modes
            assert fused.ws.graph is graph and fused.key == key
            for k in before:
                if k != "cuda_rng":
                    assert torch.equal(before[k], after[k]), k
            torch.cuda.set_rng_state(before["cuda_rng"], dev)
            fs = model.cfg.feature_samples
            c1 = torch.rand([8, fs, fs, 2], device=dev) * 2 - 1
            c2 = torch.rand([8, fs, fs, 2], device=dev) * 2 - 1
            assert torch.equal(torch.cuda.get_rng_state(dev), after["cuda_rng"])
            assert len(seen) == 1
            twin = _metric(27, dev)
            twin.update(seen[0][0], seen[0][1], val["label"], c1, c2)
            assert torch.equal(metric.counts, twin.counts)
            assert int(metric.counts.sum()) == 2 * 8 * fs ** 4
            torch.cuda.set_rng_state(before["cuda_rng"], dev)  # the next step draws what it would have drawn
        losses.append(model.training_step(steps[1], 1).item())
        return losses, _train_state(model, dev)

    def dist(a, b):
        return max(float((a[1][k].double() - b[1][k].double()).abs().max()) for k in ("param", "exp_avg", "exp_avg_sq"))

    # The step's fp32 atomics make identical runs differ in the last bits, and the largest difference over the state
    # takes few distinct values, some rare (1e-7, 6e-7 and 2e-6 have been seen on unchanged code): one pair of plain
    # runs is too small a sample of the spread to hold the run with correspondence_pr_step to 4x of it.  The spread is
    # the largest distance among the plain runs; while it does not cover that run, more plain runs are drawn, up to
    # 16.  A step that left another RNG state behind would change every coordinate and dropout draw of the next one,
    # which no number of plain runs reproduces.
    plain = [run(False) for _ in range(2)]
    pr = run(True)
    while True:
        noise = max(dist(a, b) for i, a in enumerate(plain) for b in plain[i + 1:])
        diff = max(dist(a, pr) for a in plain)
        if diff <= 4 * noise or len(plain) == 16:
            break
        plain.append(run(False))
    print(f"run-to-run {noise:.3e} over {len(plain)} plain runs, with correspondence_pr_step {diff:.3e}")
    ref = plain[0]
    assert torch.equal(ref[1]["cuda_rng"], pr[1]["cuda_rng"])
    if noise == 0 and all(a[0] == ref[0] for a in plain):
        assert ref[0] == pr[0] and diff == 0
    else:
        assert diff <= 4 * noise
