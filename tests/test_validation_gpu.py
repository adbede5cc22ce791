"""LitUnsupervisedSegmenter.validation_step / validation_epoch_end (train_segmentation.py:254-371) on the GPU.

  * the reference's own validation (tests/golden/validation.pt, oracle/make_golden_validation.py) on the seeded
    ViT-S/8 at 32 px: the same preview dict, and the same predictions and confusion counts except at pixels whose
    fp64 top-2 margin on the reference's code is within what the difference between the two codes (bf16 ViT here,
    fp32 there) and the fp32 bars can move the logits;
  * full size against an fp64 evaluation of :260-269 on the same code: argmax maps equal off near-ties (the bars of
    tests/test_probes_fp64_gpu.py), confusion counts equal to the masked bincount of the returned maps exactly;
  * validation leaves training alone: parameters, gradients, Adam moments and the RNG bit-identical across it, training
    graphs neither re-captured nor replaced, train / eval modes restored, and the later steps as close to a run
    without validation as two runs without it are;
  * a validation_step issued right after training_step sees the updated parameters.
"""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _probes_fp64 as R  # noqa: E402
from _parity_util import make_batch, make_model  # noqa: E402

pytestmark = pytest.mark.gpu
U = R.U
ALPHA = 2.0


def _model(arch, dev, n_classes=27, seed=0, **over):
    import stego_oracle as O
    from stego_b200.config import make_cfg
    from stego_b200.segmenter import LitUnsupervisedSegmenter
    cfg = make_cfg(model_type=arch, random_backbone_init=True, **over)
    torch.manual_seed(seed)
    model = LitUnsupervisedSegmenter(n_classes, cfg).to(dev)
    model.net.model.load_state_dict(O.perturb_vit_state(O.vit_random_state(arch, 8, seed=3)))
    model.train()
    return model


def _capture_code(model):
    """Keep the code each net() call returns (the exact input of the fused probe pass)."""
    seen = []
    fwd = model.net.forward

    def rec(img, *a, **k):
        out = fwd(img, *a, **k)
        seen.append(out[1].detach().clone())
        return out
    model.net.forward = rec
    return seen


def _reference_fp64(code, lin_w, lin_b, clusters, H, W, code_delta=None):
    """fp64 linear logits / cluster cosines of :260-269 on `code` [B, C, h, w], image by image in bands of rows.  Returns
    the argmax maps and the 'safe' masks: pixels whose top-2 margin exceeds twice the largest bar of the pixel.
    Bars (tests/test_probes_fp64_gpu.py::_eval_case): linear E_z = interp((C + 3) u Ml) + 8 u sum_t |l_t| + lambda term;
    cluster alpha E_cos + 2 u alpha |cos| with E_cos = E_dv / |v| + |cos| eta.  code_delta: a second code's difference
    from this one, whose effect is added: interp(|W| |dx|) on the logits, 2 interp(|dx|) / |v| on the cosines."""
    B, C, h, w = code.shape
    n_lin, n_clu = lin_w.shape[0], clusters.shape[0]
    Wl = lin_w.view(n_lin, C)
    out = {k: torch.empty(B, H, W, dtype=dt, device=code.device)
           for k, dt in (("la", torch.long), ("ca", torch.long), ("ls", torch.bool), ("cs", torch.bool))}
    for b in range(B):
        x = code[b].double()
        dx = None if code_delta is None else code_delta[b].double().reshape(C, h * w).abs()
        for y0 in range(0, H, 64):
            rows = (y0, min(H, y0 + 64))
            e = R.eval_band(x, Wl, lin_b, clusters, ALPHA, H, W, rows)
            cr = e["corners"]
            E_z = cr.interp((C + 3) * U * e["Ml"]) + 8 * U * sum(t.abs() for t in cr.gather(e["l"])) + cr.lam_term(e["l"])
            vn, cos = e["vnorm"], e["cos"]
            E_dv = cr.interp((1.5 * C + 8) * U * e["Mdc"]) + 8 * U * sum(t.abs() for t in cr.gather(e["dc"])) + \
                cr.lam_term(e["dc"])
            xn = x.reshape(C, -1).norm(dim=0, keepdim=True)
            lam_n = 2 * (cr.ey + cr.ex) * torch.stack(cr.gather(xn)).amax(0)[0]
            A = e["wxn"]
            eta = 3 * U * A / vn + (C + 18) * 2.0 ** -53 * A ** 2 / (2 * vn ** 2) + lam_n / vn + 4 * U
            eta = torch.where(eta < 0.5, eta, torch.full_like(eta, float("inf")))
            E_s = ALPHA * (E_dv / vn + cos.abs() * eta) + 2 * U * ALPHA * cos.abs()
            if dx is not None:
                E_z = E_z + cr.interp(Wl.double().abs() @ dx)
                E_s = E_s + ALPHA * 2 * cr.interp(dx.norm(dim=0, keepdim=True)) / vn
            sl = (b, slice(rows[0], rows[1]))
            for logits, bar, arg, safe in ((e["z"], E_z, "la", "ls"), (ALPHA * cos, E_s, "ca", "cs")):
                top2 = logits.topk(2, 0)
                out[arg][sl] = top2.indices[0].view(-1, W)
                out[safe][sl] = (top2.values[0] - top2.values[1] > 2 * bar.amax(0)).view(-1, W)
            del e
    return out


# ================================================================================================
# the reference's own validation, 32 px
# ================================================================================================
@pytest.mark.parametrize("extra", [0, 2])
def test_golden_validation_step(cuda_dev, extra):
    import make_golden_validation as MV
    dev = cuda_dev
    g = torch.load(os.path.join(os.path.dirname(__file__), "golden", "validation.pt"), weights_only=False)[f"extra{extra}"]
    model = _model("vit_small", dev, extra_clusters=extra, n_images=MV.N_IMAGES)
    named = dict(model.named_parameters())
    with torch.no_grad():
        for k, v in MV.params(extra).items():
            named[k].copy_(v)
    codes = _capture_code(model)
    n_near = n_valid_near = n_diff = 0
    for i, batch in enumerate(MV.inputs()):
        prev = model.validation_step({k: v.to(dev) for k, v in batch.items()}, i)
        want = g["steps"][i]
        assert list(prev) == want["keys"] == ["img", "linear_preds", "cluster_preds", "label"]
        assert {k: tuple(v.shape) for k, v in prev.items()} == want["shapes"]
        assert {k: str(v.dtype) for k, v in prev.items()} == want["dtypes"]
        assert all(v.device.type == "cpu" for v in prev.values())
        ref_code = want["code"].to(dev)
        ref = _reference_fp64(ref_code, named["linear_probe.weight"].detach(), named["linear_probe.bias"].detach(),
                              named["cluster_probe.clusters"].detach(), MV.RES, MV.RES, code_delta=codes[-1] - ref_code)
        label = batch["label"].to(dev)
        valid = (label >= 0) & (label < 27)
        for got, ref_arg, safe, name in ((prev["linear_preds"], ref["la"], ref["ls"], "linear"),
                                         (prev["cluster_preds"], ref["ca"], ref["cs"], "cluster")):
            n = got.shape[0]
            got, ref_pred = got.to(dev), want[f"{name}_preds"].to(dev).long()
            # the fp64 argmax of the reference's code is the reference's own prediction off its fp32 near-ties
            assert torch.equal(ref_pred[safe[:n]], ref_arg[:n][safe[:n]]), name
            assert torch.equal(got[safe[:n]], ref_pred[safe[:n]]), (name, int((got != ref_pred)[safe[:n]].sum()))
            n_diff += int((got != ref_pred).sum())
            n_near += int((~safe).sum())
            n_valid_near += int((~safe & valid).sum())
    diff = int((model.linear_metrics.stats.cpu() - g["linear_stats"]).abs().sum() +
               (model.cluster_metrics.stats.cpu() - g["cluster_stats"]).abs().sum())
    pixels = 2 * 2 * MV.B * MV.RES * MV.RES  # two batches, two probes
    print(f"golden extra={extra}: near {n_near} of {pixels} pixel-probes, preview differences {n_diff}, stats |diff| {diff}")
    assert diff <= 2 * n_valid_near, (diff, n_valid_near)
    # the code-difference term is a worst-case (triangle-inequality) bound: about a quarter of these 4 x 4 -> 32 x 32
    # pixels fall under it, while under 0.5 % of the predictions actually differ (H100: 75 / 78 of 20480)
    assert n_near <= 0.3 * pixels, n_near
    assert n_diff <= 0.01 * 2 * 2 * MV.N_IMAGES * MV.RES * MV.RES, n_diff


# ================================================================================================
# full size against fp64 on the same code
# ================================================================================================
FULL = {
    # name: arch, B, H, W, n_classes, extra_clusters, label dtype
    "vits8_320_b16": ("vit_small", 16, 320, 320, 27, 0, torch.int64),
    "vitb8_320_b8": ("vit_base", 8, 320, 320, 27, 0, torch.int64),
    "vits8_320_3cls_extra2_u8": ("vit_small", 8, 320, 320, 3, 2, torch.uint8),
    "vits8_224x320_b8": ("vit_small", 8, 224, 320, 27, 0, torch.int32),
}


@pytest.mark.parametrize("case", list(FULL))
def test_full_size_against_fp64(cuda_dev, case):
    """27 / 27 classes at an 8x upsampling take eval_probe_vec4_kernel, 3 classes + 2 extra clusters eval_probe_kernel."""
    arch, B, H, W, n, extra, ldt = FULL[case]
    dev = cuda_dev
    model = _model(arch, dev, n_classes=n, extra_clusters=extra, n_images=B)
    with torch.no_grad():
        model.cluster_probe.clusters.normal_(generator=torch.Generator(device=dev).manual_seed(4))
    codes = _capture_code(model)
    gen = torch.Generator(device=dev).manual_seed(9)
    img = torch.randn(B, 3, H, W, device=dev, generator=gen)
    label = torch.randint(0, n, (B, H, W), device=dev, generator=gen)
    r = torch.rand(B, H, W, device=dev, generator=gen)
    label[r < 0.05] = 255 if ldt == torch.uint8 else -1
    label[(r >= 0.05) & (r < 0.08)] = n
    label = label.to(ldt)
    prev = model.validation_step(dict(img=img, label=label), 0)
    assert list(prev) == ["img", "linear_preds", "cluster_preds", "label"]
    assert all(v.device.type == "cpu" for v in prev.values())
    assert prev["img"].shape == (B, 3, H, W) and prev["img"].dtype == torch.float32
    assert prev["label"].dtype == ldt and torch.equal(prev["label"], label.cpu())
    for k in ("linear_preds", "cluster_preds"):
        assert prev[k].shape == (B, H, W) and prev[k].dtype == torch.int64
    la, ca = prev["linear_preds"].to(dev), prev["cluster_preds"].to(dev)
    assert int(la.max()) < n and int(ca.max()) < n + extra
    assert torch.equal(model.linear_metrics.stats, R.confusion(la, label, n, n))
    assert torch.equal(model.cluster_metrics.stats, R.confusion(ca, label, n + extra, n))
    ref = _reference_fp64(codes[0], model.linear_probe.weight.detach(), model.linear_probe.bias.detach(),
                          model.cluster_probe.clusters.detach(), H, W)
    for got, arg, safe, name in ((la, ref["la"], ref["ls"], "linear"), (ca, ref["ca"], ref["cs"], "cluster")):
        assert torch.equal(got[safe], arg[safe]), (case, name, int((got != arg)[safe].sum()))
        assert int((~safe).sum()) <= 2e-2 * B * H * W, (case, name, int((~safe).sum()))
    if extra:
        assert bool((ca >= n).any())  # the extra clusters are predicted, and dropped from the counts


# ================================================================================================
# validation does not change training
# ================================================================================================
def _train_state(model, dev):
    model.flush()
    torch.cuda.synchronize()
    f = model._flat
    return dict(param=f.param.clone(), grad=f.grad.clone(), exp_avg=f.exp_avg.clone(), exp_avg_sq=f.exp_avg_sq.clone(),
                cpu_rng=torch.get_rng_state(), cuda_rng=torch.cuda.get_rng_state(dev),
                adam_steps=torch.tensor([o.steps for o in f.optimizers]))


def _modes(model):
    return [m.training for m in model.modules()]


def _max_diff(a, b):
    return max(float((a[k].double() - b[k].double()).abs().max()) for k in ("param", "exp_avg", "exp_avg_sq"))


def test_validation_leaves_training_unchanged(cuda_dev):
    """4 fused steps, against 2 steps + 2 validation batches + validation_epoch_end + 2 steps.  Across validation the
    whole training state is bit-identical: parameters, gradients, Adam moments and step counts, both RNG states, the
    captured graphs (the same objects, replayed afterwards, never re-captured) and every module's train / eval mode.
    The two 4-step runs then agree as closely as two runs without validation do (bit-identical where the step itself
    is run-to-run reproducible; its split-K weight gradients accumulate with fp32 atomics)."""
    dev = cuda_dev
    steps = [make_batch(4, 64, dev, seed=10 + i) for i in range(4)]
    vals = [make_batch(4, 64, dev, seed=50 + i) for i in range(2)]
    runs = {}
    for name in ("plain", "plain_again", "with_validation"):
        model, _ = make_model("vit_small", dev, fused=True, seed=0)
        torch.manual_seed(777)
        losses = []
        for i, batch in enumerate(steps):
            if name == "with_validation" and i == 2:
                fused = model._fused
                graph, key, vit_graphs = fused.ws.graph, fused.key, dict(model.net.model._cache["graphs"])
                assert graph is not None
                before, modes = _train_state(model, dev), _modes(model)
                for j, v in enumerate(vals):
                    model.validation_step(dict(img=v["img"], label=v["label"]), j)
                    assert _modes(model) == modes
                metrics = model.validation_epoch_end([])
                assert model.global_step == 2 and not any(k.startswith("test/") for k in model.logged)
                assert sorted(metrics) == sorted(["test/linear/mIoU", "test/linear/Accuracy", "test/cluster/mIoU",
                                                  "test/cluster/Accuracy"])
                after = _train_state(model, dev)
                for k in before:
                    assert torch.equal(before[k], after[k]), k
                assert fused.ws.graph is graph and fused.key == key
                assert model.net.model._cache["graphs"] == vit_graphs
            losses.append(model.training_step(batch, i).item())
        assert model._fused.step_idx == 4  # every step took the hand-scheduled path
        if name == "with_validation":
            assert model._fused.ws.graph is graph  # replayed, not re-captured
        runs[name] = (losses, _train_state(model, dev))
    ref, again, val = runs["plain"], runs["plain_again"], runs["with_validation"]
    for k in ("cpu_rng", "cuda_rng", "adam_steps"):
        assert torch.equal(ref[1][k], val[1][k]), k
    noise = _max_diff(ref[1], again[1])
    noise_loss = max(abs(a - b) for a, b in zip(ref[0], again[0]))
    print(f"run-to-run: state {noise:.3e}, losses {noise_loss:.3e}; with validation: state "
          f"{_max_diff(ref[1], val[1]):.3e}, losses {max(abs(a - b) for a, b in zip(ref[0], val[0])):.3e}")
    if noise == 0 and noise_loss == 0:
        assert ref[0] == val[0]
        for k in ("param", "exp_avg", "exp_avg_sq"):
            assert torch.equal(ref[1][k], val[1][k]), k
    else:
        assert _max_diff(ref[1], val[1]) <= 4 * noise
        assert max(abs(a - b) for a, b in zip(ref[0], val[0])) <= 4 * noise_loss + 1e-7


def test_validation_right_after_training_step_sees_update(cuda_dev):
    """The parameter update runs on a side stream under the next step's backbone; validation_step waits for it.  Its
    predictions and counts equal those of flush() followed by an explicit eval-mode forward, and differ from the
    predictions before the step (the update is visible)."""
    from stego_b200.eval import fused_probe_log_probs
    dev = cuda_dev
    model, _ = make_model("vit_small", dev, fused=True, seed=0, n_images=4)
    val = make_batch(4, 64, dev, seed=60)
    vb = dict(img=val["img"], label=val["label"])
    before = model.validation_step(vb, 0)
    model.linear_metrics.reset()
    model.cluster_metrics.reset()
    torch.manual_seed(777)
    model.training_step(make_batch(4, 64, dev, seed=61), 0)
    got = model.validation_step(vb, 1)
    stats = (model.linear_metrics.stats.clone(), model.cluster_metrics.stats.clone())
    model.flush()
    torch.cuda.synchronize()
    model.net.eval()
    with torch.no_grad():
        code = model.net(vb["img"])[1]
    model.net.train()
    lc, cc = torch.zeros_like(stats[0]), torch.zeros_like(stats[1])
    _, _, la, ca = fused_probe_log_probs(code, model.linear_probe, model.cluster_probe, vb["label"].shape[-2:], 2.0,
                                         want_log_probs=False, want_argmax=True, label=vb["label"], linear_confusion=lc,
                                         cluster_confusion=cc)
    assert torch.equal(got["linear_preds"], la.long().cpu()) and torch.equal(got["cluster_preds"], ca.long().cpu())
    assert torch.equal(stats[0], lc) and torch.equal(stats[1], cc)
    assert not torch.equal(before["linear_preds"], got["linear_preds"])
