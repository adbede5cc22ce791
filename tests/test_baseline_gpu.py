"""GPU: evaluation of the DINO baseline (projection_type None: the probes on the backbone's 384 / 768-channel features).

  * the wide preparation kernel (eval_prep_wide_kernel) behind fused_probe_log_probs against the reference op sequence
    in fp64 (upsample, 1x1 conv, ClusterLookup, log_softmax) on the 1024 x 2048 frame and a smaller one, at 384 and
    768 channels, fp32 and bf16 code, with and without flip-TTA, with zero code pixels: log-probabilities elementwise,
    argmax equal off near-ties, confusion counts exactly those of the kernel's own predictions;
  * a bf16 code gives bit-identical outputs to the same values in fp32 (the two entries share every kernel);
  * eval_step (with and without the CRF), eval_scene and validation_step on ViT-S/8 and ViT-B/8 baseline models are
    bit-equal to the fused calls on the fp32 codes of two separate eval-mode net() calls, as for the projection head.
"""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))

pytestmark = pytest.mark.gpu


class _Lin(torch.nn.Module):
    def __init__(self, w, b):
        super().__init__()
        self.weight, self.bias = torch.nn.Parameter(w[:, :, None, None]), torch.nn.Parameter(b)


class _Clu(torch.nn.Module):
    def __init__(self, c):
        super().__init__()
        self.clusters = torch.nn.Parameter(c)


def _inputs(dev, C, h, w, n_lin, n_clu, dtype, flip, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    tok = torch.randn(2, h * w, C, device=dev, generator=g)
    tok[:, : 3 * w + 5] = 0.0  # zero code pixels: the cosine's norm clamp
    tok = tok.to(dtype)
    code = tok[:1].view(1, h, w, C).permute(0, 3, 1, 2)
    code_flipped = tok[1:].view(1, h, w, C).permute(0, 3, 1, 2) if flip else None
    W = torch.randn(n_lin, C, device=dev, generator=g) * (4.0 / (3.0 * C ** 0.5))
    b = torch.randn(n_lin, device=dev, generator=g) * 0.5
    cl = torch.randn(n_clu, C, device=dev, generator=g)
    return code, code_flipped, _Lin(W, b), _Clu(cl)


def _reference(code, code_flipped, W, b, cl, alpha, H, W_out, chunk=64):
    """fp64: (linear log-probs, cluster log-probs) [n, H, W] of one frame by the reference's op sequence, channels in
    chunks (the upsampled 768-channel fp64 code of a 1024 x 2048 frame would be 13 GB)."""
    x = code[0].double()
    if code_flipped is not None:
        x = (x + code_flipped[0].double().flip(2)) / 2
    C = x.shape[0]
    Wd, ch = W.double().reshape(-1, C), F.normalize(cl.double(), dim=1, eps=1e-12)
    z = b.double()[:, None, None].expand(-1, H, W_out).clone()
    d = torch.zeros(ch.shape[0], H, W_out, dtype=torch.float64, device=x.device)
    n2 = torch.zeros(H, W_out, dtype=torch.float64, device=x.device)
    for c0 in range(0, C, chunk):
        v = F.interpolate(x[None, c0:c0 + chunk], (H, W_out), mode="bilinear", align_corners=False)[0]
        z += torch.einsum("kc,chw->khw", Wd[:, c0:c0 + chunk], v)
        d += torch.einsum("kc,chw->khw", ch[:, c0:c0 + chunk], v)
        n2 += v.square().sum(0)
    cos = d / n2.sqrt().clamp_min(1e-12)
    return torch.log_softmax(z, 0), torch.log_softmax(alpha * cos, 0)


def _off_ties(ref_logp, margin):
    top2 = ref_logp.topk(2, dim=0).values
    return (top2[0] - top2[1]) > margin


@pytest.mark.parametrize("flip", [False, True])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("C", [384, 768])
@pytest.mark.parametrize("shape", ["c4_27", "256x512_5_7"])
def test_wide_prep_against_fp64(cuda_dev, shape, C, dtype, flip):
    from _probes_fp64 import confusion
    from stego_b200.eval import fused_probe_log_probs
    dev = cuda_dev
    h, w, n_lin, n_clu = dict(c4_27=(128, 256, 27, 27), **{"256x512_5_7": (32, 64, 5, 7)})[shape]
    H, W = 8 * h, 8 * w
    code, code_flipped, lin, clu = _inputs(dev, C, h, w, n_lin, n_clu, dtype, flip, seed=C + int(flip))
    g = torch.Generator(device=dev).manual_seed(7)
    label = torch.randint(-1, n_lin, (1, H, W), device=dev, generator=g)
    lc = torch.zeros(n_lin, n_lin, dtype=torch.long, device=dev)
    cc = torch.zeros(n_clu, n_lin, dtype=torch.long, device=dev)
    llp, clp, la, ca = fused_probe_log_probs(code, lin, clu, (H, W), 2.0, want_log_probs=True, want_argmax=True,
                                             code_flipped=code_flipped, label=label, linear_confusion=lc,
                                             cluster_confusion=cc)
    with torch.no_grad():
        rl, rc = _reference(code, code_flipped, lin.weight, lin.bias, clu.clusters, 2.0, H, W)
    for name, got, ref in (("linear", llp[0], rl), ("cluster", clp[0], rc)):
        err = float((got.double() - ref).abs().max())
        assert err < 1e-4, (name, err)
        ok = _off_ties(ref, max(4 * err, 1e-6))  # the argmax may differ only where the errors can swap the top two
        arg = (la if name == "linear" else ca)[0].long()
        assert torch.equal(arg[ok], ref.argmax(0)[ok]), name
        assert float(ok.double().mean()) > 0.9, name
    # the zero code pixels: cosine 0 for every centroid, uniform cluster log-probabilities, argmax 0
    assert torch.allclose(clp[0, :, :8, :8], torch.full_like(clp[0, :, :8, :8], -float(torch.tensor(n_clu).log())),
                          atol=1e-6)
    assert not ca[0, :8, :8].any()
    assert torch.equal(lc, confusion(la, label, n_lin, n_lin))
    assert torch.equal(cc, confusion(ca, label, n_clu, n_lin))
    assert int(lc.sum()) > 0


@pytest.mark.parametrize("flip", [False, True])
@pytest.mark.parametrize("C", [384, 768])
def test_bf16_code_bit_equal_to_fp32_of_its_values(cuda_dev, C, flip):
    from stego_b200.eval import fused_eval_crf, fused_probe_log_probs
    dev = cuda_dev
    h, w = 8, 12
    code, code_flipped, lin, clu = _inputs(dev, C, h, w, 27, 30, torch.bfloat16, flip, seed=3)
    g = torch.Generator(device=dev).manual_seed(2)
    img = torch.randn(1, 3, 64, 96, device=dev, generator=g)
    f32 = lambda t: None if t is None else t.float()
    a = fused_probe_log_probs(code, lin, clu, (64, 96), 2.0, want_argmax=True, code_flipped=code_flipped)
    b = fused_probe_log_probs(f32(code), lin, clu, (64, 96), 2.0, want_argmax=True, code_flipped=f32(code_flipped))
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    a = fused_eval_crf(code, lin, clu, img, 2.0, code_flipped=code_flipped, want_marginals=True)
    b = fused_eval_crf(f32(code), lin, clu, img, 2.0, code_flipped=f32(code_flipped), want_marginals=True)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


# ================================================================================================
# the model's eval entry points on baseline models
# ================================================================================================
def _model(dev, arch, n_classes=27, extra=0):
    import stego_oracle as O
    from stego_b200.config import make_cfg
    from stego_b200.segmenter import LitUnsupervisedSegmenter
    torch.manual_seed(0)
    dim = 384 if arch == "vit_small" else 768
    cfg = make_cfg(random_backbone_init=True, model_type=arch, projection_type=None, dim=dim,
                   correspondence_weight=0.0, extra_clusters=extra)
    model = LitUnsupervisedSegmenter(n_classes, cfg).to(dev)
    model.net.model.load_state_dict(O.perturb_vit_state(O.vit_random_state(arch, 8, seed=3)))
    with torch.no_grad():
        model.cluster_probe.clusters.normal_(generator=torch.Generator(device=dev).manual_seed(4))
        model.linear_probe.weight.mul_(8.0)
    model.train()
    return model


def _two_codes(model, img):
    """The codes of two eval-mode net() calls on img and img.flip(3) (eval_segmentation.py:124-125): fp32 features."""
    modes = [(m, m.training) for m in model.modules()]
    model.net.eval()
    with torch.no_grad():
        code1 = model.net(img)[1].clone()
        code2 = model.net(img.flip(3).contiguous())[1].clone()
    for m, mode in modes:
        m.training = mode
    return code1, code2


def _batch(dev, n, B, H, W, seed=9):
    g = torch.Generator(device=dev).manual_seed(seed)
    img = torch.randn(B, 3, H, W, device=dev, generator=g)
    label = torch.randint(-1, n, (B, H, W), device=dev, generator=g)
    return img, label


@pytest.mark.parametrize("run_crf", [False, True])
@pytest.mark.parametrize("arch,B,res", [("vit_small", 3, 64), ("vit_base", 2, 96)])
def test_eval_step_bit_equal_to_fused_calls(cuda_dev, arch, B, res, run_crf):
    from _probes_fp64 import confusion
    from stego_b200 import _lib
    from stego_b200.eval import fused_eval_crf, fused_probe_log_probs
    dev = cuda_dev
    n, extra = 27, 3
    model = _model(dev, arch, n, extra)
    img, label = _batch(dev, n, B, res, res)
    rng = torch.cuda.get_rng_state(dev)
    launches = _lib.launch_count()
    got = model.eval_step(dict(img=img, label=label), run_crf=run_crf, want_probs=True)
    assert _lib.launch_count() > launches and torch.equal(rng, torch.cuda.get_rng_state(dev))
    code1, code2 = _two_codes(model, img)
    assert code1.shape == (B, model.net.n_feats, res // 8, res // 8)
    lc = torch.zeros(n, n, dtype=torch.long, device=dev)
    cc = torch.zeros(n + extra, n, dtype=torch.long, device=dev)
    if run_crf:
        la, ca, lq, cq = fused_eval_crf(code1, model.linear_probe, model.cluster_probe, img, 2.0, code_flipped=code2,
                                        label=label, linear_confusion=lc, cluster_confusion=cc, want_marginals=True)
    else:
        lq, cq, la, ca = fused_probe_log_probs(code1, model.linear_probe, model.cluster_probe, (res, res), 2.0,
                                               want_argmax=True, code_flipped=code2, label=label, linear_confusion=lc,
                                               cluster_confusion=cc)
    for k, want in (("linear_preds", la), ("cluster_preds", ca), ("linear_probs", lq), ("cluster_probs", cq)):
        assert torch.equal(got[k], want), k
    assert torch.equal(model.test_linear_metrics.stats, lc) and torch.equal(model.test_cluster_metrics.stats, cc)
    assert torch.equal(lc, confusion(got["linear_preds"], label, n, n))
    assert torch.equal(cc, confusion(got["cluster_preds"], label, n + extra, n))
    assert len(torch.unique(got["cluster_preds"])) > 1 and len(torch.unique(got["linear_preds"])) > 1


@pytest.mark.parametrize("arch", ["vit_small", "vit_base"])
def test_eval_scene_bit_equal_to_eval_step(cuda_dev, arch):
    dev = cuda_dev
    n = 5
    model = _model(dev, arch, n)
    R, C, t = 2, 3, 32
    tiles, label = _batch(dev, n, R * C, t, t, seed=4)
    got = model.eval_scene(tiles, (R, C), label=label, want_probs=True, chunk=4)
    scene_stats = (model.test_linear_metrics.stats.clone(), model.test_cluster_metrics.stats.clone())
    model.test_linear_metrics.reset()
    model.test_cluster_metrics.reset()
    parts = [model.eval_step(dict(img=tiles[i:i + 4], label=label[i:i + 4]), want_probs=True) for i in (0, 4)]
    stitch = lambda m: m.reshape(R, C, t, t).transpose(1, 2).reshape(R * t, C * t)  # [R*C, t, t] -> [R t, C t]
    for k in ("linear", "cluster"):
        preds = torch.cat([p[k + "_preds"] for p in parts])
        probs = torch.cat([p[k + "_probs"] for p in parts])  # [R*C, n, t, t]
        assert torch.equal(got[k + "_preds"], stitch(preds)), k
        assert torch.equal(got[k + "_probs"], torch.stack([stitch(probs[:, c]) for c in range(probs.shape[1])])), k
    assert torch.equal(scene_stats[0], model.test_linear_metrics.stats)
    assert torch.equal(scene_stats[1], model.test_cluster_metrics.stats)


def test_validation_step_on_the_baseline(cuda_dev):
    from _probes_fp64 import confusion
    from stego_b200.eval import fused_probe_log_probs
    dev = cuda_dev
    n = 27
    model = _model(dev, "vit_small", n)
    img, label = _batch(dev, n, 4, 64, 64)
    out = model.validation_step(dict(img=img, label=label), 0)
    code1, _ = _two_codes(model, img)
    _, _, la, ca = fused_probe_log_probs(code1, model.linear_probe, model.cluster_probe, (64, 64), 2.0,
                                         want_log_probs=False, want_argmax=True)
    assert torch.equal(out["linear_preds"], la[:4].long().cpu()) and torch.equal(out["cluster_preds"], ca[:4].long().cpu())
    assert torch.equal(model.linear_metrics.stats, confusion(la, label, n, n))
    assert torch.equal(model.cluster_metrics.stats, confusion(ca, label, n, n))


def test_eval_against_reference_golden(cuda_dev):
    """eval_step (flip-TTA) and fused_probe_log_probs without the mirror against the reference's own evaluation of the
    baseline (tests/golden/baseline.pt): the backbone runs in bf16 here and in fp32 there, so the predictions agree
    wherever the reference's top-2 margin exceeds twice the largest log-probability difference, and the confusion
    counts are exactly those of the predictions returned."""
    from _probes_fp64 import confusion
    from stego_b200.eval import fused_probe_log_probs
    import make_golden_baseline as MB
    import make_golden_eval_step as ME
    dev = cuda_dev
    g = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "baseline.pt"), weights_only=False)
    n, extra = MB.N_CLASSES, MB.EXTRA
    model = _model(dev, "vit_small", n, extra)
    with torch.no_grad():
        for k, v in MB.params().items():
            dict(model.named_parameters())[k].copy_(v)
    for key in ("tta", "no_tta"):
        model.test_linear_metrics.reset()
        model.test_cluster_metrics.reset()
        for batch, want in zip(ME.inputs(), g[key]):
            img, label = batch["img"].to(dev), batch["label"].to(dev)
            if key == "tta":
                got = model.eval_step(dict(img=img, label=label), want_probs=True)
            else:
                code, _ = _two_codes(model, img)
                lq, cq, la, ca = fused_probe_log_probs(code, model.linear_probe, model.cluster_probe, label.shape[-2:],
                                                       2.0, want_argmax=True)
                got = dict(linear_probs=lq, cluster_probs=cq, linear_preds=la, cluster_preds=ca)
            for k in ("linear", "cluster"):
                ref = want[k + "_probs"].to(dev).double()
                diff = float((got[k + "_probs"].detach().double() - ref).abs().max())
                assert diff < 5e-2, (key, k, diff)
                ok = _off_ties(ref.transpose(0, 1).reshape(ref.shape[1], -1), 2 * diff).reshape(ref.shape[0], *ref.shape[2:])
                assert torch.equal(got[k + "_preds"].long()[ok], want[k + "_preds"].to(dev).long()[ok]), (key, k)
                assert float(ok.double().mean()) > 0.5, (key, k)
            if key == "tta":
                assert torch.equal(model.test_linear_metrics.stats, confusion(got["linear_preds"], label, n, n))
                assert torch.equal(model.test_cluster_metrics.stats, confusion(got["cluster_preds"], label, n + extra, n))
                model.test_linear_metrics.reset()
                model.test_cluster_metrics.reset()


# ================================================================================================
# training: the wide probe kernels against fp64, and the step against the reference's
# ================================================================================================
TRAIN = {"c1": (32, 28, 224), "c2": (32, 40, 320), "c3": (16, 56, 448)}  # B, h = w, H = W (the c1-c3 shapes)


@pytest.mark.parametrize("shape,C,n,ldt,ignore,view", [
    ("c1", 384, 27, torch.int64, "random", "contiguous"),
    ("c2", 768, 32, torch.int32, "random", "contiguous"),
    ("c3", 384, 5, torch.uint8, "random", "contiguous"),
    ("c3", 768, 27, torch.int64, "tiles", "contiguous"),
    ("c1", 768, 27, torch.int64, "all", "contiguous"),
    ("c1", 384, 27, torch.int64, "random", "batch_strided"),
])
def test_wide_linear_probe_ce_fp64(cuda_dev, shape, C, n, ldt, ignore, view):
    from _probes_fp64 import linear_inputs, linear_ce_ref
    from stego_b200.segmenter import linear_probe_ce
    dev = cuda_dev
    B, h, H = TRAIN[shape]
    code, weight, bias, label = linear_inputs(B, C, h, h, H, H, n, label_dtype=ldt, ignore=ignore, seed=C + n,
                                              device=dev)
    x = code.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)  # tokens-major, as the step's code
    if view == "batch_strided":
        big = torch.zeros(2 * B, h, h, C, device=dev)
        big[::2] = x.permute(0, 2, 3, 1)
        x = big[::2].permute(0, 3, 1, 2)
    W = weight.clone().requires_grad_(True)
    b = bias.clone().requires_grad_(True)
    loss = linear_probe_ce(x, W.view(n, C, 1, 1), b, label)
    loss.backward()
    ref = linear_ce_ref(code, weight, bias, label, n)
    if ignore == "all":
        assert torch.isnan(loss) and not W.grad.any() and not b.grad.any()
        return
    assert abs(float(loss) - float(ref["loss"])) < 1e-5 * max(1.0, abs(float(ref["loss"]))), (float(loss), float(ref["loss"]))
    X = code.double().reshape(B, C, h * h)
    dl = ref["dl"]
    bound_w = ref["s"] * torch.einsum("bkr,bcr->kc", dl.abs(), X.abs())
    bound_b = ref["s"] * dl.abs().sum((0, 2))
    assert bool(((W.grad.double().reshape(n, C) - ref["dW"]).abs() <= 1e-4 * bound_w + 1e-9).all())
    assert bool(((b.grad.double() - ref["db"]).abs() <= 1e-4 * bound_b + 1e-9).all())


def _cluster_wide(x_rows, clusters, want_grad=True):
    from stego_b200 import _lib, ops
    dev = x_rows.device
    rows, C = x_rows.shape
    n = clusters.shape[0]
    loss = torch.empty(2, device=dev)
    assign = torch.empty(rows, dtype=torch.int32, device=dev)
    inv = torch.empty(rows, device=dev)
    dnc = torch.zeros(n, C, device=dev)
    dcl = torch.zeros(n, C, device=dev)
    _lib.check(_lib.load().stego_cluster_lookup_wide(
        _lib.ptr(x_rows), C, rows, C, _lib.ptr(clusters), n, _lib.ptr(assign), _lib.ptr(inv),
        _lib.ptr(ops.probe_scratch(dev)), _lib.ptr(loss), _lib.ptr(dnc) if want_grad else None,
        _lib.ptr(dcl) if want_grad else None, _lib.stream()), "stego_cluster_lookup_wide")
    return loss[0], assign, dnc, dcl


@pytest.mark.parametrize("shape,C,n,regime", [
    ("c1", 384, 27, "random"), ("c2", 768, 64, "random"), ("c3", 384, 64, "ties"), ("c1", 768, 27, "zeros"),
    ("c2", 384, 33, "zerorow"), ("c3", 768, 5, "sharp"),
])
def test_wide_cluster_lookup_fp64(cuda_dev, shape, C, n, regime):
    from _probes_fp64 import cluster_inputs, normalize_bwd
    import torch.nn.functional as F_
    dev = cuda_dev
    B, h, _ = TRAIN[shape]
    x, cl = cluster_inputs(regime, B, C, h * h, n, seed=C + n, device=dev)
    rows = x.permute(0, 2, 1).reshape(-1, C).contiguous()
    loss, assign, dnc, dcl = _cluster_wide(rows, cl)
    xd = rows.double()
    xh = xd / xd.norm(dim=1, keepdim=True).clamp_min(1e-12)
    ch = cl.double() / cl.double().norm(dim=1, keepdim=True).clamp_min(1e-12)
    ip = xh @ ch.t()                                         # [rows, n]
    top2 = ip.topk(min(2, n), dim=1).values
    ok = (top2[:, 0] - top2[:, 1]) > 1e-5 if n > 1 else torch.ones_like(top2[:, 0], dtype=torch.bool)
    assert torch.equal(assign.long()[ok], ip.argmax(1)[ok])
    if regime == "ties":  # exact ties by construction (a duplicated centroid, mirrored channels): the first one wins
        assert not bool((assign == 1).any()) and not bool((assign == 3).any())
    elif regime == "zeros":  # a zero pixel's cosines are all 0: argmax 0
        assert not bool(assign.view(B, h * h)[:, ::7].any())
    else:
        assert float(ok.double().mean()) > 0.9
    a = assign.long()
    best = ip.gather(1, a[:, None])[:, 0]                    # the kernel's choice, in fp64
    assert abs(float(loss) + float(best.mean())) < 1e-5, (float(loss), -float(best.mean()))
    gs = -1.0 / rows.shape[0]
    onehot = F_.one_hot(a, n).double()
    ref_dnc = gs * onehot.t() @ xh
    bound = abs(gs) * onehot.t() @ xh.abs()
    assert bool(((dnc.double() - ref_dnc).abs() <= 1e-4 * bound + 1e-12).all())
    # the centroid normalisation's backward (cluster_norm_bwd_kernel, fp32) on the kernel's own dnc: its error is
    # bounded by the size of the terms it combines, |dnc_k| and |c_k| <c_k, dnc_k> / |c_k|^2, over |c_k|
    cd, dn = cl.double(), dnc.double()
    nrm = cd.norm(dim=1, keepdim=True)
    ref_dcl = normalize_bwd(cd, dn)
    terms = (dn.abs() + cd.abs() * (cd * dn).abs().sum(1, keepdim=True) / nrm.square().clamp_min(1e-24))
    bound = terms.amax(1, keepdim=True) / nrm.clamp_min(1e-12)
    assert bool(((dcl.double() - ref_dcl).abs() <= 1e-5 * bound).all())
    again = _cluster_wide(rows, cl)
    assert torch.equal(loss, again[0]) and torch.equal(assign, again[1]) and torch.equal(dcl, again[3])


def _train_model(dev, seed=0):
    import make_golden_baseline as MB
    model = _model(dev, "vit_small", MB.N_CLASSES, MB.EXTRA)
    with torch.no_grad():
        for k, v in MB.params().items():
            dict(model.named_parameters())[k].copy_(v)
    model.configure_optimizers()
    return model


def _run_steps(model, dev):
    import make_golden_baseline as MB
    out = []
    for i, batch in enumerate(MB.step_batches()):
        torch.manual_seed(777 + i)
        loss = model.training_step({k: v.to(dev) for k, v in batch.items()}, i)
        model.flush()
        out.append(dict(loss=loss.detach().clone(), logged={k: float(v) for k, v in model.logged.items()},
                        params={k: v.detach().clone() for k, v in model.named_parameters()
                                if k.startswith(("linear_probe", "cluster_probe", "net.cluster1"))}))
    return out


def test_training_step_against_reference_golden(cuda_dev):
    """Two baseline training steps: the probes' losses and parameters against the fp64 restatement on the step's own
    (bf16) backbone features tightly, and against the reference's fp32 run (tests/golden/baseline.pt) to the bf16
    backbone's difference; cluster1 untouched, bit-identical cluster probe across two runs, eval_step leaving the
    training state alone."""
    import baseline_oracle as BO
    import make_golden_baseline as MB
    from stego_b200 import _lib
    dev = cuda_dev
    g = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "baseline.pt"), weights_only=False)
    model = _train_model(dev)
    c1 = model.net.cluster1[0].weight.detach().clone(), model.net.cluster1[0].bias.detach().clone()
    launches = _lib.launch_count()
    got = _run_steps(model, dev)
    assert _lib.launch_count() > launches
    # the restatement in fp64 on the features the step saw
    p = {k: v.double().cpu() for k, v in MB.params().items()}
    state = {k: (torch.zeros_like(v), torch.zeros_like(v)) for k, v in p.items()}
    for i, (batch, s, want) in enumerate(zip(MB.step_batches(), got, g["train"])):
        with torch.no_grad():
            B, _, H, W = batch["img"].shape
            tok = model.net.backbone_tokens(batch["img"].to(dev)).double().cpu()
            code = tok.view(B, H // 8, W // 8, -1).permute(0, 3, 1, 2)
        q = {k: v.clone().requires_grad_(True) for k, v in p.items()}
        lin, clu = BO.probe_losses(code, q, batch["label"], MB.N_CLASSES)
        grads = torch.autograd.grad(lin + clu, list(q.values()))
        with torch.no_grad():
            for (k, v), gr in zip(p.items(), grads):
                _adam(v, gr, *state[k], i + 1)
        assert abs(s["logged"]["loss/linear"] - float(lin)) < 1e-4 * abs(float(lin)), (s["logged"], float(lin))
        assert abs(s["logged"]["loss/cluster"] - float(clu)) < 1e-4, (s["logged"], float(clu))
        for k, v in p.items():
            err = float((s["params"][k].double().cpu() - v).abs().max())
            assert err < 1e-5, (i, k, err)
        for k in ("loss/linear", "loss/cluster", "loss/total"):
            assert abs(s["logged"][k] - want["logged"][k]) < 2e-2 * max(1.0, abs(want["logged"][k])), (k, s["logged"][k])
        for k, v in want["params"].items():
            # Adam's first steps move every entry by about lr = 5e-3 whatever the gradient's size: an entry whose
            # gradient is within the bf16 features' difference of 0 may move the other way
            d = (s["params"][k].cpu() - v).abs()
            assert float(d.max()) < 2.1e-2 and float((d < 1e-3).double().mean()) > 0.95, (i, k)
        assert torch.equal(s["params"]["net.cluster1.0.weight"], c1[0])
        assert torch.equal(s["params"]["net.cluster1.0.bias"], c1[1])
    # two runs from one seed
    again = _run_steps(_train_model(dev), dev)
    for a, b in zip(got, again):
        assert torch.equal(a["loss"], b["loss"])
        for k in ("cluster_probe.clusters", "linear_probe.weight", "linear_probe.bias"):
            assert torch.equal(a["params"][k], b["params"][k]), k
    # eval_step between steps leaves the training state alone: parameters, Adam moments, gradients, backbone graphs
    snap = {k: v.detach().clone() for k, v in model.state_dict().items()}
    flat = {k: getattr(model._flat, k).detach().clone() for k in ("param", "grad", "exp_avg", "exp_avg_sq")}
    graphs = dict(model.net.model._cache.get("graphs", {}))
    model.eval_step(dict(img=MB.step_batches()[0]["img"].to(dev)))
    model.flush()
    assert all(torch.equal(v, model.state_dict()[k]) for k, v in snap.items())
    for k, v in flat.items():
        assert torch.equal(v, getattr(model._flat, k)), k
    after = model.net.model._cache.get("graphs", {})
    assert all(after.get(k) is v for k, v in graphs.items())  # the training graphs kept, none replaced
    # and the next step trains on from the same state as without the eval_step
    third = _run_steps(model, dev)[0]
    ref_model = _train_model(dev)
    _run_steps(ref_model, dev)
    ref_third = _run_steps(ref_model, dev)[0]
    for k in ("cluster_probe.clusters", "linear_probe.weight", "linear_probe.bias"):
        assert torch.equal(third["params"][k], ref_third["params"][k]), k


def _adam(p, g, m, v, step, lr=5e-3):
    import stego_oracle as O
    O.adam_step(p, g, m, v, step, lr)


@pytest.mark.parametrize("C", [384, 768])
def test_wide_prep_nearly_cancelling_neighbours_fp64(cuda_dev, C):
    """Odd columns nearly cancel the even column to their left (|v| = 1e-3 of sum_t w_t |x_t| at some output pixels):
    the cosine's norm comes from the fp64 Gram entries, so the error is that of the fp32 dots alone,
    about C * U * sum_t w_t |<x_t, c_k>|_abs / |v|."""
    from _probes_fp64 import anticorrelated_code
    from stego_b200.eval import fused_probe_log_probs
    dev = cuda_dev
    h, w, n = 32, 64, 27
    H, W = 8 * h, 8 * w
    code = anticorrelated_code(1, C, h, w, 1e-3, seed=C, device=dev)
    tok = code.permute(0, 2, 3, 1).contiguous()
    x = tok.permute(0, 3, 1, 2)
    _, _, lin, clu = _inputs(dev, C, h, w, n, n, torch.float32, False, seed=5)
    _, clp, _, ca = fused_probe_log_probs(x, lin, clu, (H, W), 2.0, want_argmax=True)
    with torch.no_grad():
        _, rc = _reference(x, None, lin.weight, lin.bias, clu.clusters, 2.0, H, W)
        xd = x[0].double()
        ch = F.normalize(clu.clusters.double(), dim=1, eps=1e-12)
        Mdc = torch.einsum("kc,chw->khw", ch.abs(), xd.abs()).amax(0, keepdim=True)  # [1, h, w]
        S = F.interpolate(Mdc[None], (H, W), mode="bilinear", align_corners=False)[0, 0]
        vn2 = torch.zeros(H, W, dtype=torch.float64, device=dev)
        for c0 in range(0, C, 64):
            vn2 += F.interpolate(xd[None, c0:c0 + 64], (H, W), mode="bilinear", align_corners=False)[0].square().sum(0)
        bar = 2.0 * 2 * 4 * C * 2.0 ** -24 * S / vn2.sqrt().clamp_min(1e-30) + 1e-5  # alpha * 2 * (cos error)
    err = (clp[0].double() - rc).abs().amax(0)
    assert bool((err <= bar).all()), float((err / bar).max())
    assert float((S / vn2.sqrt()).max()) > 20  # the case is badly conditioned somewhere
    top2 = rc.topk(2, dim=0).values
    ok = (top2[0] - top2[1]) > 2 * bar
    assert torch.equal(ca[0].long()[ok], rc.argmax(0)[ok]) and float(ok.double().mean()) > 0.5


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("C", [384, 768])
def test_wide_crf_unaries_fp64(cuda_dev, C, dtype):
    """stego_eval_crf_unary(_bf16) on a wide code against pydensecrf's unary_from_softmax (-log(clip(p, 1e-5, 1))) and
    the initial Q = softmax(-U) of the fp64 log-probabilities, both probes, with flip-TTA."""
    from stego_b200 import _lib
    from stego_b200.eval import _eval_codes, _probe_tables
    dev = cuda_dev
    h, w, n_lin, n_clu = 16, 32, 27, 30
    H, W = 8 * h, 8 * w
    code, code_flipped, lin, clu = _inputs(dev, C, h, w, n_lin, n_clu, dtype, True, seed=11)
    x, xf, ld, bf16 = _eval_codes(code, code_flipped)
    assert bf16 == (dtype == torch.bfloat16)
    wl, bl, cl = _probe_tables(lin, clu, C)
    scratch = torch.empty(h * w, 80, device=dev)
    unary = torch.empty(H * W, 64, device=dev)
    Q = torch.empty(H * W, 64, device=dev)
    name = "stego_eval_crf_unary_bf16" if bf16 else "stego_eval_crf_unary"
    _lib.check(getattr(_lib.load(), name)(_lib.ptr(x), _lib.ptr(xf), ld, C, 1, h, w, H, W, _lib.ptr(wl), _lib.ptr(bl),
                                          n_lin, _lib.ptr(cl), n_clu, 2.0, _lib.ptr(scratch), _lib.ptr(unary),
                                          _lib.ptr(Q), _lib.stream()), name)
    with torch.no_grad():
        rl, rc = _reference(code, code_flipped, lin.weight, lin.bias, clu.clusters, 2.0, H, W)
    for off, ref, n in ((0, rl, n_lin), (32, rc, n_clu)):
        u_ref = -ref.exp().clamp(1e-5, 1.0).log().reshape(n, -1).t()  # [H*W, n]
        q_ref = torch.softmax(-u_ref, 1)
        u, q = unary[:, off:off + n].double(), Q[:, off:off + n].double()
        assert float((u - u_ref).abs().max()) < 1e-4, float((u - u_ref).abs().max())
        assert float((q - q_ref).abs().max()) < 1e-5, float((q - q_ref).abs().max())
        assert not unary[:, off + n:off + 32].any() and not Q[:, off + n:off + 32].any()
