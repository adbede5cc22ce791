"""LitUnsupervisedSegmenter.eval_step (eval_segmentation.py:122-141) and its flip-TTA backbone pass on the GPU.

  * stego_vit_patchify_tta is bit-equal to stego_vit_patchify of img and of img.flip(3) (fp32 / bf16, patch 8 / 16);
  * the 2B tokens of one mirrored backbone pass are bit-equal, half for half, to separate patch_features /
    key_features calls on img and img.flip(3), eagerly and replayed as a graph;
  * eval_step's predictions, probabilities and both `final/` confusion matrices are bit-equal to fused_probe_log_probs
    (or fused_eval_crf with run_crf) on the codes of two separate eval-mode net() calls, and the counts equal a masked
    bincount of the returned predictions;
  * end to end against the reference loop in fp32 torch on the GPU (oracle/eval_step_oracle.py): argmax maps equal
    wherever the reference's top-2 margin exceeds twice the largest log-probability difference;
  * eval_step leaves training alone (state, generators, graphs, modes) and sees the update of the step before it.
"""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from _parity_util import make_batch, make_model  # noqa: E402

pytestmark = pytest.mark.gpu


# ================================================================================================
# the mirrored patchify
# ================================================================================================
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("p", [8, 16])
@pytest.mark.parametrize("B,H,W", [(2, 224, 224), (2, 320, 320), (2, 224, 320), (1, 224, 320), (1, 320, 224)])
def test_patchify_tta_bit_equal(cuda_dev, dtype, p, B, H, W):
    from stego_b200 import ops
    g = torch.Generator(device=cuda_dev).manual_seed(B * H + W + p)
    img = torch.randn(B, 3, H, W, device=cuda_dev, generator=g).to(dtype)
    got = ops.patchify_tta(img, p)
    n = B * (H // p) * (W // p)
    assert got.shape == (2 * n, 3 * p * p)
    assert torch.equal(got[:n], ops.patchify(img, p))
    assert torch.equal(got[n:], ops.patchify(img.flip(3).contiguous(), p))


# ================================================================================================
# one backbone pass over the frame and its mirror
# ================================================================================================
@pytest.mark.parametrize("arch,res", [("vit_small", 224), ("vit_base", 320)])
def test_tta_tokens_bit_equal_to_separate_calls(cuda_dev, arch, res):
    import stego_oracle as O
    from stego_b200.dino import vision_transformer as vits
    B = 16
    vit = vits.__dict__[arch](patch_size=8).to(cuda_dev)
    vit.load_state_dict(O.perturb_vit_state(O.vit_random_state(arch, 8, seed=3)))
    g = torch.Generator(device=cuda_dev).manual_seed(5)
    img = torch.randn(B, 3, res, res, device=cuda_dev, generator=g)
    flipped = img.flip(3).contiguous()
    for fn in (vit.patch_features, vit.key_features):
        want = torch.cat([fn(img), fn(flipped)], 0)
        eager = fn(img, mirror=True)
        assert eager.shape == (2 * B, (res // 8) ** 2, vit.embed_dim)
        assert torch.equal(eager, want), fn.__name__
        graphed = fn(img, use_graph=True, mirror=True)
        assert torch.equal(graphed, want), fn.__name__
        graphed = fn(img.flip(0).contiguous(), use_graph=True, mirror=True)  # the graph's static input is refilled
        assert torch.equal(graphed[:B], want[:B].flip(0)) and torch.equal(graphed[B:], want[B:].flip(0))
    keys = sorted(k[0] for k in vit._cache["graphs"])
    assert keys == ["KK+mirror", "feat+mirror"]
    static_in = vit.graph_input("feat+mirror", img.shape, img.device)
    assert static_in.shape == img.shape  # the graph holds B frames, not 2B


# ================================================================================================
# eval_step against the fused eval calls on two separate net() calls
# ================================================================================================
CASES = {
    # name: model overrides, n_classes, B, H, W, label dtype or None, label size (None: the frames')
    "feat_i64": (dict(), 27, 4, 64, 96, torch.int64, None),
    "kk_u8": (dict(dino_feat_type="KK"), 27, 4, 64, 64, torch.uint8, None),
    "linear_head_i32": (dict(projection_type="linear"), 27, 4, 64, 64, torch.int32, None),
    "3cls_extra2_i64": (dict(extra_clusters=2), 3, 3, 48, 64, torch.int64, None),
    "3cls_extra2_u8_label_96x128": (dict(extra_clusters=2), 3, 3, 48, 64, torch.uint8, (96, 128)),
    "no_label": (dict(), 27, 2, 64, 64, None, None),
    "bf16_frames_b1": (dict(), 27, 1, 64, 64, torch.int64, None),
    "vitb8_320_b4": (dict(model_type="vit_base"), 27, 4, 320, 320, torch.int64, None),
}


def _model(dev, over, n_classes, seed=0):
    import stego_oracle as O
    from stego_b200.config import make_cfg
    from stego_b200.segmenter import LitUnsupervisedSegmenter
    arch = over.get("model_type", "vit_small")
    torch.manual_seed(seed)
    model = LitUnsupervisedSegmenter(n_classes, make_cfg(random_backbone_init=True, **over)).to(dev)
    model.net.model.load_state_dict(O.perturb_vit_state(O.vit_random_state(arch, 8, seed=3)))
    with torch.no_grad():
        model.cluster_probe.clusters.normal_(generator=torch.Generator(device=dev).manual_seed(4))
    model.train()
    return model


def _case_batch(dev, case):
    _, n, B, H, W, ldt, lsize = CASES[case]
    g = torch.Generator(device=dev).manual_seed(9)
    img = torch.randn(B, 3, H, W, device=dev, generator=g)
    if case.startswith("bf16"):
        img = img.to(torch.bfloat16)
    if ldt is None:
        return dict(img=img)
    lh, lw = lsize or (H, W)
    label = torch.randint(0, n, (B, lh, lw), device=dev, generator=g)
    r = torch.rand(B, lh, lw, device=dev, generator=g)
    label[r < 0.05] = 255 if ldt == torch.uint8 else -1
    label[(r >= 0.05) & (r < 0.08)] = n
    return dict(img=img, label=label.to(ldt))


def _two_codes(model, img):
    """The codes of two eval-mode net() calls on img and img.flip(3): eval_segmentation.py:124-125."""
    model.flush()
    modes = [(m, m.training) for m in model.modules()]
    model.net.eval()
    with torch.no_grad():
        code1 = model.net(img)[1].clone()
        code2 = model.net(img.flip(3).contiguous())[1].clone()
    for m, mode in modes:
        m.training = mode
    return code1, code2


def _confusion(preds, label, n, rows):
    import eval_step_oracle as EO
    return EO.confusion(preds, label.long(), n, rows).to(preds.device)


@pytest.mark.parametrize("run_crf", [False, True])
@pytest.mark.parametrize("case", list(CASES))
def test_eval_step_bit_equal_to_fused_calls(cuda_dev, case, run_crf):
    from stego_b200 import _lib
    from stego_b200.eval import fused_eval_crf, fused_probe_log_probs
    over, n, B, H, W, ldt, lsize = CASES[case]
    if run_crf and (lsize is not None or over.get("model_type") == "vit_base"):
        pytest.skip("the CRF runs at the frames' size; ViT-B is covered without it")
    dev = cuda_dev
    model = _model(dev, over, n)
    batch = _case_batch(dev, case)
    img, label = batch["img"], batch.get("label")
    extra = over.get("extra_clusters", 0)
    rng = (torch.get_rng_state(), torch.cuda.get_rng_state(dev))
    modes = [m.training for m in model.modules()]
    launches = _lib.launch_count()
    got = model.eval_step(batch, run_crf=run_crf, want_probs=True)
    assert _lib.launch_count() > launches
    assert torch.equal(rng[0], torch.get_rng_state()) and torch.equal(rng[1], torch.cuda.get_rng_state(dev))
    assert modes == [m.training for m in model.modules()]
    assert sorted(got) == ["cluster_preds", "cluster_probs", "linear_preds", "linear_probs"]
    size = tuple(label.shape[-2:]) if label is not None else (H, W)
    for k, rows in (("linear", n), ("cluster", n + extra)):
        assert got[k + "_preds"].shape == (B,) + size and got[k + "_preds"].dtype == torch.uint8
        assert got[k + "_preds"].device == img.device
        assert got[k + "_probs"].shape == (B, rows) + size and got[k + "_probs"].dtype == torch.float32

    code1, code2 = _two_codes(model, img)
    lc = torch.zeros(n, n, dtype=torch.long, device=dev)
    cc = torch.zeros(n + extra, n, dtype=torch.long, device=dev)
    stats = dict(linear_confusion=lc, cluster_confusion=cc) if label is not None else {}
    if run_crf:
        la, ca, lq, cq = fused_eval_crf(code1, model.linear_probe, model.cluster_probe, img, 2.0, code_flipped=code2,
                                        label=label, want_marginals=True, **stats)
    else:
        lq, cq, la, ca = fused_probe_log_probs(code1, model.linear_probe, model.cluster_probe, size, 2.0,
                                               want_log_probs=True, want_argmax=True, code_flipped=code2, label=label,
                                               **stats)
    for k, want in (("linear_preds", la), ("cluster_preds", ca), ("linear_probs", lq), ("cluster_probs", cq)):
        assert torch.equal(got[k], want), (case, k)
    if label is None:
        assert not model.test_linear_metrics.stats.any() and not model.test_cluster_metrics.stats.any()
    else:
        assert torch.equal(model.test_linear_metrics.stats, lc) and torch.equal(model.test_cluster_metrics.stats, cc)
        assert torch.equal(lc, _confusion(got["linear_preds"], label, n, n))
        assert torch.equal(cc, _confusion(got["cluster_preds"], label, n, n + extra))
        assert int(lc.sum()) > 0
    assert not model.linear_metrics.stats.any() and not model.cluster_metrics.stats.any()  # validation's: untouched
    # a second call accumulates, and without want_probs returns the predictions alone
    again = model.eval_step(batch, run_crf=run_crf)
    assert sorted(again) == ["cluster_preds", "linear_preds"]
    assert torch.equal(again["linear_preds"], la) and torch.equal(again["cluster_preds"], ca)
    if label is not None:
        assert torch.equal(model.test_linear_metrics.stats, 2 * lc)


def test_refused_before_anything_is_enqueued(cuda_dev):
    from stego_b200 import _lib
    model = _model(cuda_dev, dict(extra_clusters=6), 27)
    batch = _case_batch(cuda_dev, "feat_i64")
    n0 = _lib.launch_count()
    with pytest.raises(ValueError, match="33 cluster-probe rows"):
        model.eval_step(batch)
    model = _model(cuda_dev, dict(), 27)
    with pytest.raises(ValueError, match="does not match img"):
        model.eval_step(dict(img=batch["img"], label=batch["label"][:, :32]), run_crf=True)
    with pytest.raises(RuntimeError, match="CUDA"):
        model.eval_step(dict(img=batch["img"], label=batch["label"].cpu()))
    torch.cuda.synchronize()
    assert _lib.launch_count() == n0
    assert not model.test_linear_metrics.stats.any() and not model.test_cluster_metrics.stats.any()


# ================================================================================================
# end to end against the reference loop in fp32 on the GPU
# ================================================================================================
@pytest.mark.parametrize("case", ["feat_i64", "kk_u8", "3cls_extra2_i64"])
def test_against_fp32_reference_loop(cuda_dev, case):
    """The reference loop (oracle/eval_step_oracle.py: fp32 ViT, F.interpolate, conv, log_softmax, ClusterLookup) on
    the same frames and weights.  With d the largest log-probability difference, a pixel whose reference top-2 margin
    exceeds 2 d must have the same argmax; d is what the bf16 ViT operands move the code by."""
    import eval_step_oracle as EO
    import stego_oracle as O
    over, n, B, H, W, _, _ = CASES[case]
    dev = cuda_dev
    model = _model(dev, over, n)
    batch = _case_batch(dev, case)
    got = model.eval_step(batch, want_probs=True)
    vit = {k: v.to(dev) for k, v in O.perturb_vit_state(O.vit_random_state("vit_small", 8, seed=3)).items()}
    head = {k[len("net."):]: v.detach() for k, v in model.named_parameters() if k.startswith("net.cluster")}
    with torch.no_grad():
        ref = EO.eval_loop(lambda im: EO.net_code(vit, head, im, feat_type=over.get("dino_feat_type", "feat")),
                           model.linear_probe.weight.detach(), model.linear_probe.bias.detach(),
                           model.cluster_probe.clusters.detach(), batch["img"], batch["label"], n)
    for k in ("linear", "cluster"):
        lp = ref[k + "_probs"]
        d = float((got[k + "_probs"] - lp).abs().max())
        top2 = lp.topk(2, 1).values
        safe = (top2[:, 0] - top2[:, 1]) > 2 * d
        agree = got[k + "_preds"].long() == ref[k + "_preds"]
        print(f"{case} {k}: max |d log p| {d:.3e}, near-tie pixels {float((~safe).double().mean()):.4f}, "
              f"argmax agreement {float(agree.double().mean()):.5f}")
        assert bool(agree[safe].all()), (case, k, int((~agree)[safe].sum()))
        assert d < 2e-2, (case, k, d)  # H100: 1.8e-3 ... 4.5e-3
        assert float(agree.double().mean()) > 0.97, (case, k)


# ================================================================================================
# eval_step and training
# ================================================================================================
def _train_state(model, dev):
    model.flush()
    torch.cuda.synchronize()
    f = model._flat
    return dict(param=f.param.clone(), grad=f.grad.clone(), exp_avg=f.exp_avg.clone(), exp_avg_sq=f.exp_avg_sq.clone(),
                cpu_rng=torch.get_rng_state(), cuda_rng=torch.cuda.get_rng_state(dev),
                adam_steps=torch.tensor([o.steps for o in f.optimizers]))


def _max_diff(a, b):
    return max(float((a[k].double() - b[k].double()).abs().max()) for k in ("param", "exp_avg", "exp_avg_sq"))


def test_eval_step_leaves_training_unchanged(cuda_dev):
    """4 fused steps, against 2 steps + eval_step (with and without CRF, fp32 and bf16 frames) + 2 steps.  Across the
    evaluation the training state is bit-identical (parameters, gradients, Adam moments and step counts, both RNG
    states), the training graphs are the same objects (replayed afterwards, never re-captured), the modes are restored;
    the two 4-step runs agree as closely as two runs without evaluation do."""
    dev = cuda_dev
    steps = [make_batch(4, 64, dev, seed=10 + i) for i in range(4)]
    evals = [make_batch(4, 64, dev, seed=50 + i) for i in range(2)]
    runs = {}
    for name in ("plain", "plain_again", "with_eval"):
        model, _ = make_model("vit_small", dev, fused=True, seed=0)
        torch.manual_seed(777)
        losses = []
        for i, batch in enumerate(steps):
            if name == "with_eval" and i == 2:
                fused = model._fused
                graph, key, vit_graphs = fused.ws.graph, fused.key, dict(model.net.model._cache["graphs"])
                assert graph is not None
                before, modes = _train_state(model, dev), [m.training for m in model.modules()]
                for j, v in enumerate(evals):
                    img = v["img"] if j == 0 else v["img"].to(torch.bfloat16)
                    for run_crf in (False, True):
                        model.eval_step(dict(img=img, label=v["label"]), run_crf=run_crf)
                        assert [m.training for m in model.modules()] == modes
                after = _train_state(model, dev)
                for k in before:
                    assert torch.equal(before[k], after[k]), k
                assert fused.ws.graph is graph and fused.key == key
                now = model.net.model._cache["graphs"]
                assert all(now[k] is v for k, v in vit_graphs.items())
                assert sorted(k[0] for k in set(now) - set(vit_graphs)) == ["feat+mirror", "feat+mirror"]
                assert int(model.test_linear_metrics.stats.sum()) > 0
            losses.append(model.training_step(batch, i).item())
        assert model._fused.step_idx == 4
        if name == "with_eval":
            assert model._fused.ws.graph is graph
        runs[name] = (losses, _train_state(model, dev))
    ref, again, val = runs["plain"], runs["plain_again"], runs["with_eval"]
    for k in ("cpu_rng", "cuda_rng", "adam_steps"):
        assert torch.equal(ref[1][k], val[1][k]), k
    noise = _max_diff(ref[1], again[1])
    noise_loss = max(abs(a - b) for a, b in zip(ref[0], again[0]))
    print(f"run-to-run: state {noise:.3e}, losses {noise_loss:.3e}; with eval_step: state "
          f"{_max_diff(ref[1], val[1]):.3e}, losses {max(abs(a - b) for a, b in zip(ref[0], val[0])):.3e}")
    if noise == 0 and noise_loss == 0:
        assert ref[0] == val[0]
        for k in ("param", "exp_avg", "exp_avg_sq"):
            assert torch.equal(ref[1][k], val[1][k]), k
    else:
        assert _max_diff(ref[1], val[1]) <= 4 * noise
        assert max(abs(a - b) for a, b in zip(ref[0], val[0])) <= 4 * noise_loss + 1e-7


def test_eval_step_right_after_training_step_sees_update(cuda_dev):
    from stego_b200.eval import fused_probe_log_probs
    dev = cuda_dev
    model, _ = make_model("vit_small", dev, fused=True, seed=0)
    ev = make_batch(4, 64, dev, seed=60)
    eb = dict(img=ev["img"], label=ev["label"])
    before = model.eval_step(eb)
    model.test_linear_metrics.reset()
    model.test_cluster_metrics.reset()
    torch.manual_seed(777)
    model.training_step(make_batch(4, 64, dev, seed=61), 0)
    got = model.eval_step(eb)
    code1, code2 = _two_codes(model, eb["img"])
    lc, cc = torch.zeros_like(model.test_linear_metrics.stats), torch.zeros_like(model.test_cluster_metrics.stats)
    _, _, la, ca = fused_probe_log_probs(code1, model.linear_probe, model.cluster_probe, eb["label"].shape[-2:], 2.0,
                                         want_log_probs=False, want_argmax=True, code_flipped=code2, label=eb["label"],
                                         linear_confusion=lc, cluster_confusion=cc)
    assert torch.equal(got["linear_preds"], la) and torch.equal(got["cluster_preds"], ca)
    assert torch.equal(model.test_linear_metrics.stats, lc) and torch.equal(model.test_cluster_metrics.stats, cc)
    assert not torch.equal(before["linear_preds"], got["linear_preds"])
