"""CPU: the evaluation loop body LitUnsupervisedSegmenter.eval_step runs (eval_segmentation.py:122-141).

  * oracle/eval_step_oracle.py, the plain-torch restatement the GPU tests hold eval_step to, reproduces the reference's
    own loop (tests/golden/eval_step.pt, written by oracle/make_golden_eval_step.py): codes and log-probabilities to
    fp32 rounding, argmax maps and confusion matrices exactly;
  * eval_step refuses what its kernels would refuse before anything is enqueued, and leaves the metrics untouched;
  * the header declares stego_vit_patchify_tta and the library exports it; the entry refuses the patchify rules' bad
    arguments without a GPU.
"""
import ctypes
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
GOLD = os.path.join(ROOT, "tests", "golden", "eval_step.pt")


# ================================================================================================
# the oracle loop against the reference's own outputs
# ================================================================================================
def test_oracle_loop_matches_reference_golden():
    import eval_step_oracle as EO
    import make_golden_eval_step as MG
    import stego_oracle as O
    g = torch.load(GOLD, weights_only=False)
    assert (g["n_classes"], g["extra_clusters"]) == (MG.N_CLASSES, MG.EXTRA)
    p = MG.params()
    vit = O.perturb_vit_state(O.vit_random_state("vit_small", 8, seed=3))
    head = {k[len("net."):]: v for k, v in p.items() if k.startswith("net.")}
    lin_stats = torch.zeros(MG.N_CLASSES, MG.N_CLASSES, dtype=torch.long)
    clu_stats = torch.zeros(MG.N_CLASSES + MG.EXTRA, MG.N_CLASSES, dtype=torch.long)
    with torch.no_grad():
        for batch, want in zip(MG.inputs(), g["steps"]):
            got = EO.eval_loop(lambda im: EO.net_code(vit, head, im), p["linear_probe.weight"], p["linear_probe.bias"],
                               p["cluster_probe.clusters"], batch["img"], batch["label"], MG.N_CLASSES)
            for k in ("code1", "code2"):
                err = float((got[k] - want[k]).abs().max() / want[k].abs().max())
                assert err < 1e-5, (k, err)
            for k in ("linear_probs", "cluster_probs"):
                assert got[k].shape == want[k].shape == (2, want[k].shape[1]) + tuple(batch["label"].shape[-2:])
                assert float((got[k] - want[k]).abs().max()) < 1e-5, k
            for k in ("linear_preds", "cluster_preds"):
                assert torch.equal(got[k].to(torch.uint8), want[k]), (k, int((got[k] != want[k].long()).sum()))
            lin_stats += got["linear_stats"]
            clu_stats += got["cluster_stats"]
            assert torch.equal(lin_stats, want["linear_stats"]) and torch.equal(clu_stats, want["cluster_stats"])
    assert int(clu_stats.sum()) > 0 and bool((g["steps"][0]["cluster_preds"] >= MG.N_CLASSES).any())


# ================================================================================================
# argument errors, before anything is enqueued
# ================================================================================================
def _model(n_classes=5, **over):
    from stego_b200.config import make_cfg
    from stego_b200.segmenter import LitUnsupervisedSegmenter
    torch.manual_seed(0)
    return LitUnsupervisedSegmenter(n_classes, make_cfg(random_backbone_init=True, **over))


def _batch(B=2, H=32, W=48, label_hw=None, dtype=torch.int64):
    g = torch.Generator().manual_seed(3)
    lh, lw = label_hw or (H, W)
    return dict(img=torch.randn(B, 3, H, W, generator=g), label=torch.randint(0, 5, (B, lh, lw), generator=g).to(dtype))


def _refused(model, batch, exc, words, **kw):
    stats = (model.test_linear_metrics.stats.clone(), model.test_cluster_metrics.stats.clone())
    modes = [m.training for m in model.modules()]
    with pytest.raises(exc) as e:
        model.eval_step(batch, **kw)
    for w in words:
        assert w in str(e.value), (w, str(e.value))
    assert torch.equal(stats[0], model.test_linear_metrics.stats)
    assert torch.equal(stats[1], model.test_cluster_metrics.stats)
    assert modes == [m.training for m in model.modules()]


@pytest.mark.parametrize("run_crf", [False, True])
def test_cpu_tensors_refused(run_crf):
    model = _model()
    _refused(model, _batch(), RuntimeError, ["CUDA"], run_crf=run_crf)
    _refused(model, dict(img=_batch()["img"]), RuntimeError, ["CUDA"], run_crf=run_crf)


def test_crf_label_must_have_the_frames_size():
    """fused_eval_crf's own rule (the dense CRF runs at image resolution), raised from its own check."""
    model = _model()
    _refused(model, _batch(label_hw=(48, 48)), ValueError, ["fused_eval_crf", "does not match img"], run_crf=True)


@pytest.mark.parametrize("H,W", [(32, 36), (36, 32), (32, 44)])
def test_frames_not_whole_patches_refused(H, W):
    model = _model()
    for run_crf in (False, True):
        _refused(model, _batch(H=H, W=W), ValueError, ["patches", "multiple of 8"], run_crf=run_crf)


def test_patch_size_rule():
    """The model only builds patch 8 and 16; a featurizer whose patch size was changed afterwards is refused."""
    model = _model()
    model.net.patch_size = 12
    _refused(model, _batch(H=36, W=48), ValueError, ["patch 8 or 16"])


@pytest.mark.parametrize("case", ["projection_none", "33_cluster_rows", "32_classes_1_extra"])
def test_refused_probe_sizes(case):
    if case == "projection_none":
        model, words = _model(projection_type=None), ["projection_type None", "384 channels"]
    elif case == "33_cluster_rows":
        model, words = _model(n_classes=30, extra_clusters=3), ["33 cluster-probe rows"]
    else:
        model, words = _model(n_classes=32, extra_clusters=1), ["33 cluster-probe rows"]
    for run_crf in (False, True):
        _refused(model, _batch(), ValueError, words, run_crf=run_crf)


def test_bad_labels_refused():
    model = _model()
    _refused(model, _batch(dtype=torch.float32), ValueError, ["label dtype"])
    b = _batch()
    _refused(model, dict(img=b["img"], label=b["label"][:1]), ValueError, ["per frame"])
    _refused(model, _batch(label_hw=(2, 3)), ValueError, ["upsampling only"])
    _refused(model, dict(img=b["img"].double(), label=b["label"]), ValueError, ["fp32 or bf16"])


# ================================================================================================
# the C-ABI entry
# ================================================================================================
def test_header_declares_and_library_exports_patchify_tta():
    from stego_b200 import _lib
    protos = _lib.header_prototypes()
    assert protos["stego_vit_patchify_tta"] == ("int", ["const void*", "int", "void*", "int", "int", "int", "int",
                                                        "void*"])
    assert hasattr(ctypes.CDLL(_lib.LIB_PATH), "stego_vit_patchify_tta")
    # the existing entries keep their signatures
    assert protos["stego_vit_patchify"] == ("int", ["const float*", "void*", "int", "int", "int", "int", "void*"])
    assert protos["stego_vit_patchify_bf16"] == ("int", ["const void*", "void*", "int", "int", "int", "int", "void*"])


@pytest.mark.parametrize("args,words", [
    (dict(patch=12), "patch size 12 unsupported"),
    (dict(W=36), "bad image"),
    (dict(H=20), "bad image"),
    (dict(B=0), "bad image"),
    (dict(img=8), "not 16-byte aligned"),
    (dict(img=0), "null pointer"),
])
def test_patchify_tta_refuses_bad_arguments(args, words):
    """Refused before any CUDA call (host addresses stand in for the buffers)."""
    from stego_b200 import _lib
    buf = torch.zeros(64, dtype=torch.float32)
    a = dict(img=buf.data_ptr(), bf16=0, out=buf.data_ptr(), B=2, H=32, W=32, patch=8)
    a.update({k: (buf.data_ptr() + v if k == "img" and v else v) for k, v in args.items()})
    for bf16 in (0, 1):
        rc = _lib.load().stego_vit_patchify_tta(a["img"], bf16, a["out"], a["B"], a["H"], a["W"], a["patch"], 0)
        assert rc != 0 and words in _lib.last_error() and "stego_vit_patchify_tta" in _lib.last_error()
