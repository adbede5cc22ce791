"""CPU: the DINO baseline configuration (projection_type None, dim = the backbone's width; the paper's "DINO" row).

  * construction accepts dim 384 for ViT-S and 768 for ViT-B with projection_type None, and no other width above 96;
  * its state-dict keys are the reference's for that configuration: cluster1 present, no cluster2;
  * training_step refuses, before anything is launched, what the baseline cannot train: another dim, the correspondence,
    reconstruction, aug-alignment and CRF terms;
  * the header declares the bf16 eval entries and the library exports them; the eval entries refuse every width but
    1..96 (fp32) and 384 / 768 (fp32 or bf16) without touching the GPU.
"""
import ctypes
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BF16_ENTRIES = ["stego_eval_probes_bf16", "stego_eval_probes_mosaic_bf16", "stego_eval_crf_unary_bf16",
                "stego_eval_crf_unary_mosaic_bf16"]


def _model(n_classes=5, **over):
    from stego_b200.config import make_cfg
    from stego_b200.segmenter import LitUnsupervisedSegmenter
    torch.manual_seed(0)
    return LitUnsupervisedSegmenter(n_classes, make_cfg(random_backbone_init=True, **over))


@pytest.mark.parametrize("arch,dim", [("vit_small", 384), ("vit_base", 768)])
def test_baseline_builds_at_the_backbone_width(arch, dim):
    m = _model(model_type=arch, projection_type=None, dim=dim)
    assert m.net.dim == m.net.n_feats == dim
    assert m.linear_probe.weight.shape == (5, dim, 1, 1) and m.cluster_probe.clusters.shape == (5, dim)
    keys = set(m.state_dict())
    assert {"net.cluster1.0.weight", "net.cluster1.0.bias"} <= keys
    assert not any(k.startswith("net.cluster2") for k in keys)


@pytest.mark.parametrize("over", [
    dict(projection_type=None, dim=97),
    dict(projection_type=None, dim=383),
    dict(projection_type=None, dim=768),                        # ViT-S is 384 wide
    dict(model_type="vit_base", projection_type=None, dim=384),  # ViT-B is 768 wide
    dict(projection_type="linear", dim=384),                     # a head is at most 96 wide
    dict(projection_type="nonlinear", dim=384),
])
def test_other_wide_codes_refused_at_construction(over):
    with pytest.raises(RuntimeError, match="96"):
        _model(**over)


def _step_batch():
    g = torch.Generator().manual_seed(1)
    return dict(img=torch.randn(2, 3, 32, 32, generator=g), img_pos=torch.randn(2, 3, 32, 32, generator=g),
                label=torch.randint(0, 5, (2, 32, 32), generator=g))


@pytest.mark.parametrize("over,words", [
    (dict(dim=70), "reference cannot run"),
    (dict(dim=384, correspondence_weight=1.0), "correspondence_weight"),
    (dict(dim=384, correspondence_weight=0.0, rec_weight=1.0), "rec_weight"),
    (dict(dim=384, correspondence_weight=0.0, aug_alignment_weight=1.0), "aug_alignment_weight"),
    (dict(dim=384, correspondence_weight=0.0, crf_weight=1.0), "crf_weight"),
])
def test_baseline_step_refusals_before_any_launch(over, words):
    from stego_b200 import _lib
    m = _model(projection_type=None, **over)
    rng = torch.get_rng_state()
    n = _lib.launch_count()
    with pytest.raises(ValueError, match=words):
        m.training_step(_step_batch(), 0)
    assert _lib.launch_count() == n and m.global_step == 0 and torch.equal(rng, torch.get_rng_state())


def test_eval_refusal_keeps_naming_the_width():
    """projection_type None with the probes at another dim: the reference cannot run it either."""
    m = _model(projection_type=None)
    with pytest.raises(ValueError) as e:
        m.eval_step(dict(img=torch.randn(1, 3, 32, 32)))
    assert "projection_type None" in str(e.value) and "384 channels" in str(e.value)


def test_header_declares_and_library_exports_bf16_entries():
    from stego_b200 import _lib
    protos = _lib.header_prototypes()
    lib = _lib.load()
    for name in BF16_ENTRIES + ["stego_cluster_lookup_wide", "stego_linear_probe_ce_wide"]:
        assert name in protos, name
        getattr(lib, name)
    # same arguments as the fp32 entries, the code pointers untyped
    for name in BF16_ENTRIES:
        want = list(protos[name[:-len("_bf16")]][1])
        want[0] = want[1] = "const void*"
        assert protos[name][1] == want, name


def _probes(lib, name, C):
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    lr = ctypes.cast((ctypes.c_double * 16)(), ctypes.c_void_p)
    return getattr(lib, name)(p, None, C, C, 1, 2, 2, 16, 16, p, p, 5, p, 5, 2.0, lr, p, p, None, None, None, 0, 0,
                              None, None, None)


@pytest.mark.parametrize("name,C", [("stego_eval_probes", 97), ("stego_eval_probes", 383), ("stego_eval_probes", 769),
                                    ("stego_eval_probes_bf16", 70), ("stego_eval_probes_bf16", 96),
                                    ("stego_eval_probes_bf16", 500)])
def test_eval_entries_refuse_other_widths(name, C):
    from stego_b200 import _lib
    lib = _lib.load()
    n = _lib.launch_count()
    assert _probes(lib, name, C) != 0
    assert _lib.launch_count() == n


# ================================================================================================
# the oracle restatement against the reference's own evaluation of the baseline
# ================================================================================================
GOLD = os.path.join(ROOT, "tests", "golden", "baseline.pt")


def test_oracle_matches_reference_golden():
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import baseline_oracle as BO
    import eval_step_oracle as EO
    import make_golden_baseline as MB
    import make_golden_eval_step as ME
    import stego_oracle as O
    g = torch.load(GOLD, weights_only=False)
    assert (g["n_classes"], g["extra_clusters"], g["dim"]) == (MB.N_CLASSES, MB.EXTRA, 384)
    p = MB.params()
    vit = O.perturb_vit_state(O.vit_random_state("vit_small", 8, seed=3))
    code_fn = lambda im: BO.net_code(vit, im)
    n = MB.N_CLASSES
    for key, tta in (("no_tta", False), ("tta", True)):
        lin_stats = torch.zeros(n, n, dtype=torch.long)
        clu_stats = torch.zeros(n + MB.EXTRA, n, dtype=torch.long)
        with torch.no_grad():
            for batch, want in zip(ME.inputs(), g[key]):
                # without TTA the mirrored code is the code of the unflipped frame, mirrored: the average is the code
                fn = code_fn if tta else (lambda im, b=batch: code_fn(b["img"]).flip(dims=[3]) if im is not b["img"]
                                          else code_fn(im))
                got = EO.eval_loop(fn, p["linear_probe.weight"], p["linear_probe.bias"], p["cluster_probe.clusters"],
                                   batch["img"], batch["label"], n)
                if tta:
                    err = float((got["code1"] - want["code1"]).abs().max() / want["code1"].abs().max())
                    assert err < 1e-5, err
                for k in ("linear_probs", "cluster_probs"):
                    assert float((got[k] - want[k]).abs().max()) < 1e-5, (key, k)
                for k in ("linear_preds", "cluster_preds"):
                    assert torch.equal(got[k].to(torch.uint8), want[k]), (key, k)
                lin_stats += got["linear_stats"]
                clu_stats += got["cluster_stats"]
                assert torch.equal(lin_stats, want["linear_stats"]) and torch.equal(clu_stats, want["cluster_stats"])
    assert int(clu_stats.sum()) > 0


def test_state_dict_keys_are_the_reference_s():
    g = torch.load(GOLD, weights_only=False)
    m = _model(extra_clusters=2, projection_type=None, dim=384, correspondence_weight=0.0)
    assert sorted(m.state_dict().keys()) == g["state_dict_keys"]


def test_wide_probe_entries_refuse_other_widths_and_classes():
    from stego_b200 import _lib
    lib = _lib.load()
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    n = _lib.launch_count()
    for C, k in ((383, 5), (96, 5), (768, 65), (384, 0)):
        assert lib.stego_cluster_lookup_wide(p, C, 4, C, p, k, p, p, p, p, p, p, None) != 0, (C, k)
    assert lib.stego_cluster_lookup_wide(p, 384, 4, 384, p, 5, p, p, p, p, None, p, None) != 0  # no dnc scratch
    for C in (97, 383, 384, 768, 769):  # the wide widths have their own entry
        assert lib.stego_linear_probe_ce(p, C, C, p, p, 5, p, 8, 1, 2, 2, 16, 16, p, p, p, p, 1.0, p, p, None) != 0
    for C in (70, 96, 383, 769):
        assert lib.stego_linear_probe_ce_wide(p, C, C, p, p, 5, p, 8, 1, 2, 2, 16, 16, p, p, p, p, p, 1.0, p, p,
                                              None) != 0
    # the backward without its fixed-point scratch
    assert lib.stego_linear_probe_ce_wide(p, 384, 384, p, p, 5, p, 8, 1, 2, 2, 16, 16, p, p, None, p, p, 1.0, p, p,
                                          None) != 0
    assert _lib.launch_count() == n


def test_training_restatement_matches_reference_golden():
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import baseline_oracle as BO
    import make_golden_baseline as MB
    import stego_oracle as O
    g = torch.load(GOLD, weights_only=False)
    vit = O.perturb_vit_state(O.vit_random_state("vit_small", 8, seed=3))
    got = BO.training_steps(vit, MB.params(), MB.step_batches(), MB.N_CLASSES)
    assert len(got) == len(g["train"]) == 2
    for s, want in zip(got, g["train"]):
        for k in ("loss/linear", "loss/cluster", "loss/total"):
            assert abs(s["logged"][k] - want["logged"][k]) < 1e-5, (k, s["logged"][k], want["logged"][k])
        for k, v in want["params"].items():
            assert float((s["params"][k] - v).abs().max()) < 1e-6, k
    # the probes moved: Adam at lr 5e-3
    assert float((g["train"][1]["params"]["cluster_probe.clusters"] - MB.params()["cluster_probe.clusters"]).abs().max()) > 1e-3
