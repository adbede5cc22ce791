"""CPU: the attention-map / last-n-block oracle (oracle/vit_maps_oracle.py) against the reference's own outputs
(tests/golden/vit_small8_32px_maps.pt, written by oracle/make_golden_vit_maps.py), the n-edge semantics of
get_intermediate_feat, and argument checks of the attention-matrix entry points that run before any CUDA call."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import stego_oracle as O  # noqa: E402
import vit_maps_oracle as VM  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden", "vit_small8_32px_maps.pt")


def _inputs():
    sd = O.perturb_vit_state(O.vit_random_state("vit_small", 8, seed=3))
    torch.manual_seed(11)
    return sd, torch.randn(2, 3, 32, 32)


def _close(a, b):
    assert a.shape == b.shape
    assert (a - b).abs().max().item() <= 1e-5 * max(1.0, b.abs().max().item())


def test_oracle_matches_reference_fixture():
    g = torch.load(GOLD)
    sd, img = _inputs()
    with torch.no_grad():
        feat, attn, qkv = VM.vit_intermediate(sd, img, "vit_small", 8, n=3)
        layers, _, _ = VM.vit_intermediate(sd, img, "vit_small", 8, n=2)
        _, last, _ = VM.vit_intermediate(sd, img, "vit_small", 8, n=1)
    assert len(feat) == len(attn) == len(qkv) == len(g["feat3"]) == 3 and len(layers) == len(g["layers2"]) == 2
    _close(last[0], g["last_selfattention"])
    assert g["last_selfattention"].shape == (2, 6, 17, 17)
    for a, b in zip(feat, g["feat3"]):
        _close(a, b)
    for a, b in zip(attn, g["attn3"]):
        _close(a, b)
    for a, b in zip(qkv, g["qkv3"]):
        _close(a, b)
        assert b.shape == (3, 2, 6, 17, 64)
    for a, b in zip(layers, g["layers2"]):
        _close(a, b)
    # the last of get_intermediate_feat(n=3) is the output of get_intermediate_feat(n=1) (vit_small8_32px.pt)
    _close(feat[-1], torch.load(os.path.join(ROOT, "tests", "golden", "vit_small8_32px.pt"))["tokens"])


def test_n_edges():
    """n <= 0 keeps no block; n >= depth keeps every block; the kept blocks are the last n, oldest first."""
    sd, img = _inputs()
    img = img[:1]
    with torch.no_grad():
        for n in (0, -1):
            assert VM.vit_intermediate(sd, img, "vit_small", 8, n=n) == ([], [], [])
        all12 = VM.vit_intermediate(sd, img, "vit_small", 8, n=12)
        all40 = VM.vit_intermediate(sd, img, "vit_small", 8, n=40)
        two = VM.vit_intermediate(sd, img, "vit_small", 8, n=2)
    assert [len(t) for t in all12] == [len(t) for t in all40] == [12, 12, 12]
    for a, b in zip(all12, all40):
        for x, y in zip(a, b):
            assert torch.equal(x, y)
    for a, b in zip(all12, two):
        for x, y in zip(a[-2:], b):
            assert torch.equal(x, y)
    for attn in all12[1]:
        assert torch.allclose(attn.sum(-1), torch.ones(()), atol=1e-5)


def test_vit_entry_points_without_gpu():
    """get_intermediate_feat / get_intermediate_layers follow the reference for n <= 0 (empty lists); the computing
    entry points refuse CPU tensors (no CPU fallback); DinoFeaturizer rejects n < 1 (the reference indexes feat[0])."""
    from stego_b200.config import make_cfg
    from stego_b200.dino import vision_transformer as V
    from stego_b200.modules import DinoFeaturizer
    torch.manual_seed(0)
    vit = V.vit_small(patch_size=8)
    img = torch.randn(1, 3, 16, 16)
    assert vit.get_intermediate_feat(img, n=0) == ([], [], [])
    assert vit.get_intermediate_layers(img, n=-2) == []
    for call in (lambda: vit.get_last_selfattention(img), lambda: vit.get_intermediate_feat(img, n=2),
                 lambda: vit.get_intermediate_layers(img, n=3)):
        with pytest.raises(RuntimeError, match="no CPU fallback"):
            call()
    feat = DinoFeaturizer(70, make_cfg(random_backbone_init=True))
    with pytest.raises(ValueError):
        feat(img, n=0)


def test_attention_probs_abi_rejects_bad_arguments():
    from stego_b200 import _lib
    lib = _lib.load()
    ok = dict(qkv=256, probs=256, B=2, N=17, E=384, heads=6)

    def call(**kw):
        a = {**ok, **kw}
        return lib.stego_attention_probs(a["qkv"], a["probs"], a["B"], a["N"], a["E"], a["heads"], 0)

    assert call(qkv=0) == -1 and "null pointer" in _lib.last_error()
    assert call(probs=0) == -1 and "null pointer" in _lib.last_error()
    assert call(E=320) == -1 and "head_dim" in _lib.last_error()
    assert call(probs=258) == -1 and "aligned" in _lib.last_error()
    for bad in (dict(B=0), dict(N=0), dict(heads=0), dict(N=-5)):
        assert call(**bad) == -1 and "bad sizes" in _lib.last_error()
    assert call(B=70000) == -1 and "65535" in _lib.last_error()
