"""CPU: dino_feat_type "KK" (src/modules.py:98-101, the last block's keys as the teacher features).

  * the oracle's "KK" step (oracle/kk_oracle.py keys -> stego_oracle.training_losses) reproduces the REFERENCE's own
    training_step with dino_feat_type "KK" (oracle/make_golden_kk_step.py, stub-Lightning harness) at the bars of
    test_true_labels.py, and the oracle's descriptors reproduce the reference's get_feats (src/precompute_knns.py:15-21);
  * stego_linear_rows_f32, the projection of the "KK" kNN descriptors, rejects bad arguments before any CUDA call, and
    its Python wrapper refuses CPU tensors.
"""
import os
import sys
import tempfile

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))


def _golden():
    return torch.load(os.path.join(ROOT, "tests", "golden", "kk_step.pt"))


def _oracle_keys():
    import kk_oracle as KK
    import lightning_harness as H
    import make_golden_kk_step as MK
    with tempfile.TemporaryDirectory() as td:
        sd = H.write_random_dino_checkpoint(os.path.join(td, "dino.pth"), "vit_small")
    batch = MK.step_batch()
    with torch.no_grad():
        f = KK.vit_image_keys(sd, batch["img"], "vit_small", 8)
        fp = KK.vit_image_keys(sd, batch["img_pos"], "vit_small", 8)
    return batch, f, fp


def test_oracle_matches_reference_training_step_with_keys():
    import make_golden as MG
    import stego_oracle as O
    want = _golden()["training_step"]
    batch, f, fp = _oracle_keys()
    assert f.shape == (MG.STEP_B, 384, 8, 8)
    p0 = MG.step_params()
    masks, masks_pos, c1, c2, perms = MG.step_draws()  # same RNG order as the "feat" step: net() draws its noises
    hp = {k[len("net."):]: v.clone().requires_grad_(True) for k, v in p0.items() if k.startswith("net.")}
    probes = {k: v.clone().requires_grad_(True) for k, v in p0.items() if not k.startswith("net.")}
    out = O.training_losses(f, fp, hp, probes, batch["label"], masks, masks_pos, c1, c2, perms, O.LossCfg(), 27)
    out["total"].backward()
    assert abs(want["loss"] - out["total"].item()) < 2e-6 * abs(out["total"].item())
    for k_log, k_or in [("loss/pos_intra", "pos_intra"), ("loss/pos_inter", "pos_inter"), ("loss/neg_inter", "neg_inter"),
                        ("loss/linear", "linear"), ("loss/cluster", "cluster"), ("cd/pos_intra", "cd_intra"),
                        ("cd/pos_inter", "cd_inter"), ("cd/neg_inter", "cd_neg")]:
        assert abs(want["logged"][k_log] - out[k_or].item()) < 1e-5 * abs(out[k_or].item()) + 1e-7, k_log
    mine_g = {("net." + k): v.grad for k, v in hp.items()}
    mine_g.update({k: v.grad for k, v in probes.items()})
    for k in MG.STEP_NAMES:
        g = want["grads"][k]
        idx = g["idx"].long()
        mine = mine_g[k].reshape(-1)
        assert abs(mine.norm().item() - g["norm"]) <= 1e-4 * mine.norm().item() + 1e-10, k
        assert (g["values"] - mine[idx]).norm() <= 1e-4 * mine[idx].norm() + 1e-10, k
        p = p0[k].reshape(-1)[idx].clone()
        O.adam_step(p, g["values"], torch.zeros_like(p), torch.zeros_like(p), 1, 5e-4 if k.startswith("net.") else 5e-3)
        assert (want["params_after"][k] - p).abs().max().item() < 1e-7, k


def test_keys_step_differs_from_feat_step():
    """The golden "KK" step is not the "feat" step: the teacher choice reaches the loss."""
    feat = torch.load(os.path.join(ROOT, "tests", "golden", "reference_pins.pt"))["training_step"]
    kk = _golden()["training_step"]
    assert abs(feat["loss"] - kk["loss"]) > 1e-4 * abs(kk["loss"])


def test_oracle_matches_reference_get_feats_with_keys():
    import stego_oracle as O
    want = _golden()["descriptors"]
    _, f, fp = _oracle_keys()
    got = O.knn_descriptors(torch.cat([f, fp], 0))
    assert got.shape == want.shape == (4, 384)
    assert (got - want).abs().max().item() < 1e-6


def test_linear_rows_symbol_and_argument_checks():
    from stego_b200 import _lib, ops
    assert "stego_linear_rows_f32" in _lib.header_prototypes()
    lib = _lib.load()
    P = 1 << 12  # a 16-byte-aligned non-null value: the checks run before any pointer is touched

    def call(x=P, w=P, ldw=384, bias=0, out=P, B=2, N=384, K=384):
        return lib.stego_linear_rows_f32(x, w, ldw, bias, out, B, N, K, 0)

    for kw, msg in [(dict(x=0), "null pointer"), (dict(w=0), "null pointer"), (dict(out=0), "null pointer"),
                    (dict(B=0), "bad sizes"), (dict(N=-1), "bad sizes"), (dict(K=100), "bad sizes"),
                    (dict(ldw=376), "ldw"), (dict(ldw=390), "ldw"), (dict(x=P + 4), "aligned"),
                    (dict(w=P + 8), "aligned")]:
        assert call(**kw) == -1, kw
        assert msg in _lib.last_error(), (kw, _lib.last_error())
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.linear_rows_f32(torch.zeros(2, 384), torch.zeros(384, 384, dtype=torch.bfloat16))


def test_unknown_feat_type_is_refused():
    from types import SimpleNamespace
    from stego_b200.knn import knn_descriptors
    from stego_b200.modules import DinoFeaturizer
    net = SimpleNamespace(feat_type="QQ")
    with pytest.raises(ValueError, match="Unknown feat type"):
        knn_descriptors(net, torch.zeros(1, 3, 8, 8))
    fake = SimpleNamespace(feat_type="QQ", patch_size=8, model=SimpleNamespace(eval=lambda: None))
    with pytest.raises(ValueError, match="Unknown feat type"):
        DinoFeaturizer.backbone_tokens(fake, torch.zeros(1, 3, 8, 8))
