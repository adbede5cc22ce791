"""CPU: pins the oracle's restatement of the training step (oracle/stego_oracle.py::training_losses, adam_step —
src/train_segmentation.py:112-245, 373-383) against the REFERENCE's own LitUnsupervisedSegmenter.training_step, executed
unmodified through the stub-Lightning harness (oracle/lightning_harness.py) by oracle/make_golden.py; its outputs are
stored in tests/golden/reference_pins.pt."""
import os
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))


def _pins():
    return torch.load(os.path.join(ROOT, "tests", "golden", "reference_pins.pt"))


def test_oracle_training_step_matches_reference_training_step():
    import lightning_harness as H
    import make_golden as MG
    import stego_oracle as O
    want = _pins()["training_step"]
    B = MG.STEP_B
    with tempfile.TemporaryDirectory() as td:
        sd = H.write_random_dino_checkpoint(os.path.join(td, "dino.pth"), "vit_small")
    batch = H.make_batch(B, MG.STEP_RES, "cpu")
    p0 = MG.step_params()
    masks, masks_pos, c1, c2, perms = MG.step_draws()
    with torch.no_grad():
        f = O.vit_image_feat(sd, batch["img"], "vit_small", 8)
        fp = O.vit_image_feat(sd, batch["img_pos"], "vit_small", 8)
    hp = {k[len("net."):]: v.clone().requires_grad_(True) for k, v in p0.items() if k.startswith("net.")}
    probes = {k: v.clone().requires_grad_(True) for k, v in p0.items() if not k.startswith("net.")}
    out = O.training_losses(f, fp, hp, probes, batch["label"], masks, masks_pos, c1, c2, perms, O.LossCfg(), 27)
    out["total"].backward()
    assert abs(want["loss"] - out["total"].item()) < 2e-6 * abs(out["total"].item())
    for k_log, k_or in [("loss/pos_intra", "pos_intra"), ("loss/pos_inter", "pos_inter"), ("loss/neg_inter", "neg_inter"),
                        ("loss/linear", "linear"), ("loss/cluster", "cluster"), ("cd/pos_intra", "cd_intra"),
                        ("cd/pos_inter", "cd_inter"), ("cd/neg_inter", "cd_neg")]:
        assert abs(want["logged"][k_log] - out[k_or].item()) < 1e-5 * abs(out[k_or].item()) + 1e-7, k_log
    want_g = {("net." + k): v.grad for k, v in hp.items()}
    want_g.update({k: v.grad for k, v in probes.items()})
    for k in MG.STEP_NAMES:
        g = want["grads"][k]
        idx = g["idx"].long()
        mine = want_g[k].reshape(-1)
        # the reference's gradient (a fixed sample of it, and its full norm) against the oracle's
        assert abs(mine.norm().item() - g["norm"]) <= 1e-4 * mine.norm().item() + 1e-10, k
        assert (g["values"] - mine[idx]).norm() <= 1e-4 * mine[idx].norm() + 1e-10, k
        # the reference's torch.optim.Adam update vs the oracle's adam_step on the reference's gradient
        p = p0[k].reshape(-1)[idx].clone()
        O.adam_step(p, g["values"], torch.zeros_like(p), torch.zeros_like(p), 1, 5e-4 if k.startswith("net.") else 5e-3)
        assert (want["params_after"][k] - p).abs().max().item() < 1e-7, k


def test_knn_oracle_matches_lifted_reference_lines():
    """The kNN restatement (oracle knn_descriptors / knn_indices) against the reference's own statements: `get_feats`
    (src/precompute_knns.py:15-21) and the slab loop (:83-92), lifted as TEXT from the reference file and executed by
    oracle/make_golden.py on the same feature maps."""
    import make_golden as MG
    import stego_oracle as O
    want = _pins()["knn"]
    want_feats, want_nn = want["normed_feats"], want["nearest_neighbors"]
    desc = torch.cat([O.knn_descriptors(f) for f in MG.knn_feature_maps()], 0)
    assert torch.allclose(desc, want_feats, atol=1e-7)
    idx, _ = O.knn_indices(desc, k=30, n_batches=4)
    assert idx.shape == want_nn.shape == (40, 30)
    assert torch.equal(idx, want_nn)
