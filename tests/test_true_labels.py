"""CPU: the pieces of cfg.use_true_labels (train_segmentation.py:135-140) that need no GPU.

  * oracle/true_labels_oracle.py, the restatement the GPU tests check against, reproduces the REFERENCE's own
    training_step with use_true_labels (oracle/make_golden_true_labels.py, stub-Lightning harness) and the reference
    module's 6-tuple on a one-hot signal at 4x the code's resolution, at the bars of test_reference_harness.py;
  * stego_sample_labels_fwd is referenced from exactly one function of the package (corr.build_label_tiles), as the
    shared entry points of test_step_stages.py are;
  * the symbol is exported and rejects bad arguments before any CUDA call.
"""
import os
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def _golden():
    return torch.load(os.path.join(ROOT, "tests", "golden", "true_labels_step.pt"))


def test_oracle_matches_reference_training_step_with_true_labels():
    import lightning_harness as H
    import make_golden as MG
    import make_golden_true_labels as MT
    import stego_oracle as O
    import true_labels_oracle as TL
    want = _golden()["training_step"]
    B = MG.STEP_B
    with tempfile.TemporaryDirectory() as td:
        sd = H.write_random_dino_checkpoint(os.path.join(td, "dino.pth"), "vit_small")
    batch = MT.step_batch()
    assert (batch["label"] == -1).any() and (batch["label_pos"] == -1).any()
    assert not torch.equal(batch["label"], batch["label_pos"])
    p0 = MG.step_params()
    masks, masks_pos, c1, c2, perms = MG.step_draws()  # the RNG order is the shipped step's: net() draws its noises
    with torch.no_grad():
        f = O.vit_image_feat(sd, batch["img"], "vit_small", 8)
        fp = O.vit_image_feat(sd, batch["img_pos"], "vit_small", 8)
    hp = {k[len("net."):]: v.clone().requires_grad_(True) for k, v in p0.items() if k.startswith("net.")}
    probes = {k: v.clone().requires_grad_(True) for k, v in p0.items() if not k.startswith("net.")}
    out = TL.training_losses(f, fp, hp, probes, batch["label"], batch["label_pos"], masks, masks_pos, c1, c2, perms,
                             O.LossCfg(), 27)
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


def test_oracle_matches_reference_module_on_one_hot_signal():
    import make_golden_true_labels as MT
    import stego_oracle as O
    import true_labels_oracle as TL
    want = _golden()["module"]
    label, label_pos, code, code_pos = MT.module_inputs()
    assert tuple(label.shape[-2:]) == (4 * code.shape[-2], 4 * code.shape[-1]) and (label == -1).any()
    code.requires_grad_(True)
    code_pos.requires_grad_(True)
    sig, sig_pos = TL.label_signals(label, label_pos, MT.N_CLASSES)
    assert sig.shape[1] == 28 and sig.dtype == torch.float32
    perms = list(want["perms"])
    o = O.correlation_loss(sig, sig_pos, code, code_pos, want["coords1"], want["coords2"], perms, O.LossCfg())
    loss = .67 * o[0] + .25 * o[2] + .63 * o[4].mean()
    loss.backward()
    for got, ref in ((o[0], want["pos_intra_loss"]), (o[2], want["pos_inter_loss"]),
                     (o[4].mean(), want["neg_inter_loss_mean"]), (loss, want["total"])):
        assert abs(got.item() - ref.item()) < 1e-6 + 1e-5 * abs(ref.item())
    assert (torch.stack([o[1].mean(), o[3].mean(), o[5].mean()]) - want["cd_means"]).abs().max() < 1e-6
    assert (o[3].detach().reshape(-1)[::53] - want["inter_cd_sub"]).abs().max() < 1e-6
    assert (o[4].detach().reshape(-1)[::53] - want["neg_loss_sub"]).abs().max() < 1e-6
    for mine, ref in ((code.grad, want["code_grad"]), (code_pos.grad, want["code_pos_grad"])):
        assert (mine - ref).norm() <= 1e-5 * ref.norm()


def test_sample_labels_entry_point_has_one_call_site():
    from test_step_stages import _referencing_functions, SHARED_ENTRY_POINTS
    SHARED_ENTRY_POINTS.append("stego_sample_labels_fwd")
    try:
        sites = _referencing_functions()["stego_sample_labels_fwd"]
    finally:
        SHARED_ENTRY_POINTS.remove("stego_sample_labels_fwd")
    assert sites == {"stego_b200/corr.py:build_label_tiles"}, sites


def test_sample_labels_symbol_and_argument_checks():
    import ctypes
    from stego_b200 import _lib
    assert hasattr(ctypes.CDLL(_lib.LIB_PATH), "stego_sample_labels_fwd")
    lib = _lib.load()
    P = 4096  # a non-null address: every case below must be refused before anything is read

    def call(label=P, label_pos=P, nbytes=8, c1=P, c2=P, perms=P, tiles=P, B=2, n=27, cpad=64, H=8, W=8, fs=11,
             nslots=7):
        return lib.stego_sample_labels_fwd(label, label_pos, nbytes, c1, c2, perms, tiles, B, n, cpad, H, W, fs, nslots,
                                           1, 0)

    for kw, what in [(dict(label=0), "null"), (dict(label_pos=0), "null"), (dict(c1=0), "null"),
                     (dict(tiles=0), "null tiles"), (dict(perms=0), "perms"), (dict(nbytes=2), "label_bytes"),
                     (dict(n=256, cpad=256), "n_classes"), (dict(n=300, cpad=320), "n_classes"),
                     (dict(n=0), "n_classes"), (dict(n=27, cpad=32), "Cpad"), (dict(n=100, cpad=64), "Cpad"),
                     (dict(n=27, cpad=384), "Cpad"), (dict(H=1), "H="), (dict(W=1), "W="), (dict(fs=65), "feature_samples")]:
        rc = call(**kw)
        assert rc != 0 and what in _lib.last_error(), (kw, rc, _lib.last_error())


def test_teacher_width_and_shapes_checked_on_the_host():
    import pytest
    from stego_b200 import corr
    assert [corr.teacher_width(c) for c in (1, 28, 64, 65, 101, 256, 257, 320, 385, 768)] == \
        [64, 64, 64, 128, 128, 256, 384, 320, 768, 768]
    with pytest.raises(RuntimeError, match="channels"):
        corr.teacher_width(800)
