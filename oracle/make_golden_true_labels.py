"""Generate tests/golden/true_labels_step.pt from the REAL reference: its training step with use_true_labels=True.

    STEGO_REFERENCE_SRC=<reference checkout>/src python oracle/make_golden_true_labels.py

Two outputs of the reference's own code on the CPU, on seeded inputs the tests rebuild without it:
  * `training_step`: src/train_segmentation.py:112-245 (text unmodified, stub-Lightning base, oracle/lightning_harness.py)
    with cfg.use_true_labels (:135-140) at ViT-S/8, B = 2, 64x64 images (8x8 code), labels with -1 entries: loss,
    logged terms, sampled gradients and the parameters after the reference's torch.optim.Adam update;
  * `module`: src/modules.py ContrastiveCorrelationLoss on the one-hot signal one_hot_feats(label + 1, 28) at 4x the
    code's resolution, with the coordinate / permutation draws it made.
Only outputs and draws are stored; the inputs are rebuilt from their seeds (step_batch, module_inputs).
"""
from __future__ import annotations

import os
import sys
import tempfile
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import lightning_harness as H  # noqa: E402
import make_golden as MG  # noqa: E402
import reference_shim  # noqa: E402
import stego_oracle as O  # noqa: E402
import true_labels_oracle as TL  # noqa: E402

OUT = os.path.join(HERE, "..", "tests", "golden", "true_labels_step.pt")
N_CLASSES = 27
MOD_B, MOD_CODE, MOD_LABEL = 3, 10, 40  # module case: code 10x10, labels 40x40


def step_batch():
    """The step's batch: lightning_harness.make_batch with a label_pos of its own (both contain -1)."""
    batch = H.make_batch(MG.STEP_B, MG.STEP_RES, "cpu")
    g = torch.Generator().manual_seed(5)
    batch["label_pos"] = torch.randint(-1, N_CLASSES, (MG.STEP_B, MG.STEP_RES, MG.STEP_RES), generator=g)
    return batch


def module_inputs():
    """Region labels (piecewise constant, 5x5-pixel blocks, some unlabelled) at 4x the code's resolution."""
    g = torch.Generator().manual_seed(21)
    blocks = torch.randint(-1, N_CLASSES, (2, MOD_B, MOD_LABEL // 5, MOD_LABEL // 5), generator=g)
    lab = blocks.repeat_interleave(5, -1).repeat_interleave(5, -2)
    code = torch.randn(MOD_B, 70, MOD_CODE, MOD_CODE, generator=g)
    code_pos = code + 0.5 * torch.randn(MOD_B, 70, MOD_CODE, MOD_CODE, generator=g)
    return lab[0], lab[1], code, code_pos


def reference_step(ts):
    from stego_b200.config import make_cfg
    with tempfile.TemporaryDirectory() as td:
        ck = os.path.join(td, "dino.pth")
        H.write_random_dino_checkpoint(ck, "vit_small")
        cfg = make_cfg(pretrained_weights=ck, use_true_labels=True)
        torch.manual_seed(0)
        m = ts.LitUnsupervisedSegmenter(N_CLASSES, cfg)
    params = dict(m.named_parameters())
    with torch.no_grad():
        for k, v in MG.step_params().items():
            params[k].copy_(v)
    m.train()
    torch.manual_seed(777)
    loss = m.training_step(step_batch(), 0)
    return dict(loss=float(loss.detach()), logged={k: float(v) for k, v in m.logged.items()},
                grads={k: MG._sample(params[k].grad) for k in MG.STEP_NAMES},
                params_after={k: params[k].detach().reshape(-1)[MG._sample(params[k].grad)["idx"].long()].clone()
                              for k in MG.STEP_NAMES})


def reference_module(ref):
    label, label_pos, code, code_pos = module_inputs()
    code.requires_grad_(True)
    code_pos.requires_grad_(True)
    ns = types.SimpleNamespace(**O.LossCfg().__dict__)
    sig, sig_pos = TL.label_signals(label, label_pos, N_CLASSES)
    torch.manual_seed(31)
    o = ref.ContrastiveCorrelationLoss(ns)(sig, sig_pos, None, None, code, code_pos)
    loss = .67 * o[0] + .25 * o[2] + .63 * o[4].mean()
    loss.backward()
    torch.manual_seed(31)
    c1, c2, perms = O.draw_loss_randomness(MOD_B, O.LossCfg())
    return dict(coords1=c1, coords2=c2, perms=torch.stack(perms),
                pos_intra_loss=o[0].detach(), pos_inter_loss=o[2].detach(), neg_inter_loss_mean=o[4].mean().detach(),
                cd_means=torch.stack([o[1].mean(), o[3].mean(), o[5].mean()]).detach(), total=loss.detach(),
                inter_cd_sub=o[3].detach().reshape(-1)[::53].clone(), neg_loss_sub=o[4].detach().reshape(-1)[::53].clone(),
                code_grad=code.grad.clone(), code_pos_grad=code_pos.grad.clone())


def main():
    sys.path.insert(0, os.path.join(HERE, ".."))
    ref, _ = reference_shim.import_reference()
    ts = H.load_reference_segmenter("reference")
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    torch.save(dict(recipe="oracle/make_golden_true_labels.py", training_step=reference_step(ts),
                    module=reference_module(ref)), OUT)
    print(OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main()
