"""Generate tests/golden/kk_step.pt from the REAL reference: its training step with dino_feat_type "KK".

    STEGO_REFERENCE_SRC=<reference checkout>/src python oracle/make_golden_kk_step.py

Outputs of the reference's own code on the CPU, on seeded inputs the tests rebuild without it:
  * `training_step`: src/train_segmentation.py:112-245 (text unmodified, stub-Lightning base, oracle/lightning_harness.py)
    with cfg.dino_feat_type = "KK" (src/modules.py:98-101: the last block's keys are the teacher features) at ViT-S/8,
    B = 2, 64x64 images: loss, logged terms, sampled gradients and the parameters after the reference's
    torch.optim.Adam update;
  * `descriptors`: get_feats of src/precompute_knns.py:15-21 — F.normalize(model(img).mean([2, 3]), dim=1) with model =
    the reference's DinoFeaturizer(...)[0] — for the step's images, the featurizer in eval mode (no Dropout2d draw).
Only outputs are stored; the inputs are rebuilt from their seeds (lightning_harness.make_batch, make_golden.step_params).
"""
from __future__ import annotations

import os
import sys
import tempfile

import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import lightning_harness as H  # noqa: E402
import make_golden as MG  # noqa: E402

OUT = os.path.join(HERE, "..", "tests", "golden", "kk_step.pt")
N_CLASSES = 27


def step_batch():
    return H.make_batch(MG.STEP_B, MG.STEP_RES, "cpu")


def reference_step(ts):
    from stego_b200.config import make_cfg
    with tempfile.TemporaryDirectory() as td:
        ck = os.path.join(td, "dino.pth")
        H.write_random_dino_checkpoint(ck, "vit_small")
        cfg = make_cfg(pretrained_weights=ck, dino_feat_type="KK")
        torch.manual_seed(0)
        m = ts.LitUnsupervisedSegmenter(N_CLASSES, cfg)
    params = dict(m.named_parameters())
    with torch.no_grad():
        for k, v in MG.step_params().items():
            params[k].copy_(v)
    m.train()
    batch = step_batch()
    torch.manual_seed(777)
    loss = m.training_step(batch, 0)
    step = dict(loss=float(loss.detach()), logged={k: float(v) for k, v in m.logged.items()},
                grads={k: MG._sample(params[k].grad) for k in MG.STEP_NAMES},
                params_after={k: params[k].detach().reshape(-1)[MG._sample(params[k].grad)["idx"].long()].clone()
                              for k in MG.STEP_NAMES})
    m.net.eval()
    with torch.no_grad():
        imgs = torch.cat([batch["img"], batch["img_pos"]], 0)
        descriptors = F.normalize(m.net(imgs)[0].mean([2, 3]), dim=1)  # precompute_knns.py:19
    return step, descriptors


def main():
    sys.path.insert(0, os.path.join(HERE, ".."))
    ts = H.load_reference_segmenter("reference")
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    step, desc = reference_step(ts)
    torch.save(dict(recipe="oracle/make_golden_kk_step.py", training_step=step, descriptors=desc), OUT)
    print(OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main()
