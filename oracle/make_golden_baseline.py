"""Generate tests/golden/baseline.pt from the REAL reference's training step and evaluation loop body on the DINO
baseline.

    STEGO_REFERENCE_SRC=<reference checkout>/src python oracle/make_golden_baseline.py

The model is the reference's own LitUnsupervisedSegmenter (oracle/lightning_harness.py) with projection_type None,
dim 384 and correspondence_weight 0: DinoFeaturizer returns the ViT-S/8 features as the code (src/modules.py:108-113)
and the probes are Conv2d(384, n) / ClusterLookup(384, n).  The ViT is the seeded random one of the other fixtures;
the probes are seeded (params()).  The loop body of eval_segmentation.py (:121-141, run_crf False) is lifted as text,
as make_golden_eval_step.py does, and run on its two batches: without flip-TTA it is the same body with the mirrored
code replaced by the code itself, i.e. `code = code1`.
Training: two of the reference's own training_step calls (correspondence_weight 0, so only the probes learn) on
step_batches(), recording the loss, every logged term and the probe parameters after each Adam update.
Stored (data only; model and batches regenerate from their seeds): per training step the above; per eval batch and TTA
setting (without TTA the first
batch only) both log-probability maps, both argmax maps and both confusion matrices after the batch, and with TTA the
reference's code of the frames.
"""
from __future__ import annotations

import os
import sys
import tempfile
import types

import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import lightning_harness as H  # noqa: E402
import make_golden_eval_step as ME  # noqa: E402

OUT = os.path.join(HERE, "..", "tests", "golden", "baseline.pt")
N_CLASSES, EXTRA, DIM = ME.N_CLASSES, ME.EXTRA, 384
RECIPE = ("ViT: perturb_vit_state(vit_random_state('vit_small', 8, seed=3)); projection_type None, dim 384; probes: "
          "params(); eval batches: make_golden_eval_step.inputs(); eval_segmentation.py:121-141 per batch, "
          "run_crf=False, with and without flip-TTA; train: step_batches(), two training_step calls, "
          "correspondence_weight 0")


def params() -> dict:
    """Seeded probes on the 384 backbone channels for 5 classes + 2 extra clusters."""
    g = torch.Generator().manual_seed(43)
    return {"linear_probe.weight": torch.randn(N_CLASSES, DIM, 1, 1, generator=g) * 0.1,
            "linear_probe.bias": torch.randn(N_CLASSES, generator=g) * 0.1,
            "cluster_probe.clusters": torch.randn(N_CLASSES + EXTRA, DIM, generator=g)}


def loop_body(tta: bool) -> str:
    body = ME.loop_body()
    if tta:
        return body
    # the same body without the mirrored pass: the averaged code is the code itself
    line = "code = (code1 + code2.flip(dims=[3])) / 2"
    assert line in body, body
    return body.replace(line, "code = code1")


def reference_eval() -> dict:
    import make_golden_validation as MV
    from stego_b200.config import make_cfg
    ts = H.load_reference_segmenter("reference")
    ts.UnsupervisedMetrics = MV._metric_class()
    out = {}
    for tta in (False, True):
        with tempfile.TemporaryDirectory() as td:
            ck = os.path.join(td, "dino.pth")
            H.write_random_dino_checkpoint(ck, "vit_small")
            cfg = make_cfg(pretrained_weights=ck, extra_clusters=EXTRA, projection_type=None, dim=DIM,
                           correspondence_weight=0.0, submitting_to_aml=False, azureml_logging=False)
            torch.manual_seed(0)
            m = ts.LitUnsupervisedSegmenter(N_CLASSES, cfg)
        named = dict(m.named_parameters())
        with torch.no_grad():
            for k, v in params().items():
                named[k].copy_(v)
        m.eval()
        codes = []
        net = m.net

        def par_model(img):  # the reference net, keeping the codes it returns
            o = net(img)
            codes.append(o[1].clone())
            return o

        body = compile(loop_body(tta), "eval_segmentation.py", "exec")
        steps = []
        for i, batch in enumerate(ME.inputs()[:2 if tta else 1]):  # without TTA the first batch (a small file)
            env = dict(torch=torch, F=F, batch=batch, par_model=par_model, model=m,
                       cfg=types.SimpleNamespace(run_crf=False), pool=None, batched_crf=None, i=i)
            codes.clear()
            exec(body, env)
            steps.append(dict(code1=codes[0] if tta else None, linear_probs=env["linear_probs"].clone(),
                              cluster_probs=env["cluster_probs"].clone(),
                              linear_preds=env["linear_preds"].to(torch.uint8),
                              cluster_preds=env["cluster_preds"].to(torch.uint8),
                              linear_stats=m.test_linear_metrics.stats.clone(),
                              cluster_stats=m.test_cluster_metrics.stats.clone()))
        out["tta" if tta else "no_tta"] = steps
        out["state_dict_keys"] = sorted(m.state_dict().keys())
    return out


def step_batches():
    """The two training batches: ViT-S/8 frames of 64 x 64, B = 2, labels in [-1, N_CLASSES)."""
    return [H.make_batch(2, 64, "cpu", seed=s, n_classes=N_CLASSES) for s in (1, 2)]


def reference_train() -> dict:
    """Two of the reference's training steps (src/train_segmentation.py:112-245, text unmodified) on the baseline:
    every logged loss and the probes after each step's Adam update (the net has no parameter with a gradient)."""
    from stego_b200.config import make_cfg
    ts = H.load_reference_segmenter("reference")
    with tempfile.TemporaryDirectory() as td:
        ck = os.path.join(td, "dino.pth")
        H.write_random_dino_checkpoint(ck, "vit_small")
        # use_true_labels: as written, training_step reads feats_pos (:140) even when correspondence_weight is 0 and
        # net(img_pos) did not run; the one-hot label signal of use_true_labels takes that branch instead and is unused
        # without the correspondence loss
        cfg = make_cfg(pretrained_weights=ck, extra_clusters=EXTRA, projection_type=None, dim=DIM,
                       correspondence_weight=0.0, use_true_labels=True)
        torch.manual_seed(0)
        m = ts.LitUnsupervisedSegmenter(N_CLASSES, cfg)
    named = dict(m.named_parameters())
    with torch.no_grad():
        for k, v in params().items():
            named[k].copy_(v)
    m.train()
    steps = []
    for i, batch in enumerate(step_batches()):
        torch.manual_seed(777 + i)
        loss = m.training_step(batch, i)
        steps.append(dict(loss=float(loss.detach()), logged={k: float(v) for k, v in m.logged.items()},
                          params={k: named[k].detach().clone() for k in params()}))
    return dict(train=steps)


def main():
    torch.set_num_threads(1)
    sys.path.insert(0, os.path.join(HERE, ".."))
    g = dict(recipe=RECIPE, n_classes=N_CLASSES, extra_clusters=EXTRA, dim=DIM, **reference_eval(), **reference_train())
    for s in g["train"]:
        print(s["loss"], s["logged"])
    torch.save(g, OUT)
    for k in ("no_tta", "tta"):
        for s in g[k]:
            print(k, tuple(s["linear_probs"].shape), s["linear_stats"].sum().item(), s["cluster_stats"].sum().item())
    print(OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main()
