"""Generate tests/golden/validation.pt from the REAL reference's validation path.

    STEGO_REFERENCE_SRC=<reference checkout>/src python oracle/make_golden_validation.py

The reference's own `validation_step` and `validation_epoch_end` (src/train_segmentation.py:254-371, class text
unmodified through oracle/lightning_harness.py) over its own modules.py on the CPU, with the reference's
`UnsupervisedMetrics` (src/utils.py:203-274) lifted as TEXT onto a minimal torchmetrics `Metric` stand-in (`add_state` /
`reset`), in place of the harness's no-op metrics.  The seeded ViT-S/8 of tests/golden/vit_small8_32px.pt, the seeded
head and probes of oracle/make_golden.py (step_params), 27 classes, extra_clusters 0 and 2.

Stored (data only; the model and the batch are regenerated from their seeds by `inputs` / `params`): both confusion
matrices, the preview dict's predictions, the low-res code the reference computed, `compute()` of both metrics with the
Hungarian assignment and histogram, and `map_clusters` of the preview and of every cluster id.
"""
from __future__ import annotations

import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import lightning_harness as H  # noqa: E402
import make_golden as MG  # noqa: E402

OUT = os.path.join(HERE, "..", "tests", "golden", "validation.pt")
B, RES, N_CLASSES, N_IMAGES = 6, 32, 27, 5
EXTRA = (0, 2)
RECIPE = ("ViT: perturb_vit_state(vit_random_state('vit_small', 8, seed=3)); head / linear probe: make_golden.step_params(); "
          "clusters: params(extra); batch: inputs(); reference validation_step x2 (batch, then batch[::-1]) + "
          "validation_epoch_end at global_step 3")


def inputs():
    """Two validation batches: img [B, 3, 32, 32] and int64 labels in [-1, 27] (-1 and 27 are ignored)."""
    g = torch.Generator().manual_seed(21)
    img = torch.randn(B, 3, RES, RES, generator=g)
    label = torch.randint(-1, N_CLASSES + 1, (B, RES, RES), generator=g)
    return [dict(img=img, label=label), dict(img=img.flip(0).contiguous(), label=label.flip(0).contiguous())]


def params(extra: int) -> dict:
    """step_params() with the cluster probe widened to 27 + extra centroids (extra rows from their own seed)."""
    p = MG.step_params()
    g = torch.Generator().manual_seed(30 + extra)
    p["cluster_probe.clusters"] = torch.cat([p["cluster_probe.clusters"], torch.randn(extra, 70, generator=g)], 0)
    return p


def _metric_class():
    """utils.py's UnsupervisedMetrics class text, executed over a Metric base that keeps its states as attributes."""
    import ast

    import numpy as np
    from scipy.optimize import linear_sum_assignment

    class Metric:
        def __init__(self, dist_sync_on_step=False):
            self._defaults = {}

        def add_state(self, name, default, dist_reduce_fx=None):
            self._defaults[name] = default.clone()
            setattr(self, name, default.clone())

        def reset(self):
            for k, v in self._defaults.items():
                setattr(self, k, v.clone())

    text = open(os.path.join(H.reference_src(), "utils.py")).read()
    src = next(ast.get_source_segment(text, n) for n in ast.parse(text).body
               if isinstance(n, ast.ClassDef) and n.name == "UnsupervisedMetrics")
    env = dict(Metric=Metric, torch=torch, np=np, linear_sum_assignment=linear_sum_assignment)
    exec(src, env)
    return env["UnsupervisedMetrics"]


def reference_validation(extra: int) -> dict:
    import tempfile
    sys.path.insert(0, os.path.join(HERE, ".."))
    from stego_b200.config import make_cfg
    ts = H.load_reference_segmenter("reference")
    ts.UnsupervisedMetrics = _metric_class()
    # `super().validation_epoch_end(outputs)` (:278) resolves to the stub LightningModule: a no-op as in Lightning
    H._LightningModule.validation_epoch_end = lambda self, outputs: None
    with tempfile.TemporaryDirectory() as td:
        ck = os.path.join(td, "dino.pth")
        H.write_random_dino_checkpoint(ck, "vit_small")
        cfg = make_cfg(pretrained_weights=ck, extra_clusters=extra, n_images=N_IMAGES, submitting_to_aml=False,
                       azureml_logging=False)
        torch.manual_seed(0)
        m = ts.LitUnsupervisedSegmenter(N_CLASSES, cfg)
    named = dict(m.named_parameters())
    with torch.no_grad():
        for k, v in params(extra).items():
            named[k].copy_(v)
    m.train()
    m.trainer.is_global_zero = False  # skips the matplotlib figures (:285-359)
    m.global_step = 3
    out = dict(steps=[])
    for i, batch in enumerate(inputs()):
        with torch.no_grad():
            m.net.eval()
            code = m.net(batch["img"])[1]
        preview = m.validation_step(batch, i)
        out["steps"].append(dict(code=code.clone(), linear_preds=preview["linear_preds"].to(torch.uint8),
                                 cluster_preds=preview["cluster_preds"].to(torch.uint8),
                                 keys=list(preview.keys()),
                                 shapes={k: tuple(v.shape) for k, v in preview.items()},
                                 dtypes={k: str(v.dtype) for k, v in preview.items()}))
    out["linear_stats"] = m.linear_metrics.stats.clone()
    out["cluster_stats"] = m.cluster_metrics.stats.clone()
    m.validation_epoch_end([])
    out["logged"] = {k: float(v) for k, v in m.logged.items()}
    cm = m.cluster_metrics
    out["assignments"] = [torch.as_tensor(a).clone() for a in cm.assignments]
    out["histogram"] = cm.histogram.clone()
    out["map_preview"] = cm.map_clusters(out["steps"][0]["cluster_preds"].long()).to(torch.int8)
    out["map_all"] = cm.map_clusters(torch.arange(N_CLASSES + extra))
    out["stats_after_epoch_end"] = (int(m.linear_metrics.stats.abs().sum()), int(cm.stats.abs().sum()))
    return out


def main():
    torch.set_num_threads(1)
    g = dict(recipe=RECIPE)
    for extra in EXTRA:
        g[f"extra{extra}"] = reference_validation(extra)
        print(extra, g[f"extra{extra}"]["logged"], g[f"extra{extra}"]["map_all"].tolist())
    torch.save(g, OUT)
    print(OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main()
