"""Generate tests/golden/scene.pt from the REAL reference's scene evaluation (src/plot_potsdam.py).

    STEGO_REFERENCE_SRC=<reference checkout>/src python oracle/make_golden_scene.py

plot_potsdam.py cannot be imported (hydra, a data set, a checkpoint), so two pieces of `my_app` are lifted as TEXT:
  * the loop body (:44-59): the statements of its `with torch.no_grad():` block after `if i > 100: break`, executed
    once per loader batch, with its `.cuda()` calls dropped (it runs on the CPU);
  * the scene (:61-83): `test_cluster_metrics.compute()` and the statements from `img_num = 6` up to `reshaped_preds`,
    without the two that need a display (`print`, `unnorm(...)`).  The scene size is substituted into the stitching
    lines: `15, 15` -> `R, C` (tiles per column and per row), `320` -> `T` (the tile side), and `img_num` is 0.
It runs over the reference's own LitUnsupervisedSegmenter (oracle/lightning_harness.py) and UnsupervisedMetrics (lifted
as in make_golden_validation.py); `par_model` is its eval-mode `net`.  The stitching reshapes the cluster
probabilities with the image's channel count 3, so the model has 3 classes and no extra clusters, as Potsdam does.

The model: the seeded ViT-S/8 of tests/golden/vit_small8_32px.pt, the seeded head of make_golden.step_params (dim 70)
and seeded probes (params()).  The scene: 3 x 4 tiles of 32 x 32 in loader batches of 5 (inputs()).
Stored (data only; the model and the tiles are regenerated from their seeds): the stitched image, cluster
log-probabilities and label, the cluster metrics' confusion matrix, its assignment and the mapped predictions.
"""
from __future__ import annotations

import ast
import os
import sys
import tempfile
import textwrap
from collections import defaultdict

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import lightning_harness as H  # noqa: E402
import make_golden as MG  # noqa: E402

OUT = os.path.join(HERE, "..", "tests", "golden", "scene.pt")
N_CLASSES, DIM = 3, 70
R, C, T, BATCH = 3, 4, 32, 5
RECIPE = ("ViT: perturb_vit_state(vit_random_state('vit_small', 8, seed=3)); head: make_golden.step_params() net.*; "
          "probes: params(); tiles: inputs(); plot_potsdam.py:44-59 per batch of 5, :61-83 for the 3 x 4 scene")


def inputs():
    """R*C tiles [12, 3, 32, 32] and int64 labels [12, 32, 32] in [-1, N_CLASSES] (-1 and N_CLASSES are ignored)."""
    g = torch.Generator().manual_seed(51)
    img = torch.randn(R * C, 3, T, T, generator=g)
    label = torch.randint(-1, N_CLASSES + 1, (R * C, T, T), generator=g)
    return img, label


def params() -> dict:
    """The head of make_golden.step_params() and seeded probes for 3 classes."""
    p = {k: v for k, v in MG.step_params().items() if k.startswith("net.")}
    g = torch.Generator().manual_seed(52)
    p["linear_probe.weight"] = torch.randn(N_CLASSES, DIM, 1, 1, generator=g) * 0.1
    p["linear_probe.bias"] = torch.randn(N_CLASSES, generator=g) * 0.1
    p["cluster_probe.clusters"] = torch.randn(N_CLASSES, DIM, generator=g)
    return p


def _my_app():
    text = open(os.path.join(H.reference_src(), "plot_potsdam.py")).read()
    fn = next(n for n in ast.walk(ast.parse(text)) if isinstance(n, ast.FunctionDef) and n.name == "my_app")
    return text, fn


def loop_body() -> str:
    """The statements of the loader loop's `with torch.no_grad():` block after `if i > 100: break`, as text."""
    text, fn = _my_app()
    loop = next(n for n in fn.body if isinstance(n, ast.For))
    block = next(n for n in loop.body if isinstance(n, ast.With))
    stmts = [textwrap.dedent(ast.get_source_segment(text, s, padded=True)) for s in block.body if not isinstance(s, ast.If)]
    return "\n".join(stmts).replace(".cuda()", "")


def scene_body() -> str:
    """`test_cluster_metrics.compute()` and the statements from `img_num = 6` to `reshaped_preds = ...`, without the
    print and the display image, with the scene size substituted."""
    text, fn = _my_app()
    i0 = next(i for i, s in enumerate(fn.body) if isinstance(s, ast.For))
    stmts = []
    for s in fn.body[i0 + 1:]:
        src = ast.get_source_segment(text, s)
        if src.startswith("print(") or src.startswith("reshaped_img"):
            continue
        stmts.append(src)
        if src.startswith("reshaped_preds"):
            break
    body = "\n".join(stmts)
    for a, b in (("img_num = 6", "img_num = 0"), ("15, 15", "R, C"), ("320 * 15, 320 * 15", "T * R, T * C"),
                 ("15 * 15", "R * C"), ("320", "T")):
        assert a in body, a
        body = body.replace(a, b)
    return body


def reference_scene() -> dict:
    import make_golden_validation as MV
    from stego_b200.config import make_cfg
    ts = H.load_reference_segmenter("reference")
    ts.UnsupervisedMetrics = MV._metric_class()
    with tempfile.TemporaryDirectory() as td:
        ck = os.path.join(td, "dino.pth")
        H.write_random_dino_checkpoint(ck, "vit_small")
        cfg = make_cfg(pretrained_weights=ck, extra_clusters=0, submitting_to_aml=False, azureml_logging=False)
        torch.manual_seed(0)
        m = ts.LitUnsupervisedSegmenter(N_CLASSES, cfg)
    named = dict(m.named_parameters())
    with torch.no_grad():
        for k, v in params().items():
            named[k].copy_(v)
    m.eval()
    img, label = inputs()
    outputs = defaultdict(list)
    body = compile(loop_body(), "plot_potsdam.py", "exec")
    for i, t0 in enumerate(range(0, R * C, BATCH)):
        batch = dict(img=img[t0:t0 + BATCH], label=label[t0:t0 + BATCH])
        with torch.no_grad():  # the block's own `with`
            exec(body, dict(torch=torch, F=F, batch=batch, par_model=m.net, model=m, outputs=outputs, i=i))
    env = dict(torch=torch, np=np, model=m, outputs=outputs, R=R, C=C, T=T)
    exec(compile(scene_body(), "plot_potsdam.py", "exec"), env)
    metric = m.test_cluster_metrics
    return dict(image=env["full_image"].clone(), cluster_probs=env["full_cluster_prob"].clone(),
                label=env["reshaped_label"].clone(), cluster_stats=metric.stats.clone(),
                assignments=tuple(torch.as_tensor(np.asarray(a)) for a in metric.assignments),
                mapped_preds=torch.as_tensor(np.asarray(env["reshaped_preds"])).reshape(R * T, C * T).clone())


def main():
    torch.set_num_threads(1)
    sys.path.insert(0, os.path.join(HERE, ".."))
    g = dict(recipe=RECIPE, n_classes=N_CLASSES, grid=(R, C), tile=T, batch=BATCH, **reference_scene())
    torch.save(g, OUT)
    print({k: tuple(v.shape) for k, v in g.items() if isinstance(v, torch.Tensor)}, int(g["cluster_stats"].sum()))
    print(OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main()
