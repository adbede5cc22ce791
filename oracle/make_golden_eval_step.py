"""Generate tests/golden/eval_step.pt from the REAL reference's evaluation loop body.

    STEGO_REFERENCE_SRC=<reference checkout>/src python oracle/make_golden_eval_step.py

src/eval_segmentation.py cannot be imported (hydra, seaborn, a DataLoader over a data set), so the body of its
`with torch.no_grad():` block (:121-141, up to the PiCIE branch) is lifted as TEXT and executed once per batch, with
cfg.run_crf = False (the dense CRF needs pydensecrf).  Only its `.cuda()` calls are dropped: it runs on the CPU.  It runs
over the reference's own LitUnsupervisedSegmenter (src/train_segmentation.py, class text unmodified through
oracle/lightning_harness.py) and modules.py: `par_model` is its eval-mode `net`, and its `test_linear_metrics` /
`test_cluster_metrics` are the reference's UnsupervisedMetrics (src/utils.py, lifted as in make_golden_validation.py).

The model: the seeded ViT-S/8 of tests/golden/vit_small8_32px.pt, the seeded head of make_golden.step_params (dim 70),
5 classes + 2 extra clusters with seeded probes (params()).  Two batches of 2 frames (inputs()): 32x48 frames with
32x48 labels, and 32x32 frames with 48x48 labels (the output follows the label's size).
Stored (data only; the model and the batches are regenerated from their seeds): per batch the reference's two codes,
both log-probability maps and both argmax maps, and both confusion matrices after each batch.
"""
from __future__ import annotations

import ast
import os
import sys
import tempfile
import textwrap
import types

import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import lightning_harness as H  # noqa: E402
import make_golden as MG  # noqa: E402

OUT = os.path.join(HERE, "..", "tests", "golden", "eval_step.pt")
N_CLASSES, EXTRA, DIM = 5, 2, 70
RECIPE = ("ViT: perturb_vit_state(vit_random_state('vit_small', 8, seed=3)); head: make_golden.step_params() net.*; "
          "probes: params(); batches: inputs(); eval_segmentation.py:121-141 per batch, run_crf=False")


def inputs():
    """Two batches: img [2, 3, 32, 48] with int64 labels [2, 32, 48], img [2, 3, 32, 32] with labels [2, 48, 48]; labels
    in [-1, N_CLASSES] (-1 and N_CLASSES are ignored by the metrics)."""
    g = torch.Generator().manual_seed(41)
    out = []
    for (h, w), (lh, lw) in (((32, 48), (32, 48)), ((32, 32), (48, 48))):
        img = torch.randn(2, 3, h, w, generator=g)
        label = torch.randint(-1, N_CLASSES + 1, (2, lh, lw), generator=g)
        out.append(dict(img=img, label=label))
    return out


def params() -> dict:
    """The head of make_golden.step_params() and seeded probes for 5 classes + 2 extra clusters."""
    p = {k: v for k, v in MG.step_params().items() if k.startswith("net.")}
    g = torch.Generator().manual_seed(42)
    p["linear_probe.weight"] = torch.randn(N_CLASSES, DIM, 1, 1, generator=g) * 0.1
    p["linear_probe.bias"] = torch.randn(N_CLASSES, generator=g) * 0.1
    p["cluster_probe.clusters"] = torch.randn(N_CLASSES + EXTRA, DIM, generator=g)
    return p


def loop_body() -> str:
    """The statements of eval_segmentation.py's `with torch.no_grad():` block before `if run_picie:`, as text."""
    text = open(os.path.join(H.reference_src(), "eval_segmentation.py")).read()
    for node in ast.walk(ast.parse(text)):
        if isinstance(node, ast.With) and any(isinstance(s, ast.Assign) and "code1" in ast.unparse(s.targets[0])
                                              for s in node.body):
            stmts = []
            for s in node.body:
                if isinstance(s, ast.If) and ast.unparse(s.test) == "run_picie":
                    break
                stmts.append(textwrap.dedent(ast.get_source_segment(text, s, padded=True)))
            return "\n".join(stmts).replace(".cuda()", "")
    raise KeyError("eval_segmentation.py: no loop body with code1")


def reference_eval() -> dict:
    import make_golden_validation as MV
    from stego_b200.config import make_cfg
    ts = H.load_reference_segmenter("reference")
    ts.UnsupervisedMetrics = MV._metric_class()
    with tempfile.TemporaryDirectory() as td:
        ck = os.path.join(td, "dino.pth")
        H.write_random_dino_checkpoint(ck, "vit_small")
        cfg = make_cfg(pretrained_weights=ck, extra_clusters=EXTRA, submitting_to_aml=False, azureml_logging=False)
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
        out = net(img)
        codes.append(out[1].clone())
        return out

    body = compile(loop_body(), "eval_segmentation.py", "exec")
    out = dict(steps=[])
    for i, batch in enumerate(inputs()):
        env = dict(torch=torch, F=F, batch=batch, par_model=par_model, model=m, cfg=types.SimpleNamespace(run_crf=False),
                   pool=None, batched_crf=None, i=i)
        codes.clear()
        exec(body, env)
        out["steps"].append(dict(code1=codes[0], code2=codes[1], linear_probs=env["linear_probs"].clone(),
                                 cluster_probs=env["cluster_probs"].clone(),
                                 linear_preds=env["linear_preds"].to(torch.uint8),
                                 cluster_preds=env["cluster_preds"].to(torch.uint8),
                                 linear_stats=m.test_linear_metrics.stats.clone(),
                                 cluster_stats=m.test_cluster_metrics.stats.clone()))
    return out


def main():
    torch.set_num_threads(1)
    sys.path.insert(0, os.path.join(HERE, ".."))
    g = dict(recipe=RECIPE, n_classes=N_CLASSES, extra_clusters=EXTRA, **reference_eval())
    torch.save(g, OUT)
    for s in g["steps"]:
        print(tuple(s["linear_probs"].shape), s["linear_stats"].sum().item(), s["cluster_stats"].sum().item())
    print(OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main()
