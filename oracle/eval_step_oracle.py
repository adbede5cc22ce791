"""Restatement of the reference's evaluation loop body (src/eval_segmentation.py:122-141, run_crf=False) in plain torch,
over the functional ViT and head of oracle/stego_oracle.py:

    code = (net(img) + net(img.flip(3)).flip(3)) / 2
    code = F.interpolate(code, label.shape[-2:], mode='bilinear', align_corners=False)
    linear_probs  = log_softmax(linear_probe(code)); cluster_probs = cluster_probe(code, 2, log_probs=True)
    preds = probs.argmax(1); test_*_metrics.update(preds, label)

`eval_loop` is what LitUnsupervisedSegmenter.eval_step computes.  tests/test_eval_step.py checks it against the
reference's own outputs (tests/golden/eval_step.pt, oracle/make_golden_eval_step.py) on the CPU, and
tests/test_eval_step_gpu.py runs it in fp32 on the GPU against eval_step.
"""
from __future__ import annotations

import os
import sys
from typing import Dict, Optional

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import kk_oracle  # noqa: E402
import stego_oracle as O  # noqa: E402


def net_code(vit_sd: Dict[str, torch.Tensor], head_sd: Dict[str, torch.Tensor], img: torch.Tensor,
             arch: str = "vit_small", patch: int = 8, feat_type: str = "feat") -> torch.Tensor:
    """The eval-mode DinoFeaturizer's code (src/modules.py:83-118, dropout off): the head on the last block's
    final-norm tokens ("feat") or keys ("KK"), [B, dim, h, w].  head_sd without cluster2 entries: the linear head."""
    feat = kk_oracle.image_feat(vit_sd, img, arch, feat_type, patch)
    code = F.conv2d(feat, head_sd["cluster1.0.weight"], head_sd["cluster1.0.bias"])
    if "cluster2.0.weight" in head_sd:
        hid = torch.relu(F.conv2d(feat, head_sd["cluster2.0.weight"], head_sd["cluster2.0.bias"]))
        code = code + F.conv2d(hid, head_sd["cluster2.2.weight"], head_sd["cluster2.2.bias"])
    return code


def confusion(preds: torch.Tensor, target: torch.Tensor, n_classes: int, n_rows: int) -> torch.Tensor:
    """UnsupervisedMetrics.update (src/utils.py:219-229): int64 [n_rows, n_classes] counts of (pred, actual) over the
    pixels with 0 <= actual < n_classes and 0 <= pred < n_classes."""
    actual, preds = target.reshape(-1).long(), preds.reshape(-1).long()
    mask = (actual >= 0) & (actual < n_classes) & (preds >= 0) & (preds < n_classes)
    return torch.bincount(n_rows * actual[mask] + preds[mask], minlength=n_classes * n_rows) \
        .reshape(n_classes, n_rows).t()


def eval_loop(code_fn, linear_w: torch.Tensor, linear_b: torch.Tensor, clusters: torch.Tensor, img: torch.Tensor,
              label: Optional[torch.Tensor], n_classes: int, alpha: float = 2.0) -> Dict[str, torch.Tensor]:
    """One batch of eval_segmentation.py:124-141 (run_crf=False).  code_fn(img) -> code [B, dim, h, w].  Returns the two
    codes, both log-probability maps, both argmax maps (int64) and, with a label, both confusion matrices of the batch
    (the reference's `final/linear` and `final/cluster` updates).  The output size is the label's, else the image's."""
    code1 = code_fn(img)
    code2 = code_fn(img.flip(dims=[3]))
    code = (code1 + code2.flip(dims=[3])) / 2
    size = label.shape[-2:] if label is not None else img.shape[-2:]
    code = F.interpolate(code, size, mode="bilinear", align_corners=False)
    linear_probs = torch.log_softmax(F.conv2d(code, linear_w.reshape(linear_w.shape[0], -1, 1, 1), linear_b), dim=1)
    cluster_probs = O.cluster_lookup(code, clusters, alpha, log_probs=True)
    out = dict(code1=code1, code2=code2, linear_probs=linear_probs, cluster_probs=cluster_probs,
               linear_preds=linear_probs.argmax(1), cluster_preds=cluster_probs.argmax(1))
    if label is not None:
        out["linear_stats"] = confusion(out["linear_preds"], label, n_classes, linear_w.shape[0])
        out["cluster_stats"] = confusion(out["cluster_preds"], label, n_classes, clusters.shape[0])
    return out
