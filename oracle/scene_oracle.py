"""Restatement of the reference's scene evaluation (src/plot_potsdam.py:44-57 per loader batch, :65-83 for one scene) in
plain torch, over the loop body of oracle/eval_step_oracle.py:

    per batch of tiles:  code = (net(img) + net(img.flip(3)).flip(3)) / 2;  code = F.interpolate(code, label size)
                         cluster_prob = cluster_probe(code, 2, log_probs=True);  test_cluster_metrics.update(argmax)
    one scene:           tile i -> tile row i // C, tile column i % C of an R t x C t mosaic (image, probabilities, label)
                         probs = dense_crf(mosaic image, mosaic probs)        (commented out in the reference, :76-77)
                         preds = test_cluster_metrics.map_clusters(probs.argmax(0))

`scene_loop` is what LitUnsupervisedSegmenter.eval_scene computes (the linear probe evaluated beside the cluster probe, as
eval_segmentation does).  tests/test_eval_scene.py checks it against the reference's own lines (tests/golden/scene.pt,
oracle/make_golden_scene.py) on the CPU; tests/test_eval_scene_gpu.py runs its stitching against eval_scene.
"""
from __future__ import annotations

import os
import sys
from typing import Dict, Optional, Sequence

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import crf_oracle  # noqa: E402
import eval_step_oracle as EO  # noqa: E402


def stitch(t: torch.Tensor, R: int, C: int) -> torch.Tensor:
    """[R*C, ..., h, w] tiles in row-major tile order -> [..., R*h, C*w]: tile i at tile row i // C, tile column i % C."""
    h, w = t.shape[-2:]
    mid = t.shape[1:-2]
    k = len(mid)
    x = t.reshape(R, C, *mid, h, w)
    # [R, C, mid..., h, w] -> [mid..., R, h, C, w]
    x = x.permute(*range(2, 2 + k), 0, 2 + k, 1, 3 + k)
    return x.reshape(*mid, R * h, C * w)


def hungarian(stats: torch.Tensor, n_classes: int, extra_clusters: int) -> torch.Tensor:
    """UnsupervisedMetrics.compute's assignment + map_clusters (src/utils.py:231-255) as a cluster -> class table
    (int64 [n_classes + extra_clusters], -1 for the clusters the assignment leaves out)."""
    from scipy.optimize import linear_sum_assignment
    rows, cols = linear_sum_assignment(stats.cpu().numpy(), maximize=True)
    cluster_to_class = cols
    if extra_clusters > 0:
        for m in sorted(set(range(n_classes + extra_clusters)) - set(rows)):
            if m == cluster_to_class.shape[0]:
                cluster_to_class = np.append(cluster_to_class, -1)
            else:
                cluster_to_class = np.insert(cluster_to_class, m + 1, -1)
    return torch.as_tensor(cluster_to_class, dtype=torch.long)


def scene_loop(code_fn, linear_w: torch.Tensor, linear_b: torch.Tensor, clusters: torch.Tensor, tiles: torch.Tensor,
               label: Optional[torch.Tensor], grid: Sequence[int], n_classes: int, batch: int = 64,
               run_crf: bool = False, alpha: float = 2.0) -> Dict[str, torch.Tensor]:
    """plot_potsdam.py:44-83 for one scene of R*C tiles [R*C, 3, t, t'] (with the linear probe beside the cluster probe).
    Returns the stitched image [3, R t, C t'], log-probabilities [n, R t, C t'] (or, with run_crf, the CRF marginals of
    crf_oracle.dense_crf on the stitched image and log-probabilities), argmax maps, the stitched label and, with a label,
    both confusion matrices (per tile without the CRF, of the CRF predictions against the stitched label with it)."""
    R, C = int(grid[0]), int(grid[1])
    parts = {k: [] for k in ("linear_probs", "cluster_probs", "linear_preds", "cluster_preds")}
    lin_stats = torch.zeros(linear_w.shape[0], n_classes, dtype=torch.long)
    clu_stats = torch.zeros(clusters.shape[0], n_classes, dtype=torch.long)
    for t0 in range(0, tiles.shape[0], batch):
        img = tiles[t0:t0 + batch]
        lab = label[t0:t0 + batch] if label is not None else None
        o = EO.eval_loop(code_fn, linear_w, linear_b, clusters, img, lab, n_classes, alpha)
        for k in parts:
            parts[k].append(o[k])
        if lab is not None and not run_crf:
            lin_stats += o["linear_stats"].cpu()
            clu_stats += o["cluster_stats"].cpu()
    out = {k: stitch(torch.cat(v, 0), R, C) for k, v in parts.items()}
    out["image"] = stitch(tiles, R, C)
    out["label"] = stitch(label, R, C) if label is not None else None
    if run_crf:
        for probe in ("linear", "cluster"):
            q = torch.as_tensor(crf_oracle.dense_crf(out["image"].double().cpu(), out[f"{probe}_probs"].double().cpu()))
            out[f"{probe}_probs"] = q
            out[f"{probe}_preds"] = q.argmax(0)
        if label is not None:
            lin_stats = EO.confusion(out["linear_preds"], out["label"].cpu(), n_classes, linear_w.shape[0])
            clu_stats = EO.confusion(out["cluster_preds"], out["label"].cpu(), n_classes, clusters.shape[0])
    if label is not None:
        out["linear_stats"], out["cluster_stats"] = lin_stats, clu_stats
    return out
