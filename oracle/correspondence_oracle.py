"""Restatement of the correspondence precision-recall diagnostic of src/plot_pr_curves.py (LitRecalibrator).

  get_net_fd (:108-121)   fd = tensor_correlation(norm(sample(f, coords1)), norm(sample(f, coords2))) of one image's
                          samples, ld = tensor_correlation of the sampled one-hot maps one_hot(label + 1, n + 1)
  plot_pr (:160-167)      preds = prep_fd(fd) (global min-max), targets = ld.to(int64), sklearn's
                          precision_recall_curve / average_precision_score

plus the exact positive rule stego_b200.correspondence uses (both samples pure with the same class), so that the two
can be compared.  Plain torch on the CPU; oracle/make_golden_correspondence.py pins it to the reference's own lines.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

import stego_oracle as O


def net_fd(feats: torch.Tensor, coords1: torch.Tensor, coords2: torch.Tensor) -> torch.Tensor:
    """[B, fs, fs, fs, fs] cosine of the samples of the same image at coords1 (rows) and coords2 (columns)."""
    s1 = O.l2_normalize(O.bilinear_sample(feats, coords1))
    s2 = O.l2_normalize(O.bilinear_sample(feats, coords2))
    return O.correlation(s1, s2)


def one_hot_map(label: torch.Tensor, n_classes: int) -> torch.Tensor:
    """[B, n + 1, H, W] fp32 one_hot(label + 1); labels outside 0 .. n - 1 are class 0 (the reference's -1)."""
    lab = label.long()
    cls = torch.where((lab >= 0) & (lab < n_classes), lab + 1, torch.zeros_like(lab))
    return F.one_hot(cls, n_classes + 1).to(torch.float).permute(0, 3, 1, 2)


def label_ld(label: torch.Tensor, n_classes: int, coords1: torch.Tensor, coords2: torch.Tensor) -> torch.Tensor:
    """The reference's ld: correlation of the (unnormalised) sampled one-hot maps, [B, fs, fs, fs, fs] fp32."""
    oh = one_hot_map(label, n_classes)
    return O.correlation(O.bilinear_sample(oh, coords1), O.bilinear_sample(oh, coords2))


def pure_ids(label: torch.Tensor, n_classes: int, coords: torch.Tensor) -> torch.Tensor:
    """[B, fs, fs] class of each sample when every tap with a non-zero weight has that class, else -1.  Sample (i, j)
    is `sample`'s output pixel (i, j), which reads coords[b, j, i]."""
    oh = one_hot_map(label, n_classes)
    # a tap with a non-zero weight contributes a positive amount to its class channel only: the sample is pure with
    # class c exactly when channel c is the only non-zero channel
    s = O.bilinear_sample(oh, coords)                      # [B, n + 1, fs, fs]
    nz = (s > 0).sum(1)
    return torch.where(nz == 1, s.argmax(1), torch.full_like(nz, -1))


def exact_targets(label, n_classes, coords1, coords2) -> torch.Tensor:
    """[B, fs, fs, fs, fs] bool: both samples pure with the same class (ld == 1 in exact arithmetic)."""
    a = pure_ids(label, n_classes, coords1)
    b = pure_ids(label, n_classes, coords2)
    B, fs = a.shape[0], a.shape[1]
    return ((a.reshape(B, fs, fs, 1, 1) == b.reshape(B, 1, 1, fs, fs)) & (a.reshape(B, fs, fs, 1, 1) >= 0))


def prep_fd(fd: torch.Tensor) -> torch.Tensor:
    """plot_pr_curves.py:34-37: global min-max rescale, flattened."""
    fd = fd.clone()
    fd -= fd.min()
    fd /= fd.max()
    return fd.reshape(-1)


def load_golden(path: str) -> dict:
    """tests/golden/correspondence_pr.pt with the compactly stored inputs widened back to what the reference ran on:
    feats / code (bf16 values) as fp32, labels (int8) as int64."""
    g = torch.load(path)
    g["feats"], g["code"] = g["feats"].float(), g["code"].float()
    g["label"] = g["label"].long()
    return g


def average_precision(scores, targets) -> float:
    from sklearn.metrics import average_precision_score
    return float(average_precision_score(np.asarray(targets).reshape(-1).astype(np.int64),
                                         np.asarray(scores, dtype=np.float64).reshape(-1)))
