"""Fused evaluation probes: the inner loop of the reference's `eval_segmentation.py` (:124-141) without
materialising the upsampled code.

    code = F.interpolate(code, label.shape[-2:], mode='bilinear', align_corners=False)
    linear_probs  = torch.log_softmax(model.linear_probe(code), dim=1)
    cluster_probs = model.cluster_probe(code, 2, log_probs=True)

becomes `fused_probe_log_probs(code_lowres, model.linear_probe, model.cluster_probe, label.shape[-2:], 2)`.
At 1024x2048 the reference moves 587 MB (fp32 upsampled code) per image per probe before it even starts;
the fused kernel reads the 9 MB low-res code and writes only the outputs (stego_eval_probes, eval_probes.cu).
"""
from __future__ import annotations

from typing import Optional, Sequence, Tuple

import torch

from . import _lib, ops


def fused_probe_log_probs(code: torch.Tensor, linear_probe: torch.nn.Module, cluster_probe: torch.nn.Module,
                          size: Sequence[int], alpha: float = 2.0, want_log_probs: bool = True,
                          want_argmax: bool = False, code_flipped: Optional[torch.Tensor] = None,
                          label: Optional[torch.Tensor] = None, linear_confusion: Optional[torch.Tensor] = None,
                          cluster_confusion: Optional[torch.Tensor] = None):
    """code: low-res [B, C, h, w] (any strides, CUDA).  Returns (linear_log_probs, cluster_log_probs) [B,n,H,W]
    fp32, and with want_argmax also (linear_argmax, cluster_argmax) uint8 [B,H,W].

    code_flipped: the code of `img.flip(dims=[3])` — the kernel then evaluates the flip-TTA average
    `(code + code_flipped.flip(dims=[3])) / 2` (eval_segmentation.py:124-126) without materialising it.
    label [B,H,W] (+ int64 `linear_confusion [n_lin, n_classes]` / `cluster_confusion [n_clu, n_classes]`, accumulated
    in place): UnsupervisedMetrics.update for both probes (utils.py:219-229) fused into the same pass."""
    _lib.require_cuda(code)
    if not code.is_cuda:
        raise RuntimeError("stego_b200.eval: CUDA tensors required (no CPU fallback)")
    B, C, h, w = code.shape
    H, W = int(size[0]), int(size[1])
    x = ops.tokens_major(code)
    ld = x.stride(3)
    xf = None
    if code_flipped is not None:
        assert code_flipped.shape == code.shape
        xf = ops.tokens_major(code_flipped)
        if xf.stride(3) != ld:  # one ld for both codes
            xf = xf.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
            x = x.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
            ld = x.stride(3)
    wl = linear_probe.weight.detach().float().reshape(linear_probe.weight.shape[0], C).contiguous()
    bl = linear_probe.bias.detach().float().contiguous()
    cl = cluster_probe.clusters.detach().float().contiguous()
    n_lin, n_clu = wl.shape[0], cl.shape[0]
    dev = code.device
    scratch = torch.empty(B * h * w, 80, dtype=torch.float32, device=dev)  # eval_probes.cu EV_LD
    lin = torch.empty(B, n_lin, H, W, dtype=torch.float32, device=dev) if want_log_probs else None
    clu = torch.empty(B, n_clu, H, W, dtype=torch.float32, device=dev) if want_log_probs else None
    la = torch.empty(B, H, W, dtype=torch.uint8, device=dev) if want_argmax else None
    ca = torch.empty(B, H, W, dtype=torch.uint8, device=dev) if want_argmax else None
    lab, lab_bytes, n_cls = None, 0, 0
    if label is not None:
        _lib.require_cuda(label, linear_confusion, cluster_confusion)
        lab, lab_bytes = ops.probe_label(label, B, H, W)
        n_cls = n_lin
        for t, n in ((linear_confusion, n_lin), (cluster_confusion, n_clu)):
            if t is not None:
                assert t.dtype == torch.int64 and t.is_contiguous() and tuple(t.shape) == (n, n_cls)
        if linear_confusion is None and cluster_confusion is None:
            raise ValueError("label given without a confusion matrix to accumulate into")
    rc = _lib.load().stego_eval_probes(_lib.ptr(x), _lib.ptr(xf), ld, C, B, h, w, H, W, _lib.ptr(wl), _lib.ptr(bl), n_lin,
                                       _lib.ptr(cl), n_clu, float(alpha), _lib.ptr(scratch), _lib.ptr(lin), _lib.ptr(clu),
                                       _lib.ptr(la), _lib.ptr(ca), _lib.ptr(lab), lab_bytes, n_cls,
                                       _lib.ptr(linear_confusion), _lib.ptr(cluster_confusion), _lib.stream())
    _lib.check(rc, "stego_eval_probes")
    if want_argmax:
        return lin, clu, la, ca
    return lin, clu


class UnsupervisedMetrics:
    """src/utils.py:203-274 without the torchmetrics base class: the [pred, actual] confusion counts, Hungarian matching of
    clusters to classes on the host (scipy), mIoU and accuracy.  `stats` is the int64 tensor the fused probe kernel
    accumulates into (pass it as `linear_confusion` / `cluster_confusion` to `fused_probe_log_probs`); `update` is the
    reference's torch.bincount path for predictions that come from elsewhere (e.g. after the CRF)."""

    def __init__(self, prefix: str, n_classes: int, extra_clusters: int, compute_hungarian: bool, device=None):
        self.prefix, self.n_classes, self.extra_clusters = prefix, n_classes, extra_clusters
        self.compute_hungarian = compute_hungarian
        self.stats = torch.zeros(n_classes + extra_clusters, n_classes, dtype=torch.int64, device=device)

    def update(self, preds: torch.Tensor, target: torch.Tensor):
        with torch.no_grad():
            actual, preds = target.reshape(-1), preds.reshape(-1)
            mask = (actual >= 0) & (actual < self.n_classes) & (preds >= 0) & (preds < self.n_classes)
            n = self.n_classes + self.extra_clusters
            self.stats += torch.bincount(n * actual[mask].long() + preds[mask].long(), minlength=self.n_classes * n) \
                .reshape(self.n_classes, n).t().to(self.stats.device)

    def reset(self):
        self.stats.zero_()

    def map_clusters(self, clusters: torch.Tensor) -> torch.Tensor:
        """utils.py:231-243: cluster ids -> the class ids the Hungarian matching of the last `compute()` assigned them.
        With extra clusters, the unmatched ones map to -1 by the reference's own insertion rule (each missing index m
        inserts -1 at position m + 1 of the assignment vector, or appends it at the end)."""
        import numpy as np
        cluster_to_class = self.assignments[1]
        if self.extra_clusters > 0:
            missing = sorted(set(range(self.n_classes + self.extra_clusters)) - set(self.assignments[0]))
            for m in missing:
                if m == cluster_to_class.shape[0]:
                    cluster_to_class = np.append(cluster_to_class, -1)
                else:
                    cluster_to_class = np.insert(cluster_to_class, m + 1, -1)
        return torch.as_tensor(cluster_to_class, device=clusters.device)[clusters]

    def compute(self):
        import numpy as np
        from scipy.optimize import linear_sum_assignment
        stats = self.stats.detach().cpu()
        if self.compute_hungarian:
            self.assignments = linear_sum_assignment(stats, maximize=True)
            if self.extra_clusters == 0:
                self.histogram = stats[np.argsort(self.assignments[1]), :]
            else:
                self.assignments_t = linear_sum_assignment(stats.t(), maximize=True)
                histogram = stats[self.assignments_t[1], :]
                missing = list(set(range(self.n_classes + self.extra_clusters)) - set(self.assignments[0]))
                new_row = stats[missing, :].sum(0, keepdim=True)
                histogram = torch.cat([histogram, new_row], dim=0)
                new_col = torch.zeros(self.n_classes + 1, 1, dtype=histogram.dtype)
                self.histogram = torch.cat([histogram, new_col], dim=1)
        else:
            self.assignments = (torch.arange(self.n_classes).unsqueeze(1), torch.arange(self.n_classes).unsqueeze(1))
            self.histogram = stats
        hist = self.histogram.double()
        tp = torch.diag(hist)
        fp = hist.sum(0) - tp
        fn = hist.sum(1) - tp
        iou = tp / (tp + fp + fn)
        opc = tp.sum() / hist.sum()
        return {self.prefix + "mIoU": 100 * iou[~torch.isnan(iou)].mean().item(), self.prefix + "Accuracy": 100 * opc.item()}
