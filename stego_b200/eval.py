"""Fused evaluation probes: the inner loop of the reference's `eval_segmentation.py` (:124-141) without
materialising the upsampled code.

    code = F.interpolate(code, label.shape[-2:], mode='bilinear', align_corners=False)
    linear_probs  = torch.log_softmax(model.linear_probe(code), dim=1)
    cluster_probs = model.cluster_probe(code, 2, log_probs=True)

becomes `fused_probe_log_probs(code_lowres, model.linear_probe, model.cluster_probe, label.shape[-2:], 2)`.
At 1024x2048 the reference moves 587 MB (fp32 upsampled code) per image per probe before it even starts;
the fused kernel reads the 9 MB low-res code and writes only the outputs (stego_eval_probes, eval_probes.cu).

With `run_crf=True` the reference then runs the dense CRF on each probe's log-probabilities of every frame
(eval_segmentation.py:133-141); `fused_eval_crf` is that whole loop body as one batched call (crf.cu's mean field
with both probes in one row).
"""
from __future__ import annotations

from typing import Optional, Sequence

import torch

from . import _lib, crf, ops


def fused_probe_log_probs(code: torch.Tensor, linear_probe: torch.nn.Module, cluster_probe: torch.nn.Module,
                          size: Sequence[int], alpha: float = 2.0, want_log_probs: bool = True,
                          want_argmax: bool = False, code_flipped: Optional[torch.Tensor] = None,
                          label: Optional[torch.Tensor] = None, linear_confusion: Optional[torch.Tensor] = None,
                          cluster_confusion: Optional[torch.Tensor] = None):
    """code: low-res [B, C, h, w] (any strides, CUDA; C <= 96, or 384 / 768 for projection_type None, where a bf16
    tokens-major code is read in place).  Returns (linear_log_probs, cluster_log_probs) [B,n,H,W]
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
    if code_flipped is not None:
        assert code_flipped.shape == code.shape
    codes = _eval_codes(code, code_flipped)
    tables = _probe_tables(linear_probe, cluster_probe, C)
    n_lin, n_clu = tables[0].shape[0], tables[2].shape[0]
    dev = code.device
    scratch = torch.empty(B * h * w, _EV_LD, dtype=torch.float32, device=dev)
    lin = torch.empty(B, n_lin, H, W, dtype=torch.float32, device=dev) if want_log_probs else None
    clu = torch.empty(B, n_clu, H, W, dtype=torch.float32, device=dev) if want_log_probs else None
    la = torch.empty(B, H, W, dtype=torch.uint8, device=dev) if want_argmax else None
    ca = torch.empty(B, H, W, dtype=torch.uint8, device=dev) if want_argmax else None
    lab = None
    if label is not None:
        _lib.require_cuda(label, linear_confusion, cluster_confusion)
        lab, _ = ops.probe_label(label, B, H, W)
        for t, n in ((linear_confusion, n_lin), (cluster_confusion, n_clu)):
            if t is not None:
                assert t.dtype == torch.int64 and t.is_contiguous() and tuple(t.shape) == (n, n_lin)
        if linear_confusion is None and cluster_confusion is None:
            raise ValueError("label given without a confusion matrix to accumulate into")
    _launch_probes(codes, tables, H, W, alpha, scratch, lin, clu, la, ca, lab, linear_confusion, cluster_confusion)
    if want_argmax:
        return lin, clu, la, ca
    return lin, clu


# the code widths of projection_type None (the backbone's own features): the probe kernels also read them in bf16
WIDE_DIMS = (384, 768)


def _tokens_major_bf16(t: torch.Tensor) -> bool:
    B, _, h, w = t.shape
    return (t.dtype == torch.bfloat16 and t.stride(1) == 1 and t.stride(2) == w * t.stride(3)
            and (B == 1 or t.stride(0) == h * w * t.stride(3)))


def _probe_codes(code: torch.Tensor, code_flipped: Optional[torch.Tensor]):
    """(x, xf, ld): the code and the flipped image's code (or None) as tokens-major fp32 views with one row stride ld."""
    x = ops.tokens_major(code)
    ld = x.stride(3)
    xf = None
    if code_flipped is not None:
        xf = ops.tokens_major(code_flipped)
        if xf.stride(3) != ld:  # one ld for both codes
            xf = xf.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
            x = x.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
            ld = x.stride(3)
    return x, xf, ld


def _eval_codes(code: torch.Tensor, code_flipped: Optional[torch.Tensor]):
    """(x, xf, ld, bf16): _probe_codes, except that bf16 tokens-major views of 384 / 768 channels with one row stride
    (the backbone's tokens) stay bf16 (bf16 = True), read in place by the probe kernels."""
    if (code.shape[1] in WIDE_DIMS and _tokens_major_bf16(code) and
            (code_flipped is None or (_tokens_major_bf16(code_flipped) and code_flipped.stride(3) == code.stride(3)))):
        return code.detach(), None if code_flipped is None else code_flipped.detach(), code.stride(3), True
    return (*_probe_codes(code, code_flipped), False)


def _probe_tables(linear_probe: torch.nn.Module, cluster_probe: torch.nn.Module, C: int):
    """(weight [n_lin, C], bias [n_lin], clusters [n_clu, C]) as contiguous fp32."""
    wl = linear_probe.weight.detach().float().reshape(linear_probe.weight.shape[0], C).contiguous()
    bl = linear_probe.bias.detach().float().contiguous()
    cl = cluster_probe.clusters.detach().float().contiguous()
    return wl, bl, cl


_EV_LD = 80  # eval_probes.cu EV_LD: floats per low-res pixel of the probe kernels' scratch


def _launch_probes(codes, tables, H: int, W: int, alpha: float, scratch: torch.Tensor, lin_log_probs, clu_log_probs,
                   lin_argmax, clu_argmax, label=None, lin_confusion=None, clu_confusion=None, mosaic=None) -> None:
    """One stego_eval_probes[_mosaic][_bf16] pass, the entry picked from the code's dtype and the placement.  codes:
    _eval_codes' (x, xf, ld, bf16) of a [B, C, h, w] code; tables: _probe_tables'; scratch [B*h*w, 80] fp32.  The
    outputs are the caller's tensors, each optional: log-probabilities [B, n, H, W], argmax maps [B, H, W] uint8 and,
    with label ([B, H, W] as ops.probe_label gives it), the int64 confusion counts.  mosaic: None for those frame
    layouts, or (tile0, tile_rows, tiles_per_row, pitch): the outputs are mosaic planes (stego_eval_probes_mosaic)."""
    x, xf, ld, bf16 = codes
    wl, bl, cl = tables
    B, C, h, w = x.shape
    name = "stego_eval_probes" + ("_mosaic" if mosaic else "") + ("_bf16" if bf16 else "")
    _lib.check(getattr(_lib.load(), name)(
        _lib.ptr(x), _lib.ptr(xf), ld, C, B, h, w, H, W, _lib.ptr(wl), _lib.ptr(bl), wl.shape[0], _lib.ptr(cl),
        cl.shape[0], float(alpha), _lib.ptr(scratch), _lib.ptr(lin_log_probs), _lib.ptr(clu_log_probs),
        _lib.ptr(lin_argmax), _lib.ptr(clu_argmax), _lib.ptr(label), 0 if label is None else label.element_size(),
        0 if label is None else wl.shape[0], _lib.ptr(lin_confusion), _lib.ptr(clu_confusion), *(mosaic or ()),
        _lib.stream()), name)


def _launch_crf_unary(codes, tables, H: int, W: int, alpha: float, scratch: torch.Tensor, unary: torch.Tensor,
                      Q: torch.Tensor, mosaic=None, probes: int = 3) -> None:
    """One stego_eval_crf_unary[_mosaic][_bf16] pass, the entry picked as in _launch_probes: the CRF's unary and initial
    Q rows into the caller's unary / Q, [B*H*W, 64] fp32 for frames.  mosaic: (tile0, tile_rows, tiles_per_row, pitch),
    the rows placed in a mosaic (stego_eval_crf_unary_mosaic), whose rows hold probes = 3 (both, 64 floats), 1 (the
    linear probe, 32) or 2 (the cluster probe, 32)."""
    x, xf, ld, bf16 = codes
    wl, bl, cl = tables
    B, C, h, w = x.shape
    name = "stego_eval_crf_unary" + ("_mosaic" if mosaic else "") + ("_bf16" if bf16 else "")
    _lib.check(getattr(_lib.load(), name)(
        _lib.ptr(x), _lib.ptr(xf), ld, C, B, h, w, H, W, _lib.ptr(wl), _lib.ptr(bl), wl.shape[0], _lib.ptr(cl),
        cl.shape[0], float(alpha), _lib.ptr(scratch), _lib.ptr(unary), _lib.ptr(Q),
        *((probes, *mosaic) if mosaic else ()), _lib.stream()), name)


# ----------------------------------------------------------------------------------------------------------------------
# CRF-refined evaluation
# ----------------------------------------------------------------------------------------------------------------------
_CRF_LD = 64  # crf.cu rows of two probes: linear probe in [0, 32), cluster probe in [32, 64)


_LABEL_DTYPES = (torch.uint8, torch.int32, torch.int64)


def _check_crf_args(code, linear_probe, cluster_probe, img, code_flipped, label, linear_confusion, cluster_confusion):
    """Every argument of fused_eval_crf checked before anything is launched: shapes, dtypes and limits first (ValueError),
    then the device (RuntimeError: CUDA tensors only).  Returns (B, C, h, w, H, W, n_lin, n_clu)."""
    if code.dim() != 4 or img.dim() != 4 or img.shape[1] != 3 or img.shape[0] != code.shape[0]:
        raise ValueError(f"fused_eval_crf: code [B, C, h, w] and img [B, 3, H, W] expected, got {tuple(code.shape)} and "
                         f"{tuple(img.shape)}")
    B, C, h, w = code.shape
    H, W = int(img.shape[2]), int(img.shape[3])
    n_lin, n_clu = int(linear_probe.weight.shape[0]), int(cluster_probe.clusters.shape[0])
    if not ((0 < C <= 96 or C in WIDE_DIMS) and 0 < n_lin <= 32 and 0 < n_clu <= 32):
        raise ValueError(f"fused_eval_crf: C={C}, n_lin={n_lin}, n_clu={n_clu} unsupported (C <= 96 or 384 / 768, "
                         f"classes <= 32)")
    if linear_probe.weight[0].numel() != C or cluster_probe.clusters.shape[1] != C:
        raise ValueError(f"fused_eval_crf: probes of {linear_probe.weight[0].numel()} / {cluster_probe.clusters.shape[1]} "
                         f"channels for a code of {C}")
    if H < h or W < w:
        raise ValueError(f"fused_eval_crf: img {H}x{W} is smaller than the code {h}x{w} (upsampling only)")
    if code_flipped is not None and code_flipped.shape != code.shape:
        raise ValueError(f"fused_eval_crf: code_flipped {tuple(code_flipped.shape)} != code {tuple(code.shape)}")
    if label is not None:
        if tuple(label.shape[-2:]) != (H, W) or label.numel() != B * H * W:
            raise ValueError(f"fused_eval_crf: label {tuple(label.shape)} does not match img {B}x{H}x{W}")
        if label.dtype not in _LABEL_DTYPES:
            raise ValueError(f"fused_eval_crf: label dtype {label.dtype} unsupported (uint8, int32 or int64)")
        if linear_confusion is None and cluster_confusion is None:
            raise ValueError("fused_eval_crf: label given without a confusion matrix to accumulate into")
    elif linear_confusion is not None or cluster_confusion is not None:
        raise ValueError("fused_eval_crf: confusion matrices given without a label")
    for t, n, name in ((linear_confusion, n_lin, "linear_confusion"), (cluster_confusion, n_clu, "cluster_confusion")):
        if t is not None and (t.dtype != torch.int64 or not t.is_contiguous() or tuple(t.shape) != (n, n_lin)):
            raise ValueError(f"fused_eval_crf: {name} must be a contiguous int64 [{n}, {n_lin}] tensor, got "
                             f"{t.dtype} {tuple(t.shape)}")
    _lib.require_cuda(code, img, code_flipped, label, linear_confusion, cluster_confusion, linear_probe.weight,
                      linear_probe.bias, cluster_probe.clusters)
    return B, C, h, w, H, W, n_lin, n_clu


def fused_eval_crf(code: torch.Tensor, linear_probe: torch.nn.Module, cluster_probe: torch.nn.Module, img: torch.Tensor,
                   alpha: float = 2.0, code_flipped: Optional[torch.Tensor] = None, label: Optional[torch.Tensor] = None,
                   linear_confusion: Optional[torch.Tensor] = None, cluster_confusion: Optional[torch.Tensor] = None,
                   want_marginals: bool = False):
    """The reference's CRF-refined eval step (eval_segmentation.py:124-141 with run_crf=True) as one batched call:

        code = (code + code_flipped.flip(3)) / 2                  # when code_flipped is given (flip-TTA)
        code = F.interpolate(code, img.shape[-2:], mode='bilinear', align_corners=False)
        linear_probs  = torch.log_softmax(linear_probe(code), dim=1)
        cluster_probs = cluster_probe(code, alpha, log_probs=True)
        lin_pred = stack([dense_crf(img[b], linear_probs[b])  for b]).argmax(1)      # src/crf.py:22-45
        clu_pred = stack([dense_crf(img[b], cluster_probs[b]) for b]).argmax(1)
        linear_metrics.update(lin_pred, label); cluster_metrics.update(clu_pred, label)

    code: low-res [B, C, h, w] (C <= 96 or 384 / 768, any strides; a bf16 tokens-major code of 384 / 768 channels is
    read in place); img: the normalised frames [B, 3, H, W]; both CUDA.  Returns
    (lin_pred, clu_pred) uint8 [B, H, W], the argmax of each probe's CRF marginals (lowest index on ties), and with
    want_marginals also (lin_Q [B, n_lin, H, W], clu_Q [B, n_clu, H, W]) fp32.  label [B, H, W] (uint8 with 255 =
    ignore, int32 or int64; the spatial size of img) with int64 `linear_confusion [n_lin, n_lin]` /
    `cluster_confusion [n_clu, n_lin]` (e.g. UnsupervisedMetrics.stats), accumulated in place: a pixel counts when
    0 <= label < n_lin and pred < n_lin (utils.py:219-229).  n_lin, n_clu <= 32 (extra clusters included).

    The log-probability maps are never written: the CRF unaries come straight from the low-res probe table.  Both probes
    share one bilateral lattice per frame, all frames run through each stage in one launch, and the splats are gathers
    in a fixed order, so two calls are bit-identical and a frame's results do not depend on the rest of the batch.
    The dense CRF itself is the one of stego_b200.crf (parameters of src/crf.py:13-19, 10 mean-field iterations).
    Host syncs: one per frame (the bilateral lattice's size from torch.unique), plus one the first time a frame size is
    seen (its cached position lattice).  Everything is checked before the first launch."""
    B, C, h, w, H, W, n_lin, n_clu = _check_crf_args(code, linear_probe, cluster_probe, img, code_flipped, label,
                                                      linear_confusion, cluster_confusion)
    dev = code.device
    lin_pred = torch.empty(B, H, W, dtype=torch.uint8, device=dev)
    clu_pred = torch.empty(B, H, W, dtype=torch.uint8, device=dev)
    lin_q = torch.empty(B, n_lin, H, W, dtype=torch.float32, device=dev) if want_marginals else None
    clu_q = torch.empty(B, n_clu, H, W, dtype=torch.float32, device=dev) if want_marginals else None
    lab = None if label is None else ops.probe_label(label, B, H, W)[0]
    _crf_pass(_eval_codes(code, code_flipped), _probe_tables(linear_probe, cluster_probe, C), img, alpha, lin_pred,
              clu_pred, lin_q, clu_q, lab, linear_confusion, cluster_confusion)
    if want_marginals:
        return lin_pred, clu_pred, lin_q, clu_q
    return lin_pred, clu_pred


def _crf_pass(codes, tables, img: torch.Tensor, alpha: float, lin_pred, clu_pred, lin_q, clu_q, label=None,
              lin_confusion=None, clu_confusion=None) -> None:
    """fused_eval_crf's work on checked arguments, into the caller's outputs (marginals and confusion counts optional):
    both probes' unary rows of the B frames img [B, 3, H, W], their lattices (one host sync per frame) and one mean
    field.  codes, tables and label as in _launch_probes."""
    B, _, H, W = img.shape
    N = H * W
    _, _, h, w = codes[0].shape
    dev = codes[0].device
    scratch = torch.empty(B * h * w, _EV_LD, dtype=torch.float32, device=dev)
    unary = torch.empty(B * N, _CRF_LD, dtype=torch.float32, device=dev)
    Q = torch.empty(B * N, _CRF_LD, dtype=torch.float32, device=dev)
    _launch_crf_unary(codes, tables, H, W, alpha, scratch, unary, Q)
    lg = crf._position_lattice(H, W, dev)
    lb = crf._bilateral_lattice(crf.prepare_image(frame) for frame in img.detach())
    n_lin, n_clu = tables[0].shape[0], tables[2].shape[0]
    crf._launch_mean_field(B, N, lg, lb, unary, Q, [(n_lin, lin_q, lin_pred, lin_confusion),
                                                    (n_clu, clu_q, clu_pred, clu_confusion)],
                           label=label, n_classes=0 if label is None else n_lin)


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
