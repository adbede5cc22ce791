"""Correspondence precision-recall: do feature / code correlations predict label co-occurrence?

The STEGO paper's diagnostic of `src/plot_pr_curves.py` (LitRecalibrator, :95-220), as a streaming metric.  For each
image, every pair (row sample i at coords1, column sample j at coords2) of the S = feature_samples^2 samples is scored
by the cosine of the two sampled, L2-normalised vectors (`tensor_correlation(norm(sample(f, coords1)),
norm(sample(f, coords2)))`, get_net_fd :108-121) for two methods: "code" (the head's output, the reference's
"STEGO (Ours)") and "feats" (the backbone features, "DINO").  A pair is positive when both samples are *pure* with the
same class: every bilinear tap with a non-zero weight has that class, where a tap's class is label + 1 for
0 <= label < n_classes and 0 otherwise (unlabelled pairs count as positives, as in the reference).

Instead of concatenating B S^2 scores per batch on the host and handing them to sklearn (:152-167), the correlation
kernel bins the scores in its epilogue: `corr_kernel<CP_PR>` adds int64 counts [method][negative, positive][PR_BINS]
on the device, and `compute()` turns the counts into sklearn's average precision and curve.

Deviations from the reference, on purpose:
- Targets.  The reference takes `ld.to(int64)` of the fp32 label correlation; the fp32 bilinear weights of a pure
  sample do not always sum to exactly 1, so some pairs with ld = 1 exactly become ld = 0.99999994 and count as negatives
  there.  The rule here is the exact one (ld == 1 in exact arithmetic).
- Scores.  `prep_fd`'s global min-max rescale is monotone and does not change the AP; it is not applied.  Scores are
  binned at k = clamp(floor((score + 1) * PR_BINS / 2), 0, PR_BINS - 1), so `ap` is sklearn's AP with the bin index as
  the score, and `ap_bounds` bound the AP of the unbinned fp32 scores.
- The reference script runs its MoCo and CRF baselines too; those models are not part of this package.
"""
from __future__ import annotations

import types
from typing import Dict

import numpy as np
import torch

from . import _lib, corr, ops

PR_BINS = 4096  # STEGO_PR_BINS
METHODS = ("feats", "code")  # index 0 / 1 of the counts' first axis


def _pr_spec(fs: int):
    """A correspondence spec with no negatives: slot 0 samples at coords1, slot 1 at coords2 (of the same image)."""
    cfg = types.SimpleNamespace(feature_samples=fs, neg_samples=0, pointwise=False, zero_clamp=False, stabalize=False,
                                pos_intra_shift=0.0, pos_inter_shift=0.0, neg_inter_shift=0.0)
    return corr.TiledLossSpec(cfg, n_neg=0)


def _psi_diff(x: np.ndarray, p: np.ndarray) -> np.ndarray:
    """psi(x + p) - psi(x) for x >= 1.  Below 16 from scipy's digamma; above, where the two digammas are close and their
    difference would lose digits, as log1p(p / x) + r(x + p) - r(x) with the asymptotic series
    r(z) = psi(z) - ln z = -1/(2z) - 1/(12z^2) + 1/(120z^4) - 1/(252z^6) + 1/(240z^8) (truncation < 1e-14 at z >= 16)."""
    from scipy.special import digamma
    x = np.asarray(x, dtype=np.float64)
    p = np.asarray(p, dtype=np.float64)
    big = x >= 16.0
    xs = np.where(big, x, 16.0)

    def r(z):
        z2 = 1.0 / (z * z)
        return -0.5 / z - z2 * (1.0 / 12 - z2 * (1.0 / 120 - z2 * (1.0 / 252 - z2 / 240)))

    return np.where(big, np.log1p(p / xs) + (r(xs + p) - r(xs)), digamma(x + p) - digamma(np.minimum(x, 16.0)))


def _digamma_sum(a: np.ndarray, c: np.ndarray, p: np.ndarray) -> np.ndarray:
    """sum_{i=1}^{p} (a + i) / (c + i) = p - (c - a) (psi(c + p + 1) - psi(c + 1)), elementwise (p = 0 gives 0)."""
    return p - (c - a) * _psi_diff(np.asarray(c, dtype=np.float64) + 1.0, p)


def pr_from_counts(neg: np.ndarray, pos: np.ndarray) -> Dict[str, object]:
    """Precision-recall summary of one method's counts (negatives / positives per bin, bin index = score), float64.

    ap: sklearn's average_precision_score(y, bin_index); precision, recall: precision_recall_curve(y, bin_index)'s
    first two outputs; ap_bounds: (lo, hi), the smallest and largest AP over every order of the pairs inside each bin
    (its negatives first / its positives first), which contain the AP of any scores that bin this way;
    num_pairs, num_pos."""
    neg = np.asarray(neg, dtype=np.float64)
    pos = np.asarray(pos, dtype=np.float64)
    nz = np.nonzero((neg + pos) > 0)[0][::-1]  # the thresholds: non-empty bins, highest score first
    fp_k, tp_k = neg[nz], pos[nz]
    tps, fps = np.cumsum(tp_k), np.cumsum(fp_k)
    n_pos = float(tps[-1]) if len(tps) else 0.0
    n_pairs = int(neg.sum() + pos.sum())
    out: Dict[str, object] = {"num_pairs": n_pairs, "num_pos": int(pos.sum())}
    if n_pairs == 0:
        out.update(ap=float("nan"), ap_bounds=(float("nan"), float("nan")), precision=np.ones(1), recall=np.zeros(1))
        return out
    precision = tps / (tps + fps)
    recall = np.ones_like(tps) if n_pos == 0 else tps / n_pos
    # sklearn's output order: lowest threshold first, then the (precision 1, recall 0) end point
    out["precision"] = np.hstack((precision[::-1], 1.0))
    out["recall"] = np.hstack((recall[::-1], 0.0))
    r = out["recall"]
    out["ap"] = float(-np.sum(np.diff(r) * out["precision"][:-1]))  # sklearn's _binary_uninterpolated_average_precision
    if n_pos == 0:
        out["ap_bounds"] = (out["ap"], out["ap"])
        return out
    a = tps - tp_k            # TP before the bin
    c = a + fps - fp_k        # TP + FP before the bin
    hi = _digamma_sum(a, c, tp_k).sum() / n_pos
    lo = _digamma_sum(a, c + fp_k, tp_k).sum() / n_pos
    out["ap_bounds"] = (float(lo), float(hi))
    return out


class CorrespondencePR:
    """Streaming correspondence precision-recall of the head's code and the backbone features (plot_pr_curves.py).

    `update` adds one batch's pair counts on the device (no host synchronisation), `reset` zeroes them and `compute`
    copies them to the host once and returns {"code": {...}, "feats": {...}} with the fields of `pr_from_counts`.
    The counts (`counts`, int64 [2 (feats, code)][2 (negative, positive)][PR_BINS]) add up across batches; under
    torch.distributed one all_reduce of `counts` gives the global metric."""

    def __init__(self, n_classes: int, device=None):
        if not 1 <= int(n_classes) <= 255:
            raise RuntimeError(f"stego_b200: CorrespondencePR takes n_classes 1..255, got {n_classes}")
        self.n_classes = int(n_classes)
        dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.counts = torch.zeros(len(METHODS), 2, PR_BINS, dtype=torch.int64, device=dev)

    def reset(self) -> None:
        self.counts.zero_()

    def update(self, feats: torch.Tensor, code: torch.Tensor, label: torch.Tensor, coords1: torch.Tensor,
               coords2: torch.Tensor) -> None:
        """feats [B, E, h, w] (fp32 or bf16, E <= 768), code [B, D, h', w'] (D <= 96), label [B, H, W] or
        [B, 1, H, W] (int64, int32 or uint8, any resolution), coords1 / coords2 [B, fs, fs, 2] in [-1, 1] (values
        beyond are clamped to the border, as grid_sample does), fs 1..64.  Any memory layout (NCHW, channels-last)."""
        _lib.require_cuda(feats, code, label, coords1, coords2)
        for t in (feats, code, label, coords1, coords2):
            if t.device != self.counts.device:
                raise RuntimeError(f"stego_b200: CorrespondencePR input on {t.device}, counts on {self.counts.device}")
        if feats.dim() != 4 or code.dim() != 4:
            raise RuntimeError("stego_b200: feats and code must be [B, C, h, w]")
        B = feats.shape[0]
        if code.shape[0] != B or label.shape[0] != B:
            raise RuntimeError(f"stego_b200: batch sizes differ: feats {B}, code {code.shape[0]}, "
                               f"label {label.shape[0]}")
        if coords1.dim() != 4 or coords1.shape[0] != B or coords1.shape[1] != coords1.shape[2] \
                or coords1.shape[3] != 2 or coords2.shape != coords1.shape:
            raise RuntimeError(f"stego_b200: coords must both be [B, fs, fs, 2], got {tuple(coords1.shape)} and "
                               f"{tuple(coords2.shape)}")
        fs = coords1.shape[1]
        if not 1 <= fs <= corr.MAX_TILED_FS:
            raise RuntimeError(f"stego_b200: feature_samples={fs} is outside 1..{corr.MAX_TILED_FS}")
        if label.dtype not in (torch.int64, torch.int32, torch.uint8):
            raise RuntimeError(f"stego_b200: label dtype {label.dtype} unsupported (int64, int32, uint8)")
        if label.dim() == 4 and label.shape[1] != 1 or label.dim() not in (3, 4):
            raise RuntimeError(f"stego_b200: label must be [B, H, W] or [B, 1, H, W], got {tuple(label.shape)}")
        for name, t in (("feats", feats), ("code", code)):
            if t.dtype not in (torch.float32, torch.bfloat16):
                raise RuntimeError(f"stego_b200: {name} must be fp32 or bf16, got {t.dtype}")
        E, D = feats.shape[1], code.shape[1]
        if not 1 <= E <= 768:
            raise RuntimeError(f"stego_b200: feature channels {E} unsupported (1..768)")
        if not 1 <= D <= 96:
            raise RuntimeError(f"stego_b200: code dim {D} unsupported (1..96)")
        H, W = label.shape[-2], label.shape[-1]
        if min(H, W, feats.shape[2], feats.shape[3], code.shape[2], code.shape[3]) < 2:
            raise RuntimeError("stego_b200: feats, code and label need at least 2 x 2 pixels")
        spec = _pr_spec(fs)
        c1 = coords1.detach().to(torch.float32).contiguous()
        c2 = coords2.detach().to(torch.float32).contiguous()
        lab, nbytes = ops.probe_label(label, B, H, W)
        lib = _lib.load()
        ids = torch.empty(2, B, spec.rows, dtype=torch.int32, device=feats.device)
        _lib.check(lib.stego_sample_label_ids(_lib.ptr(lab), nbytes, _lib.ptr(c1), _lib.ptr(c2), _lib.ptr(ids), B,
                                              self.n_classes, H, W, fs, _lib.stream()), "stego_sample_label_ids")
        f = feats.detach()
        e_pad = corr.teacher_width(E)
        ftiles = corr.build_tiles(f, f, c1, c2, None, spec, e_pad)
        cd = code.detach()
        ctiles = corr.build_tiles(cd, cd, c1, c2, None, spec, corr.CODE_PAD)
        _lib.check(lib.stego_corr_pr(_lib.ptr(ftiles), _lib.ptr(ctiles), _lib.ptr(ids), _lib.ptr(self.counts), B, fs,
                                     e_pad, D, _lib.stream()), "stego_corr_pr")

    def compute(self) -> Dict[str, Dict[str, object]]:
        """One device-to-host copy of the counts, then `pr_from_counts` per method (float64, host)."""
        c = self.counts.cpu().numpy()
        return {m: pr_from_counts(c[k, 0], c[k, 1]) for k, m in enumerate(METHODS)}


# ---------------------------------------------------------------------------------------------------------------------
# Dense correspondence heatmaps (src/plot_dino_correspondence.py:39-58)
# ---------------------------------------------------------------------------------------------------------------------
def _strides(t: torch.Tensor):
    return (int(s) for s in t.stride())


def correspondence_heatmaps(feats: torch.Tensor, target: torch.Tensor, query_points: torch.Tensor,
                            size) -> torch.Tensor:
    """The heatmaps of `get_heatmaps` for a batch: out[b, p] = F.interpolate(clamp(c - c.mean(), 0), size, bilinear,
    align_corners=True) with c[j] = <normalize(sample(feats, query_points)[b, :, p]), normalize(target[b, :, j])>
    (F.normalize's eps 1e-12) over every position j of target[b].  `target = feats` gives the "Self Correspondence"
    maps, the features of the KNN image the "KNN Correspondence" maps.

    feats [B, E, h, w] and target [B, E, h', w']: fp32 or bf16, any memory layout, 1 <= E <= 768; query_points
    [B, P, 1, 2] (x, y) in [-1, 1] (values beyond are clamped to the border, as grid_sample does); size = (H, W).
    Returns fp32 [B, P, H, W] on the device, without synchronising with the host."""
    _lib.require_cuda(feats, target, query_points)
    for t in (target, query_points):
        if t.device != feats.device:
            raise RuntimeError(f"stego_b200: correspondence_heatmaps input on {t.device}, feats on {feats.device}")
    if feats.dim() != 4 or target.dim() != 4:
        raise RuntimeError("stego_b200: feats and target must be [B, C, h, w]")
    B, E, h, w = feats.shape
    if target.shape[0] != B or target.shape[1] != E:
        raise RuntimeError(f"stego_b200: target {tuple(target.shape)} does not match feats {tuple(feats.shape)} in "
                           "batch and channels")
    if query_points.dim() != 4 or query_points.shape[0] != B or query_points.shape[2] != 1 \
            or query_points.shape[3] != 2:
        raise RuntimeError(f"stego_b200: query_points must be [B, P, 1, 2], got {tuple(query_points.shape)}")
    if not query_points.is_floating_point():
        raise RuntimeError(f"stego_b200: query_points must be floating point, got {query_points.dtype}")
    for name, t in (("feats", feats), ("target", target)):
        if t.dtype not in (torch.float32, torch.bfloat16):
            raise RuntimeError(f"stego_b200: {name} must be fp32 or bf16, got {t.dtype}")
    if not 1 <= E <= 768:
        raise RuntimeError(f"stego_b200: feature channels {E} unsupported (1..768)")
    if len(tuple(size)) != 2:
        raise RuntimeError(f"stego_b200: size must be (H, W), got {size}")
    H, W = (int(s) for s in size)
    P = query_points.shape[1]
    ht, wt = target.shape[2], target.shape[3]
    if min(B, P, h, w, ht, wt) < 1 or not 1 <= H <= 65535 or W < 1:
        raise RuntimeError(f"stego_b200: empty or oversized heatmap request: B={B} P={P} feats {h}x{w} "
                           f"target {ht}x{wt} size {H}x{W}")
    dev = feats.device
    e_pad = -(-E // 8) * 8
    t_bf16 = target.dtype == torch.bfloat16
    nseg = 2 if t_bf16 else 3
    lib = _lib.load()
    f, t = feats.detach(), target.detach()
    t_ops = torch.empty(B, ht * wt, nseg * e_pad, dtype=torch.bfloat16, device=dev)
    inv = torch.empty(B, ht * wt, dtype=torch.float32, device=dev)
    _lib.check(lib.stego_heatmap_prep_target(_lib.ptr(t), int(t_bf16), *_strides(t), B, E, ht, wt, e_pad,
                                             _lib.ptr(t_ops), _lib.ptr(inv), _lib.stream()),
               "stego_heatmap_prep_target")
    pts = query_points.detach().to(torch.float32).contiguous()
    q_ops = torch.empty(B, P, nseg * e_pad, dtype=torch.bfloat16, device=dev)
    _lib.check(lib.stego_heatmap_sample_queries(_lib.ptr(f), int(f.dtype == torch.bfloat16), *_strides(f),
                                                _lib.ptr(pts), B, P, E, h, w, e_pad, nseg, _lib.ptr(q_ops),
                                                _lib.stream()), "stego_heatmap_sample_queries")
    corr = ops.gemm_batched(q_ops, t_ops, torch.empty(B, P, ht * wt, dtype=torch.float32, device=dev))
    _lib.check(lib.stego_heatmap_finish(_lib.ptr(corr), _lib.ptr(inv), B, P, ht * wt, _lib.stream()),
               "stego_heatmap_finish")
    out = torch.empty(B, P, H, W, dtype=torch.float32, device=dev)
    _lib.check(lib.stego_heatmap_upsample(_lib.ptr(corr), _lib.ptr(out), B * P, ht, wt, H, W, _lib.stream()),
               "stego_heatmap_upsample")
    return out


def get_heatmaps(net, img: torch.Tensor, img_pos: torch.Tensor, query_points: torch.Tensor):
    """Drop-in for the reference's `get_heatmaps(net, img, img_pos, query_points)` (plot_dino_correspondence.py:39-58):
    `net(x)[0]` are the features of one image; returns the ("Self", "KNN") correspondence heatmaps as CPU fp32 tensors
    [P, H, W] and [P, H', W'] at the sizes of img and img_pos.  `net` runs in whatever mode the caller left it.  Like the
    reference it takes one image (B = 1); for a batch call `correspondence_heatmaps` directly."""
    if img.shape[0] != 1 or img_pos.shape[0] != 1 or query_points.dim() != 4 or query_points.shape[0] != 1:
        raise RuntimeError(f"stego_b200: get_heatmaps takes one image, as the reference does (img "
                           f"{tuple(img.shape)}, img_pos {tuple(img_pos.shape)}, query_points "
                           f"{tuple(query_points.shape)}); use correspondence_heatmaps for a batch")
    feats1, _ = net(img.cuda())
    feats2, _ = net(img_pos.cuda())
    qp = query_points.to(feats1.device)
    heatmap_intra = correspondence_heatmaps(feats1, feats1, qp, img.shape[2:])[0].cpu()
    heatmap_inter = correspondence_heatmaps(feats1, feats2, qp, img_pos.shape[2:])[0].cpu()
    return heatmap_intra, heatmap_inter
