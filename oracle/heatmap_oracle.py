"""fp64 restatement of the dense correspondence heatmaps of src/plot_dino_correspondence.py:39-58 (get_heatmaps), for a
batch of images, on any device:

    1. q[b, :, p] = F.normalize(grid_sample(feats, query_points.permute(0, 2, 1, 3), bilinear, border,
                                            align_corners=True))[b, :, 0, p]                  (eps 1e-12)
    2. c[b, p, j] = q[b, :, p] . target[b, :, j] / max(||target[b, :, j]||, 1e-12)
    3. c -= c.mean over j; c = clamp(c, 0)                  (on the low-resolution map, as the reference does)
    4. F.interpolate(c, (H, W), mode="bilinear", align_corners=True)

Every step runs in float64 (the inputs are converted exactly) unless asked otherwise; the kernels
(stego_b200/csrc/heatmap.cu) are compared with this at a bar of 1e-4 on values in [0, 2].
"""
from __future__ import annotations

import torch
import torch.nn.functional as F


def heatmaps(feats: torch.Tensor, target: torch.Tensor, query_points: torch.Tensor, size,
             dtype: torch.dtype = torch.float64) -> torch.Tensor:
    """[B, P, H, W] for feats [B, E, h, w], target [B, E, h', w'], query_points [B, P, 1, 2], computed in `dtype`
    (float64; float32 runs the reference's own precision, as its lines do on the GPU)."""
    f = feats.to(dtype)
    t = target.to(dtype)
    qp = query_points.to(dtype)
    B, E = f.shape[:2]
    P = qp.shape[1]
    s = F.grid_sample(f, qp.permute(0, 2, 1, 3), mode="bilinear", padding_mode="border", align_corners=True)
    q = F.normalize(s.reshape(B, E, P), dim=1, eps=1e-12)
    tn = F.normalize(t.reshape(B, E, -1), dim=1, eps=1e-12)
    c = torch.einsum("bep,bej->bpj", q, tn)
    c = (c - c.mean(-1, keepdim=True)).clamp(0)
    c = c.reshape(B, P, t.shape[2], t.shape[3])
    return F.interpolate(c, tuple(int(v) for v in size), mode="bilinear", align_corners=True)


def low_res(feats: torch.Tensor, target: torch.Tensor, query_points: torch.Tensor) -> torch.Tensor:
    """Steps 1-3 alone: float64 [B, P, h', w'] (the map the upsample reads)."""
    return heatmaps(feats, target, query_points, target.shape[2:])
