"""Restatement of the DINO baseline (projection_type None: src/modules.py:108-113, `code = image_feat`) over the
functional ViT of oracle/stego_oracle.py: its code (with eval_step_oracle.eval_loop, the reference's evaluation loop
body on that model) and its training step, where only the probes learn (correspondence_weight 0:
train_segmentation.py:210-230).  tests/test_baseline.py checks both against the reference's own outputs
(tests/golden/baseline.pt, written by oracle/make_golden_baseline.py) on the CPU; tests/test_baseline_gpu.py holds
eval_step and training_step to the same fixture.
"""
from __future__ import annotations

import os
import sys
from typing import Dict

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import kk_oracle  # noqa: E402
import stego_oracle as O  # noqa: E402


def net_code(vit_sd: Dict[str, torch.Tensor], img: torch.Tensor, arch: str = "vit_small", patch: int = 8,
             feat_type: str = "feat") -> torch.Tensor:
    """The eval-mode DinoFeaturizer's code with projection_type None: the backbone's features, [B, E, h, w]."""
    return kk_oracle.image_feat(vit_sd, img, arch, feat_type, patch)


def probe_losses(code: torch.Tensor, probes: Dict[str, torch.Tensor], label: torch.Tensor, n_classes: int):
    """(linear loss, cluster loss) of train_segmentation.py:210-223 on the detached code; probes holds
    linear_probe.weight / .bias and cluster_probe.clusters (requires_grad for the gradients)."""
    lin = O.linear_probe_loss(code, probes["linear_probe.weight"], probes["linear_probe.bias"], label, n_classes)
    clu, _ = O.cluster_lookup(code, probes["cluster_probe.clusters"], None)
    return lin, clu


def training_steps(vit_sd: Dict[str, torch.Tensor], probes: Dict[str, torch.Tensor], batches, n_classes: int,
                   arch: str = "vit_small", lr: float = 5e-3):
    """The baseline's training steps: per batch the losses of probe_losses, one backward, then torch.optim.Adam
    (lr 5e-3, train_segmentation.py:378-383) on the probes.  Returns per step the logged losses and the probes after
    the update."""
    p = {k: v.clone().requires_grad_(True) for k, v in probes.items()}
    state = {k: (torch.zeros_like(v), torch.zeros_like(v)) for k, v in p.items()}
    out = []
    for i, batch in enumerate(batches):
        code = net_code(vit_sd, batch["img"], arch).detach()
        lin, clu = probe_losses(code, p, batch["label"], n_classes)
        total = lin + clu
        grads = torch.autograd.grad(total, list(p.values()))
        with torch.no_grad():
            for (k, v), g in zip(p.items(), grads):
                O.adam_step(v, g, *state[k], i + 1, lr)
        out.append(dict(logged={"loss/linear": float(lin.detach()), "loss/cluster": float(clu.detach()),
                                "loss/total": float(total.detach())},
                        params={k: v.detach().clone() for k, v in p.items()}))
    return out
