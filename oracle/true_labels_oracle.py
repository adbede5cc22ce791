"""CPU oracle of the training step with cfg.use_true_labels.  TEST INFRASTRUCTURE ONLY.

src/train_segmentation.py:135-140: with use_true_labels the correspondence loss takes the one-hot ground truth as its
teacher signal instead of the DINO features,

    signal     = one_hot_feats(label + 1,     n_classes + 1)
    signal_pos = one_hot_feats(label_pos + 1, n_classes + 1)

(utils.py:65-66), both at label resolution; class 0 is "unlabelled" (label -1).  Everything else is the step of
stego_oracle.training_losses, whose pieces are reused here unchanged.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

import stego_oracle as O

Tensor = torch.Tensor


def one_hot_feats(labels: Tensor, n_classes: int) -> Tensor:
    """utils.py:65-66: F.one_hot(labels, n_classes) as an fp32 [B, n_classes, H, W] map (raises on labels outside
    0 .. n_classes - 1)."""
    return F.one_hot(labels, n_classes).permute(0, 3, 1, 2).to(torch.float32)


def label_signals(label: Tensor, label_pos: Tensor, n_classes: int):
    """train_segmentation.py:135-137."""
    return one_hot_feats(label + 1, n_classes + 1), one_hot_feats(label_pos + 1, n_classes + 1)


def training_losses(image_feat: Tensor, image_feat_pos: Tensor, hp, probes, label: Tensor, label_pos: Tensor, masks,
                    masks_pos, coords1, coords2, perms, cfg: O.LossCfg, n_classes: int, round_bf16: bool = False):
    """stego_oracle.training_losses (train_segmentation.py:130-225) with the teacher signal of :135-140.  The
    Dropout2d noise of the returned features (masks[2]) is drawn by the caller as the reference's net() draws it and
    scales nothing the loss reads."""
    _, code = O.head_forward(image_feat, hp, masks, round_bf16)
    _, code_pos = O.head_forward(image_feat_pos, hp, masks_pos, round_bf16)
    signal, signal_pos = label_signals(label, label_pos, n_classes)
    out6 = O.correlation_loss(signal, signal_pos, code, code_pos, coords1, coords2, perms, cfg)
    corr = O.weighted_correspondence_loss(out6, cfg)
    detached = code.detach().clone()
    lin = O.linear_probe_loss(detached, probes["linear_probe.weight"], probes["linear_probe.bias"], label, n_classes)
    clu, _ = O.cluster_lookup(detached, probes["cluster_probe.clusters"], None)
    return dict(total=corr + lin + clu, corr=corr, linear=lin, cluster=clu,
                pos_intra=out6[0], pos_inter=out6[2], neg_inter=out6[4].mean(),
                cd_intra=out6[1].mean(), cd_inter=out6[3].mean(), cd_neg=out6[5].mean(), code=code)
