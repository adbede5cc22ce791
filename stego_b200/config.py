"""Attribute-style config with the reference's shipped defaults (src/configs/train_config.yml).
The modules accept any attribute-style object (OmegaConf DictConfig, SimpleNamespace, ...); this helper is
only used by bench.py, smoke() and the tests, where Hydra / OmegaConf are not installed."""
from __future__ import annotations

from types import SimpleNamespace

TRAIN_DEFAULTS = dict(
    # model
    model_type="vit_small", arch="dino", dino_feat_type="feat", projection_type="nonlinear", dino_patch_size=8,
    granularity=1, continuous=True, dim=70, dropout=True, zero_clamp=True, pretrained_weights=None,
    extra_clusters=0, use_true_labels=False,
    # loss
    lr=5e-4, use_salience=False, stabalize=False, stop_at_zero=True, pointwise=True, feature_samples=11,
    neg_samples=5, aug_alignment_weight=0.0, correspondence_weight=1.0,
    neg_inter_weight=0.63, pos_inter_weight=0.25, pos_intra_weight=0.67,
    neg_inter_shift=0.46, pos_inter_shift=0.12, pos_intra_shift=0.18,
    rec_weight=0.0, repulsion_weight=0.0, crf_weight=0.0,
    alpha=.5, beta=.15, gamma=.05, w1=10.0, w2=3.0, shift=0.00, crf_samples=1000,
    reset_probe_steps=None, hist_freq=100, batch_size=16, res=224, dataset_name="cocostuff27", output_root="../",
    n_images=5,  # images per validation_step preview
    # stego_b200 execution switches (not in the reference config; read with getattr(..., default) by the modules)
    cuda_graph=True,   # replay the frozen ViT as one CUDA graph per input shape
    fused_step=True,   # hand-scheduled training step (fused_step.py) instead of the autograd-stitched one
    overlap_update=True,  # parameter update on the side stream under the next step's backbone
    p2p_update=True,   # N > 1: gradient all-reduce fused into Adam over NVLink peer memory (NCCL all-reduce as the fallback)
    fused_rec_crf=False,  # rec_weight / crf_weight > 0 on the hand-scheduled step (fp32 img and dim <= 80 for the CRF
                          # term) instead of the autograd-stitched one
)


def make_cfg(**overrides) -> SimpleNamespace:
    d = dict(TRAIN_DEFAULTS)
    d.update(overrides)
    return SimpleNamespace(**d)
