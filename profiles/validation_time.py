"""Images per second of LitUnsupervisedSegmenter.validation_step (ViT-S/8 and ViT-B/8, 320 x 320, B = 16, 27 classes)
against the reference's validation op sequence (src/train_segmentation.py:260-269) in PyTorch eager on the same card.

    python profiles/validation_time.py [--out FILE]

Prints one JSON line.  Times are CUDA-event times over repeated calls after a warm-up; each call ends with the preview
dict copied to the host (5 images, as the reference's), so both sides include that synchronising copy.  The eager side
is the reference's fp32 computation with torch's default math settings: the DINO ViT forward and the head
(modules.py:90-118, eval mode), F.interpolate to the label size, the linear probe 1x1 conv and argmax, ClusterLookup
with alpha None and argmax, and UnsupervisedMetrics.update's bincount for both probes (utils.py:219-229).
"""
import argparse
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
from _measure import card, emit, window_ms  # noqa: E402

B, RES, N_CLASSES, N_IMAGES = 16, 320, 27, 5
WINDOW = dict(warmup=2, min_window_s=1.0, min_iters=5, max_iters=200)


def eager_validation(sd, head, lin_w, lin_b, clusters, img, label, arch):
    """train_segmentation.py:260-275 in torch eager (fp32), with UnsupervisedMetrics.update's bincount."""
    import stego_oracle as O
    n, k = N_CLASSES, clusters.shape[0]
    with torch.no_grad():
        feats = O.vit_image_feat(sd, img, arch, 8)
        _, code = O.head_forward(feats, head, None)
        code = F.interpolate(code, label.shape[-2:], mode="bilinear", align_corners=False)
        linear_preds = F.conv2d(code, lin_w, lin_b).argmax(1)
        _, probs = O.cluster_lookup(code, clusters, None)
        cluster_preds = probs.argmax(1)
        stats = []
        for preds, rows in ((linear_preds, n), (cluster_preds, k)):
            actual, p = label.reshape(-1), preds.reshape(-1)
            mask = (actual >= 0) & (actual < n) & (p >= 0) & (p < n)
            stats.append(torch.bincount(rows * actual[mask] + p[mask], minlength=n * rows).reshape(n, rows).t())
        return dict(img=img[:N_IMAGES].cpu(), linear_preds=linear_preds[:N_IMAGES].cpu(),
                    cluster_preds=cluster_preds[:N_IMAGES].cpu(), label=label[:N_IMAGES].cpu()), stats


def case(arch, dev):
    import stego_oracle as O
    from stego_b200.config import make_cfg
    from stego_b200.segmenter import LitUnsupervisedSegmenter
    cfg = make_cfg(model_type=arch, random_backbone_init=True)
    torch.manual_seed(0)
    model = LitUnsupervisedSegmenter(N_CLASSES, cfg).to(dev)
    sd = O.perturb_vit_state(O.vit_random_state(arch, 8, seed=3))
    model.net.model.load_state_dict(sd)
    model.train()
    g = torch.Generator(device=dev).manual_seed(0)
    img = torch.randn(B, 3, RES, RES, device=dev, generator=g)
    label = torch.randint(-1, N_CLASSES, (B, RES, RES), device=dev, generator=g)
    batch = dict(img=img, label=label)
    t_ours, n_ours = window_ms(lambda: model.validation_step(batch, 0), **WINDOW)

    sdd = {k: v.to(dev) for k, v in sd.items()}
    head = {k[len("net."):]: v.detach() for k, v in model.named_parameters() if k.startswith("net.cluster")}
    lw, lb = model.linear_probe.weight.detach(), model.linear_probe.bias.detach()
    cl = model.cluster_probe.clusters.detach()
    t_eager, n_eager = window_ms(lambda: eager_validation(sdd, head, lw, lb, cl, img, label, arch), **WINDOW)

    # agreement of the two on this batch (bf16 ViT here, fp32 there: near-ties differ)
    model.linear_metrics.reset()
    model.cluster_metrics.reset()
    ours = model.validation_step(batch, 0)
    ref, _ = eager_validation(sdd, head, lw, lb, cl, img, label, arch)
    agree = {k: float((ours[k] == ref[k]).double().mean()) for k in ("linear_preds", "cluster_preds")}
    return dict(arch=arch, B=B, res=RES, n_classes=N_CLASSES, ours_ms=round(t_ours, 3), ours_calls=n_ours,
                ours_images_per_s=round(B * 1e3 / t_ours, 1), eager_ms=round(t_eager, 3), eager_calls=n_eager,
                eager_images_per_s=round(B * 1e3 / t_eager, 1), speedup_vs_eager=round(t_eager / t_ours, 2),
                preview_pred_agreement=agree)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    emit(dict(card=card(), cases=[case(arch, dev) for arch in ("vit_small", "vit_base")], gpu_info_after=card()), a.out)


if __name__ == "__main__":
    main()
