"""Cost of the DINO baseline (projection_type None: the probes on the backbone's 384 / 768 channels) against the
shipped configuration (nonlinear head, dim 70), on one GPU:

  * training: LitUnsupervisedSegmenter.training_step at c1 (ViT-S/8 224², B = 32) and at ViT-B/8 320², B = 32: the
    shipped step (hand-scheduled, correspondence loss) and the baseline's (autograd path: the frozen backbone on img
    alone, then the wide probe kernels and Adam);
  * evaluation: eval_step on 1024 x 2048 frames (BASELINE.json configs[4]), B = 1 and 4, 27 classes, labels at the
    frames' size, with and without run_crf, for head70_vit_small (the shipped code), baseline384_vit_small and
    baseline768_vit_base.

    python profiles/baseline_time.py [--out profiles/baseline_time_h100.json]

Per case: ms per call (CUDA events over at least 0.5 s of back-to-back calls after a warm-up, the median of three
rounds).  Then, in separate torch.profiler runs, the CUDA time of the wide kernels against the whole call's kernel time:
the probe kernels of one baseline training step (linear_logits_wide, linear_ce, wide_wgrad, cluster_wide_fwd,
cluster_norm_bwd) and the preparation kernel of one eval_step at B = 4 (eval_prep_kernel for the head's code,
eval_prep_wide_kernel for the backbone's): whether they stay negligible next to the backbone.  Prints one JSON object
with the card.
"""
from __future__ import annotations

import argparse
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
from _measure import card, emit, window_ms  # noqa: E402

MODELS = {
    "head70_vit_small": dict(model_type="vit_small"),
    "baseline384_vit_small": dict(model_type="vit_small", projection_type=None, dim=384, correspondence_weight=0.0),
    "baseline768_vit_base": dict(model_type="vit_base", projection_type=None, dim=768, correspondence_weight=0.0),
}
H, W, N_CLASSES, ROUNDS = 1024, 2048, 27, 3
WINDOW = dict(warmup=1, min_window_s=0.5, min_iters=2, max_iters=50)


def make_model(over, dev):
    import stego_oracle as O
    from stego_b200.config import make_cfg
    from stego_b200.segmenter import LitUnsupervisedSegmenter
    torch.manual_seed(0)
    model = LitUnsupervisedSegmenter(N_CLASSES, make_cfg(random_backbone_init=True, **over)).to(dev)
    model.net.model.load_state_dict(O.perturb_vit_state(O.vit_random_state(over["model_type"], 8, seed=3)))
    model.train()
    return model


def make_batch(B, dev):
    g = torch.Generator(device=dev).manual_seed(0)
    return dict(img=torch.randn(B, 3, H, W, device=dev, generator=g),
                label=torch.randint(-1, N_CLASSES, (B, H, W), device=dev, generator=g))


TRAIN_CASES = (("vit_small", 224, 32), ("vit_base", 320, 32))
TRAIN_WINDOW = dict(warmup=3, min_window_s=0.5, min_iters=5, max_iters=200)
WIDE_TRAIN_KERNELS = ("linear_logits_wide", "linear_ce_kernel", "linear_ce_finish", "wide_wgrad", "cluster_wide_fwd",
                      "cluster_norm_bwd", "sum_partials")


def train_model(arch, baseline, dev):
    over = dict(model_type=arch)
    if baseline:
        over.update(projection_type=None, dim=384 if arch == "vit_small" else 768, correspondence_weight=0.0)
    model = make_model(over, dev)
    model.configure_optimizers()
    return model


def train_batch(B, res, dev):
    g = torch.Generator(device=dev).manual_seed(1)
    img = torch.randn(B, 3, res, res, device=dev, generator=g)
    return dict(img=img, img_pos=img + 0.3 * torch.randn(B, 3, res, res, device=dev, generator=g),
                label=torch.randint(-1, N_CLASSES, (B, res, res), device=dev, generator=g))


def profile_kernels(fn, names):
    """CUDA time of the kernels whose name contains one of `names`, and of every kernel, in one call of fn."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    per, total = {}, 0.0
    for e in prof.key_averages():
        t = e.device_time_total / 1e3  # ms
        total += t
        for n in names:
            if n in e.key:
                per[n] = round(per.get(n, 0.0) + t, 4)
    part = sum(per.values())
    return dict(kernels_ms=per, selected_ms=round(part, 4), all_kernels_ms=round(total, 3),
                share=round(part / total, 5) if total else None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    result = dict(card=card(), frame=[H, W], n_classes=N_CLASSES, train=[], train_kernels=[], cases=[], kernels=[])
    for arch, res, B in TRAIN_CASES:
        batch = train_batch(B, res, dev)
        for baseline in (False, True):
            model = train_model(arch, baseline, dev)
            step = lambda: model.training_step(batch, 0)
            times = [window_ms(step, **TRAIN_WINDOW)[0] for _ in range(ROUNDS)]
            ms = statistics.median(times)
            result["train"].append(dict(arch=arch, res=res, B=B, baseline=baseline, code_channels=model.net.dim,
                                        ms=round(ms, 3), images_per_s=round(B * 1e3 / ms, 1),
                                        rounds_ms=[round(t, 3) for t in times]))
            if baseline:
                result["train_kernels"].append(dict(arch=arch, res=res, B=B,
                                                    **profile_kernels(step, WIDE_TRAIN_KERNELS)))
            del model
            torch.cuda.empty_cache()
    for name, over in MODELS.items():
        model = make_model(over, dev)
        for B in (1, 4):
            batch = make_batch(B, dev)
            for run_crf in (False, True):
                times = [window_ms(lambda: model.eval_step(batch, run_crf=run_crf), **WINDOW)[0] for _ in range(ROUNDS)]
                ms = statistics.median(times)
                result["cases"].append(dict(model=name, code_channels=model.net.dim, B=B, run_crf=run_crf,
                                            ms=round(ms, 3), frames_per_s=round(B * 1e3 / ms, 2),
                                            rounds_ms=[round(t, 3) for t in times]))
            del batch
            torch.cuda.empty_cache()
        batch = make_batch(4, dev)
        result["kernels"].append(dict(model=name, B=4, run_crf=False,
                                      **profile_kernels(lambda: model.eval_step(batch), ("eval_prep", "eval_probe"))))
        del model
        torch.cuda.empty_cache()
    result["card_after"] = card()
    emit(result, a.out)


if __name__ == "__main__":
    main()
