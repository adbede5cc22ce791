"""Cost of LitUnsupervisedSegmenter.eval_step, the evaluation loop body of eval_segmentation.py:122-141, against

  * stitched: the package calls a caller made before it — two eager eval-mode net() calls (img, then a torch-flipped
    img.flip(3)), then fused_probe_log_probs (or fused_eval_crf with run_crf) with code / code_flipped and both
    `final/` confusion matrices;
  * eager: the reference loop in PyTorch eager (fp32) on the same card (oracle/eval_step_oracle.py: two ViT + head
    passes, F.interpolate, the linear probe conv and log_softmax, ClusterLookup, argmax, UnsupervisedMetrics.update's
    bincount).  With run_crf this package's crf.batched_crf stands in for the reference's pydensecrf pool.

at the eval_config shape (ViT-B/8, 320 x 320, 16 frames) and at ViT-S/8, 224 x 224, 16 frames, 27 classes, labels at
the frames' size, each with run_crf False and True.

    python profiles/eval_step_time.py [--out profiles/eval_step_time_h100.json]

Per case and path: ms per batch (CUDA events over at least 0.5 s of back-to-back calls after a warm-up; the three paths
alternate, three rounds, the median kept) and frames per second.  Prints one JSON object with the card.
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

CASES = (("vit_base", 320, 16), ("vit_small", 224, 16))
N_CLASSES, ROUNDS = 27, 3
WINDOW = dict(warmup=2, min_window_s=0.5, min_iters=3, max_iters=200)


def paths(arch, res, B, run_crf, dev):
    import eval_step_oracle as EO
    import stego_oracle as O
    from stego_b200 import crf
    from stego_b200.config import make_cfg
    from stego_b200.eval import fused_eval_crf, fused_probe_log_probs
    from stego_b200.segmenter import LitUnsupervisedSegmenter
    torch.manual_seed(0)
    model = LitUnsupervisedSegmenter(N_CLASSES, make_cfg(model_type=arch, random_backbone_init=True)).to(dev)
    sd = O.perturb_vit_state(O.vit_random_state(arch, 8, seed=3))
    model.net.model.load_state_dict(sd)
    model.train()
    g = torch.Generator(device=dev).manual_seed(0)
    img = torch.randn(B, 3, res, res, device=dev, generator=g)
    label = torch.randint(-1, N_CLASSES, (B, res, res), device=dev, generator=g)
    batch = dict(img=img, label=label)
    lp, cp = model.linear_probe, model.cluster_probe
    stats = dict(linear_confusion=model.test_linear_metrics.stats, cluster_confusion=model.test_cluster_metrics.stats)

    def ours():
        return model.eval_step(batch, run_crf=run_crf)

    def stitched():
        model.flush()
        with model._net_in_eval_mode(), torch.no_grad():
            _, code1 = model.net(img)
            _, code2 = model.net(img.flip(dims=[3]))
            if run_crf:
                return fused_eval_crf(code1, lp, cp, img, 2.0, code_flipped=code2, label=label, **stats)
            return fused_probe_log_probs(code1, lp, cp, label.shape[-2:], 2.0, want_log_probs=False, want_argmax=True,
                                         code_flipped=code2, label=label, **stats)

    sdd = {k: v.to(dev) for k, v in sd.items()}
    head = {k[len("net."):]: v.detach() for k, v in model.named_parameters() if k.startswith("net.cluster")}
    lw, lb, cl = lp.weight.detach(), lp.bias.detach(), cp.clusters.detach()
    lin_stats, clu_stats = torch.zeros_like(stats["linear_confusion"]), torch.zeros_like(stats["cluster_confusion"])

    def eager():
        with torch.no_grad():
            r = EO.eval_loop(lambda im: EO.net_code(sdd, head, im, arch), lw, lb, cl, img, label, N_CLASSES)
            if not run_crf:
                lin_stats.add_(r["linear_stats"])
                clu_stats.add_(r["cluster_stats"])
                return r
            la = crf.batched_crf(None, img, r["linear_probs"]).argmax(1)
            ca = crf.batched_crf(None, img, r["cluster_probs"]).argmax(1)
            lin_stats.add_(EO.confusion(la, label, N_CLASSES, N_CLASSES))
            clu_stats.add_(EO.confusion(ca, label, N_CLASSES, cl.shape[0]))
            return la, ca

    return dict(eval_step=ours, stitched=stitched, eager=eager)


def case(arch, res, B, run_crf, dev):
    fns = paths(arch, res, B, run_crf, dev)
    times = {k: [] for k in fns}
    for _ in range(ROUNDS):
        for k, fn in fns.items():
            times[k].append(window_ms(fn, **WINDOW)[0])
    ms = {k: statistics.median(v) for k, v in times.items()}
    out = dict(arch=arch, res=res, B=B, n_classes=N_CLASSES, run_crf=run_crf)
    for k, t in ms.items():
        out[f"{k}_ms"] = round(t, 3)
        out[f"{k}_frames_per_s"] = round(B * 1e3 / t, 1)
        out[f"{k}_rounds_ms"] = [round(x, 3) for x in times[k]]
    out["speedup_vs_stitched"] = round(ms["stitched"] / ms["eval_step"], 3)
    out["speedup_vs_eager"] = round(ms["eager"] / ms["eval_step"], 2)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    result = dict(card=card(), cases=[])
    for arch, res, B in CASES:
        for run_crf in (False, True):
            result["cases"].append(case(arch, res, B, run_crf, dev))
            torch.cuda.empty_cache()
    result["card_after"] = card()
    emit(result, a.out)


if __name__ == "__main__":
    main()
