"""Cost of the CRF-refined evaluation step (eval_segmentation.py:124-141 with run_crf=True): the batched call
stego_b200.eval.fused_eval_crf against the stitched GPU sequence it replaces (fused_probe_log_probs -> crf.dense_crf
per frame and probe -> argmax -> UnsupervisedMetrics.update), alternated in one run, at

  * ref: the reference's eval shape, 16 frames at 320 x 320 from a ViT-B/8 code [16, 70, 40, 40], 27 classes;
  * c4:  one 1024 x 2048 frame from a [1, 70, 128, 256] code.

    python profiles/eval_crf_time.py [--out profiles/eval_crf_time_h100.json]

Per shape and path: ms per frame (CUDA events over at least 0.5 s of back-to-back calls after a warm-up, three
alternated rounds), this library's kernel launches per batch (_lib.launch_count), host synchronisations per batch
(torch's sync debug mode, counted on one call), and the bytes each path writes per frame into its per-pixel maps,
computed from the shapes (lattice values are data-dependent and not included).  Prints one JSON object.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import warnings

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from stego_b200 import _lib, crf  # noqa: E402
from stego_b200.eval import UnsupervisedMetrics, fused_eval_crf, fused_probe_log_probs  # noqa: E402
from stego_b200.modules import ClusterLookup  # noqa: E402
from _measure import call_ms, card, emit  # noqa: E402

SHAPES = {"ref": (16, 70, 40, 40, 320, 320), "c4": (1, 70, 128, 256, 1024, 2048)}
N_CLS = 27


def inputs(B, C, h, w, H, W, dev):
    g = torch.Generator().manual_seed(0)
    lin = torch.nn.Conv2d(C, N_CLS, (1, 1)).to(dev)
    clu = ClusterLookup(C, N_CLS).to(dev)
    with torch.no_grad():
        lin.weight.copy_(torch.randn(N_CLS, C, 1, 1, generator=g) * (4.0 / C ** 0.5))
        clu.clusters.copy_(torch.randn(N_CLS, C, generator=g))
    code = torch.randn(B, C, h, w, generator=g).to(dev)
    code2 = torch.randn(B, C, h, w, generator=g).to(dev)
    # piecewise-constant frames + noise, normalised like the loader
    img01 = F.interpolate(torch.rand(B, 3, 8, 8, generator=g), (H, W), mode="nearest") * 0.8 + \
        0.1 * torch.rand(B, 3, H, W, generator=g)
    mean = torch.tensor([0.485, 0.456, 0.406]).view(1, 3, 1, 1)
    std = torch.tensor([0.229, 0.224, 0.225]).view(1, 3, 1, 1)
    img = ((img01 - mean) / std).to(dev)
    label = torch.randint(-1, N_CLS, (B, H, W), generator=g).to(dev)
    return lin, clu, code, code2, img, label


def fused(lin, clu, code, code2, img, label, lm, cm):
    return fused_eval_crf(code, lin, clu, img, 2.0, code_flipped=code2, label=label, linear_confusion=lm.stats,
                          cluster_confusion=cm.stats)


def stitched(lin, clu, code, code2, img, label, lm, cm):
    H, W = img.shape[-2:]
    ll, cl = fused_probe_log_probs(code, lin, clu, (H, W), 2.0, code_flipped=code2)
    lp = torch.stack([crf.dense_crf(img[b], ll[b]) for b in range(img.shape[0])]).argmax(1)
    cp = torch.stack([crf.dense_crf(img[b], cl[b]) for b in range(img.shape[0])]).argmax(1)
    lm.update(lp, label)
    cm.update(cp, label)


def syncs(fn):
    fn()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("warn")
    try:
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            fn()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    return sum("synchroniz" in str(w.message) for w in caught)


def launches(fn):
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    fn()
    torch.cuda.synchronize()
    return _lib.launch_count() - n0


def bytes_written(H, W, path):
    """Per frame, into per-pixel maps: the stitched path writes both [27, H, W] log-prob maps, and per CRF the [N][32]
    unary and Q rows, ten Q updates and the [27, H, W] marginals; the batched call writes the [N][64] unary and Q rows,
    ten Q updates and the two uint8 label maps."""
    N = H * W
    if path == "stitched":
        return 2 * N_CLS * N * 4 + 2 * (2 * N * 32 * 4 + 10 * N * 32 * 4 + N_CLS * N * 4)
    return 2 * N * 64 * 4 + 10 * N * 64 * 4 + 2 * N


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    res = {"card": card(), "shapes": {}}
    for name, (B, C, h, w, H, W) in SHAPES.items():
        lin, clu, code, code2, img, label = inputs(B, C, h, w, H, W, dev)
        lm = UnsupervisedMetrics("l/", N_CLS, 0, False, dev)
        cm = UnsupervisedMetrics("c/", N_CLS, 0, False, dev)
        runs = {"fused_eval_crf": lambda: fused(lin, clu, code, code2, img, label, lm, cm),
                "stitched": lambda: stitched(lin, clu, code, code2, img, label, lm, cm)}
        r = {"batch": B, "frame": [H, W], "code": [B, C, h, w], "ms_per_frame": {k: [] for k in runs}}
        for _ in range(args.rounds):
            for k, fn in runs.items():  # single calls timed back to back until they add up to 0.5 s
                fn()
                torch.cuda.synchronize()
                n, total = 0, 0.0
                while total < 500.0:
                    total += call_ms(fn)[0]
                    n += 1
                r["ms_per_frame"][k].append(round(total / n / B, 3))
        r["launches_per_batch"] = {k: launches(fn) for k, fn in runs.items()}
        r["host_syncs_per_batch"] = {k: syncs(fn) for k, fn in runs.items()}
        r["bytes_written_per_frame"] = {"fused_eval_crf": bytes_written(H, W, "fused"),
                                        "stitched": bytes_written(H, W, "stitched")}
        res["shapes"][name] = r
        print(name, json.dumps(r), file=sys.stderr, flush=True)
        del lin, clu, code, code2, img, label
        torch.cuda.empty_cache()
    emit(res, args.out, indent=1)


if __name__ == "__main__":
    main()
