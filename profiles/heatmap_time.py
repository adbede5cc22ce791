"""Cost of the dense correspondence heatmaps (correspondence_heatmaps / get_heatmaps) against the reference's lines.

    python profiles/heatmap_time.py [--out profiles/heatmap_time_h100.json]

Shapes: the reference's figure (B = 1, P = 3, ViT-S E = 384, 64 x 64 map -> 512 x 512), its movie (P = 280, same
maps) and a batch (B = 16, P = 16, E = 768, 40 x 40 -> 320 x 320), each with a KNN target map of the same size.
Ours: CUDA events around REPS calls of correspondence_heatmaps after a warm-up, and around REPS launches of each of its
five steps alone (target prep, query sampler, batched GEMM, finish, upsample) on preallocated buffers; the upsample's
achieved write rate is its output bytes (B P H W x 4) over its time, beside the least time those bytes take at the H100
SXM data sheet's 3.35 TB/s.  Reference: its lines (plot_dino_correspondence.py:43-56: grid_sample, F.normalize, the
einsum, mean, clamp, F.interpolate) in eager fp32 on the same GPU, timed the same way.  The two alternate, ROUNDS
times.  For the figure and the movie the drop-in (get_heatmaps on precomputed features: both maps, then the copies to
the host) is timed with a host clock against the reference's lines with their .cpu(), and the copies alone.  The card's
name, power limit and clock are read in the same run.  Prints one JSON object.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import heatmap_oracle as HO  # noqa: E402
from stego_b200 import _lib, ops  # noqa: E402
from stego_b200.correspondence import correspondence_heatmaps, get_heatmaps  # noqa: E402
from _measure import card, emit, host_ms, window_ms  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
REPS, ROUNDS = 20, 3
WINDOW = dict(warmup=0, min_window_s=0.0, min_iters=REPS, max_iters=REPS)
FIGURE = [[-.1, 0.0], [.5, .8], [-.7, -.7]]
CASES = [("figure", 1, 3, 384, 64, 512), ("movie", 1, 280, 384, 64, 512), ("batch", 16, 16, 768, 40, 320)]


def _points(name, B, P, dev):
    if name == "figure":
        return torch.tensor(FIGURE, device=dev).reshape(1, 3, 1, 2)
    if name == "movie":
        key, pts = [[-.7, -.7], [-.1, 0.0], [.5, .8]], []
        for i in range(3):
            pts.extend([key[i]] * 60)
            if i < 2:
                pts.extend(np.stack([np.linspace(key[i][0], key[i + 1][0], 50),
                                     np.linspace(key[i][1], key[i + 1][1], 50)], axis=1).tolist())
        return torch.tensor(pts, dtype=torch.float32, device=dev).reshape(1, len(pts), 1, 2)
    g = torch.Generator().manual_seed(1)
    return (torch.rand(B, P, 1, 2, generator=g) * 2 - 1).to(dev)


def _feats(B, E, h, seed, dev):
    """fp32 NCHW view of tokens-major storage, as DinoFeaturizer returns it."""
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, h * h, E, generator=g).to(dev).view(B, h, h, E).permute(0, 3, 1, 2)


def _steps(f, t, qp, H, W):
    """The five steps of correspondence_heatmaps as closures over preallocated buffers (fp32 target: nseg 3)."""
    lib = _lib.load()
    B, E, h, w = f.shape
    P, hw, ep = qp.shape[1], h * w, -(-E // 8) * 8
    dev = f.device
    t_ops = torch.empty(B, hw, 3 * ep, dtype=torch.bfloat16, device=dev)
    q_ops = torch.empty(B, P, 3 * ep, dtype=torch.bfloat16, device=dev)
    inv = torch.empty(B, hw, device=dev)
    corr = torch.empty(B, P, hw, device=dev)
    out = torch.empty(B, P, H, W, device=dev)
    pts = qp.contiguous()
    s = lambda x: [int(v) for v in x.stride()]  # noqa: E731
    return {
        "target_prep": lambda: lib.stego_heatmap_prep_target(_lib.ptr(t), 0, *s(t), B, E, h, w, ep, _lib.ptr(t_ops),
                                                             _lib.ptr(inv), _lib.stream()),
        "query_sample": lambda: lib.stego_heatmap_sample_queries(_lib.ptr(f), 0, *s(f), _lib.ptr(pts), B, P, E, h, w,
                                                                 ep, 3, _lib.ptr(q_ops), _lib.stream()),
        "gemm": lambda: ops.gemm_batched(q_ops, t_ops, corr),
        "finish": lambda: lib.stego_heatmap_finish(_lib.ptr(corr), _lib.ptr(inv), B, P, hw, _lib.stream()),
        "upsample": lambda: lib.stego_heatmap_upsample(_lib.ptr(corr), _lib.ptr(out), B * P, h, w, H, W,
                                                       _lib.stream()),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    res = {"card": card(), "reps": REPS, "rounds": ROUNDS, "hbm_bytes_per_s_datasheet": HBM_BYTES_PER_S, "cases": []}
    for name, B, P, E, h, res_px in CASES:
        f, fp = _feats(B, E, h, 1, dev), _feats(B, E, h, 2, dev)
        qp = _points(name, B, P, dev)
        size = (res_px, res_px)
        out_bytes = B * P * res_px * res_px * 4
        ours = lambda: correspondence_heatmaps(f, fp, qp, size)  # noqa: E731
        ref = lambda: HO.heatmaps(f, fp, qp, size, dtype=torch.float32)  # noqa: E731
        err = float((ours() - ref()).abs().max())
        steps = _steps(f, fp, qp, *size)
        for k, fn in steps.items():
            rc = fn()
            if isinstance(rc, int):
                _lib.check(rc, k)
        torch.cuda.synchronize()
        t_ours, t_ref, t_steps = [], [], {k: [] for k in steps}
        for _ in range(ROUNDS):
            t_ours.append(window_ms(ours, **WINDOW)[0])
            t_ref.append(window_ms(ref, **WINDOW)[0])
            for k, fn in steps.items():
                t_steps[k].append(window_ms(fn, **WINDOW)[0])
        med = {k: float(np.median(v)) for k, v in t_steps.items()}
        row = dict(case=name, B=B, P=P, E=E, map=[h, h], size=list(size), max_abs_diff_vs_reference_fp32=err,
                   ours_ms=float(np.median(t_ours)), ours_ms_all=t_ours, reference_ms=float(np.median(t_ref)),
                   reference_ms_all=t_ref, step_ms=med, step_ms_all=t_steps, output_bytes=out_bytes,
                   upsample_write_bound_ms=out_bytes / HBM_BYTES_PER_S * 1e3,
                   upsample_write_gb_per_s=out_bytes / (med["upsample"] * 1e-3) / 1e9)
        if B == 1:  # the drop-in: both maps and the copies to the host
            img = torch.zeros(1, 3, *size, device=dev)
            calls = [0]

            def net(x):  # get_heatmaps asks for the image's features, then the KNN image's
                calls[0] += 1
                return (f if calls[0] % 2 else fp), None

            def ref_maps():
                return [HO.heatmaps(f, t, qp, size, dtype=torch.float32)[0] for t in (f, fp)]

            get_heatmaps(net, img, img, qp)
            d_ours, d_ref, d_copy = [], [], []
            for _ in range(ROUNDS):
                d_ours.append(host_ms(lambda: get_heatmaps(net, img, img, qp), 1))
                d_ref.append(host_ms(lambda: [m.cpu() for m in ref_maps()], 1))
                maps = ref_maps()  # the copies alone
                d_copy.append(host_ms(lambda: [m.cpu() for m in maps], 1))
                del maps
            row.update(drop_in_ours_ms=float(np.median(d_ours)), drop_in_ours_ms_all=d_ours,
                       drop_in_reference_ms=float(np.median(d_ref)), drop_in_reference_ms_all=d_ref,
                       drop_in_reference_copy_ms=float(np.median(d_copy)))
        res["cases"].append(row)
        print(json.dumps(row), file=sys.stderr)
        del f, fp, steps
        torch.cuda.empty_cache()
    res["card_after"] = card()
    emit(res, args.out, indent=1)


if __name__ == "__main__":
    main()
