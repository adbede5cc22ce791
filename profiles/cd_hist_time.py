"""Cost of the cd histograms (hist_freq steps) at the c1 shape (B = 32, 28 x 28 code, ViT-S features E = 384, D = 70,
5 negatives): the correlation-loss forward with the histogram epilogue minus the plain forward — the only launch a
histogram step changes, plus its 37 KB device -> host copy — against materialising cd through cd_out and binning it
with np.histogram on the host, what add_histogram(tag, cd) would cost.

    python profiles/cd_hist_time.py [--out profiles/cd_hist_time_h100.json]

CUDA events around REPS launches each, after a warm-up; the materialising path is timed once per shape with a host
clock around a device synchronise (it ends on the host).  Prints one JSON object.
"""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from stego_b200 import corr, hist  # noqa: E402
from stego_b200.config import make_cfg  # noqa: E402
from _measure import card, emit, host_ms, window_ms  # noqa: E402

B, H, E, D = 32, 28, 384, 70
REPS = 20
WINDOW = dict(warmup=3, min_window_s=0.0, min_iters=REPS, max_iters=REPS)


def _inputs(fs, dev):
    spec = corr.make_spec(make_cfg(feature_samples=fs))
    g = torch.Generator().manual_seed(0)
    code = torch.randn(B, D, H, H, generator=g).to(dev)
    feats = torch.randn(B, E, H, H, generator=g).to(dev)
    c1 = (torch.rand(B, fs, fs, 2, generator=g) * 2 - 1).to(dev)
    c2 = (torch.rand(B, fs, fs, 2, generator=g) * 2 - 1).to(dev)
    perms = torch.stack([torch.randperm(B, generator=g) for _ in range(spec.n_neg)]).to(dev)
    ft = corr.build_tiles(feats, feats.roll(1, 0), c1, c2, perms, spec, E, raw_perms=True)
    ct = corr.build_tiles(code, code.roll(1, 0), c1, c2, perms, spec, corr.CODE_PAD, raw_perms=True)
    return spec, ft, ct


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--materialise-max-fs", type=int, default=28)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    gpu = card()
    rows = []
    for fs in (11, 28, 56):
        spec, ft, ct = _inputs(fs, dev)
        partials, row_means = spec.scratch(B, dev)
        stats = torch.empty(spec.ncalls, 4, device=dev)
        h = hist.CdHistogram(spec, B, dev)
        plain = window_ms(lambda: spec.forward(ft, ct, B, E, D, partials, row_means, stats), **WINDOW)[0] * 1e3
        with_h = window_ms(lambda: (spec.forward(ft, ct, B, E, D, partials, row_means, stats, hist=h), h.stage()),
                           **WINDOW)[0] * 1e3
        row = dict(fs=fs, S=fs * fs, forward_us=round(plain, 1), forward_with_histograms_us=round(with_h, 1),
                   histogram_cost_us=round(with_h - plain, 1))
        S = fs * fs
        cd_bytes = spec.ncalls * B * S * S * 4
        row["cd_bytes"] = cd_bytes
        if fs <= args.materialise_max_fs:
            cd = torch.empty(spec.ncalls, B, S, S, device=dev)
            fdc = torch.empty_like(cd)

            def materialise():
                spec.forward(ft, ct, B, E, D, partials, row_means, stats, cd, fdc)
                host = cd.cpu().numpy()
                for vals in (host[0], host[1], host[2:]):
                    np.histogram(vals.astype(np.float64), bins=hist.default_bins())

            spec.forward(ft, ct, B, E, D, partials, row_means, stats, cd, fdc)
            row["materialise_and_np_histogram_us"] = round(host_ms(materialise, 1) * 1e3, 1)
            del cd, fdc
        else:
            row["materialise_and_np_histogram_us"] = "not measured (cd would take %.1f GB)" % (cd_bytes / 1e9)
        rows.append(row)
        torch.cuda.empty_cache()
    emit(dict(card=gpu, shape=dict(B=B, code=H, E=E, D=D, neg_samples=5), reps=REPS, rows=rows), args.out, indent=1)


if __name__ == "__main__":
    main()
