"""Cost of one CorrespondencePR.update (both methods, one batch) against the reference's lines for the same batch.

    python profiles/corr_pr_time.py [--out profiles/corr_pr_time_h100.json]

Shapes: c1 (B = 32, 28 x 28 ViT-S features E = 384, code D = 70, 224 x 224 labels) at feature_samples 11 / 28 / 56 and
c2 (B = 32, 40 x 40 ViT-B features E = 768, 320 x 320 labels) at 11 / 40.  Ours: CUDA events around REPS updates
after a warm-up (label ids, two samplers, one corr_kernel<CP_PR> launch; the counts stay on the device).  Reference
(plot_pr_curves.py:108-121, 152-167): grid_sample + F.normalize + the tensor_correlation einsum for both methods and
one_hot + grid_sample + einsum for ld, on the same GPU, then the copy of fd and ld to the host (what the epoch-end
torch.cat works on), timed with a host clock around that copy; sklearn's average_precision_score of one method on the
host is timed separately.  Each reference part runs only where its tensors fit (REF_MAX_PAIRS, SKLEARN_MAX_PAIRS).
The two paths alternate, ROUNDS times.  Prints one JSON object.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from stego_b200 import _lib  # noqa: E402
from stego_b200.correspondence import CorrespondencePR  # noqa: E402
from _measure import card, emit, host_ms, window_ms  # noqa: E402

CASES = [("c1", 32, 28, 384, 11), ("c1", 32, 28, 384, 28), ("c1", 32, 28, 384, 56),
         ("c2", 32, 40, 768, 11), ("c2", 32, 40, 768, 40)]
D, N_CLASSES = 70, 27
REPS, ROUNDS = 20, 3
WINDOW = dict(warmup=0, min_window_s=0.0, min_iters=REPS, max_iters=REPS)
REF_MAX_PAIRS = 1_000_000_000   # 3 x pairs: fd (two methods) and ld, fp32 (up to 4 GB), on the GPU and copied to the host
SKLEARN_MAX_PAIRS = 20_000_000


def _inputs(B, h, E, fs, dev):
    g = torch.Generator().manual_seed(0)
    feats = torch.randn(B, E, h, h, generator=g).to(dev)
    code = torch.randn(B, D, h, h, generator=g).to(dev)
    small = torch.randint(-1, N_CLASSES, (B, 7, 7), generator=g)
    idx = torch.arange(8 * h) * 7 // (8 * h)
    label = small[:, idx][:, :, idx].contiguous().to(dev)
    c1 = (torch.rand(B, fs, fs, 2, generator=g) * 2 - 1).to(dev)
    c2 = (torch.rand(B, fs, fs, 2, generator=g) * 2 - 1).to(dev)
    return feats, code, label, c1, c2


def _sample(t, coords):
    return F.grid_sample(t, coords.permute(0, 2, 1, 3), padding_mode="border", align_corners=True)


def _corr(a, b):
    return torch.einsum("nchw,ncij->nhwij", a, b)


def _reference(feats, code, label, c1, c2):
    """get_net_fd for both methods and ld, then the host copies; returns (fd_code, fd_feats, ld) on the host."""
    out = []
    for f in (code, feats):
        out.append(_corr(F.normalize(_sample(f, c1), dim=1, eps=1e-10), F.normalize(_sample(f, c2), dim=1, eps=1e-10)))
    oh = F.one_hot(label + 1, N_CLASSES + 1).to(torch.float).permute(0, 3, 1, 2)
    out.append(_corr(_sample(oh, c1), _sample(oh, c2)))
    return [t.cpu() for t in out]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    res = {"card": card(), "reps": REPS, "rounds": ROUNDS, "cases": []}
    for shape, B, h, E, fs in CASES:
        x = _inputs(B, h, E, fs, dev)
        pairs = B * fs ** 4
        met = CorrespondencePR(N_CLASSES, dev)
        met.update(*x)
        n0 = _lib.launch_count()
        met.update(*x)
        launches = _lib.launch_count() - n0
        torch.cuda.synchronize()
        do_ref = 3 * pairs <= REF_MAX_PAIRS
        if do_ref:
            _reference(*x)
        ours, ref = [], []
        for _ in range(ROUNDS):
            ours.append(window_ms(lambda: met.update(*x), **WINDOW)[0])
            if do_ref:
                ref.append(host_ms(lambda: _reference(*x), 1))
        row = dict(shape=shape, B=B, feature_samples=fs, E=E, D=D, pairs_per_method=pairs,
                   ours_ms=float(np.median(ours)), ours_ms_all=ours, ours_launches=launches,
                   ours_pairs_per_s=2 * pairs / (float(np.median(ours)) * 1e-3))
        if do_ref:
            row.update(reference_gpu_and_copy_ms=float(np.median(ref)), reference_ms_all=ref)
            if pairs <= SKLEARN_MAX_PAIRS:
                from sklearn.metrics import average_precision_score
                fd_code, _, ld = _reference(*x)

                def sklearn_ap():
                    p = fd_code.reshape(-1)
                    p = (p - p.min()) / (p - p.min()).max()
                    average_precision_score(ld.to(torch.int64).reshape(-1).numpy(), p.numpy())

                row["reference_sklearn_ap_ms_per_method"] = host_ms(sklearn_ap, 1)
        else:
            row["reference"] = f"not run: fd and ld would be {3 * pairs * 4 / 1e9:.1f} GB"
        res["cases"].append(row)
        print(json.dumps(row), file=sys.stderr)
        del x, met
        torch.cuda.empty_cache()
    res["card_after"] = card()
    emit(res, args.out, indent=1)


if __name__ == "__main__":
    main()
