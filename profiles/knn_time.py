"""Time of the fused kNN search (stego_knn_topk: normalise + hi/lo planes, then similarity + top-k in one kernel) at the
sizes it is built for, k = 30: Cityscapes train (2 975 descriptors), COCO-Stuff train (118 287) at the ViT-S and ViT-B
widths — beside the same search the way the reference does it on the same GPU (src/precompute_knns.py:83-92: fp32
`einsum("nf,mf->nm")` in 16 slabs + `torch.topk`, TF32 off, the slabs kept on the device).

    python profiles/knn_time.py [--out profiles/knn_time_h100.json] [--compare-lib other/libstego_b200.so --compare-label "what it is"]

CUDA events around every call, after a warm-up call of the same shape; the median of REPS calls is reported.
`tensor_flop` is what the kernel issues to the tensor cores, 3 passes x 2 n^2 E, and `tensor_tflops` is that over the
whole call's time (prep kernel and scan included): a whole-call rate, not the GEMM's share of peak.
--compare-lib times a second build of the library (e.g. of the parent commit) on the same inputs in the same run,
alternating call by call, and counts the rows whose indices differ.  That build must be compiled with
STEGO_NVCC_DEFS="-Xcompiler -fno-gnu-unique": otherwise the two libraries share the per-kernel record of the
shared-memory opt-in (a static in a template is one object per process) and the second one's launch fails.
Prints one JSON object.
"""
from __future__ import annotations

import argparse
import ctypes
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from stego_b200 import _lib  # noqa: E402
from _measure import call_ms, card, emit  # noqa: E402

SHAPES = [(2975, 384, 20), (118287, 384, 10), (118287, 768, 10)]  # n, E, REPS
K = 30


def _bind(path):
    lib = ctypes.CDLL(path)
    ret, args = _lib.header_prototypes()["stego_knn_topk"]
    lib.stego_knn_topk.restype = _lib._CTYPES[ret]
    lib.stego_knn_topk.argtypes = [_lib._CTYPES[a] for a in args]
    lib.stego_last_error.restype = ctypes.c_char_p
    return lib


def _descriptors(n, E):
    g = torch.Generator().manual_seed(n + E)
    base = torch.randn(max(8, n // 20), E, generator=g)
    return base[torch.randint(0, base.shape[0], (n,), generator=g)] + 0.35 * torch.randn(n, E, generator=g)


def _reference_search(x):
    normed = torch.nn.functional.normalize(x, dim=1)
    step = normed.shape[0] // 16
    return torch.cat([torch.topk(torch.einsum("nf,mf->nm", normed[i:i + step], normed), K)[1]
                      for i in range(0, normed.shape[0], step)], 0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--compare-lib", default=None)
    ap.add_argument("--compare-label", default=None, help="what the compared build is, kept in the JSON")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.set_float32_matmul_precision("highest")
    gpu = card()
    libs = {"this": _lib.load()}
    if args.compare_lib:
        libs["compared"] = _bind(args.compare_lib)
    rows = []
    for n, E, reps in SHAPES:
        x = _descriptors(n, E).to(dev)
        planes = torch.empty(2, n, E, dtype=torch.bfloat16, device=dev)
        idx = {name: torch.empty(n, K, dtype=torch.long, device=dev) for name in libs}

        def call(name):
            rc = libs[name].stego_knn_topk(_lib.ptr(x), n, E, K, _lib.ptr(planes), _lib.ptr(idx[name]), 0, _lib.stream())
            assert rc == 0, (name, rc, libs[name].stego_last_error())

        times = {name: [] for name in libs}
        for name in libs:
            call(name)  # warm-up
        for _ in range(reps):
            for name in libs:  # alternating
                times[name].append(call_ms(lambda: call(name))[0])
        flop = 3 * 2 * n * n * E
        row = dict(n=n, E=E, k=K, reps=reps, tensor_flop=flop)
        for name in libs:
            ms = statistics.median(times[name])
            row[name] = dict(median_ms=round(ms, 3), min_ms=round(min(times[name]), 3), max_ms=round(max(times[name]), 3),
                             tensor_tflops=round(flop / ms / 1e9, 1))
        if args.compare_lib:
            row["rows_with_different_indices"] = int((idx["this"] != idx["compared"]).any(1).sum())
        _reference_search(x[:max(16, n // 16)])  # warm-up: one slab's worth
        torch.cuda.synchronize()
        ref_ms, ref_idx = call_ms(lambda: _reference_search(x))
        row["torch_einsum_topk_fp32_ms"] = round(ref_ms, 1)
        row["rows_differing_from_torch_fp32"] = int((ref_idx != idx["this"]).any(1).sum())
        rows.append(row)
        del x, planes, idx, ref_idx
        torch.cuda.empty_cache()
    emit(dict(card=gpu, k=K, compared=args.compare_label, rows=rows), args.out, indent=1)


if __name__ == "__main__":
    main()
