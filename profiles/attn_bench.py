"""Correctness + timing of the fused attention kernel at the bench shapes (needs an H100).
    python profiles/attn_bench.py [--check-only]
Prints one JSON object: rel-L2 error vs fp32 torch for edge shapes (`check`, `check_ok`) and µs / TFLOP/s
(algorithmic flops 4*N^2*64 per head-image) for c1 (64 x 6 x 785), c2 (64 x 12 x 1601), c3 (32 x 12 x 3137), the mean
of 10 launches timed one by one with the L2 flushed between them.  Exits 1 if a check fails (then nothing is timed)."""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from stego_b200 import _lib, ops  # noqa: E402
from _measure import call_ms, card, emit  # noqa: E402

CHECKS = [(1, 128, 1, 1.5), (2, 785, 6, 1.5), (1, 1601, 12, 1.5), (3, 50, 6, 1.5), (1, 257, 2, 1.5), (1, 3137, 2, 1.0),
          (2, 65, 6, 3.0), (1, 129, 1, 1.0), (1, 256, 3, 1.0), (2, 400, 2, 4.0), (1, 17, 1, 1.0)]


def ref(qkv, B, N, heads):
    E = heads * 64
    q, k, v = qkv.float().view(B, N, 3, heads, 64).permute(2, 0, 3, 1, 4)
    attn = ((q @ k.transpose(-2, -1)) * 0.125).softmax(-1)
    return (attn @ v).transpose(1, 2).reshape(B * N, E)


def rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--check-only", action="store_true", help="run the correctness checks only")
    args = ap.parse_args()
    if os.environ.get("STEGO_PROFILE_LIB"):  # a variant build under profiles/_variants (experiments only)
        _lib.LIB_PATH = os.path.abspath(os.environ["STEGO_PROFILE_LIB"])
    dev = torch.device("cuda:0")
    res = dict(card=card(), check=[])
    torch.manual_seed(3)
    ok = True
    for B, N, heads, scale in CHECKS:
        E = heads * 64
        qkv = (torch.randn(B * N, 3 * E, device=dev) * scale).bfloat16()
        out = torch.full((B * N, E), float("nan"), device=dev, dtype=torch.bfloat16)
        ops.attention(qkv, out, B, N, E, heads)
        torch.cuda.synchronize()
        e = rel(out, ref(qkv, B, N, heads))
        fin = bool(torch.isfinite(out.float()).all())
        res["check"].append(dict(B=B, N=N, heads=heads, scale=scale, rel_l2=e, finite=fin))
        ok &= fin and e < 1e-2
    res["check_ok"] = ok
    if ok and not args.check_only:
        res["time"] = []
        flush = torch.zeros(64 * 1024 * 1024, device=dev)
        for name, B, N, heads in [("c1", 64, 785, 6), ("c2", 64, 1601, 12), ("c3", 32, 3137, 12)]:
            E = heads * 64
            qkv = torch.randn(B * N, 3 * E, device=dev).bfloat16()
            out = torch.empty(B * N, E, device=dev, dtype=torch.bfloat16)
            for _ in range(3):
                ops.attention(qkv, out, B, N, E, heads)
            torch.cuda.synchronize()
            tot = 0.0
            iters = 10
            for _ in range(iters):
                flush.add_(1.0)
                tot += call_ms(lambda: ops.attention(qkv, out, B, N, E, heads))[0]
            ms = tot / iters
            fl = 4.0 * B * heads * N * N * 64
            res["time"].append(dict(config=name, B=B, N=N, heads=heads, us=round(ms * 1e3, 1),
                                    tflops=round(fl / ms / 1e9)))
    emit(res)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
