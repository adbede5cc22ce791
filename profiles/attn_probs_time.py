"""Kernel time of the attention-matrix kernel (stego_attention_probs) at the c1 / c2 / c3 backbone shapes, against the
HBM bound and against torch eager on the same bf16 qkv.

    python profiles/attn_probs_time.py [--out FILE]

Prints one JSON line.  Times are CUDA-event times over repeated launches after a warm-up.  The kernel writes P, fp32
[B, heads, N, N], and reads q and k once from HBM (K tiles re-read by the CTAs of one image and head come from L2), so
its bytes are 4 B h N^2 + 4 B N E and its bound is bytes / 3.35 TB/s (H100 SXM data sheet, 700 W); its two passes of
Q K^T (2 x 2 B h N^2 64 FLOP) take under a quarter of that at the data-sheet bf16 rate.  The comparator is
`(q.float() @ k.float().mT * 0.125).softmax(-1)` (fp32 matmul, TF32 off), which writes S, reads and writes it for the
scale and again for the softmax: 20 B h N^2 bytes, five times the kernel's.
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from _measure import card, emit, window_ms  # noqa: E402

PEAK_TFLOPS, PEAK_TBS = 989.0, 3.35
# config: (arch, batch, resolution, tokens N = (res / 8)^2 + 1, heads)
CONFIGS = {"c1": ("vit_small", 32, 224, 785, 6), "c2": ("vit_base", 32, 320, 1601, 12),
           "c3": ("vit_base", 16, 448, 3137, 12)}
WINDOW = dict(warmup=1, min_window_s=0.5, min_iters=10, max_iters=500)


def case(name, dev):
    from stego_b200 import ops
    _, B, _, N, heads = CONFIGS[name]
    E = heads * 64
    g = torch.Generator(device=dev).manual_seed(0)
    qkv = (2.0 * torch.randn(B * N, 3 * E, device=dev, generator=g)).to(torch.bfloat16)  # logit std about 4
    P = torch.empty(B, heads, N, N, device=dev)
    t_k, n_k = window_ms(lambda: ops.attention_probs(qkv, P, B, N, E, heads), **WINDOW)
    x = qkv.view(B, N, 3, heads, 64).permute(2, 0, 3, 1, 4)
    q, k = x[0], x[1]

    def eager():
        return (q.float() @ k.float().mT * 0.125).softmax(-1)

    ref = eager()
    max_abs = (ref - P).abs().max().item()
    del ref
    torch.cuda.empty_cache()
    t_e, n_e = window_ms(eager, **WINDOW)
    torch.cuda.empty_cache()
    out_bytes = 4 * B * heads * N * N
    nbytes = out_bytes + 4 * B * N * E
    flops = 2 * 2 * B * heads * N * N * 64
    bound_ms = nbytes / (PEAK_TBS * 1e9)
    res = dict(config=name, B=B, N=N, heads=heads, elements=B * heads * N * N, gbytes=round(nbytes / 1e9, 3),
               gflop_two_passes=round(flops / 1e9, 1), hbm_bound_ms=round(bound_ms, 4),
               tensor_bound_ms=round(flops / (PEAK_TFLOPS * 1e9), 4),
               kernel_ms=round(t_k, 4), kernel_launches=n_k, kernel_write_tbs=round(out_bytes / t_k / 1e9, 3),
               kernel_fraction_of_hbm_bound=round(bound_ms / t_k, 3),
               eager_ms=round(t_e, 4), eager_launches=n_e, eager_gbytes=round((20 * B * heads * N * N + 4 * B * N * E) / 1e9, 3),
               speedup_vs_eager=round(t_e / t_k, 2), max_abs_diff_vs_eager=max_abs)
    del P, qkv
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda:0")
    res = dict(card=card(), peaks=dict(bf16_tflops=PEAK_TFLOPS, hbm_tbs=PEAK_TBS), cases=[])
    for name in CONFIGS:
        res["cases"].append(case(name, dev))
    res["gpu_info_after"] = card()
    emit(res, args.out)


if __name__ == "__main__":
    main()
