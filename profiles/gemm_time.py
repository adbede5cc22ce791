"""Kernel time and roofline of every GEMM the training step launches, at the c1 / c2 / c3 shapes.

    python profiles/gemm_time.py [--out FILE] [--configs c1,c2,c3] [--root DIR]

Prints one JSON line.  Times are CUDA-event times over windows of at least 0.3 s after warm-up, of the same
`ops.gemm` calls the step makes (L2 not flushed; every activation operand is larger than the 50 MB L2 except the
head's weights):
  * per ViT block: qkv (bf16 out), proj (fp32 x +=), fc1 + GELU (bf16 out), fc2 (fp32 x +=), at M = images x (hw + 1);
  * patch embed (im2col GEMM, row remap + positional embedding), M = images x hw;
  * head forward (cluster1, cluster2 a / b with code +=), dgrad dH and the split-K wgrads, M = images x hw, D = 70.
TFLOP/s are algorithmic (2 M N K); bytes are the operands read once, the output written once, and the fp32 residual
read once where there is one.  The floor is the larger of FLOPs / 989 TFLOP/s (dense bf16) and bytes / 3.35 TB/s
(H100 SXM data sheet, 700 W); the card's name, power limit and max SM clock are read in the same run.
--root imports stego_b200 from another checkout (e.g. the parent commit, built) to compare kernels on one card.
"""
import argparse
import os
import sys

import torch

from _measure import card, emit, window_ms

PEAK_TFLOPS, PEAK_TBS = 989.0, 3.35
CONFIGS = {"c1": (384, 28, 64), "c2": (768, 40, 64), "c3": (768, 56, 32)}  # E, patches per side, backbone images
D, P = 70, 72  # code width and its padded fp32 row
WINDOW = dict(warmup=3, min_window_s=0.3, min_iters=10)


def cases(cfg, dev):
    from stego_b200 import ops
    E, side, imgs = CONFIGS[cfg]
    hw = side * side
    Mt, Mh = imgs * (hw + 1), imgs * hw
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    g = torch.Generator(device=dev).manual_seed(0)
    rn = lambda *s: torch.randn(*s, device=dev, generator=g)
    bf = lambda *s: (rn(*s) * 0.5).bfloat16()
    y, ao, hid_t = bf(Mt, E), bf(Mt, E), bf(Mt, 4 * E)
    x = rn(Mt, E)
    qkv, hid = torch.empty(Mt, 3 * E, device=dev, dtype=torch.bfloat16), torch.empty(Mt, 4 * E, device=dev,
                                                                                     dtype=torch.bfloat16)
    w = {n: bf(r, c) / c ** 0.5 for n, (r, c) in dict(qkv=(3 * E, E), proj=(E, E), fc1=(4 * E, E), fc2=(E, 4 * E),
                                                      pe=(E, 192), wab=(E, E)).items()}
    b = {n: rn(r) for n, r in dict(qkv=3 * E, proj=E, fc1=4 * E, fc2=E, pe=E, c=P, wab=E).items()}
    rows, pos, xt = bf(Mh, 192), rn(hw + 1, E), torch.zeros(Mt, E, device=dev)
    x1, code, hh = bf(Mh, E), torch.zeros(Mh, P, device=dev), torch.empty(Mh, E, device=dev, dtype=torch.bfloat16)
    w1p, wbp = torch.zeros(128, E, device=dev, dtype=torch.bfloat16), torch.zeros(128, E, device=dev,
                                                                                   dtype=torch.bfloat16)
    w1p[:D], wbp[:D] = bf(D, E), bf(D, E)
    dyb = torch.zeros(Mh, 128, device=dev, dtype=torch.bfloat16)
    dyb[:, :D] = bf(Mh, D)
    dh, dw, dwa = torch.empty(Mh, E, device=dev), torch.zeros(D, E, device=dev), torch.zeros(E, E, device=dev)

    def lin(M, N, K, out_b, res_b=0, extra_b=0):  # flops, bytes
        return 2.0 * M * N * K, 2.0 * (M * K + N * K) + M * N * (out_b + res_b) + extra_b

    return [
        ("vit_qkv", lin(Mt, 3 * E, E, 2),
         lambda: ops.gemm(y, w["qkv"], qkv, M=Mt, N=3 * E, K=E, bias=b["qkv"])),
        ("vit_proj_residual", lin(Mt, E, E, 4, 4),
         lambda: ops.gemm(ao, w["proj"], x, M=Mt, N=E, K=E, bias=b["proj"], residual=x)),
        ("vit_fc1_gelu", lin(Mt, 4 * E, E, 2),
         lambda: ops.gemm(y, w["fc1"], hid, M=Mt, N=4 * E, K=E, bias=b["fc1"], act=ops.ACT_GELU)),
        ("vit_fc2_residual", lin(Mt, E, 4 * E, 4, 4),
         lambda: ops.gemm(hid_t, w["fc2"], x, M=Mt, N=E, K=4 * E, bias=b["fc2"], residual=x)),
        ("patch_embed", lin(Mh, E, 192, 4, 0, 4 * (hw + 1) * E),
         lambda: ops.gemm(rows, w["pe"], xt, M=Mh, N=E, K=192, bias=b["pe"], residual=pos, row_div=hw)),
        ("head_fwd_cluster1", lin(Mh, D, E, 4),
         lambda: ops.gemm(x1, w1p, code, M=Mh, N=D, K=E, bias=b["c"])),
        ("head_fwd_a_relu", lin(Mh, E, E, 2),
         lambda: ops.gemm(x1, w["wab"], hh, M=Mh, N=E, K=E, bias=b["wab"], act=ops.ACT_RELU)),
        ("head_fwd_b_residual", lin(Mh, D, E, 4, 4),
         lambda: ops.gemm(hh, wbp, code, M=Mh, N=D, K=E, bias=b["c"], residual=code)),
        ("head_dgrad", lin(Mh, E, 128, 4),
         lambda: ops.gemm(dyb, wbp, dh, M=Mh, N=E, K=128, b_mn=True)),
        ("head_wgrad_cluster", lin(D, E, Mh, 4),
         lambda: ops.gemm(dyb, x1, dw, M=D, N=E, K=Mh, a_mn=True, b_mn=True, splits=ops.wgrad_splits(Mh, D, E, sms),
                          atomic=True)),
        ("head_wgrad_a", lin(E, E, Mh, 4),
         lambda: ops.gemm(hh, x1, dwa, M=E, N=E, K=Mh, a_mn=True, b_mn=True, splits=ops.wgrad_splits(Mh, E, E, sms),
                          atomic=True)),
    ]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--configs", default="c1,c2,c3")
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.root))
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    res = dict(card=card(), configs={})
    for cfg in args.configs.split(","):
        rows, block_ms = [], 0.0
        for name, (flops, nbytes), fn in cases(cfg, dev):
            ms, n = window_ms(fn, **WINDOW)
            t_floor = max(flops / (PEAK_TFLOPS * 1e12), nbytes / (PEAK_TBS * 1e12)) * 1e6
            bound = "tensor" if flops / PEAK_TFLOPS > nbytes / PEAK_TBS else "hbm"
            rows.append(dict(gemm=name, ms=round(ms, 4), launches=n, tflops=round(flops / ms / 1e9, 1),
                             gbs=round(nbytes / ms / 1e6, 1), floor_us=round(t_floor, 1), bound=bound,
                             over_floor=round(ms * 1e3 / t_floor, 2)))
            if name.startswith("vit_"):
                block_ms += ms
        res["configs"][cfg] = dict(gemms=rows, vit_block_linears_ms=round(block_ms, 4))
        torch.cuda.empty_cache()
    emit(res, args.out)


if __name__ == "__main__":
    main()
