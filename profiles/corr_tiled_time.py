"""Kernel times and roofline of the correspondence loss for feature_samples 11 (single-tile kernels) and 16 / 28 / 40 / 56
(multi-tile kernels) at the c1 / c2 / c3 shapes, plus training_step images/s at c1 for fs 11 / 16 / 28.

    python profiles/corr_tiled_time.py [--out FILE] [--quick]

Prints one JSON line.  Kernel times are CUDA-event times over many launches after warm-up, of the C-ABI calls the
training step makes (sampling + norm of features and code, loss forward incl. its reduction, loss backward, norm +
grid_sample backward).  FLOPs: the algorithmic count of SURVEY.md 8(d), K * 2 S^2 E (fd) + K * 2 S^2 D (cd) forward and
2 * K * 2 S^2 D (dA, dB) backward per image, K = 2 + neg_samples calls; "executed" counts what the tensor cores run:
three bf16 hi/lo passes on 128-row tiles with the code padded to 128 channels, and the backward's recompute of fd / cd.
Bytes: the operand tiles read once plus the loss's own scratch / gradient tiles.  The bound named per row is the larger
of FLOPs / 989 TFLOP/s (dense bf16) and bytes / 3.35 TB/s (H100 SXM data sheet, 700 W).
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from _measure import call_ms, card, emit, window_ms  # noqa: E402

PEAK_TFLOPS, PEAK_TBS = 989.0, 3.35
CONFIGS = {"c1": ("vit_small", 384, 28, 32), "c2": ("vit_base", 768, 40, 32), "c3": ("vit_base", 768, 56, 16)}
D, NEG = 70, 5
WINDOW = dict(warmup=1, min_window_s=0.3, min_iters=5, max_iters=200)


def kernel_case(cfg_name, fs, dev):
    from stego_b200 import _lib, corr
    from stego_b200.config import make_cfg
    _, E, h, B = CONFIGS[cfg_name]
    spec = corr.make_spec(make_cfg(feature_samples=fs, neg_samples=NEG))
    lib = _lib.load()
    g = torch.Generator(device=dev).manual_seed(0)
    tok = torch.randn(2 * B, h, h, E, device=dev, generator=g).bfloat16()  # tokens-major, as the training step holds them
    feats, feats_pos = tok[:B].permute(0, 3, 1, 2), tok[B:].permute(0, 3, 1, 2)
    code_all = torch.randn(2 * B, h, h, 72, device=dev, generator=g)[..., :D].permute(0, 3, 1, 2)
    code, code_pos = code_all[:B], code_all[B:]
    c1 = torch.rand(B, fs, fs, 2, device=dev, generator=g) * 2 - 1
    c2 = torch.rand(B, fs, fs, 2, device=dev, generator=g) * 2 - 1
    perms = torch.stack([torch.randperm(B, device=dev, generator=g) for _ in range(NEG)])
    K, S, R = spec.ncalls, fs * fs, spec.rows
    ftiles = corr.build_tiles(feats, feats_pos, c1, c2, perms, spec, E, raw_perms=True)
    ctiles = corr.build_tiles(code, code_pos, c1, c2, perms, spec, corr.CODE_PAD, raw_perms=True)
    stats = torch.empty(K, 4, device=dev)
    gscale = torch.ones(K, device=dev)
    dtiles = torch.zeros(spec.nslots, B, R, corr.DT_LD, device=dev)
    dcode = torch.zeros(2 * B, h, h, 72, device=dev)[..., :D].permute(0, 3, 1, 2)
    partials, means = spec.scratch(B, dev)
    fwd = lambda: spec.forward(ftiles, ctiles, B, E, D, partials, means, stats)
    bwd = lambda: spec.backward(ftiles, ctiles, B, E, D, stats, means, gscale, None, None, dtiles)
    sn_fwd, sn_bwd = lib.stego_sample_norm_fwd, lib.stego_sample_norm_bwd
    st = _lib.stream()
    # partials are written and read once; the multi-tile finish also writes the row means
    scratch_bytes = (2 * partials.numel() + means.numel()) * 4 if spec.tiled else partials.numel() * 4

    def sample_fwd():
        sn_fwd(_lib.ptr(tok), _lib.ptr(tok[B:]), 1, h * h * E, 1, h * E, E, 0, 0, _lib.ptr(c1), _lib.ptr(c2),
               _lib.ptr(perms), _lib.ptr(ftiles), B, E, E, h, h, fs, spec.nslots, 1, st)
        sn_fwd(_lib.ptr(code_all), _lib.ptr(code_pos), 0, h * h * 72, 1, h * 72, 72, 0, 0, _lib.ptr(c1), _lib.ptr(c2),
               _lib.ptr(perms), _lib.ptr(ctiles), B, D, corr.CODE_PAD, h, h, fs, spec.nslots, 1, st)

    def sample_bwd():
        _lib.check(sn_bwd(_lib.ptr(code_all), _lib.ptr(code_pos), h * h * 72, 1, h * 72, 72, _lib.ptr(c1), _lib.ptr(c2),
                          _lib.ptr(perms), _lib.ptr(dtiles), _lib.ptr(dcode), _lib.ptr(dcode[B:]), B, D, h, h, fs,
                          spec.nslots, 1, st), "sample_bwd")

    fwd()
    t_fwd, n_fwd = window_ms(fwd, **WINDOW)
    t_bwd, n_bwd = window_ms(bwd, **WINDOW)
    t_sf, _ = window_ms(sample_fwd, **WINDOW)
    t_sb, _ = window_ms(sample_bwd, **WINDOW)
    nT = R // 128
    alg_fwd = B * K * 2 * S * S * (E + D)
    alg_bwd = B * K * 2 * S * S * 2 * D
    unit = 2 * 128 * 128 * 3  # one 128x128 block, three hi/lo passes, per unit of K
    exe_fwd = B * K * nT * nT * unit * (E + 128)
    if spec.tiled:  # two passes (dB, dA), each recomputes fd / cd and runs one GEMM
        exe_bwd = 2 * B * K * nT * nT * unit * (E + 128 + 128)
    else:           # one pass: recompute, then both GEMMs from the same G tile
        exe_bwd = B * K * unit * (E + 128 + 2 * 128)
    tile_bytes = ftiles.numel() * 2 + ctiles.numel() * 2
    bytes_fwd = tile_bytes + scratch_bytes
    bytes_bwd = tile_bytes + dtiles.numel() * 4 * 2 + means_bytes(spec, K, B)

    def roof(flops, exe, nbytes, ms):
        t_m = nbytes / (PEAK_TBS * 1e12)
        return dict(ms=round(ms, 4), tflops=round(flops / ms / 1e9, 2), gbs=round(nbytes / ms / 1e6, 1),
                    pct_bf16_peak=round(100 * flops / ms / 1e9 / PEAK_TFLOPS, 2),
                    pct_hbm_peak=round(100 * nbytes / ms / 1e6 / (PEAK_TBS * 1e3), 2),
                    # the roofline of the algorithm, and of the work the kernels execute (hi/lo passes, padding, recompute)
                    bound="tensor" if flops / (PEAK_TFLOPS * 1e12) >= t_m else "hbm",
                    executed_tflops=round(exe / ms / 1e9, 2),
                    executed_pct_bf16_peak=round(100 * exe / ms / 1e9 / PEAK_TFLOPS, 2),
                    executed_bound="tensor" if exe / (PEAK_TFLOPS * 1e12) >= t_m else "hbm")

    out = dict(config=cfg_name, fs=fs, S=S, B=B, E=E, impl="multi-tile" if spec.tiled else "single-tile",
               alg_gflop_fwd=round(alg_fwd / 1e9, 3), alg_gflop_bwd=round(alg_bwd / 1e9, 3),
               executed_gflop_fwd=round(exe_fwd / 1e9, 3), executed_gflop_bwd=round(exe_bwd / 1e9, 3),
               mbytes_fwd=round(bytes_fwd / 1e6, 2), mbytes_bwd=round(bytes_bwd / 1e6, 2),
               fwd=roof(alg_fwd, exe_fwd, bytes_fwd, t_fwd), bwd=roof(alg_bwd, exe_bwd, bytes_bwd, t_bwd),
               sample_norm_fwd_ms=round(t_sf, 4), sample_norm_bwd_ms=round(t_sb, 4), launches=dict(fwd=n_fwd, bwd=n_bwd))
    del ftiles, ctiles, dtiles, partials
    torch.cuda.empty_cache()
    return out


def means_bytes(spec, K, B):
    return K * B * spec.rows * 4 if spec.tiled else 0


def train_step_rate(fs, dev, steps, warmup):
    from stego_b200.config import make_cfg
    from stego_b200.segmenter import LitUnsupervisedSegmenter
    arch, _, h, B = CONFIGS["c1"]
    res = h * 8
    cfg = make_cfg(model_type=arch, res=res, batch_size=B, random_backbone_init=True, feature_samples=fs)
    torch.manual_seed(0)
    model = LitUnsupervisedSegmenter(27, cfg).to(dev)
    model.train()
    model.configure_optimizers()
    g = torch.Generator().manual_seed(1000)
    batch = dict(img=torch.randn(B, 3, res, res, generator=g).to(dev),
                 img_pos=torch.randn(B, 3, res, res, generator=g).to(dev),
                 label=torch.randint(-1, 27, (B, res, res), generator=g).to(dev))
    for i in range(warmup):
        model.training_step(batch, i)
    model.flush()
    torch.cuda.synchronize()

    def timed_steps():
        for i in range(steps):
            loss = model.training_step(batch, warmup + i)
        model.flush()
        return loss

    ms, loss = call_ms(timed_steps)
    ms /= steps
    fused = model._fused is not None and model._fused.ws is not None and model._fused.ws.graph is not None
    out = dict(config="c1", fs=fs, batch=B, steps=steps, ms_per_step=round(ms, 3), images_per_s=round(B * 1e3 / ms, 1),
               fused_graph_path=bool(fused), loss=float(loss))
    del model
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    ap.add_argument("--quick", action="store_true", help="c1 only, fs 11 / 16 (a smoke run)")
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=8)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    from stego_b200 import _lib
    _lib.load()
    res = dict(card=card(), peaks=dict(bf16_tflops=PEAK_TFLOPS, hbm_tbs=PEAK_TBS), kernels=[], train_step=[])
    cfgs = ["c1"] if args.quick else ["c1", "c2", "c3"]
    fss = [11, 16] if args.quick else [11, 16, 28, 40, 56]
    for c in cfgs:
        for fs in fss:
            res["kernels"].append(kernel_case(c, fs, dev))
    for fs in ([11, 16] if args.quick else [11, 16, 28]):
        res["train_step"].append(train_step_rate(fs, dev, args.steps, args.warmup))
    res["gpu_info_after"] = card()
    emit(res, args.out)


if __name__ == "__main__":
    main()
