"""Fused correspondence loss: host orchestration of the corr_loss.cu kernels + autograd glue.

Reference semantics: src/modules.py:325-398 (ContrastiveCorrelationLoss.helper / forward).  The random
draws (coords, perms) are inputs here; `modules.ContrastiveCorrelationLoss.forward` makes them with the
same torch RNG calls, in the same order, as the reference.
"""
from __future__ import annotations

import ctypes
from typing import List, Optional, Sequence, Tuple

import torch

from . import _lib

CODE_PAD = 128   # code channels are zero-padded to two 64-wide k-blocks in the operand tiles
TILE_ROWS = 128  # feature_samples^2 <= 128
DT_LD = 72       # row stride of the gradient tiles
MAX_TILED_FS = 64  # the multi-tile kernels take feature_samples up to 64 (S = 4096 points per image)


def _i32(vals: Sequence[int]):
    return (ctypes.c_int * len(vals))(*[int(v) for v in vals])


def _f32(vals: Sequence[float]):
    return (ctypes.c_float * len(vals))(*[float(v) for v in vals])


def _same_layout(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """Return b in a's strides (copy only if needed): the kernels take one stride set per tensor pair."""
    if a.stride() == b.stride() and a.dtype == b.dtype:
        return b
    out = torch.empty_strided(a.size(), a.stride(), dtype=a.dtype, device=a.device)
    out.copy_(b)
    return out


def _zeros_strided_like(t: torch.Tensor) -> torch.Tensor:
    extent = 1 + sum((s - 1) * st for s, st in zip(t.size(), t.stride()))
    buf = torch.zeros(extent, dtype=torch.float32, device=t.device)
    return torch.as_strided(buf, t.size(), t.stride())


def _describe(spec, cfg, n_neg: Optional[int]) -> None:
    spec.fs = int(cfg.feature_samples)
    spec.n_neg = int(cfg.neg_samples if n_neg is None else n_neg)
    spec.pointwise = bool(cfg.pointwise)
    spec.zero_clamp = bool(cfg.zero_clamp)
    spec.stabilize = bool(cfg.stabalize)
    spec.nslots = 2 + spec.n_neg
    spec.ncalls = 2 + spec.n_neg
    # call 0: intra (A vs A), call 1: inter (A vs pos), calls 2..: negatives (A vs img[perm_i])
    spec.slot_of_call = [0, 1] + [2 + i for i in range(spec.n_neg)]
    spec.shifts = [float(cfg.pos_intra_shift), float(cfg.pos_inter_shift)] + [float(cfg.neg_inter_shift)] * spec.n_neg
    spec._soc, spec._shf = _i32(spec.slot_of_call), _f32(spec.shifts)  # host arrays the loss entry points read


def _loss_args(spec, ftiles, ctiles, B, E, D):
    """the leading arguments every corr-loss entry point takes"""
    return (_lib.ptr(ftiles), _lib.ptr(ctiles), B, spec.fs, E, D, spec.nslots, spec.ncalls, spec._soc, spec._shf,
            int(spec.pointwise), int(spec.zero_clamp), int(spec.stabilize))


class LossSpec:
    """Static description of one ContrastiveCorrelationLoss evaluation (which calls, which shifts) for the
    single-tile kernels: all S = feature_samples^2 <= 128 points of an image in one 128-row tile.  Each spec knows its
    entry points: `scratch` allocates what `forward` needs, `forward` / `backward` launch the loss kernels."""
    tiled = False
    rows = TILE_ROWS  # operand / gradient tile rows per (slot, image)

    def __init__(self, cfg, n_neg: Optional[int] = None):
        _describe(self, cfg, n_neg)
        if self.fs * self.fs > TILE_ROWS:
            raise RuntimeError(f"stego_b200: feature_samples={self.fs} exceeds the 128-row tile (max 11)")

    def scratch(self, B, device):
        """(partials, row_means) for `forward`; the single-tile kernels keep their row means in registers, so
        row_means is empty."""
        return (torch.empty(self.ncalls, B, 8, dtype=torch.float32, device=device),
                torch.empty(0, dtype=torch.float32, device=device))

    def forward(self, ftiles, ctiles, B, E, D, partials, row_means, stats, cd=None, fdc=None, elems=None):
        _lib.check(_lib.load().stego_corr_loss_fwd(
            *_loss_args(self, ftiles, ctiles, B, E, D), _lib.ptr(partials), _lib.ptr(stats), _lib.ptr(cd),
            _lib.ptr(fdc), _lib.ptr(elems), _lib.stream()), "stego_corr_loss_fwd")

    def backward(self, ftiles, ctiles, B, E, D, stats, row_means, gscale, gelem, gcd, dtiles):
        _lib.check(_lib.load().stego_corr_loss_bwd(
            *_loss_args(self, ftiles, ctiles, B, E, D), _lib.ptr(stats), _lib.ptr(gscale), _lib.ptr(gelem),
            _lib.ptr(gcd), _lib.ptr(dtiles), _lib.stream()), "stego_corr_loss_bwd")


class TiledLossSpec:
    """The same description for the multi-tile kernels: S points padded to whole 128-row tiles (`rows`), the fd / cd
    blocks computed per (row tile, column tile).  Any feature_samples up to MAX_TILED_FS."""
    tiled = True

    def __init__(self, cfg, n_neg: Optional[int] = None):
        _describe(self, cfg, n_neg)
        if not 1 <= self.fs <= MAX_TILED_FS:
            raise RuntimeError(f"stego_b200: feature_samples={self.fs} is outside the supported range "
                               f"1..{MAX_TILED_FS}")
        S = self.fs * self.fs
        self.rows = (S + TILE_ROWS - 1) // TILE_ROWS * TILE_ROWS
        self.n_tiles = self.rows // TILE_ROWS

    def scratch(self, B, device):
        """(per-row partials, row means) for `forward`; `backward` reads the row means."""
        return (torch.empty(self.ncalls, B, self.n_tiles, self.rows, 4, dtype=torch.float32, device=device),
                torch.empty(self.ncalls, B, self.rows, dtype=torch.float32, device=device))

    def forward(self, ftiles, ctiles, B, E, D, partials, row_means, stats, cd=None, fdc=None, elems=None):
        _lib.check(_lib.load().stego_corr_loss_tiled_fwd(
            *_loss_args(self, ftiles, ctiles, B, E, D), _lib.ptr(partials), _lib.ptr(row_means), _lib.ptr(stats),
            _lib.ptr(cd), _lib.ptr(fdc), _lib.ptr(elems), _lib.stream()), "stego_corr_loss_tiled_fwd")

    def backward(self, ftiles, ctiles, B, E, D, stats, row_means, gscale, gelem, gcd, dtiles):
        _lib.check(_lib.load().stego_corr_loss_tiled_bwd(
            *_loss_args(self, ftiles, ctiles, B, E, D), _lib.ptr(stats), _lib.ptr(row_means), _lib.ptr(gscale),
            _lib.ptr(gelem), _lib.ptr(gcd), _lib.ptr(dtiles), _lib.stream()), "stego_corr_loss_tiled_bwd")


def make_spec(cfg, n_neg: Optional[int] = None):
    """The loss implementation for cfg.feature_samples: the single-tile kernels up to 11 (S <= 128), the multi-tile
    kernels from 12 to MAX_TILED_FS; above that a RuntimeError."""
    fs = int(cfg.feature_samples)
    if fs * fs <= TILE_ROWS:
        return LossSpec(cfg, n_neg)
    return TiledLossSpec(cfg, n_neg)


def build_tiles(src: torch.Tensor, src_pos: torch.Tensor, coords1: torch.Tensor, coords2: torch.Tensor,
                perms: Optional[torch.Tensor], spec: LossSpec, c_pad: int,
                chan_scale: Optional[torch.Tensor] = None, chan_scale_pos: Optional[torch.Tensor] = None,
                raw_perms: bool = False) -> torch.Tensor:
    """sample + norm for every slot -> bf16 hi/lo tiles [2][nslots][B][spec.rows][c_pad]."""
    B, C, H, W = src.shape
    src_pos = _same_layout(src, src_pos)
    tiles = torch.empty(2, spec.nslots, B, spec.rows, c_pad, dtype=torch.bfloat16, device=src.device)
    sb, sc, sy, sx = src.stride()
    rc = _lib.load().stego_sample_norm_fwd(
        _lib.ptr(src), _lib.ptr(src_pos), int(src.dtype == torch.bfloat16), sb, sc, sy, sx,
        _lib.ptr(chan_scale), _lib.ptr(chan_scale_pos), _lib.ptr(coords1), _lib.ptr(coords2), _lib.ptr(perms),
        _lib.ptr(tiles), B, C, c_pad, H, W, spec.fs, spec.nslots, int(raw_perms), _lib.stream())
    _lib.check(rc, "stego_sample_norm_fwd")
    return tiles


def _prep_common(feats, feats_pos, code, code_pos, coords1, coords2, perms, spec: LossSpec):
    _lib.require_cuda(feats, feats_pos, code, code_pos, coords1, coords2)
    B, E, H, W = feats.shape
    D = code.shape[1]
    if feats.dtype not in (torch.float32, torch.bfloat16):
        raise RuntimeError("stego_b200: feats must be fp32 or bf16")
    if E % 64 != 0 or E > 768:
        raise RuntimeError(f"stego_b200: feature channels {E} unsupported (multiple of 64, <= 768)")
    if D > 96:
        raise RuntimeError(f"stego_b200: code dim {D} unsupported (<= 96)")
    if code.shape[2:] != feats.shape[2:] or code.shape[0] != B:
        raise RuntimeError("stego_b200: feats/code shape mismatch")
    coords1 = coords1.to(torch.float32).contiguous()
    coords2 = coords2.to(torch.float32).contiguous()
    if spec.n_neg > 0:
        perms_t = torch.stack([p.to(device=feats.device, dtype=torch.long) for p in perms]).contiguous() \
            if not torch.is_tensor(perms) else perms.to(device=feats.device, dtype=torch.long).contiguous()
        assert perms_t.shape == (spec.n_neg, B)
    else:
        perms_t = None
    return B, E, D, H, W, coords1, coords2, perms_t


class _CorrLossFn(torch.autograd.Function):
    """(code, code_pos) -> per-call mean losses [ncalls], cd [ncalls,B,S,S] or None, loss elems or None."""

    @staticmethod
    def forward(ctx, code, code_pos, feats, feats_pos, coords1, coords2, perms, spec: LossSpec, want_elems: bool,
                chan_scale, chan_scale_pos, raw_perms=False, pair=False):
        # pair=True: `code` is the [2B, D, h, w] output of ONE head pass over img ++ img_pos (code_pos is None); its
        # gradient is then produced in one buffer instead of two tensors that autograd has to re-assemble.
        if pair:
            half = code.shape[0] // 2
            code_all = code.detach()
            if code_all.dtype != torch.float32:
                code_all = code_all.float()
            code_f, code_pos_f = code_all[:half], code_all[half:]
            B, E, D, H, W, coords1, coords2, perms_t = _prep_common(feats, feats_pos, code_f, code_pos_f, coords1,
                                                                     coords2, perms, spec)
        else:
            B, E, D, H, W, coords1, coords2, perms_t = _prep_common(feats, feats_pos, code, code_pos, coords1, coords2,
                                                                     perms, spec)
            code_f = code.detach()
            if code_f.dtype != torch.float32:
                code_f = code_f.float()
            code_pos_f = _same_layout(code_f, code_pos.detach().to(torch.float32))
        ctx.pair = bool(pair)
        dev = code.device
        ftiles = build_tiles(feats.detach(), feats_pos.detach(), coords1, coords2, perms_t, spec, E, chan_scale,
                             chan_scale_pos, raw_perms)
        ctiles = build_tiles(code_f, code_pos_f, coords1, coords2, perms_t, spec, CODE_PAD, raw_perms=raw_perms)
        ctx.raw_perms = bool(raw_perms)
        S = spec.fs * spec.fs
        stats = torch.empty(spec.ncalls, 4, dtype=torch.float32, device=dev)
        cd = fdc = elems = None
        if want_elems:
            cd = torch.empty(spec.ncalls, B, S, S, dtype=torch.float32, device=dev)
            fdc = torch.empty_like(cd)
            elems = torch.empty_like(cd)
        partials, row_means = spec.scratch(B, dev)
        spec.forward(ftiles, ctiles, B, E, D, partials, row_means, stats, cd, fdc, elems)
        ctx.spec = spec
        ctx.dims = (B, E, D, H, W)
        ctx.code_dtype = (code.dtype, code_pos.dtype if code_pos is not None else code.dtype)
        ctx.save_for_backward(ftiles, ctiles, stats, code_f, code_pos_f, coords1, coords2,
                              perms_t if perms_t is not None else torch.empty(0, device=dev), row_means)
        losses = stats[:, 0].clone()
        cd_means = stats[:, 1].clone()
        ctx.mark_non_differentiable(cd_means)
        if want_elems:
            return losses, cd_means, cd, elems
        return losses, cd_means, None, None

    @staticmethod
    def backward(ctx, g_losses, _g_cd_means, g_cd, g_elems):
        spec: LossSpec = ctx.spec
        B, E, D, H, W = ctx.dims
        ftiles, ctiles, stats, code_f, code_pos_f, coords1, coords2, perms_t, row_means = ctx.saved_tensors
        perms_arg = perms_t if spec.n_neg > 0 else None
        dev = code_f.device
        gscale = (g_losses if g_losses is not None else torch.zeros(spec.ncalls, device=dev)).to(torch.float32).contiguous()
        gel = g_elems.to(torch.float32).contiguous() if g_elems is not None else None
        gcd = g_cd.to(torch.float32).contiguous() if g_cd is not None else None
        dtiles = torch.zeros(spec.nslots, B, spec.rows, DT_LD, dtype=torch.float32, device=dev)
        spec.backward(ftiles, ctiles, B, E, D, stats, row_means, gscale, gel, gcd, dtiles)
        if ctx.pair:
            # code_f / code_pos_f are the two halves of one tensor: one zero-filled buffer with its layout
            full_size = (2 * B,) + tuple(code_f.shape[1:])
            dall = _zeros_strided_like(torch.as_strided(code_f, full_size, code_f.stride()))
            dcode, dcode_pos = dall[:B], dall[B:]
        else:
            dcode = _zeros_strided_like(code_f)
            dcode_pos = _zeros_strided_like(code_f)
        sb, sc, sy, sx = code_f.stride()
        rc = _lib.load().stego_sample_norm_bwd(
            _lib.ptr(code_f), _lib.ptr(code_pos_f), sb, sc, sy, sx, _lib.ptr(coords1), _lib.ptr(coords2),
            _lib.ptr(perms_arg), _lib.ptr(dtiles), _lib.ptr(dcode), _lib.ptr(dcode_pos), B, D, H, W, spec.fs,
            spec.nslots, int(ctx.raw_perms), _lib.stream())
        _lib.check(rc, "stego_sample_norm_bwd")
        d0, d1 = ctx.code_dtype
        if ctx.pair:
            return (dall.to(d0), None) + (None,) * 11
        return (dcode.to(d0), dcode_pos.to(d1)) + (None,) * 11


def corr_loss(feats, feats_pos, code, code_pos, coords1, coords2, perms, spec: LossSpec, want_elems: bool = False,
              chan_scale=None, chan_scale_pos=None, raw_perms: bool = False, pair: bool = False):
    """raw_perms=True: `perms` holds the raw torch.randperm draws and the sampling kernel applies super_perm's
    fix-up itself (saves the eq/add/remainder launches of modules.super_perm).
    pair=True: `code` holds code ++ code_pos ([2B, D, h, w], one head pass) and `code_pos` is None.
    spec: a LossSpec (single-tile kernels) or a TiledLossSpec (multi-tile kernels); make_spec picks by feature_samples.
    Returns (losses[ncalls], cd_means[ncalls], cd[ncalls,B,S,S]|None, loss_elems|None).
    losses[k] is the mean of helper call k (0 intra, 1 inter, 2.. negatives); differentiable wrt code/code_pos."""
    return _CorrLossFn.apply(code, code_pos, feats, feats_pos, coords1, coords2, perms, spec, want_elems,
                             chan_scale, chan_scale_pos, raw_perms, pair)
