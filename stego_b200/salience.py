"""Salient sampling locations of the correspondence loss (cfg.use_salience; reference src/modules.py:298-311, 357-364).

`salience_coords` returns what `ContrastiveCorrelationLoss.draw_coords` returns with use_salience — the same bits, and
the CPU and CUDA generators left in the same state — from two kernel launches (stego_salience_counts,
stego_salience_coords) and three torch.rand draws, with one host wait: the reference's torch.nonzero and per-image
boolean indexing make the host wait for the device 2B + 2 times.  That one wait cannot go: the reference's randint for
an image with nonzeros runs on the CPU generator (modules.py:307 passes no device) and the one for an empty image on
the CUDA generator, so the state both generators are left in depends on which images are empty.  The host makes the
CPU draws itself; the kernel replays the empty images' CUDA draws from (seed, offset).
"""
from __future__ import annotations

import torch

from . import _lib

MAX_PIXELS = 1 << 28  # torch's CUDA randint draws 64-bit values from a range of 2^28 on: not reproduced here
_DIRECT = {torch.float32: 4, torch.uint8: 1, torch.bool: 1, torch.int8: 1}


def mask_view(mask: torch.Tensor, B: int = None):
    """[B, H, W] or [B, 1, H, W] mask -> (contiguous [B, H, W] tensor the kernel reads, bytes per element).  fp32 and
    one-byte masks are read as they are; other floating types are converted to fp32, as the reference's
    `.to(torch.float32)` does, and integer masks become `mask != 0` (exact: no nonzero integer converts to 0.0)."""
    if not isinstance(mask, torch.Tensor):
        raise TypeError("stego_b200.salience: masks must be tensors")
    if mask.dim() == 4 and mask.shape[1] == 1:
        mask = mask[:, 0]
    if mask.dim() != 3:
        raise ValueError(f"stego_b200.salience: masks must be [B, H, W] or [B, 1, H, W], got {tuple(mask.shape)}")
    if B is not None and mask.shape[0] != B:
        raise ValueError(f"stego_b200.salience: expected {B} masks, got {mask.shape[0]}")
    _, H, W = mask.shape
    if min(mask.shape) < 1 or H * W >= MAX_PIXELS:
        raise ValueError(f"stego_b200.salience: mask shape {tuple(mask.shape)}: B, H, W >= 1 and H * W < 2^28")
    if not mask.is_cuda:
        raise RuntimeError("stego_b200.salience: CUDA tensors required (no CPU fallback)")
    if mask.dtype not in _DIRECT:
        mask = mask.to(torch.float32) if mask.dtype.is_floating_point else mask != 0
    if mask.dtype == torch.bool:
        mask = mask.view(torch.uint8)
    return mask.contiguous(), _DIRECT[mask.dtype]


def masks_supported(mask, mask_pos, B: int, device) -> bool:
    """True when the pair can go to the kernel: CUDA tensors on `device`, [B, H, W] (H > 1: the reference's squeeze(1)
    would drop H = 1) or [B, 1, H, W], one shape, within the kernel's limits."""
    if not (isinstance(mask, torch.Tensor) and isinstance(mask_pos, torch.Tensor)):
        return False
    if not (mask.is_cuda and mask.device == device and mask_pos.device == device and mask.shape == mask_pos.shape):
        return False
    shape = tuple(mask.shape)
    if len(shape) == 4 and shape[1] == 1:
        shape = shape[:1] + shape[2:]
    elif len(shape) != 3 or shape[1] == 1:
        return False
    return shape[0] == B and min(shape) >= 1 and shape[1] * shape[2] < MAX_PIXELS and not mask.dtype.is_complex


def scratch_for(B: int, H: int, W: int, device):
    """The kernel's scratch for [B, H, W] masks (None when the bitmaps fit in shared memory)."""
    n = int(_lib.load().stego_salience_scratch_bytes(B, H, W))
    return torch.empty(n // 4, dtype=torch.int32, device=device) if n else None


def launch(m1, m2, mask_bytes, fs, seed, offsets, draws, u_reg1, u_reg2, u_keep, out1, out2, scratch=None):
    """stego_salience_coords on prepared operands (mask_view outputs, contiguous fp32 uniforms); draws [2B, 2 fs^2]
    int32 on the device; offsets [2B] int64 on the device, or None to take the empty units' draws from `draws`."""
    B, H, W = m1.shape
    _lib.check(_lib.load().stego_salience_coords(
        _lib.ptr(m1), _lib.ptr(m2), mask_bytes, B, H, W, fs, _signed64(seed), _lib.ptr(offsets), _lib.ptr(draws),
        _lib.ptr(u_reg1), _lib.ptr(u_reg2), _lib.ptr(u_keep), _lib.ptr(out1), _lib.ptr(out2), _lib.ptr(scratch),
        _lib.stream()), "stego_salience_coords")


def counts(m1, m2, mask_bytes):
    """[2B] int32 device tensor: the nonzeros of each (map, image) unit."""
    B, H, W = m1.shape
    out = torch.empty(2 * B, dtype=torch.int32, device=m1.device)
    _lib.check(_lib.load().stego_salience_counts(_lib.ptr(m1), _lib.ptr(m2), mask_bytes, B, H, W, _lib.ptr(out),
                                                 _lib.stream()), "stego_salience_counts")
    return out


def _signed64(v: int) -> int:
    return v - (1 << 64) if v >= 1 << 63 else v


def draw_into(mask, mask_pos, fs: int, out1, out2, keep, scratch=None) -> None:
    """The use_salience draws into caller buffers: out1 / out2 [B, fs, fs, 2] fp32 receive coords1 / coords2, keep
    [B, fs, fs] fp32 is scratch for the keep uniforms.  Generator consumption, in the reference's order, per unit
    (map, image): a CPU randint(count, (fs^2,)) for an image with nonzeros, a CUDA one (offset + 4) without; then
    rand(reg1), rand(reg2), rand(keep) on the device.  Enqueued on the current stream after one wait for the counts."""
    B = out1.shape[0]
    _draw(*mask_view(mask, B), *mask_view(mask_pos, B), fs, out1, out2, keep, scratch)


def _draw(m1, nbytes, m2, nbytes2, fs, out1, out2, keep, scratch):
    if m1.shape != m2.shape:
        raise ValueError(f"stego_b200.salience: mask shapes differ: {tuple(m1.shape)} vs {tuple(m2.shape)}")
    if m1.device != m2.device:
        raise ValueError("stego_b200.salience: the two masks are on different devices")
    if nbytes2 != nbytes:  # e.g. an fp32 mask with a bool mask_pos: read both as fp32
        m1, m2, nbytes = m1.to(torch.float32), m2.to(torch.float32), 4
    dev, B, n = m1.device, m1.shape[0], fs * fs
    cnt = counts(m1, m2, nbytes).cpu().tolist()  # the one host wait: which generator each randint call uses
    gen = torch.cuda.default_generators[dev.index]
    draws = torch.zeros(2 * B, 2 * n, dtype=torch.int32, pin_memory=True)
    offsets = torch.zeros(2 * B, dtype=torch.int64, pin_memory=True)
    for u, c in enumerate(cnt):
        if c > 0:
            draws[u, :n] = torch.randint(c, size=(n,))  # modules.py:307: the CPU generator
        else:
            off = gen.get_offset()  # modules.py:305: randint(H, (n, 2)) on the device, offset + 4
            offsets[u] = off
            gen.set_offset(off + 4)
    draws, offsets = draws.to(dev, non_blocking=True), offsets.to(dev, non_blocking=True)
    torch.rand(out1.shape, device=dev, out=out1)
    torch.rand(out2.shape, device=dev, out=out2)
    torch.rand(keep.shape, device=dev, out=keep)
    launch(m1, m2, nbytes, fs, gen.initial_seed(), offsets, draws, out1, out2, keep, out1, out2, scratch)


def salience_coords(salience: torch.Tensor, salience_pos: torch.Tensor, feature_samples: int):
    """(coords1, coords2), each [B, fs, fs, 2] fp32: `ContrastiveCorrelationLoss.draw_coords(feats, salience,
    salience_pos)` with cfg.use_salience, bit for bit, with the same consumption of the CPU and CUDA generators.
    Masks: [B, H, W] or [B, 1, H, W] of any dtype (a pixel is salient when nonzero; fp32 NaN is), H * W < 2^28;
    feature_samples 1..64.  One host wait (the 2B counts), where the reference waits 2B + 2 times."""
    fs = int(feature_samples)
    if not 1 <= fs <= 64:
        raise ValueError(f"stego_b200.salience: feature_samples={fs} (1..64)")
    m1, nbytes = mask_view(salience)
    B, H, W = m1.shape
    m2, nbytes2 = mask_view(salience_pos, B)
    dev = m1.device
    out1 = torch.empty(B, fs, fs, 2, dtype=torch.float32, device=dev)
    out2 = torch.empty_like(out1)
    keep = torch.empty(B, fs, fs, dtype=torch.float32, device=dev)
    _draw(m1, nbytes, m2, nbytes2, fs, out1, out2, keep, scratch_for(B, H, W, dev))
    return out1, out2
