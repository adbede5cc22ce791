"""Dense-CRF post-processing on the GPU: drop-in for the reference's `src/crf.py` (`dense_crf`, `batched_crf`), which
hands every frame to pydensecrf on a pool of CPU processes (src/eval_segmentation.py:52-54,118,133-135).

Same parameters (src/crf.py:13-19) and the same preparation of image and unaries (src/crf.py:23-33); the mean-field
inference with permutohedral-lattice filtering runs as the sm_90a kernels of csrc/crf.cu.  pydensecrf itself is a
third-party dependency that is not part of the reference tree, so parity of this stage is UNPINNED: the kernels follow
the published densecrf algorithm and are tested against its CPU restatement oracle/crf_oracle.py (DESIGN.md).
No CPU fallback: CUDA tensors only.
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import torch
import torch.nn.functional as F

from . import _lib

MAX_ITER = 10
POS_W = 3
POS_XY_STD = 1
Bi_W = 4
Bi_XY_STD = 67
Bi_RGB_STD = 3

_LD = 32  # floats per pixel / lattice-point row (classes padded to a warp)


class _Lattice:
    """One permutohedral lattice: per-pixel vertex ids + barycentric weights, neighbour tables, symmetric norm."""
    __slots__ = ("d", "N", "M", "offset", "bary", "n1", "n2", "norm")


def _unpack(keys: torch.Tensor, d: int, bits: int) -> torch.Tensor:
    bias = 1 << (bits - 1)
    mask = (1 << bits) - 1
    return torch.stack([((keys >> (bits * (d - 1 - i))) & mask) - bias for i in range(d)], 1)


def _pack(coords: torch.Tensor, d: int, bits: int) -> torch.Tensor:
    bias = 1 << (bits - 1)
    mask = (1 << bits) - 1
    key = torch.zeros(coords.shape[0], dtype=torch.long, device=coords.device)
    for i in range(d):
        key = (key << bits) | ((coords[:, i] + bias) & mask)
    return key


def _build_lattice(H: int, W: int, d: int, sxy: float, srgb: float, image_u8: Optional[torch.Tensor], dev) -> _Lattice:
    """Lattice construction, once per image (the position-only lattice is cached per frame size by the caller):
    the embedding of every pixel is a kernel; de-duplicating the vertex keys and finding the blur neighbours are a sort
    and binary searches (torch.unique / searchsorted)."""
    lib = _lib.load()
    N = H * W
    keys = torch.empty(N, d + 1, dtype=torch.long, device=dev)
    bary = torch.empty(N, d + 1, dtype=torch.float32, device=dev)
    _lib.check(lib.stego_crf_lattice(H, W, d, float(sxy), float(srgb), _lib.ptr(image_u8), _lib.ptr(keys), _lib.ptr(bary),
                                     _lib.stream()), "stego_crf_lattice")
    uniq, inv = torch.unique(keys.reshape(-1), return_inverse=True)  # sorted
    M = int(uniq.numel())
    bits = 60 // d
    coords = _unpack(uniq, d, bits)
    n1 = torch.empty(d + 1, M, dtype=torch.int32, device=dev)
    n2 = torch.empty(d + 1, M, dtype=torch.int32, device=dev)
    for j in range(d + 1):  # permutohedral.cpp: neighbours along axis j are key -+ 1 with coordinate j moved by +- d
        k1, k2 = coords - 1, coords + 1
        if j < d:
            k1[:, j] = coords[:, j] + d
            k2[:, j] = coords[:, j] - d
        for dst, kk in ((n1, k1), (n2, k2)):
            q = _pack(kk, d, bits)
            pos = torch.searchsorted(uniq, q).clamp_(max=M - 1)
            dst[j] = torch.where(uniq[pos] == q, pos, torch.full_like(pos, -1)).to(torch.int32)
    lat = _Lattice()
    lat.d, lat.N, lat.M = d, N, M
    lat.offset = inv.reshape(N, d + 1).to(torch.int32).contiguous()
    lat.bary = bary
    lat.n1, lat.n2 = n1.contiguous(), n2.contiguous()
    # NORMALIZE_SYMMETRIC: norm = 1 / sqrt(K 1 + 1e-20), K 1 = slice(blur(splat(ones)))
    values = torch.zeros(M + 1, _LD, dtype=torch.float32, device=dev)
    tmp = torch.zeros(M + 1, _LD, dtype=torch.float32, device=dev)
    _lib.check(lib.stego_crf_splat_blur(d, N, M, 1, _lib.ptr(lat.offset), _lib.ptr(lat.bary), 0, 0, _lib.ptr(lat.n1),
                                        _lib.ptr(lat.n2), _lib.ptr(values), _lib.ptr(tmp), _lib.stream()), "stego_crf_splat_blur")
    blurred = tmp if (d + 1) % 2 else values
    lat.norm = torch.empty(N, dtype=torch.float32, device=dev)
    _lib.check(lib.stego_crf_norm(d, N, _lib.ptr(lat.offset), _lib.ptr(lat.bary), _lib.ptr(blurred), _lib.ptr(lat.norm),
                                  _lib.stream()), "stego_crf_norm")
    return lat


_POSITION_LATTICES: Dict[Tuple[int, int, float, int], _Lattice] = {}


def prepare_image(image_tensor: torch.Tensor) -> torch.Tensor:
    """src/crf.py:23: `np.array(VF.to_pil_image(unnorm(image_tensor)))[:, :, ::-1]` on the device: un-normalise with the
    ImageNet statistics (src/utils.py:140-141), x 255, truncate to uint8, reverse the channel order -> [H, W, 3] uint8.
    (Values outside [0, 255] are clamped; the reference's float->uint8 cast of such values is undefined.)"""
    dev = image_tensor.device
    mean = torch.tensor([0.485, 0.456, 0.406], device=dev).view(3, 1, 1)
    std = torch.tensor([0.229, 0.224, 0.225], device=dev).view(3, 1, 1)
    img = (image_tensor.detach().float() * std + mean).mul(255).clamp_(0, 255).to(torch.uint8)
    return img.flip(0).permute(1, 2, 0).contiguous()


def mean_field(logits_full: torch.Tensor, image_u8: torch.Tensor, n_iter: int = MAX_ITER, want_argmax: bool = False):
    """logits_full: [C, H, W] class scores at frame resolution (softmax is taken inside); image_u8: [H, W, 3] uint8.
    Returns Q [C, H, W] fp32 (and the argmax map [H, W] uint8)."""
    _lib.require_cuda(logits_full, image_u8)
    lib = _lib.load()
    C, H, W = logits_full.shape
    if C > _LD:
        raise RuntimeError(f"stego_b200.crf: {C} classes unsupported (<= {_LD})")
    dev = logits_full.device
    N = H * W
    key = (H, W, float(POS_XY_STD), dev.index)
    if key not in _POSITION_LATTICES:
        _POSITION_LATTICES[key] = _build_lattice(H, W, 2, POS_XY_STD, 0.0, None, dev)
    lg = _POSITION_LATTICES[key]
    lb = _build_lattice(H, W, 5, Bi_XY_STD, Bi_RGB_STD, image_u8, dev)
    logits = logits_full.detach().float().contiguous()
    unary = torch.empty(N, _LD, dtype=torch.float32, device=dev)
    Q = torch.empty(N, _LD, dtype=torch.float32, device=dev)
    _lib.check(lib.stego_crf_unary(_lib.ptr(logits), _lib.ptr(unary), _lib.ptr(Q), N, C, _lib.stream()), "stego_crf_unary")
    vg = torch.empty(2, lg.M + 1, _LD, dtype=torch.float32, device=dev)
    vb = torch.empty(2, lb.M + 1, _LD, dtype=torch.float32, device=dev)
    q_out = torch.empty(C, H, W, dtype=torch.float32, device=dev)
    arg = torch.empty(H, W, dtype=torch.uint8, device=dev) if want_argmax else None
    for it in range(n_iter):
        vg.zero_()
        vb.zero_()
        _lib.check(lib.stego_crf_splat_blur(2, N, lg.M, C, _lib.ptr(lg.offset), _lib.ptr(lg.bary), _lib.ptr(lg.norm), _lib.ptr(Q),
                                            _lib.ptr(lg.n1), _lib.ptr(lg.n2), _lib.ptr(vg[0]), _lib.ptr(vg[1]), _lib.stream()),
                   "stego_crf_splat_blur")
        _lib.check(lib.stego_crf_splat_blur(5, N, lb.M, C, _lib.ptr(lb.offset), _lib.ptr(lb.bary), _lib.ptr(lb.norm), _lib.ptr(Q),
                                            _lib.ptr(lb.n1), _lib.ptr(lb.n2), _lib.ptr(vb[0]), _lib.ptr(vb[1]), _lib.stream()),
                   "stego_crf_splat_blur")
        last = it == n_iter - 1
        _lib.check(lib.stego_crf_update(_lib.ptr(unary), _lib.ptr(lg.offset), _lib.ptr(lg.bary), _lib.ptr(vg[1]), _lib.ptr(lg.norm),
                                        _lib.ptr(lb.offset), _lib.ptr(lb.bary), _lib.ptr(vb[0]), _lib.ptr(lb.norm), float(POS_W),
                                        float(Bi_W), _lib.ptr(Q), _lib.ptr(q_out) if last else 0,
                                        _lib.ptr(arg) if (last and want_argmax) else 0, N, C, _lib.stream()), "stego_crf_update")
    if n_iter == 0:
        q_out.copy_(Q[:, :C].t().reshape(C, H, W))
        if want_argmax:
            arg.copy_(q_out.argmax(0).to(torch.uint8))
    return (q_out, arg) if want_argmax else q_out


def dense_crf(image_tensor: torch.Tensor, output_logits: torch.Tensor, want_argmax: bool = False):
    """src/crf.py:22-45 `dense_crf(image_tensor [3, H, W] normalised, output_logits [C, h, w]) -> Q [C, H, W]` (a CUDA
    tensor here; the reference returns a numpy array)."""
    if not (image_tensor.is_cuda and output_logits.is_cuda):
        raise RuntimeError("stego_b200.crf.dense_crf: CUDA tensors required (no CPU fallback)")
    image = prepare_image(image_tensor)
    H, W = image.shape[:2]
    logits = output_logits.detach().float()
    if tuple(logits.shape[-2:]) != (H, W):
        logits = F.interpolate(logits.unsqueeze(0), size=(H, W), mode="bilinear", align_corners=False).squeeze(0)
    return mean_field(logits, image, MAX_ITER, want_argmax)


def batched_crf(pool, img_tensor: torch.Tensor, prob_tensor: torch.Tensor) -> torch.Tensor:
    """src/crf.py:57-59 `batched_crf(pool, img_tensor [B,3,H,W], prob_tensor [B,C,h,w]) -> [B,C,H,W]`; `pool` (the reference's
    multiprocessing.Pool) is accepted and ignored: the frames run back to back on the current CUDA stream."""
    return torch.stack([dense_crf(i, p) for i, p in zip(img_tensor, prob_tensor)], 0)
