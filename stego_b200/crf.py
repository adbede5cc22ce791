"""Dense-CRF post-processing on the GPU: drop-in for the reference's `src/crf.py` (`dense_crf`, `batched_crf`), which
hands every frame to pydensecrf on a pool of CPU processes (src/eval_segmentation.py:52-54,118,133-135).

Same parameters (src/crf.py:13-19) and the same preparation of image and unaries (src/crf.py:23-33); the mean-field
inference with permutohedral-lattice filtering runs as the sm_90a kernels of csrc/crf.cu.  pydensecrf itself is a
third-party dependency that is not part of the reference tree, so parity of this stage is UNPINNED: the kernels follow
the published densecrf algorithm and are tested against its CPU restatement oracle/crf_oracle.py (DESIGN.md).
No CPU fallback: CUDA tensors only.
"""
from __future__ import annotations

from typing import Dict, Iterable, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F

from . import _lib

MAX_ITER = 10
POS_W = 3
POS_XY_STD = 1
Bi_W = 4
Bi_XY_STD = 67
Bi_RGB_STD = 3

_LD = 32  # floats per pixel / lattice-point row of one probe (classes padded to a warp)


class _Lattice:
    """One permutohedral lattice: per-pixel vertex ids + barycentric weights, neighbour tables, CSR slot list,
    symmetric norm."""
    __slots__ = ("d", "N", "M", "offset", "bary", "n1", "n2", "norm", "rowptr", "slots")


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


def lattice_key_bound(H: int, W: int, d: int, sxy: float, srgb: float = 0.0) -> Tuple[float, int]:
    """(bound, limit): stego_crf_lattice's bound on the lattice coordinates of an H x W frame and the largest value its
    packed keys hold (60 // d bits per coordinate, biased); the kernel refuses a frame with bound >= limit.  The same
    arithmetic as crf.cu, so a caller can refuse such a frame before it launches anything."""
    fmax = max(W, H) / sxy * 2 + (3 * 255.0 / srgb if d == 5 else 0.0)
    return (d + 1) * 0.8165 * fmax + 2 * (d + 1), 1 << (60 // d - 1)


def _lattice_points(H: int, W: int, d: int, sxy: float, srgb: float, image_u8: Optional[torch.Tensor], dev) -> _Lattice:
    """Lattice construction without the normalisation: the embedding of every pixel is a kernel; de-duplicating the
    vertex keys and finding the blur neighbours are a sort and binary searches (torch.unique / searchsorted).  The
    (pixel, vertex) slots of every point form a CSR list: `slots` sorted by point, ascending slot index within a point
    (a stable sort of the point ids), and `rowptr` [M + 1]; the gather splat sums them in that order.  One host sync,
    for the number of lattice points."""
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
    ids = lat.offset.reshape(-1)
    order = torch.argsort(ids, stable=True)
    lat.slots = order.to(torch.int32)
    lat.rowptr = torch.searchsorted(ids[order], torch.arange(M + 1, dtype=torch.int32, device=dev)).to(torch.int32)
    return lat


def _norm(lat: _Lattice) -> None:
    """lat.norm, densecrf's NORMALIZE_SYMMETRIC factor 1 / sqrt(K 1 + 1e-20), by stego_crf_norm (a gather ones-splat)."""
    dev = lat.offset.device
    values = torch.empty(lat.M, dtype=torch.float32, device=dev)
    tmp = torch.empty(lat.M, dtype=torch.float32, device=dev)
    lat.norm = torch.empty(lat.N, dtype=torch.float32, device=dev)
    _lib.check(_lib.load().stego_crf_norm(lat.d, lat.N, lat.M, _lib.ptr(lat.offset), _lib.ptr(lat.bary),
                                          _lib.ptr(lat.rowptr), _lib.ptr(lat.slots), _lib.ptr(lat.n1), _lib.ptr(lat.n2),
                                          _lib.ptr(values), _lib.ptr(tmp), _lib.ptr(lat.norm), _lib.stream()),
               "stego_crf_norm")


_POSITION_LATTICES: Dict[Tuple[int, int, int], _Lattice] = {}


def _position_lattice(H: int, W: int, dev, cache: bool = True) -> _Lattice:
    """The Gaussian kernel's lattice of an H x W frame with its normalisation, cached per frame size: it depends on
    pixel positions only, so every frame of that size shares it.  cache=False builds it for the caller alone (a scene
    mosaic's lattice takes GBs and would stay for the life of the process); a cached copy is still reused."""
    key = (H, W, dev.index)
    if key not in _POSITION_LATTICES:
        lat = _lattice_points(H, W, 2, POS_XY_STD, 0.0, None, dev)
        _norm(lat)
        if not cache:
            return lat
        _POSITION_LATTICES[key] = lat
    return _POSITION_LATTICES[key]


def _bilateral_lattice(images_u8: Iterable[torch.Tensor]) -> _Lattice:
    """The bilateral lattices of B frames ([H, W, 3] uint8 each, prepare_image's layout), concatenated into one lattice
    over the B*H*W pixels (point ids, neighbour tables and slots offset by each frame's base), with its normalisation.
    One host sync per frame (the number of lattice points)."""
    frames = []
    for image in images_u8:
        H, W = image.shape[:2]
        frames.append(_lattice_points(H, W, 5, Bi_XY_STD, Bi_RGB_STD, image, image.device))
    if len(frames) == 1:
        out = frames[0]
    else:
        B, N, dev = len(frames), frames[0].N, frames[0].offset.device
        bases, m = [], 0
        for lat in frames:
            bases.append(m)
            m += lat.M
        out = _Lattice()
        out.d, out.N, out.M = 5, B * N, m
        out.offset = torch.cat([lat.offset + base for lat, base in zip(frames, bases)])
        out.bary = torch.cat([lat.bary for lat in frames])
        out.n1, out.n2 = (torch.cat([torch.where(t >= 0, t + base, t) for t, base in zip(ts, bases)], 1).contiguous()
                          for ts in ([lat.n1 for lat in frames], [lat.n2 for lat in frames]))
        slots_per_frame = N * 6
        out.slots = torch.cat([lat.slots + b * slots_per_frame for b, lat in enumerate(frames)])
        out.rowptr = torch.cat([lat.rowptr[:-1] + b * slots_per_frame for b, lat in enumerate(frames)] +
                               [torch.full((1,), B * slots_per_frame, dtype=torch.int32, device=dev)])
    _norm(out)
    return out


def _free_device_memory(dev) -> int:
    """Bytes a new allocation on dev can take: the device's free memory plus what torch's caching allocator holds
    unused."""
    free, _ = torch.cuda.mem_get_info(dev)
    return int(free) + int(torch.cuda.memory_reserved(dev) - torch.cuda.memory_allocated(dev))


def check_value_buffers(Mg: int, Mb: int, row: int, dev, what: str) -> None:
    """Refuses a mean field whose value buffers (val / tmp of both lattices: 2 (Mg + Mb) rows of `row` fp32) do not fit
    the free device memory, with a RuntimeError that names the sizes, instead of failing inside the allocation."""
    need = 2 * (Mg + Mb) * row * 4
    free = _free_device_memory(dev)
    if need > free:
        raise RuntimeError(f"{what}: the mean field's value buffers need {need / 2**30:.2f} GiB (position lattice {Mg} "
                           f"points, bilateral lattice {Mb} points, rows of {row} floats, two buffers each) but "
                           f"{free / 2**30:.2f} GiB of device memory is free")


def _launch_mean_field(B: int, N: int, lg: _Lattice, lb: _Lattice, unary: torch.Tensor, Q: torch.Tensor,
                       slots: Sequence[tuple], n_iter: int = MAX_ITER, label: Optional[torch.Tensor] = None,
                       n_classes: int = 0) -> None:
    """stego_crf_mean_field over B frames of N pixels: lg the position lattice of one frame (shared by the B frames), lb
    the frames' bilateral lattice, unary / Q rows of 32 floats per slot.  slots: one or two probe slots in row order,
    (n, marginals [B, n, N], argmax [B, N], int64 confusion), each output optional; the confusion counts are taken
    against label ([B, N] as ops.probe_label gives it) for classes below n_classes.  The value buffers, [2, B * lg.M, row]
    and [2, lb.M, row], are allocated here."""
    (n0, q0, p0, c0), (n1, q1, p1, c1) = slots[0], (slots[1] if len(slots) == 2 else (0, None, None, None))
    row = _LD * len(slots)
    val_g = torch.empty(2, B * lg.M, row, dtype=torch.float32, device=unary.device)
    val_b = torch.empty(2, lb.M, row, dtype=torch.float32, device=unary.device)
    _lib.check(_lib.load().stego_crf_mean_field(
        B, N, n0, n1, n_iter, _lib.ptr(unary), _lib.ptr(Q),
        _lib.ptr(lg.offset), _lib.ptr(lg.bary), _lib.ptr(lg.rowptr), _lib.ptr(lg.slots), _lib.ptr(lg.n1), _lib.ptr(lg.n2),
        _lib.ptr(lg.norm), lg.M,
        _lib.ptr(lb.offset), _lib.ptr(lb.bary), _lib.ptr(lb.rowptr), _lib.ptr(lb.slots), _lib.ptr(lb.n1), _lib.ptr(lb.n2),
        _lib.ptr(lb.norm), lb.M, float(POS_W), float(Bi_W),
        _lib.ptr(val_g[0]), _lib.ptr(val_g[1]), _lib.ptr(val_b[0]), _lib.ptr(val_b[1]), _lib.ptr(q0), _lib.ptr(q1),
        _lib.ptr(p0), _lib.ptr(p1), _lib.ptr(label), 0 if label is None else label.element_size(), n_classes,
        _lib.ptr(c0), _lib.ptr(c1), _lib.stream()), "stego_crf_mean_field")


_IMAGENET_STATS: Dict[torch.device, Tuple[torch.Tensor, torch.Tensor]] = {}


def prepare_image(image_tensor: torch.Tensor) -> torch.Tensor:
    """src/crf.py:23: `np.array(VF.to_pil_image(unnorm(image_tensor)))[:, :, ::-1]` on the device: un-normalise with the
    ImageNet statistics (src/utils.py:140-141), x 255, truncate to uint8, reverse the channel order -> [H, W, 3] uint8.
    (Values outside [0, 255] are clamped; the reference's float->uint8 cast of such values is undefined.)"""
    dev = image_tensor.device
    if dev not in _IMAGENET_STATS:  # built once per device: a tensor from a host list is a synchronising copy
        _IMAGENET_STATS[dev] = (torch.tensor([0.485, 0.456, 0.406], device=dev).view(3, 1, 1),
                                torch.tensor([0.229, 0.224, 0.225], device=dev).view(3, 1, 1))
    mean, std = _IMAGENET_STATS[dev]
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
    lg = _position_lattice(H, W, dev)
    lb = _bilateral_lattice([image_u8])
    logits = logits_full.detach().float().contiguous()
    unary = torch.empty(N, _LD, dtype=torch.float32, device=dev)
    Q = torch.empty(N, _LD, dtype=torch.float32, device=dev)
    _lib.check(lib.stego_crf_unary(_lib.ptr(logits), _lib.ptr(unary), _lib.ptr(Q), N, C, _lib.stream()), "stego_crf_unary")
    q_out = torch.empty(C, H, W, dtype=torch.float32, device=dev)
    arg = torch.empty(H, W, dtype=torch.uint8, device=dev) if want_argmax else None
    if n_iter > 0:
        _launch_mean_field(1, N, lg, lb, unary, Q, [(C, q_out, arg, None)], n_iter)
    else:
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
