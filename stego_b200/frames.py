"""Loader frames and labels on the GPU from decoded images of any size (reference src/utils.py:165-183 get_transform).

The reference's loaders run, per image in their host workers,

    img   = Normalize(mean, std)(ToTensor()(CenterCrop(res)(Resize(res, Image.NEAREST)(pil_rgb))))
    label = remap(ToTargetTensor()(CenterCrop(res)(Resize(res, Image.NEAREST)(pil_label))))

`load_frames` / `load_labels` take the decoded bytes (uint8 HWC RGB / HW label maps, as np.array(pil_image) gives
them) of a whole batch and build the same tensors on the device.  The host computes, per distinct image size, Pillow's
nearest-neighbour source row and column of every output pixel with the crop folded in (`pillow_nearest_index`,
`output_size`, `crop_offsets`), and packs the records, those tables and the image bytes into one pinned staging buffer:
one host-to-device copy and one launch per call (stego_frames_rgb8 / stego_labels_u8), no synchronisation and nothing
read back.  The label remap of a data set is a 256-entry int64 table (`label_lut`) applied in the same kernel.
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib

MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)  # src/utils.py:140 normalize (ImageNet statistics)
REC_WORDS = 4  # int64 words per record: byte offset, H, W, first table word
ROW_REC_WORDS = 7  # stego_store_rows_u8's records: those four, then the output's height, width and store byte offset
CROPS = ("center", None)


def pillow_nearest_index(n_in: int, n_out: int) -> np.ndarray:
    """The source index Pillow's Image.resize(..., NEAREST) reads for each of n_out outputs along an axis of n_in
    samples: int64 [n_out], -1 where Pillow writes its fill value 0 instead.

    Pillow scales with an affine map (ImagingScaleAffine): the position starts at scale / 2 and adds scale = n_in / n_out
    once per output pixel, in double precision, and is truncated.  This is not floor((x + .5) n_in / n_out): the sum
    drifts from the closed form by a few ulps, enough to land on the other side of an integer for some size pairs
    (2 -> 7, 8 -> 7, 14 -> 3203, ...).  A position that reaches n_in is not read; Pillow leaves that pixel at 0.
    np.cumsum adds sequentially, in the same order and precision as Pillow's loop."""
    scale = n_in / n_out
    steps = np.full(n_out, scale)
    steps[0] = scale * 0.5
    idx = np.cumsum(steps).astype(np.int64)
    idx[idx >= n_in] = -1
    return idx


def output_size(h: int, w: int, res: int, crop) -> tuple:
    """(height, width) of T.Resize(res) (crop "center": the shorter side becomes res, the longer int(res * long /
    short), torchvision's _compute_resized_output_size) or of T.Resize((res, res)) (crop None, as get_transform does)."""
    if crop is None:
        return res, res
    short, long = (w, h) if w <= h else (h, w)
    new_short, new_long = res, int(res * long / short)
    return (new_long, new_short) if w <= h else (new_short, new_long)


def crop_offsets(h: int, w: int, res: int) -> tuple:
    """(top, left) of T.CenterCrop(res) on an h x w image with h, w >= res: int(round((side - res) / 2.0)), Python's
    round-half-to-even (a side of 321 crops at 0, 323 at 2)."""
    return int(round((h - res) / 2.0)), int(round((w - res) / 2.0))


def index_tables(h: int, w: int, res: int, crop) -> tuple:
    """(rows, cols): int32 [res] source row / column of every output pixel of get_transform(res, ., crop) on an h x w
    image, -1 where Pillow writes its fill value."""
    oh, ow = output_size(h, w, res, crop)
    top, left = crop_offsets(oh, ow, res)
    rows = pillow_nearest_index(h, oh)[top:top + res]  # the identity when oh == h, as Pillow's copy
    cols = pillow_nearest_index(w, ow)[left:left + res]
    return rows.astype(np.int32), cols.astype(np.int32)


def label_lut(mapping, ignore_from: int = 255, default: int = 0) -> torch.Tensor:
    """int64 [256] table for load_labels: id -> mapping[id] for id < ignore_from (`default` for ids the mapping lacks),
    -1 for ids >= ignore_from.  The COCO-Stuff remap of src/data.py:303-309 (255 -> -1, fine -> coarse, unmapped -> 0)
    is label_lut(dataset.fine_to_coarse); ignore_from=256 maps every id through the mapping."""
    if not isinstance(ignore_from, int) or not 0 <= ignore_from <= 256:
        raise ValueError(f"stego_b200.frames.label_lut: ignore_from={ignore_from!r} (an int in 0..256)")
    table = [int(mapping.get(i, default)) if i < ignore_from else -1 for i in range(256)]
    return torch.tensor(table, dtype=torch.int64)


def _as_arrays(items, channels: int, who: str) -> list:
    if isinstance(items, (np.ndarray, torch.Tensor)) or not hasattr(items, "__len__"):
        raise TypeError(f"stego_b200.frames.{who}: pass a list of images (uint8 arrays or CPU tensors)")
    if len(items) < 1 or len(items) > 65535:
        raise ValueError(f"stego_b200.frames.{who}: {len(items)} images (1..65535)")
    out = []
    for k, x in enumerate(items):
        if isinstance(x, torch.Tensor):
            if x.device.type != "cpu":
                raise ValueError(f"stego_b200.frames.{who}: image {k} is on {x.device}; pass the decoded host bytes")
            if x.dtype != torch.uint8:
                raise ValueError(f"stego_b200.frames.{who}: image {k} is {x.dtype}, not uint8")
            x = x.numpy()
        elif not isinstance(x, np.ndarray):
            raise TypeError(f"stego_b200.frames.{who}: image {k} is a {type(x).__name__}, not an array or tensor")
        if x.dtype != np.uint8:
            raise ValueError(f"stego_b200.frames.{who}: image {k} is {x.dtype}, not uint8")
        want = "H x W x 3 (RGB)" if channels == 3 else "H x W"
        if x.ndim != (3 if channels == 3 else 2) or (channels == 3 and x.shape[2] != 3):
            raise ValueError(f"stego_b200.frames.{who}: image {k} has shape {x.shape}, not {want}")
        if x.shape[0] < 1 or x.shape[1] < 1 or x.shape[0] > 1 << 20 or x.shape[1] > 1 << 20:
            raise ValueError(f"stego_b200.frames.{who}: image {k} is {x.shape[0]} x {x.shape[1]} (1..2^20 per side)")
        out.append(x)
    return out


def _check_common(res, crop, who: str) -> None:
    if isinstance(res, bool) or not isinstance(res, int) or not 1 <= res <= 8192:
        raise ValueError(f"stego_b200.frames.{who}: res={res!r} (an int in 1..8192)")
    if crop not in CROPS:
        raise ValueError(f"stego_b200.frames.{who}: crop={crop!r} (\"center\" or None, as get_transform)")


def _require_cuda(who: str) -> torch.device:
    if not torch.cuda.is_available():
        raise RuntimeError(f"stego_b200.frames.{who}: needs a CUDA device (no CPU fallback)")
    return torch.device("cuda", torch.cuda.current_device())


def _stage(arrays, res: int, crop, lut=None, dest=None):
    """The pinned staging buffer: records, index tables (one per distinct image size), the LUT, then the image bytes.
    crop "random" stages the whole Resize(res) output of each image (no crop) for stego_store_rows_u8: 7-word records
    ending with (oh, ow, dest[i]), dest[i] being image i's byte offset in the ragged store.
    Returns (host uint8 tensor, table words, byte offset of the LUT or None)."""
    B = len(arrays)
    tables, table_of, words = [], {}, 0
    for x in arrays:
        key = x.shape[:2]
        if key not in table_of:
            table_of[key] = words  # output rows then output columns
            if crop == "random":
                oh, ow = output_size(key[0], key[1], res, "center")
                pair = (pillow_nearest_index(key[0], oh).astype(np.int32),
                        pillow_nearest_index(key[1], ow).astype(np.int32))
            else:
                pair = index_tables(key[0], key[1], res, crop)
            tables.extend(pair)
            words += pair[0].size + pair[1].size
    table = np.concatenate(tables)
    rec_words = ROW_REC_WORDS if crop == "random" else REC_WORDS
    head = 8 * rec_words * B
    pos = head + 4 * table.size
    lut_at = None
    if lut is not None:
        lut_at = pos = (pos + 7) // 8 * 8
        pos += 8 * 256
    offsets = []
    for x in arrays:
        offsets.append(pos)
        pos += x.size
    staging = torch.empty(pos, dtype=torch.uint8, pin_memory=True)
    buf = staging.numpy()
    rec = np.array([(off, x.shape[0], x.shape[1], table_of[x.shape[:2]]) for off, x in zip(offsets, arrays)],
                   dtype=np.int64)
    if crop == "random":
        sizes = [output_size(x.shape[0], x.shape[1], res, "center") for x in arrays]
        rec = np.concatenate([rec, np.array(sizes, dtype=np.int64), np.asarray(dest, dtype=np.int64)[:, None]], 1)
    buf[:head] = rec.reshape(-1).view(np.uint8)
    buf[head:head + 4 * table.size] = table.view(np.uint8)
    if lut is not None:
        buf[lut_at:lut_at + 8 * 256] = lut.view(np.uint8)
    for off, x in zip(offsets, arrays):
        buf[off:off + x.size] = x.reshape(-1)
    return staging, table.size, lut_at


def _as_lut(lut) -> np.ndarray:
    if isinstance(lut, torch.Tensor):
        if lut.device.type != "cpu":
            raise ValueError("stego_b200.frames.load_labels: lut must be a host table (label_lut builds one)")
        lut = lut.numpy()
    lut = np.asarray(lut)
    if lut.shape != (256,) or not (np.issubdtype(lut.dtype, np.integer)):
        raise ValueError(f"stego_b200.frames.load_labels: lut must be 256 integers, got {lut.dtype} {lut.shape}")
    return np.ascontiguousarray(lut, dtype=np.int64)


def load_frames(images, res: int, crop="center") -> torch.Tensor:
    """get_transform(res, False, crop) of every image, stacked: fp32 [B, 3, res, res] on the current CUDA device, bit-equal
    to torchvision's Resize(NEAREST), CenterCrop, ToTensor and Normalize of the same PIL images.

    images: B uint8 arrays or CPU tensors H x W x 3 (np.array(pil_image.convert("RGB"))), sizes may differ.  One
    host-to-device copy and one launch on the current stream; the caller is not synchronised."""
    _check_common(res, crop, "load_frames")
    arrays = _as_arrays(images, 3, "load_frames")
    dev = _require_cuda("load_frames")
    staging, words, _ = _stage(arrays, res, crop)
    staged = staging.to(dev, non_blocking=True)
    out = torch.empty(len(arrays), 3, res, res, dtype=torch.float32, device=dev)
    _lib.check(_lib.load().stego_frames_rgb8(staging.data_ptr(), _lib.ptr(staged), staging.numel(), words, len(arrays),
                                             res, *MEAN, *STD, _lib.ptr(out), _lib.stream()), "stego_frames_rgb8")
    return out


def load_labels(labels, res: int, crop="center", lut=None) -> torch.Tensor:
    """get_transform(res, True, crop) of every label map followed by a data set's remap: int64 [B, res, res] on the
    current CUDA device, lut[id] of each pixel (label_lut builds the table; None keeps the ids, as DirectoryDataset).

    labels: B uint8 arrays or CPU tensors H x W (np.array of a PIL "L" / "P" image), sizes may differ.  One
    host-to-device copy (the table travels with the maps) and one launch; the caller is not synchronised."""
    _check_common(res, crop, "load_labels")
    arrays = _as_arrays(labels, 1, "load_labels")
    table = None if lut is None else _as_lut(lut)
    dev = _require_cuda("load_labels")
    staging, words, lut_at = _stage(arrays, res, crop, table)
    staged = staging.to(dev, non_blocking=True)
    out = torch.empty(len(arrays), res, res, dtype=torch.int64, device=dev)
    lut_ptr = 0 if lut_at is None else _lib.ptr(staged) + lut_at
    _lib.check(_lib.load().stego_labels_u8(staging.data_ptr(), _lib.ptr(staged), staging.numel(), words, len(arrays),
                                           res, lut_ptr, _lib.ptr(out), _lib.stream()), "stego_labels_u8")
    return out
