"""Oracle of the loader frames and labels (src/utils.py:165-183 get_transform and the data sets' remaps).  TEST
INFRASTRUCTURE ONLY.

Restates, in numpy on the decoded bytes, what the reference's loader does with a PIL image:
  * T.Resize(res, NEAREST): torchvision's output size (shorter side res, longer int(res * long / short); (res, res)
    with crop None), then Pillow's affine nearest-neighbour scaling: the source position starts at scale / 2, adds
    scale = in / out once per output pixel in double precision and is truncated; a position that reaches the input
    size leaves Pillow's fill value 0.  A size that does not change is not resampled.
  * T.CenterCrop(res): top / left = int(round((side - res) / 2.0)), round half to even.
  * ToTensor + Normalize: fp32 x / 255, then - mean, then / std (each rounded to fp32).
  * ToTargetTensor: int64, then the remap table of the data set.
Written independently of stego_b200.frames (a plain Python loop for the positions) so the two check each other.
"""
from __future__ import annotations

import numpy as np

MEAN = np.array([0.485, 0.456, 0.406], dtype=np.float32)
STD = np.array([0.229, 0.224, 0.225], dtype=np.float32)


def pillow_axis(n_in: int, n_out: int) -> np.ndarray:
    if n_in == n_out:
        return np.arange(n_out)
    scale = n_in / n_out
    pos, out = scale * 0.5, []
    for _ in range(n_out):
        i = int(pos)
        out.append(i if i < n_in else -1)
        pos += scale
    return np.array(out, dtype=np.int64)


def resized_size(h: int, w: int, res: int, crop):
    if crop is None:
        return res, res
    if w <= h:
        return int(res * h / w), res
    return res, int(res * w / h)


def gather(arr: np.ndarray, res: int, crop) -> np.ndarray:
    """Resize(res, NEAREST) then CenterCrop(res) (or Resize((res, res))) of an H x W (x C) uint8 array."""
    h, w = arr.shape[:2]
    oh, ow = resized_size(h, w, res, crop)
    top, left = int(round((oh - res) / 2.0)), int(round((ow - res) / 2.0))
    rows = pillow_axis(h, oh)[top:top + res]
    cols = pillow_axis(w, ow)[left:left + res]
    out = arr[np.clip(rows, 0, None)][:, np.clip(cols, 0, None)].copy()
    out[rows < 0] = 0
    out[:, cols < 0] = 0
    return out


def frame(rgb: np.ndarray, res: int, crop="center") -> np.ndarray:
    """get_transform(res, False, crop) of an H x W x 3 uint8 image: fp32 [3, res, res]."""
    x = gather(rgb, res, crop).transpose(2, 0, 1).astype(np.float32)
    x = x / np.float32(255)
    return (x - MEAN[:, None, None]) / STD[:, None, None]


def label(lab: np.ndarray, res: int, crop="center", table=None) -> np.ndarray:
    """get_transform(res, True, crop) of an H x W uint8 label map and the remap `table` (int64 [256] or None)."""
    x = gather(lab, res, crop).astype(np.int64)
    return x if table is None else np.asarray(table, dtype=np.int64)[x]


def coco_table(coco: dict, variant: str) -> np.ndarray:
    """Coco.__getitem__'s remap (src/data.py:303-319) of every label byte: "27", "3" (coarse_labels) or "stuff"
    (exclude_things).  coco: the data set's fine_to_coarse, cocostuff3_coarse_classes and first_stuff_index, as the
    fixture stores them."""
    fine_to_coarse = coco["fine_to_coarse"]
    ids = np.arange(256)
    coarse = np.array([fine_to_coarse.get(i, 0) for i in ids], dtype=np.int64)
    coarse[ids == 255] = -1
    if variant == "27":
        return coarse
    if variant == "stuff":
        return coarse - coco["first_stuff_index"]
    out = -np.ones(256, dtype=np.int64)
    for i, c in enumerate(coco["cocostuff3_coarse_classes"]):
        out[coarse == c] = i
    return out


def cityscapes_table() -> np.ndarray:
    """CityscapesSeg.__getitem__'s target - 7 with negatives -> -1 (src/data.py:359-360)."""
    t = np.arange(256, dtype=np.int64) - 7
    t[t < 0] = -1
    return t
