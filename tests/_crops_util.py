"""Synthetic Coco and Cityscapes source trees and the JPEG corpus shared by tests/test_crops.py and
tests/test_crops_gpu.py."""
import os

import numpy as np
import torch
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CORPUS_SIZES = [(1, 1), (1, 2), (2, 1), (1, 5), (5, 1), (3, 3), (4, 4), (5, 7), (7, 5), (6, 9), (15, 17), (16, 16),
                (17, 33), (33, 17), (213, 320), (320, 213), (512, 1024), (1, 2048), (2048, 1)]
CONTENTS = ("noise", "flat", "saturated", "gray", "gradient")
# (h, w) of the synthetic originals: odd and even sides, both orientations, one grayscale file in each tree
TREE_SIZES = [(37, 50), (48, 33), (61, 64), (40, 40)]


def corpus_image(h: int, w: int, content: str, seed: int = 0) -> np.ndarray:
    rng = np.random.default_rng(seed * 7919 + h * 131 + w)
    if content == "noise":
        return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    if content == "flat":
        return np.broadcast_to(rng.integers(0, 256, 3).astype(np.uint8), (h, w, 3)).copy()
    if content == "saturated":  # pure primaries and black / white: drives the range limit
        return (rng.integers(0, 2, (h, w, 3)) * 255).astype(np.uint8)
    if content == "gray":
        return np.repeat(rng.integers(0, 256, (h, w, 1), dtype=np.uint8), 3, axis=2)
    yy, xx = np.mgrid[0:h, 0:w]
    return np.stack([xx * 255 // max(w - 1, 1), yy * 255 // max(h - 1, 1),
                     (xx + yy) * 255 // max(h + w - 2, 1)], -1).astype(np.uint8)


def fine_to_coarse() -> dict:
    return torch.load(os.path.join(ROOT, "tests", "golden", "evalset.pt"), weights_only=False)["fine_to_coarse"]


def _image(k: int, h: int, w: int, rng) -> Image.Image:
    if k == 1:
        return Image.fromarray(rng.integers(0, 256, (h, w), dtype=np.uint8), "L")
    yy, xx = np.mgrid[0:h, 0:w]
    smooth = np.stack([(xx * 7 + yy * 3) % 256, (yy * 11) % 256, (xx * 5) % 256], -1).astype(np.uint8)
    return Image.fromarray(np.clip(smooth.astype(int) + rng.integers(-20, 21, (h, w, 3)), 0, 255).astype(np.uint8))


def make_coco_tree(root: str, image_set: str = "train") -> str:
    """{root}/cocostuff with the curated list Coco reads for cocostuff27 (subset None; val: 7), JPEG images (one
    grayscale) and PNG fine labels (ids 0..181 and 255)."""
    split = {"train": "train2017", "val": "val2017"}[image_set]
    listing = "Coco164kFull_Stuff_Coarse.txt" if image_set == "train" else "Coco164kFull_Stuff_Coarse_7.txt"
    base = os.path.join(root, "cocostuff")
    for d in ("curated", "images", "annotations"):
        os.makedirs(os.path.join(base, d, split), exist_ok=True)
    rng = np.random.default_rng(5)
    ids = []
    for k, (h, w) in enumerate(TREE_SIZES):
        img_id = f"{100 + 7 * k:012d}"
        ids.append(img_id)
        _image(k, h, w, rng).save(os.path.join(base, "images", split, img_id + ".jpg"), quality=90)
        label = rng.choice(np.r_[np.arange(182), 255], (h, w)).astype(np.uint8)
        Image.fromarray(label).save(os.path.join(base, "annotations", split, img_id + ".png"))
    with open(os.path.join(base, "curated", split, listing), "w") as f:
        f.write("".join(i + "\n" for i in ids))
    return root


def make_cityscapes_tree(root: str, image_set: str = "train") -> str:
    """{root}/cityscapes with leftImg8bit PNG images (one grayscale) and gtFine labelIds (ids 0..33 and 255) in two
    cities."""
    rng = np.random.default_rng(6)
    for k, (h, w) in enumerate(TREE_SIZES):
        city = ("aachen", "bochum")[k % 2]
        name = f"{city}_{k:06d}_000019"
        img_dir = os.path.join(root, "cityscapes", "leftImg8bit", image_set, city)
        gt_dir = os.path.join(root, "cityscapes", "gtFine", image_set, city)
        os.makedirs(img_dir, exist_ok=True)
        os.makedirs(gt_dir, exist_ok=True)
        _image(k, h, w, rng).save(os.path.join(img_dir, name + "_leftImg8bit.png"))
        label = rng.choice(np.r_[np.arange(34), 255], (h, w)).astype(np.uint8)
        Image.fromarray(label).save(os.path.join(gt_dir, name + "_gtFine_labelIds.png"))
    return root
