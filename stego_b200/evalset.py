"""The evaluation sets kept resident on the GPU (or in pinned host memory): the validation and evaluation batches of
the reference's uncropped classes, Coco (cocostuff27 / cocostuff15 / cocostuff3), CityscapesSeg, Potsdam and
PotsdamRaw, decoded once and gathered in one launch per batch.

The reference validates with ContrastiveSegDataset(dataset_name, crop_type=None, image_set="val",
get_transform(res, ., "center"), mask=True) under a shuffle=False DataLoader (src/train_segmentation.py:449-476), and
eval_segmentation.py reads the same sets.  The transform has no randomness, so every pass re-decodes the same files
into the same frames.  `EvalSet` decodes each file once in DataLoader workers, runs the transform once on the GPU (the
store build of dataset.ResidentDataset: stego_frames_store_rgb8 / stego_labels_store_u8) and keeps

    images uint8 [n, 3, res, res] and the raw label bytes uint8 [n, res, res]: 4 * res^2 bytes per sample,

on the device (location="cuda") or in pinned host memory read over PCIe (location="host").  A batch is then one launch
(stego_evalset_batch): the frames normalised as load_frames computes them, the label bytes through the class's
256-entry table (`label_table`) and the class's mask:

    kind                                     label (per byte b)                               mask
    cocostuff27  Coco(subset None; val: 7)   coarse(b) = fine_to_coarse[b], 0 if unmapped,    bool, label >= 0
                                             -1 for b = 255
    cocostuff15  Coco(subset 7, no things)   coarse(b) - 12                                   bool, label >= 0
    cocostuff3   Coco(subset 6, coarse)      index of coarse(b) in (23, 22, 21), else -1      bool, label >= 0
    cityscapes   CityscapesSeg               b - 7, negatives -1                              bool, label == -1 [1, res, res]
    potsdam(raw) Potsdam / PotsdamRaw        {0, 4} -> 0, {1, 5} -> 1, {2, 3} -> 2, 255 -> -1, fp32, label > 0
                                             others 0

Coco's 182-entry fine -> coarse table is the COCO-Stuff class hierarchy; the caller passes it (`fine_to_coarse`, as
`Coco(...).fine_to_coarse` holds it), as for frames.label_lut.
"""
from __future__ import annotations

import os

import numpy as np
import torch
from PIL import Image
from torch.utils.data import Dataset

from .dataset import LOCATIONS, MASK_IS_IGNORE, MASK_IS_POSITIVE, _check_int, _Store, image_size, shard

COCO_KINDS = ("cocostuff27", "cocostuff15", "cocostuff3")
KINDS = COCO_KINDS + ("cityscapes", "potsdam", "potsdamraw")
MASK_IS_NONNEG = 2  # stego_evalset_batch's third mask rule: bool (label >= 0), Coco's
COCO_SPLITS = {"train": ["train2017"], "val": ["val2017"], "train+val": ["train2017", "val2017"]}
COCO_LISTS = {None: "Coco164kFull_Stuff_Coarse.txt", 6: "Coco164kFew_Stuff_6.txt", 7: "Coco164kFull_Stuff_Coarse_7.txt"}
COCO3_CLASSES = (23, 22, 21)  # the coarse ids of ground-, plant- and sky-stuff: cocostuff3's labels 0, 1, 2
COCO_FIRST_STUFF = 12         # cocostuff15 drops the 12 coarse thing classes
CITYSCAPES_FIRST_NONVOID = 7
CITYSCAPES_SPLITS = ("train", "test", "val")  # torchvision Cityscapes, mode="fine"
POTSDAM_SPLITS = {"train": ["labelled_train.txt"], "unlabelled_train": ["unlabelled_train.txt"],
                  "val": ["labelled_test.txt"], "train+val": ["labelled_train.txt", "labelled_test.txt"],
                  "all": ["all.txt"]}
POTSDAM_COARSE = {0: 0, 4: 0, 1: 1, 5: 1, 2: 2, 3: 2, 255: -1}  # roads and cars, buildings and clutter, vegetation
POTSDAMRAW_GRID = (38, 15, 15)  # images, tile rows, tile columns


def _fail(who: str, msg: str):
    raise ValueError(f"stego_b200.evalset.{who}: {msg}")


def coco_subset(kind: str, image_set: str):
    """The `subset` ContrastiveSegDataset gives Coco for `kind` (src/data.py:467-484): cocostuff3 6, cocostuff15 7,
    cocostuff27 None, except 7 for its val split."""
    if kind == "cocostuff3":
        return 6
    if kind == "cocostuff15" or image_set == "val":
        return 7
    return None


def label_table(kind: str, fine_to_coarse=None) -> torch.Tensor:
    """int64 [256]: the label a class returns for each label byte (table above).  fine_to_coarse: Coco's
    {fine id: coarse id} mapping, needed for the Coco kinds only."""
    who = "label_table"
    if kind not in KINDS:
        _fail(who, f"kind={kind!r} (one of {', '.join(KINDS)})")
    ids = range(256)
    if kind in COCO_KINDS:
        if fine_to_coarse is None or not hasattr(fine_to_coarse, "items"):
            _fail(who, f"{kind} needs Coco's fine_to_coarse mapping {{fine id: coarse id}}")
        mapping = {int(k): int(v) for k, v in fine_to_coarse.items()}
        if any(not 0 <= k < 255 for k in mapping) or any(not 0 <= v < 255 for v in mapping.values()):
            _fail(who, "fine_to_coarse maps ids in 0..254 to coarse ids in 0..254")
        coarse = [-1 if b == 255 else mapping.get(b, 0) for b in ids]
        if kind == "cocostuff27":
            table = coarse
        elif kind == "cocostuff15":
            table = [c - COCO_FIRST_STUFF for c in coarse]
        else:
            table = [COCO3_CLASSES.index(c) if c in COCO3_CLASSES else -1 for c in coarse]
    elif kind == "cityscapes":
        table = [max(b - CITYSCAPES_FIRST_NONVOID, -1) for b in ids]
    else:
        table = [POTSDAM_COARSE.get(b, 0) for b in ids]
    return torch.tensor(table, dtype=torch.int64)


# ---- file listings, in each reference class's order ----------------------------------------------------------------
def coco_files(root: str, kind: str, image_set: str) -> tuple:
    """Coco(root, image_set, subset=coco_subset(kind, image_set)) (src/data.py:232-279): the ids of
    {root}/cocostuff/curated/{split}/{list} in file order, split by split, as images/{split}/{id}.jpg and
    annotations/{split}/{id}.png."""
    if kind not in COCO_KINDS:
        _fail("coco_files", f"kind={kind!r} (one of {', '.join(COCO_KINDS)})")
    if image_set not in COCO_SPLITS:
        _fail("coco_files", f"image_set={image_set!r} (one of {', '.join(COCO_SPLITS)})")
    base, listing = os.path.join(root, "cocostuff"), COCO_LISTS[coco_subset(kind, image_set)]
    images, labels = [], []
    for split in COCO_SPLITS[image_set]:
        with open(os.path.join(base, "curated", split, listing)) as f:
            for img_id in (line.rstrip() for line in f.readlines()):
                images.append(os.path.join(base, "images", split, img_id + ".jpg"))
                labels.append(os.path.join(base, "annotations", split, img_id + ".png"))
    return images, labels


def cityscapes_files(root: str, image_set: str) -> tuple:
    """CityscapesSeg(root, image_set) (src/data.py:325-350), i.e. torchvision's Cityscapes(root/cityscapes, image_set,
    mode="fine", target_type="semantic"): os.listdir of leftImg8bit/{split} (unsorted), then of each city, and the
    target gtFine/{split}/{city}/{name up to _leftImg8bit}_gtFine_labelIds.png."""
    if image_set not in CITYSCAPES_SPLITS:
        _fail("cityscapes_files", f"image_set={image_set!r} (one of {', '.join(CITYSCAPES_SPLITS)})")
    images_dir = os.path.join(root, "cityscapes", "leftImg8bit", image_set)
    targets_dir = os.path.join(root, "cityscapes", "gtFine", image_set)
    if not os.path.isdir(images_dir) or not os.path.isdir(targets_dir):
        _fail("cityscapes_files", f"{images_dir} or {targets_dir} is missing")
    images, labels = [], []
    for city in os.listdir(images_dir):
        for name in os.listdir(os.path.join(images_dir, city)):
            images.append(os.path.join(images_dir, city, name))
            labels.append(os.path.join(targets_dir, city, name.split("_leftImg8bit")[0] + "_gtFine_labelIds.png"))
    return images, labels


def potsdam_files(root: str, image_set: str) -> tuple:
    """Potsdam(root, image_set) (src/data.py:121-144): the ids of the split's text files under {root}/potsdam, as
    imgs/{id}.mat and gt/{id}.mat."""
    if image_set not in POTSDAM_SPLITS:
        _fail("potsdam_files", f"image_set={image_set!r} (one of {', '.join(POTSDAM_SPLITS)})")
    base, ids = os.path.join(root, "potsdam"), []
    for split_file in POTSDAM_SPLITS[image_set]:
        with open(os.path.join(base, split_file)) as f:
            ids.extend(line.rstrip() for line in f.readlines())
    return ([os.path.join(base, "imgs", i + ".mat") for i in ids], [os.path.join(base, "gt", i + ".mat") for i in ids])


def potsdamraw_files(root: str) -> tuple:
    """PotsdamRaw(root, ...) (src/data.py:181-197): the 38 x 15 x 15 tiles {im}_{row}_{col}.mat under
    {root}/potsdamraw/processed/imgs and gt, whatever the split."""
    base = os.path.join(root, "potsdamraw", "processed")
    n_im, n_h, n_w = POTSDAMRAW_GRID
    names = [f"{i}_{h}_{w}.mat" for i in range(n_im) for h in range(n_h) for w in range(n_w)]
    return [os.path.join(base, "imgs", f) for f in names], [os.path.join(base, "gt", f) for f in names]


class _EvalFiles(Dataset):
    """(image array, label array) per index, decoded as the reference's classes open them: reader "pil" converts the
    image to RGB and reads the label as it is (Coco, CityscapesSeg); reader "mat" reads scipy .mat files, "img"'s first
    three channels and "gt", 255 everywhere when the gt file does not exist (Potsdam, PotsdamRaw)."""

    def __init__(self, images: list, labels: list, reader: str):
        self.images, self.labels, self.reader = images, labels, reader

    def __getitem__(self, index):
        if self.reader == "pil":
            with Image.open(self.images[index]) as im:
                img = np.asarray(im.convert("RGB"))
            with Image.open(self.labels[index]) as im:
                return img, np.asarray(im)
        return read_mat(self.images[index], self.labels[index])

    def __len__(self):
        return len(self.images)


def read_mat(image_path: str, label_path: str) -> tuple:
    """A Potsdam tile: uint8 "img" [H, W, C >= 3] cut to RGB, uint8 "gt" [H, W] (all 255 when its file is missing).
    Only uint8 is taken: to_pil_image would rescale any other dtype, which the store does not reproduce."""
    from scipy.io import loadmat
    img = loadmat(image_path)["img"]
    if img.dtype != np.uint8 or img.ndim != 3 or img.shape[2] < 3:
        _fail("read_mat", f"{image_path}: img is {img.dtype} {img.shape}; a uint8 [H, W, C >= 3] array is needed")
    img = np.ascontiguousarray(img[..., :3])
    try:
        gt = loadmat(label_path)["gt"]
    except FileNotFoundError:
        return img, np.full(img.shape[:2], 255, dtype=np.uint8)
    if gt.dtype != np.uint8 or gt.ndim != 2:
        _fail("read_mat", f"{label_path}: gt is {gt.dtype} {gt.shape}; a uint8 [H, W] array is needed")
    return img, gt


def source_sizes(images: list, labels: list, reader: str) -> np.ndarray:
    """int64 [n, 4]: each image's height, width and its label map's, from the file headers (scipy's whosmat for the
    .mat tiles; a missing gt file is the image's size): the row sizes a crop="random" store is made with."""
    from scipy.io import whosmat
    out = []
    for image, label in zip(images, labels):
        if reader == "pil":
            out.append(image_size(image) + image_size(label))
            continue
        hw = next(shape[:2] for name, shape, _ in whosmat(image) if name == "img")
        lhw = next((shape[:2] for name, shape, _ in whosmat(label) if name == "gt"), hw) if os.path.exists(label) else hw
        out.append(tuple(hw) + tuple(lhw))
    return np.array(out, dtype=np.int64).reshape(-1, 4)


class EvalSet(_Store):
    """An evaluation set of one of KINDS resident in memory, n samples at res (4 * res^2 bytes each with crop "center"
    or None; with "random" each row's whole Resize(res) output).

    Rows are filled in order by `append` (images uint8 H x W x 3, label maps uint8 H x W) or built from the files by
    the `coco` / `cityscapes` / `potsdam` / `potsdamraw` constructors; `frames` and `batches` need all n.  `batches`
    is the training loader of ContrastiveSegDataset(root, kind, None, "train", ...) (dataset._Store.batches), crop the
    loader's (train_config.yml loader_crop_type)."""

    _PREFIX = "stego_b200.evalset"
    _ENTRY = "stego_evalset_batch"

    def __init__(self, n: int, res: int, kind: str, location: str = "cuda", fine_to_coarse=None, crop="center",
                 sizes=None):
        who = "EvalSet"
        if kind not in KINDS:
            _fail(who, f"kind={kind!r} (one of {', '.join(KINDS)}); the five-crop and directory sets are "
                       f"dataset.ResidentDataset's")
        if location not in LOCATIONS:
            _fail(who, f"location={location!r} (\"cuda\" or \"host\")")
        lut = label_table(kind, fine_to_coarse)
        n = _check_int(n, "n", 1, 1 << 40, who)
        res = _check_int(res, "res", 1, 8192, who)
        self.kind = kind
        self._mask_kind = (MASK_IS_NONNEG if kind in COCO_KINDS else MASK_IS_IGNORE if kind == "cityscapes" else
                           MASK_IS_POSITIVE)
        self._allocate(n, res, location, True, lut, crop, sizes)

    @classmethod
    def _from_files(cls, images, labels, reader, res, kind, location, batch_size, num_workers, fine_to_coarse=None,
                    crop="center"):
        if not images:
            _fail(f"EvalSet.{kind}", "the listing names no files")
        if len(images) != len(labels):
            _fail(f"EvalSet.{kind}", f"{len(images)} images but {len(labels)} label files")
        sizes = source_sizes(images, labels, reader) if crop == "random" else None
        store = cls(len(images), res, kind, location, fine_to_coarse, crop, sizes)
        store._fill(_EvalFiles(images, labels, reader), batch_size, num_workers)
        return store

    @classmethod
    def coco(cls, root: str, kind: str, image_set: str, res: int, fine_to_coarse, location: str = "cuda",
             batch_size: int = 64, num_workers: int = 0, crop="center") -> "EvalSet":
        """ContrastiveSegDataset(root, kind, None, image_set, ...)'s Coco (`coco_files`), decoded once in
        DataLoader(num_workers) workers."""
        images, labels = coco_files(root, kind, image_set)
        return cls._from_files(images, labels, "pil", res, kind, location, batch_size, num_workers, fine_to_coarse,
                               crop)

    @classmethod
    def cityscapes(cls, root: str, image_set: str, res: int, location: str = "cuda", batch_size: int = 64,
                   num_workers: int = 0, crop="center") -> "EvalSet":
        """ContrastiveSegDataset(root, "cityscapes", None, image_set, ...)'s CityscapesSeg (`cityscapes_files`)."""
        images, labels = cityscapes_files(root, image_set)
        return cls._from_files(images, labels, "pil", res, "cityscapes", location, batch_size, num_workers, crop=crop)

    @classmethod
    def potsdam(cls, root: str, image_set: str, res: int, location: str = "cuda", batch_size: int = 64,
                num_workers: int = 0, crop="center") -> "EvalSet":
        """ContrastiveSegDataset(root, "potsdam", None, image_set, ...)'s Potsdam (`potsdam_files`, `read_mat`)."""
        images, labels = potsdam_files(root, image_set)
        return cls._from_files(images, labels, "mat", res, "potsdam", location, batch_size, num_workers, crop=crop)

    @classmethod
    def potsdamraw(cls, root: str, res: int, location: str = "cuda", batch_size: int = 64,
                   num_workers: int = 0, crop="center") -> "EvalSet":
        """ContrastiveSegDataset(root, "potsdamraw", None, ...)'s PotsdamRaw (`potsdamraw_files`, `read_mat`)."""
        images, labels = potsdamraw_files(root)
        return cls._from_files(images, labels, "mat", res, "potsdamraw", location, batch_size, num_workers, crop=crop)

    # ---- reading --------------------------------------------------------------------------------------------------
    def _shaped(self, label, mask):
        """The class's per-sample shapes, batched: label [B, res, res]; mask [B, 1, res, res] for CityscapesSeg,
        [B, res, res] otherwise."""
        return label, mask.unsqueeze(1) if self.kind == "cityscapes" else mask

    def frames(self, batch_size: int, dtype=torch.float32, mask: bool = True, rank: int = 0, world_size: int = 1):
        """The batches of DataLoader(ContrastiveSegDataset(..., mask=mask), batch_size, shuffle=False) with
        get_transform(res, ., "center") (a crop="random" store yields the centre windows, crop None the squashed
        frames): dicts of ind
        (int64, CPU), img (dtype), label (int64 [B, res, res]) and with `mask` the class's mask (Coco: bool
        [B, res, res]; CityscapesSeg: bool [B, 1, res, res]; Potsdam, PotsdamRaw: fp32 [B, res, res]), on the store's
        device.  With world_size > 1, rank `rank`'s samples of DistributedSampler(shuffle=False), padding included.
        One launch per batch on the current stream with fresh outputs; nothing synchronises the host."""
        who = "EvalSet.frames"
        self._require_full(who)
        batch_size = _check_int(batch_size, "batch_size", 1, 65535, who)
        self._check_dtype(dtype, who)
        world_size = _check_int(world_size, "world_size", 1, 1 << 20, who)
        rank = _check_int(rank, "rank", 0, world_size - 1, who)
        order = np.asarray(shard(list(range(self.n)), rank, world_size), dtype=np.int64)
        for start in range(0, order.size, batch_size):
            ind = order[start:start + batch_size]
            img, label, m = self._gather(ind, dtype)
            batch = dict(ind=torch.from_numpy(ind), img=img, label=label)
            if mask:
                batch["mask"] = self._shaped(label, m)[1]
            yield batch
