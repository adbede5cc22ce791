"""The cropped training sets built from the uncropped Coco and Cityscapes originals: the reference's crop_datasets.py
(src/crop_datasets.py) as a host writer of its file tree and as a GPU builder of the resident store that
`ResidentDataset.cropped` reads from that tree.

The reference trains from `{root}/cropped/{name}_{crop_type}_crop_{crop_ratio}/`, which its crop script writes: for
source image `item` (in Coco's / CityscapesSeg's file order) five crop windows (`crop_windows`), each saved as
`img/{image_set}/{item * 5 + k}.jpg` with Pillow's default JPEG settings (quality 75, 4:2:0, islow DCT) and
`label/{image_set}/{item * 5 + k}.png` holding label + 1.  CroppedDataset then decodes those files, so the model trains
on the crops after a lossy encode and decode.

`write_cropped` writes that tree on the host.  `build_store` (ResidentDataset.crops) builds the same rows without
files: each original is decoded once in DataLoader workers and staged as it is; per crop one record (source, top, left,
height, width).  stego_jpeg_crops_codec runs the encoder and decoder arithmetic per 16 x 16 MCU of every window, and
stego_jpeg_crops_store_rgb8 rebuilds only the pixels get_transform(res, False, "center") reads of each decoded crop,
writing the store's bytes.  The label rows are the existing label gather (stego_labels_store_u8) with the window
folded into its index tables; the store keeps the source's raw label bytes and maps them through the class's table
(`evalset.label_table`), which equals CroppedDataset's byte - 1 of the PNG the reference writes.
"""
from __future__ import annotations

import os

import numpy as np
import torch
from PIL import Image
from torch.utils.data import DataLoader, Dataset

from . import _lib, evalset, frames
from .dataset import _as_list, _check_int

DATASETS = ("cocostuff27", "cityscapes")
CROP_TYPES = ("five", "random")
CROPS_PER_IMAGE = 5
REC_WORDS = 9  # stego_jpeg_crops_*: source offset, H, W, top, left, h, w, first table word, workspace offset


def _fail(who: str, msg: str):
    raise ValueError(f"stego_b200.crops.{who}: {msg}")


def _check_args(who: str, dataset_name, crop_type, crop_ratio, fine_to_coarse) -> None:
    if dataset_name not in DATASETS:
        _fail(who, f"dataset_name={dataset_name!r} (one of {', '.join(DATASETS)}, the sets crop_datasets.py reads)")
    if crop_type not in CROP_TYPES:
        _fail(who, f"crop_type={crop_type!r} (\"five\" or \"random\")")
    if isinstance(crop_ratio, bool) or not isinstance(crop_ratio, (int, float)) or not 0 < crop_ratio <= 1:
        _fail(who, f"crop_ratio={crop_ratio!r} (a number in (0, 1])")
    if dataset_name == "cocostuff27" and fine_to_coarse is None:
        _fail(who, "cocostuff27 needs Coco's fine_to_coarse mapping {fine id: coarse id}")


def crop_windows(h: int, w: int, crop_type: str, crop_ratio, item: int) -> list:
    """The five (top, left, height, width) windows RandomCropComputer cuts from source image `item` of size h x w, in
    their file order item * 5 + k (src/crop_datasets.py:14-74).  The crop size is (int(h * ratio), int(w * ratio)).

    "five": torchvision's five_crop order top-left, top-right, bottom-left, bottom-right, centre (the centre at
    int(round((side - crop) / 2.0))).  "random": _random_crops(img, size, item, 5): top = hash((item, i, 0)) % (h - ch)
    and left = hash((item, i, 1)) % (w - cw) with this interpreter's hash; a crop as tall or as wide as its image is
    refused there (the reference divides by zero)."""
    who = "crop_windows"
    if crop_type not in CROP_TYPES:
        _fail(who, f"crop_type={crop_type!r} (\"five\" or \"random\")")
    ch, cw = int(h * crop_ratio), int(w * crop_ratio)
    if ch < 1 or cw < 1:
        _fail(who, f"a {h} x {w} image at crop_ratio {crop_ratio} gives an empty {ch} x {cw} crop")
    if ch > h or cw > w:
        _fail(who, f"a {ch} x {cw} crop does not fit a {h} x {w} image")
    if crop_type == "five":
        ct, cl = int(round((h - ch) / 2.0)), int(round((w - cw) / 2.0))
        return [(0, 0, ch, cw), (0, w - cw, ch, cw), (h - ch, 0, ch, cw), (h - ch, w - cw, ch, cw), (ct, cl, ch, cw)]
    if ch == h or cw == w:
        _fail(who, f"a random {ch} x {cw} crop of a {h} x {w} image: the reference's offset draw divides by zero")
    return [(hash((item, i, 0)) % (h - ch), hash((item, i, 1)) % (w - cw), ch, cw) for i in range(CROPS_PER_IMAGE)]


def source_files(root: str, dataset_name: str, image_set: str) -> tuple:
    """(images, labels) of the uncropped set crop_datasets.py reads: Coco(subset None; val: 7) or CityscapesSeg."""
    if dataset_name == "cocostuff27":
        return evalset.coco_files(root, "cocostuff27", image_set)
    return evalset.cityscapes_files(root, image_set)


def cropped_dir(root: str, dataset_name: str, crop_type: str, crop_ratio) -> str:
    return os.path.join(root, "cropped", "{}_{}_crop_{}".format(dataset_name, crop_type, crop_ratio))


class _Writer(Dataset):
    """RandomCropComputer.__getitem__: the five crops of source `item` written as JPEG and label + 1 PNG files."""

    def __init__(self, images, labels, table, crop_type, crop_ratio, img_dir, label_dir):
        self.files = evalset._EvalFiles(images, labels, "pil")
        self.table = table
        self.crop_type, self.crop_ratio, self.img_dir, self.label_dir = crop_type, crop_ratio, img_dir, label_dir

    def __getitem__(self, item):
        img, raw = self.files[item]
        if raw.shape != img.shape[:2]:
            _fail("write_cropped", f"{self.files.labels[item]} is {raw.shape}, its image {img.shape[:2]}")
        label = (self.table[raw] + 1).astype(np.uint8)
        for k, (top, left, h, w) in enumerate(crop_windows(img.shape[0], img.shape[1], self.crop_type,
                                                           self.crop_ratio, item)):
            n = item * CROPS_PER_IMAGE + k
            Image.fromarray(img[top:top + h, left:left + w]).save(os.path.join(self.img_dir, f"{n}.jpg"), "JPEG")
            Image.fromarray(label[top:top + h, left:left + w]).save(os.path.join(self.label_dir, f"{n}.png"), "PNG")
        return True

    def __len__(self):
        return len(self.files)


def write_cropped(root: str, dataset_name: str, crop_type: str, crop_ratio, image_set: str, num_workers: int = 0,
                  fine_to_coarse=None) -> str:
    """Write the tree RandomCropComputer(cfg, dataset_name, image_set, crop_type, crop_ratio) writes, on the host, for
    the reference's own scripts: {root}/cropped/{dataset_name}_{crop_type}_crop_{crop_ratio}/img/{image_set}/{i}.jpg
    (Pillow's default JPEG) and label/{image_set}/{i}.png (uint8 label + 1), i = item * 5 + k.  fine_to_coarse: Coco's
    {fine id: coarse id} table (cocostuff27 only).  Returns the set's directory."""
    who = "write_cropped"
    _check_args(who, dataset_name, crop_type, crop_ratio, fine_to_coarse)
    images, labels = source_files(root, dataset_name, image_set)
    if not images:
        _fail(who, "the listing names no files")
    table = evalset.label_table(dataset_name, fine_to_coarse).numpy()
    base = cropped_dir(root, dataset_name, crop_type, crop_ratio)
    img_dir, label_dir = os.path.join(base, "img", image_set), os.path.join(base, "label", image_set)
    os.makedirs(img_dir, exist_ok=True)
    os.makedirs(label_dir, exist_ok=True)
    writer = _Writer(images, labels, table, crop_type, crop_ratio, img_dir, label_dir)
    for _ in DataLoader(writer, 1, shuffle=False, num_workers=num_workers, collate_fn=_as_list):
        pass
    return base


# ---- the GPU build ------------------------------------------------------------------------------------------------
def _stage(arrays: list, windows: list, tables_of):
    """The pinned staging buffer of stego_jpeg_crops_*: records, tables (one set per distinct key of tables_of), the
    source images.  windows: per crop (source index, top, left, h, w); tables_of(h, w) -> (key, rows, cols) or None.
    Returns (staging, table words, workspace bytes)."""
    C = len(windows)
    tables, table_of = [], {}
    for _, _, _, h, w in windows:
        t = tables_of(h, w)
        if t is not None and t[0] not in table_of:
            table_of[t[0]] = sum(x.size for x in tables)
            tables.extend(t[1:])
    table = np.concatenate(tables).astype(np.int32) if tables else np.zeros(0, dtype=np.int32)
    head = 8 * REC_WORDS * C
    pos = head + 4 * table.size
    offsets = []
    for x in arrays:
        offsets.append(pos)
        pos += x.size
    rec = np.zeros((C, REC_WORDS), dtype=np.int64)
    ws = 0
    for k, (s, top, left, h, w) in enumerate(windows):
        t = tables_of(h, w)
        rec[k] = (offsets[s], arrays[s].shape[0], arrays[s].shape[1], top, left, h, w,
                  table_of[t[0]] if t is not None else 0, ws)
        ws += h * w + 2 * ((h + 1) // 2) * ((w + 1) // 2)
    staging = torch.empty(pos, dtype=torch.uint8, pin_memory=True)
    buf = staging.numpy()
    buf[:head] = rec.reshape(-1).view(np.uint8)
    buf[head:head + 4 * table.size] = table.view(np.uint8)
    for off, x in zip(offsets, arrays):
        buf[off:off + x.size] = x.reshape(-1)
    return staging, table.size, ws


def _run(arrays: list, windows: list, res: int, tables_of, store: torch.Tensor, n: int, r0: int) -> None:
    """Codec and store launches for the crops `windows` of `arrays`, into rows r0 .. of `store` ([n, 3, res, res])."""
    lib = _lib.load()
    dev = frames._require_cuda("crops")
    with torch.cuda.device(dev):
        staging, words, ws_bytes = _stage(arrays, windows, tables_of)
        staged = staging.to(dev, non_blocking=True)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        _lib.check(lib.stego_jpeg_crops_codec(staging.data_ptr(), _lib.ptr(staged), staging.numel(), words,
                                              len(windows), _lib.ptr(ws), ws_bytes, _lib.stream()),
                   "stego_jpeg_crops_codec")
        _lib.check(lib.stego_jpeg_crops_store_rgb8(staging.data_ptr(), _lib.ptr(staged), staging.numel(), words,
                                                   len(windows), res, _lib.ptr(ws), ws_bytes, _lib.ptr(store), n, r0,
                                                   _lib.stream()), "stego_jpeg_crops_store_rgb8")


def jpeg_roundtrip(images, windows) -> list:
    """The decoded crops, as np.asarray(Image.open(jpeg).convert("RGB")) of each crop saved with Pillow's defaults
    returns them, computed by the crop kernels: uint8 [h, w, 3] CUDA tensors, one per (source index, top, left, h, w)
    window of `images` (uint8 H x W x 3 arrays)."""
    arrays = frames._as_arrays(images, 3, "jpeg_roundtrip")
    windows = [tuple(int(v) for v in win) for win in windows]
    if not 1 <= len(windows) <= 65535:
        _fail("jpeg_roundtrip", f"{len(windows)} windows (1..65535)")
    for s, top, left, h, w in windows:
        if not 0 <= s < len(arrays):
            _fail("jpeg_roundtrip", f"window of source {s}: there are {len(arrays)} images")
    side = max(max(h, w) for _, _, _, h, w in windows)
    if side > 8192:
        _fail("jpeg_roundtrip", f"a {side}-pixel window side (up to 8192)")
    dev = frames._require_cuda("jpeg_roundtrip")

    def identity(h, w):  # the crop itself, top-left in a side x side frame
        pad = lambda m: np.concatenate([np.arange(m), np.full(side - m, -1)])
        return (h, w), pad(h), pad(w)

    out = torch.empty(len(windows), 3, side, side, dtype=torch.uint8, device=dev)
    _run(arrays, windows, side, identity, out, len(windows), 0)
    return [out[k, :, :h, :w].permute(1, 2, 0) for k, (_, _, _, h, w) in enumerate(windows)]


def _stage_labels(labels: list, windows: list, res: int):
    """frames._stage's layout for the label crops: each record addresses its source map (stride W) and its tables are
    get_transform's of the crop size shifted by the window's origin (-1 stays -1)."""
    B = len(windows)
    tables, table_of = [], {}
    for s, top, left, h, w in windows:
        if (h, w, top, left) not in table_of:
            rows, cols = frames.index_tables(h, w, res, "center")
            table_of[(h, w, top, left)] = res * len(tables)
            tables.extend([np.where(rows >= 0, rows + top, -1), np.where(cols >= 0, cols + left, -1)])
    table = np.concatenate(tables).astype(np.int32)
    head = 8 * frames.REC_WORDS * B
    pos = head + 4 * table.size
    offsets = []
    for x in labels:
        offsets.append(pos)
        pos += x.size
    staging = torch.empty(pos, dtype=torch.uint8, pin_memory=True)
    buf = staging.numpy()
    rec = np.array([(offsets[s], labels[s].shape[0], labels[s].shape[1], table_of[(h, w, top, left)])
                    for s, top, left, h, w in windows], dtype=np.int64)
    buf[:head] = rec.reshape(-1).view(np.uint8)
    buf[head:head + 4 * table.size] = table.view(np.uint8)
    for off, x in zip(offsets, labels):
        buf[off:off + x.size] = x.reshape(-1)
    return staging, table.size


def _append(store, images: list, labels: list, first_item: int, crop_type: str, crop_ratio) -> None:
    """Rows store.count .. of the five crops of each (image, label) pair, source `first_item + i` for pair i."""
    arrays = frames._as_arrays(images, 3, "ResidentDataset.crops")
    label_arrays = frames._as_arrays(labels, 1, "ResidentDataset.crops")
    windows = []
    for i, (x, y) in enumerate(zip(arrays, label_arrays)):
        if y.shape != x.shape[:2]:
            _fail("ResidentDataset.crops", f"source {first_item + i}: label map {y.shape}, image {x.shape[:2]}")
        windows.extend((i,) + win for win in crop_windows(x.shape[0], x.shape[1], crop_type, crop_ratio,
                                                          first_item + i))
    C = len(windows)
    if store.count + C > store.n:
        _fail("ResidentDataset.crops", f"{C} crops after {store.count} overflow the {store.n}-row store")
    res = store.res

    def gathered(h, w):
        return (h, w), *frames.index_tables(h, w, res, "center")

    _run(arrays, windows, res, gathered, store.images, store.n, store.count)
    lib = _lib.load()
    with torch.cuda.device(store.device):
        staging, words = _stage_labels(label_arrays, windows, res)
        staged = staging.to(store.device, non_blocking=True)
        _lib.check(lib.stego_labels_store_u8(staging.data_ptr(), _lib.ptr(staged), staging.numel(), words, C, res,
                                             _lib.ptr(store.labels), store.n, store.count, _lib.stream()),
                   "stego_labels_store_u8")
    store.count += C


def build_store(cls, root: str, dataset_name: str, crop_type: str, crop_ratio, image_set: str, res: int,
                location: str = "cuda", batch_size: int = 64, num_workers: int = 0, fine_to_coarse=None):
    """ResidentDataset.crops: see there."""
    who = "ResidentDataset.crops"
    _check_args(who, dataset_name, crop_type, crop_ratio, fine_to_coarse)
    batch_size = _check_int(batch_size, "batch_size", 1, 65535, who)
    images, labels = source_files(root, dataset_name, image_set)
    if not images:
        _fail(who, "the listing names no files")
    store = cls(CROPS_PER_IMAGE * len(images), res, "cropped", location)
    store._lut = evalset.label_table(dataset_name, fine_to_coarse).to(store.device)
    # batch_size counts store rows, as for `cropped`: the originals of one build launch cut into about that many crops
    per_launch = max(1, batch_size // CROPS_PER_IMAGE)
    loader = DataLoader(evalset._EvalFiles(images, labels, "pil"), per_launch, shuffle=False, num_workers=num_workers,
                        collate_fn=_as_list)
    item = 0
    for batch in loader:
        _append(store, [b[0] for b in batch], [b[1] for b in batch], item, crop_type, crop_ratio)
        item += len(batch)
    return store
