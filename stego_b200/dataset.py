"""A training set kept resident on the GPU (or in pinned host memory): frames, labels and kNN positives of every step
gathered in one launch, the batches of the reference's training loader bit for bit.

The reference trains from `ContrastiveSegDataset` (src/data.py:419-565) over `CroppedDataset` (the five-crop sets) or
`DirectoryDataset`, read with get_transform(res, ., "center"): a nearest resize and a centre crop, with no randomness.
Its host workers open and decode the anchor and its kNN positive for every sample of every step.  The frames are a
function of the index alone, so `ResidentDataset` decodes each file once, runs the transform once on the GPU (the
gather of stego_b200/frames.py, writing the raw bytes: stego_frames_store_rgb8 / stego_labels_store_u8) and keeps

    images uint8 [n, 3, res, res] and labels uint8 [n, res, res]: 4 * res^2 bytes per sample (200,704 B at 224^2),

on the device (location="cuda") or in pinned host memory read over PCIe (location="host").  Each step is then one
launch (stego_dataset_batch) that gathers the 2B rows of its anchors and positives, normalises the frames with the
arithmetic of load_frames, maps the label bytes through the class's remap and writes its mask.

What is drawn per step is drawn on the host, in the reference's order and from private generators (`Sampler`): the
shuffle order (RandomSampler, or DistributedSampler with set_epoch), and per sample the data set's numpy seed, the
neighbour rank and the aug seed, with the numpy streams of DataLoader(num_workers=W) workers.  The global numpy,
`random` and torch generators never move; in particular torch.manual_seed is never called, so the CUDA generators the
training step's dropout draws from are untouched.

`crop` is the loader's crop (train_config.yml loader_crop_type, get_transform(res, ., crop)): "center" (the default),
None (Resize((res, res)): the image squashed to res x res; fixed rows as for "center") or "random" (Resize(res) then
RandomCrop(res), a window drawn per sample per epoch).  A "random" store keeps each row's whole Resize(res) output
(image uint8 [3, oh, ow], label uint8 [lh, lw]: a ragged layout with a row table of byte offsets and sizes, `sizes`
given up front), and each step's windows are drawn by `Sampler` and cut by the gather (stego_store_batch_window).
"""
from __future__ import annotations

import math
import os

import numpy as np
import torch
from PIL import Image
from torch.utils.data import DataLoader, Dataset

from . import _lib, frames

KINDS = ("cropped", "directory")
LOCATIONS = ("cuda", "host")
MASK_IS_IGNORE, MASK_IS_POSITIVE = 0, 1  # stego_dataset_batch's mask_kind: CroppedDataset's, DirectoryDataset's
SEED_HIGH = 2147483647                    # np.random.randint(2147483647), src/data.py:102, 387, 527
RRC_SCALE, RRC_RATIO = (0.8, 1.0), (3.0 / 4.0, 4.0 / 3.0)  # the geometric aug of src/train_segmentation.py:408-411
REFUSED = {"cocostuff3": "Coco", "cocostuff15": "Coco", "cocostuff27": "Coco (uncropped)", "cityscapes": "CityscapesSeg",
           "potsdam": "Potsdam", "potsdamraw": "PotsdamRaw"}
CROPS = ("center", "random", None)
ROW_WORDS = 6  # the ragged store's row table: image byte offset, oh, ow, label byte offset, lh, lw
WINDOW_WORDS = 5  # stego_store_batch_window's record: row, image top, left, label top, left


def _generate_state(base_seed: int, worker_id: int) -> list:
    """The four uint32 words a DataLoader worker seeds numpy with (torch/utils/data/_utils/worker.py _generate_state,
    a SeedSequence-style hash of [worker_id, base_seed low, base_seed high, 0])."""
    mask = 0xFFFFFFFF
    mult_a, mult_b, mix_l, mix_r, shift = 0x931E8875, 0x58F38DED, 0xCA01F9DD, 0x4973F715, 16
    hash_a = 0x43B0D7E5

    def hashed(value):
        nonlocal hash_a
        value = (value ^ hash_a) & mask
        hash_a = (hash_a * mult_a) & mask
        value = (value * hash_a) & mask
        return (value ^ (value >> shift)) & mask

    def mix(x, y):
        r = (((mix_l * x) & mask) - ((mix_r * y) & mask)) & mask
        return (r ^ (r >> shift)) & mask

    pool = [hashed(v) for v in (worker_id, base_seed & mask, base_seed >> 32, 0)]
    for i_src in range(4):
        for i_dst in range(4):
            if i_src != i_dst:
                pool[i_dst] = mix(pool[i_dst], hashed(pool[i_src]))
    hash_b, state = 0x8B51F9DD, []
    for v in pool:
        v = (v ^ hash_b) & mask
        hash_b = (hash_b * mult_b) & mask
        v = (v * hash_b) & mask
        state.append((v ^ (v >> shift)) & mask)
    return state


def shard(indices: list, rank: int, world_size: int) -> list:
    """Rank `rank`'s share of `indices` as DistributedSampler(drop_last=False) deals it: the list padded with its own
    head to a multiple of world_size, then every world_size-th entry from position rank."""
    total = math.ceil(len(indices) / world_size) * world_size
    pad = total - len(indices)
    indices = indices + (indices[:pad] if pad <= len(indices) else (indices * math.ceil(pad / len(indices)))[:pad])
    return indices[rank:total:world_size]


def _draw_int64(g: torch.Generator) -> int:
    """torch.empty((), dtype=torch.int64).random_(): the DataLoader's base seed and RandomSampler's epoch seed."""
    return int(torch.empty((), dtype=torch.int64).random_(generator=g).item())


def _random_crop(g: torch.Generator, h: int, w: int, res: int) -> tuple:
    """(top, left) of T.RandomCrop(res) on an h x w image (RandomCrop.get_params, src/utils.py:167): nothing drawn when
    the image is already res x res, else randint(0, h - res + 1) then randint(0, w - res + 1), from `g`."""
    if h == res and w == res:
        return 0, 0
    top = int(torch.randint(0, h - res + 1, size=(1,), generator=g))
    return top, int(torch.randint(0, w - res + 1, size=(1,), generator=g))


def _window(g: torch.Generator, seed: int, size, res: int) -> tuple:
    """(top, left, label top, label left) of one sample of a random-crop loader: the class's torch.manual_seed(seed),
    the image's RandomCrop, the reseed, the label's RandomCrop over its own resized size (h, w, lh, lw).  Leaves `g`
    where the label's draws leave the class's generator."""
    g.manual_seed(seed)
    top, left = _random_crop(g, int(size[0]), int(size[1]), res)
    g.manual_seed(seed)
    return (top, left) + _random_crop(g, int(size[2]), int(size[3]), res)


def _after_geometric_aug(seed: int, res: int) -> torch.Tensor:
    """The CPU generator state a single-process reference loader leaves after a sample whose aug seed is `seed`: its
    last draws are the geometric pair on coord (src/data.py:559-560): RandomHorizontalFlip, then RandomResizedCrop on
    [2, res, res].  Made on a forked default generator, so the caller's state is unchanged."""
    import torchvision.transforms as T
    with torch.random.fork_rng(devices=[]):
        torch.default_generator.manual_seed(seed)
        torch.rand(1)
        T.RandomResizedCrop.get_params(torch.empty(1, 1, 1).expand(2, res, res), list(RRC_SCALE), list(RRC_RATIO))
        return torch.get_rng_state()


class Sampler:
    """The host draws of the reference's training loader, `DataLoader(ContrastiveSegDataset(...), batch_size,
    shuffle=True, num_workers=loader_workers)` after seed_everything(seed), per batch: (ind, ind_pos, seed) int64
    arrays.  Iterating gives one iterator per epoch.

    - Order: RandomSampler, seeded per epoch from the main process's torch generator (drawn after the DataLoader
      iterator's base seed); with world_size > 1, DistributedSampler(shuffle=True, seed=seed) with set_epoch(epoch) and
      its padding.  The last batch may be partial.
    - Per sample, from the numpy stream of the process that loads it: dataset[ind]'s np.random.randint, whose
      torch.manual_seed seeds the neighbour rank torch.randint(1, num_neighbors + 1, []); then dataset[ind_pos]'s draw
      and the aug seed.
    - With `sizes` (int [n, 4]: each row's Resize(res) image height, width and label height, width; a random-crop
      loader): dataset[ind]'s image and label RandomCrop draw from its seed before the neighbour rank (`_window`), and
      dataset[ind_pos] draws its own windows from its seed.  Each batch is then (ind, ind_pos, seed, windows), windows
      int64 [2B, 4] (top, left, label top, label left) of the anchors, then of the positives.
    - loader_workers = 0: one numpy stream for the whole run (np.random.seed(seed)), and the main torch generator is
      the one the samples reseed: each epoch's seeds follow the state its last sample's geometric aug draws leave
      (src/train_segmentation.py:408-429).  W >= 1: a fresh worker set per epoch; worker w seeds numpy with
      _generate_state(base_seed, w), and batch i goes to worker i % W.
    """

    def __init__(self, nns, batch_size: int, num_neighbors: int, seed: int, loader_workers: int = 0, rank: int = 0,
                 world_size: int = 1, res: int = 224, sizes=None):
        self.nns = nns
        self.sizes = None if sizes is None else np.asarray(sizes, dtype=np.int64)
        self.n = nns.shape[0]
        self.batch_size, self.num_neighbors, self.seed = batch_size, num_neighbors, seed
        self.workers, self.rank, self.world_size, self.res = loader_workers, rank, world_size, res
        self.main = torch.Generator()
        self.main.manual_seed(seed)
        self.np_main = np.random.RandomState(seed)
        self.epoch = 0
        self._open = None

    def __iter__(self):
        return self

    def __next__(self):
        if self._open is not None and self.workers == 0:
            for _ in self._open:  # the next epoch starts from the state this one's last sample leaves
                pass
        base = _draw_int64(self.main)
        order = self.order()
        self._open = self._epoch(order, base)
        self.epoch += 1
        return self._open

    def order(self) -> list:
        """This epoch's sample order (this rank's share with world_size > 1)."""
        if self.world_size == 1:
            g = torch.Generator()
            g.manual_seed(_draw_int64(self.main))
            return torch.randperm(self.n, generator=g).tolist()
        g = torch.Generator()
        g.manual_seed(self.seed + self.epoch)
        return shard(torch.randperm(self.n, generator=g).tolist(), self.rank, self.world_size)

    def _epoch(self, order: list, base: int):
        B = self.batch_size
        streams = ([self.np_main] if self.workers == 0 else
                   [np.random.RandomState(_generate_state(base, w)) for w in range(self.workers)])
        g = torch.Generator()
        aug_seed = None
        for i, start in enumerate(range(0, len(order), B)):
            rs = streams[i % len(streams)]
            ind = order[start:start + B]
            pos, seeds, windows, windows_pos = [], [], [], []
            for j in ind:
                s = int(rs.randint(SEED_HIGH))
                if self.sizes is None:
                    g.manual_seed(s)
                else:
                    windows.append(_window(g, s, self.sizes[j], self.res))
                k = int(torch.randint(low=1, high=self.num_neighbors + 1, size=[], generator=g))
                pos.append(int(self.nns[j][k]))
                s = int(rs.randint(SEED_HIGH))
                if self.sizes is not None:
                    windows_pos.append(_window(g, s, self.sizes[pos[-1]], self.res))
                aug_seed = int(rs.randint(SEED_HIGH))
                seeds.append(aug_seed)
            if self.workers == 0 and start + B >= len(order):
                self.main.set_state(_after_geometric_aug(aug_seed, self.res))
            batch = (np.asarray(ind, dtype=np.int64), np.asarray(pos, dtype=np.int64), np.asarray(seeds, dtype=np.int64))
            if self.sizes is not None:
                batch += (np.asarray(windows + windows_pos, dtype=np.int64).reshape(-1, 4),)
            yield batch


def _check_int(value, name: str, lo: int, hi: int, who: str) -> int:
    if isinstance(value, bool) or not isinstance(value, (int, np.integer)) or not lo <= value <= hi:
        raise ValueError(f"stego_b200.dataset.{who}: {name}={value!r} (an int in {lo}..{hi})")
    return int(value)


class _Files(Dataset):
    """(image array, label array or None) per index, decoded as the reference's class opens them."""

    def __init__(self, images: list, labels, convert: bool):
        self.images, self.labels, self.convert = images, labels, convert

    def __getitem__(self, index):
        with Image.open(self.images[index]) as im:
            img = np.asarray(im.convert("RGB") if self.convert else im)
        if self.labels is None:
            return img, None
        with Image.open(self.labels[index]) as im:
            return img, np.asarray(im)

    def __len__(self):
        return len(self.images)


def _as_list(batch):
    return batch


def image_size(path: str) -> tuple:
    """(height, width) of an image file from its header, without decoding it."""
    with Image.open(path) as im:
        return im.size[1], im.size[0]


def source_sizes(images: list, labels) -> np.ndarray:
    """int64 [n, 4]: each image's height, width and its label map's (the image's without labels), from the headers:
    the row sizes a crop="random" store is made with."""
    out = []
    for k, path in enumerate(images):
        h, w = image_size(path)
        out.append((h, w) + (image_size(labels[k]) if labels is not None else (h, w)))
    return np.array(out, dtype=np.int64).reshape(-1, 4)


def _pinned_or_device(location: str, device, shape) -> torch.Tensor:
    if location == "cuda":
        return torch.empty(shape, dtype=torch.uint8, device=device)
    return torch.empty(shape, dtype=torch.uint8, pin_memory=True)


class _Store:
    """n samples in device or pinned host memory, filled in order by `append` and read by one gather launch per batch:
    what ResidentDataset and evalset.EvalSet share.  crop "center" / None: uint8 rows of res x res frames [n, 3, res,
    res] and label maps [n, res, res].  crop "random": each row's whole Resize(res) output at its byte offset in one
    flat image store and one flat label store, described by the pinned row table `rows` int64 [n, 6] (image offset,
    oh, ow, label offset, lh, lw).  A subclass sets the batch entry, its mask rule and the label table, and calls
    _allocate once its own arguments are checked."""

    _PREFIX = "stego_b200.dataset"
    _ENTRY = "stego_dataset_batch"

    def _allocate(self, n: int, res: int, location: str, has_labels: bool, lut: torch.Tensor, crop="center",
                  sizes=None) -> None:
        who = type(self).__name__
        if crop not in CROPS:
            raise ValueError(f"{self._PREFIX}.{who}: crop={crop!r} (\"center\", \"random\" or None)")
        self.n, self.res, self.location, self.has_labels, self.crop = n, res, location, bool(has_labels), crop
        self.device = frames._require_cuda(who)
        self.sizes = self.rows = None
        if crop == "random":
            self._allocate_ragged(sizes, who)
        else:
            if sizes is not None:
                raise ValueError(f"{self._PREFIX}.{who}: sizes are for crop=\"random\" (a ragged store) only")
            self.images = _pinned_or_device(location, self.device, (n, 3, res, res))
            self.labels = _pinned_or_device(location, self.device, (n, res, res)) if has_labels else None
        self._lut = lut.to(self.device)
        self.count = 0
        # pinned index records, used in turn: one is refilled once the launch that read it two steps earlier has run
        self._ring = [torch.empty(0, dtype=torch.int64), torch.empty(0, dtype=torch.int64)]
        self._ring_done = [None, None]
        self._slot = 0

    def _allocate_ragged(self, sizes, who: str) -> None:
        """The row table from each row's source sizes (H, W, label H, label W) and the flat stores, each rounded up to
        a multiple of 16 bytes (the gather's aligned loads stay inside)."""
        src = np.asarray(sizes, dtype=np.int64) if sizes is not None else None
        if src is None or src.shape != (self.n, 4) or (src < 1).any() or (src > 1 << 20).any():
            raise ValueError(f"{self._PREFIX}.{who}: crop=\"random\" needs sizes, int [n={self.n}, 4]: each row's "
                             f"image height, width and label height, width (1..2^20)")
        out = np.array([frames.output_size(int(h), int(w), self.res, "center") +
                        frames.output_size(int(lh), int(lw), self.res, "center") for h, w, lh, lw in src], np.int64)
        self._source_sizes, self.sizes = src, out
        img_bytes = 3 * out[:, 0] * out[:, 1]
        lab_bytes = out[:, 2] * out[:, 3] if self.has_labels else np.zeros(self.n, np.int64)
        self.rows = torch.empty(self.n, ROW_WORDS, dtype=torch.int64, pin_memory=True)
        rows = self.rows.numpy()
        rows[:, 0] = np.cumsum(img_bytes) - img_bytes
        rows[:, 1:3] = out[:, 0:2]
        rows[:, 3] = np.cumsum(lab_bytes) - lab_bytes
        rows[:, 4:6] = out[:, 2:4]
        round16 = lambda v: max(16, (int(v) + 15) // 16 * 16)  # noqa: E731
        self.images = _pinned_or_device(self.location, self.device, (round16(img_bytes.sum()),))
        self.labels = (_pinned_or_device(self.location, self.device, (round16(lab_bytes.sum()),))
                       if self.has_labels else None)

    @property
    def nbytes(self) -> int:
        return self.images.numel() + (self.labels.numel() if self.labels is not None else 0)

    def append(self, images, labels=None) -> None:
        """Transform and store the next len(images) samples: images as load_frames takes them (uint8 H x W x 3), labels
        as load_labels (uint8 H x W), one per image (None without labels); with crop="random", of the sizes the store
        was made with.  One build launch per store; the caller is not synchronised."""
        who = f"{type(self).__name__}.append"
        arrays = frames._as_arrays(images, 3, who)
        if self.has_labels:
            if labels is None:
                raise ValueError(f"{self._PREFIX}.{who}: this store keeps labels; pass one label map per image")
            label_arrays = frames._as_arrays(labels, 1, who)
            if len(label_arrays) != len(arrays):
                raise ValueError(f"{self._PREFIX}.{who}: {len(label_arrays)} label maps for {len(arrays)} images")
        elif labels is not None:
            raise ValueError(f"{self._PREFIX}.{who}: this store was made with has_labels=False")
        B = len(arrays)
        if self.count + B > self.n:
            raise ValueError(f"{self._PREFIX}.{who}: {B} samples after {self.count} overflow the {self.n}-row store")
        lib = _lib.load()
        with torch.cuda.device(self.device):
            if self.crop == "random":
                for k, x in enumerate(arrays):
                    want = self._source_sizes[self.count + k]
                    got = x.shape[:2] + (label_arrays[k].shape if self.has_labels else tuple(want[2:]))
                    if tuple(int(v) for v in want) != tuple(got):
                        raise ValueError(f"{self._PREFIX}.{who}: sample {self.count + k} is {got[0]} x {got[1]} with a "
                                         f"{got[2]} x {got[3]} label; the store was made for {tuple(want)}")
                rows = self.rows.numpy()[self.count:self.count + B]
                parts = [(arrays, self.images, rows[:, 0], 3)]
                if self.has_labels:
                    parts.append((label_arrays, self.labels, rows[:, 3], 1))
                for items, store, dest, channels in parts:
                    staging, words, _ = frames._stage(items, self.res, "random", dest=dest)
                    staged = staging.to(self.device, non_blocking=True)
                    _lib.check(lib.stego_store_rows_u8(staging.data_ptr(), _lib.ptr(staged), staging.numel(), words,
                                                       B, channels, _lib.ptr(store), store.numel(), _lib.stream()),
                               "stego_store_rows_u8")
            else:
                staging, words, _ = frames._stage(arrays, self.res, self.crop)
                staged = staging.to(self.device, non_blocking=True)
                _lib.check(lib.stego_frames_store_rgb8(staging.data_ptr(), _lib.ptr(staged), staging.numel(), words,
                                                       B, self.res, _lib.ptr(self.images), self.n, self.count,
                                                       _lib.stream()), "stego_frames_store_rgb8")
                if self.has_labels:
                    staging, words, _ = frames._stage(label_arrays, self.res, self.crop)
                    staged = staging.to(self.device, non_blocking=True)
                    _lib.check(lib.stego_labels_store_u8(staging.data_ptr(), _lib.ptr(staged), staging.numel(), words,
                                                         B, self.res, _lib.ptr(self.labels), self.n, self.count,
                                                         _lib.stream()), "stego_labels_store_u8")
        self.count += B

    def _fill(self, files: Dataset, batch_size: int, num_workers: int) -> None:
        """Append every (image, label or None) item of `files`, decoded in DataLoader(num_workers) workers."""
        loader = DataLoader(files, batch_size, shuffle=False, num_workers=num_workers, collate_fn=_as_list)
        for batch in loader:
            self.append([b[0] for b in batch], [b[1] for b in batch] if self.has_labels else None)

    # ---- reading --------------------------------------------------------------------------------------------------
    def _require_full(self, who: str) -> None:
        if self.count != self.n:
            raise ValueError(f"{self._PREFIX}.{who}: the store holds {self.count} of its {self.n} samples")

    def _record(self, index: np.ndarray) -> torch.Tensor:
        """The next pinned record holding `index` (int64, any shape), reused once the launch that read it last has
        run."""
        if self._ring[0].numel() < index.size:  # both records grow together, once their readers have run
            for j in (0, 1):
                if self._ring_done[j] is not None:
                    self._ring_done[j].synchronize()
                self._ring[j] = torch.empty(index.size, dtype=torch.int64, pin_memory=True)
        i = self._slot
        self._slot ^= 1
        if self._ring_done[i] is not None:
            self._ring_done[i].synchronize()
        self._ring[i].numpy()[:index.size] = index.reshape(-1)
        return i

    def center_windows(self, index: np.ndarray) -> np.ndarray:
        """int64 [len(index), 4]: the CenterCrop(res) window (top, left, label top, label left) of each row of a
        crop="random" store: what get_transform(res, ., "center") reads of its Resize(res) output."""
        out = self.sizes[index]
        return np.array([frames.crop_offsets(h, w, self.res) + frames.crop_offsets(lh, lw, self.res)
                         for h, w, lh, lw in out], dtype=np.int64).reshape(-1, 4)

    def _gather(self, index: np.ndarray, dtype, windows: np.ndarray = None) -> tuple:
        """(img, label, mask) of the store rows `index`, one launch on the current stream.  A crop="random" store reads
        the res x res window (top, left, label top, label left) `windows[s]` of each row, their centres by default."""
        count, res = index.size, self.res
        with torch.cuda.device(self.device):
            if self.crop == "random":
                if windows is None:
                    windows = self.center_windows(index)
                i = self._record(np.concatenate([index.reshape(-1, 1), windows], 1).astype(np.int64))
            else:
                i = self._record(index)
            img = torch.empty(count, 3, res, res, dtype=dtype, device=self.device)
            label = torch.empty(count, res, res, dtype=torch.int64, device=self.device)
            mask_dtype = torch.float32 if self._mask_kind == MASK_IS_POSITIVE else torch.bool
            mask = torch.empty(count, res, res, dtype=mask_dtype, device=self.device)
            lib = _lib.load()
            outputs = (*frames.MEAN, *frames.STD, int(dtype == torch.bfloat16), self._mask_kind, _lib.ptr(img),
                       _lib.ptr(label), _lib.ptr(mask), _lib.stream())
            if self.crop == "random":
                labels = self.labels
                _lib.check(lib.stego_store_batch_window(
                    _lib.ptr(self.images), self.images.numel(), _lib.ptr(labels),
                    0 if labels is None else labels.numel(), self.rows.data_ptr(), self.n, res,
                    self._ring[i].data_ptr(), count, _lib.ptr(self._lut), *outputs), "stego_store_batch_window")
            else:
                _lib.check(getattr(lib, self._ENTRY)(
                    _lib.ptr(self.images), _lib.ptr(self.labels), self.n, res, self._ring[i].data_ptr(), count,
                    _lib.ptr(self._lut), *outputs), self._ENTRY)
            done = torch.cuda.Event()
            done.record()
            self._ring_done[i] = done
        return img, label, mask

    def _check_dtype(self, dtype, who: str) -> None:
        if dtype not in (torch.float32, torch.bfloat16):
            raise ValueError(f"{self._PREFIX}.{who}: dtype={dtype} (torch.float32 or torch.bfloat16)")

    def batches(self, nns, batch_size: int, num_neighbors: int, seed: int, loader_workers: int = 0, rank: int = 0,
                world_size: int = 1, dtype=torch.float32, res: int = None):
        """The training loader: an iterator over epochs, each yielding the dicts training_step takes, those of
        DataLoader(ContrastiveSegDataset(..., mask=True, pos_images=True, pos_labels=True), batch_size, shuffle=True,
        num_workers=loader_workers) after seed_everything(seed) (the draws: `Sampler`), read with the store's crop.

        ind, ind_pos (int64) and seed (B aug seeds, int64, from which the fused step builds the aug views) are CPU
        tensors; img, img_pos (dtype), label, label_pos, mask and mask_pos are on the store's device, in the class's
        per-sample shapes, one launch per step on the current stream with fresh outputs.  The host runs at most two
        steps ahead of the device.

        nns: the kNN table [n, k] (precompute_knns), host array or tensor; num_neighbors 1 .. k - 1.  res, if given,
        must be the store's."""
        who = f"{type(self).__name__}.batches"
        self._require_full(who)
        if res is not None and res != self.res:
            raise ValueError(f"{self._PREFIX}.{who}: res={res!r} but the store holds {self.res}^2 frames")
        self._check_dtype(dtype, who)
        nns = np.asarray(nns.detach().cpu() if isinstance(nns, torch.Tensor) else nns)
        if nns.ndim != 2 or not np.issubdtype(nns.dtype, np.integer):
            raise ValueError(f"{self._PREFIX}.{who}: nns must be an integer table [n, k], got {nns.dtype} "
                             f"{nns.shape}")
        if nns.shape[0] != self.n:
            raise ValueError(f"{self._PREFIX}.{who}: nns has {nns.shape[0]} rows for a {self.n}-sample store")
        if nns.size and (nns.min() < 0 or nns.max() >= self.n):
            raise ValueError(f"{self._PREFIX}.{who}: nns holds indices outside 0..{self.n - 1}")
        if nns.shape[1] < 2:
            raise ValueError(f"{self._PREFIX}.{who}: nns has {nns.shape[1]} column(s); a positive needs 2 or more")
        batch_size = _check_int(batch_size, "batch_size", 1, 32767, who)
        num_neighbors = _check_int(num_neighbors, "num_neighbors", 1, nns.shape[1] - 1, who)
        seed = _check_int(seed, "seed", 0, (1 << 32) - 1, who)
        loader_workers = _check_int(loader_workers, "loader_workers", 0, 1024, who)
        world_size = _check_int(world_size, "world_size", 1, 1 << 20, who)
        rank = _check_int(rank, "rank", 0, world_size - 1, who)
        sampler = Sampler(nns, batch_size, num_neighbors, seed, loader_workers, rank, world_size, self.res,
                          self.sizes if self.crop == "random" else None)
        for epoch in sampler:
            yield self._epoch(epoch, dtype)

    def _epoch(self, plan, dtype):
        for ind, pos, seeds, *windows in plan:
            B = ind.size
            img, label, mask = self._gather(np.concatenate([ind, pos]), dtype, *windows)
            label, mask = self._shaped(label, mask)
            yield dict(ind=torch.from_numpy(ind), img=img[:B], img_pos=img[B:], ind_pos=torch.from_numpy(pos),
                       label=label[:B], label_pos=label[B:], mask=mask[:B], mask_pos=mask[B:],
                       seed=torch.from_numpy(seeds))


class ResidentDataset(_Store):
    """The training set of a CroppedDataset (kind="cropped") or DirectoryDataset (kind="directory") resident in memory.

    n samples at res: 4 * res^2 bytes each (3 * res^2 of image, res^2 of label), 200,704 B at 224^2.  location="cuda"
    keeps them in device memory, location="host" in pinned host memory that the batch kernel reads over PCIe; the
    caller chooses from the set's size.  Rows are filled in order by `append` (or the `cropped` / `directory`
    constructors); `frames` and `batches` need all n."""

    def __init__(self, n: int, res: int, kind: str = "cropped", location: str = "cuda", has_labels: bool = True,
                 crop="center", sizes=None):
        who = "ResidentDataset"
        if kind in REFUSED:
            raise ValueError(f"stego_b200.dataset.{who}: {kind!r} is read by {REFUSED[kind]}, which is not a training "
                             f"set class of this store; EvalSet.{'coco' if 'Coco' in REFUSED[kind] else kind}(..., "
                             f"\"train\", ...) (stego_b200.evalset) holds and trains from it")
        if kind not in KINDS:
            raise ValueError(f"stego_b200.dataset.{who}: kind={kind!r} (\"cropped\" or \"directory\")")
        if location not in LOCATIONS:
            raise ValueError(f"stego_b200.dataset.{who}: location={location!r} (\"cuda\" or \"host\")")
        if kind == "cropped" and not has_labels:
            raise ValueError(f"stego_b200.dataset.{who}: a CroppedDataset always has labels")
        n = _check_int(n, "n", 1, 1 << 40, who)
        res = _check_int(res, "res", 1, 8192, who)
        self.kind = kind
        self._mask_kind = MASK_IS_IGNORE if kind == "cropped" else MASK_IS_POSITIVE
        # CroppedDataset: label = byte - 1; DirectoryDataset: the byte, or -1 everywhere without a label folder
        ids = torch.arange(256, dtype=torch.int64)
        lut = ids - 1 if kind == "cropped" else (ids if has_labels else torch.full((256,), -1, dtype=torch.int64))
        self._allocate(n, res, location, has_labels, lut, crop, sizes)

    @classmethod
    def _from_files(cls, images, labels, convert, res, kind, location, batch_size, num_workers, crop):
        sizes = source_sizes(images, labels) if crop == "random" else None
        store = cls(len(images), res, kind, location, labels is not None, crop, sizes)
        store._fill(_Files(images, labels, convert), batch_size, num_workers)
        return store

    @classmethod
    def cropped(cls, root: str, dataset_name: str, crop_type: str, crop_ratio, image_set: str, res: int,
                location: str = "cuda", batch_size: int = 64, num_workers: int = 0, crop="center") -> "ResidentDataset":
        """CroppedDataset(root, dataset_name, crop_type, crop_ratio, image_set, ...) (src/data.py:370-400): the files
        {root}/cropped/{dataset_name}_{crop_type}_crop_{crop_ratio}/img/{image_set}/{i}.jpg (converted to RGB) and
        label/{image_set}/{i}.png, decoded once in DataLoader(num_workers) workers.  crop: the loader's
        (get_transform(res, ., crop))."""
        base = os.path.join(root, "cropped", "{}_{}_crop_{}".format(dataset_name, crop_type, crop_ratio))
        img_dir, label_dir = os.path.join(base, "img", image_set), os.path.join(base, "label", image_set)
        n = len(os.listdir(img_dir))
        if n != len(os.listdir(label_dir)):
            raise ValueError(f"stego_b200.dataset.ResidentDataset.cropped: {n} images but "
                             f"{len(os.listdir(label_dir))} label files under {base}")
        images = [os.path.join(img_dir, f"{i}.jpg") for i in range(n)]
        labels = [os.path.join(label_dir, f"{i}.png") for i in range(n)]
        return cls._from_files(images, labels, True, res, "cropped", location, batch_size, num_workers, crop)

    @classmethod
    def crops(cls, root: str, dataset_name: str, crop_type: str, crop_ratio, image_set: str, res: int,
              location: str = "cuda", batch_size: int = 64, num_workers: int = 0,
              fine_to_coarse=None, crop="center") -> "ResidentDataset":
        """The store `cropped(root, dataset_name, crop_type, crop_ratio, image_set, res, location)` reads from the tree
        the reference's crop_datasets.py writes, built straight from the uncropped originals (stego_b200/crops.py):
        dataset_name "cocostuff27" (Coco, subset None; val: 7) or "cityscapes" (CityscapesSeg), crop_type "five" or
        "random".  Each original is decoded once in DataLoader(num_workers) workers, max(1, batch_size // 5) originals
        (their 5x crops: about batch_size rows) per build launch; its five crops go through the JPEG round trip of
        Pillow's default save and decode on the GPU.  The
        rows, frames() and batches() equal those of `cropped` on the written tree byte for byte; the label rows hold
        the source's raw bytes, read through the class's table.  fine_to_coarse: Coco's {fine id: coarse id} table
        (cocostuff27 only).  crop: "center" only; a crop keeps its original's aspect, so its Resize(res) output is not
        res x res, and the JPEG rebuild writes the centre window alone (train with "random" or None from `cropped`
        on the written tree)."""
        if crop != "center":
            raise ValueError(f"stego_b200.dataset.ResidentDataset.crops: crop={crop!r}; this builder writes the "
                             f"\"center\" rows only (cropped(..., crop=...) reads the written tree with any crop)")
        from . import crops
        return crops.build_store(cls, root, dataset_name, crop_type, crop_ratio, image_set, res, location, batch_size,
                                 num_workers, fine_to_coarse)

    @classmethod
    def directory(cls, root: str, path: str, image_set: str, res: int, location: str = "cuda", batch_size: int = 64,
                  num_workers: int = 0, crop="center") -> "ResidentDataset":
        """DirectoryDataset(root, path, image_set, ...) (src/data.py:75-118): sorted listdir of {root}/{path}/imgs/
        {image_set} and, when {root}/{path}/labels exists, of labels/{image_set}; the images are read as they are
        (no convert), so they must decode to RGB."""
        base = os.path.join(root, path)
        img_dir, label_dir = os.path.join(base, "imgs", image_set), os.path.join(base, "labels", image_set)
        names = sorted(os.listdir(img_dir))
        if not names:
            raise ValueError(f"stego_b200.dataset.ResidentDataset.directory: no images in {img_dir}")
        labels = None
        if os.path.exists(os.path.join(base, "labels")):
            label_names = sorted(os.listdir(label_dir))
            if len(label_names) != len(names):
                raise ValueError(f"stego_b200.dataset.ResidentDataset.directory: {len(names)} images but "
                                 f"{len(label_names)} label files")
            labels = [os.path.join(label_dir, f) for f in label_names]
        images = [os.path.join(img_dir, f) for f in names]
        return cls._from_files(images, labels, False, res, "directory", location, batch_size, num_workers, crop)

    def _shaped(self, label, mask):
        """The shapes the reference's classes return, batched: CroppedDataset label [B, res, res] and mask
        [B, 1, res, res]; DirectoryDataset label and mask [B, 1, res, res] with a label folder, [B, res, res] without."""
        B, res = label.shape[0], self.res
        if self.kind == "cropped":
            return label, mask.view(B, 1, res, res)
        if self.has_labels:
            return label.view(B, 1, res, res), mask.view(B, 1, res, res)
        return label, mask

    def frames(self, batch_size: int, dtype=torch.float32, rank: int = 0, world_size: int = 1):
        """Batches {"img", "label", "mask"} of the samples in index order: get_transform(res, ., "center") of each
        image (of crop None: its squashed frame), as a shuffle=False loader yields them (precompute_knns(net,
        store.frames(b)) runs on them unchanged; a crop="random" store yields the centre windows).
        With world_size > 1, rank `rank`'s samples of DistributedSampler(shuffle=False), padding included."""
        who = "ResidentDataset.frames"
        self._require_full(who)
        batch_size = _check_int(batch_size, "batch_size", 1, 65535, who)
        self._check_dtype(dtype, who)
        world_size = _check_int(world_size, "world_size", 1, 1 << 20, who)
        rank = _check_int(rank, "rank", 0, world_size - 1, who)
        order = np.asarray(shard(list(range(self.n)), rank, world_size), dtype=np.int64)
        for start in range(0, order.size, batch_size):
            img, label, mask = self._gather(order[start:start + batch_size], dtype)
            label, mask = self._shaped(label, mask)
            yield dict(img=img, label=label, mask=mask)
