"""Generate tests/golden/uncropped.pt from the REAL reference training loader on the uncropped classes:
ContrastiveSegDataset (src/data.py:419-565) with crop_type=None over Coco (cocostuff27 "train"), CityscapesSeg "train",
Potsdam "train" and a DirectoryDataset, with the transforms my_app builds (src/train_segmentation.py:408-434) and
get_transform(res, ., loader_crop_type) for loader_crop_type "center", "random" and None, under
DataLoader(batch_size=4, shuffle=True, num_workers=W) for W = 0 and 2, at res 32 and 30, on the CPU.

    STEGO_REFERENCE_SRC=<reference checkout>/src python oracle/make_golden_uncropped.py

The input is a seeded synthetic tree in each class's layout (make_golden_evalset's file writers) holding the same 6
images and label maps (label bytes 0..40), of mixed aspect (portrait and landscape) with one 16 x 16 image, whose
Resize(res) output is exactly res x res at res 32 (the branch where RandomCrop draws nothing), and one directory sample
whose label map is smaller than its image.  Each run
seeds torch, numpy and random with SEED and reads 2.5 epochs.  A subclass records the aug seed each __getitem__ passes
to _set_seed, and the (top, left) every RandomCrop.get_params call returns inside that __getitem__ (anchor image, its
label, positive image, its label); it drops img_aug / coord_aug.  Everything else is the reference's own code.

The fixture stays small: the classes share their images, so the img rows are kept once per res, as bytes of `values`
(make_golden_evalset.as_bytes), in frames[res]["full"] (a list of [3, oh, ow]) and frames[res]["squashed"] (a list of
[3, res, res]), and equal PNG files are one bytes object in `tree`.  Labels are int8 and masks packed bits.

Stored per case f"{layout}_{res}":
  * full: per index the reference's Resize(res) output without a crop (the same ContrastiveSegDataset with the cropper
    left out): img_index (its entry of frames[res]["full"]), label (int8, with label_dtype) and mask (np.packbits of
    the 0 / 1 mask, with mask_shape and mask_dtype), each in the class's per-sample shape; squashed: the same of the
    crop None runs' rows (img_index into frames[res]["squashed"]);
  * paths: CityscapesSeg's image paths in the reference's order (os.listdir's; None for the other classes);
  * runs[(crop, W)]: sizes (samples per batch) and draws int64 [samples, 11]: ind, ind_pos, seed, then the anchor's
    (top, left, label top, label left) and the positive's (zeros for "center" and None).
Every batch is checked here to equal the gather of those rows: the windows of `full` ("random"; "center": the
CenterCrop offsets), or the rows of `squashed` (None).
"""
from __future__ import annotations

import os
import random
import sys
import tempfile
from types import SimpleNamespace

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import reference_shim  # noqa: E402
from make_golden_evalset import _mat, as_bytes, value_table  # noqa: E402
from make_golden_evalset import _png as _png_bytes  # noqa: E402
from make_golden_frames import _import_reference_loaders  # noqa: E402

OUT = os.path.join(HERE, "..", "tests", "golden", "uncropped.pt")
N, K, NUM_NEIGHBORS, BATCH, SEED = 6, 4, 3, 4, 11
RESOLUTIONS = (32, 30)
WORKERS = (0, 2)
CROPS = ("center", "random", None)
LAYOUTS = ("cocostuff27", "cityscapes", "potsdam", "directory")
SIZES = [(16, 16), (40, 21), (19, 45), (33, 70), (64, 30), (25, 25)]  # (H, W); the first is res x res at 32


def tree():
    rng = np.random.default_rng(77)
    files = {}
    samples = [(rng.integers(0, 256, (H, W, 3), dtype=np.uint8), rng.integers(0, 41, (H, W), dtype=np.uint8))
               for H, W in SIZES]
    pngs = {}

    def _png(arr, mode=None):  # one bytes object per distinct file, so the fixture holds it once
        key = (arr.tobytes(), arr.shape, mode)
        if key not in pngs:
            pngs[key] = _png_bytes(arr, mode)
        return pngs[key]

    def sample(k):
        return samples[k]

    ids = [f"00000001{k:04d}" for k in range(N)]
    for k, img_id in enumerate(ids):
        img, lab = sample(k)
        files[f"cocostuff/images/train2017/{img_id}.jpg"] = _png(img)
        files[f"cocostuff/annotations/train2017/{img_id}.png"] = _png(lab, "L")
    files["cocostuff/curated/train2017/Coco164kFull_Stuff_Coarse.txt"] = "\n".join(ids).encode() + b"\n"
    for k in range(N):
        img, lab = sample(k)
        city = ("aachen", "bonn")[k % 2]
        stem = f"{city}_{k:06d}_000019"
        files[f"cityscapes/leftImg8bit/train/{city}/{stem}_leftImg8bit.png"] = _png(img)
        files[f"cityscapes/gtFine/train/{city}/{stem}_gtFine_labelIds.png"] = _png(lab, "L")
    pids = [f"top_potsdam_2_{k}_RGBIR_{k}" for k in range(N)]
    for k, pid in enumerate(pids):
        img, lab = sample(k)
        ir = rng.integers(0, 256, img.shape[:2] + (1,), dtype=np.uint8)
        files[f"potsdam/imgs/{pid}.mat"] = _mat("img", np.concatenate([img, ir], 2))
        if k != 4:
            files[f"potsdam/gt/{pid}.mat"] = _mat("gt", (lab % 7).astype(np.uint8))
    files["potsdam/labelled_train.txt"] = "\n".join(pids).encode() + b"\n"
    for k in range(N):
        img, lab = sample(k)
        if k == 3:  # a label map of its own size
            lab = rng.integers(0, 28, (26, 51), dtype=np.uint8)
            files[f"myset/labels/train/im{k:02d}.png"] = _png(lab, "L")
        else:
            files[f"myset/labels/train/im{k:02d}.png"] = _png(lab % 28, "L")
        files[f"myset/imgs/train/im{k:02d}.png"] = _png(img)
    return files


def nns_table():
    rng = np.random.default_rng(5)
    nns = np.zeros((N, K), dtype=np.int64)
    for i in range(N):
        nns[i] = [i] + list(rng.permutation([j for j in range(N) if j != i])[:K - 1])
    return nns


def make_dataset(data, utils, root, layout, res, img_t, lab_t, cfg, record):
    import torchvision.transforms as T

    class Recording(data.ContrastiveSegDataset):
        def _set_seed(self, seed):
            self.last_seed = seed
            super()._set_seed(seed)

        def __getitem__(self, ind):
            windows = []
            original = T.RandomCrop.get_params

            def get_params(img, output_size):
                i, j, h, w = original(img, output_size)
                windows.extend((i, j))
                return i, j, h, w

            T.RandomCrop.get_params = staticmethod(get_params)
            try:
                ret = super().__getitem__(ind)
            finally:
                T.RandomCrop.get_params = staticmethod(original)
            ret.pop("img_aug", None)
            ret.pop("coord_aug", None)
            ret["seed"] = self.last_seed
            ret["win"] = torch.tensor(windows + [0] * (8 - len(windows)), dtype=torch.int64)
            return ret

    geometric = T.Compose([T.RandomHorizontalFlip(), T.RandomResizedCrop(size=res, scale=(0.8, 1.0))])
    photometric = T.Compose([T.ColorJitter(brightness=.3, contrast=.3, saturation=.3, hue=.1), T.RandomGrayscale(.2),
                             T.RandomApply([T.GaussianBlur((5, 5))])])
    kw = dict(aug_geometric_transform=geometric, aug_photometric_transform=photometric, num_neighbors=NUM_NEIGHBORS,
              pos_images=True, pos_labels=True) if record else {}
    return Recording(pytorch_data_dir=root, dataset_name=layout, crop_type=None, image_set="train", transform=img_t,
                     target_transform=lab_t, cfg=cfg, mask=True, **kw)


def run(ds):
    from torch.utils.data import DataLoader
    batches = []
    for W in WORKERS:
        random.seed(SEED)
        np.random.seed(SEED)
        torch.manual_seed(SEED)
        loader = DataLoader(ds, BATCH, shuffle=True, num_workers=W)
        out = []
        per_epoch = -(-N // BATCH)
        for epoch in range(3):
            for i, b in enumerate(loader):
                if epoch == 2 and i == per_epoch // 2:
                    break
                out.append(b)
        batches.append(out)
    return batches


def main():
    if not reference_shim.available():
        raise RuntimeError("set STEGO_REFERENCE_SRC to the reference's src directory")
    import torchvision.transforms as T
    from PIL import Image
    utils, data = _import_reference_loaders()
    files, nns = tree(), nns_table()
    values = value_table(utils)
    cases, frames = {}, {res: dict(full=[], squashed=[]) for res in RESOLUTIONS}

    def frame_index(res, part, row):
        """The entry of frames[res][part] equal to the bytes of `row`, appended if new."""
        b = as_bytes(row, values)
        for k, known in enumerate(frames[res][part]):
            if known.shape == b.shape and torch.equal(known, b):
                return k
        frames[res][part].append(b)
        return len(frames[res][part]) - 1

    def rows_of(imgs, labels, masks, res, part):
        assert all(lab.min() >= -128 and lab.max() < 128 for lab in labels)
        assert all(((m == 0) | (m == 1)).all() for m in masks)
        return dict(img_index=torch.tensor([frame_index(res, part, x) for x in imgs], dtype=torch.int64),
                    label=[lab.to(torch.int8) for lab in labels], mask_shape=[tuple(m.shape) for m in masks],
                    mask=[torch.from_numpy(np.packbits(m.to(torch.bool).numpy().reshape(-1))) for m in masks],
                    label_dtype=str(labels[0].dtype).replace("torch.", ""),
                    mask_dtype=str(masks[0].dtype).replace("torch.", ""))
    with tempfile.TemporaryDirectory() as root:
        for rel, blob in files.items():
            os.makedirs(os.path.dirname(os.path.join(root, rel)), exist_ok=True)
            with open(os.path.join(root, rel), "wb") as f:
                f.write(blob)
        os.makedirs(os.path.join(root, "nns"), exist_ok=True)
        for layout in LAYOUTS:
            for res in RESOLUTIONS:
                cfg = SimpleNamespace(model_type="vit_small", res=res, dir_dataset_name="myset",
                                      dir_dataset_n_classes=27, crop_ratio=0.5, crop_type=None)
                name = "myset" if layout == "directory" else layout
                np.savez_compressed(os.path.join(root, "nns", f"nns_vit_small_{name}_train_None_{res}.npz"), nns=nns)
                # the Resize(res) output of each index, no crop
                full_ds = make_dataset(data, utils, root, layout, res,
                                       T.Compose([T.Resize(res, Image.NEAREST), T.ToTensor(), utils.normalize]),
                                       T.Compose([T.Resize(res, Image.NEAREST), utils.ToTargetTensor()]), cfg, False)
                full = [full_ds[i] for i in range(N)]
                # CityscapesSeg lists its files with os.listdir: the order this file system gave, kept with the rows
                images = full_ds.dataset.inner_loader.images if layout == "cityscapes" else None
                case = dict(full=rows_of([f["img"] for f in full], [f["label"] for f in full],
                                         [f["mask"] for f in full], res, "full"), runs={},
                            paths=None if images is None else [os.path.relpath(p, root) for p in images])
                squashed = None
                for crop in CROPS:
                    ds = make_dataset(data, utils, root, layout, res, utils.get_transform(res, False, crop),
                                      utils.get_transform(res, True, crop), cfg, True)
                    for W, batches in zip(WORKERS, run(ds)):
                        if crop is None and squashed is None:
                            rows = {}
                            for b in batches:
                                for key, ik in (("img", "ind"), ("label", "ind"), ("mask", "ind"),
                                                ("img_pos", "ind_pos"), ("label_pos", "ind_pos"),
                                                ("mask_pos", "ind_pos")):
                                    for j, i in enumerate(b[ik].tolist()):
                                        rows.setdefault(key.replace("_pos", ""), {})[i] = b[key][j]
                            assert all(len(v) == N for v in rows.values())
                            squashed = {k: [rows[k][i] for i in range(N)] for k in ("img", "label", "mask")}
                            case["squashed"] = rows_of(squashed["img"], squashed["label"], squashed["mask"], res,
                                                       "squashed")
                        for b in batches:
                            check(b, crop, res, full, squashed)
                        case["runs"][(crop, W)] = dict(sizes=[len(b["ind"]) for b in batches], draws=torch.cat(
                            [torch.cat([b["ind"][:, None], b["ind_pos"][:, None], b["seed"][:, None].to(torch.int64),
                                        b["win"]], 1) for b in batches]))
                        print(layout, res, crop, W, len(batches), "batches")
                cases[f"{layout}_{res}"] = case
    torch.save(dict(tree=files, nns=torch.from_numpy(nns), num_neighbors=NUM_NEIGHBORS, batch_size=BATCH, seed=SEED,
                    values=values, frames=frames, cases=cases), OUT)
    print(f"wrote {OUT}: {os.path.getsize(OUT)} bytes")


def _crop(t, top, left, res):
    return t[..., top:top + res, left:left + res]


def check(b, crop, res, full, squashed):
    """Every sample of batch b is the gather of the stored rows (the docstring above)."""
    for j in range(len(b["ind"])):
        for side, ik, w0 in (("", "ind", 0), ("_pos", "ind_pos", 4)):
            i = int(b[ik][j])
            f = full[i]
            if crop is None:
                want = dict(img=squashed["img"][i], label=squashed["label"][i], mask=squashed["mask"][i])
            else:
                if crop == "random":
                    top, left, ltop, lleft = b["win"][j][w0:w0 + 4].tolist()
                else:
                    top, left = (int(round((s - res) / 2.0)) for s in f["img"].shape[-2:])
                    ltop, lleft = (int(round((s - res) / 2.0)) for s in f["label"].shape[-2:])
                want = dict(img=_crop(f["img"], top, left, res), label=_crop(f["label"], ltop, lleft, res),
                            mask=_crop(f["mask"], ltop, lleft, res))
            assert torch.equal(b["img" + side][j], want["img"]), (crop, i, "img")
            assert torch.equal(b["label" + side][j], want["label"]), (crop, i, "label")
            assert torch.equal(b["mask" + side][j], want["mask"]), (crop, i, "mask")


if __name__ == "__main__":
    main()
