"""Generate tests/golden/dataset.pt from the REAL reference training loader: ContrastiveSegDataset (src/data.py:419-565)
over CroppedDataset and DirectoryDataset, with the transforms my_app builds (src/train_segmentation.py:408-434), under
DataLoader(batch_size=4, shuffle=True, num_workers=W) for W = 0, 1 and 3, on the CPU.

    STEGO_REFERENCE_SRC=<reference checkout>/src python oracle/make_golden_dataset.py

The input is 13 seeded synthetic images of mixed sizes with label maps, written into temporary five-crop and directory
layouts (the .jpg names hold PNG bytes: PIL decodes by content, losslessly), and a seeded nns table.  Each run seeds
torch, numpy and random with SEED (as seed_everything does) and reads 2.5 epochs, so every epoch ends in a partial
batch and the last one stops halfway.  A subclass records the aug seed each __getitem__ passes to _set_seed and drops
img_aug / coord_aug; everything else is the reference's own code.

Stored: the decoded inputs, the nns table, per (layout, res, W) the batches' ind, ind_pos and seed (one table of the
samples in loader order, and the batch sizes), and the reference's per-index rows of img, label and mask (their dtypes
and per-sample shapes).  Every batch's img, img_pos, label, label_pos, mask and mask_pos are checked here to equal
those rows gathered at ind / ind_pos, so a batch of the fixture is the gather of the rows.  The img rows are the same
for every layout at one res (checked) and are stored once per res; labels are stored as int16 and masks as bool, with
the dtypes the reference returned.
"""
from __future__ import annotations

import os
import random
import sys
import tempfile
from types import SimpleNamespace

import numpy as np
import torch
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import reference_shim  # noqa: E402
from make_golden_frames import _import_reference_loaders  # noqa: E402

OUT = os.path.join(HERE, "..", "tests", "golden", "dataset.pt")
N, K, NUM_NEIGHBORS, BATCH, SEED = 13, 6, 4, 4, 5
RESOLUTIONS = (32, 30)
WORKERS = (0, 1, 3)
LAYOUTS = ("cropped", "directory", "directory_unlabelled")


def inputs():
    rng = np.random.default_rng(2024)
    images, labels = [], []
    for k in range(N):
        H, W = int(rng.integers(12, 70)), int(rng.integers(12, 70))
        images.append(rng.integers(0, 256, (H, W, 3), dtype=np.uint8))
        lab = rng.integers(0, 28, (H, W), dtype=np.uint8)
        lab[rng.random((H, W)) < 0.05] = 255
        labels.append(lab)
    nns = np.zeros((N, K), dtype=np.int64)
    for i in range(N):
        others = rng.permutation([j for j in range(N) if j != i])[:K - 1]
        nns[i] = [i] + list(others)
    return images, labels, nns


def write_layout(root: str, layout: str, images, labels, nns, res: int, cfg):
    if layout == "cropped":
        base = os.path.join(root, "cropped", f"cocostuff27_five_crop_{cfg.crop_ratio}")
        for sub in ("img/train", "label/train"):
            os.makedirs(os.path.join(base, sub), exist_ok=True)
        for i, (img, lab) in enumerate(zip(images, labels)):
            Image.fromarray(img).save(os.path.join(base, "img/train", f"{i}.jpg"), format="PNG")
            Image.fromarray(lab, mode="L").save(os.path.join(base, "label/train", f"{i}.png"))
        name, crop = "cocostuff27", "five"
    else:
        base = os.path.join(root, cfg.dir_dataset_name)
        os.makedirs(os.path.join(base, "imgs/train"), exist_ok=True)
        if layout == "directory":
            os.makedirs(os.path.join(base, "labels/train"), exist_ok=True)
        for i, (img, lab) in enumerate(zip(images, labels)):
            Image.fromarray(img).save(os.path.join(base, "imgs/train", f"im{i:02d}.png"))
            if layout == "directory":
                Image.fromarray(lab, mode="L").save(os.path.join(base, "labels/train", f"im{i:02d}.png"))
        name, crop = cfg.dir_dataset_name, None
    os.makedirs(os.path.join(root, "nns"), exist_ok=True)
    np.savez_compressed(os.path.join(root, "nns", f"nns_{cfg.model_type}_{name}_train_{crop}_{res}.npz"), nns=nns)
    return ("cocostuff27", "five") if layout == "cropped" else ("directory", None)


def run(data, utils, root, dataset_name, crop_type, res, cfg, workers):
    import torchvision.transforms as T
    from torch.utils.data import DataLoader

    class Recording(data.ContrastiveSegDataset):
        def _set_seed(self, seed):
            self.last_seed = seed
            super()._set_seed(seed)

        def __getitem__(self, ind):
            ret = super().__getitem__(ind)
            del ret["img_aug"], ret["coord_aug"]
            ret["seed"] = self.last_seed
            return ret

    geometric = T.Compose([T.RandomHorizontalFlip(), T.RandomResizedCrop(size=res, scale=(0.8, 1.0))])
    photometric = T.Compose([T.ColorJitter(brightness=.3, contrast=.3, saturation=.3, hue=.1), T.RandomGrayscale(.2),
                             T.RandomApply([T.GaussianBlur((5, 5))])])
    ds = Recording(pytorch_data_dir=root, dataset_name=dataset_name, crop_type=crop_type, image_set="train",
                   transform=utils.get_transform(res, False, "center"),
                   target_transform=utils.get_transform(res, True, "center"), cfg=cfg,
                   aug_geometric_transform=geometric, aug_photometric_transform=photometric,
                   num_neighbors=NUM_NEIGHBORS, mask=True, pos_images=True, pos_labels=True)
    random.seed(SEED)
    np.random.seed(SEED)
    torch.manual_seed(SEED)
    loader = DataLoader(ds, BATCH, shuffle=True, num_workers=workers)
    batches = []
    per_epoch = -(-N // BATCH)
    for epoch in range(3):
        for i, b in enumerate(loader):
            if epoch == 2 and i == per_epoch // 2:
                break
            batches.append(b)
    return batches


def main():
    if not reference_shim.available():
        raise RuntimeError("set STEGO_REFERENCE_SRC to the reference's src directory")
    utils, data = _import_reference_loaders()
    images, labels, nns = inputs()
    cfg = SimpleNamespace(dir_dataset_n_classes=27, dir_dataset_name="myset", crop_ratio=0.5, crop_type="five",
                          model_type="vit_small", res=None)
    cases, frames = {}, {}
    with tempfile.TemporaryDirectory() as tmp:
        for layout in LAYOUTS:
            for res in RESOLUTIONS:
                root = os.path.join(tmp, f"{layout}_{res}")
                cfg.res = res
                dataset_name, crop_type = write_layout(root, layout, images, labels, nns, res, cfg)
                case = dict(rows=None, runs={})
                for W in WORKERS:
                    batches = run(data, utils, root, dataset_name, crop_type, res, cfg, W)
                    if case["rows"] is None:  # the per-index rows, from the first run's batches
                        rows = {}
                        for b in batches:
                            for key, ik in (("img", "ind"), ("label", "ind"), ("mask", "ind"), ("img_pos", "ind_pos"),
                                            ("label_pos", "ind_pos"), ("mask_pos", "ind_pos")):
                                name = key.replace("_pos", "")
                                for j, idx in enumerate(b[ik].tolist()):
                                    rows.setdefault(name, {})[idx] = b[key][j]
                        assert all(len(rows[k]) == N for k in rows), {k: len(v) for k, v in rows.items()}
                        case["rows"] = {k: torch.stack([v[i] for i in range(N)]) for k, v in rows.items()}
                    R = case["rows"]
                    for b in batches:
                        for key, ik in (("img", "ind"), ("label", "ind"), ("mask", "ind"), ("img_pos", "ind_pos"),
                                        ("label_pos", "ind_pos"), ("mask_pos", "ind_pos")):
                            want = R[key.replace("_pos", "")][b[ik]]
                            assert b[key].dtype == want.dtype and torch.equal(b[key], want), (layout, res, W, key)
                    # one int64 [samples, 3] table (ind, ind_pos, seed) and the batch sizes per run
                    case["runs"][W] = dict(sizes=[len(b["ind"]) for b in batches], draws=torch.stack(
                        [torch.cat([b[k].to(torch.int64) for b in batches]) for k in ("ind", "ind_pos", "seed")], 1))
                R = case["rows"]
                # the fixture stays small: the frames depend on the image and res alone, so each res keeps one copy
                # (checked equal across the layouts); labels go as int16 and the 0 / 1 masks as bool, each with the
                # dtype the reference returned, and the tests convert back before comparing
                img = R.pop("img")
                if res in frames:
                    assert torch.equal(frames[res], img), (layout, res)
                frames[res] = img
                assert R["label"].abs().max() < 1 << 15
                R["label_dtype"] = str(R["label"].dtype).replace("torch.", "")
                R["label"] = R["label"].to(torch.int16)
                assert ((R["mask"] == 0) | (R["mask"] == 1)).all()
                R["mask_dtype"] = str(R["mask"].dtype).replace("torch.", "")
                R["mask"] = R["mask"].to(torch.bool)
                cases[f"{layout}_{res}"] = case
    torch.save(dict(images=[torch.from_numpy(x) for x in images], labels=[torch.from_numpy(x) for x in labels],
                    nns=torch.from_numpy(nns), num_neighbors=NUM_NEIGHBORS, batch_size=BATCH, seed=SEED, frames=frames,
                    cases=cases), OUT)
    print(f"wrote {OUT}: {os.path.getsize(OUT)} bytes")


if __name__ == "__main__":
    main()
