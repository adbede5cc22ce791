"""Cost of a validation pass fed by a resident evaluation set (stego_b200.evalset.EvalSet) against one fed by a
reference-style validation DataLoader.

    python profiles/evalset_time.py [--out FILE]

Prints one JSON object with the card name and power limit read in the same run.  The set is N_VAL synthetic 640 x 480
COCO-Stuff-style images (JPEG, quality 95) with PNG annotations of bytes 0..181 and 255, in the cocostuff27 val
layout, written to a temporary directory; the fine -> coarse table is a stand-in of the real one's size (182 ids).
  * `build`: EvalSet.coco at res 320 from those files, decoding in 8 DataLoader workers, host clock per sample to the
    synchronise after the last row (decode included), and EvalSet.append of already decoded arrays (decode excluded).
  * `batch`: the gather kernel alone (one launch: B = 16 rows, normalised fp32 frames, int64 labels, bool masks) at
    res 320, store on the device and in pinned host memory, CUDA events over a window.  `bytes_read` = 16 * 4 res^2
    store bytes, `bytes_written` = 16 * (12 + 8 + 1) res^2; the HBM bound is (read + written) / 3.35 TB/s (H100 SXM
    HBM3), the PCIe bound of the host store bytes_read / 64 GB/s (PCIe 5.0 x16, one direction, nominal).
  * `validate`: one full pass of LitUnsupervisedSegmenter.validate(store, 16) (validation_step over every batch, then
    validation_epoch_end), ViT-S/8 and ViT-B/8, 320 x 320, 27 classes, store on the device and in pinned host memory,
    images/s by host clock per pass after one warm-up pass; and the same pass fed by
    DataLoader(shuffle=False, batch_size=16, num_workers=8, pin_memory=True) over a reference-style data set that opens
    each image with PIL, converts it to RGB, runs torchvision's Resize(320, NEAREST) / CenterCrop / ToTensor /
    Normalize, and remaps the annotation with the Coco class's per-id loop (a new loader iterator per pass, as each
    validation epoch makes one), with validation_step per batch and validation_epoch_end.
"""
import argparse
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from _measure import card, emit, host_ms, window_ms  # noqa: E402

HBM_BYTES_PER_S, PCIE_BYTES_PER_S = 3.35e12, 64e9
WINDOW = dict(warmup=3, min_window_s=0.5, min_iters=10)
N_VAL, H, W, RES, B, WORKERS, PASSES = 480, 480, 640, 320, 16, 8, 2
FINE_TO_COARSE = {i: (i * 7) % 27 for i in range(182)}  # a stand-in with the real table's size: the loop's cost


def _write_coco(root):
    """N_VAL image / annotation pairs in the cocostuff27 val layout (list 7); returns the decoded arrays."""
    from PIL import Image
    rng = np.random.default_rng(0)
    base = os.path.join(root, "cocostuff")
    for sub in ("images/val2017", "annotations/val2017", "curated/val2017"):
        os.makedirs(os.path.join(base, sub), exist_ok=True)
    ids = [f"{i:012d}" for i in range(N_VAL)]
    img0 = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    lab0 = rng.integers(0, 182, (H, W), dtype=np.uint8)
    lab0[rng.random((H, W)) < 0.05] = 255
    images, labels = [], []
    for i, img_id in enumerate(ids):
        img, lab = np.roll(img0, 7 * i, axis=1), np.roll(lab0, 5 * i, axis=0)
        Image.fromarray(img).save(os.path.join(base, "images/val2017", img_id + ".jpg"), quality=95)
        Image.fromarray(lab, mode="L").save(os.path.join(base, "annotations/val2017", img_id + ".png"))
        images.append(img)
        labels.append(lab)
    with open(os.path.join(base, "curated/val2017/Coco164kFull_Stuff_Coarse_7.txt"), "w") as f:
        f.write("\n".join(ids) + "\n")
    return images, labels


class _RefCoco(torch.utils.data.Dataset):
    """A reference-style Coco validation set: PIL decode, torchvision transforms, the per-id remap loop."""

    def __init__(self, root):
        import torchvision.transforms as T
        from PIL import Image
        from stego_b200.evalset import coco_files
        from stego_b200.frames import MEAN, STD
        self.images, self.labels = coco_files(root, "cocostuff27", "val")
        self.Image = Image
        self.img_t = T.Compose([T.Resize(RES, Image.NEAREST), T.CenterCrop(RES), T.ToTensor(), T.Normalize(MEAN, STD)])
        self.lab_t = T.Compose([T.Resize(RES, Image.NEAREST), T.CenterCrop(RES)])

    def __getitem__(self, i):
        img = self.img_t(self.Image.open(self.images[i]).convert("RGB"))
        label = torch.as_tensor(np.array(self.lab_t(self.Image.open(self.labels[i]))), dtype=torch.int64)
        label[label == 255] = -1
        coarse = torch.zeros_like(label)
        for fine, c in FINE_TO_COARSE.items():
            coarse[label == fine] = c
        coarse[label == -1] = -1
        return dict(ind=i, img=img, label=coarse, mask=coarse >= 0)

    def __len__(self):
        return len(self.images)


def build(root, images, labels):
    from stego_b200.evalset import EvalSet
    ms = host_ms(lambda: EvalSet.coco(root, "cocostuff27", "val", RES, FINE_TO_COARSE, num_workers=WORKERS), 1)

    def fill():
        store = EvalSet(N_VAL, RES, "cocostuff27", fine_to_coarse=FINE_TO_COARSE)
        for i in range(0, N_VAL, 64):
            store.append(images[i:i + 64], labels[i:i + 64])

    fill()
    append_ms = host_ms(fill, 3)
    return dict(samples=N_VAL, size=[H, W], res=RES, loader_workers=WORKERS, host_cores=os.cpu_count(),
                from_files_samples_per_s=round(N_VAL / ms * 1e3), append_samples_per_s=round(N_VAL / append_ms * 1e3))


def batch(stores):
    out = []
    index = np.arange(B, dtype=np.int64) * 7 % N_VAL
    for location, store in stores.items():
        kernel_ms, calls = window_ms(lambda: store._gather(index, torch.float32), **WINDOW)
        read, written = B * 4 * RES * RES, B * 21 * RES * RES
        hbm = (read + written) / HBM_BYTES_PER_S * 1e3
        row = dict(res=RES, location=location, B=B, kernel_ms=round(kernel_ms, 4), kernel_calls=calls,
                   bytes_read=read, bytes_written=written, hbm_bound_ms=round(hbm, 4),
                   kernel_vs_hbm_bound=round(kernel_ms / hbm, 2))
        if location == "host":
            pcie = read / PCIE_BYTES_PER_S * 1e3
            row.update(pcie_bound_ms=round(pcie, 4), kernel_vs_pcie_bound=round(kernel_ms / pcie, 2))
        out.append(row)
    return out


def validate(root, stores, dev):
    from stego_b200.config import make_cfg
    from stego_b200.segmenter import LitUnsupervisedSegmenter
    loader = torch.utils.data.DataLoader(_RefCoco(root), B, shuffle=False, num_workers=WORKERS, pin_memory=True)
    out = []
    for arch in ("vit_small", "vit_base"):
        cfg = make_cfg(model_type=arch, res=RES, random_backbone_init=True)
        torch.manual_seed(0)
        model = LitUnsupervisedSegmenter(27, cfg).to(dev)
        model.train()
        model.configure_optimizers()
        row = dict(arch=arch, res=RES, B=B, images=N_VAL, passes=PASSES)
        for location, store in stores.items():
            model.validate(store, B)
            ms = host_ms(lambda: model.validate(store, B), PASSES)
            row[f"store_{location}_images_per_s"] = round(N_VAL / ms * 1e3, 1)

        def loader_pass():
            for i, b in enumerate(loader):
                model.validation_step(dict(img=b["img"].to(dev, non_blocking=True),
                                           label=b["label"].to(dev, non_blocking=True)), i)
            return model.validation_epoch_end([])

        loader_pass()
        ms = host_ms(loader_pass, PASSES)
        row.update(loader_images_per_s=round(N_VAL / ms * 1e3, 1), loader_workers=WORKERS,
                   host_cores=os.cpu_count())
        row["store_cuda_vs_loader"] = round(row["store_cuda_images_per_s"] / row["loader_images_per_s"], 2)
        out.append(row)
        del model
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from stego_b200 import _lib
    from stego_b200.evalset import EvalSet
    _lib.load()
    dev = torch.device("cuda:0")
    info = card()
    with tempfile.TemporaryDirectory() as root:
        images, labels = _write_coco(root)
        built = build(root, images, labels)
        stores = {loc: EvalSet.coco(root, "cocostuff27", "val", RES, FINE_TO_COARSE, loc, num_workers=WORKERS)
                  for loc in ("cuda", "host")}
        result = dict(card=info, build=built, batch=batch(stores), validate=validate(root, stores, dev),
                      gpu_info_after=card())
    emit(result, args.out, indent=1)


if __name__ == "__main__":
    main()
