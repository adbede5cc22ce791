"""Cost of feeding the training step from a resident data set (stego_b200.dataset.ResidentDataset) against a
reference-style host loader.

    python profiles/dataset_time.py [--out FILE]

Prints one JSON object with the card name and power limit read in the same run.
  * `build`: ResidentDataset.append of decoded 320 x 320 RGB crops with label maps (five-crop-sized) at res 224, in
    chunks of 64, host clock per sample from an idle device to the synchronise after the last chunk.  Decoding is not
    included.
  * `batch`: the batch kernel (one launch: 2B = 64 store rows gathered, normalised fp32 frames, int64 labels and bool
    masks) at B = 32, res 224 and 320, store on the device and in pinned host memory, CUDA events over a window of
    next() calls.  `bytes_read` = 64 * 4 res^2 store bytes, `bytes_written` = 64 * (12 + 8 + 1) res^2; the HBM bound
    is (read + written) / 3.35 TB/s (H100 SXM HBM3), the PCIe bound of the host store is bytes_read / 64 GB/s (PCIe
    5.0 x16, one direction, nominal).
  * `train`: c1 training images/s (ViT-S/8, res 224, B = 32, the shipped config; images/s counts anchors and
    positives, 2B per step) fed by store.batches, and fed by a DataLoader over a reference-style data set that decodes
    synthetic 320 x 320 JPEG crops and PNG labels from a temporary directory with PIL and runs torchvision's
    Resize(NEAREST) / CenterCrop / ToTensor / Normalize on the anchor and its kNN positive (num_workers 8,
    pin_memory), with the host's core count.
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
CROP, N_SET, B, K, NUM_NEIGHBORS, WORKERS = 320, 512, 32, 8, 5, 8


def _crops(n, seed=0):
    rng = np.random.default_rng(seed)
    base = rng.integers(0, 256, (CROP, CROP, 3), dtype=np.uint8)
    labs = rng.integers(0, 28, (CROP, CROP), dtype=np.uint8)
    return [np.roll(base, 7 * i, axis=1) for i in range(n)], [np.roll(labs, 5 * i, axis=0) for i in range(n)]


def _nns(n, seed=1):
    rng = np.random.default_rng(seed)
    return np.stack([np.concatenate([[i], rng.permutation(n)[:K - 1]]) for i in range(n)]).astype(np.int64)


def build(dev):
    from stego_b200.dataset import ResidentDataset
    images, labels = _crops(N_SET)

    def fill():
        store = ResidentDataset(N_SET, 224, "cropped")
        for i in range(0, N_SET, 64):
            store.append(images[i:i + 64], labels[i:i + 64])

    fill()
    ms = host_ms(fill, 3)
    return dict(samples=N_SET, size=[CROP, CROP], res=224, ms=round(ms, 2), samples_per_s=round(N_SET / ms * 1e3))


def batch(dev):
    from stego_b200.dataset import ResidentDataset
    images, labels = _crops(256)
    nns = _nns(256)
    out = []
    for res in (224, 320):
        for location in ("cuda", "host"):
            store = ResidentDataset(256, res, "cropped", location)
            store.append(images, labels)
            epochs = store.batches(nns, B, NUM_NEIGHBORS, 0, loader_workers=1)
            state = dict(epoch=next(epochs))

            def step():
                try:
                    return next(state["epoch"])
                except StopIteration:
                    state["epoch"] = next(epochs)
                    return next(state["epoch"])

            # the launch alone on one fixed record, then whole next() calls (host draws and launch)
            index = np.concatenate(store_rows(nns, 0))
            kernel_ms, calls = window_ms(lambda: store._gather(index, torch.float32), **WINDOW)
            next_ms, _ = window_ms(step, **WINDOW)
            read = 2 * B * 4 * res * res
            written = 2 * B * 21 * res * res
            hbm = (read + written) / HBM_BYTES_PER_S * 1e3
            row = dict(res=res, location=location, B=B, kernel_ms=round(kernel_ms, 4), kernel_calls=calls,
                       next_ms=round(next_ms, 4), bytes_read=read, bytes_written=written, hbm_bound_ms=round(hbm, 4),
                       kernel_vs_hbm_bound=round(kernel_ms / hbm, 2))
            if location == "host":
                pcie = read / PCIE_BYTES_PER_S * 1e3
                row.update(pcie_bound_ms=round(pcie, 4), kernel_vs_pcie_bound=round(kernel_ms / pcie, 2))
            out.append(row)
    return out


def store_rows(nns, seed):
    from stego_b200.dataset import Sampler
    return next(next(Sampler(nns, B, NUM_NEIGHBORS, seed, 1, res=224)))[:2]


class _Files(torch.utils.data.Dataset):
    """A reference-style training set: per sample, decode the anchor and a kNN positive from files and run
    get_transform(224, ., "center") on both images and labels."""

    def __init__(self, root, n, nns):
        import torchvision.transforms as T
        from PIL import Image
        from stego_b200.frames import MEAN, STD
        self.root, self.n, self.nns, self.Image = root, n, nns, Image
        self.img_t = T.Compose([T.Resize(224, Image.NEAREST), T.CenterCrop(224), T.ToTensor(), T.Normalize(MEAN, STD)])
        self.lab_t = T.Compose([T.Resize(224, Image.NEAREST), T.CenterCrop(224)])

    def _one(self, i):
        img = self.img_t(self.Image.open(os.path.join(self.root, f"{i}.jpg")).convert("RGB"))
        lab = torch.as_tensor(np.array(self.lab_t(self.Image.open(os.path.join(self.root, f"{i}.png")))),
                              dtype=torch.int64) - 1
        return img, lab, lab == -1

    def __getitem__(self, i):
        j = int(self.nns[i][np.random.randint(1, NUM_NEIGHBORS + 1)])
        (img, lab, mask), (img_p, lab_p, mask_p) = self._one(i), self._one(j)
        return dict(ind=i, img=img, label=lab, mask=mask.unsqueeze(0), img_pos=img_p, label_pos=lab_p,
                    mask_pos=mask_p.unsqueeze(0), ind_pos=j, seed=np.random.randint(2147483647))

    def __len__(self):
        return self.n


def train(dev, steps=20, warmup=5):
    from PIL import Image
    from stego_b200.config import make_cfg
    from stego_b200.dataset import ResidentDataset
    from stego_b200.segmenter import LitUnsupervisedSegmenter
    cfg = make_cfg(model_type="vit_small", res=224, random_backbone_init=True)
    torch.manual_seed(0)
    model = LitUnsupervisedSegmenter(27, cfg).to(dev)
    model.train()
    model.configure_optimizers()
    images, labels = _crops(N_SET)
    nns = _nns(N_SET)

    def run(batches):
        for i in range(warmup):
            model.training_step(next(batches), i)
        ms = host_ms(lambda: model.training_step(next(batches), 0), steps)
        return 2 * B / ms * 1e3

    def forever(epochs):
        for epoch in epochs:
            yield from epoch

    store = ResidentDataset(N_SET, 224, "cropped")
    for i in range(0, N_SET, 64):
        store.append(images[i:i + 64], labels[i:i + 64])
    store_rate = run(forever(store.batches(nns, B, NUM_NEIGHBORS, 0, loader_workers=0)))
    with tempfile.TemporaryDirectory() as root:
        for i, (img, lab) in enumerate(zip(images, labels)):
            Image.fromarray(img).save(os.path.join(root, f"{i}.jpg"), quality=95)
            Image.fromarray(lab, mode="L").save(os.path.join(root, f"{i}.png"))
        loader = torch.utils.data.DataLoader(_Files(root, N_SET, nns), B, shuffle=True, num_workers=WORKERS,
                                             pin_memory=True, persistent_workers=True)

        def host_batches():
            while True:
                for b in loader:
                    yield {k: (v.to(dev, non_blocking=True) if k not in ("ind", "ind_pos", "seed") else v)
                           for k, v in b.items()}

        loader_rate = run(host_batches())
    return dict(config="c1", B=B, steps=steps, store_images_per_s=round(store_rate, 1),
                loader_images_per_s=round(loader_rate, 1), loader_workers=WORKERS, host_cores=os.cpu_count(),
                speedup=round(store_rate / loader_rate, 2))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from stego_b200 import _lib
    _lib.load()
    dev = torch.device("cuda:0")
    emit(dict(card=card(), build=build(dev), batch=batch(dev), train=train(dev), gpu_info_after=card()), args.out,
         indent=1)


if __name__ == "__main__":
    main()
