"""Cost of the random-crop training loader on a ragged store (crop="random": each row's whole Resize(res) output,
windows cut by stego_store_batch_window) against the fixed-row gather (stego_dataset_batch).

    python profiles/uncropped_time.py [--out FILE]

Prints one JSON object with the card name and power limit read in the same run.
  * `batch`: at B = 32 (2B = 64 rows gathered: anchors and positives), res 224 and 320, store on the device and in
    pinned host memory, CUDA events over a window of launches on one fixed record: `window_ms`, the windowed gather on
    a ragged store of 2:1 (Cityscapes-shaped) 640 x 320 images, each window drawn by the loader; `fixed_ms`,
    stego_dataset_batch on a res x res store of the same images.  The bytes and bounds columns are those of
    dataset_time.py: bytes_read = 64 * 4 res^2 store bytes, bytes_written = 64 * (12 + 8 + 1) res^2, the HBM bound
    (read + written) / 3.35 TB/s (H100 SXM HBM3), the PCIe bound of the host store bytes_read / 64 GB/s (PCIe 5.0
    x16, one direction, nominal).  `next_ms`: whole next() calls on the random-crop loader (host draws, two
    RandomCrop windows per sample and its positive's, and the launch), loader_workers 1.
  * `train`: c1 training images/s (ViT-S/8, res 224, B = 32, the shipped config; anchors and positives, 2B per step)
    fed by a random-crop store of 2:1 frames, and by a center-crop store of the same frames.
"""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from _measure import card, emit, host_ms, window_ms  # noqa: E402

HBM_BYTES_PER_S, PCIE_BYTES_PER_S = 3.35e12, 64e9
WINDOW = dict(warmup=3, min_window_s=0.5, min_iters=10)
H, W, N_SET, B, K, NUM_NEIGHBORS = 320, 640, 256, 32, 8, 5


def _frames(n, seed=0):
    rng = np.random.default_rng(seed)
    base = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    labs = rng.integers(0, 34, (H, W), dtype=np.uint8)
    return [np.roll(base, 7 * i, axis=1) for i in range(n)], [np.roll(labs, 5 * i, axis=0) for i in range(n)]


def _nns(n, seed=1):
    rng = np.random.default_rng(seed)
    return np.stack([np.concatenate([[i], rng.permutation(n)[:K - 1]]) for i in range(n)]).astype(np.int64)


def _store(res, location, crop, images, labels):
    from stego_b200.evalset import EvalSet
    sizes = np.array([(H, W, H, W)] * len(images)) if crop == "random" else None
    store = EvalSet(len(images), res, "cityscapes", location, crop=crop, sizes=sizes)
    for i in range(0, len(images), 64):
        store.append(images[i:i + 64], labels[i:i + 64])
    return store


def batch(dev):
    from stego_b200.dataset import Sampler
    images, labels = _frames(N_SET)
    nns = _nns(N_SET)
    out = []
    for res in (224, 320):
        for location in ("cuda", "host"):
            ragged = _store(res, location, "random", images, labels)
            fixed = _store(res, location, "center", images, labels)
            ind, pos, _, windows = next(next(Sampler(nns, B, NUM_NEIGHBORS, 0, 1, res=res, sizes=ragged.sizes)))
            index = np.concatenate([ind, pos])
            window_time, calls = window_ms(lambda: ragged._gather(index, torch.float32, windows), **WINDOW)
            fixed_time, _ = window_ms(lambda: fixed._gather(index, torch.float32), **WINDOW)
            epochs = ragged.batches(nns, B, NUM_NEIGHBORS, 0, loader_workers=1)
            state = dict(epoch=next(epochs))

            def step():
                try:
                    return next(state["epoch"])
                except StopIteration:
                    state["epoch"] = next(epochs)
                    return next(state["epoch"])

            next_time, _ = window_ms(step, **WINDOW)
            read = 2 * B * 4 * res * res
            written = 2 * B * 21 * res * res
            hbm = (read + written) / HBM_BYTES_PER_S * 1e3
            row = dict(res=res, location=location, B=B, store_frame=[H, W], window_ms=round(window_time, 4),
                       fixed_ms=round(fixed_time, 4), kernel_calls=calls, next_ms=round(next_time, 4),
                       bytes_read=read, bytes_written=written, hbm_bound_ms=round(hbm, 4),
                       window_vs_hbm_bound=round(window_time / hbm, 2), store_bytes=ragged.nbytes,
                       fixed_store_bytes=fixed.nbytes)
            if location == "host":
                pcie = read / PCIE_BYTES_PER_S * 1e3
                row.update(pcie_bound_ms=round(pcie, 4), window_vs_pcie_bound=round(window_time / pcie, 2))
            out.append(row)
            del ragged, fixed
    return out


def train(dev, steps=20, warmup=5):
    from stego_b200.config import make_cfg
    from stego_b200.segmenter import LitUnsupervisedSegmenter
    cfg = make_cfg(model_type="vit_small", res=224, random_backbone_init=True)
    torch.manual_seed(0)
    model = LitUnsupervisedSegmenter(27, cfg).to(dev)
    model.train()
    model.configure_optimizers()
    images, labels = _frames(N_SET)
    nns = _nns(N_SET)

    def forever(epochs):
        for epoch in epochs:
            yield from epoch

    rates = {}
    for crop in ("random", "center"):
        batches = forever(_store(224, "cuda", crop, images, labels).batches(nns, B, NUM_NEIGHBORS, 0))
        for i in range(warmup):
            model.training_step(next(batches), i)
        ms = host_ms(lambda: model.training_step(next(batches), 0), steps)
        rates[crop] = round(2 * B / ms * 1e3, 1)
    return dict(config="c1", B=B, steps=steps, store_frame=[H, W], random_images_per_s=rates["random"],
                center_images_per_s=rates["center"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from stego_b200 import _lib
    _lib.load()
    dev = torch.device("cuda:0")
    emit(dict(card=card(), batch=batch(dev), train=train(dev), gpu_info_after=card()), args.out, indent=1)


if __name__ == "__main__":
    main()
