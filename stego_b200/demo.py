"""Segment a folder of images with a model (reference src/demo_segmentation.py:44-78).

The reference lists the folder, decodes each file with PIL in DataLoader workers, builds its frames with
get_transform(res, False, "center"), runs the flip-TTA probes and the dense CRF per image and writes the two argmax
maps as PNGs.  `segment_folder` keeps the decoding in the workers (they return the raw RGB bytes), builds each batch's
frames on the device with frames.load_frames, runs model.eval_step(run_crf=True) on them (the CRF's guidance image
comes from the normalised frame, as the reference's unnorm -> to_pil_image does) and copies the maps to the host once
per batch.
"""
from __future__ import annotations

import os

import numpy as np
import torch
from PIL import Image
from torch.utils.data import DataLoader, Dataset

from .frames import load_frames


class _RawImageFolder(Dataset):
    """(uint8 H x W x 3 RGB array, file name) per entry of os.listdir(root) (demo_segmentation.py's
    UnlabeledImageFolder without its transform)."""

    def __init__(self, root: str):
        self.root = root
        self.images = os.listdir(root)

    def __getitem__(self, index):
        name = self.images[index]
        with Image.open(os.path.join(self.root, name)) as im:
            return np.asarray(im.convert("RGB")), name

    def __len__(self):
        return len(self.images)


def _as_list(batch):
    return batch


def png_name(name: str) -> str:
    """demo_segmentation.py's output name: the file name without its last extension, then ".png"."""
    return ".".join(name.split(".")[:-1]) + ".png"


def segment_folder(model, image_dir: str, result_dir: str, res: int = 320, batch_size: int = 8,
                   num_workers: int = 0, devices=None) -> list:
    """Write result_dir/linear/<stem>.png and result_dir/cluster/<stem>.png, the CRF-refined linear-probe and
    cluster-probe argmax maps (uint8, res x res), for every file of image_dir, as demo_segmentation.py does with
    cfg.res = res, cfg.batch_size = batch_size and cfg.num_workers = num_workers.  Batches hold batch_size * 2 images.

    model: a LitUnsupervisedSegmenter on a CUDA device; the frames are built there.  devices: eval_step's `devices=`
    (the demo's use_ddp spreads its batches over the GPUs with nn.DataParallel; here they go to these devices).
    Returns the names written, in folder order."""
    dev = next(model.parameters()).device
    if dev.type != "cuda":
        raise RuntimeError("stego_b200.demo.segment_folder: the model must be on a CUDA device (no CPU fallback)")
    for sub in ("linear", "cluster"):
        os.makedirs(os.path.join(result_dir, sub), exist_ok=True)
    dataset = _RawImageFolder(image_dir)
    loader = DataLoader(dataset, batch_size * 2, shuffle=False, num_workers=num_workers, collate_fn=_as_list)
    written = []
    with torch.cuda.device(dev):
        for batch in loader:
            arrays, names = zip(*batch)
            frames = load_frames(list(arrays), res)
            out = model.eval_step(dict(img=frames), run_crf=True, devices=devices)
            maps = torch.stack([out["linear_preds"], out["cluster_preds"]]).cpu()  # one copy to the host
            for j, name in enumerate(names):
                stem = png_name(name)
                Image.fromarray(maps[0, j].numpy()).save(os.path.join(result_dir, "linear", stem))
                Image.fromarray(maps[1, j].numpy()).save(os.path.join(result_dir, "cluster", stem))
                written.append(stem)
    return written
