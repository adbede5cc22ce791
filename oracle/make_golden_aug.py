"""Generate tests/golden/aug_views.pt from the REAL reference: ContrastiveSegDataset.__getitem__ (src/data.py:527-563)
with the transforms my_app builds (src/train_segmentation.py:408-416), on the CPU.

    STEGO_REFERENCE_SRC=<reference checkout>/src python oracle/make_golden_aug.py

The dataset object is a stand-in holding one (frame, label) pack and the two transforms; __getitem__ is the
reference's own method.  The frames are rebuilt by the tests from `cases()` (seeded).  Each case stores the seed
__getitem__ drew (numpy's generator is seeded first, as a loader worker's is), img_aug and coord_aug.
"""
from __future__ import annotations

import os
import sys
from types import SimpleNamespace

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import aug_oracle  # noqa: E402
import reference_shim  # noqa: E402

OUT = os.path.join(HERE, "..", "tests", "golden", "aug_views.pt")


def cases():
    """name -> (frame [3, H, W] fp32, size, numpy seed): normalised-looking frames (values well outside [0, 1]),
    square and non-square, output smaller and larger than the frame."""
    g = torch.Generator().manual_seed(17)
    out = {}
    for k, (H, W, size, np_seed) in enumerate([(24, 24, 16, 1), (24, 24, 16, 2), (20, 31, 16, 3), (12, 12, 20, 4),
                                               (17, 13, 9, 5), (32, 32, 32, 6)]):
        frame = torch.randn(3, H, W, generator=g) * 1.2 + 0.2
        out[f"case{k}_{H}x{W}_to_{size}"] = (frame, size, np_seed)
    return out


def main():
    if not reference_shim.available():
        raise RuntimeError("set STEGO_REFERENCE_SRC to the reference's src directory")
    sys.path.insert(0, reference_shim.REFERENCE_SRC)
    from data import ContrastiveSegDataset  # noqa: E402  (the reference's own class)
    golden = {}
    for name, (frame, size, np_seed) in sorted(cases().items()):
        geometric, photometric = aug_oracle.transforms(size)
        ds = SimpleNamespace(dataset=[(frame, torch.zeros(frame.shape[1:], dtype=torch.int64))], pos_images=False,
                             pos_labels=False, extra_transform=None, mask=False, aug_geometric_transform=geometric,
                             aug_photometric_transform=photometric)
        ds._set_seed = lambda s, ds=ds: ContrastiveSegDataset._set_seed(ds, s)
        np.random.seed(np_seed)
        seed = int(np.random.randint(2147483647))  # what __getitem__ is about to draw
        np.random.seed(np_seed)
        ret = ContrastiveSegDataset.__getitem__(ds, 0)
        golden[name] = dict(seed=seed, img_aug=ret["img_aug"], coord_aug=ret["coord_aug"])
    torch.save(golden, OUT)
    print(f"wrote {OUT}: {len(golden)} cases")


if __name__ == "__main__":
    main()
