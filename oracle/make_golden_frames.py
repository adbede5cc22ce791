"""Generate tests/golden/frames.pt from the REAL reference: get_transform (src/utils.py:165-183) and the label code of
Coco (27 classes, 3 classes, exclude_things; src/data.py:296-319), CityscapesSeg (src/data.py:349-362) and
DirectoryDataset (src/data.py:93-115), on the CPU.

    STEGO_REFERENCE_SRC=<reference checkout>/src python oracle/make_golden_frames.py

The images and label maps are seeded synthetic uint8 arrays, written as PNG files into a temporary data-set layout and
read back by the reference's own classes (Coco, DirectoryDataset); CityscapesSeg's __getitem__ runs on a stand-in whose
inner loader returns the same PIL images.  src/utils.py imports plotting, download and metrics packages the loaders do
not use; those missing here are stubbed before the import.  The fixture stores each case's inputs and outputs, and
Coco's class tables (fine_to_coarse, cocostuff3_coarse_classes, first_stuff_index) for the tests to build their remaps.
"""
from __future__ import annotations

import os
import sys
import tempfile
import types
from types import SimpleNamespace

import numpy as np
import torch
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import reference_shim  # noqa: E402

OUT = os.path.join(HERE, "..", "tests", "golden", "frames.pt")


def closed_form_disagrees(H: int, W: int, res: int) -> bool:
    """floor((x + .5) in / out) differs from Pillow's resize of an index image inside the centre crop of
    get_transform(res, ., "center") of an H x W image."""
    from torchvision.transforms.functional import _compute_resized_output_size
    oh, ow = _compute_resized_output_size((H, W), [res])
    top, left = int(round((oh - res) / 2.0)), int(round((ow - res) / 2.0))
    for n_in, n_out, at in ((H, oh, top), (W, ow, left)):
        a = np.arange(n_in, dtype=np.int32)[None, :]
        pil = np.asarray(Image.fromarray(a, mode="I").resize((n_out, 1), Image.NEAREST))[0]
        closed = np.minimum(np.floor((np.arange(n_out) + 0.5) * n_in / n_out), n_in - 1).astype(np.int64)
        if not np.array_equal(pil[at:at + res], closed[at:at + res]):
            return True
    return False


def sizes():
    """(H, W, res, crop) cases: portrait / landscape / square, exactly res, 1 x 1, smaller than res, both round-half-even
    crop cases (resized long side res + 1 crops at 0, res + 3 at 2) and, per res, the first small size where the closed
    form disagrees with Pillow inside the crop."""
    out = [(48, 64, 32, "center"), (64, 48, 32, "center"), (32, 32, 32, "center"), (1, 1, 32, "center"),
           (17, 23, 40, "center"), (40, 41, 40, "center"), (40, 43, 40, "center"), (57, 56, 56, "center"),
           (59, 56, 56, "center"), (90, 61, 56, None), (20, 77, 40, None), (120, 33, 56, "center")]
    for res in (32, 40, 56):
        out.append(next((h, w, res, "center") for h in range(2, 64) for w in range(h, 64)
                        if closed_form_disagrees(h, w, res)))
    return out


def arrays(k: int, H: int, W: int):
    rng = np.random.default_rng(1000 + k)
    rgb = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    lab = rng.integers(0, 256, (H, W), dtype=np.uint8)
    lab[rng.random((H, W)) < 0.1] = 255
    return rgb, lab


def _import_reference_loaders():
    """The reference's utils (get_transform) and data modules, with absent imports stubbed."""
    sys.path.insert(0, reference_shim.REFERENCE_SRC)
    stubs = {"matplotlib": {}, "matplotlib.pyplot": {}, "wget": {}, "torch._six": {"string_classes": (str, bytes)},
             "torchmetrics": {"Metric": object}, "torch.utils.tensorboard": {},
             "torch.utils.tensorboard.summary": {"hparams": None}, "tqdm": {"tqdm": lambda x, *a, **k: x}}
    for name, attrs in stubs.items():
        try:
            __import__(name)
        except ImportError:
            mod = types.ModuleType(name)
            mod.__dict__.update(attrs)
            sys.modules[name] = mod
    sys.modules.pop("utils", None)  # reference_shim may have seeded a stub without get_transform
    import data  # noqa: E402
    import utils  # noqa: E402
    return utils, data


def main():
    if not reference_shim.available():
        raise RuntimeError("set STEGO_REFERENCE_SRC to the reference's src directory")
    utils, data = _import_reference_loaders()
    cases = []
    coco_tables = None
    with tempfile.TemporaryDirectory() as root:
        for k, (H, W, res, crop) in enumerate(sizes()):
            rgb, lab = arrays(k, H, W)
            img_t, lab_t = utils.get_transform(res, False, crop), utils.get_transform(res, True, crop)
            case = dict(H=H, W=W, res=res, crop=crop, image=torch.from_numpy(rgb), label=torch.from_numpy(lab))
            # Coco: one image per data-set tree (the .jpg name holds PNG bytes: PIL decodes by content, losslessly)
            coco_root = os.path.join(root, f"coco{k}")
            for sub in ("curated/val2017", "images/val2017", "annotations/val2017"):
                os.makedirs(os.path.join(coco_root, "cocostuff", sub))
            with open(os.path.join(coco_root, "cocostuff/curated/val2017/Coco164kFull_Stuff_Coarse.txt"), "w") as f:
                f.write("img\n")
            Image.fromarray(rgb).save(os.path.join(coco_root, "cocostuff/images/val2017/img.jpg"), format="PNG")
            Image.fromarray(lab, mode="L").save(os.path.join(coco_root, "cocostuff/annotations/val2017/img.png"))
            for variant, coarse, things in (("27", False, False), ("3", True, False), ("stuff", False, True)):
                ds = data.Coco(coco_root, "val", img_t, lab_t, coarse_labels=coarse, exclude_things=things)
                frame, label, _ = ds[0]
                case["frame"] = frame
                case["coco" + variant] = label
                coco_tables = dict(fine_to_coarse=dict(ds.fine_to_coarse),
                                   cocostuff3_coarse_classes=list(ds.cocostuff3_coarse_classes),
                                   first_stuff_index=int(ds.first_stuff_index))
            stand_in = SimpleNamespace(inner_loader=[(Image.fromarray(rgb), Image.fromarray(lab, mode="L"))],
                                       transform=img_t, target_transform=lab_t, first_nonvoid=7)
            frame_c, case["cityscapes"], _ = data.CityscapesSeg.__getitem__(stand_in, 0)
            assert torch.equal(frame_c, case["frame"])
            dir_root = os.path.join(root, f"dir{k}")
            for sub in ("imgs/val", "labels/val"):
                os.makedirs(os.path.join(dir_root, "set", sub))
            Image.fromarray(rgb).save(os.path.join(dir_root, "set/imgs/val/a.png"))
            Image.fromarray(lab, mode="L").save(os.path.join(dir_root, "set/labels/val/a.png"))
            frame_d, case["directory"], _ = data.DirectoryDataset(dir_root, "set", "val", img_t, lab_t)[0]
            assert torch.equal(frame_d, case["frame"])
            for key in ("coco27", "coco3", "cocostuff", "cityscapes", "directory"):
                assert case[key].dtype == torch.int64 and case[key].abs().max() < 1 << 15
                case[key] = case[key].to(torch.int16)  # the fixture stays small; the tests compare as int64
            cases.append(case)
    torch.save(dict(cases=cases, coco=coco_tables), OUT)
    print(f"wrote {OUT}: {len(cases)} cases")


if __name__ == "__main__":
    main()
