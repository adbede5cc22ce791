"""The cropped training sets built on the GPU (stego_b200/crops.py, csrc/jpeg.cu) against the host path they replace.

  * the crop kernels' decoded crops equal Pillow's own JPEG round trip of each crop, for every corpus image and for
    windows at every offset parity (and every offset modulo 16) inside a larger original;
  * ResidentDataset.crops equals ResidentDataset.cropped read from write_cropped's tree of the same synthetic Coco
    and Cityscapes originals: the store's image bytes, frames() and batches() (loader_workers 0 and 2), for both
    crop types, ratios 0.5 and 0.7, res 224 and 320 and both store locations; precompute_knns gives the same table.
"""
import io

import numpy as np
import pytest
import torch
from PIL import Image

from _crops_util import CONTENTS, CORPUS_SIZES, corpus_image, fine_to_coarse, make_cityscapes_tree, make_coco_tree

pytestmark = pytest.mark.gpu


def pillow_roundtrip(rgb: np.ndarray) -> np.ndarray:
    f = io.BytesIO()
    Image.fromarray(np.ascontiguousarray(rgb)).save(f, "JPEG")
    f.seek(0)
    with Image.open(f) as im:
        return np.asarray(im.convert("RGB"))


@pytest.mark.parametrize("content", CONTENTS)
def test_codec_equals_pillow_on_corpus(cuda_dev, content):
    from stego_b200.crops import jpeg_roundtrip
    images = [corpus_image(h, w, content) for h, w in CORPUS_SIZES]
    got = jpeg_roundtrip(images, [(i, 0, 0, h, w) for i, (h, w) in enumerate(CORPUS_SIZES)])
    for img, out in zip(images, got):
        np.testing.assert_array_equal(out.cpu().numpy(), pillow_roundtrip(img), err_msg=f"{img.shape}")


@pytest.mark.parametrize("content", ["noise", "gradient", "saturated"])
def test_codec_windows_at_every_offset(cuda_dev, content):
    from stego_b200.crops import jpeg_roundtrip
    src = corpus_image(90, 120, content, seed=1)
    windows = [(0, top, left, h, w) for top in range(17) for left in range(17)
               for h, w in ((33, 47), (16, 16), (2, 5), (45, 30)) if (top + left) % 3 == 0 or top % 16 == left % 16]
    windows += [(0, 0, 0, 90, 120), (0, 89, 119, 1, 1), (0, 1, 3, 89, 117)]
    got = jpeg_roundtrip([src], windows)
    for (_, top, left, h, w), out in zip(windows, got):
        np.testing.assert_array_equal(out.cpu().numpy(), pillow_roundtrip(src[top:top + h, left:left + w]),
                                      err_msg=f"window {top}, {left}, {h} x {w}")


# ---- the store against the written tree -------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def trees(tmp_path_factory):
    from stego_b200 import crops
    out = {}
    for name, make in (("cocostuff27", make_coco_tree), ("cityscapes", make_cityscapes_tree)):
        root = str(tmp_path_factory.mktemp(name))
        make(root, "train")
        f2c = fine_to_coarse() if name == "cocostuff27" else None
        for crop_type in ("five", "random"):
            for ratio in (0.5, 0.7):
                crops.write_cropped(root, name, crop_type, ratio, "train", fine_to_coarse=f2c)
        out[name] = (root, f2c)
    return out


def _batches_equal(a: dict, b: dict):
    assert a.keys() == b.keys()
    for k in a:
        assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape, k
        assert torch.equal(a[k].cpu(), b[k].cpu()), k


CASES = [(n, t, r, res, loc) for n in ("cocostuff27", "cityscapes") for t in ("five", "random") for r in (0.5, 0.7)
         for res, loc in ((224, "cuda"), (320, "host"))] + [("cityscapes", "five", 0.5, 320, "cuda"),
                                                              ("cocostuff27", "random", 0.7, 224, "host")]


@pytest.mark.parametrize("name,crop_type,ratio,res,location", CASES)
def test_crops_store_equals_cropped_tree(cuda_dev, trees, name, crop_type, ratio, res, location):
    from stego_b200.dataset import ResidentDataset
    root, f2c = trees[name]
    got = ResidentDataset.crops(root, name, crop_type, ratio, "train", res, location, batch_size=3,
                                fine_to_coarse=f2c)
    want = ResidentDataset.cropped(root, name, crop_type, ratio, "train", res, location, batch_size=7)
    torch.cuda.synchronize()
    assert got.n == want.n == got.count == want.count
    assert torch.equal(got.images.cpu(), want.images.cpu())
    for a, b in zip(got.frames(6), want.frames(6)):
        _batches_equal(a, b)
    nns = np.stack([np.roll(np.arange(got.n), -s) for s in range(4)], 1)
    for workers in (0, 2):
        ea, eb = got.batches(nns, 4, 3, seed=11, loader_workers=workers), want.batches(nns, 4, 3, seed=11,
                                                                                    loader_workers=workers)
        for _ in range(2):
            for a, b in zip(next(ea), next(eb)):
                _batches_equal(a, b)


def test_crops_store_with_loader_workers(cuda_dev, trees):
    from stego_b200.dataset import ResidentDataset
    root, _ = trees["cityscapes"]
    a = ResidentDataset.crops(root, "cityscapes", "random", 0.7, "train", 224, num_workers=2, batch_size=1)
    b = ResidentDataset.crops(root, "cityscapes", "random", 0.7, "train", 224, batch_size=4)
    torch.cuda.synchronize()
    assert torch.equal(a.images, b.images) and torch.equal(a.labels, b.labels)


def test_precompute_knns_on_both_stores(cuda_dev, trees):
    from stego_b200.config import make_cfg
    from stego_b200.dataset import ResidentDataset
    from stego_b200.knn import precompute_knns
    from stego_b200.modules import DinoFeaturizer
    cfg = make_cfg(random_backbone_init=True)
    torch.manual_seed(0)
    net = DinoFeaturizer(70, cfg).to(cuda_dev).eval()
    root, f2c = trees["cocostuff27"]
    got = ResidentDataset.crops(root, "cocostuff27", "five", 0.5, "train", 224, fine_to_coarse=f2c)
    want = ResidentDataset.cropped(root, "cocostuff27", "five", 0.5, "train", 224)
    assert torch.equal(precompute_knns(net, got.frames(4), k=5), precompute_knns(net, want.frames(4), k=5))
