"""The cropped training sets on the host: the JPEG oracle against Pillow's own round trip, the crop windows against
torchvision and the reference's rule, the written tree against what the reference's crop script writes, refusals.

  * oracle/jpeg_oracle.py equals np.asarray(Image.open(saved).convert("RGB")) of Pillow's default save byte for byte
    on every corpus size (1 x 1 up to 512 x 1024 and 1 x 2048, odd and non-multiple-of-16 sides) and content (noise,
    flat, saturated, grayscale as RGB, gradients);
  * libjpeg's reciprocal quantisation gives the same integers as the oracle's rounded division;
  * crop_windows equals five_crop / crop on tensors and tests/golden/crop_windows.pt (oracle/make_golden_crops.py);
  * write_cropped writes the reference's names, label + 1 PNGs and JPEGs byte-equal to a live Pillow save of the crop.
"""
import io
import os
import sys

import numpy as np
import pytest
import torch
from PIL import Image

from _crops_util import CONTENTS, CORPUS_SIZES, ROOT, corpus_image, fine_to_coarse, make_cityscapes_tree, make_coco_tree

sys.path.insert(0, os.path.join(ROOT, "oracle"))
import jpeg_oracle  # noqa: E402

from stego_b200 import crops, evalset  # noqa: E402


def pillow_roundtrip(rgb: np.ndarray) -> np.ndarray:
    f = io.BytesIO()
    Image.fromarray(rgb).save(f, "JPEG")
    f.seek(0)
    with Image.open(f) as im:
        return np.asarray(im.convert("RGB"))


@pytest.mark.parametrize("size", CORPUS_SIZES, ids=lambda s: f"{s[0]}x{s[1]}")
@pytest.mark.parametrize("content", CONTENTS)
def test_jpeg_oracle_equals_pillow(size, content):
    img = corpus_image(*size, content)
    got = jpeg_oracle.roundtrip(img)
    assert got.shape == img.shape and got.dtype == np.uint8
    np.testing.assert_array_equal(got, pillow_roundtrip(img))


def test_jpeg_oracle_every_small_size():
    rng = np.random.default_rng(3)
    for h in range(1, 21):
        for w in range(1, 21):
            img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
            np.testing.assert_array_equal(jpeg_oracle.roundtrip(img), pillow_roundtrip(img), err_msg=f"{h} x {w}")


def test_reciprocal_quantisation_is_division():
    """libjpeg-turbo quantises with 16-bit reciprocals (compute_reciprocal): equal to rounding |x| / d half up."""
    x = np.arange(0, 1 << 15, dtype=np.int64)
    for q in np.unique(np.concatenate([jpeg_oracle.LUMA_Q.ravel(), jpeg_oracle.CHROMA_Q.ravel(), np.arange(1, 256)])):
        d = int(8 * q)
        b = d.bit_length() - 1
        r = 16 + b
        fq, fr, c = (1 << r) // d, (1 << r) % d, d // 2
        if fr == 0:
            fq, r = fq >> 1, r - 1
        elif fr <= d // 2:
            c += 1
        else:
            fq += 1
        got = ((x + c) * fq) >> r
        want = jpeg_oracle.quantize(x, np.int64(q))
        np.testing.assert_array_equal(got, want, err_msg=f"q={q}")
        np.testing.assert_array_equal(jpeg_oracle.quantize(-x, np.int64(q)), -want)


def test_quality_75_tables():
    assert jpeg_oracle.LUMA_Q[0].tolist() == [8, 6, 5, 8, 12, 20, 26, 31]
    assert jpeg_oracle.CHROMA_Q[0].tolist() == [9, 9, 12, 24, 50, 50, 50, 50]
    assert jpeg_oracle.CHROMA_Q.max() == 50 and jpeg_oracle.LUMA_Q.min() == 5


# ---- crop windows ----------------------------------------------------------------------------------------------------
def _windows_by_torchvision(H, W, crop_type, ratio, item):
    import torchvision.transforms.functional as TF
    img = torch.arange(H * W).view(1, H, W)
    size = [int(H * ratio), int(W * ratio)]
    if crop_type == "five":
        parts = TF.five_crop(img, size)
    else:
        parts = [TF.crop(img, hash((item, i, 0)) % (H - size[0]), hash((item, i, 1)) % (W - size[1]), *size)
                 for i in range(5)]
    return [(int(p[0, 0, 0]) // W, int(p[0, 0, 0]) % W, p.shape[1], p.shape[2]) for p in parts]


@pytest.mark.parametrize("crop_type", ["five", "random"])
@pytest.mark.parametrize("size", [(480, 640), (427, 640), (33, 17), (4, 3), (1024, 2048)])
@pytest.mark.parametrize("ratio", [0.5, 0.7, 0.9])
def test_crop_windows_equal_torchvision(crop_type, size, ratio):
    for item in (0, 3, 12345):
        want = _windows_by_torchvision(*size, crop_type, ratio, item)
        assert crops.crop_windows(*size, crop_type, ratio, item) == want


def test_crop_windows_golden():
    gold = torch.load(os.path.join(ROOT, "tests", "golden", "crop_windows.pt"), weights_only=False)
    assert gold["libjpeg_turbo"]  # the libjpeg-turbo the JPEG oracle was pinned against
    for case in gold["cases"]:
        args = (*case["size"], case["crop_type"], case["ratio"], case["item"])
        if case["windows"] is None:
            with pytest.raises(ValueError, match="divides by zero"):
                crops.crop_windows(*args)
        else:
            assert crops.crop_windows(*args) == [tuple(w) for w in case["windows"]], case


def test_crop_windows_refusals():
    with pytest.raises(ValueError, match="empty"):
        crops.crop_windows(1, 40, "five", 0.5, 0)
    with pytest.raises(ValueError, match="divides by zero"):
        crops.crop_windows(40, 40, "random", 1.0, 0)
    with pytest.raises(ValueError, match="crop_type"):
        crops.crop_windows(40, 40, "ten", 0.5, 0)


# ---- the written tree ------------------------------------------------------------------------------------------------
def _jpeg_bytes(rgb: np.ndarray) -> bytes:
    f = io.BytesIO()
    Image.fromarray(rgb).save(f, "JPEG")
    return f.getvalue()


def _crop_like_reference(rgb: np.ndarray, top, left, h, w) -> np.ndarray:
    """RandomCropComputer's image bytes: ToTensor, crop, mul(255).add_(0.5).clamp_(0, 255) to uint8."""
    import torchvision.transforms as T
    t = T.ToTensor()(Image.fromarray(rgb))[:, top:top + h, left:left + w]
    return t.mul(255).add_(0.5).clamp_(0, 255).permute(1, 2, 0).to(torch.uint8).numpy()


@pytest.mark.parametrize("dataset_name", ["cocostuff27", "cityscapes"])
@pytest.mark.parametrize("crop_type", ["five", "random"])
def test_write_cropped_matches_reference_files(tmp_path, dataset_name, crop_type):
    root = str(tmp_path)
    (make_coco_tree if dataset_name == "cocostuff27" else make_cityscapes_tree)(root, "train")
    f2c = fine_to_coarse() if dataset_name == "cocostuff27" else None
    base = crops.write_cropped(root, dataset_name, crop_type, 0.7, "train", fine_to_coarse=f2c)
    assert base == os.path.join(root, "cropped", f"{dataset_name}_{crop_type}_crop_0.7")
    images, labels = crops.source_files(root, dataset_name, "train")
    table = evalset.label_table(dataset_name, f2c).numpy()
    n = 5 * len(images)
    assert sorted(os.listdir(os.path.join(base, "img", "train"))) == sorted(f"{i}.jpg" for i in range(n))
    assert sorted(os.listdir(os.path.join(base, "label", "train"))) == sorted(f"{i}.png" for i in range(n))
    for item, (ip, lp) in enumerate(zip(images, labels)):
        with Image.open(ip) as im:
            rgb = np.asarray(im.convert("RGB"))
        with Image.open(lp) as im:
            raw = np.asarray(im)
        for k, (top, left, h, w) in enumerate(crops.crop_windows(*rgb.shape[:2], crop_type, 0.7, item)):
            i = item * 5 + k
            with open(os.path.join(base, "img", "train", f"{i}.jpg"), "rb") as f:
                assert f.read() == _jpeg_bytes(_crop_like_reference(rgb, top, left, h, w)), (item, k)
            with Image.open(os.path.join(base, "label", "train", f"{i}.png")) as im:
                got = np.asarray(im)
            want = (table[raw[top:top + h, left:left + w]] + 1).astype(np.uint8)
            np.testing.assert_array_equal(got, want)
            # CroppedDataset's label (byte - 1) is the class's label of the source byte
            np.testing.assert_array_equal(got.astype(np.int64) - 1, table[raw[top:top + h, left:left + w]])


def test_reference_byte_conversion_is_identity():
    """The crop script's mul(255).add_(0.5) of ToTensor's x / 255 returns every byte unchanged, so the store may stage
    the decoded bytes as they are."""
    x = np.arange(256, dtype=np.uint8).reshape(16, 16, 1).repeat(3, 2)
    np.testing.assert_array_equal(_crop_like_reference(x, 0, 0, 16, 16), x)


def test_refusals(tmp_path):
    root = make_coco_tree(str(tmp_path))
    with pytest.raises(ValueError, match="dataset_name"):
        crops.write_cropped(root, "potsdam", "five", 0.5, "train")
    with pytest.raises(ValueError, match="crop_type"):
        crops.write_cropped(root, "cityscapes", "six", 0.5, "train")
    for bad in (0, 1.5, -0.5, True, "0.5"):
        with pytest.raises(ValueError, match="crop_ratio"):
            crops.write_cropped(root, "cityscapes", "five", bad, "train")
    with pytest.raises(ValueError, match="fine_to_coarse"):
        crops.write_cropped(root, "cocostuff27", "five", 0.5, "train")
    from stego_b200.dataset import ResidentDataset
    with pytest.raises(ValueError, match="dataset_name"):
        ResidentDataset.crops(root, "cocostuff15", "five", 0.5, "train", 224)
    with pytest.raises(ValueError, match="fine_to_coarse"):
        ResidentDataset.crops(root, "cocostuff27", "five", 0.5, "train", 224)
    with pytest.raises(ValueError, match="crop_type"):
        ResidentDataset.crops(root, "cityscapes", None, 0.5, "train", 224)
    with pytest.raises(ValueError, match="image_set"):
        crops.write_cropped(root, "cityscapes", "five", 0.5, "nope")
