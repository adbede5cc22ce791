"""GPU: loader frames and labels built on the device (stego_b200.frames) and the folder demo (stego_b200.demo) against
the host route the reference takes.

  * load_frames is torch.equal to torchvision's Resize(NEAREST) / CenterCrop / ToTensor / Normalize of the same PIL
    images over 200+ seeded size pairs at res 224 and 320 (1 x 1, exactly res, portrait and landscape, 4000 x 3000,
    sizes where floor((x + .5) in / out) is not Pillow's index), and with crop None;
  * load_labels with each remap table equals the reference's loaders (tests/golden/frames.pt) and the reference's
    COCO-Stuff remap loop on torchvision's label transform;
  * eval_step on load_frames output equals eval_step on host-built frames, with and without the CRF: predictions,
    probabilities and both confusion matrices;
  * segment_folder writes the same PNG bytes as the host-built-frames route;
  * a call is one host-to-device copy, one launch, no device-to-host copy and no synchronisation.
"""
import io
import os
import sys

import numpy as np
import pytest
import torch
import torchvision.transforms as T
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from _parity_util import make_model  # noqa: E402
from test_frames import CASES, GOLD, _want, all_luts, coco_luts  # noqa: E402

from stego_b200 import _lib, demo, frames  # noqa: E402

pytestmark = pytest.mark.gpu


def host_transform(res, crop="center", is_label=False):
    """get_transform(res, is_label, crop) of src/utils.py:165-183, built from torchvision as the reference builds it."""
    size = res if crop is not None else (res, res)
    steps = [T.Resize(size, Image.NEAREST)] + ([T.CenterCrop(res)] if crop is not None else [])
    if is_label:
        return T.Compose(steps + [T.Lambda(lambda t: torch.as_tensor(np.array(t), dtype=torch.int64).unsqueeze(0))])
    return T.Compose(steps + [T.ToTensor(), T.Normalize(frames.MEAN, frames.STD)])


def _size_pairs(res):
    rng = np.random.default_rng(res)
    fixed = [(1, 1), (res, res), (res, res + 1), (res + 3, res), (res - 1, res + 7), (480, 640), (640, 480),
             (3000, 4000), (4000, 3000), (1024, 2048), (2, 7), (8, 7), (7, 2), (14, 3203), (3203, 14), (3, 4), (3, 14)]
    rand = [tuple(int(x) for x in rng.integers(1, 1400, 2)) for _ in range(100 - len(fixed))]
    return fixed + rand


def _rgb(rng, h, w):
    return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)


@pytest.mark.parametrize("res", [224, 320])
def test_load_frames_equals_torchvision(cuda_dev, res):
    rng = np.random.default_rng(res + 1)
    pairs = _size_pairs(res)
    images = [_rgb(rng, h, w) for h, w in pairs]
    for crop in ("center", None):
        tf = host_transform(res, crop)
        for k in range(0, len(images), 25):
            chunk = images[k:k + 25]
            got = frames.load_frames(chunk, res, crop=crop)
            want = torch.stack([tf(Image.fromarray(x)) for x in chunk])
            assert got.device == cuda_dev and got.dtype == torch.float32 and got.shape == want.shape
            for j in range(len(chunk)):
                assert torch.equal(got[j].cpu().view(torch.int32), want[j].view(torch.int32)), (crop, pairs[k + j])


def test_load_frames_takes_tensors_and_the_fixture(cuda_dev):
    """The reference's own frames (fixture), from CPU tensors, one case per call and all sizes of a res in one call."""
    for c in CASES:
        got = frames.load_frames([c["image"]], c["res"], crop=c["crop"])
        assert torch.equal(got[0].cpu().view(torch.int32), c["frame"].view(torch.int32)), (c["H"], c["W"])
    group = [c for c in CASES if c["res"] == 40 and c["crop"]]
    got = frames.load_frames([c["image"] for c in group], 40).cpu()
    assert torch.equal(got.view(torch.int32), torch.stack([c["frame"] for c in group]).view(torch.int32))


def test_load_labels_equals_reference_remaps(cuda_dev):
    luts = all_luts()
    for res in (32, 40, 56):
        cases = [c for c in CASES if c["res"] == res]
        for crop in ("center", None):
            group = [c for c in cases if c["crop"] == crop]
            if not group:
                continue
            for key, lut in luts.items():
                got = frames.load_labels([c["label"] for c in group], res, crop=crop, lut=lut)
                assert got.dtype == torch.int64 and got.shape == (len(group), res, res)
                for j, c in enumerate(group):
                    assert np.array_equal(got[j].cpu().numpy(), _want(c, key)), (key, c["H"], c["W"])
    # the reference's COCO-Stuff loop (src/data.py:303-309) on torchvision's label transform, larger maps
    f2c = GOLD["coco"]["fine_to_coarse"]
    rng = np.random.default_rng(3)
    labs = [rng.integers(0, 256, (h, w), dtype=np.uint8) for h, w in _size_pairs(320)[:40]]
    got = frames.load_labels(labs, 320, lut=frames.label_lut(f2c))
    tf = host_transform(320, is_label=True)
    for j, lab in enumerate(labs):
        label = tf(Image.fromarray(lab, mode="L")).squeeze(0)
        label[label == 255] = -1
        coarse = torch.zeros_like(label)
        for fine, c in f2c.items():
            coarse[label == fine] = c
        coarse[label == -1] = -1
        assert torch.equal(got[j].cpu(), coarse), lab.shape
    ident = frames.load_labels(labs[:5], 320)
    for j in range(5):
        assert torch.equal(ident[j].cpu(), tf(Image.fromarray(labs[j], mode="L"))[0])


def test_one_copy_one_launch_no_sync(cuda_dev):
    rng = np.random.default_rng(11)
    images = [_rgb(rng, h, w) for h, w in ((480, 640), (640, 427), (333, 500))]
    labels = [x[..., 0].copy() for x in images]
    lut = frames.label_lut({i: i % 27 for i in range(255)})
    frames.load_frames(images, 320)
    frames.load_labels(labels, 320, lut=lut)  # warm the pinned and device allocators
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    for call in (lambda: frames.load_frames(images, 320), lambda: frames.load_labels(labels, 320, lut=lut)):
        n0 = _lib.launch_count()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            torch.cuda.set_sync_debug_mode("error")  # raises on a synchronisation or a device-to-host copy
            try:
                call()
            finally:
                torch.cuda.set_sync_debug_mode(0)
            torch.cuda.synchronize()
        assert _lib.launch_count() - n0 == 1
        names = [e.name for e in prof.events()]
        assert sum("HtoD" in n for n in names) == 1, names
        assert not any("DtoH" in n for n in names), names


def _model(dev):
    model, _ = make_model("vit_small", dev, fused=True, seed=0)
    return model


def _confusions(model):
    return model.test_linear_metrics.stats.clone(), model.test_cluster_metrics.stats.clone()


@pytest.mark.parametrize("run_crf", [False, True])
def test_eval_step_on_device_frames(cuda_dev, run_crf):
    res = 96
    rng = np.random.default_rng(21)
    images = [_rgb(rng, h, w) for h, w in ((120, 160), (96, 96), (200, 97), (75, 300))]
    labels = [rng.integers(0, 256, x.shape[:2], dtype=np.uint8) for x in images]
    lut = coco_luts()["coco27"]
    model = _model(cuda_dev)
    outs = []
    for route in ("device", "host"):
        model.test_linear_metrics.reset()
        model.test_cluster_metrics.reset()
        if route == "device":
            img, label = frames.load_frames(images, res), frames.load_labels(labels, res, lut=lut)
        else:
            img = torch.stack([host_transform(res)(Image.fromarray(x)) for x in images]).to(cuda_dev)
            ids = torch.stack([host_transform(res, is_label=True)(Image.fromarray(x, mode="L"))[0] for x in labels])
            label = lut[ids].to(cuda_dev)
        out = model.eval_step(dict(img=img, label=label), run_crf=run_crf, want_probs=True)
        torch.cuda.synchronize()
        outs.append(({k: v.clone() for k, v in out.items()}, _confusions(model)))
    (a, ca), (b, cb) = outs
    assert set(a) == {"linear_preds", "cluster_preds", "linear_probs", "cluster_probs"}
    for k in a:
        assert torch.equal(a[k], b[k]), k
    assert torch.equal(ca[0], cb[0]) and torch.equal(ca[1], cb[1]) and int(ca[0].sum()) > 0


def _write_folder(path, rng):
    """12 files, JPEG and PNG, mixed sizes and orientations."""
    sizes = [(120, 160), (160, 120), (96, 96), (97, 230), (300, 101), (64, 200), (150, 150), (99, 98), (240, 320),
             (320, 240), (111, 222), (80, 80)]
    for k, (h, w) in enumerate(sizes):
        im = Image.fromarray(_rgb(rng, h, w))
        if k % 3 == 2:
            im = im.convert("L")  # a grey file: converted to RGB on decoding
        ext = "jpg" if k % 2 else "png"
        im.save(os.path.join(path, f"img.{k}.{ext}"))


def test_segment_folder_matches_host_route(cuda_dev, tmp_path):
    res, batch_size = 96, 4
    src = tmp_path / "images"
    src.mkdir()
    _write_folder(str(src), np.random.default_rng(5))
    model = _model(cuda_dev)
    written = demo.segment_folder(model, str(src), str(tmp_path / "gpu"), res=res, batch_size=batch_size,
                                  num_workers=2)
    names = os.listdir(str(src))
    assert written == [demo.png_name(n) for n in names] and len(set(written)) == 12
    # the host route: demo_segmentation.py's transform on PIL images, the same eval_step, the same PNG writer
    tf = host_transform(res)
    for sub in ("linear", "cluster"):
        os.makedirs(str(tmp_path / "host" / sub))
    for k in range(0, len(names), 2 * batch_size):
        chunk = names[k:k + 2 * batch_size]
        img = torch.stack([tf(Image.open(str(src / n)).convert("RGB")) for n in chunk]).to(cuda_dev)
        out = model.eval_step(dict(img=img), run_crf=True)
        for j, n in enumerate(chunk):
            for sub, key in (("linear", "linear_preds"), ("cluster", "cluster_preds")):
                Image.fromarray(out[key][j].cpu().numpy()).save(str(tmp_path / "host" / sub / demo.png_name(n)))
    for stem in written:
        for sub in ("linear", "cluster"):
            got = (tmp_path / "gpu" / sub / stem).read_bytes()
            want = (tmp_path / "host" / sub / stem).read_bytes()
            assert got == want, (sub, stem)
            assert Image.open(io.BytesIO(got)).size == (res, res)
