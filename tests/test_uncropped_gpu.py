"""GPU: training batches from the uncropped classes (EvalSet.coco / cityscapes / potsdam "train",
ResidentDataset.directory) with the loader crops "center", "random" and None, against the reference loader's batches
in tests/golden/uncropped.pt (oracle/make_golden_uncropped.py), bit for bit.

  * every golden batch (2.5 epochs, W = 0 and 2 loader workers) is reproduced with torch.equal: img / img_pos in fp32
    and bf16 (the golden frame rounded), label / label_pos, mask / mask_pos with their dtypes and shapes, ind, ind_pos
    and seed; res 32 (the aligned-load path of the windowed gather) and 30 (its byte path), the store on the device and
    in pinned host memory;
  * windows at (0, 0) and at the far corner of every row;
  * frames() of a "random" store equals load_frames / load_labels with crop="center", and precompute_knns runs on it;
  * a fused training step on a Potsdam store batch is bit-identical to one on the golden batch (fp32 label > 0 mask,
    use_salience);
  * next() runs under torch.cuda.set_sync_debug_mode("error"); records outside the row table are refused on the host.
"""
import os

import numpy as np
import pytest
import torch

from _parity_util import NAMES, make_model, params_of, rel
from test_uncropped import load_gold

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "uncropped.pt")
CASES = [f"{layout}_{res}" for layout in ("cocostuff27", "cityscapes", "potsdam", "directory") for res in (32, 30)]


@pytest.fixture(scope="module")
def gold():
    return load_gold(GOLD)


@pytest.fixture(scope="module")
def tree(gold, tmp_path_factory):
    root = str(tmp_path_factory.mktemp("uncropped"))
    for rel_path, blob in gold["tree"].items():
        os.makedirs(os.path.dirname(os.path.join(root, rel_path)), exist_ok=True)
        with open(os.path.join(root, rel_path), "wb") as f:
            f.write(blob)
    return root


def _fine_to_coarse():
    return torch.load(os.path.join(ROOT, "tests", "golden", "evalset.pt"))["fine_to_coarse"]


def _store(gold, root, case, crop, location="cuda"):
    from stego_b200.dataset import ResidentDataset
    from stego_b200.evalset import EvalSet
    layout, res = case.rsplit("_", 1)
    res = int(res)
    if layout == "cocostuff27":
        return EvalSet.coco(root, "cocostuff27", "train", res, _fine_to_coarse(), location, crop=crop)
    if layout == "cityscapes":  # in the reference's os.listdir order
        images = [os.path.join(root, p) for p in gold["cases"][case]["paths"]]
        labels = [p.replace("/leftImg8bit/", "/gtFine/").split("_leftImg8bit")[0] + "_gtFine_labelIds.png"
                  for p in images]
        return EvalSet._from_files(images, labels, "pil", res, "cityscapes", location, 64, 0, crop=crop)
    if layout == "potsdam":
        return EvalSet.potsdam(root, "train", res, location, crop=crop)
    return ResidentDataset.directory(root, "myset", "train", res, location, crop=crop)


def _frame(values, b):
    return torch.stack([values[c][b[c].long()] for c in range(3)])


def _expected(gold, case, crop, i, window=None):
    """(img fp32, label int64, mask) of index i as the reference returns it, window (top, left, label top, label left)
    for "random"."""
    c = gold["cases"][case]
    res = int(case.rsplit("_", 1)[1])
    rows = c["squashed" if crop is None else "full"]
    img, lab, m = _frame(gold["values"], rows["img"][i]), rows["label"][i], rows["mask"][i]
    if crop is None:
        return img, lab, m
    if window is None:
        window = [int(round((s - res) / 2.0)) for s in tuple(img.shape[-2:]) + tuple(lab.shape[-2:])]
    t, l, lt, ll = (int(v) for v in window)
    return (img[..., t:t + res, l:l + res], lab[..., lt:lt + res, ll:ll + res], m[..., lt:lt + res, ll:ll + res])


def _check_batch(gold, case, crop, b, want_draws, dtype):
    B = want_draws.shape[0]
    assert b["ind"].tolist() == want_draws[:, 0].tolist()
    assert b["ind_pos"].tolist() == want_draws[:, 1].tolist()
    assert b["seed"].tolist() == want_draws[:, 2].tolist()
    for side, ik, w0 in (("", 0, 3), ("_pos", 1, 7)):
        rows = [_expected(gold, case, crop, int(want_draws[j, ik]),
                          want_draws[j, w0:w0 + 4] if crop == "random" else None) for j in range(B)]
        img, label, mask = (torch.stack([r[k] for r in rows]) for k in range(3))
        got_img = b["img" + side].cpu()
        assert got_img.dtype == dtype and torch.equal(got_img, img.to(dtype)), ("img" + side)
        assert torch.equal(b["label" + side].cpu(), label), ("label" + side)
        got_mask = b["mask" + side].cpu()
        assert got_mask.dtype == mask.dtype and torch.equal(got_mask, mask), ("mask" + side)


@pytest.mark.parametrize("location", ["cuda", "host"])
@pytest.mark.parametrize("crop", ["center", "random", None])
@pytest.mark.parametrize("case", CASES)
def test_batches_match_reference_loader(cuda_dev, gold, tree, case, crop, location):
    store = _store(gold, tree, case, crop, location)
    for W in (0, 2):
        run = gold["cases"][case]["runs"][(crop, W)]
        parts = torch.split(run["draws"], run["sizes"])
        for dtype in (torch.float32, torch.bfloat16):
            got = []
            for epoch in store.batches(gold["nns"], gold["batch_size"], gold["num_neighbors"], gold["seed"],
                                       loader_workers=W, dtype=dtype):
                for b in epoch:
                    got.append(b)
                    if len(got) == len(parts):
                        break
                if len(got) == len(parts):
                    break
            for b, want in zip(got, parts):
                _check_batch(gold, case, crop, b, want, dtype)


@pytest.mark.parametrize("case", ["cityscapes_30", "cityscapes_32", "directory_30"])
def test_edge_windows(cuda_dev, gold, tree, case):
    """Each row read at window (0, 0) and at its far corner (oh - res, ow - res), label likewise."""
    store = _store(gold, tree, case, "random")
    res = store.res
    index = np.arange(store.n, dtype=np.int64)
    for far in (False, True):
        windows = (np.stack([store.sizes[:, 0] - res, store.sizes[:, 1] - res, store.sizes[:, 2] - res,
                             store.sizes[:, 3] - res], 1) if far else np.zeros((store.n, 4), np.int64))
        img, label, mask = store._gather(index, torch.float32, windows)
        label, mask = store._shaped(label, mask)
        for i in range(store.n):
            want = _expected(gold, case, "random", i, windows[i])
            assert torch.equal(img[i].cpu(), want[0]), (i, far)
            assert torch.equal(label[i].cpu(), want[1]), (i, far)
            assert torch.equal(mask[i].cpu(), want[2]), (i, far)


def test_frames_of_a_random_store_are_the_center_frames(cuda_dev, gold, tree):
    from stego_b200.config import make_cfg
    from stego_b200.evalset import _EvalFiles, coco_files, label_table
    from stego_b200.frames import load_frames, load_labels
    from stego_b200.knn import precompute_knns
    from stego_b200.modules import DinoFeaturizer
    f2c = _fine_to_coarse()
    store = _store(gold, tree, "cocostuff27_30", "random")
    files = _EvalFiles(*coco_files(tree, "cocostuff27", "train"), "pil")
    images, labels = zip(*[files[i] for i in range(len(files))])
    got = list(store.frames(4))
    img = torch.cat([b["img"] for b in got])
    label = torch.cat([b["label"] for b in got])
    assert torch.equal(img, load_frames(list(images), 30, crop="center"))
    assert torch.equal(label, load_labels(list(labels), 30, crop="center", lut=label_table("cocostuff27", f2c)))
    cfg = make_cfg(random_backbone_init=True)
    torch.manual_seed(0)
    net = DinoFeaturizer(70, cfg).to(cuda_dev).eval()
    big = _store(gold, tree, "cocostuff27_32", "random")
    nns = precompute_knns(net, big.frames(4), k=3)
    assert nns.shape == (big.n, 3)


def test_training_step_on_store_batch_is_bit_identical(cuda_dev, gold, tree):
    case = "potsdam_32"
    store = _store(gold, tree, case, "random")
    run = gold["cases"][case]["runs"][("random", 0)]
    want = torch.split(run["draws"], run["sizes"])[0]
    got = next(next(store.batches(gold["nns"], gold["batch_size"], gold["num_neighbors"], gold["seed"])))
    golden = dict(ind=want[:, 0].clone(), ind_pos=want[:, 1].clone(), seed=want[:, 2].clone())
    for side, ik, w0 in (("", 0, 3), ("_pos", 1, 7)):
        rows = [_expected(gold, case, "random", int(want[j, ik]), want[j, w0:w0 + 4]) for j in range(want.shape[0])]
        for k, key in enumerate(("img", "label", "mask")):
            golden[key + side] = torch.stack([r[k] for r in rows]).to(cuda_dev)
    assert golden["mask"].dtype == torch.float32
    results = []
    for batch in (got, golden):
        model, _ = make_model("vit_small", cuda_dev, fused=True, res=32, use_salience=True)
        torch.manual_seed(777)
        loss = model.training_step(batch, 0)
        assert model._fused is not None and model._fused.step_idx == 1, "the fused step did not run"
        torch.cuda.synchronize()
        results.append((loss.detach().clone(), params_of(model)))
    assert torch.equal(results[0][0], results[1][0])
    for k in NAMES:
        if k.startswith("net."):
            assert torch.equal(results[0][1][k], results[1][1][k]), k
        else:  # the probes' weight gradients are fp32 atomic sums, whose order differs from run to run
            assert rel(results[0][1][k], results[1][1][k]) < 1e-6, k


@pytest.mark.parametrize("location", ["cuda", "host"])
def test_next_does_not_synchronise(cuda_dev, gold, tree, location):
    store = _store(gold, tree, "cityscapes_32", "random", location)
    epochs = store.batches(gold["nns"], 4, gold["num_neighbors"], gold["seed"], loader_workers=2)
    epoch = next(epochs)
    next(epoch)  # the first step sizes the record ring
    torch.cuda.set_sync_debug_mode("error")
    try:
        b = next(epoch)
        epoch = next(epochs)
        for _ in range(2):
            b = next(epoch)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert b["img"].shape == (2, 3, 32, 32)  # the epoch's last batch: 6 samples in batches of 4


def test_refusals(cuda_dev, gold, tree):
    from stego_b200.dataset import ResidentDataset
    store = _store(gold, tree, "directory_30", "random")
    with pytest.raises(ValueError, match="res=32"):
        next(store.batches(gold["nns"], 4, 1, 0, res=32))
    far = np.array([[int(store.sizes[0, 0]) - 29, 0, 0, 0]], dtype=np.int64)
    with pytest.raises(RuntimeError, match="window"):
        store._gather(np.array([0], dtype=np.int64), torch.float32, far)
    with pytest.raises(RuntimeError, match="row"):
        store._gather(np.array([store.n], dtype=np.int64), torch.float32, np.zeros((1, 4), np.int64))
    with pytest.raises(ValueError, match="crop"):
        ResidentDataset(4, 32, "directory", crop="left")
    with pytest.raises(ValueError, match="sizes"):
        ResidentDataset(4, 32, "directory", crop="random")
    with pytest.raises(ValueError, match="sizes"):
        ResidentDataset(4, 32, "directory", sizes=np.ones((4, 4)))
    torch.cuda.synchronize()


def test_abi_symbols():
    from stego_b200 import _lib
    protos = _lib.header_prototypes()
    lib = _lib.load()
    for name in ("stego_store_batch_window", "stego_store_rows_u8"):
        assert name in protos and hasattr(lib, name)
