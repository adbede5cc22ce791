"""GPU: the resident training set (stego_b200.dataset.ResidentDataset) against the reference loader's batches in
tests/golden/dataset.pt (oracle/make_golden_dataset.py), bit for bit.

  * every golden batch (2.5 epochs, W = 0, 1 and 3 loader workers, partial batches) is reproduced with torch.equal:
    img / img_pos, label / label_pos, mask / mask_pos with their dtypes and shapes, ind, ind_pos and seed; for the
    five-crop and directory layouts (with and without labels), res 32 and 30, the store on the device and in pinned
    host memory, fp32 frames and bf16 ones (the golden fp32 frame rounded to bf16);
  * the store's frames equal load_frames of the same decoded arrays, and precompute_knns over store.frames() equals it
    over load_frames batches;
  * a fused training step (shipped config plus use_salience, use_true_labels and the aug term fed by the seeds) on a
    store batch is bit-identical to one on the golden batch: the loss and the head parameters after the update (the
    probes within the run-to-run spread of their atomic gradient sums);
  * next() runs under torch.cuda.set_sync_debug_mode("error"): no synchronising call.
"""
import os

import pytest
import torch

from _parity_util import NAMES, make_model, params_of, rel
from test_dataset import load_gold

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "dataset.pt")
CASES = ["cropped_32", "cropped_30", "directory_32", "directory_30", "directory_unlabelled_32",
         "directory_unlabelled_30"]


@pytest.fixture(scope="module")
def gold():
    return load_gold(GOLD)


def _store(gold, case, location, dev):
    from stego_b200.dataset import ResidentDataset
    layout, res = case.rsplit("_", 1)
    kind = "cropped" if layout == "cropped" else "directory"
    has_labels = layout != "directory_unlabelled"
    images = [x.numpy() for x in gold["images"]]
    labels = [x.numpy() for x in gold["labels"]]
    store = ResidentDataset(len(images), int(res), kind, location, has_labels)
    for lo, hi in ((0, 5), (5, 6), (6, len(images))):  # several appends: rows land at r0 > 0
        store.append(images[lo:hi], labels[lo:hi] if has_labels else None)
    return store


def _expected(gold, case, idx, key, dtype=torch.float32):
    """The reference's rows `idx` of img / label / mask, in the dtypes it returned (img in `dtype`)."""
    rows = gold["cases"][case]["rows"]
    if key == "img":
        return gold["frames"][int(case.rsplit("_", 1)[1])][idx].to(dtype)
    return rows[key][idx].to(getattr(torch, rows[key + "_dtype"]))


def _run(store, gold, workers, n, dtype):
    out = []
    for epoch in store.batches(gold["nns"], gold["batch_size"], gold["num_neighbors"], gold["seed"],
                               loader_workers=workers, dtype=dtype):
        for b in epoch:
            out.append(b)
            if len(out) == n:
                return out


@pytest.mark.parametrize("location", ["cuda", "host"])
@pytest.mark.parametrize("case", CASES)
def test_batches_equal_reference_loader(cuda_dev, gold, case, location):
    store = _store(gold, case, location, cuda_dev)
    for workers in (0, 1, 3):
        want_run = gold["cases"][case]["runs"][workers]
        for dtype in (torch.float32, torch.bfloat16):
            got_run = _run(store, gold, workers, len(want_run), dtype)
            for want, got in zip(want_run, got_run):
                for k in ("ind", "ind_pos", "seed"):
                    assert got[k].device.type == "cpu" and got[k].dtype == torch.int64
                    assert torch.equal(got[k], want[k]), (case, workers, k)
                for key, ik in (("img", "ind"), ("img_pos", "ind_pos"), ("label", "ind"), ("label_pos", "ind_pos"),
                                ("mask", "ind"), ("mask_pos", "ind_pos")):
                    exp = _expected(gold, case, want[ik], key.replace("_pos", ""), dtype).to(cuda_dev)
                    assert got[key].is_cuda and got[key].dtype == exp.dtype and got[key].shape == exp.shape, \
                        (case, workers, key, got[key].dtype, exp.dtype, got[key].shape, exp.shape)
                    assert torch.equal(got[key], exp), (case, location, workers, dtype, key)


@pytest.mark.parametrize("location", ["cuda", "host"])
@pytest.mark.parametrize("res", [32, 30, 224])
def test_store_frames_equal_load_frames(cuda_dev, gold, location, res):
    from stego_b200.dataset import ResidentDataset
    from stego_b200.frames import load_frames, load_labels
    images = [x.numpy() for x in gold["images"]]
    labels = [x.numpy() for x in gold["labels"]]
    store = ResidentDataset(len(images), res, "directory", location)
    store.append(images, labels)
    got = list(store.frames(5))
    assert [b["img"].shape[0] for b in got] == [5, 5, 3]
    want = load_frames(images, res)
    assert torch.equal(torch.cat([b["img"] for b in got]), want)
    assert torch.equal(torch.cat([b["label"] for b in got]).squeeze(1), load_labels(labels, res))


def test_precompute_knns_on_the_store(cuda_dev, gold):
    from stego_b200.config import make_cfg
    from stego_b200.dataset import ResidentDataset
    from stego_b200.frames import load_frames
    from stego_b200.knn import precompute_knns
    from stego_b200.modules import DinoFeaturizer
    cfg = make_cfg(random_backbone_init=True)
    torch.manual_seed(0)
    net = DinoFeaturizer(70, cfg).to(cuda_dev).eval()
    images = [x.numpy() for x in gold["images"]]
    store = ResidentDataset(len(images), 224, "cropped")
    store.append(images, [x.numpy() for x in gold["labels"]])
    got = precompute_knns(net, store.frames(4), k=5)
    want = precompute_knns(net, [load_frames(images[i:i + 4], 224) for i in range(0, len(images), 4)], k=5)
    assert torch.equal(got, want)


def test_training_step_on_store_batch_is_bit_identical(cuda_dev, gold):
    case, res = "cropped_32", 32
    over = dict(res=res, use_salience=True, use_true_labels=True, aug_alignment_weight=0.6)
    store = _store(gold, case, "cuda", cuda_dev)
    got = _run(store, gold, 1, 1, torch.float32)[0]
    want_idx = gold["cases"][case]["runs"][1][0]
    golden = dict(ind=want_idx["ind"], ind_pos=want_idx["ind_pos"], seed=want_idx["seed"])
    for key, ik in (("img", "ind"), ("img_pos", "ind_pos"), ("label", "ind"), ("label_pos", "ind_pos"),
                    ("mask", "ind"), ("mask_pos", "ind_pos")):
        golden[key] = _expected(gold, case, want_idx[ik], key.replace("_pos", "")).to(cuda_dev)
    results = []
    for batch in (got, golden):
        model, _ = make_model("vit_small", cuda_dev, fused=True, **over)
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
def test_next_does_not_synchronise(cuda_dev, gold, location):
    store = _store(gold, "cropped_32", location, cuda_dev)
    epochs = store.batches(gold["nns"], 4, gold["num_neighbors"], gold["seed"], loader_workers=3)
    epoch = next(epochs)
    next(epoch)  # the first step sizes the record ring
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(2):
            b = next(epoch)
        epoch = next(epochs)
        for _ in range(3):
            b = next(epoch)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert b["img"].shape == (4, 3, 32, 32)
