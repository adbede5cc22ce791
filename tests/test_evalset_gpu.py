"""GPU: the resident evaluation sets (stego_b200.evalset.EvalSet) against the reference's validation loader in
tests/golden/evalset.pt (oracle/make_golden_evalset.py), bit for bit, and validate() / eval_step on their batches.

  * every fixture batch (DataLoader(batch_size=3, shuffle=False), partial last batch) is reproduced with torch.equal:
    ind, img, label and mask with their dtypes and shapes, and no mask with mask=False; for Coco (cocostuff27 / 15 / 3),
    CityscapesSeg, Potsdam and PotsdamRaw built from the fixture's files, res 32 and 30, the store on the device and in
    pinned host memory, fp32 frames and bf16 ones (the fixture's fp32 frame rounded to bf16);
  * frames() runs under torch.cuda.set_sync_debug_mode("error");
  * validate() on a store gives the confusion counts and metrics of the validation_step loop over load_frames /
    load_labels batches of the same files;
  * a 2-process validate() over the padded DistributedSampler shards sums to the one-process counts of those shards
    (tests/ddp_evalset_worker.py);
  * eval_step(run_crf=True) on store batches equals eval_step on the fixture's batches.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
from PIL import Image

from test_evalset import KINDS, expected_rows, listing, load_gold, write_tree

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def gold():
    return load_gold()


@pytest.fixture(scope="module")
def tree(gold, tmp_path_factory):
    root = str(tmp_path_factory.mktemp("evalset_tree"))
    write_tree(gold, root)
    return root


def build(gold, tree, kind, res, location):
    from stego_b200.evalset import EvalSet
    if kind.startswith("cocostuff"):
        return EvalSet.coco(tree, kind, "val", res, gold["fine_to_coarse"], location, batch_size=2)
    if kind == "cityscapes":
        return EvalSet.cityscapes(tree, "val", res, location, batch_size=2)
    if kind == "potsdam":
        return EvalSet.potsdam(tree, "val", res, location, batch_size=2)
    return EvalSet.potsdamraw(tree, res, location, batch_size=256, num_workers=4)


def expected(gold, kind, res, rows, dtype):
    case = gold["cases"][f"{kind}_{res}"]
    return (case["img"][rows].to(dtype), case["label"][rows].to(getattr(torch, case["label_dtype"])),
            case["mask"][rows].to(getattr(torch, case["mask_dtype"])))


@pytest.mark.parametrize("location", ["cuda", "host"])
@pytest.mark.parametrize("res", [32, 30])
@pytest.mark.parametrize("kind", KINDS)
def test_batches_equal_reference_loader(cuda_dev, gold, tree, kind, res, location):
    store = build(gold, tree, kind, res, location)
    images, _ = listing(tree, kind)
    rows = expected_rows(gold, kind, res, [os.path.relpath(p, tree) for p in images])
    assert store.n == len(images) == rows.numel()
    B = gold["batch_size"]
    for dtype in (torch.float32, torch.bfloat16):
        for mask in (True, False):
            got = list(store.frames(B, dtype, mask=mask))
            assert [b["ind"].numel() for b in got] == [min(B, store.n - s) for s in range(0, store.n, B)]
            for k, b in enumerate(got):
                ind = torch.arange(k * B, k * B + b["ind"].numel())
                assert b["ind"].device.type == "cpu" and b["ind"].dtype == torch.int64 and torch.equal(b["ind"], ind)
                assert set(b) == ({"ind", "img", "label", "mask"} if mask else {"ind", "img", "label"})
                want = dict(zip(("img", "label", "mask"), expected(gold, kind, res, rows[ind], dtype)))
                for key in ("img", "label", "mask") if mask else ("img", "label"):
                    g, w = b[key], want[key].to(cuda_dev)
                    assert g.is_cuda and g.dtype == w.dtype and g.shape == w.shape, (key, g.dtype, w.dtype, g.shape,
                                                                                     w.shape)
                    assert torch.equal(g, w), (kind, res, location, dtype, key, k)


@pytest.mark.parametrize("location", ["cuda", "host"])
def test_frames_do_not_synchronise(cuda_dev, gold, tree, location):
    store = build(gold, tree, "cityscapes", 32, location)
    it = store.frames(2, rank=1, world_size=2)
    next(it)  # the first batch sizes the record ring
    torch.cuda.set_sync_debug_mode("error")
    try:
        rest = list(it)
        more = list(store.frames(2, torch.bfloat16, rank=1, world_size=2))
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert len(rest) == 1 and len(more) == 2 and more[0]["mask"].shape == (2, 1, 32, 32)


def _snapshot_counts(model):
    """The two validation confusion matrices as validation_epoch_end sees them just before its reset."""
    seen = {}
    for name in ("linear_metrics", "cluster_metrics"):
        m = getattr(model, name)
        reset = m.reset

        def snap(m=m, reset=reset, name=name):
            seen[name] = m.stats.clone()
            reset()
        m.reset = snap
    return seen


def _decoded(tree, kind):
    images, labels = listing(tree, kind)
    out_i, out_l = [], []
    for ip, lp in zip(images, labels):
        with Image.open(ip) as im:
            out_i.append(np.array(im.convert("RGB")))
        with Image.open(lp) as im:
            out_l.append(np.array(im))
    return out_i, out_l


@pytest.mark.parametrize("location", ["cuda", "host"])
@pytest.mark.parametrize("kind", ["cocostuff27", "cityscapes"])
def test_validate_equals_validation_step_loop(cuda_dev, gold, tree, kind, location):
    from _parity_util import make_model
    from stego_b200.evalset import label_table
    from stego_b200.frames import load_frames, load_labels
    res, B = 32, 2
    store = build(gold, tree, kind, res, location)
    lut = label_table(kind, gold["fine_to_coarse"] if kind.startswith("coco") else None)
    images, labels = _decoded(tree, kind)
    results = []
    for use_store in (True, False):
        model, _ = make_model("vit_small", cuda_dev, fused=True, seed=0)
        seen = _snapshot_counts(model)
        if use_store:
            metrics = model.validate(store, B)
            assert model.last_validation_preview["img"].shape[0] == B
        else:
            for i in range(0, len(images), B):
                batch = dict(img=load_frames(images[i:i + B], res), label=load_labels(labels[i:i + B], res, lut=lut))
                model.validation_step(batch, i // B)
            metrics = model.validation_epoch_end([])
        results.append((seen["linear_metrics"], seen["cluster_metrics"], metrics))
    assert results[0][0].sum() > 0
    assert torch.equal(results[0][0], results[1][0]) and torch.equal(results[0][1], results[1][1])
    assert results[0][2] == results[1][2]


def test_ddp_validate_sums_to_one_process_counts(cuda_dev):
    world = 2
    port = 29800 + os.getpid() % 90
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr",
           "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tests", "ddp_evalset_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    lines = [json.loads(l.split(" ", 1)[1]) for l in r.stdout.splitlines() if l.startswith("DDP_EVALSET_RESULT ")]
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert len(lines) == world and all(l["ok"] for l in lines), lines
    assert all(l["metrics"] == lines[0]["metrics"] for l in lines)


def test_eval_step_crf_on_store_batches(cuda_dev, gold, tree):
    from _parity_util import make_model
    kind, res = "cocostuff27", 32
    store = build(gold, tree, kind, res, "cuda")
    images, _ = listing(tree, kind)
    rows = expected_rows(gold, kind, res, [os.path.relpath(p, tree) for p in images])
    outs = []
    for use_store in (True, False):
        model, _ = make_model("vit_small", cuda_dev, fused=True, seed=0)
        preds = []
        for k, b in enumerate(store.frames(gold["batch_size"])):
            if not use_store:
                img, label, _ = expected(gold, kind, res, rows[b["ind"]], torch.float32)
                b = dict(img=img.to(cuda_dev), label=label.to(cuda_dev))
            out = model.eval_step(b, run_crf=True)
            preds.append((out["linear_preds"].clone(), out["cluster_preds"].clone()))
        torch.cuda.synchronize()
        outs.append((preds, model.test_linear_metrics.stats.clone(), model.test_cluster_metrics.stats.clone()))
    for (a0, a1), (b0, b1) in zip(outs[0][0], outs[1][0]):
        assert torch.equal(a0, b0) and torch.equal(a1, b1)
    assert outs[0][1].sum() > 0
    assert torch.equal(outs[0][1], outs[1][1]) and torch.equal(outs[0][2], outs[1][2])
