"""CPU: the `devices=` argument of eval_step, eval_scene, knn_topk and precompute_knns, and the kNN row-range entries.

  * every refusal of a device list raises a ValueError before anything is launched: a duplicate, a CPU device, an
    ordinal out of range, a first device other than the inputs', a pair without peer access (the device count and
    the peer query patched, so no GPU is needed);
  * devices=None and a list of one device select the single-device call;
  * the slices are contiguous and nearly equal, whole 128-row blocks for the kNN search, with idle devices when there
    are more devices than items;
  * the header declares stego_knn_prep and stego_knn_topk_rows, the library exports them, and they refuse row0 off a
    128-row block, ranges past n and k above 32 without touching the GPU.
"""
import ctypes
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


@pytest.fixture
def four_gpus(monkeypatch):
    """Four visible devices; 0 and 3 cannot reach each other."""
    monkeypatch.setattr(torch.cuda, "device_count", lambda: 4)
    monkeypatch.setattr(torch.cuda, "can_device_access_peer", lambda a, b: {a, b} != {0, 3})


REFUSED = {
    "duplicate": ([0, 1, 1], "twice"),
    "cpu": ([0, torch.device("cpu")], "CUDA devices"),
    "out_of_range": ([0, 4], "out of range"),
    "negative": ([0, -1], "out of range"),
    "no_peer_access": ([0, 3], "peer access"),
    "empty": ([], "at least one"),
    "not_a_device": ([0, "cuda:1"], "ordinals or torch.device"),
    "bare_int": (1, "sequence"),
}


@pytest.mark.parametrize("case", list(REFUSED))
def test_check_devices_refusals(four_gpus, case):
    from stego_b200.devices import check_devices
    devices, words = REFUSED[case]
    with pytest.raises(ValueError, match=words):
        check_devices(devices, torch.device("cuda", 0), "who")


def test_check_devices_accepts_and_selects(four_gpus):
    from stego_b200.devices import check_devices
    c0 = torch.device("cuda", 0)
    assert check_devices(None, c0, "who") is None
    assert check_devices([0], c0, "who") is None
    assert check_devices([torch.device("cuda", 0)], c0, "who") is None
    assert check_devices([0, torch.device("cuda", 2), 1], c0, "who") == [c0, torch.device("cuda", 2),
                                                                          torch.device("cuda", 1)]
    with pytest.raises(ValueError, match="first device"):
        check_devices([1, 0], c0, "who")


def test_split():
    from stego_b200.devices import split
    assert split(10, 3) == [(0, 3), (3, 6), (6, 10)]
    assert split(2, 4) == [(0, 0), (0, 1), (1, 1), (1, 2)]
    assert split(129, 3, 128) == [(0, 0), (0, 128), (128, 129)]
    for n, parts, align in ((118287, 8, 128), (300, 2, 128), (15, 8, 1), (1, 2, 128)):
        s = split(n, parts, align)
        assert s[0][0] == 0 and s[-1][1] == n and all(a[1] == b[0] for a, b in zip(s, s[1:]))
        assert all(a % align == 0 for a, b in s if b > a)
        sizes = [b - a for a, b in s if b > a]
        assert max(sizes) - min(sizes) <= align


def _model():
    from stego_b200.config import make_cfg
    from stego_b200.segmenter import LitUnsupervisedSegmenter
    torch.manual_seed(0)
    return LitUnsupervisedSegmenter(5, make_cfg(random_backbone_init=True))


@pytest.mark.parametrize("case", ["duplicate", "cpu", "out_of_range", "no_peer_access", "primary"])
def test_refusals_before_any_launch(four_gpus, case):
    from stego_b200 import _lib
    from stego_b200.knn import knn_topk, precompute_knns
    devices = [0, 1] if case == "primary" else REFUSED[case][0]  # the inputs are on the CPU, not cuda:0
    model = _model()
    img = torch.randn(2, 3, 64, 64)
    label = torch.zeros(2, 64, 64, dtype=torch.long)
    feats = torch.randn(300, 64)
    rng = torch.get_rng_state()
    n = _lib.launch_count()
    calls = [lambda: model.eval_step(dict(img=img, label=label), devices=devices),
             lambda: model.eval_step(dict(img=img), run_crf=True, devices=devices),
             lambda: model.eval_scene(img, (1, 2), label, devices=devices),
             lambda: knn_topk(feats, 5, devices=devices),
             lambda: precompute_knns(model.net, [img], 1, devices=devices)]
    for call in calls:
        with pytest.raises(ValueError):
            call()
    assert _lib.launch_count() == n and torch.equal(rng, torch.get_rng_state())


def test_header_declares_and_library_exports_knn_row_entries():
    from stego_b200 import _lib
    protos = _lib.header_prototypes()
    assert protos["stego_knn_prep"] == ("int", ["const float*", "int", "int", "void*", "void*"])
    assert protos["stego_knn_topk_rows"] == ("int", ["const void*", "int", "int", "int", "int", "int", "long long*",
                                                     "float*", "void*"])
    lib = _lib.load()
    for name in ("stego_knn_prep", "stego_knn_topk_rows", "stego_knn_topk"):
        getattr(lib, name)


FAKE = 1 << 20  # an aligned, never dereferenced address: every refusal returns before a launch


@pytest.mark.parametrize("n,E,k,row0,nrows,words", [
    (300, 384, 5, 64, 100, "multiple of 128"),
    (300, 384, 5, -128, 100, "multiple of 128"),
    (300, 384, 5, 256, 45, "not within"),
    (300, 384, 5, 128, 0, "not within"),
    (300, 384, 33, 0, 300, "k=33"),
    (300, 384, 0, 0, 300, "k=0"),
    (3, 384, 5, 0, 3, "k=5"),
    (300, 100, 5, 0, 300, "multiple of 64"),
])
def test_knn_topk_rows_refusals(n, E, k, row0, nrows, words):
    from stego_b200 import _lib
    lib = _lib.load()
    c = _lib.launch_count()
    rc = lib.stego_knn_topk_rows(FAKE, n, E, k, row0, nrows, FAKE, 0, 0)
    assert rc == -1 and words in _lib.last_error()
    assert lib.stego_knn_topk_rows(0, n, E, k, 0, n, FAKE, 0, 0) == -1
    assert lib.stego_knn_prep(FAKE, n, 100, FAKE, 0) == -1 and "multiple of 64" in _lib.last_error()
    assert lib.stego_knn_prep(FAKE, n, E, FAKE + 2, 0) == -1
    assert _lib.launch_count() == c
    assert isinstance(ctypes.c_int(rc).value, int)
