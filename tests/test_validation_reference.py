"""CPU: UnsupervisedMetrics.compute / map_clusters and LitUnsupervisedSegmenter.validation_epoch_end against the
reference's own validation path (tests/golden/validation.pt, written by oracle/make_golden_validation.py from
src/train_segmentation.py:254-371 and src/utils.py:203-274), with extra_clusters 0 and 2.

The Hungarian assignment, the histogram and the cluster -> class table are integer results and match exactly.  mIoU and
accuracy are ratios: the reference divides int64 counts in float32, this class in float64, so they agree to float32
rounding (a relative 1e-6 is 16 float32 ulps)."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "validation.pt")
KEYS = ["test/linear/mIoU", "test/linear/Accuracy", "test/cluster/mIoU", "test/cluster/Accuracy"]


def _gold(extra):
    return torch.load(GOLD, weights_only=False)[f"extra{extra}"]


def _close(got, want):
    assert set(got) == set(want) == set(KEYS), (sorted(got), sorted(want))
    for k in KEYS:
        assert abs(got[k] - want[k]) <= 1e-6 * abs(want[k]), (k, got[k], want[k])


@pytest.mark.parametrize("extra", [0, 2])
def test_compute_and_map_clusters_match_reference(extra):
    from stego_b200.eval import UnsupervisedMetrics
    g = _gold(extra)
    lin = UnsupervisedMetrics("test/linear/", 27, 0, False)
    clu = UnsupervisedMetrics("test/cluster/", 27, extra, True)
    lin.stats.copy_(g["linear_stats"])
    clu.stats.copy_(g["cluster_stats"])
    _close({**lin.compute(), **clu.compute()}, g["logged"])
    for got, want in zip(clu.assignments, g["assignments"]):
        assert torch.equal(torch.as_tensor(got), want)
    assert torch.equal(clu.histogram.to(g["histogram"].dtype), g["histogram"])
    table = clu.map_clusters(torch.arange(27 + extra))
    assert table.dtype == torch.int64 and torch.equal(table, g["map_all"])
    assert int((table == -1).sum()) == extra  # the unmatched extra clusters
    preview = g["steps"][0]["cluster_preds"].long()
    assert torch.equal(clu.map_clusters(preview).to(torch.int8), g["map_preview"])


def test_map_clusters_insertion_rule():
    """utils.py:237-241 inserts -1 at position m + 1 for an unmatched cluster m (not at m), or appends it when m is the
    table's current length: unmatched clusters 0 and 4 of 3 classes + 2 extra."""
    import numpy as np
    from stego_b200.eval import UnsupervisedMetrics
    m = UnsupervisedMetrics("x/", 3, 2, True)
    m.assignments = (np.array([1, 2, 3]), np.array([2, 0, 1]))
    assert m.map_clusters(torch.arange(5)).tolist() == [2, -1, 0, 1, -1]
    m.assignments = (np.array([0, 1, 2]), np.array([2, 0, 1]))
    assert m.map_clusters(torch.arange(5)).tolist() == [2, 0, 1, -1, -1]


@pytest.mark.parametrize("extra", [0, 2])
def test_validation_epoch_end_matches_reference(extra):
    """Reference keys and values, logged only once global_step > 2, both metrics reset afterwards."""
    sys.path.insert(0, ROOT)
    from stego_b200.config import make_cfg
    from stego_b200.segmenter import LitUnsupervisedSegmenter
    g = _gold(extra)
    torch.manual_seed(0)
    model = LitUnsupervisedSegmenter(27, make_cfg(random_backbone_init=True, extra_clusters=extra))
    assert model.cfg.n_images == 5
    for step, logs in ((2, False), (3, True)):
        model.logged.clear()
        model.global_step = step
        model.linear_metrics.stats.copy_(g["linear_stats"])
        model.cluster_metrics.stats.copy_(g["cluster_stats"])
        out = model.validation_epoch_end([])
        _close(out, g["logged"])
        if logs:
            _close(model.logged, g["logged"])
        else:
            assert not model.logged
        assert not model.linear_metrics.stats.any() and not model.cluster_metrics.stats.any()
        assert torch.equal(model.cluster_metrics.map_clusters(torch.arange(27 + extra)), g["map_all"])
