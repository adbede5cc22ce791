"""The TensorBoard bucket rule behind the cd histograms, checked without a GPU: the library's edge and threshold tables,
the bucket trimming of summary.make_histogram, a restatement of the device bucket function (tb_bucket in
csrc/tb_hist.cuh), and the histograms the reference's own training step logs (tests/golden/cd_histograms.pt)."""
import os

import numpy as np
import pytest
import torch

from stego_b200 import hist

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cd_histograms.pt")


def _golden():
    return torch.load(GOLDEN, weights_only=False)


def test_edges_are_tensorboards_default_bins(tmp_path):
    try:
        from torch.utils.tensorboard import SummaryWriter
    except ImportError:
        want = _golden()["default_bins"].numpy()
    else:
        w = SummaryWriter(log_dir=str(tmp_path))
        want = np.array(w.default_bins, dtype=np.float64)
        w.close()
    got = hist.default_bins()
    assert got.shape == (hist.N_EDGES,) and got.tobytes() == want.tobytes()
    assert got.tobytes() == _golden()["default_bins"].numpy().tobytes()


def test_thresholds_round_each_edge_outward():
    e, t = hist.default_bins(), hist.thresholds()
    assert t.dtype == np.float32 and t.shape == (hist.N_EDGES + 1,)
    below = np.nextafter(t[:-1], np.float32(-np.inf))
    assert np.all(t[:-1].astype(np.float64) >= e) and np.all(below.astype(np.float64) < e)
    above = np.nextafter(t[-1], np.float32(np.inf))
    assert float(t[-1]) <= e[-1] < float(above)
    assert t[hist.N_EDGES // 2] == 0.0


def _make_histogram(values):
    from torch.utils.tensorboard.summary import make_histogram
    return make_histogram(values, hist.default_bins().tolist())


@pytest.mark.parametrize("support", ["first", "last", "single", "scattered", "around_zero"])
def test_trim_matches_make_histogram(support):
    pytest.importorskip("tensorboard")
    e = hist.default_bins()
    mids = (e[:-1] + e[1:]) / 2
    if support == "first":
        vals = np.array([e[0], e[0], mids[3]])
    elif support == "last":
        vals = np.array([e[-1], mids[-1], mids[-7]])
    elif support == "single":
        vals = np.full(5, mids[900])
    elif support == "scattered":
        vals = mids[[10, 400, 401, 773, 774, 1200, 1500]].repeat(3)
    else:
        vals = np.array([-0.0, 0.0, 5e-13, -5e-13, 0.3, -0.2])
    counts, _ = np.histogram(vals, bins=e)
    limits, kept = hist.trim(counts)
    want = _make_histogram(vals)
    assert limits.tolist() == list(want.bucket_limit) and kept.tolist() == list(want.bucket)


def _bucket_restated(x: np.float32, t: np.ndarray) -> int:
    """tb_bucket (csrc/tb_hist.cuh) on the host, fp32 comparisons throughout."""
    pos, nb = 774, hist.N_BINS
    if not (x >= t[0] and x <= t[hist.N_EDGES]):
        return -1
    ax = abs(x)
    if ax < np.float32(1e-12):
        k = pos if x >= 0 else pos - 1
    else:
        j = min(int(np.log2(np.float64(ax) * 1e12) * 7.272540897), pos - 1)
        k = pos + 1 + j if x > 0 else pos - 2 - j
    k = max(0, min(k, nb - 1))
    while k < nb - 1 and x >= t[k + 1]:
        k += 1
    while k > 0 and x < t[k]:
        k -= 1
    return k


def test_bucket_rule_restatement_matches_np_histogram():
    e, t = hist.default_bins(), hist.thresholds()
    f = e.astype(np.float32)
    cand = np.concatenate([f, np.nextafter(f, np.float32(np.inf)), np.nextafter(f, np.float32(-np.inf)),
                           np.array([0.0, -0.0, 1e-45, -1e-45, 1e-40, 3e38, -3e38, 1.2e20, -1.2e20], np.float32),
                           np.random.default_rng(1).standard_normal(2000).astype(np.float32)])
    for x in cand:
        counts, _ = np.histogram(np.array([np.float64(x)]), bins=e)
        want = int(np.argmax(counts)) if counts.sum() else -1
        assert _bucket_restated(np.float32(x), t) == want, x
    assert _bucket_restated(np.float32(-0.0), t) == 774  # [0, 1e-12), as numpy puts -0.0


def test_golden_reference_histograms_reproduced():
    g = _golden()
    recs = g["records"]
    assert [(r["tag"], r["step"]) for r in recs] == [("intra_cd", 1), ("inter_cd", 1), ("neg_cd", 1)]
    for r in recs:
        v = r["values"].reshape(-1).double().numpy()
        counts, _ = np.histogram(v, bins=hist.default_bins())
        stats = np.array([v.min(), v.max(), v.sum(), v.dot(v)])
        f = hist.fields(counts, stats, v.size)
        assert f["bucket_limits"] == r["bucket_limit"] and f["bucket_counts"] == r["bucket"]
        assert f["num"] == r["num"] and f["min"] == r["min"] and f["max"] == r["max"]
        assert abs(f["sum"] - r["sum"]) <= 1e-12 * np.abs(v).sum()
        assert abs(f["sum_squares"] - r["sum_squares"]) <= 1e-12 * r["sum_squares"]
