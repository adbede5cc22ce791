"""CPU: the host side of the correspondence precision-recall metric (stego_b200/correspondence.py) and its oracle.

- `pr_from_counts` against sklearn on integer bin-index scores (ap, precision, recall), the bounds against sklearn on
  unbinned fp32 scores, the digamma form against an explicit loop, the no-positive case;
- the oracle (oracle/correspondence_oracle.py) against the reference's own lines stored in
  tests/golden/correspondence_pr.pt (oracle/make_golden_correspondence.py), and the exact positive rule against the
  reference's `ld.to(int64)` targets;
- argument errors of CorrespondencePR.update."""
import os
import sys

import numpy as np
import pytest
import torch
from sklearn.metrics import average_precision_score, precision_recall_curve

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))

from stego_b200 import correspondence as CP  # noqa: E402

U = 2.0 ** -24


def _counts(bins, y, nb=CP.PR_BINS):
    return np.bincount(bins[y == 0], minlength=nb), np.bincount(bins[y == 1], minlength=nb)


def _bin(scores):
    s = torch.as_tensor(scores, dtype=torch.float32)
    return torch.clamp(torch.floor((s + 1.0) * (CP.PR_BINS // 2)), 0, CP.PR_BINS - 1).long().numpy()


@pytest.mark.parametrize("seed,n,frac", [(0, 1000, 0.3), (1, 50000, 0.05), (2, 7, 0.5), (3, 20000, 0.9)])
def test_counts_equal_sklearn_on_bin_indices(seed, n, frac):
    rng = np.random.default_rng(seed)
    y = (rng.random(n) < frac).astype(np.int64)
    bins = rng.integers(0, CP.PR_BINS, n)
    bins[y == 1] = np.minimum(bins[y == 1] + 700, CP.PR_BINS - 1)  # some signal, and ties in the top bin
    r = CP.pr_from_counts(*_counts(bins, y))
    assert r["ap"] == pytest.approx(average_precision_score(y, bins), rel=1e-13, abs=1e-15)
    p, rc, _ = precision_recall_curve(y, bins)
    np.testing.assert_allclose(r["precision"], p, rtol=1e-14, atol=0)
    np.testing.assert_allclose(r["recall"], rc, rtol=1e-14, atol=0)
    assert r["num_pairs"] == n and r["num_pos"] == int(y.sum())
    lo, hi = r["ap_bounds"]
    assert lo <= r["ap"] + 1e-12 and r["ap"] <= hi + 1e-12


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_bounds_contain_sklearn_ap_of_unbinned_scores(seed):
    rng = np.random.default_rng(seed)
    n = 400000
    y = (rng.random(n) < 0.15).astype(np.int64)
    s = np.where(y == 1, rng.normal(0.6, 0.15, n), rng.normal(0.2, 0.15, n)).astype(np.float32)
    if seed == 2:
        s = np.round(s * 300) / 300  # many exact ties inside bins
    r = CP.pr_from_counts(*_counts(_bin(s), y))
    lo, hi = r["ap_bounds"]
    ap = average_precision_score(y, s)
    assert lo - 1e-12 <= ap <= hi + 1e-12
    assert hi - lo < 5e-3


def _loop_sum(a, c, p):
    return sum((a + i) / (c + i) for i in range(1, p + 1))


@pytest.mark.parametrize("a,c,p", [(0, 0, 1), (0, 0, 50), (3, 10, 7), (1000, 123456, 999), (10 ** 6, 3 * 10 ** 6, 4000),
                                   (5, 5, 20)])
def test_digamma_form_equals_loop(a, c, p):
    got = float(CP._digamma_sum(np.float64(a), np.float64(c), np.float64(p)))
    assert got == pytest.approx(_loop_sum(a, c, p), rel=1e-12, abs=1e-12)


def test_no_positives_matches_sklearn():
    rng = np.random.default_rng(5)
    y = np.zeros(500, dtype=np.int64)
    bins = rng.integers(100, 140, 500)
    r = CP.pr_from_counts(*_counts(bins, y))
    with pytest.warns(UserWarning):
        ap = average_precision_score(y, bins)
    with pytest.warns(UserWarning):
        p, rc, _ = precision_recall_curve(y, bins)
    assert r["ap"] == ap
    np.testing.assert_array_equal(r["precision"], p)
    np.testing.assert_array_equal(r["recall"], rc)
    assert r["num_pos"] == 0


def test_all_positives_and_single_bin():
    r = CP.pr_from_counts(np.zeros(CP.PR_BINS), np.bincount([7, 7, 9], minlength=CP.PR_BINS))
    y, s = np.ones(3, dtype=np.int64), np.array([7, 7, 9])
    assert r["ap"] == average_precision_score(y, s) == 1.0
    assert r["ap_bounds"] == pytest.approx((1.0, 1.0))
    neg = np.zeros(CP.PR_BINS)
    neg[3] = 5
    pos = np.zeros(CP.PR_BINS)
    pos[3] = 2
    r = CP.pr_from_counts(neg, pos)
    y = np.array([0] * 5 + [1] * 2)
    assert r["ap"] == pytest.approx(average_precision_score(y, np.full(7, 3)), rel=1e-15)
    lo, hi = r["ap_bounds"]
    assert lo == pytest.approx((1 / 6 + 2 / 7) / 2) and hi == pytest.approx(1.0)


# ---------------------------------------------------------------------------------------------------------------------
# oracle vs the reference's lines (golden fixture)
# ---------------------------------------------------------------------------------------------------------------------
def _golden():
    import correspondence_oracle as CO
    return CO.load_golden(os.path.join(ROOT, "tests", "golden", "correspondence_pr.pt"))


def test_oracle_reproduces_reference_lines():
    import correspondence_oracle as CO
    g = _golden()
    for m in ("code", "feats"):
        fd = CO.net_fd(g[m], g["coords1"], g["coords2"])
        torch.testing.assert_close(fd, g["fd"][m], rtol=0, atol=2e-6)
        ap = CO.average_precision(CO.prep_fd(g["fd"][m]).numpy(), g["ld"].to(torch.int64).numpy())
        assert ap == g["ap_reference"][m]
        exact = CO.exact_targets(g["label"], g["n_classes"], g["coords1"], g["coords2"])
        assert CO.average_precision(g["fd"][m].numpy(), exact.numpy()) == g["ap_exact"][m]
    ld = CO.label_ld(g["label"], g["n_classes"], g["coords1"], g["coords2"])
    torch.testing.assert_close(ld, g["ld"], rtol=0, atol=0)


def test_exact_rule_against_reference_targets():
    """The exact positives contain the reference's `ld.to(int64)` positives; every pair where they differ has ld
    within 4 u of 1 (a pure sample's fp32 weights sum to 1 up to rounding)."""
    import correspondence_oracle as CO
    g = _golden()
    exact = CO.exact_targets(g["label"], g["n_classes"], g["coords1"], g["coords2"])
    ref = g["ld"].to(torch.int64) == 1
    assert bool((ref & ~exact).sum() == 0)
    diff = exact & ~ref
    assert int(diff.sum()) > 0  # the fixture exercises the deviation
    assert float((g["ld"][diff] - 1).abs().max()) <= 4 * U
    # off the exact positives ld is at most 1 - (smallest weight), i.e. well away from 1
    assert float(g["ld"][~exact].max()) < 1 - 4 * U


# ---------------------------------------------------------------------------------------------------------------------
# argument errors (raised on the host before any launch)
# ---------------------------------------------------------------------------------------------------------------------
def _args(B=2, fs=4, E=64, D=8, H=8, W=8):
    return dict(feats=torch.randn(B, E, H, W), code=torch.randn(B, D, H, W),
                label=torch.randint(-1, 5, (B, 16, 16)), coords1=torch.rand(B, fs, fs, 2) * 2 - 1,
                coords2=torch.rand(B, fs, fs, 2) * 2 - 1)


def _metric():
    m = CP.CorrespondencePR.__new__(CP.CorrespondencePR)
    m.n_classes = 5
    m.counts = torch.zeros(2, 2, CP.PR_BINS, dtype=torch.int64)
    return m


def test_rejects_cpu_tensors():
    with pytest.raises(RuntimeError, match="CUDA"):
        _metric().update(**_args())


def test_rejects_bad_n_classes():
    for n in (0, 256, 300):
        with pytest.raises(RuntimeError, match="n_classes"):
            CP.CorrespondencePR(n, "cpu")


class _FakeCuda:
    """Skip the device check so that the shape / dtype checks after it run on the CPU."""

    def __enter__(self):
        self._orig = CP._lib.require_cuda
        CP._lib.require_cuda = lambda *t: None
        return self

    def __exit__(self, *exc):
        CP._lib.require_cuda = self._orig


@pytest.mark.parametrize("bad,match", [
    (dict(code=torch.randn(3, 8, 8, 8)), "batch sizes"),
    (dict(label=torch.randint(0, 5, (3, 16, 16))), "batch sizes"),
    (dict(coords2=torch.rand(2, 5, 5, 2)), "coords"),
    (dict(coords1=torch.rand(2, 65, 65, 2), coords2=torch.rand(2, 65, 65, 2)), "feature_samples"),
    (dict(label=torch.zeros(2, 16, 16, dtype=torch.int16)), "label dtype"),
    (dict(label=torch.zeros(2, 16, 16)), "label dtype"),
    (dict(feats=torch.randn(2, 800, 8, 8)), "feature channels"),
    (dict(code=torch.randn(2, 97, 8, 8)), "code dim"),
    (dict(feats=torch.randn(2, 64, 8, 8, dtype=torch.float64)), "fp32 or bf16"),
])
def test_rejects_bad_arguments(bad, match):
    a = _args()
    a.update(bad)
    with _FakeCuda(), pytest.raises(RuntimeError, match=match):
        _metric().update(**a)
