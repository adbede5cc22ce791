"""CPU: the dense correspondence heatmaps' oracle and argument checks (stego_b200/correspondence.py).

- the fp64 restatement (oracle/heatmap_oracle.py) against the reference's own get_heatmaps lines stored in
  tests/golden/correspondence_heatmaps.pt (oracle/make_golden_heatmaps.py), and the fixture's coverage: the clamp and
  the border points change values;
- argument errors of correspondence_heatmaps and get_heatmaps, raised on the host before any launch, and refusal of CPU
  tensors."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import heatmap_oracle as HO  # noqa: E402
from stego_b200 import correspondence as CP  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "correspondence_heatmaps.pt")


def _golden():
    return torch.load(GOLDEN)


@pytest.mark.parametrize("which", ["intra", "inter"])
def test_oracle_matches_reference_lines(which):
    g = _golden()
    f = g["feats"].float()
    tgt, size = (f, g["img_size"]) if which == "intra" else (g["feats_pos"].float(), g["pos_size"])
    ref = g["heatmap_" + which]
    P = g["query_points"].shape[1]
    assert ref.dtype == torch.float32 and tuple(ref.shape) == (P,) + tuple(size)
    o = HO.heatmaps(f, tgt, g["query_points"], size)[0]
    # the reference's fp32 lines against fp64: a few fp32 roundings of values <= 2
    assert float((o - ref.double()).abs().max()) <= 1e-5


def test_fixture_exercises_clamp_and_border():
    g = _golden()
    f = g["feats"].float()
    lr = HO.low_res(f, f, g["query_points"])[0]
    assert 0.2 < float((lr == 0).double().mean()) < 0.8  # the clamp zeroes a good part of every map
    assert bool((lr.flatten(1).max(1).values > 0).all())
    qp = g["query_points"]
    assert float(qp.abs().max()) > 1.0  # points beyond the border
    # beyond the border grid_sample clamps: (1.3, -1.2) samples the same point as (1, -1)
    pts = qp[0, :, 0]
    i = int(((pts - torch.tensor([1.3, -1.2])).abs().sum(1) < 1e-6).nonzero()[0])
    j = int(((pts - torch.tensor([1.0, -1.0])).abs().sum(1) < 1e-6).nonzero()[0])
    assert torch.equal(g["heatmap_intra"][i], g["heatmap_intra"][j])


# ---------------------------------------------------------------------------------------------------------------------
# argument errors (raised on the host before any launch)
# ---------------------------------------------------------------------------------------------------------------------
def _args(B=2, E=64, h=8, w=8, P=3):
    return dict(feats=torch.randn(B, E, h, w), target=torch.randn(B, E, h + 2, w - 1),
                query_points=torch.rand(B, P, 1, 2) * 2 - 1, size=(32, 24))


class _FakeCuda:
    """Skip the device check so that the shape / dtype checks after it run on the CPU."""

    def __enter__(self):
        self._orig = CP._lib.require_cuda
        CP._lib.require_cuda = lambda *t: None
        return self

    def __exit__(self, *exc):
        CP._lib.require_cuda = self._orig


def test_rejects_cpu_tensors():
    with pytest.raises(RuntimeError, match="CUDA"):
        CP.correspondence_heatmaps(**_args())


@pytest.mark.parametrize("bad,match", [
    (dict(feats=torch.randn(2, 64, 8)), r"\[B, C, h, w\]"),
    (dict(target=torch.randn(3, 64, 8, 8)), "does not match"),
    (dict(target=torch.randn(2, 32, 8, 8)), "does not match"),
    (dict(query_points=torch.rand(2, 3, 2)), "query_points"),
    (dict(query_points=torch.rand(1, 3, 1, 2)), "query_points"),
    (dict(query_points=torch.rand(2, 3, 2, 2)), "query_points"),
    (dict(query_points=torch.zeros(2, 3, 1, 2, dtype=torch.int64)), "floating point"),
    (dict(feats=torch.randn(2, 64, 8, 8, dtype=torch.float64)), "fp32 or bf16"),
    (dict(target=torch.randn(2, 64, 8, 8, dtype=torch.float16)), "fp32 or bf16"),
    (dict(feats=torch.randn(2, 800, 8, 8), target=torch.randn(2, 800, 8, 8)), "feature channels"),
    (dict(size=(32,)), "size"),
    (dict(size=(0, 32)), "empty or oversized"),
    (dict(size=(70000, 4)), "empty or oversized"),
    (dict(query_points=torch.rand(2, 0, 1, 2)), "empty or oversized"),
])
def test_rejects_bad_arguments(bad, match):
    a = _args()
    a.update(bad)
    with _FakeCuda(), pytest.raises(RuntimeError, match=match):
        CP.correspondence_heatmaps(**a)


def test_get_heatmaps_takes_one_image():
    calls = []

    def net(x):
        calls.append(x)
        return x, None

    qp = torch.zeros(2, 3, 1, 2)
    with pytest.raises(RuntimeError, match="one image"):
        CP.get_heatmaps(net, torch.zeros(2, 3, 16, 16), torch.zeros(2, 3, 16, 16), qp)
    assert not calls  # refused before the featurizer runs
