"""Which correspondence-loss implementation a configuration selects (no GPU needed)."""
import pytest

from stego_b200 import corr
from stego_b200.config import make_cfg


@pytest.mark.parametrize("fs", [1, 5, 11])
def test_single_tile_up_to_11(fs):
    spec = corr.make_spec(make_cfg(feature_samples=fs))
    assert type(spec) is corr.LossSpec and not spec.tiled and spec.rows == 128


@pytest.mark.parametrize("fs,rows", [(12, 256), (16, 256), (23, 640), (28, 896), (56, 3200), (64, 4096)])
def test_multi_tile_from_12_to_64(fs, rows):
    spec = corr.make_spec(make_cfg(feature_samples=fs, neg_samples=3))
    assert type(spec) is corr.TiledLossSpec and spec.tiled
    assert spec.rows == rows and spec.n_tiles == rows // 128
    assert spec.nslots == spec.ncalls == 5 and spec.slot_of_call == [0, 1, 2, 3, 4]


def test_above_cap_refused():
    with pytest.raises(RuntimeError, match="1..64"):
        corr.make_spec(make_cfg(feature_samples=65))
    with pytest.raises(RuntimeError, match="feature_samples"):
        corr.LossSpec(make_cfg(feature_samples=12))
