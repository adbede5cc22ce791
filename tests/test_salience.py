"""CPU: the use_salience coordinate draws (src/modules.py:298-311, 357-364).

tests/golden/salience.pt holds what the reference's own sample_nonzero_locations and its coordinate lines returned on
the CPU (oracle/make_golden_salience.py); oracle/salience_oracle.py, modules.sample_nonzero_locations and
ContrastiveCorrelationLoss.draw_coords must reproduce it bit for bit, generator consumption included.  The wrapper of
the kernel (stego_b200/salience.py) and the C ABI reject what they cannot compute before touching a device."""
import os
import sys
from types import SimpleNamespace

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import make_golden_salience as MGS  # noqa: E402
import salience_oracle as SO  # noqa: E402

GOLDEN = torch.load(os.path.join(ROOT, "tests", "golden", "salience.pt"))
CASES = MGS.cases()


def _bits(t):
    return t.contiguous().view(torch.int32)


def test_fixture_covers_the_edges():
    assert set(GOLDEN) == set(CASES)
    fss = {c[2] for c in CASES.values()}
    assert {1, 11, 16} <= fss
    masks = [m for c in CASES.values() for m in c[:2]]
    per_image = [(m[i] != 0).sum().item() for m in masks for i in range(m.shape[0])]
    assert 0 in per_image and 1 in per_image
    assert any(bool((m[i] != 0).all()) and m[i].numel() > 1 for m in masks for i in range(m.shape[0]))
    assert any(m.shape[1] != m.shape[2] and m.shape[1] < m.shape[2] for m in masks)
    assert any(m.shape[1] > m.shape[2] for m in masks)
    assert any(bool(torch.isnan(m).any()) for m in masks)
    assert any(bool(((m == 0) & torch.signbit(m)).any()) for m in masks)


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_and_modules_reproduce_reference(name):
    from stego_b200 import modules
    sal, sal_pos, fs = CASES[name]
    want = GOLDEN[name]
    shape = [sal.shape[0], fs, fs, 2]
    for fn in (SO.sample_nonzero_locations, modules.sample_nonzero_locations):
        torch.manual_seed(want["seed"])
        assert torch.equal(_bits(fn(sal, shape)), _bits(want["nz1"])), fn
        assert torch.equal(_bits(fn(sal_pos, shape)), _bits(want["nz2"])), fn
    torch.manual_seed(want["seed"])
    c1, c2 = SO.draw_coords(sal, sal_pos, fs)
    assert torch.equal(_bits(c1), _bits(want["coords1"])) and torch.equal(_bits(c2), _bits(want["coords2"]))
    assert torch.equal(torch.randint(1 << 30, (4,)), want["next"])
    torch.manual_seed(want["seed"])
    lossfn = modules.ContrastiveCorrelationLoss(SimpleNamespace(use_salience=True, feature_samples=fs))
    c1, c2 = lossfn.draw_coords(torch.empty(sal.shape[0], 1), sal, sal_pos)
    assert torch.equal(_bits(c1), _bits(want["coords1"])) and torch.equal(_bits(c2), _bits(want["coords2"]))
    assert torch.equal(torch.randint(1 << 30, (4,)), want["next"])


def test_oracle_from_draws_matches_generator_path():
    """nonzero_locations_from_draws with the values randint would have returned is sample_nonzero_locations."""
    sal, _, fs = CASES["square_mixed_fs11"]
    n = fs * fs
    torch.manual_seed(5)
    want = SO.sample_nonzero_locations(sal, [sal.shape[0], fs, fs, 2])
    torch.manual_seed(5)
    draws = torch.zeros(sal.shape[0], 2 * n, dtype=torch.int64)
    for i in range(sal.shape[0]):
        count = int((sal[i] != 0).sum())
        # randint(high) on the CPU returns values in [0, high): the same values through `% high` stay themselves
        draws[i, :2 * n if count == 0 else n] = torch.randint(sal.shape[1] if count == 0 else count,
                                                              (2 * n if count == 0 else n,))
    assert torch.equal(_bits(SO.nonzero_locations_from_draws(sal, fs, draws)), _bits(want))


def test_wrapper_rejects_bad_shapes_sizes_and_cpu_tensors():
    from stego_b200 import salience
    ok = torch.ones(2, 8, 8)
    with pytest.raises(RuntimeError, match="CUDA"):
        salience.salience_coords(ok, ok, 11)
    with pytest.raises(RuntimeError, match="CUDA"):
        salience.salience_coords(ok[:, None], ok[:, None], 11)
    for bad in (torch.ones(8, 8), torch.ones(2, 3, 8, 8), torch.ones(1, 2, 2, 8, 8), torch.ones(2, 0, 8),
                torch.ones(0, 8, 8)):
        with pytest.raises(ValueError, match="mask"):
            salience.salience_coords(bad, bad, 11)
    huge = torch.empty(1, 1 << 14, 1 << 14, device="meta")  # H * W = 2^28: torch's 64-bit randint range
    with pytest.raises(ValueError, match="2\\^28"):
        salience.salience_coords(huge, huge, 11)
    for fs in (0, 65):
        with pytest.raises(ValueError, match="feature_samples"):
            salience.salience_coords(ok, ok, fs)
    with pytest.raises(TypeError):
        salience.salience_coords(None, ok, 11)
    assert not salience.masks_supported(ok, ok, 2, torch.device("cpu"))


def test_c_abi_rejects_before_any_cuda_call():
    import re
    from stego_b200 import _lib
    lib = _lib.load()
    P = 256  # never dereferenced: every call below fails its argument checks first

    def call(sal=P, draws=P, mask_bytes=4, B=2, H=8, W=8, fs=11, scratch=0):
        return lib.stego_salience_coords(sal, P, mask_bytes, B, H, W, fs, 1, 0, draws, P, P, P, P, P, scratch, 0)

    cases = [(dict(sal=0), "null pointer"), (dict(draws=0), "null pointer"), (dict(mask_bytes=2), "mask_bytes"),
             (dict(B=0), ">= 1"), (dict(H=0), ">= 1"), (dict(W=0), ">= 1"), (dict(H=1 << 14, W=1 << 14), "2\\^28"),
             (dict(fs=0), "feature_samples"), (dict(fs=65), "feature_samples"), (dict(H=1024, W=2048), "scratch")]
    for kw, msg in cases:
        assert call(**kw) == -1, kw
        assert re.search(msg, _lib.last_error()), (kw, _lib.last_error())
    for args, msg in [((0, P, 4, 2, 8, 8, P), "null pointer"), ((P, P, 3, 2, 8, 8, P), "mask_bytes"),
                      ((P, P, 4, 2, 0, 8, P), ">= 1"), ((P, P, 1, 1, 1 << 14, 1 << 14, P), "2\\^28")]:
        assert lib.stego_salience_counts(*args, 0) == -1, args
        assert re.search(msg, _lib.last_error()), (args, _lib.last_error())


def test_scratch_rule():
    from stego_b200 import _lib
    lib = _lib.load()
    assert lib.stego_salience_scratch_bytes(32, 224, 224) == 0
    assert lib.stego_salience_scratch_bytes(16, 448, 448) == 0
    assert lib.stego_salience_scratch_bytes(1, 384, 1024) == 0        # 12 288 words: the shared-memory limit
    assert lib.stego_salience_scratch_bytes(1, 384, 1025) == 16 * ((384 * 1025 + 31) // 32)
    assert lib.stego_salience_scratch_bytes(3, 1024, 2048) == 3 * 16 * (1024 * 2048 // 32)
    assert lib.stego_salience_scratch_bytes(0, 8, 8) == 0
