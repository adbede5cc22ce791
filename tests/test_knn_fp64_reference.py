"""tests/_knn_fp64.py on the CPU: the fp64 kNN reference against the oracle (oracle/stego_oracle.py::knn_indices, the
reference's einsum + topk) where similarities are separated and against a brute-force loop where they tie, and the
input builders against the edges they claim to build."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "oracle"))
import _knn_fp64 as R  # noqa: E402


def brute_force(feats, k):
    """per row: itself, then the others by (similarity descending, index ascending), as a Python sort"""
    xn = R.normalize64(feats)
    s = (xn @ xn.T).tolist()
    n = len(s)
    idx = [sorted(range(n), key=lambda j: (j != i, -s[i][j], j))[:min(k + 1, n)] for i in range(n)]
    return torch.tensor(idx), torch.tensor([[s[i][j] for j in row] for i, row in enumerate(idx)], dtype=torch.float64)


def test_reference_matches_oracle_where_separated():
    import stego_oracle as O
    n, E, k = 300, 64, 10
    x = R.clustered(n, E, 0)
    ref = R.knn_reference(x, k, chunk=64)  # 4 full chunks and one of 44 rows
    want_idx, want_val = O.knn_indices(R.normalize64(x), k + 1)
    assert (want_val[:, :-1] - want_val[:, 1:]).min().item() > 1e-9   # no ties: topk's order is the only order
    assert torch.equal(ref["idx"], want_idx)
    assert (ref["val"] - want_val).abs().max().item() < 1e-14
    assert torch.equal(ref["idx"][:, 0], torch.arange(n))


@pytest.mark.parametrize("n,k,chunk", [(40, 7, 16), (40, 7, 4096), (9, 9, 4), (33, 32, 33), (1, 1, 8)])
def test_reference_matches_brute_force_with_ties(n, k, chunk):
    x = R.exact_lattice(n, 64, n + k)
    gather = torch.randint(0, n, (n, 5), generator=torch.Generator().manual_seed(0))
    ref = R.knn_reference(x, k, chunk=chunk, gather=gather)
    idx, val = brute_force(x, k)
    assert ref["idx"].shape == (n, min(k + 1, n))
    assert torch.equal(ref["idx"], idx) and torch.equal(ref["val"], val)
    xn = R.normalize64(x)
    assert torch.equal(ref["gathered"], (xn @ xn.T).gather(1, gather))
    if n > 8:
        assert (val[:, 1:-1] == val[:, 2:]).double().mean().item() > 0.3  # the ties are there


def test_reference_puts_self_before_an_earlier_duplicate_and_a_zero_row_first():
    x, z = R.scaled_rows(50, 64, 3)
    x[7] = 4.0 * x[30]                               # a duplicate with a lower index than its original
    ref = R.knn_reference(x, 5)
    assert torch.equal(ref["idx"][:, 0], torch.arange(50))
    assert ref["idx"][30, 1].item() == 7 and ref["idx"][7, 1].item() == 30
    assert ref["idx"][z].tolist() == [z, 0, 1, 2, 3, 4] and (ref["val"][z] == 0).all()
    assert (ref["val"][torch.arange(50) != z, 0] - 1).abs().max().item() < 1e-15
    norms = x.norm(dim=1)
    assert norms[z] == 0 and norms[norms > 0].max() / norms[norms > 0].min() > 1e8


@pytest.mark.parametrize("n,E", [(300, 64), (1000, 384)])
def test_exact_lattice_is_exact_and_plants_its_duplicates(n, E):
    x = R.exact_lattice(n, E, 5)
    assert ((x != 0).sum(1) == 16).all()
    assert len(x.norm(dim=1).unique()) > 3           # the rows are un-normalised
    xn32 = x / x.norm(dim=1, keepdim=True)           # fp32, as the kernel normalises
    assert torch.equal(xn32.abs().unique(), torch.tensor([0.0, 0.25]))
    assert torch.equal(xn32.bfloat16().float(), xn32)                # hi plane exact, lo plane zero
    s32, s64 = xn32 @ xn32.T, R.normalize64(x) @ R.normalize64(x).T
    assert torch.equal(s32.double(), s64)
    assert torch.equal((s64 * 16).round() / 16, s64) and len(s64.unique()) <= 33
    plants = R.lattice_plants(n)
    for a, b in plants:
        assert torch.equal(xn32[a], xn32[b])
    same_tile_other_half = [(a, b) for a, b in plants if a // 128 == b // 128 and a // 64 != b // 64]
    next_tile_lower_half = [(a, b) for a, b in plants if abs(a // 128 - b // 128) == 1 and abs(a - b) >= 64
                            and min(a, b) % 128 >= 64 and max(a, b) % 128 < 64]
    far = [(a, b) for a, b in plants if abs(a - b) >= 128]
    last_block = [(a, b) for a, b in plants if max(a, b) // 128 == (n - 1) // 128 and min(a, b) // 128 == 0]
    copy_first = [(a, b) for a, b in plants if b < a]
    assert same_tile_other_half and next_tile_lower_half and far and last_block and copy_first
    dup = (s64 == 1).sum(1) - 1                      # random duplicates from the small pool, besides the plants
    assert (dup > 0).double().mean().item() > 0.5


def test_near_duplicates_are_where_they_claim():
    n, E = 1000, 384
    x, pairs, eps = R.near_duplicates(n, E, 2)
    base = R.clustered(n, E, 2)
    assert pairs.shape == (64, 2) and len(pairs.flatten().unique()) == 128
    a, b = pairs[:, 0], pairs[:, 1]
    assert torch.equal(x[a], base[a])                # originals untouched
    for level in R.EPS_LEVELS:
        sel = eps == level
        assert sel.sum() >= 8 and (b[sel] < a[sel]).any() and (b[sel] > a[sel]).any()
        rel = (x[b[sel]].double() - x[a[sel]].double()).norm(dim=1) / x[a[sel]].double().norm(dim=1)
        if level == 0:
            assert torch.equal(x[b[sel]], x[a[sel]])
        elif level > 1e-7:                           # 1e-7 is at fp32's resolution: most of it rounds away
            assert ((rel / level).log2().abs() < 0.5).all()
        else:
            assert (rel > 0).all() and (rel < 4 * level).all()
    pr = set(map(tuple, pairs.tolist()))
    assert (63, 64) in pr and (128, 127) in pr and (10, n - 5) in pr and (n - 6, 11) in pr
    # a near copy is the nearest other row of its original (the neighbours of a cluster are 0.35 sigma away)
    ref = R.knn_reference(x, 3)
    assert torch.equal(ref["idx"][a, 1], b) and torch.equal(ref["idx"][b, 1], a)


@pytest.mark.parametrize("E", [64, 384, 768, 1024])
def test_error_bar_covers_the_emulated_operand_path(E):
    """The normalisation and hi / lo terms of sim_error_bar against what they bound: knn_prep_kernel's arithmetic
    restated in torch (fp32 normalisation, bf16 hi / lo planes), the three passes summed exactly."""
    x = R.clustered(400, E, E)
    inv = 1.0 / x.pow(2).sum(1, keepdim=True).sqrt().clamp_min(1e-12)
    v = x * inv
    hi = v.bfloat16()
    lo = (v - hi.float()).bfloat16()
    assert torch.equal((v - hi.float()).double(), v.double() - hi.double())  # the subtraction is exact
    hi, lo = hi.double(), lo.double()
    s = hi @ hi.T + hi @ lo.T + lo @ hi.T
    xn = R.normalize64(x)
    err = (s - xn @ xn.T).abs().max().item()
    operand_part = 2 * (E / 64 + 6) * R.U + 3 * 2.0 ** -16
    assert 0 < err < operand_part < R.sim_error_bar(E)
    assert R.sim_error_bar(E) < 3e-4                 # still far below the spacing of neighbours (~1e-3)
