"""The fused kNN search (stego_knn_topk: csrc/knn.cu through stego_b200/knn.py) against the float64 reference of
tests/_knn_fp64.py, up to the sizes it is built for (COCO-Stuff train: 118 287 descriptors, 925 row blocks).

  exact      exact_lattice inputs: every similarity is a multiple of 1/16 that bf16 and fp32 carry exactly, so indices
             and values are compared with torch.equal at every position, and almost every position is a tie: the order
             (self first, then similarity descending, index ascending) is what is being tested.  Sizes on every edge of
             the 128 x 128 tile, its 64-column halves and 32-column scan chunks, k up to KNN_MAXK and n == k, and three
             sizes with more row blocks than the device has SMs (the persistent loop runs 2, 3 and 3 times per CTA).
  parity     clustered / near-duplicate / badly scaled descriptors at the data-set sizes, against sim_error_bar(E):
             values, the fp64 similarity of every returned index, completeness and exact indices wherever the fp64
             similarities are separated by more than two bars, with the covered fraction asserted.  Nothing is masked
             out of the value checks.
  calls      determinism, return_values, views, streams, and the raw C ABI on buffers carved out of larger ones.

The measured maxima are written beside the bars to $STEGO_PARITY_DIR when it is set.
"""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _knn_fp64 as R  # noqa: E402
from _parity_util import record  # noqa: E402

pytestmark = pytest.mark.gpu

EDGE_N = [1, 2, 31, 32, 33, 63, 64, 65, 96, 97, 127, 128, 129, 191, 193, 255, 256, 257, 1000]
EDGE_K = [1, 2, 30, 31, 32]
# least share of positions 1..k-1 the exact-index check must reach on clustered descriptors (fp64 on the CPU gives 0.72 at
# E = 384 and 0.49 at E = 768, whose bar is wider, at every n tried from 3 000 to 40 000)
MIN_COVER = {384: 0.5, 768: 0.3}


def _knn(x, k, dev, values=True):
    from stego_b200.knn import knn_topk
    return knn_topk(x.to(dev), k, return_values=values)


def _sms(dev):
    return torch.cuda.get_device_properties(dev).multi_processor_count


def _first_diff(a, b):
    bad = (a != b).nonzero()
    return None if bad.numel() == 0 else (bad[0].tolist(), a[tuple(bad[0])].item(), b[tuple(bad[0])].item())


def _assert_exact(x, k, dev):
    n = x.shape[0]
    ref = R.knn_reference(x, k, dev)
    idx, val = _knn(x, k, dev)
    assert idx.shape == (n, k) and idx.dtype == torch.long and val.shape == (n, k) and val.dtype == torch.float32
    assert torch.equal(idx, ref["idx"][:, :k]), ("index", n, k, _first_diff(idx, ref["idx"][:, :k]))
    assert torch.equal(val.double(), ref["val"][:, :k]), ("value", n, k, _first_diff(val.double(), ref["val"][:, :k]))
    return ref


# ------------------------------------------------------------------------------------------------
# exact answers, ties everywhere
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("E", [64, 384])
@pytest.mark.parametrize("n", EDGE_N)
def test_exact_order_on_tile_edges(cuda_dev, n, E):
    x = R.exact_lattice(n, E, 1000 * E + n)
    for k in EDGE_K:
        if k <= n:
            ref = _assert_exact(x, k, cuda_dev)
    if n >= 63:  # the order among ties is what decided these answers
        assert (ref["val"][:, 1:-1] == ref["val"][:, 2:]).double().mean().item() > 0.3


@pytest.mark.parametrize("E", [64, 128, 384, 768, 1024])
def test_exact_order_across_widths(cuda_dev, E):
    _assert_exact(R.exact_lattice(1500, E, E), 30, cuda_dev)


@pytest.mark.parametrize("blocks_per_sm,extra", [(1, 1), (2, 77), (3, 0)])
def test_exact_order_with_more_row_blocks_than_sms(cuda_dev, blocks_per_sm, extra):
    """Every CTA walks several row blocks: the private lists and the threshold start afresh, the mbarrier stage and
    phase carry over on the producer and both consumer warpgroups, the merge buffer is reused."""
    n = blocks_per_sm * R.TILE * _sms(cuda_dev) + extra
    assert (n + R.TILE - 1) // R.TILE > _sms(cuda_dev)
    ref = _assert_exact(R.exact_lattice(n, 384, n), 30, cuda_dev)
    record(f"knn_fp64_exact_{blocks_per_sm}x_sms_plus_{extra}",
           dict(n=n, E=384, k=30, sms=_sms(cuda_dev), row_blocks=(n + R.TILE - 1) // R.TILE, compared="torch.equal",
                tied_positions=(ref["val"][:, 1:-1] == ref["val"][:, 2:]).double().mean().item()))


# ------------------------------------------------------------------------------------------------
# fp64 parity at the data-set sizes
# ------------------------------------------------------------------------------------------------
def _assert_parity(name, x, k, dev, min_cover):
    n, E = x.shape
    bar = R.sim_error_bar(E)
    idx, val = _knn(x, k, dev)
    ref = R.knn_reference(x, k, dev, gather=idx)
    val = val.double()
    ri, rv = ref["idx"], ref["val"]
    rows = torch.arange(n, device=dev)
    # well formed: indices in range, none twice in a row, the row itself first, the rest by descending similarity
    assert torch.isfinite(val).all()
    assert idx.min().item() >= 0 and idx.max().item() < n
    srt = idx.sort(1).values
    assert (srt[:, 1:] != srt[:, :-1]).all()
    assert torch.equal(idx[:, 0], rows)
    assert (val[:, 1:-1] >= val[:, 2:]).all()
    # values, position by position, and the fp64 similarity of every returned index: both unmasked
    err_val = (val - rv[:, :k]).abs().max().item()
    err_own = (val - ref["gathered"]).abs().max().item()
    # completeness: whoever is more than two bars above the kernel's k-th similarity in fp64 was returned
    must = rv[:, 1:] > val[:, k - 1:k] + 2 * bar
    present = (ri[:, 1:, None] == idx[:, None, :]).any(2)
    missing = int((must & ~present).sum())
    # exact indices wherever fp64 separates a position from both neighbours by more than two bars (position 1's upper
    # neighbour is the row itself, which is pinned)
    gap = rv[:, :-1] - rv[:, 1:]                       # gap[:, j]: position j to position j + 1
    clear = torch.ones(n, k, dtype=torch.bool, device=dev)
    clear[:, 1:] = gap[:, 1:] > 2 * bar
    clear[:, 2:] &= gap[:, 1:-1] > 2 * bar
    cover = clear[:, 1:].double().mean().item()
    wrong = int((idx != ri[:, :k])[clear].sum())
    self_not_largest = int((val[:, 1] > val[:, 0]).sum()) if k > 1 else 0
    record(f"knn_fp64_{name}", dict(n=n, E=E, k=k, bar=bar, max_value_error=err_val, max_returned_pair_error=err_own,
                                    covered_fraction_of_exact_index_check=cover, wrong_indices=wrong, missing=missing,
                                    rows_with_a_neighbour_above_self=self_not_largest))
    assert err_val <= bar and err_own <= bar, (err_val, err_own, bar)
    assert missing == 0 and wrong == 0, (missing, wrong)
    assert cover > min_cover, cover
    return idx, val, ref


def _size(which, dev):
    return dict(cityscapes=2975, coco=118287, two_passes=2 * R.TILE * _sms(dev) + 77)[which]


@pytest.mark.parametrize("which,E", [("cityscapes", 384), ("coco", 384), ("two_passes", 768)])
def test_parity_clustered(cuda_dev, which, E):
    n = _size(which, cuda_dev)
    _assert_parity(f"clustered_{which}_E{E}", R.clustered(n, E, n + E), 30, cuda_dev, MIN_COVER[E])


@pytest.mark.parametrize("which,E", [("cityscapes", 384), ("coco", 384), ("two_passes", 768)])
def test_parity_and_self_first_with_near_duplicates(cuda_dev, which, E):
    """Exact and near copies of a row (eps 0, 1e-7, 1e-5, 1e-3 relative), before and after their original and across
    half tiles, tiles and row blocks: the row itself still comes first, its copy second."""
    n = _size(which, cuda_dev)
    x, pairs, eps = R.near_duplicates(n, E, n + E)
    idx, val, _ = _assert_parity(f"near_duplicates_{which}_E{E}", x, 30, cuda_dev, MIN_COVER[E])
    a, b = pairs[:, 0].to(cuda_dev), pairs[:, 1].to(cuda_dev)
    assert torch.equal(idx[a, 1], b) and torch.equal(idx[b, 1], a)
    same = (eps == 0).to(cuda_dev)
    # a bitwise copy has bitwise the row's own similarity (same operand planes, same order): only the rule separates them
    assert torch.equal(val[a[same], 1], val[a[same], 0]) and torch.equal(val[b[same], 1], val[b[same], 0])
    assert (b[same] < a[same]).any()                  # ... also where (value desc, index asc) would put the copy first


@pytest.mark.parametrize("n,E,k", [(2975, 384, 30), (1000, 64, 32), (130, 128, 5)])
def test_parity_scaled_rows_and_zero_row(cuda_dev, n, E, k):
    """Row norms from 1e-6 to 1e6 leave the answer alone; an all-zero row (every similarity exactly 0) lists itself,
    then the lowest indices."""
    x, z = R.scaled_rows(n, E, n)
    idx, val, _ = _assert_parity(f"scaled_rows_n{n}_E{E}", x, k, cuda_dev, 0.3)
    assert idx[z].tolist() == [z] + [j for j in range(k) if j != z][:k - 1]
    assert (val[z] == 0).all()


# ------------------------------------------------------------------------------------------------
# call-level properties
# ------------------------------------------------------------------------------------------------
def test_calls_are_deterministic_and_layout_independent(cuda_dev):
    n, E, k = 5000, 384, 30
    x, _, _ = R.near_duplicates(n, E, 9)
    x = x.to(cuda_dev)
    idx, val = _knn(x, k, cuda_dev)
    idx2, val2 = _knn(x, k, cuda_dev)
    assert torch.equal(idx, idx2) and torch.equal(val, val2)
    idx3, none = _knn(x, k, cuda_dev, values=False)
    assert none is None and torch.equal(idx, idx3)
    wide = torch.full((n, 2 * E + 3), 7.0, device=cuda_dev)
    wide[:, 1:2 * E + 1:2] = x
    view = wide[:, 1:2 * E + 1:2]
    assert not view.is_contiguous()
    idx4, val4 = _knn(view, k, cuda_dev)
    assert torch.equal(idx, idx4) and torch.equal(val, val4)
    side = torch.cuda.Stream(cuda_dev)
    side.wait_stream(torch.cuda.current_stream(cuda_dev))
    with torch.cuda.stream(side):
        idx5, val5 = _knn(x, k, cuda_dev)
    side.synchronize()
    assert torch.equal(idx, idx5) and torch.equal(val, val5)


@pytest.mark.parametrize("n,E,k", [(300, 64, 7), (129, 128, 32), (1, 64, 1)])
def test_c_abi_writes_only_its_outputs(cuda_dev, n, E, k):
    """idx_out, val_out and planes_scratch carved out of larger pre-filled buffers: nothing outside [n][k] and
    2 n E is touched — the rows of the last row block past n in particular."""
    from stego_b200 import _lib
    lib = _lib.load()
    pad = 8192  # more than the (128 - n % 128) * k elements a whole last row block would spill
    x = R.exact_lattice(n, E, 4).to(cuda_dev)
    ibuf = torch.full((n * k + 2 * pad,), -7, dtype=torch.long, device=cuda_dev)
    vbuf = torch.full((n * k + 2 * pad,), -7.0, device=cuda_dev)
    pbuf = torch.full((2 * n * E + 2 * pad,), 12345.0, dtype=torch.bfloat16, device=cuda_dev)
    rc = lib.stego_knn_topk(_lib.ptr(x), n, E, k, _lib.ptr(pbuf[pad:]), _lib.ptr(ibuf[pad:]), _lib.ptr(vbuf[pad:]),
                            _lib.stream())
    _lib.check(rc, "stego_knn_topk")
    torch.cuda.synchronize()
    idx, val = _knn(x, k, cuda_dev)
    assert torch.equal(ibuf[pad:pad + n * k].view(n, k), idx) and torch.equal(vbuf[pad:pad + n * k].view(n, k), val)
    for buf, fill, size in ((ibuf, -7, n * k), (vbuf, -7.0, n * k), (pbuf, 12345.0, 2 * n * E)):
        assert (buf[:pad] == fill).all() and (buf[pad + size:] == fill).all()
    planes = pbuf[pad:pad + 2 * n * E].float().view(2, n, E)
    assert (planes[0].abs() <= 0.25).all() and (planes[1] == 0).all()  # normalised lattice rows: hi exact, lo zero


def test_c_abi_rejects_bad_arguments_without_launching(cuda_dev):
    from stego_b200 import _lib
    from stego_b200.knn import knn_topk
    lib = _lib.load()
    n, E = 5, 64
    x = torch.randn(n, E, device=cuda_dev)
    planes = torch.zeros(2 * n * E + 8, dtype=torch.bfloat16, device=cuda_dev)
    idx = torch.full((n * 32,), -7, dtype=torch.long, device=cuda_dev)
    torch.cuda.synchronize()
    before = _lib.launch_count()
    call = lambda k, p, i: lib.stego_knn_topk(_lib.ptr(x), n, E, k, p, i, 0, _lib.stream())
    for k, p, i, msg in ((7, _lib.ptr(planes), _lib.ptr(idx), "k=7"), (0, _lib.ptr(planes), _lib.ptr(idx), "k=0"),
                         (3, _lib.ptr(planes) + 2, _lib.ptr(idx), "aligned"), (3, _lib.ptr(planes), 0, "null"),
                         (3, 0, _lib.ptr(idx), "null")):
        rc = call(k, p, i)
        assert rc != 0 and msg in _lib.last_error(), (k, rc, _lib.last_error())
    assert _lib.launch_count() == before
    torch.cuda.synchronize()
    assert (idx == -7).all()
    with pytest.raises(RuntimeError, match="k=7"):
        knn_topk(x, 7)
    with pytest.raises(RuntimeError, match="stego_knn_topk"):  # k = 0: the empty output has no address to pass
        knn_topk(x, 0)
    assert call(5, _lib.ptr(planes), _lib.ptr(idx)) == 0   # n == k on the same buffers is accepted
