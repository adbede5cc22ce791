"""The fp64 CRF references of tests/_crf_fp64.py pinned on the CPU to the fp32 restatement oracle/crf_oracle.py on
small frames, to their own exact identities, and to stego_b200.crf's key packing; and the input builders checked for
the edges they claim."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _crf_fp64 as R  # noqa: E402
from _parity_util import ROOT  # noqa: E402,F401  (puts oracle/ on sys.path)

import crf_oracle as CO  # noqa: E402

# (name, H, W, d, sxy, image kind)
FRAMES = [("pos", 12, 17, 2, 1.0, None), ("pos_1x37", 1, 37, 2, 1.0, None), ("pos_37x1", 37, 1, 2, 1.0, None),
          ("bil_piecewise", 14, 19, 5, 67.0, "piecewise"), ("bil_noise", 9, 13, 5, 67.0, "noise"),
          ("bil_black", 6, 7, 5, 67.0, "black"), ("bil_saturated", 6, 7, 5, 67.0, "saturated"),
          ("bil_constant", 8, 11, 5, 67.0, "constant"), ("bil_2x2", 2, 2, 5, 67.0, "noise")]


def _frame(H, W, d, sxy, kind, seed=None):
    img = None if d == 2 else R.image(kind, H, W, H * W if seed is None else seed)
    f64 = R.features(H, W, d, sxy, R.BI_RGB_STD, img)
    if d == 2:
        f32 = CO.gaussian_features(H, W, sxy)
    else:
        f32 = CO.bilateral_features(img.numpy(), sxy, R.BI_RGB_STD)
    return img, f64, f32


def _key_bar(e, d):
    """what separates a decision the fp32 restatement must take like fp64: twice the fp32 bound on elevated
    (gamma_{d+10} of its |terms|, tests/test_crf_fp64_gpu.py) plus the subtractions"""
    return 2 * R.gamma(d + 10) * e["elev_abs"].amax(1) + 8 * R.U * (d + 1)


@pytest.mark.parametrize("name,H,W,d,sxy,kind", FRAMES, ids=[f[0] for f in FRAMES])
def test_embedding_and_tables_match_restatement(name, H, W, d, sxy, kind):
    """Same vertices, offsets and neighbour tables as the restatement on frames where every pixel is an exact tie
    (identical in both precisions) or clear of a tie by more than the fp32 bar; barycentric weights within it."""
    _, f64, f32 = _frame(H, W, d, sxy, kind)
    e = R.embed(f64)
    clear = (e["margin"] == 0) | (e["margin"] > _key_bar(e, d))
    assert clear.all(), f"{name}: {int((~clear).sum())} near-tie pixels"
    lat = CO.Permutohedral(f32)
    want = torch.from_numpy(lat.keys[lat.offset])                              # [N, d+1, d]
    assert torch.equal(e["vertices"][..., :d], want)
    t = R.lattice_tables(e["vertices"])
    assert t["M"] == lat.M
    assert torch.equal(t["offset"], torch.from_numpy(lat.offset))
    assert torch.equal(t["n1"], torch.from_numpy(lat.n1)) and torch.equal(t["n2"], torch.from_numpy(lat.n2))
    assert torch.equal(t["points"][:, :d], torch.from_numpy(lat.keys))
    bary_bar = 2 * R.gamma(d + 10) * e["elev_abs"].amax(1, keepdim=True) / (d + 1) + 4 * R.gamma(6)
    assert ((e["bary"] - torch.from_numpy(lat.bary).double()).abs() <= bary_bar).all()


@pytest.mark.parametrize("name,H,W,d,sxy,kind", FRAMES + [("pos_big", 64, 128, 2, 1.0, None),
                                                          ("bil_noise_big", 48, 64, 5, 67.0, "noise"),
                                                          ("bil_far", 3, 5380, 5, 67.0, "saturated")],
                         ids=[f[0] for f in FRAMES] + ["pos_big", "bil_noise_big", "bil_far"])
def test_embedding_identities(name, H, W, d, sxy, kind):
    """sum_r bary_r vertex_r = elevated, bary >= 0, sum bary = 1, the vertices form a lattice simplex."""
    _, f64, _ = _frame(H, W, d, sxy, kind)
    e = R.embed(f64)
    rec = (e["bary"][:, :, None] * e["vertices"].double()).sum(1)
    assert ((rec - e["elevated"]).abs() <= 1e-12 * (1 + e["elev_abs"])).all()
    assert (e["bary"] >= -1e-12).all()
    assert ((e["bary"].sum(1) - 1).abs() < 1e-12).all()
    assert R.is_simplex(e["vertices"]).all()
    # a vertex set that is not a simplex is refused
    bad = e["vertices"].clone()
    bad[0, 1, 0] += d + 1
    bad[0, 1, 1] -= d + 1
    assert not R.is_simplex(bad)[0]


@pytest.mark.parametrize("d,kind", [(2, None), (5, "noise"), (5, "piecewise")])
def test_tables_match_fixed_width_packing(d, kind):
    """The mixed-radix numbering is the order of stego_b200.crf's sorted fixed-width keys, neighbours included, and
    the CSR list is the stable sort crf._lattice_points makes; the concatenation matches crf._bilateral_lattice's
    bases."""
    from stego_b200 import crf
    H, W = 23, 31
    _, f64, _ = _frame(H, W, d, 1.0 if d == 2 else 7.0, kind, seed=3)
    e = R.embed(f64)
    t = R.lattice_tables(e["vertices"])
    bits = 60 // d
    keys = crf._pack(e["vertices"][..., :d].reshape(-1, d), d, bits)
    uniq, inv = torch.unique(keys, return_inverse=True)
    assert torch.equal(inv.reshape(-1, d + 1), t["offset"])
    assert torch.equal(crf._unpack(uniq, d, bits), t["points"][:, :d])
    assert torch.equal(R.unpack(keys.reshape(-1, d + 1), d, bits), e["vertices"])
    ids = t["offset"].reshape(-1)
    order = torch.argsort(ids, stable=True)
    assert torch.equal(t["slots"], order)
    assert torch.equal(t["rowptr"], torch.searchsorted(ids[order], torch.arange(t["M"] + 1)))
    # n2 undoes n1 along every axis
    for j in range(d + 1):
        has = t["n1"][j] >= 0
        assert torch.equal(t["n2"][j][t["n1"][j][has]], torch.arange(t["M"])[has])
    cat, bases = R.concat([t, t])
    assert cat["M"] == 2 * t["M"] and bases.tolist() == [0, t["M"]]
    assert torch.equal(cat["offset"][H * W:], t["offset"] + t["M"])
    assert torch.equal(cat["slots"][t["slots"].numel():], t["slots"] + H * W * (d + 1))
    assert int(cat["rowptr"][-1]) == 2 * H * W * (d + 1)


def _oracle_lattice(lat):
    return R.lattice(torch.from_numpy(lat.offset), torch.from_numpy(lat.bary), torch.from_numpy(lat.n1),
                     torch.from_numpy(lat.n2), lat.M)


@pytest.mark.parametrize("H,W,C", [(14, 19, 5), (9, 13, 27), (2, 2, 3)])
def test_filter_norm_and_mean_field_match_restatement(H, W, C):
    """On the restatement's own lattices: the filter, the normalisation and the 10-iteration marginals are within
    fp32 distance of it; the filter is adjoint to its reversed-axis twin."""
    img = R.image("piecewise", H, W, seed=H)
    kg = CO.DenseKernel(CO.gaussian_features(H, W, R.POS_XY_STD))
    kb = CO.DenseKernel(CO.bilateral_features(img.numpy(), R.BI_XY_STD, R.BI_RGB_STD))
    lg, lb = _oracle_lattice(kg.lattice), _oracle_lattice(kb.lattice)
    g = torch.Generator().manual_seed(C)
    x = torch.rand(H * W, C, generator=g, dtype=torch.float64)
    y = torch.rand(H * W, C, generator=g, dtype=torch.float64)
    for k, lat in ((kg, lg), (kb, lb)):
        out = R.filter(lat, x, bars=True)
        want = torch.from_numpy(k.lattice.compute(x.float().numpy())).double()
        mag = R.slice_(lat, out["mag"][-1])[1] * R.alpha(lat["d"])
        assert ((out["out"] - want).abs() <= 1e-5 * mag + 1e-30).all()
        n, nb = R.norm(lat, bars=True)
        assert ((n - torch.from_numpy(k.norm).double()).abs() <= 1e-5 * n).all()
        assert (nb["bar"] > 0).all() and (nb["bar"] < 1e-5 * n).all()
        rev = R.filter(lat, y, reverse=True)["out"]
        lhs, rhs = (out["out"] * y).sum(), (x * rev).sum()
        assert abs(float(lhs - rhs)) <= 1e-12 * float(lhs)
        # ... and the forward filter itself is not symmetric in the pass order (the adjoint check has teeth)
        if H * W > 4:
            assert not torch.allclose(R.filter(lat, y)["out"], rev, rtol=1e-9, atol=0)
    logits = R.logits("random", H * W, C, seed=H + C)
    U, _ = R.unary_from_logits(logits)
    want = CO.mean_field(U.float().numpy(), [kg, kb], [CO.POS_W, CO.Bi_W], CO.MAX_ITER)
    seq = R.mean_field(U, lg, lb, R.MAX_ITER, record=True)
    assert len(seq) == R.MAX_ITER + 1
    assert ((seq[0] - R.softmax(-U)).abs() == 0).all()
    err = (seq[-1] - torch.from_numpy(want).double()).abs().max().item()
    assert err < 2e-5, err
    assert ((seq[-1].sum(1) - 1).abs() < 1e-12).all()


def test_unary_reference():
    """softmax, the clip at 1e-5 and -log against the restatement's unary_from_softmax"""
    z = R.logits("random", 200, 27, seed=1)
    U, p = R.unary_from_logits(z)
    want = CO.unary_from_softmax(p.float().numpy().T).T
    assert np.abs(U.numpy() - want).max() < 1e-5


def test_builders_produce_their_edges():
    H, W = 16, 24
    assert (R.image("black", H, W) == 0).all() and (R.image("saturated", H, W) == 255).all()
    c = R.image("constant", H, W, seed=2)
    assert (c == c[0, 0]).all()
    n = R.image("noise", 64, 64, seed=2)
    assert int(n.min()) == 0 and int(n.max()) == 255
    pw = R.image("piecewise", H, W, seed=2)
    assert pw.reshape(-1, 3).unique(dim=0).shape[0] > 16
    # the normalised frames round-trip through the reference's own image preparation
    frames = torch.stack([pw, n[:H, :W], R.image("saturated", H, W), R.image("black", H, W)])
    x = R.normalised(frames)
    for b in range(frames.shape[0]):
        assert np.array_equal(CO.prepare_image(x[b]), frames[b].numpy())
    # black: exactly zero colour coordinates, every pixel an exact rank tie; constant: one colour, the lattice of the
    # colour-free frame (the most slots per point)
    e = R.embed(R.features(H, W, 5, R.BI_XY_STD, R.BI_RGB_STD, R.image("black", H, W)))
    assert (e["elevated"][:, 3:] == 0).all() and (e["margin"] == 0).all()
    ec = R.lattice_tables(R.embed(R.features(H, W, 5, R.BI_XY_STD, R.BI_RGB_STD, c))["vertices"])
    en = R.lattice_tables(R.embed(R.features(H, W, 5, R.BI_XY_STD, R.BI_RGB_STD, n[:H, :W]))["vertices"])
    assert ec["counts"].max() > 4 * en["counts"].max() and ec["M"] < en["M"]
    # unaries
    N, C = 500, 27
    U, p = R.unary_from_logits(R.logits("onehot", N, C))
    assert ((p < 1e-5).sum(1) == C - 1).all()
    assert ((U == -np.log(1e-5)).sum(1) == C - 1).all()
    _, p = R.unary_from_logits(R.logits("straddle", N, C))
    off = p[p < 0.5]
    assert (off > 1e-5).sum() > 1000 and (off < 1e-5).sum() > 1000 and ((off / 1e-5 - 1).abs() < 2e-3).all()
    z = R.logits("uniform", N, C)
    assert (z == z[0, 0]).all()
