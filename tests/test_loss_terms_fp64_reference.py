"""CPU pins of the fp64 loss-term references (tests/_loss_terms_fp64.py): ContrastiveCRFLoss against the oracle
(oracle/stego_oracle.py::contrastive_crf_loss, itself pinned to the reference module) run in float64 with its autograd
gradient, the pixel cosine against (F.normalize(a) * F.normalize(b)).sum(1) in float64 with autograd (the exact-eps
case included), and the input builders against the edges they claim to produce."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _loss_terms_fp64 as R  # noqa: E402


def _close(x, y, tol=1e-12):
    x, y = x.detach().double(), y.detach().double()
    return float((x - y).abs().max()) <= tol * max(float(y.abs().max()), 1e-300)


CRF_CASES = [  # B, C, Cg, H, W, n, coords, codes, params
    (2, 70, 3, 56, 56, 150, "random", "train", R.PARAMS),
    (2, 5, 3, 12, 12, 77, "repeats", "wide", (0.5, 1e-3, 0.05, 10.0, 3.0, 0.7)),
    (1, 3, 1, 1, 9, 40, "random", "onehot", (0.5, 0.15, 0.05, 0.0, 3.0, 0.0)),
    (3, 4, 2, 7, 1, 65, "corners", "dyadic", (0.5, 0.15, 0.05, 10.0, 0.0, 0.05)),
    (1, 6, 3, 9, 9, 33, "identical", "train", R.PARAMS),
]


def _codes(kind, B, C, H, W, gen):
    if kind == "wide":
        return R.wide_codes(B, C, H, W, gen)
    if kind == "onehot":
        return R.onehot_codes(B, C, H, W, gen)
    if kind == "dyadic":
        return R.dyadic_codes(B, C, H, W, gen)
    return F.normalize(torch.randn(B, C, H, W, generator=gen), dim=1)


@pytest.mark.parametrize("B,C,Cg,H,W,n,ckind,code,params", CRF_CASES)
def test_crf_reference_matches_oracle_fp64(B, C, Cg, H, W, n, ckind, code, params):
    import stego_oracle as O
    gen = torch.Generator().manual_seed(B * 100 + C + n)
    gd = (torch.rand(B, Cg, H, W, generator=gen) * 4 - 2).double()
    cl = _codes(code, B, C, H, W, gen).double()
    coords = R.coords_of(ckind, n, H, W, gen)
    ref = R.crf_loss(gd, cl, coords, *params)
    c = cl.clone().requires_grad_(True)
    # the int64 |dp|^2 divided by a Python float takes the default dtype: float64 here, so the whole oracle is fp64
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        want = O.contrastive_crf_loss(gd, c, coords, *params)
    finally:
        torch.set_default_dtype(old)
    assert want.dtype == torch.float64
    assert _close(ref["out"], want)
    for kind in ("mean", "random", "symmetric", "antisymmetric"):
        up = R.upstream(kind, B, n, gen).double()
        gw, = torch.autograd.grad((want * up).sum(), c, retain_graph=True)
        bw = R.crf_loss_bwd(ref, up, coords, cl.shape)
        assert _close(bw["dclusters"], gw), kind
        if kind == "antisymmetric":
            assert (bw["gs"] == 0).all() and (bw["dclusters"] == 0).all()
    # the pieces: out = -G s and the |term| sums
    assert torch.equal(ref["out"], -(ref["G"] * ref["s"]))
    assert (ref["absG"] >= ref["G"].abs() * (1 - 1e-15)).all()


def test_crf_builders_make_their_edges():
    gen = torch.Generator().manual_seed(0)
    H = W = 56
    r = R.repeats(R.coords_of("repeats", 1000, H, W, gen), H, W)
    assert r.sum() == 1000 and (r[4:] == 0).all() and (r[:, 4:] == 0).all() and r.max() >= 62
    d = R.coords_of("distinct", 1000, H, W, gen)
    assert R.repeats(d, H, W).max() == 1
    i = R.coords_of("identical", 100, H, W, gen)
    assert R.repeats(i, H, W).max() == 100
    cn = R.coords_of("corners", 64, H, W, gen)
    assert set(map(tuple, cn.t().tolist())) <= {(0, 0), (0, W - 1), (H - 1, 0), (H - 1, W - 1)}
    # one-hot codes: G is exactly 0 or 1, both occur
    oh = R.onehot_codes(2, 5, 8, 8, gen)
    ref = R.crf_loss(torch.zeros(2, 3, 8, 8), oh, R.random_coords(50, 8, 8, gen), *R.PARAMS)
    assert ((ref["G"] == 0) | (ref["G"] == 1)).all() and (ref["G"] == 0).any() and (ref["G"] == 1).any()
    # dyadic codes: the fp32 Gram chain is exact, in either order
    dy = R.dyadic_codes(1, 80, 4, 4, gen)
    v = dy.reshape(80, 16)
    acc = torch.zeros(16, 16)
    for k in range(80):
        acc = acc + v[k][:, None] * v[k][None, :]
    assert torch.equal(acc.double(), v.double().t() @ v.double())
    # un-normalised codes span 1e-3 ... 1e3 per pixel
    w = R.wide_codes(1, 70, 40, 40, gen).norm(dim=1)
    assert float(w.min()) < 1e-2 and float(w.max()) > 1e2
    # training inputs: ImageNet-normalised guidance, unit-norm codes at 56^2
    g, c = R.training_inputs(2, 70, gen)
    assert g.shape == (2, 3, 56, 56) and c.shape == (2, 70, 56, 56)
    assert float(g.min()) < -1.5 and float(g.max()) > 2.0
    assert _close(c.double().norm(dim=1), torch.ones(2, 56, 56), 1e-6)
    # antisymmetric upstream gradients cancel exactly in fp32 as well
    a = R.upstream("antisymmetric", 2, 65, gen)
    assert (a + a.transpose(1, 2) == 0).all()


def test_crf_fp32_params_are_what_the_abi_receives():
    p32 = R.fp32_params(R.PARAMS + (1e-3,))
    for x, y in zip(p32, R.PARAMS + (1e-3,)):
        assert x == float(torch.tensor(y, dtype=torch.float32)) and abs(x - y) <= 2 ** -24 * abs(y)
    assert R.f32(0.15) != 0.15 and R.f32(0.5) == 0.5


@pytest.mark.parametrize("kind,C", [(k, C) for k in ("random", "parallel", "antiparallel", "orthogonal", "onehot")
                                     for C in (1, 33, 70) if not (k == "onehot" and C == 1)])  # one-hot pairs need C >= 2
def test_pixel_cosine_reference_matches_autograd_fp64(kind, C):
    gen = torch.Generator().manual_seed(C)
    a, b = R.cosine_pairs(kind, 2, C, 5, 6, gen)
    a[0, :, 0, 0] = 0  # a zero vector: clamped norm
    _pin_cosine(a, b, torch.randn(2, 5, 6, generator=gen))


def test_pixel_cosine_reference_at_eps():
    """F.normalize's clamp_min passes the gradient at |a| == eps: the tangential term is there at exactly eps, one fp32
    step above, and absent below."""
    a, b, xs = R.eps_vectors(4)
    g = torch.ones(a.shape[0], 1, 1)
    ref = _pin_cosine(a, b, g)
    da = ref["da"][:, :, 0, 0]
    assert float(ref["na"][0]) == R.EPS32 and xs[0] == R.EPS32
    ia = 1 / R.EPS32
    assert abs(da[0, 0]) < 1e-15 * ia and da[0, 1] > 0.4 * ia  # exactly eps: d/da_0 = ia (b_hat_0 - cos) = 0
    assert da[1, 0] > 0.8 * ia                                  # one step below: no tangential term, ia b_hat_0
    assert abs(da[2, 0]) < 1e-15 * ia                           # one step above
    assert (ref["da"][4] == ref["bh"][4] / R.EPS32).all()  # zero vector: ia b_hat
    # the builders' edges: the fp32 norm the kernels form (sqrt of the fp32 square) is x itself for the three
    # boundary values, and the fp32 sums of squares of the large ones are finite
    for x in xs[:3]:
        t = torch.tensor(x, dtype=torch.float32)
        assert float(torch.sqrt(t * t)) == x
    assert xs[1] < R.EPS32 < xs[2]
    for x in xs[5:]:
        t = torch.tensor(x, dtype=torch.float32)
        assert torch.isfinite(t * t)


def _pin_cosine(a, b, g):
    ad, bd = a.double().requires_grad_(True), b.double().requires_grad_(True)
    want = (F.normalize(ad, dim=1, eps=R.EPS32) * F.normalize(bd, dim=1, eps=R.EPS32)).sum(1)
    wa, wb = torch.autograd.grad((want * g.double()).sum(), (ad, bd))
    ref = R.pixel_cosine(a, b, ga=g)
    # relative to sum_c |a_hat_c b_hat_c| (orthogonal pairs cancel to ~1e-9)
    assert float(((ref["cos"] - want.detach()).abs() / (ref["absab"] * ref["ia"] * ref["ib"]).clamp_min(1e-300)).max()) <= 1e-14
    # relative to the magnitude of each pixel's terms, g ia (|b_hat| + |cos| |a_hat|): the gradient itself cancels for
    # (anti)parallel pairs and C = 1, and the zero and eps vectors' gradients are 1/eps-scaled
    cos = ref["cos"].abs()[:, None]
    for got, w, i, x, y in ((ref["da"], wa, ref["ia"], ref["ah"], ref["bh"]), (ref["db"], wb, ref["ib"], ref["bh"], ref["ah"])):
        scale = ((g.double().abs() * i)[:, None] * (y.abs() + cos * x.abs())).amax(1, keepdim=True).clamp_min(1e-300)
        assert float(((got - w).abs() / scale).max()) <= 1e-14
    return ref
