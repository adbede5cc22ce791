"""The optional loss-term kernels against the float64 references of tests/_loss_terms_fp64.py, elementwise:
ContrastiveCRFLoss (csrc/crf_loss.cu: gather, Gram x pairwise-kernel tile, recomputing backward, atomic scatter) and
the per-pixel cosine of the reconstruction / augmentation-alignment terms (csrc/cosine_loss.cu, warp-per-pixel and
thread-per-pixel paths), stand-alone and inside the autograd training step.

Bars (u = 2^-24, gamma_k = k u / (1 - k u); no fast-math in build.py, so sqrtf and '/' are correctly rounded and expf
is within 2 ulp (CUDA C Programming Guide, mathematical functions), i.e. 4u relative above the subnormal range and
2^-148 absolute in it; every |term| sum comes from the reference, the parameters are the fp32 values the C ABI gets;
each rounding also carries eta = 2^-150 absolute, the gradual-underflow term of the rounding model, which the pairwise
kernel's products reach: e^-100 times a Gram entry of 1e-4 is below the smallest subnormal):
  crf forward   t1 = -cd inv2a - gd inv2b with cd an exact integer, inv2a = fl(1 / 2 alpha) (one rounding), the three
                guidance differences, their squares and two sums: |dt1| <= gamma_3 tp + gamma_8 tg, |dt2| <= gamma_3 |t2|.
                |de| <= e (|dt| (1 + 2 |dt|) + 4u) + 2^-148.  s = w1 e1 + w2 e2 - shift: three roundings per term,
                |ds| <= |w1| |de1| + |w2| |de2| + gamma_3 (|w1| e1 + |w2| e2 + |shift|).  The Gram entry is a C-term
                FMA chain: |dG| <= gamma_C sum_k |c_a c_b|.  out = -(G s) rounds once:
                |dout| <= |s| |dG| + |G| |ds| + |dG| |ds| + u (|G| + |dG|) (|s| + |ds|).
  crf backward  W = -fl(g_ab + g_ba) s rounds twice: |dW| <= |gs| |ds| + gamma_2 |gs| (|s| + |ds|).  d sel is a chain of
                NP = ceil(n / 64) 64 FMAs (the zero padding included): |d dsel| <= gamma_NP sum_b (|W| + |dW|) |sel_b| +
                sum_b |dW| |sel_b|.  A pixel sampled r times receives r atomics onto zero: gamma_r of the sum of its
                |dsel| + bars, added to the sum of the bars.  The PTX ISA has atom / red .add.f32 flush subnormal inputs and
                results to zero, so each atomic also carries 2 * 2^-126 absolute: one-hot codes reach it, where a
                gradient of -1.2e-38 (a far pair's W summed over one class) comes back as 0.
  cosine        the sums of squares and of products are k-term chains: k = C on the thread path, ceil(C / 32) + 5
                (the lane chain and five shuffle levels) on the warp path: eS = gamma_k.  1 / max(sqrt(.), eps) carries
                eN = eS / 2 + eS^2 + gamma_2 of relative error (max is 1-Lipschitz, so the clamp adds none).
                cos = sab ia ib: |dcos| <= (1 + eN)^2 eS ia ib sum |a b| + |cos| ((1 + eN)^2 (1 + gamma_2) - 1).
                d/da = fl(fl(g ia) fl(fl(b ib) - k fl(a ia))) with k = cos where |a| >= eps: a_hat, b_hat carry
                eH = eN + u + eN u, so |dt| <= |b_hat| eH + (|cos| + |dcos|) |a_hat| eH + |dcos| |a_hat| (1 + eH), plus the
                fma's u (|t| + |dt|); |d da| <= |g| ia [((1 + eN)(1 + gamma_2) - 1) |t| + (1 + eN)(1 + gamma_2) |dt|].
                The bar carries u (|b_hat| + |cos| |a_hat|) + |dcos| |a_hat|, not u |t|: where t cancels (nearly
                parallel pairs) no relative accuracy is asked for.  A pixel whose norm is within the fp32 norm's error
                of eps may take either side of the clamp: its bar also carries the whole tangential term
                |g| ia (|cos| + |dcos|) |a_hat| (1 + eH).  The exact-eps vectors have an exact fp32 norm (the CPU test
                checks sqrt(fl(x^2)) = x), so they get no such band.
The largest error / bar per quantity is printed and written to $STEGO_PARITY_DIR when that is set.
"""
import math
import os
import sys

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _loss_terms_fp64 as R  # noqa: E402
from _parity_util import record  # noqa: E402

pytestmark = pytest.mark.gpu
U, G = R.U, R.gamma
ETA = 2.0 ** -150  # the absolute error of one rounding in fp32's subnormal range (half the smallest subnormal)
TINY = 2.0 ** -126  # the smallest normal fp32
NAN = float("nan")


def _ratio(err, bar):
    err, bar = err.detach().double(), bar.detach().double()
    if not err.numel():
        return 0.0
    return float(torch.where(err == 0, torch.zeros_like(err), err / bar).max())


class Ratios(dict):
    """largest err / bar per quantity; `check` asserts after everything is recorded"""

    def add(self, name, got, ref, bar):
        r = _ratio((got.double() - ref.double()).abs(), bar)
        self[name] = max(self.get(name, 0.0), r)
        return r

    def check(self, tag):
        print(tag, {k: f"{v:.3g}" for k, v in self.items()})
        record(tag, dict(self))
        bad = {k: v for k, v in self.items() if not v <= 1.0}
        assert not bad, (tag, bad)


# ================================================================================================
# ContrastiveCRFLoss
# ================================================================================================
def crf_bars(ref, C, p32):
    """forward bar [B, n, n] and the bound on |s_kernel - s| (see the module docstring)"""
    _, _, _, w1, w2, shift = p32
    dt1 = G(3) * ref["tp"] + G(8) * ref["tg"]
    dt2 = G(3) * ref["t2"].abs()
    de1 = ref["e1"] * (dt1 * (1 + 2 * dt1) + 4 * U) + 2.0 ** -148
    de2 = ref["e2"] * (dt2 * (1 + 2 * dt2) + 4 * U) + 2.0 ** -148
    ds = abs(w1) * de1 + abs(w2) * de2 + G(3) * (abs(w1) * ref["e1"] + abs(w2) * ref["e2"] + abs(shift)) + 3 * ETA
    dG = G(C) * ref["absG"] + C * ETA
    s, Gm = ref["s"].abs(), ref["G"].abs()
    return s * dG + Gm * ds + dG * ds + U * (Gm + dG) * (s + ds) + ETA, ds


def crf_bwd_bar(ref, gout, coords, shape, ds, n):
    gs = (gout.double() + gout.double().transpose(1, 2)).abs()
    wbar = gs * ds + G(2) * gs * (ref["s"].abs() + ds) + 2 * ETA
    bw = R.crf_loss_bwd(ref, gout, coords, shape, wbar=wbar)
    NP = -(-n // 64) * 64
    dsel_bar = G(NP) * (bw["dsel_abs"] + bw["dsel_werr"]) + bw["dsel_werr"] + NP * ETA
    r = bw["repeats"].double()
    gr = (r * U / (1 - r * U))[None, None]
    bar = R.scatter(dsel_bar, coords, shape) + gr * R.scatter(bw["dsel"].abs() + dsel_bar, coords, shape) + r * 2 * TINY
    return bw, bar


def _crf_run(gd, cl, coords, p, gouts):
    """forward and, per upstream gradient (None: .mean()), the backward through the public module"""
    from stego_b200.modules import ContrastiveCRFLoss
    mod = ContrastiveCRFLoss(coords.shape[1], *p)
    c = cl.detach().requires_grad_(True)
    out = mod.forward_with_coords(gd, c, coords)
    grads = []
    for go in gouts:
        if go is None:
            g, = torch.autograd.grad(out.mean(), c, retain_graph=True)
        else:
            g, = torch.autograd.grad(out, c, go, retain_graph=True)
        grads.append(g)
    return out.detach(), grads


def _crf_check(tag, gd, cl, coords, p, kinds=("mean", "random", "symmetric", "antisymmetric"), seed=0):
    dev = cl.device
    B, C, H, W = cl.shape
    n = coords.shape[1]
    gen = torch.Generator().manual_seed(seed)
    gouts = [None if k == "mean" else R.upstream(k, B, n, gen).to(dev) for k in kinds]
    out, grads = _crf_run(gd, cl, coords, p, gouts)
    p32 = R.fp32_params(p)
    ref = R.crf_loss(gd, cl, coords, *p32)
    fbar, ds = crf_bars(ref, C, p32)
    rat = Ratios()
    rat.add("out", out, ref["out"], fbar)
    assert torch.isfinite(out).all()
    for k, go, g in zip(kinds, gouts, grads):
        if go is None:
            go = torch.full((B, n, n), 1.0 / (B * n * n), dtype=torch.float32, device=dev)
        bw, bar = crf_bwd_bar(ref, go, coords, cl.shape, ds, n)
        if g.dtype == torch.bfloat16:  # autograd returns a bf16 leaf's gradient in bf16: one more rounding, 2^-8
            bar = bar + 2.0 ** -8 * (bw["dclusters"].abs() + bar)
        rat.add(f"dclusters_{k}", g, bw["dclusters"], bar)
        if k == "antisymmetric":  # g_ab + g_ba == 0 exactly, so W and the whole gradient are exactly zero
            assert (g == 0).all()
        del bw, bar
    rat.check(tag)
    return out, grads, ref


CRF_SHAPES = [  # B, C, Cg, H, W, n
    (32, 70, 3, 56, 56, 1000), (16, 70, 3, 56, 56, 1000),
    *[(2, 70, 3, 56, 56, n) for n in (1, 3, 4, 63, 64, 65, 127, 128, 129, 1024, 2000)],
    *[(3, C, 3, 56, 40, 203) for C in (1, 3, 4, 5, 27, 64, 77, 79, 80)],
    (2, 70, 1, 56, 40, 300), (2, 70, 2, 1, 56, 130), (2, 70, 3, 56, 1, 130),
]


@pytest.mark.parametrize("B,C,Cg,H,W,n", CRF_SHAPES)
def test_crf_loss_fp64_shapes(cuda_dev, B, C, Cg, H, W, n):
    gen = torch.Generator().manual_seed(B * 7919 + C * 31 + n)
    gd, cl = R.training_inputs(B, C, gen, dev=cuda_dev)
    gd = gd[:, :Cg].contiguous()
    if H != 56 or W != 56:
        gd = F.interpolate(gd, (H, W), mode="bilinear", align_corners=False)
        cl = F.normalize(F.interpolate(cl, (H, W), mode="bilinear", align_corners=False), dim=1, eps=R.EPS)
    coords = R.random_coords(n, H, W, gen).to(cuda_dev)
    _crf_check(f"crf_B{B}_C{C}_Cg{Cg}_{H}x{W}_n{n}", gd, cl, coords, R.PARAMS)


REGIMES = {  # name: (params, codes, coords)
    "sharp": ((0.5, 1e-3, 0.05, 10.0, 3.0, 0.0), "train", "random"),
    "shift": ((0.5, 0.15, 0.05, 10.0, 3.0, 0.7), "train", "random"),
    "w1_zero": ((0.5, 0.15, 0.05, 0.0, 3.0, 0.0), "train", "random"),
    "w2_zero": ((0.5, 0.15, 0.05, 10.0, 0.0, 0.0), "train", "random"),
    "onehot": (R.PARAMS, "onehot", "random"),
    "wide": ((0.5, 0.15, 0.05, 10.0, 3.0, 0.3), "wide", "random"),
    "distinct": (R.PARAMS, "train", "distinct"),
    "repeats": (R.PARAMS, "train", "repeats"),
    "identical": ((0.5, 0.15, 0.05, 10.0, 3.0, 0.2), "train", "identical"),
    "corners": (R.PARAMS, "train", "corners"),
}


@pytest.mark.parametrize("regime", list(REGIMES))
def test_crf_loss_fp64_regimes(cuda_dev, regime):
    p, codes, ckind = REGIMES[regime]
    B, C, H, W, n = 4, 70, 56, 56, 1000
    gen = torch.Generator().manual_seed(len(regime))
    gd, cl = R.training_inputs(B, C, gen, dev=cuda_dev)
    if codes == "onehot":
        cl = R.onehot_codes(B, C, H, W, gen).to(cuda_dev)
    elif codes == "wide":
        cl = R.wide_codes(B, C, H, W, gen).to(cuda_dev)
    coords = R.coords_of(ckind, n, H, W, gen).to(cuda_dev)
    out, _, ref = _crf_check(f"crf_{regime}", gd, cl, coords, p)
    if codes == "onehot":  # G is exactly 0 or 1: out is exactly 0 where G = 0
        assert (out[ref["G"] == 0] == 0).all()


@pytest.mark.parametrize("layout", ["nchw", "channels_last", "sliced", "batch_slice", "bf16", "guidance_cl"])
def test_crf_loss_fp64_layouts(cuda_dev, layout):
    B, C, H, W, n = 3, 70, 56, 56, 500
    gen = torch.Generator().manual_seed(11)
    gd, cl = R.training_inputs(B + 2, C + 2, gen, dev=cuda_dev)
    gd, base = gd[:B].contiguous(), cl
    cl = base[:B, :C].contiguous()
    if layout == "channels_last":
        cl = cl.contiguous(memory_format=torch.channels_last)
    elif layout == "sliced":  # a channel slice of a 72-channel channels-last tensor: padded pixel pitch
        cl = base[:B].contiguous(memory_format=torch.channels_last)[:, :C]
    elif layout == "batch_slice":
        cl = base[1:B + 1, :C]
    elif layout == "bf16":
        cl = cl.bfloat16()
    elif layout == "guidance_cl":
        gd = gd.contiguous(memory_format=torch.channels_last)
    coords = R.random_coords(n, H, W, gen).to(cuda_dev)
    _, grads, _ = _crf_check(f"crf_layout_{layout}", gd, cl, coords, R.PARAMS, kinds=("random", "antisymmetric"))
    assert grads[0].shape == cl.shape


def test_crf_loss_exact_cases(cuda_dev):
    """Dyadic codes make every Gram entry exact, so on the diagonal (a = b or the same position: cd = gd = 0, both
    exponentials are expf(-0) = 1 and s = w1 + w2 - shift exactly) out == -fl(|c|^2) (w1 + w2 - shift) bit for bit;
    the padding rows and columns of the 64-tiles are never written (NaN sentinels around out); two forwards, and
    without repeated positions two backwards, are bit-identical."""
    from stego_b200 import _lib
    lib = _lib.load()
    B, C, H, W, n = 3, 70, 56, 56, 1000
    gen = torch.Generator().manual_seed(5)
    gd, _ = R.training_inputs(B, C, gen, dev=cuda_dev)
    cl = R.dyadic_codes(B, C, H, W, gen).to(cuda_dev)
    coords = R.coords_of("repeats", n, H, W, gen).to(cuda_dev)
    p = (0.5, 0.15, 0.05, 10.0, 3.0, 0.5)
    out, _ = _crf_run(gd, cl, coords, p, [])
    sel = cl.double()[:, :, coords[0], coords[1]]
    G2 = torch.einsum("bka,bkc->bac", sel, sel)
    same = ((coords[0][:, None] == coords[0][None]) & (coords[1][:, None] == coords[1][None]))[None].expand(B, n, n)
    assert same.sum() > B * n  # repeated positions besides the diagonal
    want = -(G2 * 12.5).float()
    assert torch.equal(out[same], want[same])
    # NaN sentinels around the output of the raw entry point: only the n x n elements are written
    NP = -(-n // 64) * 64
    pad = 4096
    buf = torch.full((B * n * n + 2 * pad,), NAN, device=cuda_dev)
    sel_ws = torch.empty(B, C, NP, device=cuda_dev)
    gsel = torch.empty(B, NP, 4, device=cuda_dev)
    pos = torch.empty(NP, 2, dtype=torch.int32, device=cuda_dev)
    o = buf[pad:pad + B * n * n]
    _lib.check(lib.stego_crf_loss_fwd(gd.data_ptr(), *gd.stride(), 3, cl.data_ptr(), *cl.stride(), C, coords.data_ptr(),
                                      B, n, H, W, *map(float, p), sel_ws.data_ptr(), gsel.data_ptr(), pos.data_ptr(),
                                      o.data_ptr(), _lib.stream()), "stego_crf_loss_fwd")
    torch.cuda.synchronize()
    assert torch.isnan(buf[:pad]).all() and torch.isnan(buf[pad + B * n * n:]).all()
    assert torch.equal(o.view(B, n, n), out)
    # determinism
    gd2, cl2 = R.training_inputs(B, C, gen, dev=cuda_dev)
    up = R.upstream("random", B, n, gen).to(cuda_dev)
    for ckind, bwd_same in (("repeats", False), ("distinct", True)):
        co = R.coords_of(ckind, n, H, W, gen).to(cuda_dev)
        o1, (g1,) = _crf_run(gd2, cl2, co, R.PARAMS, [up])
        o2, (g2,) = _crf_run(gd2, cl2, co, R.PARAMS, [up])
        assert torch.equal(o1, o2)
        if bwd_same:
            assert torch.equal(g1, g2)


def test_crf_loss_refuses_unsupported(cuda_dev):
    """C <= 80 (the backward's four channel groups of CL_KMAX = 20) and at most three guidance channels: anything else is
    an error from the library, not a wrong answer."""
    from stego_b200.modules import ContrastiveCRFLoss
    gen = torch.Generator().manual_seed(0)
    coords = R.random_coords(100, 8, 8, gen).to(cuda_dev)
    mod = ContrastiveCRFLoss(100, *R.PARAMS)
    with pytest.raises(RuntimeError, match="C <= 80"):
        mod.forward_with_coords(torch.rand(2, 3, 8, 8, device=cuda_dev), torch.randn(2, 81, 8, 8, device=cuda_dev), coords)
    with pytest.raises(RuntimeError, match="guidance channels <= 3"):
        mod.forward_with_coords(torch.rand(2, 4, 8, 8, device=cuda_dev), torch.randn(2, 80, 8, 8, device=cuda_dev), coords)


# ================================================================================================
# pixel_cosine
# ================================================================================================
def cos_bars(ref, C, warp, g, kink=True):
    k = math.ceil(C / 32) + 5 if warp else C
    eS = G(k)
    eN = eS / 2 + eS * eS + G(2)
    eH = eN + U + eN * U
    cos = ref["cos"].abs()
    dcos = (1 + eN) ** 2 * eS * ref["ia"] * ref["ib"] * ref["absab"] + cos * ((1 + eN) ** 2 * (1 + G(2)) - 1)
    bars = {}
    gg = g.double().abs()
    for name, i, n, x, y in (("da", ref["ia"], ref["na"], ref["ah"], ref["bh"]), ("db", ref["ib"], ref["nb"], ref["bh"], ref["ah"])):
        on = (n >= R.EPS32)[:, None]
        kk = torch.where(on, cos[:, None], torch.zeros_like(x))
        dk = torch.where(on, dcos[:, None], torch.zeros_like(x))
        t = (y - torch.where(on, ref["cos"][:, None], torch.zeros_like(x)) * x).abs()
        dt0 = y.abs() * eH + (kk + dk) * x.abs() * eH + dk * x.abs() * (1 + eH)
        dt = dt0 + U * (t + dt0)
        f = (1 + eN) * (1 + G(2))
        bar = (gg * i)[:, None] * ((f - 1) * t + f * dt)
        if kink:
            near = ((n - R.EPS32).abs() <= (eS / 2 + eS * eS + U) * n)[:, None]
            bar = bar + torch.where(near, (gg * i)[:, None] * (cos[:, None] + dcos[:, None]) * x.abs() * (1 + eH) * (1 + G(3)),
                                    torch.zeros_like(bar))
        bars[name] = bar
    return dcos, bars


def _cos_check(tag, a, b, up, need=(True, True), kink=True, rat=None):
    from stego_b200.modules import pixel_cosine
    a_ = a.detach().requires_grad_(need[0])
    b_ = b.detach().requires_grad_(need[1])
    got = pixel_cosine(a_, b_)
    ins = [t for t, nd in zip((a_, b_), need) if nd]
    gr = torch.autograd.grad(got, ins, up)
    grads = dict(zip([nm for nm, nd in zip(("da", "db"), need) if nd], gr))
    warp = a.stride(1) == 1 and b.stride(1) == 1
    ref = R.pixel_cosine(a, b, ga=up)
    dcos, bars = cos_bars(ref, a.shape[1], warp, up, kink)
    own = rat is None
    rat = Ratios() if own else rat
    rat.add("cos", got.detach(), ref["cos"], dcos)
    for nm, g in grads.items():
        assert g.shape == a.shape
        rat.add(nm, g, ref[nm], bars[nm])
    if own:
        rat.check(tag)
    return got.detach(), grads, ref


def _cl(t):
    return t.contiguous(memory_format=torch.channels_last)


@pytest.mark.parametrize("path", ["warp", "thread"])
@pytest.mark.parametrize("C", [1, 31, 32, 33, 63, 64, 65, 70, 384, 768])
def test_pixel_cosine_fp64_channels(cuda_dev, C, path):
    gen = torch.Generator().manual_seed(C)
    rat = Ratios()
    for kind in ("random", "parallel", "antiparallel", "orthogonal", "onehot"):
        if kind == "onehot" and C < 2:
            continue
        a, b = R.cosine_pairs(kind, 4, C, 9, 11, gen)
        a[0, :, 0, 0] = 0
        b[1, :, 2, 3] = 0
        a, b = a.to(cuda_dev), b.to(cuda_dev)
        if path == "warp":
            a, b = _cl(a), _cl(b)
        up = torch.randn(4, 9, 11, generator=gen).to(cuda_dev)
        got, _, _ = _cos_check("", a, b, up, rat=rat)
        if kind == "onehot":  # disjoint supports: every product is exactly zero
            assert (got == 0).all()
    rat.check(f"cos_C{C}_{path}")


@pytest.mark.parametrize("E,side,B", [(384, 28, 32), (768, 40, 32), (768, 56, 16)])
def test_pixel_cosine_fp64_rec_shapes(cuda_dev, E, side, B):
    """the reconstruction term: a = the decoder's NCHW output, b = the channels-last backbone features (mixed layouts:
    thread path)"""
    gen = torch.Generator(device=cuda_dev).manual_seed(E + side)
    a = torch.randn(B, E, side, side, device=cuda_dev, generator=gen)
    b = _cl(torch.randn(B, E, side, side, device=cuda_dev, generator=gen) * 2)
    up = torch.full((B, side, side), -1.0 / (B * side * side), device=cuda_dev)
    _cos_check(f"cos_rec_E{E}_{side}_B{B}", a, b, up)
    _cos_check(f"cos_rec_cl_E{E}_{side}_B{B}", _cl(a), b, up)


def test_pixel_cosine_fp64_aug_shape(cuda_dev):
    """the augmentation term at c1: C = 70 codes stored on a 72-float pixel pitch (channel stride 1: warp path), and a
    batch-strided view; one operand requiring grad at a time"""
    gen = torch.Generator(device=cuda_dev).manual_seed(3)
    B, C, h = 32, 70, 28
    store = _cl(torch.randn(2 * B, 72, h, h, device=cuda_dev, generator=gen))
    a, b = store[:B, :C], store[B:, :C]
    assert a.stride(1) == 1 and a.stride(3) == 72
    up = torch.randn(B, h, h, device=cuda_dev, generator=gen)
    _cos_check("cos_aug_pitch72", a, b, up)
    _cos_check("cos_aug_only_a", a, b, up, need=(True, False))
    _cos_check("cos_aug_only_b", a, b, up, need=(False, True))
    nchw = torch.randn(2 * B, C, h, h, device=cuda_dev, generator=gen)
    _cos_check("cos_batch_strided", nchw[::2], nchw[1::2], up)


def test_pixel_cosine_broadcast_operand(cuda_dev):
    """a prototype broadcast over every pixel (stride 0): its gradient is the sum over pixels of each pixel's gradient"""
    from stego_b200.modules import pixel_cosine
    gen = torch.Generator(device=cuda_dev).manual_seed(9)
    B, C, H, W = 4, 70, 9, 11
    proto = torch.randn(B, C, device=cuda_dev, generator=gen)
    b = torch.randn(B, C, H, W, device=cuda_dev, generator=gen)
    up = torch.randn(B, H, W, device=cuda_dev, generator=gen)
    for feats in (b, _cl(b)):
        p = proto.clone().requires_grad_(True)
        got = pixel_cosine(p[:, :, None, None].expand(B, C, H, W), feats)
        dp, = torch.autograd.grad(got, p, up)
        a = proto[:, :, None, None].expand(B, C, H, W)
        ref = R.pixel_cosine(a, feats, ga=up)
        dcos, bars = cos_bars(ref, C, False, up)  # the overlapping operand is made dense NCHW: thread path
        rat = Ratios()
        rat.add("cos", got.detach(), ref["cos"], dcos)
        # the sum over H W pixels adds (HW - 1) fp32 roundings of torch's reduction
        rat.add("dproto", dp, ref["da"].sum((2, 3)),
                bars["da"].sum((2, 3)) + G(H * W) * (ref["da"].abs() + bars["da"]).sum((2, 3)))
        rat.check(f"cos_broadcast_{'cl' if feats.stride(1) == 1 else 'nchw'}")


def test_pixel_cosine_at_eps(cuda_dev):
    """a = x e_0 with x at the clamp boundary, b = (1, 0.5, 0, ...): F.normalize passes the tangential term at
    |a| == eps (clamp_min's gradient is taken where input >= min), so d/da_0 = ia (b_hat_0 - cos) = 0 there, not
    ia b_hat_0.  The fp32 norms of these vectors are exact, so no clamp band is allowed.  Both paths, cos bit-equal
    between them."""
    rat = Ratios()
    for C in (4, 70):
        a, b, _ = R.eps_vectors(C, cuda_dev)
        up = torch.ones(a.shape[0], 1, 1, device=cuda_dev)
        c1, g1, ref = _cos_check("", a, b, up, kink=False, rat=rat)
        a2 = torch.zeros(a.shape[0], 2 * C, 1, 1, device=cuda_dev)
        a2[:, ::2] = a
        c2, g2, _ = _cos_check("", a2[:, ::2], b, up, kink=False, rat=rat)  # channel stride 2: thread path
        assert torch.equal(c1, c2)  # at most two nonzero terms per sum: exact in either order
        assert torch.isfinite(g1["da"]).all() and torch.isfinite(g1["db"]).all()
        assert abs(float(g1["da"][0, 0, 0, 0])) <= 1e-6 * float(ref["ia"][0])  # the tangential term is there
    rat.check("cos_eps")


# ================================================================================================
# inside the training step
# ================================================================================================
TERMS = {"rec": dict(rec_weight=0.7), "aug": dict(aug_alignment_weight=0.6), "crf": dict(crf_weight=0.5),
         "all": dict(rec_weight=0.7, aug_alignment_weight=0.6, crf_weight=0.5)}


def _mean_bar(ref_abs, bar, N):
    """torch's fp32 mean over N elements, treated as a chain of 4 ceil(sqrt(N)) additions (its CUDA reduction keeps
    per-thread partial sums and combines them in a tree; an assumption, not a documented order) plus the division"""
    return bar.mean() + G(4 * math.ceil(math.sqrt(N)) + 1) * (ref_abs + bar).mean()


@pytest.mark.parametrize("terms", list(TERMS))
def test_training_step_loss_terms_fp64(cuda_dev, terms, monkeypatch):
    """ViT-S/8 224^2 c1 (B = 32) on the autograd path with the optional terms on: the tensors reaching pixel_cosine and
    ContrastiveCRFLoss are the fp32 restatement of train_segmentation.py:183-208 on the step's own code, features (with
    the m3 dropout mask), code_aug, coord_aug and image; the kernels' outputs and the gradients they return are within
    the bars above of fp64 on those tensors; the logged terms are their means; the decoder's weight / bias gradients
    are fp64 of the rec term on the captured tensors (only rec reaches the decoder); the total is the sum of the logged terms."""
    import stego_b200.segmenter as S
    from _parity_util import fp32_strict, make_batch, make_model
    from stego_b200.modules import norm, sample
    tf32 = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    fp32_strict()  # the decoder's convolutions in fp32, so its weight gradient has an fp32 bar
    try:
        B, res = 32, 224
        w = TERMS[terms]
        model, _ = make_model("vit_small", cuda_dev, fused=True, batch_size=B, res=res, **w)
        batch = make_batch(B, res, cuda_dev)
        g = torch.Generator().manual_seed(4)
        batch["img_aug"] = (batch["img"].cpu() + 0.2 * torch.randn(B, 3, res, res, generator=g)).to(cuda_dev)
        batch["coord_aug"] = (torch.rand(B, res, res, 2, generator=g) * 2 - 1).to(cuda_dev)
        net = model.net
        heads, masks = [], []
        head_code, draw_masks = net.head_code, net.draw_masks

        def rec_head(tok, *a, **k):
            out = head_code(tok, *a, **k)
            heads.append((tok.detach().clone(), out.detach().clone()))
            return out

        def rec_masks(*a, **k):
            m = draw_masks(*a, **k)
            masks.append([x.clone() if x is not None else None for x in m])
            return m
        monkeypatch.setattr(net, "head_code", rec_head)
        monkeypatch.setattr(net, "draw_masks", rec_masks)
        cos_calls, crf_calls = [], []
        pixel_cosine = S.pixel_cosine

        def keep(entry, key):
            def hook(gr):
                entry[key] = gr.detach().clone()
            return hook

        def rec_cos(a, b):
            out = pixel_cosine(a, b)
            e = dict(a=a.detach().clone(), b=b.detach().clone(), out=out.detach().clone(), need=(a.requires_grad, b.requires_grad))
            for t, key in ((a, "da"), (b, "db"), (out, "g")):
                if t.requires_grad:
                    t.register_hook(keep(e, key))
            cos_calls.append(e)
            return out
        monkeypatch.setattr(S, "pixel_cosine", rec_cos)
        crf_fn = model.crf_loss_fn

        class RecCrf(torch.nn.Module):
            def forward(self, guidance, clusters):
                coords = crf_fn.draw_coords(guidance.shape[2], guidance.shape[3], clusters.device)
                out = crf_fn._apply_kernel(guidance, clusters, coords)
                e = dict(guidance=guidance.detach().clone(), clusters=clusters.detach().clone(), coords=coords.clone(),
                         out=out.detach().clone())
                clusters.register_hook(keep(e, "dclusters"))
                out.register_hook(keep(e, "g"))
                crf_calls.append(e)
                return out
        model.crf_loss_fn = RecCrf()
        dec = {k: v.detach().clone() for k, v in model.decoder.state_dict().items()}
        torch.manual_seed(21)
        total = model.training_step(batch, 0)
        torch.cuda.synchronize()
        assert model._fused is not None and not model._fused.supported(batch)
        logged = model.logged
        tok, code_all = heads[0]
        code = code_all[:B]
        m3 = masks[0][2]
        fh = res // 8
        E = tok.shape[-1]
        feats_f = tok[:B].view(B, fh, fh, E).permute(0, 3, 1, 2).float() * m3.view(B, E, 1, 1)
        rat = Ratios()
        i = 0
        if "rec_weight" in w:
            e = cos_calls[i]
            i += 1
            assert torch.equal(e["b"], feats_f)
            with torch.no_grad():
                assert torch.allclose(e["a"], _decoder_at(model.decoder, dec)(code), rtol=1e-6, atol=1e-6)
            ref, N = _cos_step(rat, "rec", e, cuda_dev)
            rat.add("loss_rec", logged["loss/rec"], -ref["cos"].mean(),
                    _mean_bar(ref["cos"].abs(), ref["dcos"], N))
            # the decoder (a 1x1 convolution, segmenter.py): dW = sum_p da_p code_p^T, db = sum_p da_p
            model.flush()
            da = ref["da"] * 1.0
            cd = code.double()
            gw = torch.einsum("bepq,bkpq->ek", da, cd)
            gw_abs = torch.einsum("bepq,bkpq->ek", da.abs() + ref["bars"]["da"], cd.abs())
            gw_bar = torch.einsum("bepq,bkpq->ek", ref["bars"]["da"], cd.abs()) + G(B * fh * fh) * gw_abs
            lw = model.decoder.weight.grad
            rat.add("decoder_w", lw.view(lw.shape[0], -1), gw, gw_bar)
            gb = da.sum((0, 2, 3))
            gb_bar = ref["bars"]["da"].sum((0, 2, 3)) + G(B * fh * fh) * (da.abs() + ref["bars"]["da"]).sum((0, 2, 3))
            rat.add("decoder_b", model.decoder.bias.grad, gb, gb_bar)
        if "aug_alignment_weight" in w:
            e = cos_calls[i]
            i += 1
            coord = F.interpolate(batch["coord_aug"].permute(0, 3, 1, 2), e["b"].shape[2], mode="bilinear",
                                  align_corners=False).permute(0, 2, 3, 1)
            assert torch.equal(e["a"], sample(code, coord))
            assert e["b"].shape == code.shape and e["need"] == (True, True)
            ref, N = _cos_step(rat, "aug", e, cuda_dev)
            rat.add("loss_aug", logged["loss/aug_alignment"], -ref["cos"].mean(), _mean_bar(ref["cos"].abs(), ref["dcos"], N))
        assert i == len(cos_calls)
        if "crf_weight" in w:
            e, = crf_calls
            rs = lambda t: F.interpolate(t, 56, mode="bilinear", align_corners=False)
            assert torch.equal(e["guidance"], rs(batch["img"]))
            assert torch.equal(e["clusters"], norm(rs(code)))
            n = e["coords"].shape[1]
            p32 = R.fp32_params(R.PARAMS)
            ref = R.crf_loss(e["guidance"], e["clusters"], e["coords"], *p32)
            fbar, ds = crf_bars(ref, e["clusters"].shape[1], p32)
            rat.add("crf_out", e["out"], ref["out"], fbar)
            bw, bar = crf_bwd_bar(ref, e["g"], e["coords"], e["clusters"].shape, ds, n)
            rat.add("crf_dclusters", e["dclusters"], bw["dclusters"], bar)
            rat.add("loss_crf", logged["loss/crf"], ref["out"].mean(), _mean_bar(ref["out"].abs(), fbar, ref["out"].numel()))
        # the total is the weighted sum of the logged terms (eight fp32 additions / products at most)
        cfg = model.cfg
        parts = [cfg.pos_inter_weight * logged["loss/pos_inter"], cfg.pos_intra_weight * logged["loss/pos_intra"],
                 cfg.neg_inter_weight * logged["loss/neg_inter"], logged["loss/linear"], logged["loss/cluster"]]
        parts += [cfg.rec_weight * logged["loss/rec"]] if "rec_weight" in w else []
        parts += [cfg.aug_alignment_weight * logged["loss/aug_alignment"]] if "aug_alignment_weight" in w else []
        parts += [cfg.crf_weight * logged["loss/crf"]] if "crf_weight" in w else []
        want = sum(float(p) for p in parts)
        assert abs(float(total) - want) <= G(16) * sum(abs(float(p)) for p in parts)
        assert float(logged["loss/total"]) == float(total)
        rat.check(f"step_{terms}")
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32


def _decoder_at(decoder, state):
    """a copy of the decoder with the weights it had before the step's update"""
    import copy
    d = copy.deepcopy(decoder)
    d.load_state_dict(state)
    return d


def _cos_step(rat, name, e, dev):
    a, b = e["a"], e["b"]
    ref = R.pixel_cosine(a, b, ga=e["g"])
    warp = a.stride(1) == 1 and b.stride(1) == 1
    dcos, bars = cos_bars(ref, a.shape[1], warp, e["g"])
    ref["dcos"], ref["bars"] = dcos, bars
    rat.add(f"{name}_cos", e["out"], ref["cos"], dcos)
    for key, nd in zip(("da", "db"), e["need"]):
        if nd:
            rat.add(f"{name}_{key}", e[key], ref[key], bars[key])
    return ref, ref["cos"].numel()
