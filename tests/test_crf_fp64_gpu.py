"""The dense CRF against the float64 references of tests/_crf_fp64.py, stage by stage and elementwise: csrc/crf.cu
with one probe per row (stego_b200.crf: dense_crf / batched_crf) and with two (stego_b200.eval.fused_eval_crf), at
the c4 frame (1024 x 2048, 27 classes), the reference eval batch (16 x 320^2, n_lin != n_clu) and small edge frames.

Bars (u = 2^-24, gamma_k = k u / (1 - k u)):
  embedding    elevated: the features x * fp32(1 / sxy) (two roundings), the scale factors (five) and their product
               (one) carry 8 u relative, the running sum and j cf another d + 2: gamma_{d+10} sum |terms| (el_bar).
               Keys equal fp64's wherever the pixel's fp64 decision margin exceeds 2 max el_bar + 8 (d+1) u (an exact
               fp64 tie such as el_0 - el_2 = 72 at x = 0 need not be one in fp32).  Everywhere: the vertices form a
               lattice simplex; sum_r bary_r v_r reconstructs the exact elevated within el_bar + mean(el_bar) +
               4 gamma_5 sum_r |v_r| (the identity holds exactly for the kernel's own elevated projected on the
               hyperplane sum = 0, so only its error, spread by the projection, and the weights' arithmetic remain);
               bary >= -bar and sum bary = 1
               within 4 (d+1) gamma_6.  Against fp64 off near-ties, absolute: 2 max el_bar / (d+1) + 4 gamma_6 (a
               weight is the difference of two residuals / (d+1)): it cannot be relative, the residuals cancel
               |elevated|.
  tables       exact: M, offsets, both neighbour tables, the CSR list and the per-frame bases of the concatenation.
  splat        gamma_{m_i + 1} sum |b v| over the m_i slots of point i (summed in CSR order; the bar holds for any).
  blur pass    err' = blur(err) (1 + gamma_2) + gamma_2 blur(magnitudes)   (two roundings of old + 0.5 (a + b)).
  norm         half the relative error of the slice (propagated blur error + gamma_{d+4} of its |terms|) plus the
               correctly rounded sqrt and divide.
  update       |dt| <= the propagated error of both slices + gamma_{d+6} and gamma_2 of their |terms| + gamma_2 |U|;
               |dq| <= q (2 max |dt| + eps_i + sum_j q_j eps_j + (n + 2) u) + 2^-126, eps = __expf's
               2 + floor(1.173 |z|) ulp.  Argmax equal to fp64's wherever the fp64 top-2 gap exceeds twice the
               pixel's largest q bar, and always the lowest index among the lanes holding the maximum.
  unary        the bound of test_eval_crf_gpu.py::test_unary_matches_fp64 with exact scores: 2 ((2 + |z|) 2^-23 +
               u |z| + (n + 4) u + 3 2^-19); Q_0 = softmax(-U) stage-wise from the kernel's U with the update's q bar.
  chain        no derived bar (mean field is not contractive): max |dQ| recorded, held to 2e-3, labels equal off
               near-ties (fp64 top-2 gap > 2 max |dQ|).
The largest err / bar per quantity is written to $STEGO_PARITY_DIR when it is set.
"""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _crf_fp64 as R  # noqa: E402
from _parity_util import record  # noqa: E402

pytestmark = pytest.mark.gpu
U, G = R.U, R.gamma
LD = 32


def _lib():
    from stego_b200 import _lib
    return _lib


class Ratios(dict):
    """largest err / bar per quantity; `check` asserts after everything is recorded"""

    def add(self, name, err, bar):
        err, bar = err.detach().double(), bar.detach().double()
        r = float(torch.where(err == 0, torch.zeros_like(err), err / bar).max()) if err.numel() else 0.0
        self[name] = max(self.get(name, 0.0), r)
        return r

    def check(self, tag, **extra):
        record(tag, dict(self, **extra))
        bad = {k: v for k, v in self.items() if not v <= 1.0}
        assert not bad, (tag, bad)


def _sxy(d):
    return R.POS_XY_STD if d == 2 else R.BI_XY_STD


def _kernel_keys(H, W, d, img, dev):
    L = _lib()
    keys = torch.empty(H * W, d + 1, dtype=torch.long, device=dev)
    bary = torch.empty(H * W, d + 1, dtype=torch.float32, device=dev)
    L.check(L.load().stego_crf_lattice(H, W, d, _sxy(d), R.BI_RGB_STD, L.ptr(img), L.ptr(keys), L.ptr(bary),
                                       L.stream()), "stego_crf_lattice")
    return keys, bary


def _max_width(H, d=5, sxy=R.BI_XY_STD, srgb=R.BI_RGB_STD):
    """the widest frame stego_crf_lattice accepts: its coordinate bound (d+1) 0.8165 (2 max(H, W) / sxy + 3 * 255 /
    srgb) + 2 (d+1) below 2^(bits-1), bits = 60 / d"""
    bits = 60 // d
    ok = lambda W: (d + 1) * 0.8165 * (max(W, H) / sxy * 2 + 3 * 255.0 / srgb) + 2 * (d + 1) < 2 ** (bits - 1)
    W = H
    while ok(W + 1):
        W += 1
    return W


FAR_W = _max_width(3)

# ================================================================================================
# 1. embedding
# ================================================================================================
EMBED = [("pos_c4", 1024, 2048, 2, None), ("bil_c4_piecewise", 1024, 2048, 5, "piecewise"),
         ("bil_c4_noise", 1024, 2048, 5, "noise"), ("bil_320_noise", 320, 320, 5, "noise"),
         ("bil_black", 37, 53, 5, "black"), ("bil_saturated", 37, 53, 5, "saturated"),
         ("bil_constant", 37, 53, 5, "constant"), ("pos_1x1", 1, 1, 2, None), ("bil_1x37", 1, 37, 5, "noise"),
         ("bil_37x1", 37, 1, 5, "noise"), ("bil_2x2", 2, 2, 5, "noise"), ("bil_far", 3, FAR_W, 5, "saturated")]


@pytest.mark.parametrize("name,H,W,d,kind", EMBED, ids=[e[0] for e in EMBED])
def test_embedding(cuda_dev, name, H, W, d, kind):
    img = None if d == 2 else R.image(kind, H, W, seed=H + W).to(cuda_dev)
    keys, bary = _kernel_keys(H, W, d, img, cuda_dev)
    e = R.embed(R.features(H, W, d, _sxy(d), R.BI_RGB_STD, img, cuda_dev))
    verts = R.unpack(keys, d, 60 // d)
    el_bar = G(d + 10) * e["elev_abs"]
    key_bar = 2 * el_bar.amax(1) + 8 * (d + 1) * U
    b = bary.double()
    rat = Ratios()
    assert R.is_simplex(verts).all(), name
    assert int(e["vertices"][..., :d].abs().max()) < 2 ** (60 // d - 1)     # the packed fields cannot wrap
    rec = (b[:, :, None] * verts.double()).sum(1)
    # vertices sum to 0 and the weights to 1, so the reconstruction is the kernel's elevated projected on the
    # hyperplane sum = 0: each coordinate also carries the mean of the others' errors
    rbar = el_bar + el_bar.mean(1, keepdim=True) + 4 * G(5) * verts.double().abs().sum(1)
    rat.add("reconstruction", (rec - e["elevated"]).abs(), rbar)
    bary_bar = 2 * el_bar.amax(1, keepdim=True) / (d + 1) + 4 * G(6)
    rat.add("bary_negative", (-b).clamp_min(0), bary_bar.expand_as(b))
    rat.add("bary_sum", (b.sum(1) - 1).abs(), torch.full_like(b[:, 0], 4 * (d + 1) * G(6)))
    clear = e["margin"] > key_bar
    same = (verts == e["vertices"]).all(2).all(1)
    bad = (~same & clear).nonzero()[:4, 0].tolist()
    assert not bad, (name, int((~same & clear).sum()), [(i, float(e["margin"][i]), float(key_bar[i]), verts[i].tolist(),
                                                        e["vertices"][i].tolist(), e["elevated"][i].tolist())
                                                       for i in bad])
    rat.add("bary", (b - e["bary"])[clear].abs(), bary_bar.expand_as(b)[clear])
    near = int((~clear).sum())
    print(f"{name}: near-tie pixels {near} of {H * W}, keys differing there {int((~same).sum())}; {dict(rat)}")
    rat.check(f"crf_embed_{name}", near_ties=near, differing_keys=int((~same).sum()))


def test_argument_check_refuses_one_column_more(cuda_dev):
    """the widest accepted frame is embedded above (bil_far); one column more is refused with its message"""
    L = _lib()
    H, W = 3, FAR_W + 1
    img = torch.full((H, W, 3), 255, dtype=torch.uint8, device=cuda_dev)
    keys = torch.empty(H * W, 6, dtype=torch.long, device=cuda_dev)
    bary = torch.empty(H * W, 6, dtype=torch.float32, device=cuda_dev)
    with pytest.raises(RuntimeError, match="do not fit 12-bit keys"):
        L.check(L.load().stego_crf_lattice(H, W, 5, R.BI_XY_STD, R.BI_RGB_STD, L.ptr(img), L.ptr(keys), L.ptr(bary),
                                           L.stream()), "stego_crf_lattice")
    assert 5300 < FAR_W < 5400


# ================================================================================================
# 2. lattice tables
# ================================================================================================
def _tables_equal(lat, t):
    assert lat.M == t["M"]
    assert torch.equal(lat.offset.long(), t["offset"])
    assert torch.equal(lat.n1.long(), t["n1"]) and torch.equal(lat.n2.long(), t["n2"])
    assert torch.equal(lat.slots.long(), t["slots"]) and torch.equal(lat.rowptr.long(), t["rowptr"])
    for j in range(t["d"] + 1):
        has = lat.n1[j] >= 0
        i = torch.arange(lat.M, device=lat.n1.device)[has]
        assert torch.equal(lat.n2[j][lat.n1[j][has].long()].long(), i)


TABLES = [("pos_c4", 1, 1024, 2048, 2, None), ("bil_c4_noise", 1, 1024, 2048, 5, "noise"),
          ("bil_c4_piecewise", 1, 1024, 2048, 5, "piecewise"), ("bil_320_noise_x16", 16, 320, 320, 5, "noise"),
          ("bil_37x53_mixed", 5, 37, 53, 5, None), ("pos_1x1", 1, 1, 1, 2, None), ("bil_1x37", 2, 1, 37, 5, "noise"),
          ("bil_37x1", 2, 37, 1, 5, "constant"), ("bil_2x2", 3, 2, 2, 5, "black"),
          ("bil_far", 1, 3, FAR_W, 5, "saturated")]


@pytest.mark.parametrize("name,B,H,W,d,kind", TABLES, ids=[t[0] for t in TABLES])
def test_crf_lattice_tables(cuda_dev, name, B, H, W, d, kind):
    """crf._lattice_points (with its CSR list) and crf._bilateral_lattice's concatenation equal the tables rebuilt from
    the kernel's keys with an independent packing."""
    from stego_b200 import crf
    if d == 2:
        keys, _ = _kernel_keys(H, W, 2, None, cuda_dev)
        t = R.lattice_tables(R.unpack(keys, 2, 30))
        lat = crf._lattice_points(H, W, 2, R.POS_XY_STD, 0.0, None, cuda_dev)
        _tables_equal(lat, t)
        return
    kinds = [kind] * B if kind else list(R.IMAGES)[:B]
    imgs = torch.stack([R.image(k, H, W, seed=10 * b + H) for b, k in enumerate(kinds)]).to(cuda_dev)
    x = R.normalised(imgs.cpu()).to(cuda_dev)
    per = []
    for b in range(B):
        assert torch.equal(crf.prepare_image(x[b]), imgs[b])
        keys, _ = _kernel_keys(H, W, 5, imgs[b], cuda_dev)
        per.append(R.lattice_tables(R.unpack(keys, 5, 12)))
        if b == 0:
            lat = crf._lattice_points(H, W, 5, R.BI_XY_STD, R.BI_RGB_STD, imgs[b], cuda_dev)
            _tables_equal(lat, per[0])
        del keys
    want, bases = R.concat(per)
    got = crf._bilateral_lattice(crf.prepare_image(f) for f in x)
    _tables_equal(got, want)
    print(f"{name}: M per frame {[p['M'] for p in per]}, N {H * W}, bases {bases.tolist()}")


# ================================================================================================
# 3. filter and normalisation
# ================================================================================================
def _lat64(lat):
    return R.lattice(lat.offset, lat.bary, lat.n1, lat.n2, lat.M)


def _probs(N, C, seed, dev):
    g = torch.Generator().manual_seed(seed)
    return torch.softmax(torch.randn(N, C, generator=g) * 2, 1).to(dev)


FILTER = [("c4_piecewise", 1024, 2048, "piecewise", 27), ("320_noise", 320, 320, "noise", 32),
          ("37x53_constant", 37, 53, "constant", 3), ("37x53_black", 37, 53, "black", 1),
          ("1x37_saturated", 1, 37, "saturated", 2), ("37x1", 37, 1, "noise", 27), ("2x2", 2, 2, "noise", 27),
          ("1x1", 1, 1, "noise", 5)]


def _call_norm(lat, dev):
    L = _lib()
    v = torch.full((2, lat.M), float("nan"), device=dev)
    out = torch.empty(lat.N, device=dev)
    L.check(L.load().stego_crf_norm(lat.d, lat.N, lat.M, L.ptr(lat.offset), L.ptr(lat.bary), L.ptr(lat.rowptr),
                                    L.ptr(lat.slots), L.ptr(lat.n1), L.ptr(lat.n2), L.ptr(v[0]), L.ptr(v[1]), L.ptr(out),
                                    L.stream()), "stego_crf_norm")
    return v, out


def _setup(B, H, W, kinds, dev, seed=0):
    """crf.py's lattices for B frames and the fp64 views of them: the position lattice repeated B times and the
    concatenated bilateral lattice, both over B*N pixels"""
    from stego_b200 import crf
    imgs = torch.stack([R.image(k, H, W, seed=seed + 7 * b) for b, k in enumerate(kinds)])
    x = R.normalised(imgs).to(dev)
    lg = crf._position_lattice(H, W, dev)
    lb = crf._bilateral_lattice(crf.prepare_image(f) for f in x)
    g1 = _lat64(lg)
    t = dict(d=2, N=H * W, M=lg.M, offset=g1["offset"], n1=g1["n1"], n2=g1["n2"], rowptr=lg.rowptr.long(),
             slots=lg.slots.long(), counts=g1["counts"])
    gcat, _ = R.concat([t] * B)
    g64 = R.lattice(gcat["offset"], lg.bary.repeat(B, 1), gcat["n1"], gcat["n2"], gcat["M"])
    return x, lg, lb, g64, _lat64(lb)


def _call_mf(B, N, n_lin, n_clu, n_iter, unary, Q, lg, lb, dev):
    """stego_crf_mean_field; n_clu = 0: one probe, rows of 32 floats (else 64)"""
    L = _lib()
    ld = 64 if n_clu else LD
    vg = torch.full((2, B * lg.M, ld), float("nan"), device=dev)
    vb = torch.full((2, lb.M, ld), float("nan"), device=dev)
    lq = torch.empty(B, n_lin, N, device=dev)
    cq = torch.empty(B, n_clu, N, device=dev) if n_clu else None
    lp = torch.empty(B, N, dtype=torch.uint8, device=dev)
    cp = torch.empty(B, N, dtype=torch.uint8, device=dev) if n_clu else None
    p = L.ptr
    L.check(L.load().stego_crf_mean_field(
        B, N, n_lin, n_clu, n_iter, p(unary), p(Q), p(lg.offset), p(lg.bary), p(lg.rowptr), p(lg.slots), p(lg.n1),
        p(lg.n2), p(lg.norm), lg.M, p(lb.offset), p(lb.bary), p(lb.rowptr), p(lb.slots), p(lb.n1), p(lb.n2),
        p(lb.norm), lb.M, R.POS_W, R.BI_W, p(vg[0]), p(vg[1]), p(vb[0]), p(vb[1]), p(lq), p(cq), p(lp), p(cp), 0, 0, 0,
        0, 0, L.stream()), "stego_crf_mean_field")
    return vg, vb, lq, cq, lp, cp


@pytest.mark.parametrize("name,H,W,kind,C", FILTER, ids=[f[0] for f in FILTER])
def test_filter_one_probe(cuda_dev, name, H, W, kind, C):
    """dense_crf's rows of 32 floats: the normalisation of both of its lattices (stego_crf_norm) and the last two blur
    passes of each left in the scratch of stego_crf_mean_field(n_clu = 0, n_iter = 1)"""
    N = H * W
    _, lg, lb, g64, b64 = _setup(1, H, W, [kind], cuda_dev, seed=N)
    rat = Ratios()
    Q = torch.zeros(N, LD, device=cuda_dev)
    Q[:, :C] = _probs(N, C, H + C, cuda_dev)
    vg, vb, *_ = _call_mf(1, N, C, 0, 1, torch.zeros(N, LD, device=cuda_dev), Q, lg, lb, cuda_dev)
    for lat, l64, v, last, tag in ((lg, g64, vg, 1, "d2"), (lb, b64, vb, 0, "d5")):
        n, nb = R.norm(l64, bars=True)
        rat.add(f"norm_{tag}", (lat.norm.double() - n).abs(), nb["bar"])
        f = R.filter(l64, lat.norm.double()[:, None] * Q[:, :C].double(), bars=True)
        rat.add(f"blurred_{tag}", (v[last, :, :C].double() - f["passes"][-1]).abs(), f["err"][-1])
        rat.add(f"blurred_prev_{tag}", (v[1 - last, :, :C].double() - f["passes"][-2]).abs(), f["err"][-2])
        assert (v[:, :, C:] == 0).all(), tag
        del f
    print(f"{name}: {dict(rat)}")
    rat.check(f"crf_filter_one_probe_{name}")


def _check_q(rat, tag, q, arg, ref, n):
    """q [P, n] against ref (update dict with bars) and the argmax rules"""
    q64 = ref["q"]
    z = ref["t"] - ref["t"].amax(1, keepdim=True)
    bar = R.softmax_bar(q64, z, n, ref["dt"])
    rat.add(f"q_{tag}", (q.double() - q64).abs(), bar)
    top = q64.topk(min(2, n), 1).values
    gap = top[:, 0] - top[:, -1] if n > 1 else torch.full_like(top[:, 0], float("inf"))
    clear = gap > 2 * bar.amax(1)
    assert torch.equal(arg.long()[clear], q64.argmax(1)[clear]), tag
    first = (q == q.amax(1, keepdim=True)).float().argmax(1)         # lowest index holding the maximum
    assert torch.equal(arg.long(), first), tag


EVAL_FILTER = [("320_piecewise_x16", 16, 320, 320, "piecewise", 27, 32), ("320_noise_x2", 2, 320, 320, "noise", 27, 22),
               ("c4", 1, 1024, 2048, "piecewise", 27, 27), ("37x53_x5", 5, 37, 53, None, 3, 2),
               ("1x37_x2", 2, 1, 37, "saturated", 1, 2), ("37x1", 1, 37, 1, "black", 2, 1),
               ("2x2_x3", 3, 2, 2, "constant", 32, 27), ("1x1", 1, 1, 1, "noise", 27, 32)]


@pytest.mark.parametrize("name,B,H,W,kind,n_lin,n_clu", EVAL_FILTER, ids=[e[0] for e in EVAL_FILTER])
def test_filter_and_update_two_probes(cuda_dev, name, B, H, W, kind, n_lin, n_clu):
    """stego_crf_norm's scratch and norm, and stego_crf_mean_field(n_iter=1) with two probes: the last two blur passes
    of both lattices left in val_g / tmp_g / val_b / tmp_b, the updated marginals and the argmax maps"""
    N = H * W
    kinds = [kind] * B if kind else list(R.IMAGES)[:B]
    x, lg, lb, g64, b64 = _setup(B, H, W, kinds, cuda_dev, seed=N)
    rat = Ratios()
    for lat, l64, tag in ((lg, _lat64(lg), "g"), (lb, b64, "b")):
        v, nrm = _call_norm(lat, cuda_dev)
        n, nb = R.norm(l64, bars=True)
        f = nb["filter"]
        last = 1 if lat.d == 2 else 0
        rat.add(f"ones_last_pass_{tag}", (v[last].double() - f["passes"][-1][:, 0]).abs(), f["err"][-1][:, 0])
        rat.add(f"ones_prev_pass_{tag}", (v[1 - last].double() - f["passes"][-2][:, 0]).abs(), f["err"][-2][:, 0])
        rat.add(f"norm_{tag}", (nrm.double() - n).abs(), nb["bar"])
        assert torch.equal(nrm, lat.norm)
    g = torch.Generator().manual_seed(N + n_lin)
    Q = torch.zeros(B * N, 64)
    unary = torch.zeros(B * N, 64)
    for lo, n in ((0, n_lin), (32, n_clu)):
        Q[:, lo:lo + n] = torch.softmax(torch.randn(B * N, n, generator=g) * 2, 1)
        unary[:, lo:lo + n] = R.unary_from_logits(torch.randn(B * N, n, generator=g) * 3)[0].float()
    Q, unary = Q.to(cuda_dev), unary.to(cuda_dev)
    vg, vb, lq, cq, lp, cp = _call_mf(B, N, n_lin, n_clu, 1, unary, Q.clone(), lg, lb, cuda_dev)
    ng, nbn = lg.norm.double().repeat(B), lb.norm.double()
    # position values [B][Mg][64] of the B frames = one lattice over B*N pixels; passes 2 and 3 / 5 and 6 remain
    on = torch.zeros(64, dtype=torch.bool, device=cuda_dev)
    on[:n_lin] = True
    on[32:32 + n_clu] = True
    fg = R.filter(g64, ng[:, None] * Q[:, on].double(), bars=True)
    fb = R.filter(b64, nbn[:, None] * Q[:, on].double(), bars=True)
    for got, f, k, tag in ((vg[1], fg, -1, "g3"), (vg[0], fg, -2, "g2"), (vb[0], fb, -1, "b6"), (vb[1], fb, -2, "b5")):
        rat.add(f"blurred_{tag}", (got[:, on].double() - f["passes"][k]).abs(), f["err"][k])
        assert (got[:, ~on] == 0).all(), tag
    del fg, fb
    for lo, n, q, arg, tag in ((0, n_lin, lq, lp, "lin"), (32, n_clu, cq, cp, "clu")):
        ref = R.update(unary[:, lo:lo + n], Q[:, lo:lo + n], g64, b64, ng, nbn, bars=True)
        _check_q(rat, tag, q.permute(0, 2, 1).reshape(B * N, n), arg.reshape(-1), ref, n)
    print(f"{name}: M_g {lg.M}, M_b {lb.M}; {dict(rat)}")
    rat.check(f"crf_gather_{name}")


# ================================================================================================
# 4. one update from the fp64 chain's own Q_k, both kernels; the unaries
# ================================================================================================
UPDATE = [("c4_27", 1024, 2048, "piecewise", 27, "random"), ("37x53_1", 37, 53, "piecewise", 1, "random"),
          ("37x53_2", 37, 53, "noise", 2, "straddle"), ("37x53_3", 37, 53, "black", 3, "onehot"),
          ("37x53_27", 37, 53, "saturated", 27, "straddle"), ("37x53_32", 37, 53, "constant", 32, "random"),
          ("1x37_27", 1, 37, "noise", 27, "onehot"), ("37x1_32", 37, 1, "noise", 32, "random"),
          ("2x2_27", 2, 2, "noise", 27, "random"), ("1x1_3", 1, 1, "noise", 3, "random"),
          ("uniform_27", 37, 53, "piecewise", 27, "uniform"), ("uniform_32", 2, 2, "noise", 32, "uniform")]


def _unary_bar(U32, logits, n):
    Uref, p = R.unary_from_logits(logits)
    zz = logits.double() - logits.double().amax(1, keepdim=True)
    bound = 2 * ((2 + zz.abs()) * 2.0 ** -23 + U * zz.abs() + (n + 4) * U + 3 * 2.0 ** -19)
    return (U32.double() - Uref).abs(), bound


def _q0_bar(Q32, U32, n):
    t = -U32.double()
    z = t - t.amax(1, keepdim=True)
    q = torch.softmax(t, 1)
    return (Q32.double() - q).abs(), R.softmax_bar(q, z, n, U * z.abs())


@pytest.mark.parametrize("name,H,W,kind,C,unary", UPDATE, ids=[u[0] for u in UPDATE])
def test_update_one_and_two_probes_from_fp64_chain(cuda_dev, name, H, W, kind, C, unary):
    """crf_unary_kernel and Q_0, then for k = 0..9: Q_k of the fp64 chain rounded to fp32 through one iteration of
    stego_crf_mean_field(n_iter=1) with one probe (dense_crf's rows of 32) and with two carrying the same classes
    (fused_eval_crf's rows of 64); both give the same bits"""
    from stego_b200 import crf
    L = _lib()
    lib = L.load()
    N = H * W
    img = R.image(kind, H, W, seed=N + C).to(cuda_dev)
    z = R.logits(unary, N, C, seed=N + C).to(cuda_dev)
    Ut = torch.empty(N, LD, device=cuda_dev)
    Q0 = torch.empty(N, LD, device=cuda_dev)
    L.check(lib.stego_crf_unary(L.ptr(z.t().contiguous()), L.ptr(Ut), L.ptr(Q0), N, C, L.stream()), "stego_crf_unary")
    rat = Ratios()
    rat.add("unary", *_unary_bar(Ut[:, :C], z, C))
    rat.add("q0", *_q0_bar(Q0[:, :C], Ut[:, :C], C))
    assert (Ut[:, C:] == 0).all() and (Q0[:, C:] == 0).all()
    if unary == "uniform":
        assert (Q0[:, :C] == Q0[:, :1]).all() and (Ut[:, :C] == Ut[:, :1]).all()
    lg = crf._position_lattice(H, W, cuda_dev)
    lb = crf._bilateral_lattice([img])
    g64, b64 = _lat64(lg), _lat64(lb)
    U32 = Ut[:, :C]
    seq = R.mean_field(U32, g64, b64, R.MAX_ITER, record=True)
    eU = torch.zeros(N, 64, device=cuda_dev)
    eU[:, :C] = U32
    eU[:, 32:32 + C] = U32
    for k in range(R.MAX_ITER):
        Qk = torch.zeros(N, LD, device=cuda_dev)
        Qk[:, :C] = seq[k].float()
        _, _, q1, _, a1, _ = _call_mf(1, N, C, 0, 1, Ut, Qk, lg, lb, cuda_dev)
        ref = R.update(U32, seq[k], g64, b64, lg.norm, lb.norm, bars=True)
        _check_q(rat, "one_probe", q1[0].t(), a1[0], ref, C)
        eQ = torch.zeros(N, 64, device=cuda_dev)
        eQ[:, :C] = seq[k].float()
        eQ[:, 32:32 + C] = seq[k].float()
        _, _, lq, cq, lp, cp = _call_mf(1, N, C, C, 1, eU, eQ, lg, lb, cuda_dev)
        assert torch.equal(lq, cq) and torch.equal(lp, cp)
        assert torch.equal(q1, lq) and torch.equal(a1, lp)
        if unary == "uniform":
            assert (q1 == q1[:, :1]).all() and (a1 == 0).all(), k
    print(f"{name}: {dict(rat)}")
    rat.check(f"crf_update_{name}")


@pytest.mark.parametrize("unary", R.UNARIES)
def test_eval_unary_q0(cuda_dev, unary):
    """Q_0 of stego_eval_crf_unary (so far only its row sums were checked), stage-wise from its own unary, with a
    linear probe whose scores are the unary builders' logits (identity weights; a 1 x 1 code per frame, upsampled,
    so every pixel of a frame gets that row)"""
    from stego_b200 import _lib as L
    from stego_b200.eval import _probe_codes, _probe_tables
    from stego_b200.modules import ClusterLookup
    B, C, h, w, H, W, n_lin, n_clu = 8, 32, 1, 1, 8, 8, 27, 32
    g = torch.Generator().manual_seed(len(unary))
    lin = torch.nn.Conv2d(C, n_lin, (1, 1)).to(cuda_dev)
    z = R.logits(unary, B * h * w, n_lin, seed=3)                       # the linear probe's scores per code pixel
    with torch.no_grad():
        lin.weight.zero_()
        lin.bias.zero_()
        lin.weight[:, :, 0, 0] = torch.eye(n_lin, C)
    clu = ClusterLookup(C, n_clu).to(cuda_dev)
    with torch.no_grad():
        clu.clusters.copy_(torch.eye(n_clu, C) if unary == "uniform" else torch.randn(n_clu, C, generator=g))
    code = torch.zeros(B, C, h, w)
    code[:, :n_lin] = z.reshape(B, h, w, n_lin).permute(0, 3, 1, 2)
    if unary == "uniform":
        code[:, n_lin:] = 0.75
    code = code.to(cuda_dev)
    x, xf, ld = _probe_codes(code, None)
    wl, bl, cl = _probe_tables(lin, clu, C)
    scratch = torch.empty(B * h * w, 80, device=cuda_dev)
    unary_t = torch.empty(B * H * W, 64, device=cuda_dev)
    Q = torch.empty(B * H * W, 64, device=cuda_dev)
    L.check(L.load().stego_eval_crf_unary(L.ptr(x), L.ptr(xf), ld, C, B, h, w, H, W, L.ptr(wl), L.ptr(bl), n_lin,
                                          L.ptr(cl), n_clu, 2.0, L.ptr(scratch), L.ptr(unary_t), L.ptr(Q), L.stream()),
              "stego_eval_crf_unary")
    rat = Ratios()
    for lo, n in ((0, n_lin), (32, n_clu)):
        rat.add(f"q0_{lo}", *_q0_bar(Q[:, lo:lo + n], unary_t[:, lo:lo + n], n))
        if unary == "uniform":
            assert (Q[:, lo:lo + n] == Q[:, lo:lo + 1]).all()
    if unary == "onehot":
        # every off-winner probability of the linear probe sits at the clip: U = -log 1e-5 to the unary bound
        off = unary_t[:, :n_lin] > 5
        assert (off.sum(1) == n_lin - 1).all()
    print(f"eval unary {unary}: {dict(rat)}")
    rat.check(f"crf_eval_q0_{unary}")


# ================================================================================================
# 5. ten iterations
# ================================================================================================
def _chain_check(what, got, want):
    err = (got.double() - want).abs().max().item()
    top = want.topk(min(2, want.shape[1]), 1).values
    gap = top[:, 0] - top[:, -1] if want.shape[1] > 1 else torch.full_like(top[:, 0], float("inf"))
    clear = gap > 2 * err
    differ = got.argmax(1) != want.argmax(1)
    print(f"{what}: max |dQ| {err:.2e}, labels differing {int(differ.sum())} of {differ.numel()}")
    assert err < 2e-3, (what, err)
    assert not (differ & clear).any(), what
    return err


CHAIN = [("c4", 1, 1024, 2048, "piecewise", 27, 27), ("320_x16", 16, 320, 320, "piecewise", 27, 32),
         ("320_noise_x2", 2, 320, 320, "noise", 27, 27), ("37x53_saturated", 1, 37, 53, "saturated", 3, 2),
         ("37x53_black", 2, 37, 53, "black", 2, 3), ("37x53_constant", 1, 37, 53, "constant", 32, 32),
         ("1x37", 1, 1, 37, "noise", 27, 1), ("37x1", 1, 37, 1, "noise", 1, 27), ("2x2", 1, 2, 2, "noise", 27, 32),
         ("1x1", 1, 1, 1, "noise", 27, 3)]


@pytest.mark.parametrize("name,B,H,W,kind,n_lin,n_clu", CHAIN, ids=[c[0] for c in CHAIN])
def test_mean_field_chain(cuda_dev, name, B, H, W, kind, n_lin, n_clu):
    """crf.mean_field (dense_crf's ten iterations) per frame and fused_eval_crf for the batch against the fp64 chain
    on the same lattices (fp64 normalisation, fp64 unaries from the logits / from the probe table's unary)"""
    from stego_b200 import crf, eval as ev
    N = H * W
    kinds = [kind] * B
    imgs = torch.stack([R.image(k, H, W, seed=N + 7 * b) for b, k in enumerate(kinds)])
    rat = {}
    # dense_crf: one frame at a time, class scores given at full resolution
    lg = crf._position_lattice(H, W, cuda_dev)
    g64 = _lat64(lg)
    for b in range(min(B, 2)):
        img = imgs[b].to(cuda_dev)
        z = R.logits("random", N, n_lin, seed=N + b).to(cuda_dev)
        q, arg = crf.mean_field(z.t().reshape(n_lin, H, W).contiguous(), img, R.MAX_ITER, want_argmax=True)
        lb = crf._lattice_points(H, W, 5, R.BI_XY_STD, R.BI_RGB_STD, img, cuda_dev)
        want = R.mean_field(R.unary_from_logits(z)[0], g64, _lat64(lb))
        got = q.reshape(n_lin, N).t()
        rat["dense_crf"] = max(rat.get("dense_crf", 0.0), _chain_check(f"{name} dense_crf frame {b}", got, want))
        assert torch.equal(arg.reshape(-1).long(), got.argmax(1))
        del q, want, got, lb
    # fused_eval_crf: the batch in one call, from a low-resolution code
    from stego_b200.modules import ClusterLookup
    g = torch.Generator().manual_seed(N)
    C, h, w = 24, max(1, H // 8), max(1, W // 8)
    lin = torch.nn.Conv2d(C, n_lin, (1, 1))
    with torch.no_grad():
        lin.weight.copy_(torch.randn(n_lin, C, 1, 1, generator=g))
    clu = ClusterLookup(C, n_clu)
    with torch.no_grad():
        clu.clusters.copy_(torch.randn(n_clu, C, generator=g))
    lin, clu = lin.to(cuda_dev), clu.to(cuda_dev)
    code = torch.randn(B, C, h, w, generator=g).to(cuda_dev)
    x = R.normalised(imgs).to(cuda_dev)
    lp, cp, lq, cq = ev.fused_eval_crf(code, lin, clu, x, want_marginals=True)
    xc, xf, ld = ev._probe_codes(code, None)
    wl, bl, cl = ev._probe_tables(lin, clu, C)
    L = _lib()
    scratch = torch.empty(B * h * w, 80, device=cuda_dev)
    unary = torch.empty(B * N, 64, device=cuda_dev)
    Q = torch.empty(B * N, 64, device=cuda_dev)
    L.check(L.load().stego_eval_crf_unary(L.ptr(xc), L.ptr(xf), ld, C, B, h, w, H, W, L.ptr(wl), L.ptr(bl), n_lin,
                                          L.ptr(cl), n_clu, 2.0, L.ptr(scratch), L.ptr(unary), L.ptr(Q), L.stream()),
              "stego_eval_crf_unary")
    _, elg, elb, eg64, eb64 = _setup(B, H, W, kinds, cuda_dev, seed=N)
    for lo, n, q, p, tag in ((0, n_lin, lq, lp, "lin"), (32, n_clu, cq, cp, "clu")):
        want = R.mean_field(unary[:, lo:lo + n], eg64, eb64)
        got = q.permute(0, 2, 3, 1).reshape(B * N, n)
        rat[f"fused_{tag}"] = _chain_check(f"{name} fused {tag}", got, want)
        assert torch.equal(p.reshape(-1).long(), got.argmax(1))
        del want, got
    record(f"crf_chain_{name}", rat)
