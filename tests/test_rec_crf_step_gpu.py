"""GPU: the reconstruction and CRF terms on the hand-scheduled step (cfg.fused_rec_crf), kernels and step.

Bars (u = 2^-24, gamma_k = k u / (1 - k u); no fast-math, so sqrtf and '/' are correctly rounded).

rec (csrc/rec_loss.cu) against tests/_rec_crf_fp64.py::rec_term on the kernel's own fp32 inputs:
  r_e = b_e + sum_d W_ed c_d is a D-FMA chain and one add: |dr_e| <= gamma_{D+1} rabs_e, rabs = |W| |c| + |b|.
  f = fl(feat m3) is one rounding, u |f|.  The three row sums are chains of at most E / 64 + 7 terms (the thread's
  chunks, five shuffle levels, the two halves); gamma_E bounds them.  With rr = ||dr|| ia (the relative size of the
  decoder's error), eN = gamma_{E+4} (norm, square root, clamp, reciprocal):
    cos: |dcos| <= 2 rr + gamma_{E+8} (sum |r f| ia ib + 2 |cos|) + 2u
    |r|: rr |r| + gamma_{E+2} |r|,   |f|: gamma_{E+3} |f|
    dr_e = g ia (fh_e - k rh_e): |d dr_e| <= |g| ia [(|fh_e| + |rh_e|)(2 eN + 2 rr + gamma_8) + |dr_e^r| ia + |rh_e| |dcos|]
      with |dr_e^r| the decoder error of element e (the first-order terms of every factor; the second-order ones are
      below 2^-40 relative here)
    dcode_d = sum_e dr_e W_ed, a chain of 64 FMAs per chunk plus E / 64 adds: sum_e bar(dr_e) |W_ed| + gamma_E sum |dr W|
    dW_ed / db_e sum over all M rows (per-CTA chains, then a G-term fixed-order sum): sum_rows bar(dr_e) |c_d| +
      gamma_M sum_rows |dr_e c_d| (and the same without c for db).
  Two runs give bit-equal dW / db (no atomics).

crf (the stego_crf_mean_* entry points of csrc/crf_loss.cu):
  * the resized code and image at the samples are bit-equal to torch CUDA's F.interpolate read at those points;
  * sel = raw / max(|raw|, eps) against fp64 on the kernel's raw: the sum of squares is a ceil(C / 32) + 5 chain, eS;
    eN = eS / 2 + eS^2 + gamma_2; |d sel_k| <= |sel_k| (eN + u);
  * loss against fp64 on the kernel's own sel / gsel (scattered to their 56 x 56 positions; repeated samples carry equal
    values) with test_loss_terms_fp64_gpu.crf_bars per output, averaged (the fp64 tile sums add < 2^-40 relative), plus
    u |loss| for the final rounding; and end to end against the fp64 restatement from the code, where every sample's
    normalised vector also moves by delta_a <= 2 vbar_a / |v_a| + eN with vbar_a = (gamma_6 + 16 u max(h, w)) sqrt(C)
    max|code| (per channel four fp32 products and three sums, and ATen's fp32 lambdas, whose source position carries
    <= 4 u in_size): the Gram entry by <= delta_a + delta_b, the loss by mean_ab |s_ab| (delta_a + delta_b);
  * dcode against fp64 through the same chain from the kernel's raw: test_loss_terms_fp64_gpu.crf_bwd_bar gives the
    bar of d sel for the uniform upstream gradient; F.normalize's backward dv = (dsel - k sel <sel, dsel>) / den carries
    (|d dsel| + |d sel| sum|sel dsel| + |sel| |d dot|) / den plus (eN + gamma_3) of its own terms, with
    |d dot| <= sum (|d sel| |dsel| + |sel| |d dsel|) + eS sum |sel dsel|.  The tap weights are fp32 products a' b'
    of fp32 lambdas, each off by an ABSOLUTE d = 4 u in_size + 2 u from the fp64 a, b in [0, 1]; so
    |a' b' - a b| <= d (a + b) + d^2 + u <= 2 d + d^2 + u, however small a b is.  And where the fp64 source position
    lies within d of an integer, the fp32 one may fall on its other side: the kernel then taps the next pixel out
    (i0 - 1 or i1 + 1) with a weight <= d.  So the weight error is bounded over the 4 x 4 box [y0 - 1, y0 + 2] x
    [x0 - 1, x0 + 2] of every sample (clipped to the map), each pixel of it by (2 d + d^2 + u)(|dv| + |d dv|), and a
    pixel gets at most r atomics, r the samples whose box holds it: gamma_r of its |contributions| and 2^-125 per
    atomic (crf_dcode_bar).  With a non-dyadic scale (40 / 56, 60 / 56) a weight of a few 1e-7 lands on a pixel whose
    fp64 weight is 0: a bar relative to a b does not hold there (a 60 x 84 code, 64 samples, 80 channels, went to 1.4
    times such a bar).
  * the fused step's peak memory over a step stays below B n^2 4 bytes (no [B, n, n] tensor).

Kernel edges: rec with m3 = None (the step with dropout off) at E = 384 / 768, D = 1 / 70 / 96, bit-equal to an
all-ones m3; rec at the non-square frames' hw = 28 x 40 and 14 x 20 with M = B hw, B = 1 / 3; CRF codes of 28 x 40,
40 x 28, 14 x 20 and 60 x 84 (a downsampling resize), C = 1 / 15 / 16 / 27 / 70 / 80 in NCHW and channels-last strides
(both of ATen's bilinear kernels), guidance 224 x 320 or its transpose, n = 1 / 64 / 65 / 1000.  The same terms inside
the replayed step, stage by stage across the step's configurations: tests/test_step_rec_crf_fp64_gpu.py.

Step (switch on) against an autograd twin (switch off, no TF32) from the same generator states, at ViT-S/8 224² and
ViT-B/8 320² (B = 32) and at ViT-S/8 224² (B = 8) crossed with the aug seeds, use_salience, use_true_labels, "KK",
feature_samples = 16: both generators end equal; the CRF coordinates are bit-equal to the twin's draw; the positive
correspondence terms, cd means and the cluster loss are bit-equal; loss/rec and loss/crf are within the bars above of
fp64 on the captured tensors; loss/total within the sum of those bars and 8 u of the terms; parameter gradients (the
decoder's included) and one Adam update within test_aug_step_gpu.py's relative bar 3e-3; each term's own contribution
to the head gradients (the step with the term minus the step without it) within 1e-3 between the paths.
"""
import pytest
import torch
import torch.nn.functional as F

import _loss_terms_fp64 as R
import _rec_crf_fp64 as RC
from _parity_util import NAMES, fp32_strict, make_batch, make_model, rel, record
from test_aug_step_gpu import _one_step_each
from test_loss_terms_fp64_gpu import Ratios, crf_bars, crf_bwd_bar

pytestmark = pytest.mark.gpu
U, G = R.U, R.gamma
EPS = R.EPS32
DEC = ["decoder.weight", "decoder.bias"]


@pytest.fixture
def strict_fp32():
    """The autograd twin's decoder conv in fp32, not TF32; the previous settings are restored afterwards."""
    saved = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32, torch.get_float32_matmul_precision())
    fp32_strict()
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved[:2]
    torch.set_float32_matmul_precision(saved[2])


# ================================================================================================
# reconstruction kernels
# ================================================================================================
def _rec_inputs(E, D, M, hw, dev, seed, edge):
    g = torch.Generator().manual_seed(seed)
    P = -(-D // 8) * 8
    code = torch.zeros(M, P)
    code[:, :D] = torch.randn(M, D, generator=g)
    feat = torch.randn(M, E, generator=g).bfloat16()
    nimg = -(-M // hw)
    m3 = (torch.rand(nimg, E, generator=g) > 0.1).float() / 0.9
    m3[0, :7] = 0  # dropped channels
    W = torch.randn(E, D, 1, 1, generator=g) / D ** 0.5
    b = torch.randn(E, generator=g) * 0.1
    if edge:  # r = 0 at row 3 (zero code row, zero bias), f = 0 at row 5
        b.zero_()
        code[3] = 0
        feat[5] = 0
    return [t.to(dev) for t in (code, feat, m3, W, b)]


def _rec_run(code, feat, m3, W, b, hw, dcos):
    from stego_b200 import modules
    M, E, D = feat.shape[0], W.shape[0], W.shape[1]
    dev = code.device
    cosv, nr, nf = (torch.empty(M, device=dev) for _ in range(3))
    modules.rec_forward(code, feat, m3, hw, W, b, cosv, nr, nf)
    dg = torch.full((1,), dcos, device=dev)
    dcode = torch.zeros_like(code)
    dW, db = torch.empty_like(W), torch.empty_like(b)
    scratch = modules.rec_scratch(M, E, D, dev)
    modules.rec_backward(code, feat, m3, hw, W, b, cosv, nr, nf, dg, dcode, scratch, dW, db)
    return cosv, nr, nf, dcode, dW, db


def rec_bars(ref, code, W, M, D, E, dcos):
    rbar = G(D + 1) * ref["rabs"]
    rr = rbar.norm(dim=1) * ref["ia"]
    absrf = (ref["r"] * ref["f"]).abs().sum(1)
    cos_bar = 2 * rr + G(E + 8) * (absrf * ref["ia"] * ref["ib"] + 2 * ref["cos"].abs()) + 2 * U
    eN = G(E + 4)
    fh, rh = ref["fh"].abs(), ref["rh"].abs()
    dr_bar = abs(dcos) * ref["ia"][:, None] * ((fh + rh) * (2 * eN + 2 * rr[:, None] + G(8)) + rbar * ref["ia"][:, None] +
                                               rh * cos_bar[:, None])
    c, Wd, dr = code.double()[:, :D], W.double().view(E, D), ref["dr"]
    return dict(cos=cos_bar, nr=rr * ref["nr"] + G(E + 2) * ref["nr"], nf=G(E + 3) * ref["nf"],
                dcode=dr_bar @ Wd.abs() + G(E) * (dr.abs() @ Wd.abs()),
                dW=dr_bar.t() @ c.abs() + G(M) * (dr.abs().t() @ c.abs()),
                db=dr_bar.sum(0) + G(M) * dr.abs().sum(0))


def _rec_check(code, feat, m3, W, b, hw, tag, edge=False):
    """one forward and backward against rec_term at rec_bars; the decoder gradient repeats bit for bit"""
    M, E, D = feat.shape[0], W.shape[0], W.shape[1]
    dcos = float(torch.tensor(-0.7, dtype=torch.float32) / M)
    out = _rec_run(code, feat, m3, W, b, hw, dcos)
    cosv, nr, nf, dcode, dW, db = out
    again = _rec_run(code, feat, m3, W, b, hw, dcos)
    assert torch.equal(dW, again[4]) and torch.equal(db, again[5]), "decoder gradient not bit-reproducible"
    assert torch.equal(dcode, again[3])
    m3r = m3.repeat_interleave(hw, 0)[:M] if m3 is not None else None
    ref = RC.rec_term(code[:, :D], feat, m3r, W.view(E, D), b, dcos)
    bars = rec_bars(ref, code, W, M, D, E, dcos)
    rat = Ratios()
    rat.add("cos", cosv, ref["cos"], bars["cos"])
    rat.add("nr", nr, ref["nr"], bars["nr"])
    rat.add("nf", nf, ref["nf"], bars["nf"])
    rat.add("dcode", dcode[:, :D], ref["dcode"], bars["dcode"])
    rat.add("dW", dW.view(E, D), ref["dW"], bars["dW"])
    rat.add("db", db, ref["db"], bars["db"])
    assert (dcode[:, D:] == 0).all(), "padding columns written"
    if edge:
        assert nr[3].item() == 0 and nf[5].item() == 0 and cosv[3].item() == 0 and cosv[5].item() == 0
    rat.check(tag)
    return out


@pytest.mark.parametrize("E", [384, 768])
@pytest.mark.parametrize("D", [1, 8, 70, 96])
@pytest.mark.parametrize("edge", [False, True])
def test_rec_kernels_vs_fp64(cuda_dev, E, D, edge):
    """M = 3 x 337 rows (not a multiple of the CTA's 32), m3 with zeros; with edge, a pixel with r = 0 and one with
    f = 0 (the eps clamps)."""
    hw, M = 337, 3 * 337
    code, feat, m3, W, b = _rec_inputs(E, D, M, hw, cuda_dev, seed=E + D + edge, edge=edge)
    _rec_check(code, feat, m3, W, b, hw, f"rec_E{E}_D{D}_{'edge' if edge else 'rand'}", edge)


@pytest.mark.parametrize("E", [384, 768])
@pytest.mark.parametrize("D", [1, 70, 96])
def test_rec_kernels_without_m3(cuda_dev, E, D):
    """m3 = None (the step with dropout off) against rec_term without a mask, and bit-equal to an all-ones m3: f = feat
    * 1.0 is exact in fp32, and nothing else reads m3."""
    hw, M = 337, 3 * 337
    code, feat, m3, W, b = _rec_inputs(E, D, M, hw, cuda_dev, seed=7 * E + D, edge=True)
    none = _rec_check(code, feat, None, W, b, hw, f"rec_nom3_E{E}_D{D}", edge=True)
    ones = _rec_run(code, feat, torch.ones_like(m3), W, b, hw, float(torch.tensor(-0.7, dtype=torch.float32) / M))
    for name, a, o in zip(("cos", "nr", "nf", "dcode", "dW", "db"), none, ones):
        assert torch.equal(a, o), f"m3 = None differs from an all-ones m3 in {name}"


@pytest.mark.parametrize("E,D", [(384, 70), (768, 96)])
@pytest.mark.parametrize("hw", [28 * 40, 14 * 20])
@pytest.mark.parametrize("B", [1, 3])
def test_rec_kernels_nonsquare(cuda_dev, E, D, hw, B):
    """The step's non-square frames (28 x 40 at ViT-S/8 224 x 320, 14 x 20 at patch 16): M = B hw rows, a per-image m3
    switching at every multiple of hw (280 is not a multiple of the CTA's 32 rows)."""
    M = B * hw
    code, feat, m3, W, b = _rec_inputs(E, D, M, hw, cuda_dev, seed=hw + B + D, edge=False)
    _rec_check(code, feat, m3, W, b, hw, f"rec_E{E}_D{D}_hw{hw}_B{B}")


# ================================================================================================
# CRF kernels
# ================================================================================================
def _crf_coords(n, gen):
    c = R.random_coords(n, 56, 56, gen)
    special = torch.tensor([[0, 0, 55, 55, 0, 27, 55, 13], [0, 55, 0, 55, 30, 0, 20, 55]])  # corners, then edges
    k = min(n, special.shape[1])
    c[:, :k] = special[:, :k]
    if n >= 12:
        c[:, 8:12] = c[:, 4:8]  # repeats
    return c


def _crf_run(img, code, coords, p32, weight):
    from stego_b200 import modules
    B, C = code.shape[:2]
    n = coords.shape[1]
    NP = -(-n // 64) * 64
    dev = code.device
    gsel = torch.empty(B, NP, 4, device=dev)
    pos = torch.empty(NP, 2, dtype=torch.int32, device=dev)
    raw, sel, dsel = (torch.empty(B, C, NP, device=dev) for _ in range(3))
    nrm = torch.empty(B, NP, device=dev)
    tiles = torch.empty(B, NP // 64, NP // 64, dtype=torch.float64, device=dev)
    loss, total = torch.empty(1, device=dev), torch.zeros(1, device=dev)
    g = torch.full((1,), float(weight), device=dev).div_(B * n * n)
    dcode = torch.zeros_like(code)
    modules.crf_guidance(img, coords, gsel, pos)
    modules.crf_forward(code, coords, p32, gsel, pos, raw, sel, nrm, tiles)
    modules.crf_loss(tiles, n, weight, loss, total)
    modules.crf_backward(g, sel, nrm, gsel, pos, coords, p32, dsel, dcode)
    return dict(gsel=gsel[:, :n, :3], raw=raw[:, :, :n], sel=sel[:, :, :n], nrm=nrm[:, :n], loss=loss, total=total,
                g=g, dcode=dcode, pos=pos[:n])


def _on_map(v, coords, S=56):
    """[B, C, n] values at coords -> a [B, C, S, S] map holding them (repeated samples carry equal values)"""
    B, C, _ = v.shape
    m = torch.zeros(B, C, S * S, dtype=v.dtype, device=v.device)
    m[:, :, coords[0] * S + coords[1]] = v
    return m.view(B, C, S, S)


def crf_loss_bars(run, coords, p32, C, code, h, w):
    """(bar of the kernel's loss against fp64 on its own sel / gsel, that fp64 loss, extra end-to-end bar)"""
    sel64 = run["sel"].double()
    ref = R.crf_loss(_on_map(run["gsel"].permute(0, 2, 1).double(), coords), _on_map(sel64, coords), coords, *p32)
    fbar, ds = crf_bars(ref, C, p32)
    loss64 = ref["out"].mean()
    bar = fbar.mean() + U * loss64.abs() + 1e-12 * ref["out"].abs().mean()
    eS = G(-(-C // 32) + 5)
    eN = eS / 2 + eS ** 2 + G(2)
    vmax = code.detach().abs().amax(dim=(1, 2, 3)).double()  # per image
    vbar = (G(6) + 16 * U * max(h, w)) * vmax[:, None] * C ** 0.5
    delta = 2 * vbar / run["nrm"].double().clamp_min(1e-30) + eN  # [B, n]
    e2e = (ref["s"].abs() * (delta[:, :, None] + delta[:, None, :])).mean()
    return bar, loss64, e2e, ref, ds


def _taps64(coords, h, w):
    y0, y1, ly = RC.resize_taps(coords[0], h, 56)
    x0, x1, lx = RC.resize_taps(coords[1], w, 56)
    return ((y0, x0, (1 - ly) * (1 - lx)), (y0, x1, (1 - ly) * lx), (y1, x0, ly * (1 - lx)), (y1, x1, ly * lx))


def scatter_box(v, coords, h, w):
    """v [B, C, n] added to every pixel of each sample's 4 x 4 box [y0 - 1, y0 + 2] x [x0 - 1, x0 + 2] (clipped to the
    [B, C, h, w] map): the pixels the kernel's fp32 taps can land on"""
    B, C, _ = v.shape
    y0 = RC.resize_taps(coords[0], h, 56)[0]
    x0 = RC.resize_taps(coords[1], w, 56)[0]
    out = torch.zeros(B, C, h * w, dtype=torch.float64, device=v.device)
    for dy in range(-1, 3):
        for dx in range(-1, 3):
            yi, xi = y0 + dy, x0 + dx
            ok = ((yi >= 0) & (yi < h) & (xi >= 0) & (xi < w)).double()
            out.index_add_(2, yi.clamp(0, h - 1) * w + xi.clamp(0, w - 1), v * ok)
    return out.view(B, C, h, w)


def scatter_taps(v, coords, h, w, weights=True):
    """v [B, C, n] scattered into [B, C, h, w] through the bilinear taps (weights=False: count the nonzero taps)"""
    B, C, _ = v.shape
    out = torch.zeros(B, C, h * w, dtype=torch.float64, device=v.device)
    for yi, xi, wt in _taps64(coords, h, w):
        out.index_add_(2, yi * w + xi, v * (wt if weights else (wt != 0).double()))
    return out.view(B, C, h, w)


def crf_dcode_bar(run, ref, ds, coords, code, n, h, w):
    """bar of the kernel's dcode against fp64 through the chain from the kernel's raw (module docstring); ref is
    R.crf_loss on the fp64 normalisation of the kernel's raw"""
    B, C = code.shape[:2]
    gout = torch.full((B, n, n), run["g"].double().item(), dtype=torch.float64, device=code.device)
    bw, _ = crf_bwd_bar(ref, gout, coords, (B, C, 56, 56), ds, n)
    NP = -(-n // 64) * 64
    dsel_bar = G(NP) * (bw["dsel_abs"] + bw["dsel_werr"]) + bw["dsel_werr"]  # crf_bwd_bar's, before its scatter
    dsel, sel = bw["dsel"], ref["sel"]
    eS = G(-(-C // 32) + 5)
    eN = eS / 2 + eS ** 2 + G(2)
    selbar = sel.abs() * (eN + U)
    den = run["nrm"].double().clamp_min(EPS)[:, None]
    dotabs = (sel.abs() * dsel.abs()).sum(1, keepdim=True)
    ddot = (selbar * dsel.abs() + sel.abs() * dsel_bar).sum(1, keepdim=True) + eS * dotabs
    dv = (dsel - sel * (sel * dsel).sum(1, keepdim=True)) / den
    dv_bar = (dsel_bar + selbar * dotabs + sel.abs() * ddot) / den + (eN + G(3)) * (dsel.abs() + sel.abs() * dotabs) / den
    d = 4 * U * max(h, w) + 2 * U  # each fp32 lambda (and 1 - lambda): absolute error
    werr = 2 * d + d * d + U        # |a' b' - a b| for a, b in [0, 1], on every pixel of the sample's box
    wbox = werr * scatter_box(dv.abs() + dv_bar, coords, h, w)
    r = scatter_box(torch.ones_like(dv), coords, h, w)  # atomics per pixel, at most
    gr = r * U / (1 - r * U)
    return (scatter_taps(dv_bar, coords, h, w) + wbox + gr * (scatter_taps(dv.abs() + dv_bar, coords, h, w) + wbox) +
            r * 2 * 2.0 ** -126)


def dcode_from_raw(raw64, run, coords, p32, shape):
    """fp64 d code through normalize and the taps from the kernel's raw samples and guidance, and R.crf_loss's dict"""
    B, C, h, w = shape
    nv = raw64.norm(dim=1)
    sel = raw64 / nv.clamp_min(EPS)[:, None]
    ref = R.crf_loss(_on_map(run["gsel"].permute(0, 2, 1).double(), coords), _on_map(sel, coords), coords, *p32)
    ref["sel"] = sel
    dsel = torch.einsum("zab,zkb->zka", -2 * run["g"].double().item() * ref["s"], sel)
    k = torch.where(nv >= EPS, (sel * dsel).sum(1), torch.zeros_like(nv))
    dv = (dsel - sel * k[:, None]) / nv.clamp_min(EPS)[:, None]
    ref["dv"] = dv
    return scatter_taps(dv, coords, h, w), ref


def _crf_check(img, code, coords, tag):
    """the CRF kernels on one code map (any strides) and guidance image: the resized samples bit-equal to torch CUDA's
    F.interpolate read at them; sel, the norms, the loss and d(code) at crf_bars / crf_dcode_bar"""
    B, C, h, w = code.shape
    n = coords.shape[1]
    p32 = R.fp32_params(R.PARAMS)
    wt = 0.5
    run = _crf_run(img, code, coords, p32, wt)
    # the resized samples are torch's, bit for bit
    rs = lambda t: F.interpolate(t, 56, mode="bilinear", align_corners=False)
    ys, xs = coords[0], coords[1]
    assert torch.equal(run["raw"], rs(code)[:, :, ys, xs]), "resized code differs from F.interpolate"
    assert torch.equal(run["gsel"], rs(img)[:, :, ys, xs].permute(0, 2, 1)), "resized image differs from F.interpolate"
    assert torch.equal(run["pos"].long(), coords.t())
    rat = Ratios()
    raw64 = run["raw"].double()
    nv = raw64.norm(dim=1)
    sel64 = raw64 / nv.clamp_min(EPS)[:, None]
    eS = G(-(-C // 32) + 5)
    eN = eS / 2 + eS ** 2 + G(2)
    rat.add("sel", run["sel"], sel64, sel64.abs() * (eN + U) + 2.0 ** -149)
    rat.add("nrm", run["nrm"], nv, nv * eS)
    bar, loss64, e2e, ref, ds = crf_loss_bars(run, coords, p32, C, code, h, w)
    rat.add("loss", run["loss"], loss64, bar)
    rat.add("total", run["total"], wt * loss64, wt * bar + U * abs(wt) * loss64.abs() + 2 * U * abs(wt * loss64))
    full = RC.crf_term(img, code, coords, p32, wt)
    rat.add("loss_e2e", run["loss"], full["loss"], bar + e2e)
    # dcode through the chain from the kernel's own raw
    want, ref_raw = dcode_from_raw(raw64, run, coords, p32, code.shape)
    _, ds_raw = crf_bars(ref_raw, C, p32)
    rat.add("dcode", run["dcode"], want, crf_dcode_bar(run, ref_raw, ds_raw, coords, code, n, h, w))
    rat.check(tag)
    return run


def _crf_image(B, H, W, gen, dev):
    return ((torch.rand(B, 3, H, W, generator=gen) - torch.tensor(R.MEAN).view(1, 3, 1, 1)) /
            torch.tensor(R.STD).view(1, 3, 1, 1)).to(dev)


def _crf_code(B, C, h, w, layout, gen, dev):
    """[B, C, h, w]: "channels_last" is the step's layout (channels innermost, rows padded by two channels), "nchw"
    contiguous"""
    if layout == "channels_last":
        return torch.randn(B, h, w, C + 2, generator=gen).to(dev)[..., :C].permute(0, 3, 1, 2)
    return torch.randn(B, C, h, w, generator=gen).to(dev)


@pytest.mark.parametrize("h,S", [(28, 224), (40, 320), (56, 448)])
@pytest.mark.parametrize("n", [1, 63, 64, 65, 1000, 2000])
@pytest.mark.parametrize("C", [1, 70, 80])
def test_crf_kernels_vs_torch_and_fp64(cuda_dev, h, S, n, C):
    gen = torch.Generator().manual_seed(h * 7 + n + C)
    B = 2
    img = _crf_image(B, S, S, gen, cuda_dev)
    code = _crf_code(B, C, h, h, "channels_last", gen, cuda_dev)
    coords = _crf_coords(n, gen).to(cuda_dev)
    _crf_check(img, code, coords, f"crf_h{h}_n{n}_C{C}")
    if n == 1000:  # an NCHW-contiguous code: ATen's other kernel (the same for fewer than 16 channels)
        flat = code.contiguous()
        rs = lambda t: F.interpolate(t, 56, mode="bilinear", align_corners=False)
        run = _crf_run(img, flat, coords, R.fp32_params(R.PARAMS), 0.5)
        assert torch.equal(run["raw"], rs(flat)[:, :, coords[0], coords[1]])


@pytest.mark.parametrize("h,w", [(28, 40), (40, 28), (14, 20), (60, 84)])
@pytest.mark.parametrize("C", [1, 15, 16, 27, 70, 80])
@pytest.mark.parametrize("layout", ["nchw", "channels_last"])
@pytest.mark.parametrize("n", [1, 64, 65, 1000])
def test_crf_kernels_nonsquare(cuda_dev, h, w, C, layout, n):
    """Non-square code maps (28 x 40 and its transpose: ViT-S/8 at 224 x 320 and 320 x 224; 14 x 20: patch 16) and one
    with both sides above 56, which the resize to 56 x 56 downsamples; the guidance image 224 x 320 or its transpose,
    as the code.  Channel counts on both sides of ATen's channels-last switch at 16, each in both layouts, so both
    restatements of ATen's bilinear kernel run; 1, 64 and 65 samples (one, a full and a second 64-sample tile) and the
    default 1000."""
    gen = torch.Generator().manual_seed(h * 1000 + w * 10 + C + n)
    B = 2
    H, W = (224, 320) if w > h else (320, 224)
    img = _crf_image(B, H, W, gen, cuda_dev)
    code = _crf_code(B, C, h, w, layout, gen, cuda_dev)
    coords = _crf_coords(n, gen).to(cuda_dev)
    _crf_check(img, code, coords, f"crf_{h}x{w}_n{n}_C{C}_{layout}")


# ================================================================================================
# the step
# ================================================================================================
TERMS = dict(rec_weight=0.7, crf_weight=0.5)


def _batch(B, res, dev, variant, seed=1):
    b = make_batch(B, res, dev, seed=seed)
    if variant == "aug":
        b["seed"] = [1000 * seed + i for i in range(B)]
    if variant == "salience":
        g = torch.Generator().manual_seed(5)
        b["mask"] = (torch.rand(B, 1, res, res, generator=g) > 0.6).float().to(dev)
        b["mask_pos"] = (torch.rand(B, 1, res, res, generator=g) > 0.3).float().to(dev)
    if variant == "true_labels":
        b["label_pos"] = b["label"].roll(1, 0)
    return b


def _over(variant, res, terms=TERMS):
    over = dict(terms, res=res)
    over.update(dict(aug=dict(aug_alignment_weight=0.6), salience=dict(use_salience=True),
                     true_labels=dict(use_true_labels=True), KK=dict(dino_feat_type="KK"),
                     fs16=dict(feature_samples=16)).get(variant, {}))
    return over


class _Spy:
    """Clones of what the fused step hands the rec / crf stages (eager steps only), and the twin's CRF coordinates."""

    def __init__(self, monkeypatch, twin):
        from stego_b200 import modules
        self.rec, self.crf, self.twin_coords = [], [], []

        def wrap(name, store, keep):
            orig = getattr(modules, name)

            def f(*a, **k):
                store.append([t.clone() if isinstance(t, torch.Tensor) else t for t in keep(a)])
                return orig(*a, **k)
            monkeypatch.setattr(modules, name, f)
        wrap("rec_forward", self.rec, lambda a: a[:6])                  # code, feat, m3, hw, weight, bias
        wrap("crf_forward", self.crf, lambda a: (a[0], a[1]))           # code of img, coords
        draw = twin.crf_loss_fn.draw_coords

        def spy(h, w, device):
            c = draw(h, w, device)
            self.twin_coords.append(c.clone())
            return c
        twin.crf_loss_fn.draw_coords = spy


def _check_step(fused, twin, spy, batch):
    cfg = fused.cfg
    ws = fused._fused.ws
    img = batch["img"]
    B = img.shape[0]
    got, want = fused.logged, twin.logged
    for key in ("loss/pos_intra", "loss/pos_inter", "cd/pos_intra", "cd/pos_inter", "loss/cluster"):
        assert torch.equal(got[key], want[key]), (key, got[key].item(), want[key].item())
    rat = Ratios()
    bars = {}
    if cfg.rec_weight > 0:
        assert ws.rec and ws.rec_scratch is not None and "loss/rec" in got
        code, feat, m3, hw, W, b = spy.rec[0]
        E, D = W.shape[:2]
        m3r = m3.reshape(B, E).repeat_interleave(hw, 0) if m3 is not None else None
        dcos = ws.rec_dcos.item()
        ref = RC.rec_term(code[:, :D], feat, m3r, W.view(E, D), b, dcos)
        cbar = rec_bars(ref, code, W, feat.shape[0], D, E, dcos)["cos"]
        bars["loss/rec"] = cbar.mean() + U * ref["loss"].abs()
        rat.add("loss_rec", got["loss/rec"], ref["loss"], bars["loss/rec"])
    if cfg.crf_weight > 0:
        assert ws.crf and ws.crf_tiles is not None and "loss/crf" in got
        code, coords = spy.crf[0]
        assert torch.equal(coords, spy.twin_coords[0]), "CRF coordinates differ from the autograd draw"
        n = coords.shape[1]
        run = dict(sel=ws.crf_sel[:, :, :n], gsel=ws.crf_gsel[:, :n, :3], nrm=ws.crf_nrm[:, :n])
        p32 = R.fp32_params(R.PARAMS)
        C, h, w = code.shape[1:]
        bar, _, e2e, _, _ = crf_loss_bars(run, coords, p32, C, code, h, w)
        full = RC.crf_term(img, code, coords, p32, cfg.crf_weight)
        bars["loss/crf"] = bar + e2e
        rat.add("loss_crf", got["loss/crf"], full["loss"], bars["loss/crf"])
    rat.check(f"step_{'_'.join(k for k in ('rec', 'crf') if getattr(cfg, k + '_weight') > 0)}_B{B}_{img.shape[-1]}")
    lin_f, lin_t = got["loss/linear"].item(), want["loss/linear"].item()
    assert abs(lin_f - lin_t) <= 1e-6 * abs(lin_t), (lin_f, lin_t)
    w_of = {"loss/rec": cfg.rec_weight, "loss/crf": cfg.crf_weight, "loss/aug_alignment": cfg.aug_alignment_weight}
    opt = [k for k in w_of if k in got]
    terms = [got[k].item() for k in ("loss/pos_intra", "loss/pos_inter", "loss/neg_inter", "loss/linear", "loss/cluster")]
    bar = (abs(lin_f - lin_t) + sum(abs(w_of[k]) * abs(got[k].item() - want[k].item()) for k in opt) +
           8 * U * (sum(abs(t) for t in terms) + sum(abs(w_of[k] * got[k].item()) for k in opt)))
    assert abs(got["loss/total"].item() - want["loss/total"].item()) <= bar


def _params(model, names):
    model.flush()
    sd = dict(model.named_parameters())
    return {k: sd[k].detach().clone() for k in names}


def _grads(model, names):
    model.flush()
    sd = dict(model.named_parameters())
    return {k: sd[k].grad.detach().clone() for k in names}


ROWS = [("vit_small", 224, 32, "plain"), ("vit_base", 320, 32, "plain"), ("vit_small", 224, 8, "aug"),
        ("vit_small", 224, 8, "salience"), ("vit_small", 224, 8, "true_labels"), ("vit_small", 224, 8, "KK"),
        ("vit_small", 224, 8, "fs16")]


@pytest.mark.parametrize("arch,res,B,variant", ROWS)
def test_step_fused_vs_autograd(cuda_dev, strict_fp32, monkeypatch, arch, res, B, variant):
    over = _over(variant, res)
    fused, _ = make_model(arch, cuda_dev, fused=True, fused_rec_crf=True, **over)
    twin, _ = make_model(arch, cuda_dev, fused=False, **over)
    names = NAMES + DEC
    p0 = _params(fused, names)
    assert all(torch.equal(p0[k], v) for k, v in _params(twin, names).items())
    spy = _Spy(monkeypatch, twin)
    batch = _batch(B, res, cuda_dev, variant)
    _one_step_each(fused, twin, batch, cuda_dev)
    assert fused._fused.ws.aug == (variant == "aug")
    _check_step(fused, twin, spy, batch)
    g_f, g_t = _grads(fused, names), _grads(twin, names)
    for k in names:
        assert rel(g_f[k], g_t[k]) < 3e-3, (k, rel(g_f[k], g_t[k]))
    # one Adam update: each element moves by at most ~lr on the first step; the moves agree where the gradients do
    p_f, p_t = _params(fused, names), _params(twin, names)
    for k in names:
        d_f, d_t = p_f[k] - p0[k], p_t[k] - p0[k]
        lr = 5e-4 if not k.startswith(("linear_probe", "cluster_probe")) else 5e-3
        assert (d_f - d_t).abs().max().item() <= 2.0 * lr, k
        assert rel(d_f, d_t) < 5e-2, (k, rel(d_f, d_t))


@pytest.mark.parametrize("term", ["rec_weight", "crf_weight"])
def test_term_gradient_wiring(cuda_dev, strict_fp32, term):
    """Each term's own contribution to the head gradients (the step with it minus the step without it) agrees between
    the paths; the draws before the CRF coordinates are the same with and without the term."""
    arch, res, B = "vit_small", 224, 8
    batch = _batch(B, res, cuda_dev, "plain", seed=4)
    diffs = {}
    for fused in (True, False):
        g = {}
        for w in (TERMS[term], 0.0):
            m, _ = make_model(arch, cuda_dev, fused=fused, fused_rec_crf=fused, res=res, **{term: w})
            torch.manual_seed(777)
            m.training_step(batch, 0)
            assert (m._fused is not None and m._fused.ws is not None) == fused
            g[w] = _grads(m, NAMES)
            del m
        diffs[fused] = {k: g[TERMS[term]][k] - g[0.0][k] for k in NAMES if k.startswith("net.")}
    for k in diffs[True]:
        d_f, d_t = diffs[True][k], diffs[False][k]
        assert d_t.abs().max().item() > 0, k
        assert rel(d_f, d_t) < 1e-3, (term, k, rel(d_f, d_t))


def test_histogram_step(cuda_dev, strict_fp32):
    from types import SimpleNamespace
    models = []
    for fused in (True, False):
        m, _ = make_model("vit_small", cuda_dev, fused=fused, fused_rec_crf=fused, res=64, hist_freq=1, **TERMS)
        m.logger = SimpleNamespace(experiment=SimpleNamespace(add_histogram_raw=lambda *a, **k: None))
        models.append(m)
    batch = _batch(4, 64, cuda_dev, "plain", seed=3)
    torch.manual_seed(5)
    names = NAMES + DEC
    for s in range(2):  # step 1 logs histograms
        st, st_cpu = torch.cuda.get_rng_state(cuda_dev), torch.get_rng_state()
        models[0].training_step(batch, s)
        after = torch.cuda.get_rng_state(cuda_dev)
        torch.cuda.set_rng_state(st, cuda_dev)
        torch.set_rng_state(st_cpu)
        models[1].training_step(batch, s)
        assert torch.equal(torch.cuda.get_rng_state(cuda_dev), after)
        torch.cuda.synchronize()
        g_f, g_t = _grads(models[0], names), _grads(models[1], names)
        for k in names:
            assert rel(g_f[k], g_t[k]) < 3e-3, (s, k, rel(g_f[k], g_t[k]))
        for key in ("loss/rec", "loss/crf", "loss/cluster"):
            a, b = models[0].logged[key].item(), models[1].logged[key].item()
            assert abs(a - b) <= 1e-4 * abs(b) + 1e-6, (s, key, a, b)
    assert models[0]._fused.ws.hist is not None


def test_graph_capture_and_replay_match_eager(cuda_dev):
    """Three steps with cuda_graph=True (eager, capture, replay) log what three steps with cuda_graph=False log, with
    both terms and the aug seeds."""
    runs = {}
    for use_graph in (True, False):
        m, _ = make_model("vit_small", cuda_dev, fused=True, fused_rec_crf=True, aug_alignment_weight=0.6, res=64,
                          cuda_graph=use_graph, **TERMS)
        torch.manual_seed(9)
        logs = []
        for s, seed in enumerate((1, 2, 1)):
            m.training_step(_batch(4, 64, cuda_dev, "aug", seed=seed), s)
            torch.cuda.synchronize()
            logs.append({k: v.item() for k, v in m.logged.items()})
            ws = m._fused.ws
            assert ws.rec and ws.crf and (ws.graph is not None) == (use_graph and s >= 1), s
        runs[use_graph] = logs
    for s in range(3):
        assert "loss/rec" in runs[True][s] and "loss/crf" in runs[True][s]
        for k, v in runs[False][s].items():
            g = runs[True][s][k]
            if s == 0:
                assert g == v, (s, k, g, v)  # same kernels on the same inputs
            else:
                assert abs(g - v) <= 1e-4 * abs(v) + 1e-6, (s, k, g, v)


def test_no_pairwise_tensor(cuda_dev):
    """A replayed fused step with the CRF term allocates less than one [B, n, n] fp32 tensor."""
    B, n = 32, 1000
    m, _ = make_model("vit_small", cuda_dev, fused=True, fused_rec_crf=True, res=224, crf_samples=n, **TERMS)
    batch = _batch(B, 224, cuda_dev, "plain")
    for s in range(2):
        m.training_step(batch, s)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated(cuda_dev)
    torch.cuda.reset_peak_memory_stats(cuda_dev)
    m.training_step(batch, 2)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated(cuda_dev) - base
    record("rec_crf_peak_delta", dict(bytes=peak, bar=B * n * n * 4))
    assert m._fused.ws.graph is not None and peak < B * n * n * 4, peak


def test_terms_off_switch_changes_nothing(cuda_dev):
    """rec = crf = 0: the switch on and off allocate the same workspace, capture the same launches and log the same."""
    ms = []
    for sw in (False, True):
        m, _ = make_model("vit_small", cuda_dev, fused=True, fused_rec_crf=sw, res=64)
        torch.manual_seed(3)
        for s in range(2):
            m.training_step(make_batch(4, 64, cuda_dev, seed=s + 1), s)
        torch.cuda.synchronize()
        ms.append(m)
    a, b = (m._fused.ws for m in ms)
    assert sorted(vars(a)) == sorted(vars(b)) and not a.rec and not a.crf
    assert a.graph[0].launches == b.graph[0].launches
    for k in ms[0].logged:
        assert torch.equal(ms[0].logged[k], ms[1].logged[k]), k
