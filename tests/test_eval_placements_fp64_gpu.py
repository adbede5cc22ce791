"""The eight evaluation-frame entries (stego_eval_probes and stego_eval_crf_unary, each with and without _mosaic and
_bf16) called directly through stego_b200.eval's launchers, against float64, over one table-driven matrix:

  * code: C = 70 fp32 (eval_prep_kernel), C = 384 / 768 fp32 and bf16 tokens-major (eval_prep_wide_kernel, the bf16
    ones through the _bf16 entries);
  * frames: B = 1, 3, 6 (the preps' row index r % w, (r / w) % h across frames; 7 x 9 and 5 x 11 frames, 63 and 55
    low-res rows, also put frame boundaries inside the wide prep's 64-row blocks), low-res 8 x 8 up to 32 x 64
    upsampled x8, 7 x 9 -> 50 x 61 (the generic probe kernel), and the 1024 x 2048 frame once per code width;
    flip-TTA off and on;
    n_lin / n_clu = 27 / 27 (the four-pixel probe kernel), 5 / 7 and 32 / 32;
  * placement: frame-major, mosaics of 2 x 3, 3 x 2 and 1 x 5 tiles, and a band of tiles starting at tile0 > 0 in a
    larger grid whose row pitch is tiles_per_row * W + 8; CRF rows of both probes (64 floats) or one (32 floats).

Checks per cell: the frame-major log-probabilities, CRF unaries and initial Q elementwise against fp64; argmax maps
equal to the fp64 argmax off near-ties; confusion counts equal to a masked bincount of the kernel's own maps (also
from a mosaic launch with a label); every mosaic output bit-equal to the frame-major output placed by torch indexing,
with the NaN / 0xAB sentinel intact outside the band and in the pitch padding, and the zero tails of the CRF rows; a
bf16 code bit-identical to the fp32 code of its values through every entry.

Bars (u = 2^-24).  For C <= 96 they are test_probes_fp64_gpu.py's (_eval_case) and test_eval_crf_gpu.py's
(test_unary_matches_fp64).  For the wide prep they are derived from its arithmetic:
  * low-res logit / centroid dot: a sequential fp32 FMA chain over the C channels from the bias (wide_tile_dots), so
    its error is at most u sum_i |s_i|, s_i the exact partial sums in channel order (computed here in fp64), which is
    about sqrt(C) times tighter than (C + 1) u sum_c |terms|; plus u sum_c |terms| for the flip-TTA average's rounding
    (bf16 inputs are exact in fp32, so a code without flip is read exactly), and for the centroid dots
    (C / 64 + 8) u sum_c |terms| for the normalised table: the centroid's fp32 sum of squares (C / 32 lane terms and
    five shuffle levels), sqrt, reciprocal and the product with the entry;
  * the Gram entries are fp64 sums of exact products, so the norm's bar is _eval_case's
    (3 u A / |v| + (C + 18) 2^-53 A^2 / (2 |v|^2) + ...), with C = 768 in the fp64 term;
  * interpolation, cosine, log_softmax, unary and Q_0 as for the narrow code.
The flat 1e-4 of test_wide_prep_against_fp64 / test_wide_crf_unaries_fp64 stays where it is the tighter of the two
(large logits); the derived bar applies everywhere else, which is what catches a dropped term or a lost flip half on
small-magnitude pixels.  The largest error / bar ratios go to $STEGO_PARITY_DIR.

The baseline's CRF-refined scene (eval_scene(run_crf=True) on ViT-S/8 and ViT-B/8 models with projection_type None)
is also checked here: bit-equal to eval_step on a 1 x 1 grid, within the fp64 mean field's bars on a 2 x 3 mosaic,
one-probe rows against the two-probe run, map_clusters against the host, bands of tile rows on one device and several
devices against one.  A module fixture records every call of the eight entries; the last test asserts each ran with a
wide code, and the four fp32 ones also with C = 70.
"""
import os
import sys
from types import SimpleNamespace

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
import _crf_fp64 as F64  # noqa: E402
import _probes_fp64 as R  # noqa: E402
from _parity_util import record  # noqa: E402
from test_probes_fp64_gpu import _argmax_check, _lse_bar, _ratio  # noqa: E402

pytestmark = pytest.mark.gpu
U = R.U
ALPHA = 2.0
FLAT = 1e-4  # test_baseline_gpu.py's flat bar on the wide log-probabilities and unaries
NAN = float("nan")

ENTRIES = [f"stego_eval_{op}{m}{b}" for op in ("probes", "crf_unary") for m in ("", "_mosaic") for b in ("", "_bf16")]
CALLS = {}  # entry -> code widths it was called with
CELLS_RUN = set()  # the matrix cells run in this session (the coverage guard needs all of them)


@pytest.fixture(scope="module", autouse=True)
def _record_entry_calls():
    """Wraps the eight entries of the loaded library for this module's tests: each call records its code width."""
    from stego_b200 import _lib
    lib = _lib.load()
    with pytest.MonkeyPatch.context() as mp:
        for name in ENTRIES:
            def shim(*args, _fn=getattr(lib, name), _name=name):
                CALLS.setdefault(_name, set()).add(int(args[3]))
                return _fn(*args)
            mp.setattr(lib, name, shim)
        yield


# ================================================================================================
# 1. the entries against fp64
# ================================================================================================
CODES = {"n70": (70, torch.float32), "w384": (384, torch.float32), "w768": (768, torch.float32),
         "w384bf": (384, torch.bfloat16), "w768bf": (768, torch.bfloat16)}

FRAMES = {
    # name: B, h, w, H, W, flip, n_lin, n_clu
    "b1_8x8_x8_27": (1, 8, 8, 64, 64, False, 27, 27),
    "b3_16x16_x8_flip_5_7": (3, 16, 16, 128, 128, True, 5, 7),
    "b6_8x16_x8_flip_32": (6, 8, 16, 64, 128, True, 32, 32),
    "b6_8x8_x8_5_7": (6, 8, 8, 64, 64, False, 5, 7),
    "b3_7x9_to_50x61_flip_27": (3, 7, 9, 50, 61, True, 27, 27),
    "b6_5x11_x8_flip_27": (6, 5, 11, 40, 88, True, 27, 27),
    "b1_32x64_x8_flip_27": (1, 32, 64, 256, 512, True, 27, 27),
    "c4": (1, 128, 256, 1024, 2048, True, 27, 27),
}

PLACEMENTS = {
    # name: tile0, tile_rows, tiles_per_row, pitch beyond tiles_per_row * W
    "2x3": (0, 2, 3, 0),
    "3x2": (0, 3, 2, 0),
    "1x5": (0, 1, 5, 0),
    "band_3x3_pitch8": (2, 3, 3, 8),
    "band_1x2_pitch8": (1, 1, 2, 8),
}

CELLS = [(code, frames) for frames in FRAMES if frames != "c4" for code in CODES] + \
        [(code, "c4") for code in ("n70", "w384", "w768")]


def _placements(frames, B):
    if frames == "c4":
        return ["band_1x2_pitch8"]
    return [p for p, (t0, r, c, _) in PLACEMENTS.items() if t0 + B <= r * c]


def _inputs(dev, kind, B, h, w, flip, n_lin, n_clu, seed):
    """(code [B, C, h, w], code_flipped or None, linear probe, cluster probe): tokens-major views of one [2, B*h*w, C]
    store in the kind's dtype.  Tokens (0, 0) and (0, w - 1) of every frame and mirror are zero (the cosine's norm clamp
    at the corner pixels, with or without flip-TTA); the linear logits have a spread of about 2.7, so softmax entries
    below the CRF's 1e-5 clip occur."""
    C, dt = CODES[kind]
    g = torch.Generator(device=dev).manual_seed(seed)
    tok = torch.randn(2, B, h, w, C, device=dev, generator=g)
    tok[:, :, 0, 0] = 0.0
    tok[:, :, 0, w - 1] = 0.0
    tok = tok.to(dt)
    code = tok[0].permute(0, 3, 1, 2)
    code_flipped = tok[1].permute(0, 3, 1, 2) if flip else None
    weight = torch.randn(n_lin, C, device=dev, generator=g) * (8.0 / (3.0 * C ** 0.5))
    lin = SimpleNamespace(weight=weight[:, :, None, None], bias=torch.randn(n_lin, device=dev, generator=g) * 0.5)
    clu = SimpleNamespace(clusters=torch.randn(n_clu, C, device=dev, generator=g))
    return code, code_flipped, lin, clu


def _launch_all(codes, tables, H, W, label, placements):
    """Every entry of one code on the same inputs: the frame-major probes (label and counts) and CRF rows, and per
    placement the mosaic probes (label and counts) and CRF rows of both probes, the linear and the cluster probe.
    Outputs start as NaN / 0xAB sentinels."""
    from stego_b200 import ops
    from stego_b200.eval import _EV_LD, _launch_crf_unary, _launch_probes
    x = codes[0]
    B, _, h, w = x.shape
    dev = x.device
    n_lin, n_clu = tables[0].shape[0], tables[2].shape[0]
    scratch = torch.empty(B * h * w, _EV_LD, dtype=torch.float32, device=dev)
    lab = ops.probe_label(label, B, H, W)[0]
    f32 = lambda *s: torch.full(s, NAN, dtype=torch.float32, device=dev)
    u8 = lambda *s: torch.full(s, 0xAB, dtype=torch.uint8, device=dev)
    i64 = lambda *s: torch.zeros(s, dtype=torch.int64, device=dev)
    fm = dict(lin=f32(B, n_lin, H, W), clu=f32(B, n_clu, H, W), la=u8(B, H, W), ca=u8(B, H, W), lc=i64(n_lin, n_lin),
              cc=i64(n_clu, n_lin), unary=f32(B * H * W, 64), Q=f32(B * H * W, 64))
    _launch_probes(codes, tables, H, W, ALPHA, scratch, fm["lin"], fm["clu"], fm["la"], fm["ca"], lab, fm["lc"],
                   fm["cc"])
    _launch_crf_unary(codes, tables, H, W, ALPHA, scratch, fm["unary"], fm["Q"])
    out = {"frame": fm}
    for name in placements:
        tile0, rows, cols, extra = PLACEMENTS[name]
        pitch = cols * W + extra
        mos = (tile0, rows, cols, pitch)
        m = dict(lin=f32(n_lin, rows * H, pitch), clu=f32(n_clu, rows * H, pitch), la=u8(rows * H, pitch),
                 ca=u8(rows * H, pitch), lc=i64(n_lin, n_lin), cc=i64(n_clu, n_lin))
        _launch_probes(codes, tables, H, W, ALPHA, scratch, m["lin"], m["clu"], m["la"], m["ca"], lab, m["lc"], m["cc"],
                       mos)
        for probes, ld in ((3, 64), (1, 32), (2, 32)):
            m[f"unary{probes}"], m[f"Q{probes}"] = f32(rows * H * pitch, ld), f32(rows * H * pitch, ld)
            _launch_crf_unary(codes, tables, H, W, ALPHA, scratch, m[f"unary{probes}"], m[f"Q{probes}"], mos, probes)
        out[name] = m
    return out


def _same_bits(a, b):
    if a.dtype == torch.float32:
        a, b = a.view(torch.int32), b.view(torch.int32)
    return a.shape == b.shape and torch.equal(a, b)


def _check_placement(fm, m, name, B, H, W, tag):
    """The mosaic outputs == the frame-major ones placed by torch, the sentinels everywhere else."""
    tile0, rows, cols, extra = PLACEMENTS[name]
    pitch = cols * W + extra

    def place(t, fill):  # [B, H, W, ...] -> [rows * H, pitch, ...]
        o = torch.full((rows * H, pitch, *t.shape[3:]), fill, dtype=t.dtype, device=t.device)
        for b in range(B):
            r, c = divmod(tile0 + b, cols)
            o[r * H:(r + 1) * H, c * W:(c + 1) * W] = t[b]
        return o

    for k in ("lin", "clu"):
        assert _same_bits(m[k], place(fm[k].permute(0, 2, 3, 1), NAN).permute(2, 0, 1)), (tag, name, k)
    for k in ("la", "ca"):
        assert _same_bits(m[k], place(fm[k], 0xAB)), (tag, name, k)
    for k in ("lc", "cc"):
        assert torch.equal(m[k], fm[k]), (tag, name, k)
    for k in ("unary", "Q"):
        rows_fm = fm[k].view(B, H, W, 64)
        for probes, sl in ((3, slice(0, 64)), (1, slice(0, 32)), (2, slice(32, 64))):
            want = place(rows_fm[..., sl], NAN).reshape(-1, sl.stop - sl.start)
            assert _same_bits(m[f"{k}{probes}"], want), (tag, name, k, probes)


def _wide_lowres_bars(x, wl, bl, ch, flip, chunk=1024):
    """(E_l [n_lin, P], E_dc [n_clu, P]): the wide prep's error bars on the low-res logits and centroid dots of
    x [C, P] (fp64, the flip-averaged code), from the partial sums of its channel-order FMA chains."""
    C, P = x.shape
    E_l = torch.empty(wl.shape[0], P, dtype=torch.float64, device=x.device)
    E_dc = torch.empty(ch.shape[0], P, dtype=torch.float64, device=x.device)
    avg = 1.0 if flip else 0.0  # the flip-TTA average rounds each channel once
    for p0 in range(0, P, chunk):
        xs = x[:, p0:p0 + chunk]
        for E, tab, b0, extra in ((E_l, wl, bl, avg), (E_dc, ch, None, avg + C / 64 + 8)):
            terms = tab[:, :, None] * xs[None]  # [n, C, p], in the kernel's channel order
            s = terms.cumsum(1)
            if b0 is not None:
                s += b0[:, None, None]
            E[:, p0:p0 + chunk] = U * (s.abs().sum(1) + extra * terms.abs().sum(1))
            del terms, s
    return E_l, E_dc


def _q0_bar(Q32, U32, n):
    """Q_0 = softmax(-U) from the kernel's own unary rows (test_crf_fp64_gpu.py's stage-wise bar)"""
    t = -U32.double()
    z = t - t.amax(1, keepdim=True)
    q = torch.softmax(t, 1)
    return (Q32.double() - q).abs(), F64.softmax_bar(q, z, n, U * z.abs())


def _worst(m, key, ratio):
    """m[key] = the larger of m[key] and ratio, NaN if either is (Python's max would drop a NaN ratio)"""
    if m[key] == m[key] and not ratio <= m[key]:
        m[key] = ratio


def _check_fp64(fm, code, code_flipped, tables, label, H, W, wide, tag):
    """The frame-major outputs of one code against fp64; returns the ratios and near-tie counts.  Every element of the
    outputs must have been written: the float outputs start as NaN, the argmax maps as 0xAB."""
    B, C, h, w = code.shape
    wl, bl, cl = (t.double() for t in tables)
    n_lin, n_clu = wl.shape[0], cl.shape[0]
    ch = R.normalize_rows(cl)
    m = dict(lin_logp=0.0, clu_logp=0.0, lin_unary=0.0, clu_unary=0.0, lin_near=0, clu_near=0)
    for k in ("lin", "clu", "unary", "Q"):
        assert bool(torch.isfinite(fm[k]).all()), (tag, k, int((~torch.isfinite(fm[k])).sum()))
    assert int(fm["la"].max()) < n_lin and int(fm["ca"].max()) < n_clu, tag
    assert torch.equal(fm["lc"], R.confusion(fm["la"], label, n_lin, n_lin)), tag
    assert torch.equal(fm["cc"], R.confusion(fm["ca"], label, n_clu, n_lin)), tag
    assert int(fm["lc"].sum()) > 0, tag
    band = max(1, min(H, (1 << 16) // W if wide else (1 << 20) // W))
    scratch = torch.empty(H, W, dtype=torch.long, device=code.device)
    for b in range(B):
        xbar = R.tta_code(code[b:b + 1], None if code_flipped is None else code_flipped[b:b + 1])[0]
        x = xbar.reshape(C, h * w)
        if wide:
            E_l, E_dc = _wide_lowres_bars(x, wl, bl, ch, code_flipped is not None)
        else:
            E_l = (C + 3) * U * (bl.abs()[:, None] + wl.abs() @ x.abs())
            E_dc = (1.5 * C + 8) * U * (ch.abs() @ x.abs())
        xn = x.norm(dim=0, keepdim=True)
        for y0 in range(0, H, band):
            rows = (y0, min(H, y0 + band))
            e = R.eval_band(xbar, wl, bl, cl, ALPHA, H, W, rows)
            cr = e["corners"]
            # linear probe: the interpolated logits
            z = e["z"]
            E_z = cr.interp(E_l) + 8 * U * sum(t.abs() for t in cr.gather(e["l"])) + cr.lam_term(e["l"])
            # cluster probe: alpha * cosine
            vn, cos, A = e["vnorm"], e["cos"], e["wxn"]
            E_dv = cr.interp(E_dc) + 8 * U * sum(t.abs() for t in cr.gather(e["dc"])) + cr.lam_term(e["dc"])
            lam_n = 2 * (cr.ey + cr.ex) * torch.stack(cr.gather(xn)).amax(0)[0]
            eta = 3 * U * A / vn + (C + 18) * 2.0 ** -53 * A ** 2 / (2 * vn ** 2) + lam_n / vn + 4 * U
            eta = torch.where(eta < 0.5, eta, torch.full_like(eta, float("inf")))
            zero = vn == 0
            E_s = ALPHA * (E_dv / vn + cos.abs() * eta) + 2 * U * ALPHA * cos.abs()
            E_s = torch.where(zero[None], torch.zeros_like(E_s), E_s)
            pix = slice(b * H * W + rows[0] * W, b * H * W + rows[1] * W)
            for p, s, ds, logp, n, lo, arg in (("lin", z, E_z, e["lin_logp"], n_lin, 0, fm["la"]),
                                               ("clu", ALPHA * cos, E_s, e["clu_logp"], n_clu, 32, fm["ca"])):
                lse = torch.logsumexp(s, 0)
                bar = ds + ds.amax(0) + _lse_bar(s) + U * (logp.abs() + lse.abs())
                if wide:
                    bar = bar.clamp_max(FLAT)
                got = fm[p][b, :, rows[0]:rows[1]].reshape(n, -1).double()
                _worst(m, f"{p}_logp", _ratio((got - logp).abs(), bar))
                m[f"{p}_near"] += _argmax_check(arg[b, rows[0]:rows[1]].reshape(-1), logp, bar,
                                                scratch[rows[0]:rows[1]], tag)
                # CRF unary -log(clip(softmax(s), 1e-5, 1)) (test_eval_crf_gpu.py's bar)
                zz = s - s.amax(0)
                want = -torch.log(torch.softmax(s, 0).clamp(F64.CLIP, 1.0))
                ubar = 2 * (2 * ds.amax(0) + (2 + zz.abs()) * 2.0 ** -23 + (n + 4) * U + 3 * 2.0 ** -19)
                if wide:
                    ubar = ubar.clamp_max(FLAT)
                got_u = fm["unary"][pix, lo:lo + n].t().double()
                _worst(m, f"{p}_unary", _ratio((got_u - want).abs(), ubar))
            if zero.any():
                assert not fm["ca"][b, rows[0]:rows[1]].reshape(-1)[zero].any(), tag
            del e
    for p, lo, n in (("lin", 0, n_lin), ("clu", 32, n_clu)):
        m[f"{p}_q0"] = _ratio(*_q0_bar(fm["Q"][:, lo:lo + n], fm["unary"][:, lo:lo + n], n))
        assert not fm["unary"][:, lo + n:lo + 32].any() and not fm["Q"][:, lo + n:lo + 32].any(), tag
    m["pixels"] = B * H * W
    return m


@pytest.mark.parametrize("code_kind,frames", CELLS, ids=[f"{c}-{f}" for c, f in CELLS])
def test_entries_against_fp64_and_placed(cuda_dev, code_kind, frames):
    from stego_b200.eval import _eval_codes, _probe_tables
    dev = cuda_dev
    B, h, w, H, W, flip, n_lin, n_clu = FRAMES[frames]
    C, dt = CODES[code_kind]
    tag = f"{code_kind}_{frames}"
    CELLS_RUN.add((code_kind, frames))
    code, code_flipped, lin, clu = _inputs(dev, code_kind, B, h, w, flip, n_lin, n_clu, seed=C + 7 * B + h + W)
    g = torch.Generator(device=dev).manual_seed(17)
    label = torch.randint(-1, n_lin + 2, (B, H, W), device=dev, generator=g)
    codes = _eval_codes(code, code_flipped)
    assert codes[3] == (dt == torch.bfloat16)
    tables = _probe_tables(lin, clu, C)
    places = _placements(frames, B)
    out = _launch_all(codes, tables, H, W, label, places)
    if dt == torch.bfloat16:  # the fp32 code of the same values through the fp32 entries: the same bits everywhere
        f32 = lambda t: None if t is None else t.float()
        codes32 = _eval_codes(f32(code), f32(code_flipped))
        assert not codes32[3]
        again = _launch_all(codes32, tables, H, W, label, places)
        for p in out:
            for k in out[p]:
                assert _same_bits(out[p][k], again[p][k]), (tag, p, k)
        del again
    fm = out["frame"]
    m = _check_fp64(fm, code, code_flipped, tables, label, H, W, C > 96, tag)
    for name in places:
        _check_placement(fm, out[name], name, B, H, W, tag)
    record(f"eval_placements_{tag}", m)
    for k, v in m.items():
        if k.endswith(("_logp", "_unary", "_q0")):
            assert v <= 1.0, (tag, k, m)
    assert m["lin_near"] <= 2e-2 * B * H * W and m["clu_near"] <= 2e-2 * B * H * W, (tag, m)


# ================================================================================================
# 2. the baseline's CRF-refined scene
# ================================================================================================
def _baseline(dev, arch, n, extra=0):
    from test_baseline_gpu import _model
    return _model(dev, arch, n, extra)


def _scene(dev, R_, C_, t, n, smooth=False):
    from test_eval_scene_gpu import _scene as scene
    return scene(dev, R_, C_, t, n, smooth=smooth)


def _stats(model):
    return model.test_linear_metrics.stats.clone(), model.test_cluster_metrics.stats.clone()


def _reset(model):
    model.test_linear_metrics.reset()
    model.test_cluster_metrics.reset()


ARCHS = ["vit_small", "vit_base"]


@pytest.mark.parametrize("arch", ARCHS)
def test_baseline_crf_1x1_bit_equal_to_eval_step(cuda_dev, arch):
    model = _baseline(cuda_dev, arch, 5)
    tiles, label = _scene(cuda_dev, 1, 1, 64, 5)
    got = model.eval_scene(tiles, (1, 1), label=label, run_crf=True, want_probs=True)
    got_stats = _stats(model)
    _reset(model)
    want = model.eval_step(dict(img=tiles, label=label), run_crf=True, want_probs=True)
    for k in ("linear_preds", "cluster_preds", "linear_probs", "cluster_probs"):
        assert torch.equal(got[k], want[k][0]), k
    for a, b in zip(got_stats, _stats(model)):
        assert torch.equal(a, b)
    assert int(got_stats[0].sum()) > 0


@pytest.mark.parametrize("arch", ARCHS)
def test_baseline_crf_mosaic_against_the_fp64_mean_field(cuda_dev, arch):
    """The unary rows of stego_eval_crf_unary_mosaic_bf16 from the scene's own bf16 tokens, through tests/_crf_fp64.py's
    float64 mean field on the mosaic's lattices: eval_scene's marginals within |dQ| < 2e-3 (test_crf_fp64_gpu.py's
    ten-iteration chain) and equal labels wherever the fp64 top-2 gap exceeds twice the largest error."""
    import scene_oracle as SO
    from stego_b200 import crf
    from stego_b200.eval import _EV_LD, _eval_codes, _launch_crf_unary, _probe_tables
    R_, C_, t = 2, 3, 16
    model = _baseline(cuda_dev, arch, 5, extra=2)
    tiles, _ = _scene(cuda_dev, R_, C_, t, 5, smooth=True)
    got = model.eval_scene(tiles, (R_, C_), run_crf=True, want_probs=True)
    net, HH, WW, h = model.net, R_ * t, C_ * t, t // 8
    with model._net_in_eval_mode(), torch.no_grad():
        code = net.eval_code(net.backbone_tokens(tiles, mirror=True), h, h)
    codes = _eval_codes(code[:R_ * C_], code[R_ * C_:])
    assert codes[3], "the baseline's tokens are read in place as bf16"
    tables = _probe_tables(model.linear_probe, model.cluster_probe, net.dim)
    n_lin, n_clu = tables[0].shape[0], tables[2].shape[0]
    scratch = torch.empty(R_ * C_ * h * h, _EV_LD, device=cuda_dev)
    unary = torch.empty(HH * WW, 64, device=cuda_dev)
    Q = torch.empty(HH * WW, 64, device=cuda_dev)
    _launch_crf_unary(codes, tables, t, t, ALPHA, scratch, unary, Q, (0, R_, C_, WW), 3)
    lat64 = lambda lat: F64.lattice(lat.offset, lat.bary, lat.n1, lat.n2, lat.M)
    g64 = lat64(crf._position_lattice(HH, WW, cuda_dev, cache=False))
    image = crf.prepare_image(SO.stitch(tiles, R_, C_))
    b64 = lat64(crf._lattice_points(HH, WW, 5, F64.BI_XY_STD, F64.BI_RGB_STD, image, cuda_dev))
    m = {}
    for lo, n, probe in ((0, n_lin, "linear"), (32, n_clu, "cluster")):
        want = F64.mean_field(unary[:, lo:lo + n], g64, b64)
        q = got[f"{probe}_probs"].reshape(n, HH * WW).t()
        err = (q.double() - want).abs().max().item()
        top = want.topk(2, 1).values
        clear = (top[:, 0] - top[:, 1]) > 2 * err
        m[f"{probe}_dQ"], m[f"{probe}_near"] = err, int((~clear).sum())
        assert err < 2e-3, (probe, err)
        assert torch.equal(got[f"{probe}_preds"].reshape(-1).long()[clear], want.argmax(1)[clear]), probe
    record(f"eval_placements_baseline_crf_mosaic_{arch}", m)


@pytest.mark.parametrize("probe", ["cluster", "linear"])
def test_baseline_crf_one_probe_rows_match_the_two_probe_run(cuda_dev, probe):
    R_, C_, t = 2, 3, 32
    model = _baseline(cuda_dev, "vit_small", 27)
    tiles, label = _scene(cuda_dev, R_, C_, t, 27, smooth=True)
    both = model.eval_scene(tiles, (R_, C_), label=label, run_crf=True, want_probs=True)
    stats2 = dict(zip(("linear", "cluster"), _stats(model)))
    _reset(model)
    one = model.eval_scene(tiles, (R_, C_), label=label, run_crf=True, want_probs=True, probes=(probe,))
    assert sorted(one) == [f"{probe}_preds", f"{probe}_probs"]
    q1, q2 = one[f"{probe}_probs"], both[f"{probe}_probs"]
    assert float((q1 - q2).abs().max()) < 1e-6
    top2 = q2.topk(2, 0).values
    clear = (top2[0] - top2[1]) > 2e-6
    assert torch.equal(one[f"{probe}_preds"][clear], both[f"{probe}_preds"][clear])
    stats1 = dict(zip(("linear", "cluster"), _stats(model)))
    other = "linear" if probe == "cluster" else "cluster"
    assert int(stats1[other].sum()) == 0 and int(stats1[probe].sum()) > 0
    assert int((stats1[probe] - stats2[probe]).abs().sum()) <= 2 * int((~clear).sum())


def test_baseline_crf_map_clusters_equals_the_host_mapping(cuda_dev):
    model = _baseline(cuda_dev, "vit_small", 3, extra=2)
    tiles, label = _scene(cuda_dev, 2, 3, 32, 3)
    model.eval_scene(tiles, (2, 3), label=label)
    model.test_cluster_metrics.compute()
    raw = model.eval_scene(tiles, (2, 3), run_crf=True)["cluster_preds"]
    got = model.eval_scene(tiles, (2, 3), run_crf=True, map_clusters=True)["cluster_preds"]
    want = model.test_cluster_metrics.map_clusters(raw.long().cpu())
    assert got.dtype == torch.uint8
    assert torch.equal(torch.where(got == 255, -1, got.long()).cpu(), want.cpu())


def _scene_kw(probes):
    return dict(run_crf=True, probes=probes, want_probs=True, map_clusters=False, chunk=4)


@pytest.mark.parametrize("probes", [("linear", "cluster"), ("cluster",)])
def test_baseline_crf_scene_bands_on_one_device_equal_eval_scene(cuda_dev, probes):
    """Bands of tile rows [0, 1) and [1, 3), the second written into a staging band from tile 0 of its own rows: the
    multi-device scene's placements, run on one device."""
    R_, C_, t = 3, 4, 32
    model = _baseline(cuda_dev, "vit_small", 27)
    tiles, label = _scene(cuda_dev, R_, C_, t, 27)
    want = model.eval_scene(tiles, (R_, C_), label, **_scene_kw(probes))
    want_stats = _stats(model)
    _reset(model)
    got = model._eval_scene_bands(tiles=tiles, label=label, run_crf=True, probes=probes, want_probs=True,
                                  map_clusters=False, chunk=4, R=R_, C=C_, n_tiles=R_ * C_, H=t, W=t,
                                  bands=[(cuda_dev, 0, 1), (cuda_dev, 1, 3)])
    assert got.keys() == want.keys()
    for k in want:
        assert torch.equal(got[k], want[k]), k
    for a, b in zip(_stats(model), want_stats):
        assert torch.equal(a, b)


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2,
                    reason="needs at least 2 visible GPUs")
@pytest.mark.parametrize("arch", ARCHS)
def test_baseline_crf_scene_devices_equal_one_device(arch):
    dev = torch.device("cuda", 0)
    R_, C_, t = 3, 4, 32
    model = _baseline(dev, arch, 27)
    tiles, label = _scene(dev, R_, C_, t, 27)
    kw = _scene_kw(("linear", "cluster"))
    want = model.eval_scene(tiles, (R_, C_), label, **kw)
    want_stats = _stats(model)
    _reset(model)
    got = model.eval_scene(tiles, (R_, C_), label, devices=[0, 1], **kw)
    assert got.keys() == want.keys()
    for k in want:
        assert got[k].device == want[k].device and torch.equal(got[k], want[k]), k
    for a, b in zip(_stats(model), want_stats):
        assert torch.equal(a, b)


# ================================================================================================
# 3. coverage guard
# ================================================================================================
def test_every_entry_was_called_with_each_code_width(cuda_dev):
    """Reads what the matrix above called, so it needs the whole matrix to have run before it in this process (the
    file in order, not split by -k or across workers): it is skipped otherwise rather than reporting entries as missing
    that were only deselected."""
    if CELLS_RUN != set(CELLS):
        pytest.skip(f"{len(set(CELLS) - CELLS_RUN)} of the {len(CELLS)} matrix cells did not run before this test")
    print(f"\neval entries called (code widths): { {k: sorted(v) for k, v in sorted(CALLS.items())} }")
    missing = []
    for name in ENTRIES:
        widths = CALLS.get(name, set())
        if not widths & {384, 768}:
            missing.append((name, "wide"))
        if not name.endswith("_bf16") and 70 not in widths:
            missing.append((name, 70))
    assert not missing, missing
