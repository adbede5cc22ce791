"""The correspondence-loss kernels (csrc/corr_loss.cu through stego_b200/corr.py) against the float64 references of
tests/_corr_fp64.py, stage by stage and elementwise, at the c1-c3 shapes and feature_samples up to 64.

Bars (u = 2^-24; every |term| sum comes from the reference, see _corr_fp64.py):
  operand tiles  |hi + lo - n| <= E_n + 2^-16 (|n| + E_n): E_n from the fp32 4-tap sum (<= 5 u sum_t |a_t w_t|, FMA
                 or not, chan_scale included), the L-term sum of squares, sqrt and reciprocal; the split drops
                 |x - hi - lo| <= 2^-16 |x|.  Rows >= S and code channels >= D must be exactly zero.
  fd, cd         sum_c (E_a |b| + |a| E_b) over the split operands + 2^-16 sum_c |a b| (the dropped lo.lo) +
                 (K + 2) u sum_c |a b|, K = 3E (fd) or 3 * 128 (cd) terms.  The fp32 accumulation inside wgmma is
                 not documented as IEEE round-to-nearest; it is treated as a K-term chain, an assumption, and the
                 measured ratios are recorded rather than the bar tuned to them.
  row means      mean_j E_fd + 34 u mean_j |fd| + 2 u |m| (32 values per thread + 2 shuffles, one division / cast).
  centred fd     E_fd + E_m + u |fdc|.
  call losses    sum (|fdc - shift| + |offset|) E_cd + |cl| E_fdc + |sum cl| E_offset + L u sum |cl| (|fd| + |m| +
                 |shift|), over n = B S S, plus u |loss|; L = 80 (single tile: 64 per thread, warp, 8 warps) or 40
                 (multi-tile row partials), the fp64 finish exact by comparison.  |fd| + |m| rather than |fdc|
                 because the multi-tile path forms sum cl fd - m sum cl, which cancels on flat features.
  cd means       mean E_cd + L u mean |cd| + u |mean|.
  loss elements  |fdc + offset - shift| E_cd + |cl| (E_fdc + E_offset) + 3 u |cl| (|fdc| + |offset| + |shift|).
  d code         G's bar (from fdc, offset and up, five fp32 roundings, its own split 2^-16 |G|) through dA = G Bc,
                 dB = G^T Ac with (3 * 128 + 2 ncalls nT + 2)-term chains, the fp32 normalise backward and the
                 (hits + 2)-term gather.  Clamp kinks: clamp is 1-Lipschitz, so the forward bars need no kink rule;
                 in the backward an element with |cd - bound| < E_cd may pass or stop the gradient, so its
                 |up (fdc + offset - shift)| is added to E_G and through it to the bar of every row it touches.
                 Elsewhere (including cd exactly at a bound with E_cd = 0, the exact-kink regime) the gradient
                 must meet the bar.
The largest error / bar ratios are written to $STEGO_PARITY_DIR when it is set.  test_intended_kernels_ran checks
with torch.profiler, in a child process, that each kind of case launches the kernels it means to test.
"""
import json
import os
import subprocess
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _corr_fp64 as R  # noqa: E402
import stego_oracle as O  # noqa: E402
from _parity_util import record  # noqa: E402

pytestmark = pytest.mark.gpu
SHAPES = {"c1": (32, 28, 384), "c2": (32, 40, 768), "c3": (16, 56, 768)}
D = 70


def _ratio(err, bar):
    err, bar = err.detach(), bar.detach()
    return float(torch.where(err == 0, torch.zeros_like(err), err / bar).max()) if err.numel() else 0.0


def _to_dev(d, dev, feat_layout, code_layout):
    """Put the CPU inputs on the device in the requested layouts.
    feat_layout: "nchw32" (fp32 NCHW: the generic sampler) or "tok16" (bf16 tokens-major [2B, hw, E] of which feats and
    feats_pos are the two halves: the vec8 sampler).  code_layout: "nchw" (two fp32 tensors) or "pair72" (one
    [2B, h, w, 72] channels-last store, code ++ code_pos, pair=True)."""
    B, E, H, W = d["feats"].shape
    out = dict(d)
    if feat_layout == "tok16":
        tok = torch.cat([d["feats"], d["feats_pos"]]).permute(0, 2, 3, 1).reshape(2 * B, H * W, E)
        tok = tok.to(dev).bfloat16().contiguous()  # the reshape above is a view with NCHW strides
        f_all = tok.view(2 * B, H, W, E).permute(0, 3, 1, 2)
        out["feats"], out["feats_pos"] = f_all[:B], f_all[B:]
    else:
        out["feats"], out["feats_pos"] = d["feats"].to(dev), d["feats_pos"].to(dev)
    if code_layout == "pair72":
        store = torch.full((2 * B, H, W, 72), float("nan"), device=dev)
        store[..., :D] = torch.cat([d["code"], d["code_pos"]]).permute(0, 2, 3, 1).to(dev)
        out["store"] = store
        code_all = store[..., :D].permute(0, 3, 1, 2)
        out["code"], out["code_pos"] = code_all[:B], code_all[B:]
    else:
        out["code"], out["code_pos"] = d["code"].to(dev), d["code_pos"].to(dev)
    for k in ("coords1", "coords2", "perms", "chan_scale", "chan_scale_pos"):
        out[k] = d[k].to(dev) if d[k] is not None else None
    return out


def _run(x, cfg, want_elems, pair, raw, gl, gelem, gcd):
    """one forward + backward through corr.corr_loss; the saved operand tiles, stats and row means"""
    from stego_b200 import corr
    spec = corr.make_spec(cfg)
    if pair:  # a fresh leaf store per run: the gradient arrives in its first D channels
        store = x["store"].detach().clone().requires_grad_(True)
        code = store[..., :D].permute(0, 3, 1, 2)
        args = (code, None)
    else:
        code, code_pos = x["code"].clone().requires_grad_(True), x["code_pos"].clone().requires_grad_(True)
        args = (code, code_pos)
    perms = x["perms"] if cfg.neg_samples else None
    losses, cd_means, cd, elems = corr.corr_loss(x["feats"], x["feats_pos"], *args, x["coords1"], x["coords2"], perms,
                                                 spec, want_elems=want_elems, chan_scale=x["chan_scale"],
                                                 chan_scale_pos=x["chan_scale_pos"], raw_perms=raw, pair=pair)
    saved = [t.detach().clone() for t in losses.grad_fn.saved_tensors]
    outs, grads = [losses], [gl]
    if want_elems:
        outs += [cd, elems]
        grads += [gcd, gelem]
    torch.autograd.backward(outs, grads)
    if pair:
        B = code.shape[0] // 2
        grad = store.grad[..., :D].permute(0, 3, 1, 2)
        dc, dcp = grad[:B], grad[B:]
    else:
        dc, dcp = code.grad, code_pos.grad
    torch.cuda.synchronize()
    return dict(losses=losses.detach(), cd_means=cd_means, cd=cd, elems=elems, ftiles=saved[0], ctiles=saved[1],
                stats=saved[2], row_means=saved[8], dcode=dc, dcode_pos=dcp, tiled=spec.tiled)


def _case(dev, tag, regime, B, H, W, E, fs, n_neg=5, cfg_over=None, want_elems=True, feat_layout="tok16",
          code_layout="pair72", raw=True, seed=0, upstream=True):
    cfg = O.LossCfg(feature_samples=fs, neg_samples=n_neg, **(cfg_over or {}))
    d = R.make_inputs(regime, B, E, D, H, W, fs, n_neg, seed=seed)
    if not raw and n_neg:
        d["perms"] = R.resolve_perms(d["perms"], B, True)
    x = _to_dev(d, dev, feat_layout, code_layout)
    S, nc = fs * fs, 2 + n_neg
    g = torch.Generator(device=dev).manual_seed(seed + 11)
    gl = torch.tensor([0.67, 0.25] + [0.63 / max(n_neg, 1)] * n_neg, device=dev)
    gelem = gcd = None
    if want_elems and upstream:
        gelem = torch.randn(nc, B, S, S, device=dev, generator=g) / (B * S * S) * 30
        gcd = torch.randn(nc, B, S, S, device=dev, generator=g) / (B * S * S) * 3
    elif want_elems:
        gelem = torch.zeros(nc, B, S, S, device=dev)
        gcd = torch.zeros(nc, B, S, S, device=dev)
    got = _run(x, cfg, want_elems, code_layout == "pair72", raw, gl, gelem, gcd)
    ref = R.CorrRef(x["feats"], x["feats_pos"], x["code"].detach(), x["code_pos"].detach(), x["coords1"], x["coords2"],
                    x["perms"], cfg, x["chan_scale"], x["chan_scale_pos"], raw_perms=raw, vec8=feat_layout == "tok16")
    m = {}
    # ---- operand tiles
    for name, tiles, vals, bars, C in (("ftiles", got["ftiles"], ref.fn, ref.fE, E), ("ctiles", got["ctiles"], ref.cn,
                                                                                      ref.cE, D)):
        t = tiles.double()
        hl = t[0] + t[1]
        assert torch.equal(tiles[:, :, :, S:], torch.zeros_like(tiles[:, :, :, S:])), (tag, name, "rows >= S")
        assert torch.equal(tiles[..., C:], torch.zeros_like(tiles[..., C:])), (tag, name, "pad channels")
        r = 0.0
        for s in range(ref.nslots):
            n, En = vals[s], bars[s]
            r = max(r, _ratio((hl[s, :, :S, :C] - n).abs(), En + R.SPLIT * (n.abs() + En)))
        m[name] = r
    # ---- stats
    stats = ref.forward()
    m["loss"] = max(abs(got["losses"][k].item() - st["loss"]) / st["E_loss"] for k, st in enumerate(stats))
    m["cd_mean"] = max(_ratio(torch.tensor(abs(got["cd_means"][k].item() - st["cd_mean"])), torch.tensor(st["E_cd_mean"]))
                       for k, st in enumerate(stats))
    # ---- blocks: cd, centred fd, row means, loss elements
    acc = dict(cd=0.0, row_mean=0.0, elem=0.0)

    def visit(k, b, blk):
        if got["tiled"]:
            rm = got["row_means"][k, b, :S].double()[:, None]
            acc["row_mean"] = max(acc["row_mean"], _ratio((rm - blk["m"]).abs(), blk["Em"]))
        if want_elems:
            acc["cd"] = max(acc["cd"], _ratio((got["cd"][k, b].double() - blk["cd"]).abs(), blk["Ecd"]))
            acc["elem"] = max(acc["elem"], _ratio((got["elems"][k, b].double() - blk["elem"]).abs(), blk["Eelem"]))

    (dc, Edc), (dcp, Edcp) = ref.backward(gl, gelem, gcd, visit=visit)
    m.update(acc)
    assert torch.isfinite(got["dcode"]).all() and torch.isfinite(got["dcode_pos"]).all(), tag
    m["dcode"] = _ratio((got["dcode"].double() - dc).abs(), Edc)
    m["dcode_pos"] = _ratio((got["dcode_pos"].double() - dcp).abs(), Edcp)
    m["band_elements"] = ref.band_count
    m["max_gather_hits"] = int(max(ref.hits[0].max().item(), ref.hits[1].max().item()))
    record(f"corr_fp64_{tag}", m)
    for k, v in m.items():
        if k not in ("band_elements", "max_gather_hits"):
            assert v <= 1.0, (tag, k, m)
    return m


# ================================================================================================
# single tile (fs = 11, S = 121) at the training shapes, the fused step's layouts
# ================================================================================================
@pytest.mark.parametrize("shape", list(SHAPES))
def test_single_tile_production(cuda_dev, shape):
    """c1 / c2 / c3, fs 11, 5 negatives: bf16 tokens-major features (vec8 sampler), code ++ code_pos in one
    channels-last store padded to 72 (pair=True), raw randperm draws, chan_scale, random upstream gelem / gcd."""
    B, h, E = SHAPES[shape]
    _case(cuda_dev, f"single_{shape}", "corr", B, h, h, E, 11)


@pytest.mark.parametrize("regime", ["flat", "kinks", "border", "zeros", "tagged", "scale1e3", "scale1e-3"])
@pytest.mark.parametrize("fs", [11, 16])
def test_regimes(cuda_dev, regime, fs):
    """Every input regime of _corr_fp64.make_inputs on both implementations (fs 11 single tile, fs 16 multi-tile);
    kinks under stabalize too, so that cd sits within the band of 0.8."""
    over = dict(stabalize=True) if regime == "kinks" else None
    _case(cuda_dev, f"regime_{regime}_fs{fs}", regime, 4, 17, 21, 384, fs, cfg_over=over, seed=fs)


@pytest.mark.parametrize("fs,B", [(12, 4), (16, 4), (23, 4), (32, 2), (64, 2)])
def test_multi_tile(cuda_dev, fs, B):
    """S = 144 (second tile 16 valid rows), 256, 529, 1024 (8 tiles), 4096 (the maximum).  want_elems returns three
    [ncalls, B, S, S] fp32 tensors (about 1.4 GB per image at fs 64), so B is 2 at fs 32 and 64."""
    _case(cuda_dev, f"tiled_fs{fs}", "corr", B, 28, 28, 384, fs)


@pytest.mark.parametrize("fs", [16, 28])
@pytest.mark.parametrize("shape", ["c1", "c3"])
def test_multi_tile_training_shapes(cuda_dev, shape, fs):
    """The full training batch at c1 and c3 with fs 16 and 28, without the [ncalls, B, S, S] outputs."""
    B, h, E = SHAPES[shape]
    _case(cuda_dev, f"tiled_{shape}_fs{fs}", "corr", B, h, h, E, fs, want_elems=False)


@pytest.mark.parametrize("E,layout", [(64, "nchw32"), (384, "nchw32"), (768, "nchw32"), (128, "tok16"),
                                      (384, "tok16"), (768, "tok16")])
def test_sampler_variants(cuda_dev, E, layout):
    """generic sample_norm_kernel NV = 2 / 12 / 24 (fp32 NCHW) and sample_norm_vec8_kernel NI = 1 / 2 / 3 (bf16
    tokens-major), with two separate fp32 code tensors and resolved permutations."""
    _case(cuda_dev, f"sampler_{layout}_E{E}", "tagged", 3, 12, 10, E, 11, feat_layout=layout, code_layout="nchw",
          raw=False, seed=E)


@pytest.mark.parametrize("case", ["B1_fs11", "B1_fs16", "B2_raw", "nonsquare_fs_gt_h", "H2", "W2", "no_neg_tiled"])
def test_edges(cuda_dev, case):
    """A batch of one (the raw-perm fix-up maps every negative to image 0 itself), B = 2 with fixed points, a
    non-square map smaller than feature_samples, the smallest maps the kernels take (H or W = 2), no negatives."""
    B, H, W, fs, n_neg = {"B1_fs11": (1, 28, 28, 11, 5), "B1_fs16": (1, 28, 28, 16, 3), "B2_raw": (2, 20, 20, 13, 5),
                          "nonsquare_fs_gt_h": (3, 9, 13, 16, 2), "H2": (2, 2, 17, 11, 2), "W2": (2, 19, 2, 14, 2),
                          "no_neg_tiled": (2, 16, 16, 20, 0)}[case]
    _case(cuda_dev, f"edge_{case}", "tagged", B, H, W, 384, fs, n_neg=n_neg, seed=B * 7 + fs)


@pytest.mark.parametrize("branch", ["no_pointwise", "no_zero_clamp", "stabalize"])
@pytest.mark.parametrize("fs", [11, 23])
def test_cfg_branches(cuda_dev, branch, fs):
    over = {"no_pointwise": dict(pointwise=False), "no_zero_clamp": dict(zero_clamp=False, stabalize=True),
            "stabalize": dict(stabalize=True)}[branch]
    _case(cuda_dev, f"branch_{branch}_fs{fs}", "corr", 3, 20, 20, 384, fs, cfg_over=over, seed=fs)


@pytest.mark.parametrize("fs", [11, 32])
def test_two_launches_bit_identical(cuda_dev, fs):
    cfg = O.LossCfg(feature_samples=fs)
    d = R.make_inputs("corr", 4, 384, D, 28, 28, fs, 5, seed=3)
    x = _to_dev(d, cuda_dev, "tok16", "pair72")
    S = fs * fs
    g = torch.Generator(device=cuda_dev).manual_seed(1)
    gl = torch.tensor([0.67, 0.25] + [0.126] * 5, device=cuda_dev)
    gelem = torch.randn(7, 4, S, S, device=cuda_dev, generator=g) * 1e-5
    gcd = torch.randn(7, 4, S, S, device=cuda_dev, generator=g) * 1e-6
    a = _run(x, cfg, True, True, True, gl, gelem, gcd)
    b = _run(x, cfg, True, True, True, gl, gelem, gcd)
    for k in ("losses", "cd_means", "cd", "elems", "ftiles", "ctiles", "stats", "dcode", "dcode_pos"):
        assert torch.equal(a[k], b[k]), k


# ================================================================================================
# which kernel each kind of case runs (torch.profiler in a child process)
# ================================================================================================
def _kernel_cases(dev):
    def launch(E, layout, fs, code_layout):
        cfg = O.LossCfg(feature_samples=fs)
        d = R.make_inputs("corr", 2, E, D, 16, 16, fs, 5, seed=1)
        x = _to_dev(d, dev, layout, code_layout)
        gl = torch.ones(7, device=dev)
        return lambda: _run(x, cfg, False, code_layout == "pair72", True, gl, None, None)

    single = ("corr_kernel<false>", "corr_kernel<true>", "corr_finish_kernel", "sample_norm_bwd_kernel<3, false>")
    tiled = ("corr_tiled_kernel<0>", "corr_tiled_kernel<1>", "corr_tiled_kernel<2>", "corr_tiled_finish_kernel",
             "sample_norm_bwd_kernel<3, true>")
    return {
        "vec8_single": (launch(384, "tok16", 11, "pair72"), ("sample_norm_vec8_kernel<2, false>",) + single,
                        ("corr_tiled_kernel",)),
        "vec8_tiled": (launch(768, "tok16", 16, "pair72"), ("sample_norm_vec8_kernel<3, true>",) + tiled,
                       ("corr_kernel<",)),
        "vec8_ni1": (launch(128, "tok16", 11, "pair72"), ("sample_norm_vec8_kernel<1, false>",), ()),
        "generic_single": (launch(64, "nchw32", 11, "nchw"), ("sample_norm_kernel<2, false>",) + single,
                           ("sample_norm_vec8_kernel<", "corr_tiled_kernel")),
        "generic_tiled": (launch(768, "nchw32", 23, "nchw"), ("sample_norm_kernel<24, true>",) + tiled,
                          ("sample_norm_vec8_kernel<", "corr_kernel<")),
    }


def test_intended_kernels_ran(cuda_dev):
    """bf16 tokens-major features take the vec8 sampler, fp32 NCHW the generic one; fs <= 11 the single-tile kernels,
    fs >= 12 the multi-tile ones."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--kernel-names"], cwd=root, capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
    for case, (want, not_want) in got["expect"].items():
        names = [n.replace("(int)", "") for n in got["names"][case]]  # demangled as kernel<(int)2, false>
        for k in want:
            assert any(k in n for n in names), (case, k, names)
        for k in not_want:
            assert not any(k in n for n in names), (case, k, names)


if __name__ == "__main__" and sys.argv[1:] == ["--kernel-names"]:
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from torch.profiler import ProfilerActivity, profile
    for _ in range(2):  # the first sessions of a process can miss kernel records while the profiler initialises
        with profile(activities=[ProfilerActivity.CUDA]):
            torch.ones(1024, device="cuda").sum().item()
    names, expect = {}, {}
    for case, (fn, want, not_want) in _kernel_cases(torch.device("cuda:0")).items():
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names[case] = sorted({e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA})
        expect[case] = (list(want), list(not_want))
    print(json.dumps(dict(names=names, expect=expect)))
