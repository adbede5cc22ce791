"""The segmentation head (csrc/head.cu glue + the wgmma GEMMs of csrc/gemm.cu, through stego_b200/modules.py) and the
Adam updates (adam_kernel, p2p_adam_kernel) against the float64 references of tests/_head_fp64.py, stage by stage and
elementwise, at the c1-c3 shapes (M = 2 B h^2 = 50 176 / 102 400 / 100 352 head rows).

Bars (u = 2^-24, gamma_k = k u / (1 - k u); bf16 rounding is half an ulp, 2^-8 relative; every |term| sum comes from
the reference):
  glue           dropout3, cast_pad and relu_bwd are one fp32 operation and one bf16 rounding: bit-exact against
                 torch's own (f.float() * m).bfloat16(), .bfloat16() and where(h > 0, dh, 0).bfloat16().
  GEMM           the fp32 accumulation inside wgmma is not documented as IEEE round-to-nearest; it is treated as a
                 K-term chain (DESIGN.md section 4), an assumption: the measured ratios are recorded, not the bar tuned.
                 hid: gamma_{E+2} pre_abs through the ReLU (1-Lipschitz), then the bf16 store: 2^-8 of the stored
                 value.  code: gamma_{E+3} code_abs (two K = E chains, two bias adds and the residual or reduce-add,
                 on the kernel's own hid).  dh = dyb Wb: gamma_{130} (K = 128 padded rows + the store).
  wgrad          split-K: a chain of kb_per_split * 64 rows (ceil(ceil(M / 64) / splits) k-blocks), then `splits`
                 fp32 atomics onto zero: gamma_{64 kbps + splits}, for splits 1, ops.wgrad_splits and M // 512.
  colsum         vector path: 32 rows per warp, 8 warps per block, one atomic per block onto the caller's value:
                 gamma_{40 + blocks} (sum |x| + |out0|); scalar path: 512 rows, then one atomic per 512-row block.
  Adam           stage-wise from the given fp32 state, with 1 - beta1, 1 - beta2, lr / (1 - beta1^t) and
                 sqrt(1 - beta2^t) rounded once each from double: m = fma(1-b1, g s, m b1): gamma_3 m_abs;
                 v = fma((1-b2) g s, g s, v b2): gamma_5 v_abs; from the kernel's m, v: denom = sqrt(v) / sqrt_bc2 +
                 eps within gamma_4, q = m / denom within gamma_5, step_size q within gamma_6, p = fma(-step_size,
                 q, p) rounds that once: gamma_6 (1 + u) |upd| + u |p - upd|.  A quarter of the elements start at
                 p = 0, where the parameter is the update itself: gamma_7 |upd|.
  step losses    gamma_{ncalls+3} (sum |w s| + |extras|) for the total, gamma_{ncalls} for the means.
test_fused_step_head_fp64 applies the same bars to the replayed training step's own workspace at c1-c3.
The code against the exact head (no bf16 anywhere) gets the loose bar 6 * 2^-8 prop_abs: two bf16 roundings per
product in each layer plus the hidden layer's error through |Wb|.  The largest error / bar ratios are written to
$STEGO_PARITY_DIR when it is set.  test_intended_kernels_ran checks with torch.profiler, in a child process, that the
colsum and GEMM-epilogue cases launch the kernel they mean to test.
"""
import json
import os
import subprocess
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _head_fp64 as R  # noqa: E402
from _parity_util import grads_of, make_batch, make_model, params_of, record  # noqa: E402

pytestmark = pytest.mark.gpu
U, G = R.U, R.gamma
NAN = float("nan")


def _lib():
    from stego_b200 import _lib
    return _lib


def _ratio(err, bar):
    err, bar = err.detach().double(), bar.detach().double()
    return float(torch.where(err == 0, torch.zeros_like(err), err / bar).max()) if err.numel() else 0.0


class Ratios(dict):
    """largest err / bar per quantity; `check` asserts after everything is recorded"""

    def add(self, name, got, ref, bar):
        r = _ratio((got.double() - ref.double()).abs(), bar)
        self[name] = max(self.get(name, 0.0), r)
        return r

    def check(self, tag):
        record(tag, dict(self))
        bad = {k: v for k, v in self.items() if not v <= 1.0}
        assert not bad, (tag, bad)


def _same_bits(a, b):
    a, b = a.contiguous(), b.contiguous()
    it = {2: torch.int16, 4: torch.int32}[a.element_size()]
    return torch.equal(a.view(it), b.view(it))


# ================================================================================================
# 1. glue kernels, bit-exact
# ================================================================================================
def _special_bf16(dev):
    """+-0, the smallest bf16 subnormals, the largest bf16, values at +-300"""
    tiny = torch.tensor([1], dtype=torch.int16).view(torch.bfloat16).float().item()
    big = torch.finfo(torch.bfloat16).max
    return torch.tensor([0.0, -0.0, tiny, -tiny, 3 * tiny, big, -big, 300.0, -300.0, 1.0], device=dev)


@pytest.mark.parametrize("E,hw", [(384, 784), (768, 1600), (768, 33)])
def test_dropout3_bit_exact(cuda_dev, E, hw):
    lib = _lib()
    B = 4
    g = torch.Generator(device=cuda_dev).manual_seed(E + hw)
    f = torch.randn(B * hw, E, device=cuda_dev, generator=g)
    sp = _special_bf16(cuda_dev)
    f[:, :sp.numel()] = sp
    f = f.bfloat16()
    keep = (torch.rand(3, B, E, device=cuda_dev, generator=g) > 0.1).float()
    keep[:, 2] = 0.0  # one whole image dropped
    masks = (keep * R.DROPPED).float()
    masks[2, 0, :8] = torch.tensor([0.5, 3.0, 1e-30, 7e20, -1.0, 0.0, 2.0, 1.0])  # arbitrary multipliers too
    outs = [torch.full((B * hw, E), NAN, dtype=torch.bfloat16, device=cuda_dev) for _ in range(3)]
    _lib().check(lib.load().stego_head_dropout3(f.data_ptr(), *(m.data_ptr() for m in masks), *(o.data_ptr() for o in outs),
                                                B, hw, E, lib.stream()), "stego_head_dropout3")
    torch.cuda.synchronize()
    for k in range(3):
        want = (f.float().view(B, hw, E) * masks[k].view(B, 1, E)).bfloat16().view(B * hw, E)
        assert _same_bits(outs[k], want), k
    assert (outs[0].view(B, hw, E)[2] == 0).all()


def test_cast_pad_bit_exact(cuda_dev):
    lib = _lib()
    rows, ld_in, C, ld_out = 1031, 72, 70, 128
    g = torch.Generator(device=cuda_dev).manual_seed(0)
    x = torch.randn(rows, ld_in, device=cuda_dev, generator=g) * 1e-3
    x = torch.where(torch.rand(rows, ld_in, device=cuda_dev, generator=g) < 0.25, R.bf16_ties(x), x)
    big = torch.finfo(torch.bfloat16).max
    # the largest fp32 below the tie between the bf16 maximum and the next binade: still rounds to the maximum
    below_inf = torch.tensor(big, dtype=torch.float32).view(torch.int32) + 0x7FFF
    special = torch.tensor([0.0, -0.0, 1e-40, -1e-40, 1e-45, 2.0 ** -133, 2.0 ** -134, 3 * 2.0 ** -135, big, -big],
                           device=cuda_dev)
    x[0, :special.numel()] = special
    x[1, :2] = below_inf.view(torch.float32).to(cuda_dev) * torch.tensor([1.0, -1.0], device=cuda_dev)
    x[:, C:] = NAN  # columns the cast must not read
    out = torch.full((rows, ld_out), NAN, dtype=torch.bfloat16, device=cuda_dev)
    lib.check(lib.load().stego_cast_pad_bf16(x.data_ptr(), ld_in, C, out.data_ptr(), ld_out, rows, lib.stream()),
              "stego_cast_pad_bf16")
    torch.cuda.synchronize()
    assert _same_bits(out[:, :C], x[:, :C].bfloat16())
    assert (out[:, C:].view(torch.int16) == 0).all()  # +0, not only == 0
    assert torch.isfinite(out[1, :2].float()).all()


def test_relu_bwd_bit_exact(cuda_dev):
    lib = _lib()
    M, E = 517, 384
    g = torch.Generator(device=cuda_dev).manual_seed(1)
    dh = torch.randn(M, E, device=cuda_dev, generator=g) * 1e-2
    dh = torch.where(torch.rand(M, E, device=cuda_dev, generator=g) < 0.25, R.bf16_ties(dh), dh)
    h = torch.randn(M, E, device=cuda_dev, generator=g).bfloat16()
    sp = _special_bf16(cuda_dev).bfloat16()
    h[:, :sp.numel()] = sp
    dh[0, :4] = torch.tensor([-0.0, 0.0, 1e-40, -1e-40])
    out = torch.full((M, E), NAN, dtype=torch.bfloat16, device=cuda_dev)
    lib.check(lib.load().stego_relu_bwd_bf16(dh.data_ptr(), h.data_ptr(), out.data_ptr(), M * E, lib.stream()),
              "stego_relu_bwd_bf16")
    torch.cuda.synchronize()
    assert _same_bits(out, torch.where(h.float() > 0, dh, 0.0).bfloat16())
    assert (out[:, 0:2].view(torch.int16) == 0).all()  # h = +0 and -0 stop the gradient (+0 out)


# ================================================================================================
# 2. stego_colsum against fp64
# ================================================================================================
COLSUM = [  # (dtype, C, ld, element offset of the base, vector path?)
    (torch.float32, 72, 72, 0, True), (torch.float32, 384, 384, 0, True), (torch.float32, 72, 128, 0, True),
    (torch.bfloat16, 384, 384, 0, True), (torch.bfloat16, 768, 768, 0, True),
    (torch.float32, 70, 70, 0, False), (torch.bfloat16, 70, 70, 0, False),
    (torch.float32, 384, 384, 1, False), (torch.bfloat16, 768, 768, 4, False),
]


def _colsum(x, ld, C, rows, out):
    lib = _lib()
    lib.check(lib.load().stego_colsum(x.data_ptr(), int(x.dtype == torch.bfloat16), ld, C, rows, out.data_ptr(),
                                      lib.stream()), "stego_colsum")


def _colsum_bar(rows, vec):
    return G(40 + (rows + 255) // 256) if vec else G(512 + (rows + 511) // 512)


@pytest.mark.parametrize("rows", [1, 31, 257, 100352])
@pytest.mark.parametrize("case", COLSUM, ids=lambda c: f"{str(c[0])[6:]}_C{c[1]}_ld{c[2]}_off{c[3]}")
def test_colsum_fp64(cuda_dev, case, rows):
    dtype, C, ld, off, vec = case
    g = torch.Generator(device=cuda_dev).manual_seed(rows + C)
    base = torch.randn(rows * ld + off, device=cuda_dev, generator=g)
    base = base * 10 ** (torch.rand(base.shape, device=cuda_dev, generator=g) * 6 - 3)
    base = base.to(dtype)
    x = base[off:].view(rows, ld)
    out0 = torch.randn(C, device=cuda_dev, generator=g)
    out = out0.clone()
    _colsum(x, ld, C, rows, out)
    torch.cuda.synchronize()
    xd = x[:, :C].double()
    ref = out0.double() + xd.sum(0)
    bar = _colsum_bar(rows, vec) * (xd.abs().sum(0) + out0.double().abs())
    r = Ratios()
    r.add("colsum", out, ref, bar)
    r.check(f"head_fp64_colsum_{str(dtype)[6:]}_C{C}_ld{ld}_off{off}_rows{rows}")


# ================================================================================================
# 3. head forward
# ================================================================================================
def _round8(n):
    return (n + 7) // 8 * 8


def _forward(dev, x, B, hw, E, d, nonlinear=True, train=True):
    """modules.head_forward over fresh buffers (NaN-filled operands, code padding columns at a sentinel)"""
    from stego_b200 import modules
    M, P = B * hw, _round8(d)
    bf = dict(dtype=torch.bfloat16, device=dev)
    w1p = torch.zeros(128, E, **bf)
    wab, wbp = (torch.empty(E, E, **bf), torch.zeros(128, E, **bf)) if nonlinear else (None, None)
    modules.pack_head_weights(x["w1"], x["wa"], x["wb"], w1p, wab, wbp)
    if train:
        x1 = torch.full((M, E), NAN, **bf)
        x2 = torch.full((M, E), NAN, **bf) if nonlinear else None
    else:
        x1 = x2 = x["f"]
    hid = torch.full((M, E), NAN, **bf) if nonlinear else None
    code = torch.full((M, P), 7.0, device=dev)
    m1, m2 = (x["m1"], x["m2"] if nonlinear else None) if train else (None, None)
    modules.head_forward(x["f"], m1, m2, B, hw, x1, x2, hid, code, w1p, x["b1"], wab, x["ba"], wbp, x["bb"])
    torch.cuda.synchronize()
    return dict(x1=x1, x2=x2, hid=hid, code=code, wbp=wbp, w1p=w1p)


def _check_forward(r, k, x, B, d, nonlinear, train, exact=True, pad=7.0):
    """stage-wise checks of one forward (pad: what the code's padding columns held before it)"""
    m1, m2 = (x["m1"], x["m2"]) if train else (None, None)
    E = x["f"].shape[1]
    ref = R.head_forward(x["f"], m1, m2, B, x["w1"], x["b1"], x["wa"], x["ba"], x["wb"], x["bb"],
                         hid=k["hid"] if nonlinear else None)
    assert torch.equal(k["x1"].double(), ref["x1"]), "x1"
    if nonlinear:
        assert torch.equal(k["x2"].double(), ref["x2"]), "x2"
        relu = torch.relu(ref["pre"])
        e_pre = G(E + 2) * ref["pre_abs"]
        r.add("hid", k["hid"], relu, e_pre * (1 + R.UB) + R.UB * relu + 2.0 ** -133)
    r.add("code", k["code"][:, :d], ref["code"], G(E + 3) * ref["code_abs"])
    assert (k["code"][:, d:] == pad).all(), "padding columns of code were written"
    if exact:
        ex = R.head_forward(x["f"], m1, m2, B, x["w1"], x["b1"], x["wa"], x["ba"], x["wb"], x["bb"], rnd=False)
        r.add("code_vs_exact_head_loose", k["code"][:, :d], ex["code"], 6 * R.UB * ex["prop_abs"])


@pytest.mark.parametrize("regime", ["uniform", "outliers", "zero_pre", "dropped"])
@pytest.mark.parametrize("shape", ["c1", "c2", "c3"])
def test_head_forward_fp64(cuda_dev, shape, regime):
    Bi, h, E = R.SHAPES[shape]
    B, hw = 2 * Bi, h * h
    x = R.head_inputs(regime, B, hw, E, seed=11, device=cuda_dev)
    k = _forward(cuda_dev, x, B, hw, E, R.D)
    r = Ratios()
    _check_forward(r, k, x, B, R.D, True, True)
    if regime == "zero_pre":
        band = slice(E // 4, E // 4 + 32)
        assert (k["hid"][:, band].view(torch.int16) == 0).all()  # relu(+0) stored as +0
    r.check(f"head_fp64_forward_{shape}_{regime}")


@pytest.mark.parametrize("d", [64, 72, 96])
def test_head_forward_tma_epilogue_widths(cuda_dev, d):
    """D = 64, 72 and 96 rows are whole 16-byte units: TMA store + fp32 reduce-add for the residual."""
    Bi, h, E = R.SHAPES["c1"]
    B, hw = 2 * Bi, h * h
    x = R.head_inputs("uniform", B, hw, E, d=d, seed=12, device=cuda_dev)
    k = _forward(cuda_dev, x, B, hw, E, d)
    r = Ratios()
    _check_forward(r, k, x, B, d, True, True)
    r.check(f"head_fp64_forward_c1_D{d}")


@pytest.mark.parametrize("variant", ["linear", "eval", "linear_eval"])
def test_head_forward_linear_and_eval(cuda_dev, variant):
    Bi, h, E = R.SHAPES["c1"]
    B, hw = 2 * Bi, h * h
    nonlinear, train = "linear" not in variant, "eval" not in variant
    x = R.head_inputs("dropped", B, hw, E, nonlinear=nonlinear, seed=13, device=cuda_dev)
    k = _forward(cuda_dev, x, B, hw, E, R.D, nonlinear=nonlinear, train=train)
    r = Ratios()
    _check_forward(r, k, x, B, R.D, nonlinear, train)
    r.check(f"head_fp64_forward_{variant}")


def test_head_autograd_path_d128(cuda_dev):
    """_HeadFn (the autograd path) at D = 128: forward stage-wise and backward against fp64 from its saved operands."""
    from stego_b200.modules import _HeadFn
    Bi, h, E = R.SHAPES["c1"]
    B, hw, d = 2 * Bi, h * h, 128
    x = R.head_inputs("dropped", B, hw, E, d=d, seed=14, device=cuda_dev)
    ps = [x[n].clone().requires_grad_(True) for n in ("w1", "b1", "wa", "ba", "wb", "bb")]
    code = _HeadFn.apply(x["f"], x["m1"], x["m2"], B, hw, *ps)
    x1, x2, hid, wbp = (t.detach().clone() for t in code.grad_fn.saved_tensors)
    k = dict(x1=x1, x2=x2, hid=hid, code=torch.cat([code.detach(), torch.full_like(code[:, :1], 7.0)], 1))
    r = Ratios()
    _check_forward(r, k, x, B, d, True, True)
    dc = R.dcode_inputs("dense", B, h, h, d, d=d, seed=15, device=cuda_dev)
    code.backward(dc)
    torch.cuda.synchronize()
    ref = R.head_backward(dc, x1, x2, hid, wbp, d=d)
    M = B * hw
    sms = torch.cuda.get_device_properties(cuda_dev).multi_processor_count
    from stego_b200 import ops
    wg = lambda rows: _wgrad_bar(M, ops.wgrad_splits(M, rows, E, sms))
    r.add("db1", ps[1].grad, ref["db"], _colsum_bar(M, True) * ref["db_abs"])
    r.add("dw1", ps[0].grad, ref["dw1"], wg(d) * ref["dw1_abs"])
    r.add("dwb", ps[4].grad, ref["dwb"], wg(d) * ref["dwb_abs"])
    # dh is not kept by the autograd path: dba / dwa against the exact dh carry dh's bar through the bf16 store
    dh_bar = G(130) * ref["dh_abs"]
    mask = (hid > 0).double()
    e_dhb = (dh_bar * (1 + R.UB) + 2 * R.UB * ref["dh"].abs()) * mask  # two bf16 roundings of nearby values
    e_dba, e_dwa = e_dhb.sum(0), e_dhb.T @ x2.double().abs()
    r.add("dba", ps[3].grad, ref["dba"], e_dba + _colsum_bar(M, True) * (ref["dba_abs"] + e_dba))
    r.add("dwa", ps[2].grad, ref["dwa"], e_dwa + wg(E) * (ref["dwa_abs"] + e_dwa))
    r.check("head_fp64_autograd_D128")


# ================================================================================================
# 4. head backward
# ================================================================================================
def _wgrad_bar(M, splits):
    num_kb = (M + 63) // 64
    s = min(splits, num_kb)
    kbps = (num_kb + s - 1) // s
    s = (num_kb + kbps - 1) // kbps
    return G(64 * kbps + s)


def _backward(dev, k, dcode, E, d, splits, monkeypatch):
    from stego_b200 import modules, ops
    M = k["x1"].shape[0]
    P = dcode.shape[1]
    monkeypatch.setattr(ops, "wgrad_splits", lambda *a: splits)
    f32 = dict(dtype=torch.float32, device=dev)
    b = dict(dyb=torch.full((M, 128), NAN, dtype=torch.bfloat16, device=dev), db_pad=torch.zeros(P, **f32),
             dh=torch.full((M, E), NAN, **f32), dhb=torch.full((M, E), NAN, dtype=torch.bfloat16, device=dev),
             dw1=torch.zeros(d, E, **f32), db1=torch.full((d,), NAN, **f32), dwa=torch.zeros(E, E, **f32),
             dba=torch.zeros(E, **f32), dwb=torch.zeros(d, E, **f32), dbb=torch.full((d,), NAN, **f32))
    modules.head_backward(dcode, k["x1"], k["x2"], k["hid"], k["wbp"], b["dyb"], b["db_pad"], b["dh"], b["dhb"],
                          b["dw1"], b["db1"], b["dwa"], b["dba"], b["dwb"], b["dbb"])
    torch.cuda.synchronize()
    return b


def _check_backward(r, b, k, dcode, d, splits, ref=None):
    M, E = k["x1"].shape
    if ref is None:  # stage-wise: the kernel's own dh (deterministic: the dgrad has no atomics)
        ref = R.head_backward(dcode, k["x1"], k["x2"], k["hid"], k["wbp"], d=d, dh=b["dh"])
    dyb = torch.zeros(M, 128, dtype=torch.bfloat16, device=dcode.device)
    dyb[:, :d] = dcode[:, :d].bfloat16()
    assert _same_bits(b["dyb"], dyb), "dyb"
    assert _same_bits(b["dhb"], torch.where(k["hid"].float() > 0, b["dh"], 0.0).bfloat16()), "dhb"
    assert _same_bits(b["db1"], b["db_pad"][:d]) and _same_bits(b["dbb"], b["db_pad"][:d]), "db1 / dbb"
    cs = _colsum_bar(M, True)
    wg = _wgrad_bar(M, splits)
    r.add("db", b["db_pad"], ref["db"], cs * ref["db_abs"])
    r.add("db1", b["db1"], ref["db"][:d], cs * ref["db_abs"][:d])
    r.add("dw1", b["dw1"], ref["dw1"], wg * ref["dw1_abs"])
    r.add("dwb", b["dwb"], ref["dwb"], wg * ref["dwb_abs"])
    r.add("dh", b["dh"], ref["dh"], G(130) * ref["dh_abs"])
    r.add("dba", b["dba"], ref["dba"], cs * ref["dba_abs"])
    r.add("dwa", b["dwa"], ref["dwa"], wg * ref["dwa_abs"])
    return ref


def _split_counts(M, rows_e):
    from stego_b200 import ops
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return sorted({1, ops.wgrad_splits(M, R.D, rows_e, sms), ops.wgrad_splits(M, rows_e, rows_e, sms), max(1, M // 512)})


@pytest.mark.parametrize("kind", ["dense", "sparse"])
@pytest.mark.parametrize("shape", ["c1", "c2", "c3"])
def test_head_backward_fp64(cuda_dev, shape, kind, monkeypatch):
    Bi, h, E = R.SHAPES[shape]
    B, hw = 2 * Bi, h * h
    x = R.head_inputs("zero_pre", B, hw, E, seed=21, device=cuda_dev)
    k = _forward(cuda_dev, x, B, hw, E, R.D)
    dcode = R.dcode_inputs(kind, B, h, h, 72, seed=22, device=cuda_dev)
    r, ref, dhb0 = Ratios(), None, None
    for s in _split_counts(B * hw, E):
        b = _backward(cuda_dev, k, dcode, E, R.D, s, monkeypatch)
        if dhb0 is None:
            dhb0 = b["dhb"].clone()
        assert _same_bits(b["dhb"], dhb0)
        rs = Ratios()
        ref = _check_backward(rs, b, k, dcode, R.D, s, ref)
        for n, v in rs.items():
            key = f"{n}_splits{s}" if n.startswith("dw") else n
            r[key] = max(r.get(key, 0.0), v)
    # the cost of storing d(hidden) in bf16 before its column sum (reported; changing it is out of scope)
    dba_u = ref["dba_unrounded"]
    rel = float((ref["dba"] - dba_u).norm() / dba_u.norm().clamp_min(1e-300))
    record(f"head_fp64_backward_{shape}_{kind}_dba_bf16_storage", dict(rel_l2=rel))
    r.check(f"head_fp64_backward_{shape}_{kind}")


@pytest.mark.parametrize("M", [1, 127, 129, 511, 513, 1023, 1025, 4097, 3 * 1601])
def test_head_backward_ragged_rows(cuda_dev, M, monkeypatch):
    """Row counts that are not whole 64-row k-blocks or 128-row tiles, with one image of M pixels (odd hw)."""
    E = 384
    x = R.head_inputs("zero_pre", 1, M, E, seed=M, device=cuda_dev)
    k = _forward(cuda_dev, x, 1, M, E, R.D)
    r = Ratios()
    _check_forward(r, k, x, 1, R.D, True, True, exact=False)
    dcode = R.dcode_inputs("range", 1, 1, M, 72, seed=M + 1, device=cuda_dev)
    ref = None
    for s in _split_counts(M, E):
        b = _backward(cuda_dev, k, dcode, E, R.D, s, monkeypatch)
        ref = _check_backward(r, b, k, dcode, R.D, s, ref)
    r.check(f"head_fp64_backward_ragged_M{M}")


def test_head_backward_dynamic_range_c1(cuda_dev, monkeypatch):
    Bi, h, E = R.SHAPES["c1"]
    B, hw = 2 * Bi, h * h
    x = R.head_inputs("outliers", B, hw, E, seed=23, device=cuda_dev)
    k = _forward(cuda_dev, x, B, hw, E, R.D)
    dcode = R.dcode_inputs("range", B, h, h, 72, seed=24, device=cuda_dev)
    r, ref = Ratios(), None
    for s in _split_counts(B * hw, E):
        b = _backward(cuda_dev, k, dcode, E, R.D, s, monkeypatch)
        ref = _check_backward(r, b, k, dcode, R.D, s, ref)
    r.check("head_fp64_backward_c1_range")


FULL = {"c1": ("vit_small", 224, 32), "c2": ("vit_base", 320, 32), "c3": ("vit_base", 448, 16)}
HEAD = ["net.cluster1.0.weight", "net.cluster1.0.bias", "net.cluster2.0.weight", "net.cluster2.0.bias",
        "net.cluster2.2.weight", "net.cluster2.2.bias"]


@pytest.mark.parametrize("shape", ["c1", "c2", "c3"])
def test_fused_step_head_fp64(cuda_dev, shape):
    """The head inside the real training step: three fused steps (eager, capture, replay), then the replayed step's own
    workspace against fp64.  Forward: ws.x1 / ws.x2 bit-exact from the step's features and noises ws.M1 / ws.M2, the
    packed operands bit-equal to bf16 of the weights the step ran with (snapshotted before it: the overlapped update
    changes them afterwards), hid and code stage-wise as above.  Backward from the step's real, tap-sparse d(code)
    ws.dall: the six head gradients read from the flat gradient buffer (views the kernels accumulate into after the
    prologue's memset), ws.db_pad, dh stage-wise with the step's split counts; dyb and dhb bit-exact.  The cost of the
    bf16 storage of d(hidden) on the column sum dba is recorded."""
    from stego_b200 import ops
    arch, res, B = FULL[shape]
    model, _ = make_model(arch, cuda_dev, fused=True)
    batches = [make_batch(B, res, cuda_dev, seed=1), make_batch(B, res, cuda_dev, seed=2)]
    torch.manual_seed(777)
    for s in range(3):
        if s == 2:
            before = params_of(model)  # flushes: the parameters the replayed step runs with
        model.training_step(batches[s % 2], s)
    grads = grads_of(model)  # flushes
    torch.cuda.synchronize()
    ws = model._fused.ws
    assert ws.graph is not None and ws.eager_steps == 1, "the compared step must be a graph replay"
    B2, E, D, P, fh, fw, hw, M, nonlinear = ws.dims
    assert nonlinear and B2 == B and M == 2 * B * hw
    batch = batches[0]
    with torch.no_grad():  # the same backbone graph the step replayed, on the same images
        tok = model.net.backbone_tokens([batch["img"], batch["img_pos"]], use_graph=True).reshape(M, E).clone()
    w = {k[len("net."):]: before[k] for k in HEAD}
    assert _same_bits(ws.w1p[:D], w["cluster1.0.weight"].reshape(D, E).bfloat16())
    assert _same_bits(ws.wab, w["cluster2.0.weight"].reshape(E, E).bfloat16())
    assert _same_bits(ws.wbp[:D], w["cluster2.2.weight"].reshape(D, E).bfloat16())
    x = dict(f=tok, m1=ws.M1.view(2 * B, E), m2=ws.M2.view(2 * B, E), w1=w["cluster1.0.weight"], b1=w["cluster1.0.bias"],
             wa=w["cluster2.0.weight"], ba=w["cluster2.0.bias"], wb=w["cluster2.2.weight"], bb=w["cluster2.2.bias"])
    r = Ratios()
    _check_forward(r, dict(x1=ws.x1, x2=ws.x2, hid=ws.hid, code=ws.code), x, 2 * B, D, True, True, pad=0.0)

    dall = ws.dall.view(M, P)
    ref = R.head_backward(dall, ws.x1, ws.x2, ws.hid, ws.wbp, d=D, dh=ws.dh)
    dyb = torch.zeros(M, 128, dtype=torch.bfloat16, device=cuda_dev)
    dyb[:, :D] = dall[:, :D].bfloat16()
    assert _same_bits(ws.dyb, dyb), "dyb"
    assert _same_bits(ws.dhb, torch.where(ws.hid.float() > 0, ws.dh, 0.0).bfloat16()), "dhb"
    sms = torch.cuda.get_device_properties(cuda_dev).multi_processor_count
    wg_d, wg_e = _wgrad_bar(M, ops.wgrad_splits(M, D, E, sms)), _wgrad_bar(M, ops.wgrad_splits(M, E, E, sms))
    cs = _colsum_bar(M, True)
    g = {k: grads[k].reshape(grads[k].shape[0], -1).squeeze(1) for k in HEAD}
    r.add("db_pad", ws.db_pad, ref["db"], cs * ref["db_abs"])
    r.add("db1", g["net.cluster1.0.bias"], ref["db"][:D], cs * ref["db_abs"][:D])
    r.add("dbb", g["net.cluster2.2.bias"], ref["db"][:D], cs * ref["db_abs"][:D])
    r.add("dw1", g["net.cluster1.0.weight"], ref["dw1"], wg_d * ref["dw1_abs"])
    r.add("dwb", g["net.cluster2.2.weight"], ref["dwb"], wg_d * ref["dwb_abs"])
    r.add("dh", ws.dh, ref["dh"], G(130) * ref["dh_abs"])
    r.add("dba", g["net.cluster2.0.bias"], ref["dba"], cs * ref["dba_abs"])
    r.add("dwa", g["net.cluster2.0.weight"], ref["dwa"], wg_e * ref["dwa_abs"])
    dba_u = ref["dba_unrounded"]
    record(f"head_fp64_fused_step_{shape}_dba_bf16_storage", dict(
        rel_l2=float((ref["dba"] - dba_u).norm() / dba_u.norm()),
        max_rel_to_abs_sum=float(((ref["dba"] - dba_u).abs() / ref["dba_abs"].clamp_min(1e-300)).max()),
        dcode_nonzero_row_fraction=float((dall[:, :D] != 0).any(1).double().mean())))
    r.check(f"head_fp64_fused_step_{shape}")


# ================================================================================================
# 5. Adam
# ================================================================================================
def _adam_state(n, step, dev, seed):
    """arbitrary fp32 state: |g| 1e-12..1e2 with zeros, m of either sign (half opposite to g), v = 0 in places and
    sqrt(v / bc2) ~ eps in others, a quarter of the parameters at 0"""
    g_ = torch.Generator().manual_seed(seed)
    sgn = lambda: torch.where(torch.rand(n, generator=g_) < 0.5, -1.0, 1.0)
    g = sgn() * 10 ** (torch.rand(n, generator=g_) * 14 - 12)
    g[torch.rand(n, generator=g_) < 0.02] = 0.0
    m = 10 ** (torch.rand(n, generator=g_) * 10 - 9) * g.sign() * torch.where(torch.rand(n, generator=g_) < 0.5, -1.0, 1.0)
    bc2 = 1 - 0.999 ** step
    v = 10 ** (torch.rand(n, generator=g_) * 24 - 22)
    near_eps = torch.rand(n, generator=g_) < 0.2
    v = torch.where(near_eps, (1e-8 * 10 ** (torch.rand(n, generator=g_) - 0.5)) ** 2 * bc2, v)
    zero = torch.rand(n, generator=g_) < 0.02
    v[zero], g[zero[:n] & (torch.rand(n, generator=g_) < 0.5)] = 0.0, 0.0
    p = torch.randn(n, generator=g_)
    p[torch.rand(n, generator=g_) < 0.25] = 0.0
    return [t.float().to(dev) for t in (p, g, m, v)]


def _adam_ratios(r, before, after, step, lr, grad_scale, b1=0.9, b2=0.999, eps=1e-8):
    p, g, m, v = before
    p1, m1, v1 = after
    ref = R.adam(p, g, m, v, step, lr, b1, b2, eps, grad_scale)
    r.add("exp_avg", m1, ref["m"], G(3) * ref["m_abs"])
    r.add("exp_avg_sq", v1, ref["v"], G(5) * ref["v_abs"])
    upd = R.adam_update(m1, v1, step, lr, b1, b2, eps)  # stage-wise: from the kernel's moments
    pref = p.double() - upd
    # fma rounds y = p - step_size q once, and |y - pref| <= gamma_6 |upd|: |p1 - pref| <= gamma_6 (1 + u) |upd| + u |pref|
    r.add("param", p1, pref, G(6) * (1 + U) * upd.abs() + U * pref.abs())
    z = p == 0  # there p1 = fl(-step_size q): the update itself, gamma_6 and the final rounding
    r.add("update", (p - p1)[z], upd[z], G(7) * upd[z].abs())


def _adam_step_direct(p, g, m, v, lr, step, grad_scale, b1=0.9, b2=0.999, eps=1e-8):
    lib = _lib()
    lib.check(lib.load().stego_adam_step(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), p.numel(), lr, b1, b2,
                                         eps, step, grad_scale, lib.stream()), "stego_adam_step")


@pytest.mark.parametrize("grad_scale", [1.0, 0.5, 0.125])
@pytest.mark.parametrize("step", [1, 2, 10, 1000, 1000000])
def test_adam_step_fp64(cuda_dev, step, grad_scale):
    """stego_adam_step and FusedAdam.step, stage-wise from arbitrary fp32 state (n = 100 003, not a multiple of 256)."""
    from stego_b200.segmenter import FlatParams
    n, lr = 100003, 5e-4
    before = _adam_state(n, step, cuda_dev, seed=step * 7 + int(8 * grad_scale))
    r = Ratios()
    p, g, m, v = (t.clone() for t in before)
    _adam_step_direct(p, g, m, v, lr, step, grad_scale)
    torch.cuda.synchronize()
    assert torch.equal(g, before[1])
    _adam_ratios(r, before, (p, m, v), step, lr, grad_scale)
    # the same through FusedAdam over a flat buffer of two parameters
    params = [torch.nn.Parameter(before[0][:40000].clone()), torch.nn.Parameter(before[0][40000:].clone())]
    flat = FlatParams([params], [lr])
    flat.grad.copy_(before[1])
    flat.exp_avg.copy_(before[2])
    flat.exp_avg_sq.copy_(before[3])
    flat.grad_scale = grad_scale
    opt = flat.optimizers[0]
    opt.steps = step - 1
    opt.step()
    torch.cuda.synchronize()
    rf = Ratios()
    _adam_ratios(rf, before, (flat.param, flat.exp_avg, flat.exp_avg_sq), step, lr, grad_scale)
    assert _same_bits(flat.param, p) and _same_bits(flat.exp_avg, m) and _same_bits(flat.exp_avg_sq, v)
    r.update({f"fused_{k}": x for k, x in rf.items()})
    r.check(f"head_fp64_adam_step{step}_scale{grad_scale}")


def test_adam_1000_steps(cuda_dev):
    """1000 consecutive steps, each checked stage-wise; the drift from torch.optim.Adam (fp32, on the GPU, same
    gradients) is recorded with the loose bar 64 u sum_t |upd_t| + 2 u t |p| (each step may round p differently)."""
    n, lr = 4099, 5e-4
    gen = torch.Generator(device=cuda_dev).manual_seed(5)
    p = torch.randn(n, device=cuda_dev, generator=gen) * 1e-2
    m, v = torch.zeros_like(p), torch.zeros_like(p)
    tp = torch.nn.Parameter(p.clone())
    opt = torch.optim.Adam([tp], lr=lr)
    r = Ratios()
    upd_sum = torch.zeros(n, dtype=torch.float64, device=cuda_dev)
    for t in range(1, 1001):
        g = torch.randn(n, device=cuda_dev, generator=gen) * 10 ** (torch.rand(n, device=cuda_dev, generator=gen) * 6 - 6)
        before = [x.clone() for x in (p, g, m, v)]
        _adam_step_direct(p, g, m, v, lr, t, 1.0)
        _adam_ratios(r, before, (p, m, v), t, lr, 1.0)
        upd_sum += (p.double() - before[0].double()).abs()
        tp.grad = g.clone()
        opt.step()
    torch.cuda.synchronize()
    drift = _ratio((p.double() - tp.detach().double()).abs(), 64 * U * upd_sum + 2 * U * 1000 * p.double().abs())
    r["drift_vs_torch_adam_loose"] = drift
    r.check("head_fp64_adam_1000_steps")


# ================================================================================================
# 6. stego_p2p_adam on one GPU
# ================================================================================================
GROUPS = [(3, 1000, 5e-4, 1), (1500, 2501, 5e-3, 7), (4100, 17, 5e-3, 1000), (5000, 4999, 1e-3, 1000000)]


def _p2p(exports, p, grad, m, v, groups, grad_scale):
    lib = _lib()
    addr = torch.tensor([e.data_ptr() for e in exports], dtype=torch.int64)
    desc = torch.tensor([[s, k, lr, 0.9, 0.999, 1e-8, t] for s, k, lr, t in groups], dtype=torch.float64).reshape(-1)
    lib.check(lib.load().stego_p2p_adam(addr.data_ptr(), len(exports), p.data_ptr(), grad.data_ptr(), m.data_ptr(),
                                        v.data_ptr(), p.numel(), desc.data_ptr(), len(groups), grad_scale, lib.stream()),
              "stego_p2p_adam")
    torch.cuda.synchronize()


@pytest.mark.parametrize("world", [1, 2, 3, 8, 16])
def test_p2p_adam_single_gpu(cuda_dev, world):
    """Local buffers stand in for the ranks' exports (the kernel takes a host array of device addresses)."""
    n = 10007
    p0, g0, m0, v0 = _adam_state(n, 10, cuda_dev, seed=world)
    gen = torch.Generator(device=cuda_dev).manual_seed(world)
    exports = [g0 * torch.randn(n, device=cuda_dev, generator=gen) for _ in range(world)]
    exports[0][:4] = torch.tensor([-0.0, 0.0, 1.0, -1.0])
    scale = float(torch.tensor(1.0 / world, dtype=torch.float32))
    p, m, v = p0.clone(), m0.clone(), v0.clone()
    grad = torch.full((n,), NAN, device=cuda_dev)
    _p2p(exports, p, grad, m, v, GROUPS, scale)
    gsum = R.rank_sum_fp32(exports)
    assert _same_bits(grad, gsum), "grad: the fp32 sum in rank order"
    inside = torch.zeros(n, dtype=torch.bool, device=cuda_dev)
    r = Ratios()
    for s, k, lr, t in GROUPS:
        sl = slice(s, s + k)
        inside[sl] = True
        rg = Ratios()
        _adam_ratios(rg, (p0[sl], gsum[sl], m0[sl], v0[sl]), (p[sl], m[sl], v[sl]), t, lr, scale)
        for name, x in rg.items():
            r[name] = max(r.get(name, 0.0), x)
    out = ~inside
    assert _same_bits(p[out], p0[out]) and _same_bits(m[out], m0[out]) and _same_bits(v[out], v0[out])
    r.check(f"head_fp64_p2p_adam_world{world}")


def test_p2p_adam_world1_bit_identical_to_adam_step(cuda_dev):
    n = 10007
    p0, g0, m0, v0 = _adam_state(n, 3, cuda_dev, seed=99)
    p, m, v = p0.clone(), m0.clone(), v0.clone()
    grad = torch.empty_like(g0)
    _p2p([g0], p, grad, m, v, GROUPS, 1.0)
    pa, ma, va = p0.clone(), m0.clone(), v0.clone()
    for s, k, lr, t in GROUPS:
        sl = slice(s, s + k)
        _adam_step_direct(pa[sl], g0[sl], ma[sl], va[sl], lr, t, 1.0)
    torch.cuda.synchronize()
    assert _same_bits(grad, g0 + 0.0)
    assert _same_bits(p, pa) and _same_bits(m, ma) and _same_bits(v, va)


# ================================================================================================
# 7. stego_step_losses
# ================================================================================================
@pytest.mark.parametrize("extras", [False, True])
@pytest.mark.parametrize("ncalls", list(range(1, 17)))
def test_step_losses_fp64(cuda_dev, ncalls, extras):
    lib = _lib()
    gen = torch.Generator().manual_seed(ncalls)
    stats = (torch.randn(ncalls, 4, generator=gen) * 10 ** (torch.rand(ncalls, 4, generator=gen) * 4 - 2)).to(cuda_dev)
    w = torch.zeros(16, dtype=torch.float32)
    w[:ncalls] = torch.randn(ncalls, generator=gen)
    ex = [torch.randn(1, generator=gen).to(cuda_dev) for _ in range(2)] if extras else [None, None]
    out = torch.full((4,), NAN, device=cuda_dev)
    lib.check(lib.load().stego_step_losses(stats.data_ptr(), ncalls, w.data_ptr(), lib.ptr(ex[0]), lib.ptr(ex[1]),
                                           out.data_ptr(), lib.stream()), "stego_step_losses")
    torch.cuda.synchronize()
    s, wd = stats.double().cpu(), w[:ncalls].double()
    ws = wd * s[:, 0]
    e = sum(float(t.double()) for t in ex if t is not None) if extras else 0.0
    e_abs = sum(abs(float(t.double())) for t in ex if t is not None) if extras else 0.0
    nn = max(ncalls - 2, 1)
    neg, negcd = s[2:, 0].sum() / nn, s[2:, 1].sum() / nn
    oc = out.double().cpu()
    r = Ratios()
    r.add("total", oc[0], ws.sum() + e, G(ncalls + 3) * (ws.abs().sum() + e_abs))
    r.add("corr", oc[1], ws.sum(), G(ncalls + 2) * ws.abs().sum())
    r.add("neg_loss", oc[2], neg, G(ncalls) * s[2:, 0].abs().sum() / nn)
    r.add("neg_cd", oc[3], negcd, G(ncalls) * s[2:, 1].abs().sum() / nn)
    r.check(f"head_fp64_step_losses_n{ncalls}_{int(extras)}")


# ================================================================================================
# 8. which kernel each kind of case runs (torch.profiler in a child process)
# ================================================================================================
def _kernel_cases(dev):
    """name -> (launch, kernels that must run, kernels that must not); GEMM entries name the epilogue instantiation"""
    from stego_b200 import ops
    cases = {}
    for dtype, C, ld, off, vec in COLSUM:
        x = torch.randn(257 * ld + off, device=dev).to(dtype)[off:].view(257, ld)
        out = torch.zeros(C, device=dev)
        want, not_want = ("colsum_kernel<", "colsum_scalar_kernel") if vec else ("colsum_scalar_kernel", "colsum_kernel<")
        cases[f"colsum_{str(dtype)[6:]}_C{C}_ld{ld}_off{off}"] = (
            lambda x=x, ld=ld, C=C, out=out: _colsum(x, ld, C, 257, out), (want,), (not_want,))
    E, M = 384, 1000
    a = torch.randn(M, E, device=dev).bfloat16()
    for d, tma in ((70, False), (64, True), (72, True), (96, True)):
        w = torch.randn(128, E, device=dev).bfloat16()
        code = torch.zeros(M, _round8(d), device=dev)
        bias = torch.zeros(d, device=dev)

        def run(w=w, code=code, bias=bias, d=d):
            ops.gemm(a, w, code, M=M, N=d, K=E, bias=bias)
            ops.gemm(a, w, code, M=M, N=d, K=E, bias=bias, residual=code)
        cases[f"gemm_D{d}"] = (run, (f"tma_epi={int(tma)}",), (f"tma_epi={int(not tma)}",))
    return cases


def _names(prof_names):
    """kernel names, with the GEMM's last template argument (kTmaEpi) spelled as tma_epi=0/1"""
    out = set()
    for n in prof_names:
        out.add(n)
        if "gemm_bf16_kernel<" in n:
            last = n.split("gemm_bf16_kernel<", 1)[1].split(">", 1)[0].split(",")[-1].strip()
            out.add(f"tma_epi={int(last in ('true', '1', '(bool)1'))}")
    return out


def test_intended_kernels_ran(cuda_dev):
    """Shape alone does not pick the kernel: the colsum vector path also needs an aligned base and 16-byte rows, the
    TMA epilogue whole 16-byte output rows.  Profile each kind of case and check the kernel names."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    res = subprocess.run([sys.executable, os.path.abspath(__file__), "--kernel-names"], cwd=root, capture_output=True,
                         text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-4000:]
    got = json.loads(res.stdout.strip().splitlines()[-1])
    for case, (want, not_want) in got["expect"].items():
        names = got["names"][case]
        for w in want:
            assert any(w in n for n in names), (case, w, names)
        for w in not_want:
            assert not any(w in n for n in names), (case, w, names)


if __name__ == "__main__" and sys.argv[1:] == ["--kernel-names"]:
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from torch.profiler import ProfilerActivity, profile
    dev = torch.device("cuda:0")
    for _ in range(2):  # the first sessions of a process can miss kernel records while the profiler initialises
        with profile(activities=[ProfilerActivity.CUDA]):
            torch.ones(1024, device=dev).sum().item()
    names, expect = {}, {}
    for case, (fn, want, not_want) in _kernel_cases(dev).items():
        fn()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names[case] = sorted(_names({e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}))
        expect[case] = (list(want), list(not_want))
    print(json.dumps(dict(names=names, expect=expect)))
