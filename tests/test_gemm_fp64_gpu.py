"""The wgmma GEMM (stego_gemm_bf16 / stego_gemm_bf16_batched) against the float64 reference of tests/_gemm_fp64.py,
every output element within its derived bar (the bars are derived in that module's docstring).

Every case stores its operands with NaN in the pitch padding past K (or M / N for MN-major operands), in spare rows
and in the gaps between batch entries, so zero-fill must come from the tensor-map dimensions and never from memory.
Every output sits in a store filled with a sentinel: rows past M, columns between N and ldo, the gaps between batch
entries and the cls rows of row_div mode must keep it.  Store-mode outputs start as NaN, so an element left unwritten
fails its bar.  Every non-atomic case runs twice and must be bit-identical.

Covered: every instantiation (A_MN, B_MN) x {TMA, register epilogue} x {fp32, bf16 out} x {store, reduce-add /
in-place, residual != out, row_div} x {none, GELU, ReLU}; M, N and K edges with lda > K; tile counts around the SM
count; cancelling rows, rows at +-1e30 and 1e-30, magnitudes at the subnormal boundary and a bias that cancels the
product; split-K onto zero and onto a non-zero out; batch 1 / 2 / 7 / 64 with ragged M / N, odd N and a shared bias.
GELU and ReLU are also swept over every finite bf16 |x| <= 1e4 on an exact accumulator.  Refused calls return an error
and leave out untouched.  The largest error / bar ratios are written to $STEGO_PARITY_DIR when it is set.
test_intended_kernels_ran checks with torch.profiler, in a child process, that each instantiation case launches the
gemm_bf16_kernel<stages, A_MN, B_MN, TMA> it claims.
"""
import json
import os
import subprocess
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _gemm_fp64 as R  # noqa: E402
from _parity_util import record  # noqa: E402
from test_gemm_args import REFUSED, SENTINEL, refused_call  # noqa: E402

pytestmark = pytest.mark.gpu
NAN = float("nan")


class Ratios(dict):
    """largest err / bar per quantity; `check` asserts after everything is recorded"""

    def add(self, name, got, ref, bar):
        return self.put(name, R.ratio(got, ref, bar))

    def put(self, name, r):
        self[name] = max(self.get(name, 0.0), r) if r == r else r  # a NaN ratio is kept
        return r

    def check(self, tag):
        record(tag, dict(self))
        bad = {k: v for k, v in self.items() if not v <= 1.0}
        assert not bad, (tag, bad)


def _lib():
    from stego_b200 import _lib
    return _lib


def _same_bits(a, b):
    it = {2: torch.int16, 4: torch.int32}[a.element_size()]
    return torch.equal(a.contiguous().view(it), b.contiguous().view(it))


# ------------------------------------------------------------------------------------------------
# operands and outputs in padded, NaN-filled storage
# ------------------------------------------------------------------------------------------------
def _r8(x):
    return (x + 7) // 8 * 8


class Operand:
    """`batch` logical [rows, K] bf16 matrices stored K-major ([rows][ld]) or MN-major ([K][ld]) in one NaN-filled
    buffer: ld > the stored row, 3 spare stored rows per entry and an 8-element gap between entries."""

    def __init__(self, vals, mn, dev, ld_pad=8):
        batch, rows, K = vals.shape
        srows, scols = (K, rows) if mn else (rows, K)
        self.ld = _r8(scols) + ld_pad
        self.bs = (srows + 3) * self.ld + 8
        self.buf = torch.full((batch * self.bs + 8,), NAN, device=dev, dtype=torch.bfloat16)
        for i in range(batch):
            v = vals[i].t() if mn else vals[i]
            self.view(i, srows)[:, :scols] = v.to(dev, torch.bfloat16)
        self.vals = vals.to(dev).bfloat16().double()
        self.mn = mn

    def view(self, i, srows):
        return self.buf[i * self.bs:i * self.bs + srows * self.ld].view(srows, self.ld)

    @property
    def ptr(self):
        return self.buf.data_ptr()


class Output:
    """`batch` outputs [M][N] (row_div > 0: rows remapped r -> r + r // row_div + 1) in a sentinel-filled store with
    ldo >= N, spare rows and a gap between entries."""

    def __init__(self, batch, M, N, dtype, dev, ldo, row_div=0):
        self.rows = M + M // row_div + 1 if row_div else M
        self.M, self.N, self.ldo, self.row_div, self.batch = M, N, ldo, row_div, batch
        self.bs = (self.rows + 3) * ldo + 8
        self.buf = torch.full((batch * self.bs + 8,), SENTINEL, device=dev, dtype=dtype)
        idx = torch.arange(M, device=dev)
        orow = idx + idx // row_div + 1 if row_div else idx
        col = torch.arange(N, device=dev)
        self.index = (torch.arange(batch, device=dev).view(batch, 1, 1) * self.bs + orow.view(1, M, 1) * ldo +
                      col.view(1, 1, N))
        self.mask = torch.zeros_like(self.buf, dtype=torch.bool)
        self.mask[self.index.reshape(-1)] = True

    @property
    def ptr(self):
        return self.buf.data_ptr()

    def get(self):
        return self.buf[self.index]

    def set(self, vals):
        self.buf[self.index] = vals.to(self.buf.dtype)

    def guards_intact(self):
        return bool((self.buf[~self.mask] == SENTINEL).all())

    def tma_expected(self, atomic, residual_other):
        """the host rule of gemm_impl: the output is describable by a tensor map"""
        esz = self.buf.element_size()
        return (not atomic and not self.row_div and not residual_other and (self.ptr % 16 == 0) and
                (self.ldo * esz) % 16 == 0 and (self.bs * esz) % 16 == 0 and (self.N * esz) % 16 == 0)


def _values(kind, batch, M, N, K, g, dev):
    """logical A [batch, M, K], B [batch, N, K] (fp32 holding bf16 values) and bias [N] of one value regime
    uniform      A ~ N(0, 1), B ~ N(0, 1 / K), bias ~ N(0, 1)
    cancel       A's second half of K is minus its first, B's halves are equal, no bias: every result is 0 exactly,
                 from a large sum of |a b|
    huge         rows alternately at +-1e30 and 1e-30 scale (the rest N(0, 1))
    tiny         A, B ~ 1e-19: products near and below the fp32 subnormal boundary 1.2e-38, bias ~ 1e-37
    bias_cancel  every row of A and every batch entry of B equal, bias = -fp32(a b^T): results are the rounding
                 residue of a sum of size 1"""
    rn = lambda *s: torch.randn(*s, device=dev, generator=g)
    a = rn(batch, M, K)
    b = rn(batch, N, K) / K ** 0.5
    bias = rn(N)
    if kind == "cancel":
        h = K // 2
        a[..., h:2 * h] = -a[..., :h]
        b[..., h:2 * h] = b[..., :h]
        bias = torch.zeros_like(bias)
    elif kind == "huge":
        scale = torch.ones(M, device=dev)
        scale[0::3], scale[1::3] = 1e30, 1e-30
        scale[0::6] *= -1
        a = a * scale.view(1, M, 1)
    elif kind == "tiny":
        a, b, bias = a * 1e-19, b * K ** 0.5 * 1e-19, bias * 1e-37
    elif kind == "bias_cancel":
        a = a[:1, :1].expand(batch, M, K).contiguous()
        b = b[:1].expand(batch, N, K).contiguous()
        a, b = a.bfloat16().float(), b.bfloat16().float()
        bias = -(a[0, 0].double() @ b[0].double().t()).float()
    return a.bfloat16().float(), b.bfloat16().float(), bias


# ------------------------------------------------------------------------------------------------
# one case: build, launch twice, compare every element with its bar, check guards and determinism
# ------------------------------------------------------------------------------------------------
def run_case(dev, *, M, N, K, a_mn=False, b_mn=False, out_bf16=False, mode="store", act=0, use_bias=True,
             tma=True, vals="uniform", batch=1, splits=0, row_div=0, out0_zero=False, seed=0, batched_api=False,
             launch_only=False):
    """mode: store | reduce_add (residual is out) | residual (residual != out) | row_div | atomic (split-K with
    `splits`).  tma: ask for an output the TMA epilogue can describe (16-byte rows; only store / reduce_add), else
    ldo = N + 2 with a vector-aligned base (pairs through the register epilogue).  Returns (ratio, tma expected)."""
    g = torch.Generator(device=dev).manual_seed(seed)
    a, b, bias = _values(vals, batch, M, N, K, g, dev)
    bias = bias if use_bias else None
    A, B = Operand(a, a_mn, dev), Operand(b, b_mn, dev)
    dtype = torch.bfloat16 if out_bf16 else torch.float32
    ldo = (_r8(N) + 8) if tma else (N + 2)
    out = Output(batch, M, N, dtype, dev, ldo, row_div=row_div if mode == "row_div" else 0)
    residual = res_t = out0 = None
    if mode in ("residual", "row_div"):
        ldr = N + 3
        rrows = row_div + 1 if mode == "row_div" else M
        res_t = torch.full((rrows + 2, ldr), NAN, device=dev)
        res_t[:rrows, :N] = torch.randn(rrows, N, device=dev, generator=g)
        residual = res_t[:rrows, :N]
        res_log = residual[torch.arange(M, device=dev) % row_div + 1] if mode == "row_div" else residual
    if mode in ("reduce_add", "atomic"):
        init = torch.zeros(batch, M, N, device=dev) if out0_zero else torch.randn(batch, M, N, device=dev, generator=g)
        out.set(init)
        out0 = init
    else:
        out.set(torch.full((batch, M, N), NAN, device=dev))
    ref = R.reference(a, b, bias, act, residual=res_log.unsqueeze(0) if res_t is not None else None, out0=out0)
    start = out.buf.clone()

    lib = _lib()

    def launch(o):
        if batched_api or batch > 1:
            rc = lib.load().stego_gemm_bf16_batched(A.ptr, A.ld, A.bs, int(a_mn), B.ptr, B.ld, B.bs, int(b_mn), batch,
                                                    M, N, K, o.ptr, o.ldo, o.bs, int(out_bf16), lib.ptr(bias), act,
                                                    lib.stream())
        else:
            ldr = res_t.stride(0) if res_t is not None else (o.ldo if mode == "reduce_add" else 0)
            rptr = o.ptr if mode == "reduce_add" else lib.ptr(res_t)
            rc = lib.load().stego_gemm_bf16(A.ptr, A.ld, int(a_mn), B.ptr, B.ld, int(b_mn), M, N, K, o.ptr, o.ldo,
                                            int(out_bf16), lib.ptr(bias), act, rptr, ldr,
                                            row_div if mode == "row_div" else 0, max(splits, 1), int(mode == "atomic"),
                                            lib.stream())
        lib.check(rc, "stego_gemm_bf16")

    tma_exp = out.tma_expected(mode == "atomic", mode in ("residual", "row_div"))
    if launch_only:
        return launch, out, tma_exp
    launch(out)
    torch.cuda.synchronize()
    got = out.get()
    assert torch.isfinite(got).all() or not torch.isfinite(ref["out"]).all(), "unwritten or non-finite outputs"
    bar = R.bar(ref, K, act, out_bf16, added=mode in ("reduce_add", "residual", "row_div"),
                splits=splits if mode == "atomic" else 0)
    r = R.ratio(got, ref["out"], bar)
    assert out.guards_intact(), "a sentinel outside the output changed"
    if mode != "atomic":
        out2 = Output(batch, M, N, dtype, dev, ldo, row_div=out.row_div)
        out2.buf.copy_(start)
        launch(out2)
        torch.cuda.synchronize()
        assert _same_bits(out.buf, out2.buf), "two launches differ"
    return r, tma_exp


# ================================================================================================
# 1. every instantiation: layouts x epilogues x output types x epilogue terms x activations
# ================================================================================================
EPILOGUES = {  # name: (out_bf16, mode, tma)
    "tma_f32_store": (False, "store", True),
    "tma_bf16_store": (True, "store", True),
    "tma_f32_reduce_add": (False, "reduce_add", True),
    "reg_f32_store": (False, "store", False),
    "reg_bf16_store": (True, "store", False),
    "reg_f32_in_place": (False, "reduce_add", False),
    "reg_f32_residual": (False, "residual", False),
    "reg_bf16_residual": (True, "residual", False),
    "reg_f32_row_div": (False, "row_div", False),
    "reg_bf16_row_div": (True, "row_div", False),
}
LAYOUTS = [(False, False), (False, True), (True, False), (True, True)]
INST = dict(M=200, N=136, K=136, row_div=25)  # ragged in all three dimensions: 2 x 2 tiles, 3 k-blocks


@pytest.mark.parametrize("act", [0, 1, 2])
@pytest.mark.parametrize("epi", sorted(EPILOGUES))
@pytest.mark.parametrize("a_mn,b_mn", LAYOUTS)
def test_every_instantiation(cuda_dev, a_mn, b_mn, epi, act):
    out_bf16, mode, tma = EPILOGUES[epi]
    r = Ratios()
    ratio, tma_exp = run_case(cuda_dev, **INST, a_mn=a_mn, b_mn=b_mn, out_bf16=out_bf16, mode=mode, act=act, tma=tma,
                              seed=7 * act + len(epi))
    assert tma_exp == tma, (epi, tma_exp)
    r["out"] = ratio
    r.check(f"gemm_inst_{int(a_mn)}{int(b_mn)}_{epi}_act{act}")


# ================================================================================================
# 2. edges: M, N, K, tile counts
# ================================================================================================
EDGE_EPIS = [("tma_f32_store", 1), ("reg_bf16_residual", 2), ("tma_bf16_store", 1)]


@pytest.mark.parametrize("M", [1, 63, 64, 65, 127, 128, 129, 257, 785 * 3])
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (True, True)])
def test_edges_m(cuda_dev, M, a_mn, b_mn):
    r = Ratios()
    for epi, act in EDGE_EPIS:
        out_bf16, mode, tma = EPILOGUES[epi]
        r.put(epi, run_case(cuda_dev, M=M, N=136, K=136, a_mn=a_mn, b_mn=b_mn, out_bf16=out_bf16, mode=mode,
                                  act=act, tma=tma, seed=M)[0])
    r.check(f"gemm_edge_M{M}_{int(a_mn)}{int(b_mn)}")


@pytest.mark.parametrize("N", [8, 70, 127, 128, 129, 1152, 3072])
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True)])
def test_edges_n(cuda_dev, N, a_mn, b_mn):
    r = Ratios()
    for epi, act in EDGE_EPIS:
        out_bf16, mode, tma = EPILOGUES[epi]
        r.put(epi, run_case(cuda_dev, M=129, N=N, K=136, a_mn=a_mn, b_mn=b_mn, out_bf16=out_bf16, mode=mode,
                                  act=act, tma=tma, seed=N)[0])
    r.check(f"gemm_edge_N{N}_{int(a_mn)}{int(b_mn)}")


@pytest.mark.parametrize("K", [8, 56, 64, 72, 136, 3072])
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (True, False)])
def test_edges_k(cuda_dev, K, a_mn, b_mn):
    r = Ratios()
    for epi, act in EDGE_EPIS:
        out_bf16, mode, tma = EPILOGUES[epi]
        r.put(epi, run_case(cuda_dev, M=129, N=136, K=K, a_mn=a_mn, b_mn=b_mn, out_bf16=out_bf16, mode=mode,
                                  act=act, tma=tma, seed=K)[0])
    r.check(f"gemm_edge_K{K}_{int(a_mn)}{int(b_mn)}")


@pytest.mark.parametrize("which", range(5))
def test_tile_counts_around_sm_count(cuda_dev, which):
    """M x N tiles around the persistent grid: the second MMA warpgroup of a CTA with no tile, or one fewer"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    tiles = [1, sms - 1, sms, sms + 1, 2 * sms + 1][which]
    r = Ratios()
    for epi in ("tma_f32_reduce_add", "reg_bf16_store"):
        out_bf16, mode, tma = EPILOGUES[epi]
        r.put(epi, run_case(cuda_dev, M=128 * tiles - 5, N=128, K=72, out_bf16=out_bf16, mode=mode, act=1,
                                  tma=tma, seed=tiles)[0])
    r.check(f"gemm_tiles_{tiles}")


# ================================================================================================
# 3. value regimes
# ================================================================================================
@pytest.mark.parametrize("vals", ["cancel", "huge", "tiny", "bias_cancel"])
@pytest.mark.parametrize("epi", ["tma_f32_store", "tma_bf16_store", "tma_f32_reduce_add", "reg_f32_residual",
                                 "reg_bf16_store"])
def test_value_regimes(cuda_dev, vals, epi):
    out_bf16, mode, tma = EPILOGUES[epi]
    r = Ratios()
    for act in (0, 1, 2):
        for K in (136, 1032):
            r.put(f"act{act}", run_case(cuda_dev, M=257, N=136, K=K, out_bf16=out_bf16, mode=mode, act=act,
                                              tma=tma, vals=vals, seed=K + act)[0])
    r.check(f"gemm_vals_{vals}_{epi}")


def test_subnormal_handling_measured(cuda_dev):
    """wgmma's handling of subnormals is undocumented: measure whether fp32-subnormal products (bf16 2^-70 x 2^-70)
    and bf16-subnormal inputs (2^-130 x 1) survive, and record it.  Either way the result must be within the bars'
    (K + 2) 2^-126 absolute term."""
    dev, M, N, K = cuda_dev, 128, 128, 64
    a = torch.zeros(1, M, K, device=dev)
    b = torch.zeros(1, N, K, device=dev)
    a[0, :, 0] = 2.0 ** -70 * torch.arange(M, device=dev).remainder(7).add(1)
    a[0, :, 1] = 2.0 ** -130 * torch.arange(M, device=dev).remainder(5).add(1)
    b[0, :64, 0] = 2.0 ** -70  # columns < 64: one product k 2^-140, an fp32 subnormal
    b[0, 64:, 1] = 1.0         # columns >= 64: one bf16-subnormal input times 1
    out = Output(1, M, N, torch.float32, dev, N + 8)
    A, B = Operand(a, False, dev), Operand(b, False, dev)
    lib = _lib()
    lib.check(lib.load().stego_gemm_bf16(A.ptr, A.ld, 0, B.ptr, B.ld, 0, M, N, K, out.ptr, out.ldo, 0, 0, 0, 0, 0, 0,
                                         1, 0, lib.stream()), "stego_gemm_bf16")
    torch.cuda.synchronize()
    got = out.get()[0].double()
    want = A.vals[0] @ B.vals[0].t()
    assert bool((want != 0).all())
    record("gemm_subnormals", dict(subnormal_products_kept=bool((got[:, :64] == want[:, :64]).all()),
                                   subnormal_products_zero=bool((got[:, :64] == 0).all()),
                                   subnormal_inputs_kept=bool((got[:, 64:] == want[:, 64:]).all()),
                                   subnormal_inputs_zero=bool((got[:, 64:] == 0).all()),
                                   max_abs_err=float((got - want).abs().max())))
    assert float((got - want).abs().max()) <= (K + 2) * R.TINY


# ================================================================================================
# 4. activations on an exact accumulator
# ================================================================================================
def _all_bf16(limit=1e4):
    """every finite bf16 value with |x| <= limit, +-0 and the subnormals included"""
    x = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(torch.bfloat16).float()
    return x[torch.isfinite(x) & (x.abs() <= limit)]


@pytest.mark.parametrize("act", [1, 2])
@pytest.mark.parametrize("out_bf16", [False, True])
@pytest.mark.parametrize("tma", [True, False])
def test_activation_sweep_exact_accumulator(cuda_dev, act, out_bf16, tma):
    """A's column 0 holds x and B's column 0 is 1, so the accumulator of every element of row i is x_i exactly; every
    x passes through all 128 column positions of a tile.  GELU: |out - gelu64(x)| <= 2^-8 |gelu64(x)| [bf16] +
    (delta + 3 u |gelu64(x)|)(1 + 2^-8 [bf16]) + 2^-126 with the delta of tests/_gemm_fp64.py, and out <= 0 for every
    x < 0.  ReLU: max(x, 0) exactly, within 2^-126 if wgmma flushes a subnormal x."""
    dev = cuda_dev
    x = _all_bf16().to(dev)
    M, N, K = x.numel(), 128, 64
    a = torch.zeros(1, M, K, device=dev)
    a[0, :, 0] = x
    b = torch.zeros(1, N, K, device=dev)
    b[0, :, 0] = 1.0
    A, B = Operand(a, False, dev), Operand(b, False, dev)
    out = Output(1, M, N, torch.bfloat16 if out_bf16 else torch.float32, dev, (N + 8) if tma else (N + 2))
    assert out.tma_expected(False, False) == tma
    out.set(torch.full((1, M, N), NAN, device=dev))
    lib = _lib()
    lib.check(lib.load().stego_gemm_bf16(A.ptr, A.ld, 0, B.ptr, B.ld, 0, M, N, K, out.ptr, out.ldo, int(out_bf16), 0,
                                         act, 0, 0, 0, 1, 0, lib.stream()), "stego_gemm_bf16")
    torch.cuda.synchronize()
    assert out.guards_intact()
    got = out.get()[0].double()
    xd = x.double().view(M, 1).expand(M, N)
    r = Ratios()
    if act == 1:
        want = R.gelu64(xd)
        neg = xd < 0
        pos_for_neg = int((got[neg] > 0).sum())
        d = R.delta_gelu(out_bf16)
        ub = R.UB if out_bf16 else 0.0
        bar = ub * want.abs() + (d + 3 * R.U * want.abs()) * (1 + ub) + R.TINY
        err = (got - want).abs()
        worst = int(err.max(1).values.argmax())
        r.add("gelu", got, want, bar)
        bad_x = x[((got > 0) & neg).any(1)]
        record(f"gemm_gelu_sweep_{'bf16' if out_bf16 else 'f32'}_{'tma' if tma else 'reg'}",
               dict(max_abs_err=float(err.max()), at_x=float(x[worst]), delta=d, ratio=r["gelu"],
                    positive_outputs_for_negative_x=pos_for_neg))
        assert pos_for_neg == 0, (pos_for_neg, "x in", float(bad_x.min()), float(bad_x.max()))
    else:
        want = torch.relu(xd)
        r.add("relu", got, want, torch.full_like(want, R.TINY))
    r.check(f"gemm_act{act}_sweep_{'bf16' if out_bf16 else 'f32'}_{'tma' if tma else 'reg'}")


# ================================================================================================
# 5. split-K
# ================================================================================================
@pytest.mark.parametrize("splits", [1, 2, 7, 20, 21, 30])
@pytest.mark.parametrize("a_mn,b_mn", [(True, True), (False, False)])
@pytest.mark.parametrize("onto", ["zero", "nonzero"])
def test_split_k(cuda_dev, splits, a_mn, b_mn, onto):
    """K = 1336: 21 k-blocks, the last one ragged; splits 1, 2, 7, num_kb - 1, num_kb and more than num_kb"""
    r = Ratios()
    for M, N in ((70, 384), (200, 136)):
        r.put(f"M{M}", run_case(cuda_dev, M=M, N=N, K=1336, a_mn=a_mn, b_mn=b_mn, mode="atomic", use_bias=False,
                                      tma=False, splits=splits, out0_zero=onto == "zero", seed=splits + M)[0])
    r.check(f"gemm_splitk_{splits}_{int(a_mn)}{int(b_mn)}_{onto}")


# ================================================================================================
# 6. batched
# ================================================================================================
BATCHED = [  # batch, M, N, K, out_bf16, act, bias, tma
    (1, 121, 121, 72, False, 0, False, False),
    (2, 129, 200, 136, True, 1, True, True),
    (7, 50, 127, 72, True, 2, True, False),
    (7, 257, 136, 56, False, 1, True, True),
    (64, 65, 70, 64, False, 0, True, False),
    (64, 33, 8, 8, True, 1, True, True),
]


@pytest.mark.parametrize("case", range(len(BATCHED)))
@pytest.mark.parametrize("a_mn,b_mn", LAYOUTS)
def test_batched(cuda_dev, case, a_mn, b_mn):
    """stego_gemm_bf16_batched: NaN in the gaps between the operands' batch entries, sentinels between the outputs',
    one bias shared by every entry; N = 127 in bf16 takes the register epilogue"""
    batch, M, N, K, out_bf16, act, use_bias, tma = BATCHED[case]
    r = Ratios()
    r["out"], tma_exp = run_case(cuda_dev, M=M, N=N, K=K, a_mn=a_mn, b_mn=b_mn, out_bf16=out_bf16, act=act,
                                 use_bias=use_bias, tma=tma, batch=batch, batched_api=True, seed=case)
    assert tma_exp == (tma and (N * (2 if out_bf16 else 4)) % 16 == 0)
    r.check(f"gemm_batched_{case}_{int(a_mn)}{int(b_mn)}")


# ================================================================================================
# 7. refused calls leave out untouched
# ================================================================================================
@pytest.mark.parametrize("name", sorted(REFUSED))
def test_refused_calls_leave_out_untouched(cuda_dev, name):
    rc, before, after, word = refused_call(name, cuda_dev)
    assert rc != 0, name
    assert word in _lib().last_error(), _lib().last_error()
    assert _same_bits(before, after)


# ================================================================================================
# 8. which kernel each instantiation case runs (torch.profiler in a child process)
# ================================================================================================
def _kernel_cases(dev):
    cases = {}
    for a_mn, b_mn in LAYOUTS:
        for epi, (out_bf16, mode, tma) in EPILOGUES.items():
            launch, out, tma_exp = run_case(dev, **INST, a_mn=a_mn, b_mn=b_mn, out_bf16=out_bf16, mode=mode, act=1,
                                            tma=tma, launch_only=True)
            want = (5 if tma_exp else 6, a_mn, b_mn, tma_exp)
            cases[f"{int(a_mn)}{int(b_mn)}_{epi}"] = (lambda launch=launch, out=out: launch(out), want)
    return cases


def _template_args(name):
    """gemm_bf16_kernel<stages, A_MN, B_MN, TMA> of a demangled kernel name, as (int, bool, bool, bool), or None"""
    if "gemm_bf16_kernel<" not in name:
        return None
    args = [s.strip() for s in name.split("gemm_bf16_kernel<", 1)[1].split(">", 1)[0].split(",")]
    flag = lambda s: s in ("true", "1", "(bool)1")
    return (int(args[0]), flag(args[1]), flag(args[2]), flag(args[3]))


def test_intended_kernels_ran(cuda_dev):
    """Shape and pointers pick the instantiation: profile every instantiation case and check it launched exactly the
    gemm_bf16_kernel<stages, A_MN, B_MN, TMA> it claims (5 stages with the TMA epilogue's staging, 6 without)."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    res = subprocess.run([sys.executable, os.path.abspath(__file__), "--kernel-names"], cwd=root, capture_output=True,
                         text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-4000:]
    got = json.loads(res.stdout.strip().splitlines()[-1])
    assert len(got) == len(LAYOUTS) * len(EPILOGUES)
    for case, (want, ran) in got.items():
        assert ran == [want], (case, want, ran)


if __name__ == "__main__" and sys.argv[1:] == ["--kernel-names"]:
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from torch.profiler import ProfilerActivity, profile
    dev = torch.device("cuda:0")
    for _ in range(2):  # the first sessions of a process can miss kernel records while the profiler initialises
        with profile(activities=[ProfilerActivity.CUDA]):
            torch.ones(1024, device=dev).sum().item()
    result = {}
    for case, (fn, want) in _kernel_cases(dev).items():
        fn()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        ran = [_template_args(e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        result[case] = (list(want), [list(t) for t in ran if t is not None])
    print(json.dumps(result))
