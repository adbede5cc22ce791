"""fp64 reference of the wgmma GEMM (stego_gemm_bf16 / stego_gemm_bf16_batched: csrc/gemm.cu, csrc/epilogue.cuh) and
its elementwise error bars, shared by tests/test_gemm_fp64_gpu.py.

Plain torch and device-agnostic: the GPU tests run it in float64 on the device.  The reference returns
out = act(A B^T + bias) + residual together with the sums of |terms| the bars are made of.

Bars (u = 2^-24, gamma_k = k u / (1 - k u)).  The fp32 accumulation inside wgmma is not documented as IEEE
round-to-nearest; it is treated as a K-term chain (DESIGN.md section 4).  That is an assumption: the tests record the
measured err / bar ratios rather than tuning the bars to them.
  plain          gamma_{K+1} (sum |a b| + |bias|): K products and the bias add
  residual       one rounding more and |residual| in the sum: gamma_{K+2} (sum |a b| + |bias| + |r|); the TMA fp32
                 reduce-add (out += tile) is the same with r = the old out
  split-K        each split is a chain of 64 kb_per_split products, then `splits` fp32 atomics onto out's old value:
                 gamma_{64 kb_per_split + splits} (sum |a b| + |out0|); atomic_out takes no bias, act or residual
  activation     ReLU is 1-Lipschitz.  GELU multiplies the input bar by max |gelu'| = 1.1289 < 1.13 and adds its
                 approximation error delta plus 3 u |gelu| for the roundings of 0.5 x (1 + e) / h + |h| e:
                   fp32 outputs (Abramowitz-Stegun erf, rcp.approx + ex2.approx): DELTA_GELU_F32 = 1e-6, twice the
                   5e-7 an fp32 emulation of the formula with exact rcp / exp reaches;
                   bf16 outputs (degree-8 erf polynomial, e capped at 1): the fit's erf error in fp32 evaluation,
                   4.4e-5, times |h| <= 2.27 at the clamp |x| = 4.5255 gives 1.0e-4; beyond the clamp the output is
                   exactly 0 or x, within |h| erfc(|x| / sqrt 2) < 1.4e-5 of GELU.  DELTA_GELU_BF16 = 1.2e-4 keeps
                   20 % of margin over that derivation.  Neither delta grows with |x|.
  bf16 store     half an ulp of the stored value: bar_bf16 = bar_fp32 (1 + 2^-8) + 2^-8 |out|
  subnormals     wgmma's handling of subnormal products and inputs is not documented, so every bar carries
                 (K + 2) 2^-126: each product, the bias add and the residual may lose up to one smallest normal.
"""
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from _head_fp64 import U, UB, gamma  # noqa: E402,F401

GEMM_BK = 64
GELU_LIP = 1.13
DELTA_GELU_F32 = 1e-6
DELTA_GELU_BF16 = 1.2e-4
TINY = 2.0 ** -126


def gelu64(x):
    """exact (erf) GELU, nn.GELU's default, in x's dtype"""
    return 0.5 * x * (1.0 + torch.special.erf(x / math.sqrt(2.0)))


def act64(x, act):
    if act == 1:
        return gelu64(x)
    if act == 2:
        return torch.relu(x)
    return x


def delta_gelu(out_bf16):
    return DELTA_GELU_BF16 if out_bf16 else DELTA_GELU_F32


def split_plan(K, splits):
    """(kb_per_split, splits) as gemm_impl normalises them: no more splits than k-blocks, none of them empty"""
    num_kb = (K + GEMM_BK - 1) // GEMM_BK
    s = min(splits, num_kb)
    kbps = (num_kb + s - 1) // s
    return kbps, (num_kb + kbps - 1) // kbps


def reference(a, b, bias=None, act=0, residual=None, out0=None):
    """a [..., M, K], b [..., N, K] (the logical operands, bf16 values in any dtype), bias [N], residual and out0
    [..., M, N]: out = act(a b^T + bias) + residual (+ out0: the old value atomics add onto), all float64.
    Returns dict(out, pre (the activation's input), pre_abs (sum |a b| + |bias|), add_abs (|residual| + |out0|))."""
    A, B = a.double(), b.double()
    pre = A @ B.transpose(-1, -2)
    pre_abs = A.abs() @ B.abs().transpose(-1, -2)
    if bias is not None:
        pre = pre + bias.double()
        pre_abs = pre_abs + bias.double().abs()
    out = act64(pre, act)
    add_abs = torch.zeros_like(out)
    for t in (residual, out0):
        if t is not None:
            out = out + t.double()
            add_abs = add_abs + t.double().abs()
    return dict(out=out, pre=pre, pre_abs=pre_abs, add_abs=add_abs)


def bar(ref, K, act=0, out_bf16=False, added=False, splits=0):
    """Elementwise bound on |kernel - ref["out"]| (see the module docstring).
    added: a residual or reduce-add term is summed after the activation; splits > 0: the atomic split-K path with
    that requested split count (onto ref's out0)."""
    if splits:
        kbps, s = split_plan(K, splits)
        n = GEMM_BK * kbps + s
    else:
        n = K + 1 + int(added)
    lip = GELU_LIP if act == 1 else 1.0
    b = lip * (gamma(n) * (ref["pre_abs"] + ref["add_abs"]) + (K + 2) * TINY)
    if act == 1:
        b = b + delta_gelu(out_bf16) + 3 * U * ref["out"].abs()
    if out_bf16:
        b = b * (1 + UB) + UB * ref["out"].abs()
    return b


def ratio(got, want, b):
    """largest |got - want| / b (0 where the difference is 0; NaN if got has a NaN where want has none)"""
    err = (got.double() - want.double()).abs()
    if not err.numel():
        return 0.0
    return float(torch.where(err == 0, torch.zeros_like(err), err / b.double()).max())
