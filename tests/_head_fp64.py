"""fp64 references of the segmentation head (cluster1 + cluster2: csrc/head.cu glue around the wgmma GEMMs of
csrc/gemm.cu, driven by stego_b200/modules.py::head_forward / head_backward) and of the Adam update (adam_kernel,
p2p_adam_kernel), shared by the head tests.

Plain torch and device-agnostic: the GPU tests run these in float64 on the device and the CPU test pins them to the
oracle (oracle/stego_oracle.py), to autograd and to torch.optim.Adam.  Every reference also returns the per-element
sums of |terms| its error bar is made of; the bars themselves are derived in tests/test_head_fp64_gpu.py.

Where the kernels store bf16 the references round the same way: x = bf16(fp32(f * m)) (the product is formed in fp32
first, as dropout3_kernel does), the weights, hid = bf16(relu(x2 Wa^T + ba)), dyb = bf16(dcode) and
dhb = bf16(dh [hid > 0]).  `rnd=False` drops every one of these roundings: the exact head.
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if os.path.join(ROOT, "oracle") not in sys.path:
    sys.path.insert(0, os.path.join(ROOT, "oracle"))

U = 2.0 ** -24       # unit roundoff of fp32
UB = 2.0 ** -8        # unit roundoff of bf16 (half an ulp, relative)
D = 70                # code channels of the shipped configuration
# training shapes (images per ViT pass, feature side, feature width): M = 2 B h^2 head rows per step
SHAPES = {"c1": (32, 28, 384), "c2": (32, 40, 768), "c3": (16, 56, 768)}
DROPPED = 1.0 / 0.9   # the Dropout2d keep scale (p = 0.1)


def gamma(k):
    """gamma_k = k u / (1 - k u): the bound on k fp32 roundings in a chain (Higham, Lemma 3.1)."""
    return k * U / (1 - k * U)


def bf16(t):
    """round to bf16 (nearest even), kept in t's dtype"""
    return t.to(torch.bfloat16).to(t.dtype)


def masked(f, m, B, rnd=True):
    """Dropout2d of tokens-major features f [B*hw, E] by per-image noise m [B, E] (None: eval mode, f itself):
    bf16(fp32(f * m)) as dropout3_kernel stores it, or the exact product."""
    if m is None:
        return f.double()
    M, E = f.shape
    mm = m.reshape(B, 1, E)
    if rnd:
        x = f.float().reshape(B, M // B, E) * mm.float()
        return x.bfloat16().double().reshape(M, E)
    return (f.double().reshape(B, M // B, E) * mm.double()).reshape(M, E)


# ------------------------------------------------------------------------------------------------
# head forward
# ------------------------------------------------------------------------------------------------
def head_forward(f, m1, m2, B, w1, b1, wa=None, ba=None, wb=None, bb=None, rnd=True, hid=None):
    """code = x1 W1^T + b1 + hid Wb^T + bb with hid = relu(x2 Wa^T + ba) in float64.
    f: [M, E] tokens-major features (bf16 values); m1, m2: [B, E] noises or None (eval); weights in the parameters'
    shapes (1x1 convs or matrices); wa None is the linear head.  rnd: round where the kernels store bf16;
    hid: the kernel's own hidden activation (stage-wise: the code then depends on nothing the kernels rounded
    differently).  Returns x1, x2, pre, pre_abs (sum |x2 wa| + |ba|), hid, code, code_abs (sum of |terms| of code)
    and prop_abs (code_abs with |hid| replaced by pre_abs: what an error in the hidden layer can reach)."""
    r = bf16 if rnd else (lambda t: t)
    mat = lambda w: r(w.detach().double().reshape(w.shape[0], -1))
    x1 = masked(f, m1, B, rnd)
    W1, B1 = mat(w1), b1.detach().double()
    code = x1 @ W1.T + B1
    code_abs = x1.abs() @ W1.abs().T + B1.abs()
    out = dict(x1=x1, code=code, code_abs=code_abs, prop_abs=code_abs.clone())
    if wa is None:
        return out
    x2 = masked(f, m2, B, rnd)
    Wa, Ba, Wb, Bb = mat(wa), ba.detach().double(), mat(wb), bb.detach().double()
    pre = x2 @ Wa.T + Ba
    pre_abs = x2.abs() @ Wa.abs().T + Ba.abs()
    if hid is None:
        hid = r(torch.relu(pre))
    hid = hid.double()
    out.update(x2=x2, pre=pre, pre_abs=pre_abs, hid=hid, code=code + hid @ Wb.T + Bb,
               code_abs=code_abs + hid.abs() @ Wb.abs().T + Bb.abs(),
               prop_abs=code_abs + pre_abs @ Wb.abs().T + Bb.abs())
    return out


# ------------------------------------------------------------------------------------------------
# head backward
# ------------------------------------------------------------------------------------------------
def head_backward(dcode, x1, x2=None, hid=None, wb=None, d=D, rnd=True, dh=None):
    """The six parameter gradients from d(code) [M, >= d] in float64, with the |term| sums of each.
    x1, x2, hid: the GEMM operands the forward stored; wb [>= d, E]: the bf16 operand copy of cluster2's second conv
    (None with hid None: linear head).  dyb = bf16(dcode[:, :d]) zero padded to 128 columns; db = column sums of
    dcode over all its columns (fp32 input, not rounded); dh = dyb Wb; dhb = bf16(dh [hid > 0]).  dh: the kernel's
    own fp32 d(hidden) (stage-wise) instead of the exact one.  rnd=False drops the two bf16 roundings.
    Also dba_unrounded: the column sums of the fp32 dh [hid > 0] before its bf16 storage."""
    r = bf16 if rnd else (lambda t: t)
    dbl = lambda t: None if t is None else t.double()
    dc, x1, x2, hid, dh = dbl(dcode), dbl(x1), dbl(x2), dbl(hid), dbl(dh)
    wb = None if wb is None else wb.double()[:d]
    M = dc.shape[0]
    dy = r(dc[:, :d])
    dyb = torch.zeros(M, 128, dtype=torch.float64, device=dc.device)
    dyb[:, :d] = dy
    out = dict(dyb=dyb, db=dc.sum(0), db_abs=dc.abs().sum(0), dw1=dy.T @ x1, dw1_abs=dy.abs().T @ x1.abs())
    if hid is None:
        return out
    dh_ref = dy @ wb
    out.update(dwb=dy.T @ hid, dwb_abs=dy.abs().T @ hid.abs(), dh=dh_ref, dh_abs=dy.abs() @ wb.abs())
    if dh is None:
        dh = dh_ref
    mask = (hid > 0).double()
    dhb = r(dh * mask)
    out.update(dhb=dhb, dba=dhb.sum(0), dba_abs=dhb.abs().sum(0), dba_unrounded=(dh * mask).sum(0),
               dwa=dhb.T @ x2, dwa_abs=dhb.abs().T @ x2.abs())
    return out


# ------------------------------------------------------------------------------------------------
# input builders
# ------------------------------------------------------------------------------------------------
def head_inputs(regime, B, hw, E, d=D, nonlinear=True, seed=0, device="cpu"):
    """Features, noises and head parameters of one regime, on `device`.
    uniform   features N(0, 1) in bf16, Conv2d-default weights U(+-1/sqrt(E)), every channel kept
    outliers  as uniform, 8 feature channels at +-300 (the ViT's massive activations)
    zero_pre  as uniform, hidden units [E/4, E/4 + 32) with zero weight rows and zero bias: pre-activation exactly 0
    dropped   as uniform, Dropout2d noises with ~10 % dropped channels per image and image 1 dropped entirely
    Returns dict(f [B*hw, E] bf16, m1, m2 [B, E] fp32, w1, b1, wa, ba, wb, bb fp32 matrices / vectors)."""
    g = torch.Generator().manual_seed(seed)
    M = B * hw
    f = torch.randn(M, E, generator=g)
    if regime == "outliers":
        ch = torch.randperm(E, generator=g)[:8]
        f[:, ch] = 300.0 * torch.sign(torch.randn(M, 8, generator=g))
    f = f.bfloat16()
    k = 1.0 / E ** 0.5
    uni = lambda *s: (torch.rand(*s, generator=g) * 2 - 1) * k
    w1, b1 = uni(d, E), uni(d)
    wa, ba, wb, bb = (uni(E, E), uni(E), uni(d, E), uni(d)) if nonlinear else (None,) * 4
    if regime == "zero_pre" and nonlinear:
        band = slice(E // 4, E // 4 + 32)
        wa[band] = 0.0
        ba[band] = 0.0
    keep = torch.ones(2, B, E)
    if regime == "dropped":
        keep = (torch.rand(2, B, E, generator=g) > 0.1).float()
        keep[:, min(1, B - 1)] = 0.0
    m1, m2 = (keep * DROPPED).float()
    dev = lambda t: None if t is None else t.to(device)
    return dict(f=dev(f), m1=dev(m1), m2=dev(m2), w1=dev(w1), b1=dev(b1), wa=dev(wa), ba=dev(ba), wb=dev(wb),
                bb=dev(bb))


def bf16_ties(x):
    """fp32 values exactly halfway between x's bf16 rounding and the next bf16 number up (round-to-nearest-even must
    pick the even one)."""
    b = x.float().bfloat16()
    nxt = (b.view(torch.int16) + 1).view(torch.bfloat16)
    return (b.float() + nxt.float()) / 2


def dcode_inputs(kind, B, h, w, P, d=D, seed=0, device="cpu", fs=11, ncalls=7):
    """d(code) [B*h*w, P] fp32 (columns >= d zero, as the loss backward leaves its padding).
    dense   N(0, 1e-3), with an eighth of the entries at exact bf16 ties
    sparse  nonzero only at the 4 bilinear taps of fs^2 * ncalls random sample points per image (what the correspondence
            loss backward scatters), values N(0, 1e-2)
    range   dense with magnitudes 10^U(-8, 2) (six orders beyond bf16's exponent-independent 2^-8)"""
    g = torch.Generator().manual_seed(seed)
    M = B * h * w
    dc = torch.zeros(M, P)
    if kind == "sparse":
        n = fs * fs * ncalls
        for b in range(B):
            yx = torch.rand(n, 2, generator=g) * torch.tensor([h - 1.0, w - 1.0])
            y0, x0 = yx[:, 0].floor().long(), yx[:, 1].floor().long()
            y1, x1 = (y0 + 1).clamp_max(h - 1), (x0 + 1).clamp_max(w - 1)
            rows = torch.cat([y0 * w + x0, y0 * w + x1, y1 * w + x0, y1 * w + x1]) + b * h * w
            vals = torch.randn(rows.numel(), d, generator=g) * 1e-2
            dc[:, :d].index_add_(0, rows, vals)
    else:
        v = torch.randn(M, d, generator=g) * 1e-3
        if kind == "range":
            v = v.sign() * 10 ** (torch.rand(M, d, generator=g) * 10 - 8)
        tie = torch.rand(M, d, generator=g) < 0.125
        v = torch.where(tie, bf16_ties(v), v)
        dc[:, :d] = v
    return dc.to(device)


# ------------------------------------------------------------------------------------------------
# Adam
# ------------------------------------------------------------------------------------------------
def adam(p, g, m, v, step, lr, b1=0.9, b2=0.999, eps=1e-8, grad_scale=1.0):
    """One step of torch.optim.Adam's rule (no weight decay, no amsgrad) in float64 from the given state:
    returns m1, v1, upd (the amount subtracted from p), p1 and the |term| sums m_abs, v_abs of the two moments."""
    p, g, m, v = p.double(), g.double() * grad_scale, m.double(), v.double()
    m1 = b1 * m + (1 - b1) * g
    v1 = b2 * v + (1 - b2) * g * g
    upd = adam_update(m1, v1, step, lr, b1, b2, eps)
    return dict(m=m1, v=v1, upd=upd, p=p - upd, m_abs=(b1 * m).abs() + ((1 - b1) * g).abs(),
                v_abs=(b2 * v).abs() + (1 - b2) * g * g)


def adam_update(m1, v1, step, lr, b1=0.9, b2=0.999, eps=1e-8):
    """lr / (1 - b1^t) * m / (sqrt(v) / sqrt(1 - b2^t) + eps) in float64 from given moments."""
    bc1, bc2 = 1 - b1 ** step, 1 - b2 ** step
    return (lr / bc1) * m1.double() / (v1.double().sqrt() / bc2 ** 0.5 + eps)


def rank_sum_fp32(exports):
    """sum over ranks in rank order, in fp32, starting from +0 (what p2p_adam_kernel forms)"""
    acc = torch.zeros_like(exports[0], dtype=torch.float32)
    for e in exports:
        acc = acc + e.float()
    return acc
