"""fp64 references of the optional loss terms (DESIGN.md section 9d): ContrastiveCRFLoss (csrc/crf_loss.cu) and the
per-pixel cosine of the reconstruction / augmentation-alignment terms (csrc/cosine_loss.cu), shared by the loss-term
tests, with the input builders for the regimes where those kernels can go wrong.

Plain torch and device-agnostic: the GPU tests run these in float64 on the device, the CPU test pins them to the oracle
(oracle/stego_oracle.py::contrastive_crf_loss) and to autograd through F.normalize.  Every reference also returns the
per-element sums of |terms| its error bar is built from; the bars themselves are derived in
tests/test_loss_terms_fp64_gpu.py.
"""
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if os.path.join(ROOT, "oracle") not in sys.path:
    sys.path.insert(0, os.path.join(ROOT, "oracle"))

U = 2.0 ** -24                            # unit roundoff of fp32
PARAMS = (0.5, 0.15, 0.05, 10.0, 3.0, 0.0)  # train_config.yml: alpha, beta, gamma, w1, w2, shift
EPS = 1e-10                               # F.normalize's eps in the reference's norm (modules.py:275-276)
EPS32 = float(torch.tensor(EPS, dtype=torch.float32))  # the eps the kernels compare with (a float argument)
MEAN = (0.485, 0.456, 0.406)              # ImageNet normalisation of the training images
STD = (0.229, 0.224, 0.225)


def gamma(k):
    """gamma_k = k u / (1 - k u): the bound on k fp32 roundings in a chain (Higham, Lemma 3.1)."""
    return k * U / (1 - k * U)


def f32(x):
    """the fp32 value a Python float becomes at the C ABI, as a Python float"""
    return float(torch.tensor(x, dtype=torch.float32))


def fp32_params(params):
    return tuple(f32(p) for p in params)


# ------------------------------------------------------------------------------------------------
# ContrastiveCRFLoss
# ------------------------------------------------------------------------------------------------
def crf_loss(guidance, clusters, coords, alpha, beta, gamma_, w1, w2, shift):
    """-(G * s) of ContrastiveCRFLoss in float64, with the pieces its bars need.
    guidance [B, Cg, H, W], clusters [B, C, H, W] (any dtype, taken at their values), coords int64 [2, n].
    The parameters are used as given: pass fp32_params(...) for what the kernels receive.  Returns a dict:
      out = -G s, G = <c_a, c_b>, s = w1 e1 + w2 e2 - shift, e1 = exp(t1), e2 = exp(t2) with
      t1 = -|dp|^2 / 2 alpha - |dI|^2 / 2 beta, t2 = -|dp|^2 / 2 gamma, the two parts of t1 (tp = |dp|^2 / 2 alpha,
      tg = |dI|^2 / 2 beta), absG = sum_k |c_ak c_bk|, sel = the selected code vectors [B, C, n]."""
    ys, xs = coords[0], coords[1]
    g = guidance.double()[:, :, ys, xs]
    c = clusters.double()[:, :, ys, xs]
    dpos = ((ys[:, None] - ys[None, :]) ** 2 + (xs[:, None] - xs[None, :]) ** 2).double()[None]
    dgui = (g[:, :, :, None] - g[:, :, None, :]).square().sum(1)
    tp, tg = dpos / (2 * alpha), dgui / (2 * beta)
    t1, t2 = -tp - tg, -dpos / (2 * gamma_)
    e1, e2 = torch.exp(t1), torch.exp(t2)
    s = w1 * e1 + w2 * e2 - shift
    G = torch.einsum("bka,bkc->bac", c, c)
    absG = torch.einsum("bka,bkc->bac", c.abs(), c.abs())
    return dict(out=-(G * s), G=G, s=s, e1=e1, e2=e2, t1=t1, t2=t2, tp=tp, tg=tg, absG=absG, sel=c)


def crf_loss_bwd(ref, gout, coords, shape, wbar=None):
    """The gradient of sum(gout * out) w.r.t. clusters [B, C, H, W] in float64, from crf_loss's dict:
    W_ab = -(g_ab + g_ba) s_ab, d sel_a = sum_b W_ab sel_b, scattered to the sampled pixels with repeats summed.
    Returns dclusters, dsel [B, C, n], W, the sums sum_b |W_ab| |sel_bk| [B, C, n] and, for a per-element bound wbar on
    |W_kernel - W| [B, n, n], sum_b wbar_ab |sel_bk|; `repeats` [H, W] counts the samples of each pixel."""
    g = gout.double()
    sel = ref["sel"]
    gs = g + g.transpose(1, 2)
    W = -gs * ref["s"]
    dsel = torch.einsum("zab,zkb->zka", W, sel)
    dsel_abs = torch.einsum("zab,zkb->zka", W.abs(), sel.abs())
    dsel_werr = torch.einsum("zab,zkb->zka", wbar, sel.abs()) if wbar is not None else None
    B, C, H, Wd = shape
    return dict(dclusters=scatter(dsel, coords, shape), dsel=dsel, W=W, gs=gs, dsel_abs=dsel_abs, dsel_werr=dsel_werr,
                repeats=repeats(coords, H, Wd, g.device))


def scatter(v, coords, shape):
    """v [B, C, n] summed into [B, C, H, W] at (coords[0], coords[1]) (index_put with accumulation)"""
    B, C, H, W = shape
    out = torch.zeros(B, C, H * W, dtype=v.dtype, device=v.device)
    out.index_add_(2, coords[0] * W + coords[1], v)
    return out.view(B, C, H, W)


def repeats(coords, H, W, device=None):
    r = torch.zeros(H * W, dtype=torch.long, device=device if device is not None else coords.device)
    r.index_add_(0, (coords[0] * W + coords[1]).to(r.device), torch.ones_like(coords[0], device=r.device))
    return r.view(H, W)


# ------------------------------------------------------------------------------------------------
# pixel cosine
# ------------------------------------------------------------------------------------------------
def pixel_cosine(a, b, eps=EPS32, ga=None):
    """cos = <a / max(|a|, eps), b / max(|b|, eps)> over dim 1 in float64 and, for an upstream gradient ga [B, H, W],
    both input gradients by F.normalize's rule: clamp_min passes the gradient where |a| >= eps, so
      |a| >= eps: d/da = g ia (b_hat - cos a_hat)      |a| < eps: d/da = g ia b_hat      (ia = 1 / max(|a|, eps)).
    Also returned: na, nb (the norms), ia, ib, a_hat, b_hat, absab = sum_c |a_c b_c| ([B, H, W])."""
    a, b = a.double(), b.double()
    na, nb = a.norm(dim=1), b.norm(dim=1)
    ia, ib = 1.0 / na.clamp_min(eps), 1.0 / nb.clamp_min(eps)
    ah, bh = a * ia[:, None], b * ib[:, None]
    cos = (ah * bh).sum(1)
    out = dict(cos=cos, na=na, nb=nb, ia=ia, ib=ib, ah=ah, bh=bh, absab=(a * b).abs().sum(1))
    if ga is not None:
        g = ga.double()
        ka = torch.where(na >= eps, cos, torch.zeros_like(cos))
        kb = torch.where(nb >= eps, cos, torch.zeros_like(cos))
        out["da"] = (g * ia)[:, None] * (bh - ka[:, None] * ah)
        out["db"] = (g * ib)[:, None] * (ah - kb[:, None] * bh)
    return out


# ------------------------------------------------------------------------------------------------
# input builders
# ------------------------------------------------------------------------------------------------
def resize56(t):
    return F.interpolate(t, 56, mode="bilinear", align_corners=False)


def training_inputs(B, C, gen, side=28, dev="cpu"):
    """The training regime (train_segmentation.py:201-208): guidance = resize(img, 56) of ImageNet-normalised images in
    [0, 1], clusters = norm(resize(code, 56)) of a code at the head's resolution."""
    img = torch.rand(B, 3, 224, 224, generator=gen)
    img = (img - torch.tensor(MEAN).view(1, 3, 1, 1)) / torch.tensor(STD).view(1, 3, 1, 1)
    code = torch.randn(B, C, side, side, generator=gen)
    return resize56(img).to(dev), F.normalize(resize56(code), dim=1, eps=EPS).to(dev)


def random_coords(n, H, W, gen):
    return torch.cat([torch.randint(0, H, size=[1, n], generator=gen), torch.randint(0, W, size=[1, n], generator=gen)], 0)


def coords_of(kind, n, H, W, gen):
    """all distinct (n <= H W), heavy repeats (n samples of a 4 x 4 corner), all identical, the four corners only"""
    if kind == "random":
        return random_coords(n, H, W, gen)
    if kind == "distinct":
        flat = torch.randperm(H * W, generator=gen)[:n]
        return torch.stack([flat // W, flat % W])
    if kind == "repeats":
        return random_coords(n, min(H, 4), min(W, 4), gen)
    if kind == "identical":
        return torch.tensor([[H // 2], [W // 3]]).expand(2, n).contiguous()
    if kind == "corners":
        cy, cx = torch.tensor([0, 0, H - 1, H - 1]), torch.tensor([0, W - 1, 0, W - 1])
        k = torch.randint(0, 4, (n,), generator=gen)
        return torch.stack([cy[k], cx[k]])
    raise ValueError(kind)


def onehot_codes(B, C, H, W, gen):
    """a one-hot code per pixel: G_ab is exactly 1 (same class) or exactly 0"""
    cls = torch.randint(0, C, (B, H, W), generator=gen)
    return F.one_hot(cls, C).permute(0, 3, 1, 2).float()


def dyadic_codes(B, C, H, W, gen):
    """codes in {-1, -7/8, ..., 7/8}: every product and partial sum of the Gram chain is exact in fp32 (|G| <= C, on
    a 2^-6 grid), so out = -G * fl(s) with an exact G"""
    return torch.randint(-8, 8, (B, C, H, W), generator=gen).float() / 8


def wide_codes(B, C, H, W, gen):
    """un-normalised codes whose pixels span 1e-3 ... 1e3 in magnitude"""
    scale = 10.0 ** (torch.rand(B, 1, H, W, generator=gen) * 6 - 3)
    return torch.randn(B, C, H, W, generator=gen) * scale


def upstream(kind, B, n, gen):
    """upstream gradients of the [B, n, n] output: uniform (the .mean() path), random non-symmetric, symmetric, and exactly
    antisymmetric (fl(r_ab - r_ba) = -fl(r_ba - r_ab), so g_ab + g_ba is exactly 0 and so is W)"""
    if kind == "mean":
        return torch.full((B, n, n), 1.0 / (B * n * n))
    r = torch.randn(B, n, n, generator=gen)
    if kind == "random":
        return r
    if kind == "symmetric":
        return r + r.transpose(1, 2)
    if kind == "antisymmetric":
        return r - r.transpose(1, 2)
    raise ValueError(kind)


def cosine_pairs(kind, B, C, H, W, gen):
    """a, b [B, C, H, W] for: random, nearly parallel (b = a + 1e-4 noise: b_hat - cos a_hat cancels), antiparallel,
    orthogonal (b = the component of noise orthogonal to a, computed in fp64), and disjoint one-hot (cos exactly 0)"""
    a = torch.randn(B, C, H, W, generator=gen)
    if kind == "random":
        return a, torch.randn(B, C, H, W, generator=gen) * 3
    if kind == "parallel":
        return a, (a.double() * 2 + 1e-4 * torch.randn(B, C, H, W, generator=gen).double()).float()
    if kind == "antiparallel":
        return a, (-0.5 * a.double() + 1e-5 * torch.randn(B, C, H, W, generator=gen).double()).float()
    if kind == "orthogonal":
        r = torch.randn(B, C, H, W, generator=gen).double()
        ad = a.double()
        return a, (r - (r * ad).sum(1, keepdim=True) / (ad * ad).sum(1, keepdim=True) * ad).float()
    if kind == "onehot":
        assert C >= 2
        i = torch.randint(0, C, (B, H, W), generator=gen)
        j = (i + 1 + torch.randint(0, C - 1, (B, H, W), generator=gen)) % C
        oa = F.one_hot(i, C).permute(0, 3, 1, 2).float() * 3
        ob = F.one_hot(j, C).permute(0, 3, 1, 2).float() * 0.25
        return oa, ob
    raise ValueError(kind)


def eps_vectors(C, dev="cpu"):
    """single-component vectors x e_0 at the clamp boundary, paired with b = (1, 0.5, 0, ...): x = eps exactly (the fp32
    square root of fl(x^2) is x itself, so the fp32 norm equals eps), one fp32 step below and above it, far below,
    and zero, plus magnitudes up to where the fp32 sum of squares stays finite.  Returns a, b [K, C, 1, 1] and the
    list of x."""
    e = torch.tensor(EPS32, dtype=torch.float32)
    xs = [e, torch.nextafter(e, torch.tensor(0.0)), torch.nextafter(e, torch.tensor(1.0)), e * 2 ** -10,
          torch.tensor(0.0), torch.tensor(1e18), torch.tensor(-1e19)]
    K = len(xs)
    a = torch.zeros(K, C, 1, 1)
    b = torch.zeros(K, C, 1, 1)
    for k, x in enumerate(xs):
        a[k, 0] = x
        b[k, 0] = 1.0
        if C > 1:
            b[k, 1] = 0.5
    return a.to(dev), b.to(dev), [float(x) for x in xs]
