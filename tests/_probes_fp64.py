"""fp64 references of the probe and eval-frame kernels (csrc/probes.cu, csrc/eval_probes.cu), shared by the probe tests.

Plain torch and device-agnostic: the GPU tests run these in float64 on the device, image by image (and band by band
of output rows for the 1024 x 2048 eval frame), and the CPU test pins them to the oracle (oracle/stego_oracle.py) and
to autograd.  Every reference also returns the per-element sums of |terms| its error bar is made of; the bars
themselves are derived in tests/test_probes_fp64_gpu.py.

Bilinear upsampling (align_corners=False) is written out as four gathered corners with separable weights, so that a
band of output rows can be evaluated alone and the corners are at hand for the bars.  The source coordinate is
s = scale (d + 0.5) - 0.5 with scale = in / out in double, as F.interpolate computes it in fp64; the kernels compute
scale in fp32.  `lam_err` gives, per output coordinate, how far the kernels' fp32 weight (with or without a contracted
FMA) is from the double one: 0 when in / out is a power of two (every c1-c4 shape), ~1e-7 otherwise.
"""
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if os.path.join(ROOT, "oracle") not in sys.path:
    sys.path.insert(0, os.path.join(ROOT, "oracle"))

U = 2.0 ** -24                 # unit roundoff of fp32
LOGF_ABS = 3 * 2.0 ** -22      # __logf: 2^-21.41 absolute on [0.5, 2], else 3 ulp of a result <= ln 32 < 4
DIM, NCLS = 70, 27             # code channels and label classes of the shipped configuration
# training shapes (batch, low-res side, label side) and the eval frame (batch, h, w, H, W)
TRAIN = {"c1": (32, 28, 224), "c2": (32, 40, 320), "c3": (16, 56, 448)}
EVAL_C4 = (4, 128, 256, 1024, 2048)


# ------------------------------------------------------------------------------------------------
# bilinear upsampling by corners
# ------------------------------------------------------------------------------------------------
def _src(n_in, n_out, dtype, fma=True):
    """ATen area_pixel_compute_source_index (align_corners=False, clamped at 0) with scale = n_in / n_out in `dtype`.
    fp32: the product and the subtraction rounded separately, or contracted into one FMA."""
    d = torch.arange(n_out, dtype=torch.float64) + 0.5
    if dtype == torch.float64:
        s = (n_in / n_out) * d - 0.5
    else:
        sc = torch.tensor(float(n_in), dtype=torch.float32) / torch.tensor(float(n_out), dtype=torch.float32)
        if fma:  # exact product of two fp32 numbers in fp64, one rounding
            s = (sc.double() * d - 0.5).float().double()
        else:
            s = ((sc * d.float()).float() - 0.5).double()
    return s.clamp_min(0.0)


def axis(n_in, n_out, device="cpu"):
    """(i0, i1, lam, lam_err) for one axis: lam in double as F.interpolate's fp64 path; lam_err = the largest distance
    of the kernels' fp32 lam from it."""
    s = _src(n_in, n_out, torch.float64)
    i0 = s.floor().long().clamp_max(n_in - 1)
    i1 = torch.where(i0 < n_in - 1, i0 + 1, i0)
    lam = s - i0
    err = torch.zeros_like(lam)
    for fma in (True, False):
        s32 = _src(n_in, n_out, torch.float32, fma)
        j0 = s32.floor().long().clamp_max(n_in - 1)
        l32 = s32 - j0
        # a rounding that crosses an integer moves the pair of corners, not the value: lam 1 at i0 == lam 0 at i0 + 1
        l32 = torch.where(j0 != i0, l32 + (j0 - i0).double(), l32)
        err = torch.maximum(err, (l32 - lam).abs())
    return tuple(t.to(device) for t in (i0, i1, lam, err))


class Corners:
    """The four source pixels and weights of every output pixel of rows [y0, y1) of an H x W upsampling of h x w."""

    def __init__(self, h, w, H, W, device, rows=None):
        ya, xa = axis(h, H, device), axis(w, W, device)
        if rows is not None:
            ya = tuple(t[rows[0]:rows[1]] for t in ya)
        y0, y1, ly, ey = ya
        x0, x1, lx, ex = xa
        self.shape = (len(y0), W)
        self.idx = [(y0[:, None] * w + x0[None, :]).reshape(-1), (y0[:, None] * w + x1[None, :]).reshape(-1),
                    (y1[:, None] * w + x0[None, :]).reshape(-1), (y1[:, None] * w + x1[None, :]).reshape(-1)]
        ly, lx = ly[:, None], lx[None, :]
        self.wt = [((1 - ly) * (1 - lx)).reshape(-1), ((1 - ly) * lx).reshape(-1), (ly * (1 - lx)).reshape(-1),
                   (ly * lx).reshape(-1)]
        self.ey, self.ex = ey[:, None].expand(self.shape).reshape(-1), ex[None, :].expand(self.shape).reshape(-1)

    def gather(self, t):
        """t [n, h*w] -> the four corners, each [n, Hb*W]."""
        return [t.index_select(1, i) for i in self.idx]

    def interp(self, t):
        return sum(w * c for w, c in zip(self.wt, self.gather(t)))

    def wabs(self, t):
        """sum_t w_t |corner_t|: what rounding the weighted sum scales with"""
        return sum(w * c.abs() for w, c in zip(self.wt, self.gather(t)))

    def lam_term(self, t):
        """Error from the kernels' fp32 weights: e_y |bottom - top| + e_x |right - left| (corner differences)."""
        a, b, c, d = self.gather(t)
        return self.ey * torch.maximum((c - a).abs(), (d - b).abs()) + self.ex * torch.maximum((b - a).abs(), (d - c).abs())


def adjoint_into(out, cr, g, weights=None):
    """out [n, h*w] += interp^T g, with the corners' own weights or with `weights` [4][Hb*W]."""
    ws = cr.wt if weights is None else weights
    for i, w in zip(cr.idx, ws):
        out.index_add_(1, i, g * w)
    return out


def upsample(t, H, W):
    """t [n, h, w] -> [n, H, W] (fp64 corners; equals F.interpolate(bilinear, align_corners=False) in fp64)."""
    n, h, w = t.shape
    cr = Corners(h, w, H, W, t.device)
    return cr.interp(t.reshape(n, h * w).double()).view(n, H, W)


# ------------------------------------------------------------------------------------------------
# ClusterLookup (src/modules.py:134-161)
# ------------------------------------------------------------------------------------------------
def normalize_rows(t, eps=1e-12):
    return t / t.norm(dim=-1, keepdim=True).clamp_min(eps)


def cluster_ref(x, clusters, alpha, grad=1.0):
    """x [B, C, P] pixels (any dtype and device), clusters [n, C].  fp64:
      ip [B, n, P], S = sum_c |x_hat_c| |c_hat_kc| [B, n, P], argmax (first maximum), probs / logp [B, n, P] (alpha given),
      loss = -mean_p sum_k probs_k ip_k, dip [B, n, P] = d(sum_k probs_k ip_k) / d ip (argmax held fixed for alpha=None),
      dnc [n, C] = d(grad * loss) / d(normalised clusters), dcl [n, C] = d(grad * loss) / d clusters."""
    xd, cd = x.double(), clusters.double()
    B, C, P = xd.shape
    xh = xd / xd.norm(dim=1, keepdim=True).clamp_min(1e-12)
    ch = normalize_rows(cd)
    ip = torch.einsum("kc,bcp->bkp", ch, xh)
    S = torch.einsum("kc,bcp->bkp", ch.abs(), xh.abs())
    arg = ip.argmax(1)
    n = cd.shape[0]
    out = dict(ip=ip, S=S, arg=arg, xh=xh, ch=ch)
    if alpha is None:
        probs = F.one_hot(arg, n).permute(0, 2, 1).double()
        dip = probs
    else:
        logp = torch.log_softmax(alpha * ip, 1)
        probs = logp.exp()
        dotp = (probs * ip).sum(1, keepdim=True)
        dip = probs + alpha * probs * (ip - dotp)
        out["logp"] = logp
    out["probs"], out["dip"] = probs, dip
    out["loss"] = -(probs * ip).sum(1).mean()
    gs = -grad / (B * P)
    out["gs"] = gs
    dnc = gs * torch.einsum("bkp,bcp->kc", dip, xh)
    out["dnc"] = dnc
    out["dcl"] = normalize_bwd(cd, dnc)
    return out


def normalize_bwd(c, g, eps=1e-12):
    """d/dc of F.normalize(c, dim=1) applied to g (row-wise); below eps the clamp makes it g / eps."""
    nrm = c.norm(dim=1, keepdim=True)
    ch = c / nrm.clamp_min(eps)
    full = (g - ch * (ch * g).sum(1, keepdim=True)) / nrm.clamp_min(eps)
    return torch.where(nrm > eps, full, g / eps)


# ------------------------------------------------------------------------------------------------
# linear probe + bilinear upsample + masked CE (src/train_segmentation.py:210-218)
# ------------------------------------------------------------------------------------------------
def linear_ce_ref(code, weight, bias, label, n, grad=1.0):
    """code [B, C, h, w], weight [n, C], bias [n], label [B, H, W] (ignored: outside [0, n)).  fp64, image by image.
    Returns loss (NaN without a valid pixel, like the reference), count, dW, db, the low-res logits l [B, n, h*w] and
    logit gradient dl (= interp^T (softmax - onehot), unnormalised), and per image the quantities the bars use:
      Ml = |b| + sum_c |W x| per low-res logit, and per valid output pixel z, the CE value, E-independent sums."""
    B, C, h, w = code.shape
    H, W = label.shape[-2:]
    dev = code.device
    Wd, bd = weight.double().reshape(n, C), bias.double()
    cr = Corners(h, w, H, W, dev)
    tot, cnt = torch.zeros((), dtype=torch.float64, device=dev), 0
    dl = torch.zeros(B, n, h * w, dtype=torch.float64, device=dev)
    per = []
    for b in range(B):
        x = code[b].double().reshape(C, h * w)
        l = Wd @ x + bd[:, None]
        Ml = bd.abs()[:, None] + Wd.abs() @ x.abs()
        z = cr.interp(l)
        lab = label[b].reshape(-1).long()
        valid = (lab >= 0) & (lab < n)
        lse = torch.logsumexp(z, 0)
        li = lab.clamp(0, n - 1)
        zl = z.gather(0, li[None])[0]
        ce = (lse - zl)[valid]
        tot = tot + ce.sum()
        cnt += int(valid.sum())
        p = torch.softmax(z, 0)
        g = (p - F.one_hot(li, n).t().double()) * valid[None].double()
        adjoint_into(dl[b], cr, g)
        per.append(dict(l=l, Ml=Ml, z=z, p=p, valid=valid, lab=li, ce=lse - zl, lse=lse, g=g))
    loss = tot / cnt if cnt > 0 else torch.tensor(float("nan"), dtype=torch.float64, device=dev)
    s = grad / cnt if cnt > 0 else 0.0
    X = code.double().reshape(B, C, h * w)
    dW = s * torch.einsum("bkr,bcr->kc", dl, X)
    db = s * dl.sum((0, 2))
    return dict(loss=loss, count=cnt, dW=dW, db=db, dl=dl, s=s, per=per, corners=cr)


# ------------------------------------------------------------------------------------------------
# eval frame (src/eval_segmentation.py:124-131 + src/utils.py:219-229)
# ------------------------------------------------------------------------------------------------
def tta_code(code, code_flipped):
    """(code + code_flipped.flip(3)) / 2 in fp64, or the code itself."""
    x = code.double()
    return x if code_flipped is None else (x + code_flipped.double().flip(3)) / 2


def eval_band(xbar, weight, bias, clusters, alpha, H, W, rows):
    """One image's log-probs for output rows [rows[0], rows[1]) by the reference op sequence in fp64:
    F.interpolate of the (TTA-averaged) code xbar [C, h, w] -> 1x1 conv / log_softmax, and ClusterLookup log-probs
    (normalise the upsampled code and the centroids, alpha * cosine, log_softmax).  Also returns what the bars need:
    the corners of the low-res logits and centroid dots, |v| and sum_t w_t |x_t| (norms of the corner codes)."""
    C, h, w = xbar.shape
    cr = Corners(h, w, H, W, xbar.device, rows)
    x = xbar.reshape(C, h * w)
    Wd, bd = weight.double().reshape(-1, C), bias.double()
    ch = normalize_rows(clusters.double())
    l = Wd @ x + bd[:, None]
    v = cr.interp(x)                                      # the upsampled code [C, band]
    z = Wd @ v + bd[:, None]
    vn = v.norm(dim=0)
    cos = (ch @ v) / vn.clamp_min(1e-12)
    xn = x.norm(dim=0, keepdim=True)
    return dict(corners=cr, l=l, Ml=bd.abs()[:, None] + Wd.abs() @ x.abs(), z=z, lin_logp=torch.log_softmax(z, 0),
                dc=ch @ x, Mdc=ch.abs() @ x.abs(), vnorm=vn, cos=cos, clu_logp=torch.log_softmax(alpha * cos, 0),
                wxn=cr.interp(xn)[0], wabs_x=cr.wabs(x), ch=ch)


def confusion(pred, label, n_pred, n_cls):
    """UnsupervisedMetrics.update (src/utils.py:219-229) as [n_pred, n_cls] counts: pixels with 0 <= label < n_cls
    and 0 <= pred < n_cls (extra clusters are dropped, as the reference's mask does)."""
    a, p = label.reshape(-1).long(), pred.reshape(-1).long()
    m = (a >= 0) & (a < n_cls) & (p >= 0) & (p < n_cls)
    out = torch.zeros(n_pred, n_cls, dtype=torch.int64, device=pred.device)
    out.index_put_((p[m], a[m]), torch.ones_like(p[m]), accumulate=True)
    return out


# ------------------------------------------------------------------------------------------------
# input builders
# ------------------------------------------------------------------------------------------------
def _gen(seed, device):
    return torch.Generator(device=device).manual_seed(seed)


def cluster_inputs(regime, B, C, P, n, seed=0, device="cpu"):
    """(x [B, C, P] fp32, clusters [n, C] fp32) for one regime:
      random   : Gaussian code and centroids
      sharp    : every pixel within ~1e-2 of a centroid (cosine ~0.99 to it): with alpha 50 the softmax saturates
      ties     : centroid 1 duplicates centroid 0; centroids 2 and 3 have the same small-integer values on disjoint
                 channels 0-9 and 10-19, pixels of the first half are near centroid 0 (exact fp32 tie between 0 and 1),
                 the second half are symmetric in channels 0-9 / 10-19 (exact tie between 2 and 3): the lower index wins
      zeros    : random, with every 7th pixel all zero (the normalise clamp: all inner products 0, argmax 0)
      zerorow  : random, with centroid n - 1 all zero (the nrm <= 1e-12 branch of the centroid normalise backward)"""
    g = _gen(seed, device)
    rn = lambda *s: torch.randn(*s, generator=g, device=device)
    x, cl = rn(B, C, P), rn(n, C)
    if regime == "sharp":
        k = torch.randint(0, n, (B, P), generator=g, device=device)
        x = normalize_rows(cl)[k].permute(0, 2, 1) * 3.0 + 0.03 * rn(B, C, P)
    elif regime == "ties":
        vals = torch.tensor([1.0, -2.0, 0.5, 1.0, 2.0, -1.0, 1.0, -0.5, 2.0, 1.0], device=device)
        cl[1] = cl[0]
        cl[2].zero_(); cl[3].zero_()
        cl[2, :10], cl[3, 10:20] = vals, vals
        half = P // 2
        x[:, :, :half] = normalize_rows(cl[0])[None, :, None] * 4.0 + 0.05 * x[:, :, :half]
        sym = 0.2 * rn(B, 10, P - half)
        x[:, :10, half:] = vals[None, :, None] + sym
        x[:, 10:20, half:] = vals[None, :, None] + sym
    elif regime == "zeros":
        x[:, :, ::7] = 0.0
    elif regime == "zerorow":
        cl[n - 1] = 0.0
    elif regime != "random":
        raise ValueError(regime)
    return x.float().contiguous(), cl.float().contiguous()


def linear_inputs(B, C, h, w, H, W, n, spread=4.0, label_dtype=torch.int64, ignore="random", seed=0, device="cpu"):
    """(code [B, C, h, w] fp32, weight [n, C], bias [n], label [B, H, W]).  The logits have a spread of about
    +-spread.  Labels hit n - 1 and the ignored values (-1 and n for the signed types, n and 255 for uint8).
    ignore: 'random' (about 10 % ignored), 'tiles' (whole 16 x 16 output tiles of every image ignored), 'image'
    (image 0 entirely ignored), 'all' (every pixel ignored)."""
    g = _gen(seed, device)
    code = torch.randn(B, C, h, w, generator=g, device=device)
    weight = torch.randn(n, C, generator=g, device=device) * (spread / (3.0 * C ** 0.5))
    bias = torch.randn(n, generator=g, device=device) * 0.5
    label = torch.randint(0, n, (B, H, W), generator=g, device=device)
    label[:, ::5, ::3] = n - 1
    r = torch.rand(B, H, W, generator=g, device=device)
    bad = -1 if label_dtype != torch.uint8 else 255
    label[r < 0.05] = bad
    label[(r >= 0.05) & (r < 0.1)] = n
    if ignore == "tiles":
        ty, tx = (torch.arange(H, device=device) // 16), (torch.arange(W, device=device) // 16)
        label[:, ((ty[:, None] + 2 * tx[None, :]) % 3) == 0] = bad
    elif ignore == "image":
        label[0] = bad
    elif ignore == "all":
        label[:] = bad
    elif ignore != "random":
        raise ValueError(ignore)
    return code, weight, bias, label.to(label_dtype)


def anticorrelated_code(B, C, h, w, ratio, seed=0, device="cpu"):
    """Low-res code whose odd columns nearly cancel the even column to their left: x[2j+1] = -k x[2j] + p with
    k = (1 - lam) / lam for lam = 7/16, the weight of output column 16 j + 7 at an 8x upsampling.  There v is the
    perturbation alone, |v| = ratio * sum_t w_t |x_t| (up to the vertical mix of two rows), the conditioning the
    Gram-entry norm is sensitive to.  Other output pixels see moderate cancellation."""
    g = _gen(seed, device)
    lam = 7.0 / 16.0
    k = (1 - lam) / lam
    x = torch.randn(B, C, h, w, generator=g, device=device)
    a = x[..., 0::2]
    d = torch.randn(a.shape, generator=g, device=device)
    d = d / d.norm(dim=1, keepdim=True)
    scale = ratio * 2 * (1 - lam) * a.norm(dim=1, keepdim=True) / lam   # |lam * p| = ratio * ((1 - lam) + lam k) |a|
    x[..., 1::2] = -k * a + scale * d
    return x.float().contiguous()
