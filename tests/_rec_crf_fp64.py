"""fp64 restatements of the training step's reconstruction and CRF terms as the hand-scheduled step computes them
(csrc/rec_loss.cu, the stego_crf_mean_* entry points of csrc/crf_loss.cu), with the magnitude sums their error bars are
built from.  Plain torch and device-agnostic: the GPU tests run them in float64 on the device; tests/test_rec_crf_step.py
pins them to oracle/stego_oracle.py::contrastive_crf_loss, to tests/golden/contrastive_crf_loss.pt and to float64
autograd through F.interpolate / F.normalize / conv2d.

  rec:  r = code W^T + b (rows), f = feat * m3, cos = <r / max(|r|, eps), f / max(|f|, eps)>, loss = -mean(cos); for
        d loss_total / d cos = dcos (the same for every pixel): dr by F.normalize's rule, dcode = dr W, dW = dr^T code,
        db = sum dr.
  crf:  v = resize(code, S) and gsel = resize(img, S) at the samples (ATen's bilinear taps, align_corners=False),
        sel = v / max(|v|, eps), out = -(<sel_a, sel_b> * s_ab), loss = mean(out); for the uniform upstream gradient
        g: d sel_a = sum_b -2 g s_ab sel_b, dv = (dsel - [|v| >= eps] sel <sel, dsel>) / max(|v|, eps), scattered back
        through the taps.
"""
import torch

from _loss_terms_fp64 import EPS32, crf_loss


# ------------------------------------------------------------------------------------------------
# reconstruction
# ------------------------------------------------------------------------------------------------
def rec_term(code, feat, m3, weight, bias, dcos, eps=EPS32):
    """code [M, D], feat [M, E], m3 [M, E] (already expanded per row) or None, weight [E, D], bias [E]; dcos a float.
    Returns cos, nr, nf, loss, dcode, dW, db and, for the bars: rabs = |W| |code| + |b| [M, E], ia, ib, rh, fh."""
    c, W, b = code.double(), weight.double(), bias.double()
    f = feat.double() * (m3.double() if m3 is not None else 1.0)
    r = c @ W.t() + b
    nr, nf = r.norm(dim=1), f.norm(dim=1)
    ia, ib = 1.0 / nr.clamp_min(eps), 1.0 / nf.clamp_min(eps)
    rh, fh = r * ia[:, None], f * ib[:, None]
    cos = (rh * fh).sum(1)
    ka = torch.where(nr >= eps, cos, torch.zeros_like(cos))
    dr = (dcos * ia)[:, None] * (fh - ka[:, None] * rh)
    return dict(r=r, f=f, cos=cos, nr=nr, nf=nf, loss=-cos.mean(), dr=dr, dcode=dr @ W, dW=dr.t() @ c, db=dr.sum(0),
                rabs=c.abs() @ W.abs().t() + b.abs(), ia=ia, ib=ib, rh=rh, fh=fh)


# ------------------------------------------------------------------------------------------------
# CRF
# ------------------------------------------------------------------------------------------------
def resize_taps(idx, in_size, out_size):
    """ATen's area_pixel_compute_source_index (align_corners=False) in float64: (i0, i1, l1) per output index"""
    s = ((idx.double() + 0.5) * (in_size / out_size) - 0.5).clamp_min(0)
    i0 = s.floor().long().clamp_max(in_size - 1)
    i1 = torch.where(i0 < in_size - 1, i0 + 1, i0)
    return i0, i1, s - i0.double()


def sample_resized(t, coords, S):
    """resize(t, S)[:, :, ys, xs] in float64 for t [B, C, H, W]: [B, C, n], and the taps"""
    t = t.double()
    H, W = t.shape[-2:]
    y0, y1, ly = resize_taps(coords[0], H, S)
    x0, x1, lx = resize_taps(coords[1], W, S)
    v = ((1 - ly) * ((1 - lx) * t[:, :, y0, x0] + lx * t[:, :, y0, x1]) +
         ly * ((1 - lx) * t[:, :, y1, x0] + lx * t[:, :, y1, x1]))
    return v, (y0, y1, ly, x0, x1, lx)


def crf_term(img, code, coords, params, weight, S=56, eps=EPS32):
    """img [B, 3, H, W], code [B, C, h, w], coords int64 [2, n] on the S x S maps, params the fp32 kernel parameters,
    weight the term's weight.  Returns loss, out [B, n, n], sel, nv, dsel, dcode (of weight * loss) and, for the bars,
    crf_loss's dict (ref) and |out| summed (out_abs)."""
    gsel, _ = sample_resized(img, coords, S)
    v, (y0, y1, ly, x0, x1, lx) = sample_resized(code, coords, S)
    nv = v.norm(dim=1)
    sel = v / nv.clamp_min(eps)[:, None]
    ys, xs = coords[0], coords[1]
    # crf_loss reads guidance / clusters at (ys, xs): hand it the sampled values on an n x 1 "map" with identity coords
    n = coords.shape[1]
    ref = crf_loss(gsel[..., None], sel[..., None], torch.stack([torch.arange(n, device=ys.device), torch.zeros_like(ys)]),
                   *params)
    # crf_loss's position differences come from the identity coords: recompute s with the real positions
    alpha, beta, gamma_, w1, w2, shift = params
    dpos = ((ys[:, None] - ys[None, :]) ** 2 + (xs[:, None] - xs[None, :]) ** 2).double()[None]
    s = w1 * torch.exp(-dpos / (2 * alpha) - ref["tg"]) + w2 * torch.exp(-dpos / (2 * gamma_)) - shift
    out = -(ref["G"] * s)
    B = img.shape[0]
    g = weight / (B * n * n)
    Wm = -2 * g * s
    dsel = torch.einsum("zab,zkb->zka", Wm, sel)
    k = torch.where(nv >= eps, (sel * dsel).sum(1), torch.zeros_like(nv))
    dv = (dsel - sel * k[:, None]) / nv.clamp_min(eps)[:, None]
    Bc, C, h, w = code.shape
    dcode = torch.zeros(Bc, C, h * w, dtype=torch.float64, device=code.device)
    for yi, xi, wt in ((y0, x0, (1 - ly) * (1 - lx)), (y0, x1, (1 - ly) * lx), (y1, x0, ly * (1 - lx)), (y1, x1, ly * lx)):
        dcode.index_add_(2, yi * w + xi, dv * wt)
    return dict(loss=out.mean(), out=out, s=s, G=ref["G"], absG=ref["absG"], sel=sel, v=v, nv=nv, gsel=gsel, dsel=dsel,
                dsel_abs=torch.einsum("zab,zkb->zka", Wm.abs(), sel.abs()), dv=dv, dcode=dcode.view(Bc, C, h, w),
                out_abs=out.abs().sum(), g=g)
