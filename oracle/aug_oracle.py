"""Oracle of the aug-alignment views (img_aug, coord_aug).  TEST INFRASTRUCTURE ONLY.

`reference_views` restates src/data.py:527-563 for one sample (the lines that build img_aug / coord_aug) with the
transforms of src/train_segmentation.py:408-416, run by the installed torchvision on CPU tensors.  The reference pins
torchvision 0.8.2, whose tensor resize has no antialiasing; that release is not what runs here, and the installed one is
the oracle, as the installed torch is for every torch op.

`views_fp64` is the same arithmetic in float64 on given parameters (stego_b200.augment.draw_params): the crop box, the
factors, the Gaussian weights and the resize's tap centres are the fp32 values the views are built from, and every
operation after them is exact to fp64.  It is what
the GPU tests measure the kernel's error against.
"""
from __future__ import annotations

import math
import random

import torch
import torch.nn.functional as F
import torchvision.transforms as T

Tensor = torch.Tensor
GRAY_W = [float(torch.tensor(w, dtype=torch.float32)) for w in (0.2989, 0.587, 0.114)]  # the fp32 constants torch uses


def transforms(size: int):
    """train_segmentation.py:408-416."""
    geometric = T.Compose([T.RandomHorizontalFlip(), T.RandomResizedCrop(size=size, scale=(0.8, 1.0))])
    photometric = T.Compose([T.ColorJitter(brightness=.3, contrast=.3, saturation=.3, hue=.1), T.RandomGrayscale(.2),
                             T.RandomApply([T.GaussianBlur((5, 5))])])
    return geometric, photometric


def reference_views(img: Tensor, seed: int, size: int):
    """data.py:538-563 for pack[0] = img ([3, H, W] fp32, CPU): (img_aug [3, size, size], coord_aug [size, size, 2]).
    Seeds torch like data.py:533-535 (torch.manual_seed also reseeds CUDA: callers on a GPU machine fork it)."""
    geometric, photometric = transforms(size)

    def set_seed(s):  # data.py:533-535
        random.seed(s)
        torch.manual_seed(s)

    set_seed(seed)
    coord_entries = torch.meshgrid([torch.linspace(-1, 1, img.shape[1]), torch.linspace(-1, 1, img.shape[2])],
                                   indexing="ij")
    coord = torch.cat([t.unsqueeze(0) for t in coord_entries], 0)
    img_aug = photometric(geometric(img))
    set_seed(seed)
    coord_aug = geometric(coord)
    return img_aug, coord_aug.permute(1, 2, 0)


def _f32(x: float) -> float:
    return float(torch.tensor(x, dtype=torch.float32))


def _aa_matrix(in_size: int, out_size: int) -> Tensor:
    """[out, in] float64 weights of ATen's antialiased bilinear resize (align_corners=False) along one axis.  The scale,
    each tap centre and the inverse scale are the fp32 values ATen forms (their rounding moves a centre by up to
    2^-24 in_size pixels, which is not an arithmetic error of the filter); the weights and their sum are exact to fp64."""
    scale = _f32(in_size / out_size)
    support = max(scale, 1.0)
    invscale = _f32(1.0 / scale) if scale >= 1.0 else 1.0
    m = torch.zeros(out_size, in_size, dtype=torch.float64)
    for o in range(out_size):
        center = _f32(scale * (o + 0.5))
        lo = max(int(center - support + 0.5), 0)
        hi = min(int(center + support + 0.5), in_size)
        w = [max(0.0, 1.0 - abs((k - center + 0.5) * invscale)) for k in range(lo, hi)]
        t = sum(w)
        m[o, lo:hi] = torch.tensor(w, dtype=torch.float64) / (t if t != 0 else 1.0)
    return m


def geometry_fp64(x: Tensor, p: dict, size: int) -> Tensor:
    """hflip, crop (on the flipped frame) and the antialiased resize of [C, H, W] in float64.  torchvision returns an
    already [size, size] crop unchanged, which these weights reproduce (they are the identity there)."""
    x = x.double()
    if p["flip"]:
        x = x.flip(-1)
    top, left, h, w = p["crop"]
    x = x[:, top:top + h, left:left + w]
    return torch.einsum("oh,chw,pw->cop", _aa_matrix(h, size), x, _aa_matrix(w, size))


def gray(x: Tensor) -> Tensor:
    return GRAY_W[0] * x[0] + GRAY_W[1] * x[1] + GRAY_W[2] * x[2]


def _blend(a, b, ratio: float) -> Tensor:
    r = float(torch.tensor(ratio, dtype=torch.float32))
    return (r * a + (1.0 - r) * b).clamp(0, 1)


def rgb2hsv(x: Tensor):
    """_functional_tensor._rgb2hsv in float64: (h, s, v, maxc == minc)."""
    r, g, b = x
    maxc, minc = x.max(0).values, x.min(0).values
    eqc = maxc == minc
    cr = maxc - minc
    ones = torch.ones_like(maxc)
    s = cr / torch.where(eqc, ones, maxc)
    crd = torch.where(eqc, ones, cr)
    rc, gc, bc = (maxc - r) / crd, (maxc - g) / crd, (maxc - b) / crd
    hr = (maxc == r) * (bc - gc)
    hg = ((maxc == g) & (maxc != r)) * (2.0 + rc - bc)
    hb = ((maxc != g) & (maxc != r)) * (4.0 + gc - rc)
    h = torch.fmod((hr + hg + hb) / 6.0 + 1.0, 1.0)
    return h, s, maxc, eqc


def hsv2rgb(h, s, v, sector=None) -> Tensor:
    """_functional_tensor._hsv2rgb in float64 (the einsum's 0 / 1 mask makes any NaN candidate poison all three).
    sector(i, f) -> (i, f) may replace the sector index and fraction (the tests evaluate the other side of an edge)."""
    i = torch.floor(h * 6.0)
    f = h * 6.0 - i
    i = i.to(torch.int64)
    if sector is not None:
        i, f = sector(i, f)
    i = i % 6
    p = torch.clamp(v * (1.0 - s), 0.0, 1.0)
    q = torch.clamp(v * (1.0 - s * f), 0.0, 1.0)
    t = torch.clamp(v * (1.0 - s * (1.0 - f)), 0.0, 1.0)
    a = torch.stack([torch.stack(c) for c in ((v, q, p, p, t, v), (t, v, v, q, p, p), (p, p, t, v, v, q))])
    out = a.gather(1, i.expand(3, 1, *i.shape)).squeeze(1)
    bad = torch.isnan(p) | torch.isnan(q) | torch.isnan(t)
    return torch.where(bad, torch.full_like(out, float("nan")), out)


def adjust_hue(x: Tensor, factor: float, sector=None) -> Tensor:
    h, s, v, _ = rgb2hsv(x)
    h = torch.remainder(h + float(torch.tensor(factor, dtype=torch.float32)), 1.0)
    return hsv2rgb(h, s, v, sector)


def photometric_fp64(x: Tensor, p: dict, weights: Tensor = None, probe=None, sector=None) -> Tensor:
    """ColorJitter in fn_idx order, grayscale, blur on a float64 [3, size, size]; `probe(x, op)` sees the input of
    every op (the tests measure how close it lies to a branch boundary); `sector` goes to hsv2rgb."""
    for op in p["fn_idx"]:
        if probe is not None:
            probe(x, op)
        if op == 0:
            x = _blend(x, torch.zeros_like(x), p["brightness"])
        elif op == 1:
            x = _blend(x, gray(x).mean(), p["contrast"])
        elif op == 2:
            x = _blend(x, gray(x).expand_as(x), p["saturation"])
        else:
            x = adjust_hue(x, p["hue"], sector)
    if p["gray"]:
        x = gray(x).expand_as(x).clone()
    if p["blur"]:
        k = weights.double().view(1, 1, 5, 5).expand(3, 1, 5, 5)
        x = F.conv2d(F.pad(x[None], [2, 2, 2, 2], mode="reflect"), k, groups=3)[0]
    return x


def views_fp64(img: Tensor, p: dict, size: int, weights: Tensor = None, probe=None, sector=None):
    """(img_aug [3, size, size], coord_aug [size, size, 2]) in float64 for one sample and its drawn parameters."""
    H, W = img.shape[1], img.shape[2]
    ly = torch.tensor([-1 + 2 * k / (H - 1) if H > 1 else -1.0 for k in range(H)], dtype=torch.float64)
    lx = torch.tensor([-1 + 2 * k / (W - 1) if W > 1 else -1.0 for k in range(W)], dtype=torch.float64)
    coord = torch.stack([ly[:, None].expand(H, W), lx[None, :].expand(H, W)])
    x = photometric_fp64(geometry_fp64(img, p, size), p, weights, probe, sector)
    return x, geometry_fp64(coord, p, size).permute(1, 2, 0)


def max_taps(in_size: int, size: int) -> int:
    """Most taps one output sample of the resize reads along an axis."""
    return 2 * math.ceil(max(in_size / size, 1.0)) + 1
