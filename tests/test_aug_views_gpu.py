"""GPU: stego_aug_views (stego_b200.augment.aug_alignment_views) against float64 and against torchvision.

Every element of img_aug / coord_aug is compared with oracle/aug_oracle.views_fp64 on the same drawn parameters.

Bars (u = 2^-24, M = max(1, max |img|), n_x / n_y = most resize taps per output along x / y):
  - coord_aug: the resize is a positive-weight sum of linspace values in [-1, 1] (each fp32 linspace value within 2u of
    the exact one).  Each weight is within 4u relative of its exact value (triangle, sum, division), and the two nested
    sums add one rounding per tap.  So the error is at most (n_x + n_y + 12) u.
  - img_aug: the resize is the same sum on values up to M, so it is within (n_x + n_y + 12) u M.  A blend
    clamp(r a + (1 - r) b) with r <= 1.3 and |1 - r| <= .3 passes on at most 1.6 times its input error and adds
    3 u (1.3 M + .3 M) of its own.  Contrast's mean and saturation's grayscale are within one input error plus 4 u M.
    Hue writes v - cr g(h) with g in [0, 1] and cr g'(h) dh bounded by twice the input error.  So it passes on at most
    8 times the input error and adds 32 u M: the 1 / cr of its hue angle cancels against the cr that scales it.
    Grayscale passes on 1 times the error plus 3 u M, and the blur (weights >= 0 summing to 1 + 25 u) 1 times the error
    plus 27 u M.  The worst order amplifies the resize by 1.6^3 * 8 < 33.  The whole chain is therefore within
    bar = (33 (n_x + n_y + 12) + 33 * 40 + 40) u M.
  - Branches.  The clamp edges are continuous.  The hue op is not, for normalised inputs: hsv2rgb writes v unclamped
    but p, q and t clamped, so with v outside [0, 1] the two sides of a sector edge (the % 1.0 wrap is the edge between
    sectors 5 and 0) place v in different channels.  maxc == minc leaves s = 0, and any sector then gives v in one
    channel and clamp(v) in the other two.  maxc == 0 < cr gives s = inf, and the einsum turns the pixel into NaN.
    Where the float64 hue input lies within reach of such a boundary, the other branches are evaluated too (the other
    sector across the edge, v placed in each channel, NaN), and an element matches if it lies within the bar of any of
    them.  "Within reach" means dist(6h, Z) cr <= 6 bar for an edge (an input error e moves 6h by at most 6 e / cr),
    cr <= bar for maxc == minc, and |maxc| <= bar for maxc == 0.  The blur spreads a pixel's branch over its 5 x 5
    neighbourhood, and a NaN before contrast spreads over the image.  Such elements are asserted to be rare.
The same bars, doubled, hold against torchvision's own fp32 composition on the CPU: both lie within the bar of fp64.
"""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import aug_oracle as AO  # noqa: E402

from stego_b200 import augment  # noqa: E402

pytestmark = pytest.mark.gpu
U = 2.0 ** -24


def _frames(B, H, W, seed=0, kinds=("randn",)):
    """Normalised-looking frames: randn * 1.2 + .2 (values far outside [0, 1]).  Extra kinds, one per image: a
    constant colour, a grey frame (r = g = b: maxc == minc everywhere), saturated colours (one channel at +2.6, the
    others at -2.1, the range ImageNet normalisation gives) and a frame with maxc == 0 < maxc - minc on every third row."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 3, H, W, generator=g) * 1.2 + 0.2
    for b, kind in enumerate(kinds):
        if kind == "const":
            x[b] = torch.tensor([0.3, -1.1, 2.0]).view(3, 1, 1)
        elif kind == "grey":
            x[b] = x[b, :1].expand(3, H, W)
        elif kind == "saturated":
            ch = torch.randint(0, 3, (H, W), generator=g)
            x[b] = torch.where(torch.arange(3).view(3, 1, 1) == ch, 2.6, -2.1)
        elif kind == "zeros":  # maxc == 0 with maxc != minc on every third row
            x[b, 0, ::3] = 0.0
            x[b, 1:, ::3] = -x[b, 1:, ::3].abs() - 0.1
    return x


def _bars(H, W, size, M):
    nx, ny = AO.max_taps(W, size), AO.max_taps(H, size)
    return (33 * (nx + ny + 12) + 33 * 40 + 40) * U * M, (nx + ny + 12) * U


def _fp64(img_cpu, p, size, bar):
    """views_fp64 of one sample, the other-branch candidates of img_aug ([] when no pixel is near a boundary), the
    mask of elements they may stand for, and whether a NaN may appear there."""
    w = augment.blur_weights(p["sigma"]) if p["blur"] else None
    near = {}

    def probe(x, op):
        if op != 3:
            return
        h, _, v, _ = AO.rgb2hsv(x)
        h = torch.remainder(h + float(torch.tensor(p["hue"], dtype=torch.float32)), 1.0)
        cr = x.max(0).values - x.min(0).values
        outside = (v < bar) | (v > 1 - bar)
        near["edge"] = outside & ((6 * h - torch.round(6 * h)).abs() * cr <= 6 * bar)
        near["flat"] = outside & (cr <= bar)
        near["zero"] = (v.abs() <= bar) & (cr > 0)
    x, c = AO.views_fp64(img_cpu, p, size, w, probe)
    if not near or not (near["edge"] | near["flat"] | near["zero"]).any():
        return x, c, [], torch.zeros(3, size, size, dtype=torch.bool), False
    edge, flat = near["edge"], near["flat"]

    def other_side(place):
        def sector(i, f):
            lo = f < 0.5
            i2 = torch.where(edge, torch.where(lo, i - 1, i + 1), i)
            f2 = torch.where(edge, torch.where(lo, f + 1.0, f - 1.0), f)
            return torch.where(flat, torch.full_like(i, place), i2), torch.where(flat, torch.zeros_like(f2), f2)
        return sector
    alts = [AO.views_fp64(img_cpu, p, size, w, None, other_side(k))[0] for k in (0, 2, 4)]
    mask = edge | flat | near["zero"]
    if p["blur"]:
        mask = F.max_pool2d(mask[None, None].double(), 5, 1, 2)[0, 0].bool()
    nan_all = bool(near["zero"].any()) and p["fn_idx"].index(3) < p["fn_idx"].index(1)
    if nan_all:
        mask[:] = True
    return x, c, alts, mask.expand(3, size, size), bool(near["zero"].any())


def _compare(got, want, bar, alts=(), mask=None, nan_ok=False):
    """Max error / bar over the elements matched by the main branch, and the count matched only by another branch."""
    got, want = got.double().cpu(), want.double()
    err = (got - want).abs()
    ok = err <= bar
    other = torch.zeros_like(ok)
    if mask is not None:
        for a in alts:
            other |= (got - a).abs() <= bar
        if nan_ok:
            other |= torch.isnan(got)
        other &= mask & ~ok
    bad = ~(ok | other)
    assert not bool(bad.any()), (bad.nonzero()[:4].tolist(), got[bad][:4], want[bad][:4])
    ratio = float((err[ok] / bar).max()) if ok.any() else 0.0
    return ratio, int(other.sum())


def _run(img, seeds, size, torchvision_check=True, built=0):
    """Kernel views of the batch against fp64 (and torchvision) for every image; the other-branch elements must be
    rare among the random frames (the first `built` frames are constructed to sit on the boundaries)."""
    B, _, H, W = img.shape
    cpu = torch.get_rng_state()
    cuda = torch.cuda.get_rng_state()
    img_aug, coord_aug = augment.aug_alignment_views(img, seeds, size)
    torch.cuda.synchronize()
    assert torch.equal(torch.get_rng_state(), cpu) and torch.equal(torch.cuda.get_rng_state(), cuda)
    assert img_aug.shape == (B, 3, size, size) and coord_aug.shape == (B, size, size, 2)
    params, _ = augment.draw_records(seeds, H, W)
    M = max(1.0, float(img.abs().max()))
    bar, cbar = _bars(H, W, size, M)
    worst, others, total = 0.0, 0, 0
    for b, p in enumerate(params):
        frame = img[b].cpu()
        x, c, alts, mask, nan_ok = _fp64(frame, p, size, bar)
        r, n = _compare(img_aug[b], x, bar, alts, mask, nan_ok)
        worst = max(worst, r)
        if b >= built:
            others, total = others + n, total + x.numel()
        worst = max(worst, _compare(coord_aug[b], c, cbar)[0])
        if torchvision_check:
            with torch.random.fork_rng():
                ia, ca = AO.reference_views(frame, seeds[b], size)
            # torchvision is within the bar of the same float64 branches; on the same branch the two are within 2 bar
            _compare(ia, x, bar, alts, mask, nan_ok)
            _compare(ca, c, cbar)
            got = img_aug[b].cpu()
            same = ((got - ia).abs() <= 2 * bar) | (torch.isnan(got) & torch.isnan(ia))
            assert float(same.double().mean()) >= 0.999
            assert bool(((coord_aug[b].cpu() - ca).abs() <= 2 * cbar).all())
    assert others <= 1e-3 * max(total, 1), (others, total)
    return img_aug, coord_aug, params, worst


def _seeds_where(pred, n, H=224, W=224, start=0):
    out = []
    with torch.random.fork_rng(devices=[]):
        for s in range(start, start + 200000):
            if pred(augment.draw_params(s, H, W)):
                out.append(s)
                if len(out) == n:
                    return out
    raise AssertionError("no seed found")


@pytest.mark.parametrize("B,H,W,size", [(1, 224, 224, 224), (32, 224, 224, 224), (64, 224, 224, 224),
                                        (8, 320, 320, 320), (4, 448, 448, 448), (6, 240, 320, 224),
                                        (4, 480, 640, 224), (5, 150, 200, 320)])
def test_views_fp64(cuda_dev, B, H, W, size):
    """Batches of sizes 1..64, size 224 / 320 / 448, square and non-square frames, down- and up-sampling."""
    kinds = ("const", "grey", "saturated", "zeros")[:B]
    img = _frames(B, H, W, seed=B + H, kinds=kinds).to(cuda_dev)
    seeds = [int(s) for s in torch.randint(0, 2147483647, (B,), generator=torch.Generator().manual_seed(size + B))]
    _, _, _, worst = _run(img, seeds, size, torchvision_check=B <= 8, built=len(kinds))
    assert worst <= 1.0


def test_views_edge_parameters(cuda_dev):
    """Seeds found by search: the identity crop (the fallback on a square frame: the full frame, returned unresized),
    the widest and narrowest crop ratios among 4000 seeds, sigma near .1 and near 2, all 24 jitter orders, hue first
    (it sees the unclamped normalised values) and grayscale."""
    import itertools
    H = W = size = 224
    seeds = _seeds_where(lambda p: p["crop"] == (0, 0, 224, 224), 1)
    with torch.random.fork_rng(devices=[]):
        ratios = sorted(range(4000), key=lambda s: (lambda c: c[3] / c[2])(augment.draw_params(s, H, W)["crop"]))
    seeds += [ratios[0], ratios[-1]]
    seeds += _seeds_where(lambda p: p["blur"] and p["sigma"] < 0.12, 1)
    seeds += _seeds_where(lambda p: p["blur"] and p["sigma"] > 1.98, 1)
    for order in itertools.permutations(range(4)):
        seeds += _seeds_where(lambda p, o=list(order): p["fn_idx"] == o, 1)
    seeds += _seeds_where(lambda p: p["gray"] and p["fn_idx"][0] == 3, 1)
    kinds = ("const", "grey", "saturated", "zeros") * 3
    img = _frames(len(seeds), H, W, seed=5, kinds=kinds).to(cuda_dev)
    _, _, params, worst = _run(img, seeds, size, built=len(kinds))
    assert params[0]["crop"] == (0, 0, 224, 224)
    assert worst <= 1.0


def test_noncontiguous_reruns_and_no_host_sync(cuda_dev):
    """A channels-last view and a strided slice give the contiguous input's bits; two calls give identical bits; the
    call makes no device-to-host copy and no synchronisation (torch's sync debug mode raises on either)."""
    B, H, W, size = 6, 224, 224, 224
    base = _frames(B, H, 2 * W, seed=3).to(cuda_dev)
    sliced = base[:, :, :, ::2]
    cl = sliced.contiguous().to(memory_format=torch.channels_last)
    seeds = list(range(100, 100 + B))
    want = augment.aug_alignment_views(sliced.contiguous(), seeds, size)
    for view in (sliced, cl):
        got = augment.aug_alignment_views(view, seeds, size)
        assert all(torch.equal(g.view(torch.int32), w.view(torch.int32)) for g, w in zip(got, want))
    augment.aug_alignment_views(sliced, seeds, size)  # warm the allocator's pinned and device blocks
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        again = augment.aug_alignment_views(sliced, seeds, size)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert all(torch.equal(g.view(torch.int32), w.view(torch.int32)) for g, w in zip(again, want))
    _run(sliced, seeds, size, torchvision_check=False)


def test_training_step_aug_alignment(cuda_dev):
    """_training_step_autograd with aug_alignment_weight > 0, twice from the same model, seeds and batch: once with
    views from aug_alignment_views, once with views from the torchvision composition.  The views differ by at most
    2 bar (about 1e-4 at M = 3.6; measured well below).  The frozen backbone rounds its input to bf16 (ulp 2^-8 at
    1), so such a difference moves an input by at most one bf16 ulp where the rounding flips.  The logged term is a
    mean of cosines in [-1, 1]; a perturbation of that size moves it by a few 1e-4 at most.  So 2e-3 bounds it, and
    every term that does not read the views must agree bit for bit."""
    from _parity_util import make_batch, make_model
    B, res = 4, 224
    batch = make_batch(B, res, cuda_dev)
    seeds = [11, 12, 13, 14]
    ia, ca = augment.aug_alignment_views(batch["img"], seeds, res)
    with torch.random.fork_rng():
        ref = [AO.reference_views(batch["img"][b].cpu(), s, res) for b, s in enumerate(seeds)]
    ib = torch.stack([r[0] for r in ref]).to(cuda_dev)
    cb = torch.stack([r[1] for r in ref]).to(cuda_dev)
    logged = []
    for img_aug, coord_aug in ((ia, ca), (ib, cb)):
        model, _ = make_model("vit_small", cuda_dev, fused=True, batch_size=B, res=res, aug_alignment_weight=0.6)
        b = dict(batch, img_aug=img_aug, coord_aug=coord_aug)
        torch.manual_seed(21)
        model.training_step(b, 0)
        torch.cuda.synchronize()
        logged.append({k: float(v) for k, v in model.logged.items() if torch.is_tensor(v) and v.numel() == 1})
    a, r = logged
    assert abs(a["loss/aug_alignment"] - r["loss/aug_alignment"]) <= 2e-3, (a, r)
    for k in ("loss/pos_intra", "loss/pos_inter", "loss/neg_inter", "loss/linear", "loss/cluster"):
        assert a[k] == r[k], k
