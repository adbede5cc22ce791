"""Dense correspondence heatmaps on the GPU (stego_b200/correspondence.py, stego_b200/csrc/heatmap.cu).

  * correspondence_heatmaps against the fp64 restatement (oracle/heatmap_oracle.py) within 1e-4 (values in [0, 2]):
    the bf16 hi/lo split of the correlation GEMM is good to ~2^-16 relative per dot product, the row mean adds at most
    as much again, and the clamp and the bilinear weights (non-negative, summing to 1) carry a low-resolution bar to the
    output unchanged.  Shapes: the reference's figure and movie, c1, c2, code maps, layouts and dtypes, self and KNN
    maps of different sizes, a non-square 1024 x 2048 output, one point / one pixel, a zero vector, a constant target;
  * the reference's own lines (tests/golden/correspondence_heatmaps.pt) within 2e-4;
  * the upsample kernel alone against ATen's CUDA F.interpolate on the same map, within 4 ulp of max |map|;
  * two calls give bit-identical output;
  * get_heatmaps against an fp32 restatement of the reference's lines on the same DinoFeaturizer outputs;
  * one output of more than 2^31 elements (64-bit offsets).
"""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import heatmap_oracle as HO  # noqa: E402

pytestmark = pytest.mark.gpu
BAR = 1e-4
FIGURE_POINTS = [[-.1, 0.0], [.5, .8], [-.7, -.7]]


def _heatmaps(*a, **k):
    from stego_b200.correspondence import correspondence_heatmaps
    return correspondence_heatmaps(*a, **k)


def fmap(B, E, h, w, seed, dev, rank=4, noise=0.5):
    """Low rank plus noise [B, E, h, w] fp32: every query correlates positively with part of the map, negatively with
    the rest, so the centring and the clamp both change values."""
    g = torch.Generator(device=dev).manual_seed(seed)
    basis = torch.randn(B, rank, E, device=dev, generator=g)
    coef = torch.randn(B, h * w, rank, device=dev, generator=g)
    x = coef @ basis + noise * torch.randn(B, h * w, E, device=dev, generator=g)
    return x.transpose(1, 2).reshape(B, E, h, w).contiguous()


def points(B, P, seed, dev, spread=1.1):
    g = torch.Generator(device=dev).manual_seed(seed)
    return (torch.rand(B, P, 1, 2, device=dev, generator=g) * 2 - 1) * spread


def movie_points():
    """The reference's 280-point key-point path (plot_dino_correspondence.py:157-173): 60 frames on each key point,
    50 interpolated between consecutive ones."""
    key = [[-.7, -.7], [-.1, 0.0], [.5, .8]]
    pts = []
    for i in range(len(key)):
        pts.extend([key[i]] * 60)
        if i < len(key) - 1:
            pts.extend(np.stack([np.linspace(key[i][0], key[i + 1][0], 50),
                                 np.linspace(key[i][1], key[i + 1][1], 50)], axis=1).tolist())
    return torch.tensor(pts, dtype=torch.float32).reshape(1, len(pts), 1, 2)


def check(feats, target, qp, size, bar=BAR):
    out = _heatmaps(feats, target, qp, size)
    B, P = qp.shape[:2]
    assert out.dtype == torch.float32 and out.shape == (B, P) + tuple(size) and out.is_contiguous()
    ref = HO.heatmaps(feats, target, qp, size)
    err = float((out.double() - ref).abs().max())
    assert err <= bar, err
    return out, ref


def test_reference_figure(cuda_dev):
    f = fmap(1, 384, 64, 64, 1, cuda_dev)
    fp = fmap(1, 384, 64, 64, 2, cuda_dev)
    qp = torch.tensor(FIGURE_POINTS, device=cuda_dev).reshape(1, 3, 1, 2)
    out, ref = check(f, f, qp, (512, 512))
    assert float((ref == 0).double().mean()) > 0.05 and float(ref.max()) > 0.3
    check(f, fp, qp, (512, 512))


def test_reference_movie(cuda_dev):
    f = fmap(1, 384, 64, 64, 3, cuda_dev)
    fp = fmap(1, 384, 64, 64, 4, cuda_dev)
    qp = movie_points().to(cuda_dev)
    assert qp.shape[1] == 280
    check(f, f, qp, (512, 512))
    check(f, fp, qp, (512, 512))


@pytest.mark.parametrize("B,E,hw,res", [(32, 384, 28, 224), (32, 768, 40, 320)], ids=["c1", "c2"])
def test_training_shapes(cuda_dev, B, E, hw, res):
    f = fmap(B, E, hw, hw, 5 + E, cuda_dev)
    fp = fmap(B, E, hw, hw, 6 + E, cuda_dev)
    check(f, fp, points(B, 16, 7, cuda_dev), (res, res))


def test_code_maps(cuda_dev):
    c = fmap(4, 70, 28, 28, 8, cuda_dev, rank=3, noise=0.3)
    cp = fmap(4, 70, 28, 28, 9, cuda_dev, rank=3, noise=0.3)
    qp = points(4, 16, 10, cuda_dev)
    check(c, c, qp, (224, 224))
    check(c, cp, qp, (224, 224))


@pytest.mark.parametrize("layout", ["fp32_nchw", "fp32_channels_last", "bf16_tokens", "bf16_nchw", "mixed"])
def test_layouts_and_dtypes(cuda_dev, layout):
    f = fmap(3, 384, 20, 24, 11, cuda_dev)
    t = fmap(3, 384, 14, 18, 12, cuda_dev)  # KNN map of a different size
    if layout == "fp32_channels_last":
        f, t = f.to(memory_format=torch.channels_last), t.to(memory_format=torch.channels_last)
    elif layout == "bf16_tokens":  # tokens-major [B, hw, E] storage viewed as NCHW, as DinoFeaturizer returns
        f = f.to(torch.bfloat16).permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
        t = t.to(torch.bfloat16).permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
        assert f.stride(1) == 1
    elif layout == "bf16_nchw":
        f, t = f.to(torch.bfloat16), t.to(torch.bfloat16)
    elif layout == "mixed":
        f, t = f.to(torch.bfloat16), t[:, :, 1:, ::2]  # bf16 queries, a strided fp32 view as the target
    qp = points(3, 9, 13, cuda_dev)
    check(f, t, qp, (160, 192))
    check(f, f, qp, (100, 90))


def test_non_square(cuda_dev):
    f = fmap(1, 64, 128, 256, 14, cuda_dev)
    qp = points(1, 4, 15, cuda_dev)
    check(f, f, qp, (1024, 2048))


def test_one_point_one_pixel(cuda_dev):
    f = fmap(2, 32, 6, 5, 16, cuda_dev)
    one = fmap(2, 32, 1, 1, 17, cuda_dev)
    qp = points(2, 1, 18, cuda_dev)
    check(f, f, qp, (1, 1))
    check(f, f, qp, (1, 7))
    check(one, one, qp, (3, 4))  # a 1 x 1 map: every correlation equals its mean, the output is 0
    out = _heatmaps(f, one, qp, (5, 5))
    assert bool((out == 0).all())
    check(f, f, points(2, 1, 19, cuda_dev), (33, 31))


def test_zero_feature_vector(cuda_dev):
    """F.normalize's eps: a zero query or a zero target position correlates 0 with everything."""
    f = fmap(1, 384, 16, 16, 20, cuda_dev)
    f[0, :, 0, 0] = 0
    f[0, :, 5, 7] = 0
    qp = torch.tensor([[-1.0, -1.0], [0.3, 0.2]], device=cuda_dev).reshape(1, 2, 1, 2)  # point 0 is pixel (0, 0)
    out, ref = check(f, f, qp, (64, 64))
    assert bool((out[0, 0] == 0).all())
    check(f.to(torch.bfloat16), f.to(torch.bfloat16), qp, (64, 64))


def test_constant_target(cuda_dev):
    f = fmap(2, 384, 16, 16, 21, cuda_dev)
    for t in (f[:, :, :1, :1].expand(-1, -1, 12, 10).contiguous(),
              f[:, :, :1, :1].expand(-1, -1, 12, 10).contiguous().to(torch.bfloat16)):
        out = _heatmaps(f, t, points(2, 5, 22, cuda_dev), (48, 40))
        assert bool((out == 0).all())


def test_matches_reference_lines_fixture(cuda_dev):
    g = torch.load(os.path.join(HERE, "golden", "correspondence_heatmaps.pt"))
    qp = g["query_points"].to(cuda_dev)
    for dtype in (torch.bfloat16, torch.float32):
        f = g["feats"].to(cuda_dev, dtype)
        fp = g["feats_pos"].to(cuda_dev, dtype)
        intra = _heatmaps(f, f, qp, g["img_size"])[0].cpu()
        inter = _heatmaps(f, fp, qp, g["pos_size"])[0].cpu()
        assert float((intra - g["heatmap_intra"]).abs().max()) <= 2e-4
        assert float((inter - g["heatmap_inter"]).abs().max()) <= 2e-4


@pytest.mark.parametrize("n,h,w,H,W", [(280, 64, 64, 512, 512), (16, 40, 40, 320, 320), (3, 128, 256, 1024, 2048),
                                       (5, 7, 9, 30, 33), (2, 1, 1, 4, 8), (2, 5, 6, 1, 1), (4, 12, 12, 12, 12)])
def test_upsample_matches_aten(cuda_dev, n, h, w, H, W):
    from stego_b200 import _lib
    g = torch.Generator(device=cuda_dev).manual_seed(n * 31 + H)
    x = torch.rand(n, h, w, device=cuda_dev, generator=g) * 1.7
    x[x < 0.6] = 0
    out = torch.empty(n, H, W, device=cuda_dev)
    _lib.check(_lib.load().stego_heatmap_upsample(_lib.ptr(x), _lib.ptr(out), n, h, w, H, W, _lib.stream()),
               "stego_heatmap_upsample")
    ref = F.interpolate(x[:, None], (H, W), mode="bilinear", align_corners=True)[:, 0]
    ulp = 2.0 ** (np.floor(np.log2(float(x.abs().max()))) - 23)
    assert float((out - ref).abs().max()) <= 4 * ulp


def test_repeatable(cuda_dev):
    f = fmap(4, 384, 28, 28, 23, cuda_dev)
    fp = fmap(4, 384, 24, 30, 24, cuda_dev)
    qp = points(4, 40, 25, cuda_dev)
    a = _heatmaps(f, fp, qp, (224, 224))
    b = _heatmaps(f, fp, qp, (224, 224))
    assert torch.equal(a, b)


def test_get_heatmaps_drop_in(cuda_dev):
    """get_heatmaps against the reference's lines (restated in fp32 torch) on the same DinoFeaturizer's outputs, in
    eval mode; the featurizer's mode is left as the caller set it."""
    from stego_b200.config import make_cfg
    from stego_b200.correspondence import get_heatmaps
    from stego_b200.modules import DinoFeaturizer
    cfg = make_cfg(random_backbone_init=True)
    torch.manual_seed(0)
    net = DinoFeaturizer(cfg.dim, cfg).to(cuda_dev).eval()
    g = torch.Generator().manual_seed(26)
    img = torch.randn(1, 3, 128, 160, generator=g)
    img_pos = torch.randn(1, 3, 96, 128, generator=g)
    seen = []

    def rec(x):
        out = net(x)
        seen.append(out[0])
        return out

    for pts in (FIGURE_POINTS, [[0.25, -0.5]]):
        seen.clear()
        qp = torch.tensor(pts, device=cuda_dev).reshape(1, len(pts), 1, 2)
        intra, inter = get_heatmaps(rec, img, img_pos, qp)
        assert not net.training and len(seen) == 2
        assert intra.device.type == "cpu" and intra.shape == (len(pts), 128, 160)
        assert inter.device.type == "cpu" and inter.shape == (len(pts), 96, 128)
        f1, f2 = seen
        ref_intra = HO.heatmaps(f1, f1, qp, img.shape[2:], dtype=torch.float32)[0].cpu()
        ref_inter = HO.heatmaps(f1, f2, qp, img_pos.shape[2:], dtype=torch.float32)[0].cpu()
        assert float((intra - ref_intra).abs().max()) <= 2e-4
        assert float((inter - ref_inter).abs().max()) <= 2e-4


def test_output_beyond_2_31_elements(cuda_dev):
    free, _ = torch.cuda.mem_get_info(cuda_dev)
    if free < 12 * 2 ** 30:
        pytest.skip(f"needs 12 GB free, {free / 2 ** 30:.1f} GB available")
    P = 8200
    f = fmap(1, 64, 64, 64, 27, cuda_dev)
    qp = points(1, P, 28, cuda_dev)
    out = _heatmaps(f, f, qp, (512, 512))
    assert out.numel() > 2 ** 31
    rows = torch.tensor([0, 4095, 4096, P - 2, P - 1], device=cuda_dev)  # 4096 * 512^2 = 2^30 ... past 2^31 at the end
    ref = HO.heatmaps(f, f, qp[:, rows], (512, 512))
    assert float((out[:, rows].double() - ref).abs().max()) <= BAR
    del out
    torch.cuda.empty_cache()
