"""Dense CRF on the GPU (stego_b200.crf, csrc/crf.cu) against the CPU restatement of pydensecrf's published algorithm
(oracle/crf_oracle.py).  Parity with the reference's CRF stage itself is UNPINNED (pydensecrf is third-party, absent):
what is checked is that the CUDA path computes the same mean-field marginals as the restatement — same lattice, fp32 —
to 1e-3 and the same labels."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.join(os.path.dirname(__file__), "..", "oracle"))


def _frame(H, W, C, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    # piecewise-constant image + noise (so that the bilateral kernel has edges to respect), normalised like the loader does
    base = torch.rand(3, 4, 4, generator=g)
    img01 = torch.nn.functional.interpolate(base[None], (H, W), mode="nearest")[0] * 0.8 + 0.1 * torch.rand(3, H, W, generator=g)
    mean = torch.tensor([0.485, 0.456, 0.406]).view(3, 1, 1)
    std = torch.tensor([0.229, 0.224, 0.225]).view(3, 1, 1)
    img = (img01 - mean) / std
    logits = torch.randn(C, h, w, generator=g) * 2.0
    return img, logits


@pytest.mark.parametrize("H,W,C,h,w", [(24, 32, 5, 6, 8), (40, 56, 27, 5, 7), (64, 64, 27, 64, 64)])
def test_dense_crf_matches_oracle(cuda_dev, H, W, C, h, w):
    import crf_oracle as CO
    from stego_b200 import crf
    img, logits = _frame(H, W, C, h, w, seed=H * 100 + C)
    want = CO.dense_crf(img, logits)                                    # [C, H, W] numpy
    got, arg = crf.dense_crf(img.to(cuda_dev), logits.to(cuda_dev), want_argmax=True)
    got = got.cpu().numpy()
    assert got.shape == want.shape
    assert np.abs(got.sum(0) - 1).max() < 1e-5
    err = np.abs(got - want).max()
    agree = (got.argmax(0) == want.argmax(0)).mean()
    print(f"CRF {H}x{W} C={C}: max |dQ| {err:.2e}, label agreement {agree:.5f}")
    assert err < 2e-3, err
    assert agree > 0.999
    assert (arg.cpu().numpy() == got.argmax(0)).all()
    # the CRF did something: labels differ from the unary argmax on a piecewise-constant image with noisy unaries
    up = torch.nn.functional.interpolate(logits[None], (H, W), mode="bilinear", align_corners=False)[0]
    assert (want.argmax(0) != up.argmax(0).numpy()).mean() > 0.01


def test_crf_lattices_match_oracle(cuda_dev):
    """Lattice construction (vertex de-duplication, barycentric weights, symmetric normalisation) for both kernels."""
    import crf_oracle as CO
    from stego_b200 import crf
    H, W = 20, 28
    img, _ = _frame(H, W, 3, 4, 4, seed=3)
    image = CO.prepare_image(img)
    image_dev = crf.prepare_image(img.to(cuda_dev))
    assert (image_dev.cpu().numpy() == image).all()
    for d, feat in ((2, CO.gaussian_features(H, W, 1.0)), (5, CO.bilateral_features(image, 67.0, 3.0))):
        ok = CO.DenseKernel(feat)
        lat = crf._position_lattice(H, W, cuda_dev) if d == 2 else crf._bilateral_lattice([image_dev])
        assert lat.M == ok.lattice.M
        assert np.abs(lat.bary.cpu().numpy() - ok.lattice.bary).max() < 1e-4
        assert np.abs(lat.norm.cpu().numpy() / ok.norm - 1).max() < 1e-4
        # same partition of (pixel, vertex) slots into lattice points (ids differ: compare co-membership through the keys)
        a = lat.offset.cpu().numpy().reshape(-1)
        b = ok.lattice.offset.reshape(-1)
        first = {}
        for x, y in zip(a.tolist(), b.tolist()):
            assert first.setdefault(x, y) == y


def test_batched_crf_full_frame_properties(cuda_dev):
    """configs[4] frame (1024 x 2048, 27 classes): marginals normalise, labels mostly follow the unaries, runs per frame."""
    from stego_b200 import crf
    torch.manual_seed(0)
    H, W, C = 1024, 2048, 27
    img = torch.randn(1, 3, H, W, device=cuda_dev) * 0.5
    logp = torch.log_softmax(torch.randn(1, C, 128, 256, device=cuda_dev) * 3, 1)
    logp = torch.nn.functional.interpolate(logp, (H, W), mode="bilinear", align_corners=False)
    q = crf.batched_crf(None, img, logp)
    assert q.shape == (1, C, H, W)
    assert (q.sum(1) - 1).abs().max().item() < 1e-4
    assert torch.isfinite(q).all()
    assert (q.argmax(1) == logp.argmax(1)).float().mean().item() > 0.5


def test_dense_crf_is_reproducible(cuda_dev):
    """Two calls on the same input give bit-identical marginals and labels: every splat sums its lattice point's slots
    in a fixed order (no float atomics).  A noise frame, so the bilateral lattice has many points with several slots."""
    from stego_b200 import crf
    H, W, C = 320, 320, 27
    g = torch.Generator().manual_seed(11)
    img = torch.randn(3, H, W, generator=g).to(cuda_dev)
    logits = (torch.randn(C, 40, 40, generator=g) * 3).to(cuda_dev)
    q1, a1 = crf.dense_crf(img, logits, want_argmax=True)
    q2, a2 = crf.dense_crf(img, logits, want_argmax=True)
    assert torch.equal(q1, q2) and torch.equal(a1, a2)
