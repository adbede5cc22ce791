"""CPU oracle for the dense-CRF stage of the eval path (reference: src/crf.py:22-45 -> pydensecrf).  TEST INFRASTRUCTURE ONLY.

Parity status: **UNPINNED**.  The arithmetic lives in a third-party dependency that is neither vendored in the reference nor
installed here: `pydensecrf` (listed unpinned in environment.yml:34; the demo notebook installs
`git+https://github.com/lucasb-eyer/pydensecrf.git`, i.e. master, which wraps Philipp Kraehenbuehl's densecrf C++:
densecrf.cpp, pairwise.cpp, permutohedral.cpp).  This file restates that PUBLISHED algorithm in numpy —

  * fully connected CRF with Gaussian edge potentials, mean-field inference (Kraehenbuehl & Koltun, NIPS 2011);
  * high-dimensional Gaussian filtering on the permutohedral lattice, splat / blur / slice (Adams, Baek & Davis,
    Eurographics 2010), with densecrf's specifics: blur stencil new = old + 0.5 (n1 + n2) along each of the d+1 lattice
    axes, slice scaled by alpha = 1 / (1 + 2^-d), NORMALIZE_SYMMETRIC kernels (out = n * K(n * in), n = 1/sqrt(K 1 + 1e-20)),
    Potts compatibility (pairwise message = -w * K(Q)), Q <- softmax(-U + sum_k w_k K_k(Q)), Q_0 = softmax(-U);
  * the parameters and the image / unary preparation of the reference's own call site, src/crf.py:13-43.

Because no pydensecrf binary, source or golden vector is available offline, bit parity with the reference's CRF cannot be
claimed; tests compare the CUDA implementation with THIS restatement (same lattice, fp32) by label agreement and by the
marginals, and check the restatement itself against brute-force Gaussian filtering and against an exact O(N^2) dense
mean-field with the same conventions (tests/test_oracle_golden.py).
"""
from __future__ import annotations

from typing import Dict, Tuple

import numpy as np

# src/crf.py:13-19
MAX_ITER = 10
POS_W = 3
POS_XY_STD = 1
Bi_W = 4
Bi_XY_STD = 67
Bi_RGB_STD = 3


class Permutohedral:
    """permutohedral.cpp: Permutohedral::init / seqCompute."""

    def __init__(self, feature: np.ndarray):
        """feature: [d, N] float32."""
        feature = np.asarray(feature, dtype=np.float32)
        d, N = feature.shape
        self.d, self.N = d, N
        inv_std_dev = np.sqrt(2.0 / 3.0) * (d + 1)
        scale = (1.0 / np.sqrt((np.arange(d) + 2.0) * (np.arange(d) + 1.0)) * inv_std_dev).astype(np.float32)
        # elevate (y = E p)
        cf = feature * scale[:, None]                                  # [d, N]
        elevated = np.zeros((d + 1, N), np.float32)
        sm = np.zeros(N, np.float32)
        for j in range(d, 0, -1):
            elevated[j] = sm - j * cf[j - 1]
            sm = sm + cf[j - 1]
        elevated[0] = sm
        # closest 0-coloured simplex through rounding
        down_factor = np.float32(1.0 / (d + 1))
        up_factor = np.float32(d + 1)
        v = down_factor * elevated
        up = np.ceil(v) * up_factor
        down = np.floor(v) * up_factor
        rem0 = np.where(up - elevated < elevated - down, up, down).astype(np.float32)
        ssum = np.rint(rem0.sum(0) * down_factor).astype(np.int64)      # integer by construction
        # rank of every coordinate in the sorted order of the residuals
        rank = np.zeros((d + 1, N), np.int64)
        diff = (elevated - rem0).astype(np.float64)
        for i in range(d):
            for j in range(i + 1, d + 1):
                lt = diff[i] < diff[j]
                rank[i] += lt
                rank[j] += ~lt
        rank += ssum[None, :]
        lo, hi = rank < 0, rank > d
        rank[lo] += d + 1
        rem0[lo] += d + 1
        rank[hi] -= d + 1
        rem0[hi] -= d + 1
        # barycentric coordinates
        bary = np.zeros((d + 2, N), np.float32)
        vv = ((elevated - rem0) * down_factor).astype(np.float32)
        cols = np.arange(N)
        for i in range(d + 1):
            np.add.at(bary, (d - rank[i], cols), vv[i])
            np.add.at(bary, (d - rank[i] + 1, cols), -vv[i])
        bary[0] += 1.0 + bary[d + 1]
        # canonical simplex and the d+1 vertices of every point
        canonical = np.zeros((d + 1, d + 1), np.int64)
        for i in range(d + 1):
            canonical[i, :d - i + 1] = i
            canonical[i, d - i + 1:] = i - (d + 1)
        keys = np.zeros((N, d + 1, d), np.int64)
        rem0i = rem0.astype(np.int64)
        for r in range(d + 1):
            for i in range(d):
                keys[:, r, i] = rem0i[i] + canonical[r, rank[i]]
        flat = keys.reshape(-1, d)
        uniq, inv = np.unique(flat, axis=0, return_inverse=True)
        self.M = uniq.shape[0]
        self.offset = inv.reshape(N, d + 1)                             # lattice point of (pixel, vertex)
        self.bary = bary[:d + 1].T.copy()                              # [N, d+1]
        self.keys = uniq
        lookup = {tuple(k): i for i, k in enumerate(uniq)}
        n1 = np.full((d + 1, self.M), -1, np.int64)
        n2 = np.full((d + 1, self.M), -1, np.int64)
        for j in range(d + 1):
            k1 = uniq - 1
            k2 = uniq + 1
            if j < d:
                k1[:, j] = uniq[:, j] + d
                k2[:, j] = uniq[:, j] - d
            for i in range(self.M):
                n1[j, i] = lookup.get(tuple(k1[i]), -1)
                n2[j, i] = lookup.get(tuple(k2[i]), -1)
        self.n1, self.n2 = n1, n2

    def compute(self, inp: np.ndarray, reverse: bool = False) -> np.ndarray:
        """inp: [N, value_size] -> filtered [N, value_size] (splat, blur along the d+1 axes, slice)."""
        d, N, M = self.d, self.N, self.M
        vs = inp.shape[1]
        values = np.zeros((M + 2, vs), np.float32)
        for j in range(d + 1):
            np.add.at(values, self.offset[:, j] + 1, self.bary[:, j:j + 1] * inp)
        axes = range(d, -1, -1) if reverse else range(d + 1)
        for j in axes:
            new = np.zeros_like(values)
            new[1:M + 1] = values[1:M + 1] + 0.5 * (values[self.n1[j] + 1] + values[self.n2[j] + 1])
            values = new
        alpha = np.float32(1.0 / (1.0 + 2.0 ** (-d)))
        out = np.zeros((N, vs), np.float32)
        for j in range(d + 1):
            out += self.bary[:, j:j + 1] * values[self.offset[:, j] + 1] * alpha
        return out


class DenseKernel:
    """pairwise.cpp: DenseKernel with NORMALIZE_SYMMETRIC (pydensecrf's default for both pairwise terms)."""

    def __init__(self, feature: np.ndarray):
        self.lattice = Permutohedral(feature)
        ones = np.ones((feature.shape[1], 1), np.float32)
        self.norm = (1.0 / np.sqrt(self.lattice.compute(ones)[:, 0] + 1e-20)).astype(np.float32)

    def apply(self, Q: np.ndarray) -> np.ndarray:
        """Q: [N, C] -> n * K(n * Q)."""
        return self.lattice.compute(Q * self.norm[:, None]) * self.norm[:, None]


def gaussian_features(H: int, W: int, sxy: float) -> np.ndarray:
    """densecrf.cpp DenseCRF2D::addPairwiseGaussian: (x / sx, y / sy) per pixel, row-major pixels."""
    ys, xs = np.mgrid[0:H, 0:W]
    return np.stack([xs.reshape(-1) / sxy, ys.reshape(-1) / sxy]).astype(np.float32)


def bilateral_features(image: np.ndarray, sxy: float, srgb: float) -> np.ndarray:
    """DenseCRF2D::addPairwiseBilateral: (x / sx, y / sy, c0 / sr, c1 / sg, c2 / sb); image [H, W, 3] uint8."""
    H, W, _ = image.shape
    ys, xs = np.mgrid[0:H, 0:W]
    im = image.reshape(-1, 3).astype(np.float32)
    return np.stack([xs.reshape(-1) / sxy, ys.reshape(-1) / sxy, im[:, 0] / srgb, im[:, 1] / srgb, im[:, 2] / srgb]).astype(np.float32)


def exp_and_normalize(x: np.ndarray) -> np.ndarray:
    """densecrf.cpp expAndNormalize over the class axis (axis 1 here)."""
    e = np.exp(x - x.max(1, keepdims=True))
    return (e / e.sum(1, keepdims=True)).astype(np.float32)


def mean_field(unary: np.ndarray, kernels, weights, n_iter: int = MAX_ITER) -> np.ndarray:
    """densecrf.cpp DenseCRF::inference with Potts compatibilities: unary [N, C] (energies), returns Q [N, C]."""
    Q = exp_and_normalize(-unary)
    for _ in range(n_iter):
        tmp = -unary
        for k, w in zip(kernels, weights):
            tmp = tmp + w * k.apply(Q)            # pairwise->apply gives -w K(Q); tmp1 -= that
        Q = exp_and_normalize(tmp)
    return Q


def unary_from_softmax(probs: np.ndarray, clip: float = 1e-5) -> np.ndarray:
    """pydensecrf.utils.unary_from_softmax(sm, scale=None, clip=1e-5): -log(clip(p)), [C, N] float32."""
    return (-np.log(np.clip(probs, clip, 1.0))).reshape(probs.shape[0], -1).astype(np.float32)


def prepare_image(image_tensor) -> np.ndarray:
    """src/crf.py:23: np.array(VF.to_pil_image(unnorm(image_tensor)))[:, :, ::-1] — un-normalise with the ImageNet
    statistics (src/utils.py:140-141), x255 and truncate to uint8 (torchvision to_pil_image), reverse the channel order."""
    import torch
    mean = torch.tensor([0.485, 0.456, 0.406]).view(3, 1, 1)
    std = torch.tensor([0.229, 0.224, 0.225]).view(3, 1, 1)
    img = (image_tensor.detach().cpu().float() * std + mean).mul(255).clamp(0, 255).byte()  # (out-of-range: clamped; UB in the reference)
    return np.ascontiguousarray(img.permute(1, 2, 0).numpy()[:, :, ::-1])


def dense_crf(image_tensor, output_logits) -> np.ndarray:
    """src/crf.py:22-45 `dense_crf(image_tensor [3,H,W] normalised, output_logits [C,h,w]) -> Q [C,H,W]`."""
    import torch
    import torch.nn.functional as F
    image = prepare_image(image_tensor)
    H, W = image.shape[:2]
    logits = F.interpolate(output_logits.detach().cpu().float().unsqueeze(0), size=(H, W), mode="bilinear",
                           align_corners=False).squeeze(0)
    probs = F.softmax(logits, dim=0).numpy()
    C = probs.shape[0]
    U = unary_from_softmax(probs).T.copy()                               # [N, C]
    kernels = [DenseKernel(gaussian_features(H, W, POS_XY_STD)), DenseKernel(bilateral_features(image, Bi_XY_STD, Bi_RGB_STD))]
    Q = mean_field(U, kernels, [POS_W, Bi_W], MAX_ITER)
    return Q.T.reshape(C, H, W)


def brute_force_filter(feature: np.ndarray, inp: np.ndarray) -> np.ndarray:
    """Exact Gaussian filtering out_i = sum_j exp(-|f_i - f_j|^2 / 2) in_j — what the lattice approximates (tests only)."""
    f = feature.T.astype(np.float64)
    d2 = ((f[:, None, :] - f[None, :, :]) ** 2).sum(-1)
    return (np.exp(-0.5 * d2) @ inp.astype(np.float64)).astype(np.float32)
