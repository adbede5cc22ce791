"""Drop-in for the reference `src/modules.py` (mhamilton723/STEGO): same public names, constructor
arguments, forward signatures, parameter names and return tuples — with the hot path running on
hand-written sm_90a kernels through libstego_b200.so (include/stego_b200.h).

Hot path (CUDA kernels, no CPU / eager fallback):
    DinoFeaturizer               modules.py:17-118    frozen DINO ViT + 1x1-conv head (wgmma GEMMs, fused attention)
    ContrastiveCorrelationLoss   modules.py:314-398   fused sample/norm/einsum/loss + backward
    ClusterLookup                modules.py:134-161   fused cosine-sim / argmax / softmax probe
    norm, tensor_correlation, sample, super_perm  modules.py:275-295
API-surface only (plain torch, not on the measured path; SURVEY.md §8a row a14 and §2 "out of scope"):
    FeaturePyramidNet, DoubleConv, NetWithActivations, LambdaLayer, ResizeAndClassify, Decoder,
    ContrastiveCRFLoss, average_norm, sample_nonzero_locations
"""
from __future__ import annotations

import math
import os
import sys
from os.path import join  # noqa: F401  (reference scripts rely on star-exported names)
from typing import Optional

import numpy as np  # noqa: F401
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib, corr, ops
from .dino import vision_transformer as vits

__all__ = [
    "LambdaLayer", "DinoFeaturizer", "ResizeAndClassify", "ClusterLookup", "FeaturePyramidNet", "DoubleConv",
    "norm", "average_norm", "tensor_correlation", "sample", "super_perm", "sample_nonzero_locations",
    "ContrastiveCorrelationLoss", "Decoder", "NetWithActivations", "ContrastiveCRFLoss",
    "torch", "nn", "F", "np", "os", "join", "vits",
]


def _round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


# ==================================================================================================
# small pure functions (reference modules.py:275-295)
# ==================================================================================================
def norm(t):
    """modules.py:275-276."""
    return F.normalize(t, dim=1, eps=1e-10)


def average_norm(t):
    """modules.py:279-280."""
    return t / t.square().sum(1, keepdim=True).sqrt().mean()


def tensor_correlation(a, b):
    """modules.py:283-284: einsum nchw,ncij->nhwij — one [hw, C] x [C, ij] GEMM per image, all images in ONE launch of
    the batched wgmma GEMM.  fp32 inputs are split into bf16 hi + lo parts and the three significant products are
    folded into the K axis: [hi | lo | hi] . [hi | hi | lo]^T = hi.hi + lo.hi + hi.lo (fp32 accumulate, ~2^-16
    relative instead of bf16's 2^-9); bf16 inputs take a single pass.  Off-device there is no implementation."""
    if not (a.is_cuda and b.is_cuda):
        raise RuntimeError("stego_b200.tensor_correlation: CUDA tensors required (no CPU fallback)")
    n, c, h, w = a.shape
    _, _, i, j = b.shape
    exact_bf16 = a.dtype == torch.bfloat16 and b.dtype == torch.bfloat16
    cp = _round_up(c, 8)
    parts = 1 if exact_bf16 else 3

    def operand(x, rows, order):  # [n, rows, parts * cp] bf16, K-major
        x = x.reshape(n, c, rows).transpose(1, 2)
        buf = torch.zeros(n, rows, parts * cp, dtype=torch.bfloat16, device=x.device)
        if exact_bf16:
            buf[:, :, :c] = x
            return buf
        x = x.float()
        hi = x.to(torch.bfloat16)
        lo = (x - hi.float()).to(torch.bfloat16)
        for k, part in enumerate(order):
            buf[:, :, k * cp:k * cp + c] = hi if part == "hi" else lo
        return buf

    A = operand(a, h * w, ("hi", "lo", "hi"))
    Bm = operand(b, i * j, ("hi", "hi", "lo"))
    ld = _round_up(i * j, 4)  # 16-byte rows: the GEMM epilogue stores fp32 pairs
    out = torch.empty(n, h * w, ld, dtype=torch.float32, device=a.device)
    ops.gemm_batched(A, Bm, out[:, :, :i * j])
    return out[:, :, :i * j].reshape(n, h, w, i, j) if ld == i * j else out[:, :, :i * j].contiguous().reshape(n, h, w, i, j)


def sample(t: torch.Tensor, coords: torch.Tensor):
    """modules.py:287-288 (pure function kept as the torch op; the fused loss samples inside its own kernel)."""
    return F.grid_sample(t, coords.permute(0, 2, 1, 3), padding_mode='border', align_corners=True)


def super_perm(size: int, device: torch.device):
    """modules.py:291-295: randperm with fixed points bumped by one, mod size (duplicates possible).
    Same torch RNG call as the reference so the random stream stays aligned."""
    perm = torch.randperm(size, device=device, dtype=torch.long)
    bump = perm == torch.arange(size, device=device)
    return (perm + bump.to(perm.dtype)) % size


def sample_nonzero_locations(t, target_size):
    """modules.py:298-311 (salience sampling; off by default: use_salience False)."""
    nz = torch.nonzero(t)
    coords = torch.zeros(target_size, dtype=nz.dtype, device=nz.device)
    n = target_size[1] * target_size[2]
    for i in range(t.shape[0]):
        mine = nz[nz[:, 0] == i]
        if mine.shape[0] == 0:
            picked = torch.randint(t.shape[1], size=(n, 2), device=nz.device)
        else:
            picked = mine[torch.randint(len(mine), size=(n,)), 1:]
        coords[i] = picked.reshape(target_size[1], target_size[2], 2)
    coords = coords.to(torch.float32) / t.shape[1] * 2 - 1
    return torch.flip(coords, dims=[-1])


class LambdaLayer(nn.Module):
    def __init__(self, lambd):
        super().__init__()
        self.lambd = lambd

    def forward(self, x):
        return self.lambd(x)


# ==================================================================================================
# segmentation head (cluster1 + cluster2) as one autograd node over wgmma GEMMs
# ==================================================================================================
class _HeadFn(torch.autograd.Function):
    """code = conv1x1(E->D)(f*m1) + conv1x1(E->D)(relu(conv1x1(E->E)(f*m2)))   (modules.py:108-111)

    feat_tok: [M, E] bf16 tokens-major (frozen backbone output, no grad); masks: [B, E] fp32 or None.
    Output: code storage [M, P] fp32 (P = D rounded up to 8; columns >= D are padding)."""

    @staticmethod
    def forward(ctx, feat_tok, m1, m2, B, hw, w1, b1, wa, ba, wb, bb):
        M, E = feat_tok.shape
        D = w1.shape[0]
        dev = feat_tok.device
        P = _round_up(D, 8)
        nonlinear = wa is not None
        if m1 is not None:
            x1 = torch.empty_like(feat_tok)
            x2 = torch.empty_like(feat_tok) if nonlinear else None
            rc = _lib.load().stego_head_dropout3(_lib.ptr(feat_tok), _lib.ptr(m1), _lib.ptr(m2) if nonlinear else 0, 0,
                                                 _lib.ptr(x1), _lib.ptr(x2), 0, B, hw, E, _lib.stream())
            _lib.check(rc, "stego_head_dropout3")
        else:
            x1 = x2 = feat_tok
        # bf16 operand copies of the (small) trainable weights, zero-padded to 128 output rows
        w1p = torch.zeros(128, E, dtype=torch.bfloat16, device=dev)
        w1p[:D] = w1.detach().reshape(D, E)
        code = torch.zeros(M, P, dtype=torch.float32, device=dev)
        ops.gemm(x1, w1p, code, M=M, N=D, K=E, bias=b1.detach().float().contiguous())
        hid = wbp = wab = None
        if nonlinear:
            wab = wa.detach().reshape(E, E).to(torch.bfloat16).contiguous()
            wbp = torch.zeros(128, E, dtype=torch.bfloat16, device=dev)
            wbp[:D] = wb.detach().reshape(D, E)
            hid = torch.empty(M, E, dtype=torch.bfloat16, device=dev)
            ops.gemm(x2, wab, hid, M=M, N=E, K=E, bias=ba.detach().float().contiguous(), act=ops.ACT_RELU)
            ops.gemm(hid, wbp, code, M=M, N=D, K=E, bias=bb.detach().float().contiguous(), residual=code)
        ctx.save_for_backward(x1, x2 if nonlinear else None, hid, wab, wbp)
        ctx.dims = (M, E, D, P, nonlinear)
        ctx.shapes = (w1.shape, wa.shape if nonlinear else None, wb.shape if nonlinear else None)
        return code

    @staticmethod
    def backward(ctx, dcode):
        x1, x2, hid, wab, wbp = ctx.saved_tensors
        M, E, D, P, nonlinear = ctx.dims
        dev = dcode.device
        lib = _lib.load()
        dcode = dcode.contiguous() if dcode.stride(1) != 1 else dcode
        dyb = torch.empty(M, 128, dtype=torch.bfloat16, device=dev)
        _lib.check(lib.stego_cast_pad_bf16(_lib.ptr(dcode), dcode.stride(0), D, _lib.ptr(dyb), 128, M, _lib.stream()),
                   "stego_cast_pad_bf16")
        sms = torch.cuda.get_device_properties(dev).multi_processor_count

        def splits_for(out_rows, out_cols):
            tiles = ((out_rows + 127) // 128) * ((out_cols + 127) // 128)
            return max(1, min(M // 512, sms // tiles))  # tiles x splits = one wave of the persistent GEMM grid
        # bias gradient: column sums over the padded row (padding columns of d(code) are zero) -> vector loads
        db_pad = torch.zeros(P, dtype=torch.float32, device=dev)
        _lib.check(lib.stego_colsum(_lib.ptr(dcode), 0, dcode.stride(0), P if dcode.shape[1] >= P else D, M,
                                    _lib.ptr(db_pad), _lib.stream()), "stego_colsum")
        db = db_pad[:D].contiguous()
        dw1 = torch.zeros(D, E, dtype=torch.float32, device=dev)
        ops.gemm(dyb, x1, dw1, M=D, N=E, K=M, a_mn=True, b_mn=True, splits=splits_for(D, E), atomic=True)
        dwa = dba = dwb = dbb = None
        if nonlinear:
            dwb = torch.zeros(D, E, dtype=torch.float32, device=dev)
            ops.gemm(dyb, hid, dwb, M=D, N=E, K=M, a_mn=True, b_mn=True, splits=splits_for(D, E), atomic=True)
            dbb = db.clone()
            # dH = dY . Wb  (B operand [K=c][N=E] is MN-major), then ReLU backward -> bf16 operand
            dh = torch.empty(M, E, dtype=torch.float32, device=dev)
            ops.gemm(dyb, wbp, dh, M=M, N=E, K=128, b_mn=True)
            dhb = torch.empty(M, E, dtype=torch.bfloat16, device=dev)
            _lib.check(lib.stego_relu_bwd_bf16(_lib.ptr(dh), _lib.ptr(hid), _lib.ptr(dhb), M * E, _lib.stream()),
                       "stego_relu_bwd_bf16")
            dba = torch.zeros(E, dtype=torch.float32, device=dev)
            _lib.check(lib.stego_colsum(_lib.ptr(dhb), 1, E, E, M, _lib.ptr(dba), _lib.stream()), "stego_colsum")
            dwa = torch.zeros(E, E, dtype=torch.float32, device=dev)
            ops.gemm(dhb, x2, dwa, M=E, N=E, K=M, a_mn=True, b_mn=True, splits=splits_for(E, E), atomic=True)
        s1, sa, sb_ = ctx.shapes
        return (None, None, None, None, None, dw1.reshape(s1), db,
                dwa.reshape(sa) if nonlinear else None, dba, dwb.reshape(sb_) if nonlinear else None, dbb)


def _draw_dropout2d_noise(batch: int, channels: int, p: float, device) -> torch.Tensor:
    """The noise F.dropout2d / nn.Dropout2d draws for a [B,C,H,W] input (ATen _dropout_impl, feature
    dropout): empty([B,C,1,1]).bernoulli_(1-p).div_(1-p).  Same RNG consumption as the reference's three
    Dropout2d calls in DinoFeaturizer.forward (modules.py:109,111,116)."""
    return torch.empty(batch, channels, 1, 1, device=device).bernoulli_(1 - p).div_(1 - p)


class DinoFeaturizer(nn.Module):
    """modules.py:17-118.  `forward(img) -> (image_feat [B,E,h,w], code [B,dim,h,w])`."""

    _URLS = {("vit_small", 16): "dino_deitsmall16_pretrain/dino_deitsmall16_pretrain.pth",
             ("vit_small", 8): "dino_deitsmall8_300ep_pretrain/dino_deitsmall8_300ep_pretrain.pth",
             ("vit_base", 16): "dino_vitbase16_pretrain/dino_vitbase16_pretrain.pth",
             ("vit_base", 8): "dino_vitbase8_pretrain/dino_vitbase8_pretrain.pth"}

    def __init__(self, dim, cfg):
        super().__init__()
        self.cfg = cfg
        self.dim = dim
        self.patch_size = cfg.dino_patch_size
        self.feat_type = cfg.dino_feat_type
        arch = cfg.model_type
        if (arch, self.patch_size) not in self._URLS:
            raise ValueError("Unknown arch and patch size")
        self.model = vits.__dict__[arch](patch_size=self.patch_size, num_classes=0)
        for p in self.model.parameters():
            p.requires_grad = False
        self.model.eval()
        if torch.cuda.is_available():
            self.model.cuda()
        self.dropout = torch.nn.Dropout2d(p=.1)

        weights = getattr(cfg, "pretrained_weights", None)
        if weights is not None:
            sd = torch.load(weights, map_location="cpu")["teacher"]
            sd = {k.replace("module.", "").replace("backbone.", ""): v for k, v in sd.items()}
            msg = self.model.load_state_dict(sd, strict=False)
            print('Pretrained weights found at {} and loaded with msg: {}'.format(weights, msg))
        elif getattr(cfg, "random_backbone_init", False):
            print("DinoFeaturizer: keeping the random ViT initialisation (cfg.random_backbone_init).", file=sys.stderr)
        else:
            print("Since no pretrained weights have been provided, we load the reference pretrained DINO weights.")
            sd = torch.hub.load_state_dict_from_url(url="https://dl.fbaipublicfiles.com/dino/" + self._URLS[(arch, self.patch_size)])
            self.model.load_state_dict(sd, strict=True)

        self.n_feats = 384 if arch == "vit_small" else 768
        self.cluster1 = self.make_clusterer(self.n_feats)
        self.proj_type = cfg.projection_type
        if self.proj_type == "nonlinear":
            self.cluster2 = self.make_nonlinear_clusterer(self.n_feats)

    def make_clusterer(self, in_channels):
        return torch.nn.Sequential(torch.nn.Conv2d(in_channels, self.dim, (1, 1)))

    def make_nonlinear_clusterer(self, in_channels):
        return torch.nn.Sequential(torch.nn.Conv2d(in_channels, in_channels, (1, 1)), torch.nn.ReLU(),
                                   torch.nn.Conv2d(in_channels, self.dim, (1, 1)))

    # ---- fused internals -------------------------------------------------------------------------
    def backbone_tokens(self, img: torch.Tensor, use_graph: bool = False) -> torch.Tensor:
        """Frozen ViT -> bf16 tokens-major features [B, hw, E] (cls dropped).  use_graph: replay the kernel
        sequence as one CUDA graph (result is a static buffer valid until the next call)."""
        self.model.eval()
        first = img[0] if isinstance(img, (list, tuple)) else img  # a list of batches is concatenated on the fly
        assert first.shape[2] % self.patch_size == 0
        assert first.shape[3] % self.patch_size == 0
        return self.model.patch_features(img, use_graph=use_graph)

    def draw_masks(self, batch: int, device):
        """Dropout2d noises in the reference's call order: cluster1 input, cluster2 input, returned feats."""
        if not self.training:
            return None, None, None
        E = self.n_feats
        m1 = m2 = m3 = None
        if self.proj_type is not None:
            m1 = _draw_dropout2d_noise(batch, E, 0.1, device).view(batch, E)
            if self.proj_type == "nonlinear":
                m2 = _draw_dropout2d_noise(batch, E, 0.1, device).view(batch, E)
        if self.cfg.dropout:
            m3 = _draw_dropout2d_noise(batch, E, 0.1, device).view(batch, E)
        return m1, m2, m3

    def head_code(self, feat_tok: torch.Tensor, m1, m2, fh: int, fw: int) -> torch.Tensor:
        """cluster1 (+ cluster2) on tokens-major features -> code [B, dim, h, w] (view of padded storage)."""
        B, hw, E = feat_tok.shape
        c1 = self.cluster1[0]
        if self.proj_type == "nonlinear":
            ca, cb = self.cluster2[0], self.cluster2[2]
            store = _HeadFn.apply(feat_tok.reshape(B * hw, E), m1, m2, B, hw, c1.weight, c1.bias, ca.weight, ca.bias,
                                  cb.weight, cb.bias)
        else:
            store = _HeadFn.apply(feat_tok.reshape(B * hw, E), m1, None, B, hw, c1.weight, c1.bias, None, None, None,
                                  None)
        return store.view(B, fh, fw, -1)[..., :self.dim].permute(0, 3, 1, 2)

    # ---- reference entry point -------------------------------------------------------------------
    def forward(self, img, n=1, return_class_feat=False):
        self.model.eval()
        assert (img.shape[2] % self.patch_size == 0)
        assert (img.shape[3] % self.patch_size == 0)
        fh, fw = img.shape[2] // self.patch_size, img.shape[3] // self.patch_size
        B = img.shape[0]
        with torch.no_grad():
            if return_class_feat:
                return self.model(img).reshape(B, 1, 1, -1).permute(0, 3, 1, 2)
            if self.feat_type == "feat":
                tok = self.model.patch_features(img)  # [B, hw, E] bf16
            elif self.feat_type == "KK":
                _, _, qkv = self.model.get_intermediate_feat(img, n=n)
                k = qkv[0][1, :, :, 1:, :]  # [B, heads, hw, 64]
                tok = k.permute(0, 2, 1, 3).reshape(B, fh * fw, -1).to(torch.bfloat16).contiguous()
            else:
                raise ValueError("Unknown feat type:{}".format(self.feat_type))
        E = tok.shape[-1]
        m1, m2, m3 = self.draw_masks(B, img.device)
        if self.proj_type is not None:
            code = self.head_code(tok, m1, m2, fh, fw)
        else:
            code = tok.float().view(B, fh, fw, E).permute(0, 3, 1, 2)
        image_feat = tok.float().view(B, fh, fw, E).permute(0, 3, 1, 2)  # NCHW view of tokens-major storage
        if self.cfg.dropout and m3 is not None:
            image_feat = image_feat * m3.view(B, E, 1, 1)
        return image_feat, code


# ==================================================================================================
# ContrastiveCorrelationLoss (modules.py:314-398)
# ==================================================================================================
class ContrastiveCorrelationLoss(nn.Module):

    def __init__(self, cfg, ):
        super().__init__()
        self.cfg = cfg

    def standard_scale(self, t):
        t1 = t - t.mean()
        return t1 / t1.std()

    def draw_coords(self, orig_feats, orig_salience, orig_salience_pos):
        """RNG consumption identical to modules.py:353-367."""
        fs = self.cfg.feature_samples
        shape = [orig_feats.shape[0], fs, fs, 2]
        dev = orig_feats.device
        if self.cfg.use_salience:
            nz1 = sample_nonzero_locations(orig_salience, shape)
            nz2 = sample_nonzero_locations(orig_salience_pos, shape)
            reg1 = torch.rand(shape, device=dev) * 2 - 1
            reg2 = torch.rand(shape, device=dev) * 2 - 1
            mask = (torch.rand(shape[:-1], device=dev) > .1).unsqueeze(-1).to(torch.float32)
            return nz1 * mask + reg1 * (1 - mask), nz2 * mask + reg2 * (1 - mask)
        return torch.rand(shape, device=dev) * 2 - 1, torch.rand(shape, device=dev) * 2 - 1

    def forward(self, orig_feats: torch.Tensor, orig_feats_pos: torch.Tensor, orig_salience: torch.Tensor,
                orig_salience_pos: torch.Tensor, orig_code: torch.Tensor, orig_code_pos: torch.Tensor):
        cfg = self.cfg
        coords1, coords2 = self.draw_coords(orig_feats, orig_salience, orig_salience_pos)
        B = orig_feats.shape[0]
        perms = [super_perm(B, orig_feats.device) for _ in range(cfg.neg_samples)]
        spec = corr.make_spec(cfg)
        losses, _cd_means, cd, elems = corr.corr_loss(orig_feats, orig_feats_pos, orig_code, orig_code_pos, coords1,
                                                      coords2, perms, spec, want_elems=True)
        fs = cfg.feature_samples
        five = (fs, fs, fs, fs)
        neg = cfg.neg_samples
        return (losses[0],
                cd[0].reshape(B, *five),
                losses[1],
                cd[1].reshape(B, *five),
                elems[2:].reshape(neg * B, *five),
                cd[2:].reshape(neg * B, *five))


# ==================================================================================================
# ClusterLookup (modules.py:134-161)
# ==================================================================================================
class _ClusterLookupFn(torch.autograd.Function):

    @staticmethod
    def forward(ctx, x, clusters, alpha, want_probs, want_logp):
        B, C, H, W = x.shape
        n = clusters.shape[0]
        dev = x.device
        xf = x.detach()
        if xf.dtype != torch.float32:
            xf = xf.float()
        # the pixel index y*W + x must map to ONE stride: true for NCHW-contiguous and channels-last views
        if xf.stride(2) != W * xf.stride(3):
            xf = xf.contiguous()
        cl = clusters.detach().float().contiguous()
        loss = torch.empty(2, dtype=torch.float32, device=dev)
        scratch = torch.empty(16 * torch.cuda.get_device_properties(dev).multi_processor_count, dtype=torch.float32,
                              device=dev)
        probs = torch.empty(B, n, H, W, dtype=torch.float32, device=dev) if want_probs else None
        logp = torch.empty(B, n, H, W, dtype=torch.float32, device=dev) if want_logp else None
        rc = _lib.load().stego_cluster_lookup_fwd(
            _lib.ptr(xf), xf.stride(0), xf.stride(1), xf.stride(3), _lib.ptr(cl), B, C, n, H * W,
            int(alpha is not None), float(alpha) if alpha is not None else 0.0, 0, _lib.ptr(probs), _lib.ptr(logp),
            _lib.ptr(loss), _lib.ptr(scratch), _lib.stream())
        _lib.check(rc, "stego_cluster_lookup_fwd")
        ctx.save_for_backward(xf, cl)
        ctx.alpha = alpha
        ctx.shape = clusters.shape
        if want_probs:
            ctx.mark_non_differentiable(probs)
        if want_logp:
            ctx.mark_non_differentiable(logp)
        return loss[0], probs, logp

    @staticmethod
    def backward(ctx, g_loss, _gp, _gl):
        xf, cl = ctx.saved_tensors
        B, C, H, W = xf.shape
        n = cl.shape[0]
        dnc = torch.zeros(n, C, dtype=torch.float32, device=xf.device)
        dcl = torch.zeros(n, C, dtype=torch.float32, device=xf.device)
        alpha = ctx.alpha
        g = (g_loss if g_loss is not None else torch.zeros((), device=xf.device)).to(torch.float32).reshape(1).contiguous()
        rc = _lib.load().stego_cluster_lookup_bwd(
            _lib.ptr(xf), xf.stride(0), xf.stride(1), xf.stride(3), _lib.ptr(cl), B, C, n, H * W,
            int(alpha is not None), float(alpha) if alpha is not None else 0.0, _lib.ptr(g), _lib.ptr(dnc), _lib.ptr(dcl),
            _lib.stream())
        _lib.check(rc, "stego_cluster_lookup_bwd")
        return None, dcl.reshape(ctx.shape), None, None, None


class ClusterLookup(nn.Module):
    """modules.py:134-161.  Differentiable wrt `clusters`; `x` is treated as a constant (the reference only
    ever passes detached / no-grad features: train_segmentation.py:212,222, eval_segmentation.py:131)."""

    def __init__(self, dim: int, n_classes: int):
        super().__init__()
        self.n_classes = n_classes
        self.dim = dim
        self.clusters = torch.nn.Parameter(torch.randn(n_classes, dim))

    def reset_parameters(self):
        with torch.no_grad():
            self.clusters.copy_(torch.randn(self.n_classes, self.dim))

    def forward(self, x, alpha, log_probs=False):
        if not x.is_cuda:
            raise RuntimeError("stego_b200.ClusterLookup: CUDA tensors required (no CPU fallback)")
        if x.requires_grad and torch.is_grad_enabled():
            raise RuntimeError("stego_b200.ClusterLookup: gradients wrt the features are not implemented "
                               "(STEGO always detaches them); detach x")
        if log_probs:
            if alpha is None:
                raise TypeError("log_probs=True needs a numeric alpha (as in the reference)")
            _, _, logp = _ClusterLookupFn.apply(x, self.clusters, alpha, False, True)
            return logp
        loss, probs, _ = _ClusterLookupFn.apply(x, self.clusters, alpha, True, False)
        return loss, probs


# ==================================================================================================
# API-surface-only modules (plain torch; not on the measured path)
# ==================================================================================================
class ResizeAndClassify(nn.Module):
    """modules.py:121-131."""

    def __init__(self, dim: int, size: int, n_classes: int):
        super().__init__()
        self.size = size
        self.predictor = torch.nn.Sequential(torch.nn.Conv2d(dim, n_classes, (1, 1)), torch.nn.LogSoftmax(1))

    def forward(self, x):
        return F.interpolate(self.predictor.forward(x), self.size, mode="bilinear", align_corners=False)


class DoubleConv(nn.Module):
    """modules.py:255-272: (conv3x3 -> BN -> ReLU) x 2."""

    def __init__(self, in_channels, out_channels, mid_channels=None):
        super().__init__()
        mid = mid_channels or out_channels
        layers = []
        for cin, cout in ((in_channels, mid), (mid, out_channels)):
            layers += [nn.Conv2d(cin, cout, kernel_size=3, padding=1), nn.BatchNorm2d(cout), nn.ReLU()]
        self.double_conv = nn.Sequential(*layers)

    def forward(self, x):
        return self.double_conv(x)


class FeaturePyramidNet(nn.Module):
    """modules.py:164-252: ResNet-activation pyramid decoder (cfg.arch == 'feature-pyramid').  Kept for API
    completeness with stock torch ops; STEGO's shipped configuration uses the DINO path."""

    @staticmethod
    def _helper(x):
        return F.interpolate(x, 56, mode="bilinear", align_corners=False).unsqueeze(-1)

    def make_clusterer(self, in_channels):
        return torch.nn.Sequential(torch.nn.Conv2d(in_channels, self.dim, (1, 1)), LambdaLayer(FeaturePyramidNet._helper))

    def make_nonlinear_clusterer(self, in_channels):
        return torch.nn.Sequential(torch.nn.Conv2d(in_channels, in_channels, (1, 1)), torch.nn.ReLU(),
                                   torch.nn.Conv2d(in_channels, in_channels, (1, 1)), torch.nn.ReLU(),
                                   torch.nn.Conv2d(in_channels, self.dim, (1, 1)), LambdaLayer(FeaturePyramidNet._helper))

    def __init__(self, granularity, cut_model, dim, continuous):
        super().__init__()
        self.layer_nums = [5, 6, 7]
        self.spatial_resolutions = [7, 14, 28, 56]
        self.feat_channels = [2048, 1024, 512, 3]
        self.extra_channels = [128, 64, 32, 32]
        self.granularity = granularity
        self.encoder = NetWithActivations(cut_model, self.layer_nums)
        self.dim = dim
        self.continuous = continuous
        self.n_feats = self.dim
        self.up = nn.Upsample(scale_factor=2, mode='bilinear', align_corners=False)
        assert granularity in {1, 2, 3, 4}
        self.cluster1 = self.make_clusterer(self.feat_channels[0])
        self.cluster1_nl = self.make_nonlinear_clusterer(self.feat_channels[0])
        # decoder stage k fuses the upsampled previous stage with encoder activation k (or the image at stage 4)
        prev = self.feat_channels[0]
        for level in (2, 3, 4):
            if granularity >= level:
                out_ch = self.extra_channels[level - 1]
                setattr(self, f"conv{level}", DoubleConv(prev + self.feat_channels[level - 1], out_ch))
                setattr(self, f"cluster{level}", self.make_clusterer(out_ch))
                prev = out_ch

    def c(self, x, y):
        return torch.cat([x, y], dim=1)

    def forward(self, x):
        with torch.no_grad():
            feats = self.encoder(x)
        low_res_feats = feats[self.layer_nums[-1]]
        all_clusters = [self.cluster1(low_res_feats)]
        if self.granularity >= 2:
            f1_up = self.up(low_res_feats)
            f2 = self.conv2(self.c(f1_up, feats[self.layer_nums[-2]]))
            all_clusters.append(self.cluster2(f2))
        if self.granularity >= 3:
            f3 = self.conv3(self.c(self.up(f2), feats[self.layer_nums[-3]]))
            all_clusters.append(self.cluster3(f3))
        if self.granularity >= 4:
            f4 = self.conv4(self.c(self.up(f3), F.interpolate(x, 56, mode="bilinear", align_corners=False)))
            all_clusters.append(self.cluster4(f4))
        avg_code = torch.cat(all_clusters, 4).mean(4)
        if self.continuous:
            clusters = avg_code
        else:
            clusters = torch.log_softmax(avg_code, 1)
        return low_res_feats, clusters


class Decoder(nn.Module):
    """modules.py:401-413."""

    def __init__(self, code_channels, feat_channels):
        super().__init__()
        self.linear = torch.nn.Conv2d(code_channels, feat_channels, (1, 1))
        self.nonlinear = torch.nn.Sequential(torch.nn.Conv2d(code_channels, code_channels, (1, 1)), torch.nn.ReLU(),
                                             torch.nn.Conv2d(code_channels, code_channels, (1, 1)), torch.nn.ReLU(),
                                             torch.nn.Conv2d(code_channels, feat_channels, (1, 1)))

    def forward(self, x):
        return self.linear(x) + self.nonlinear(x)


class NetWithActivations(torch.nn.Module):
    """modules.py:416-434: run a sequential model and collect the activations of selected children."""

    def __init__(self, model, layer_nums):
        super().__init__()
        self.layers = nn.ModuleList(model.children())
        self.layer_nums = [ln if ln >= 0 else len(self.layers) + ln for ln in layer_nums]
        self.layer_nums = set(sorted(self.layer_nums))

    def forward(self, x):
        activations = {}
        for ln, l in enumerate(self.layers):
            x = l(x)
            if ln in self.layer_nums:
                activations[ln] = x
        return activations


class _PixelCosineFn(torch.autograd.Function):
    """cos[b, y, x] = <normalize(a)[b, :, y, x], normalize(b)[b, :, y, x]> (F.normalize eps 1e-10, modules.py:275-276): one
    read of each operand in the forward, one in the backward (csrc/cosine_loss.cu)."""

    @staticmethod
    def forward(ctx, a, b):
        _lib.require_cuda(a, b)
        lib = _lib.load()
        a32, b32 = a.detach().float(), b.detach().float()
        B, C, H, W = a32.shape
        assert b32.shape == a32.shape
        cosv = torch.empty(B, H, W, dtype=torch.float32, device=a.device)
        inva, invb = torch.empty_like(cosv), torch.empty_like(cosv)
        _lib.check(lib.stego_cosine_fwd(_lib.ptr(a32), *a32.stride(), _lib.ptr(b32), *b32.stride(), B, C, H, W, 1e-10,
                                        _lib.ptr(cosv), _lib.ptr(inva), _lib.ptr(invb), _lib.stream()), "stego_cosine_fwd")
        ctx.save_for_backward(a32, b32, cosv, inva, invb)
        return cosv

    @staticmethod
    def backward(ctx, g):
        a32, b32, cosv, inva, invb = ctx.saved_tensors
        lib = _lib.load()
        B, C, H, W = a32.shape
        need_a, need_b = ctx.needs_input_grad
        da = torch.empty_strided(a32.shape, a32.stride(), dtype=torch.float32, device=a32.device) if need_a else None
        db = torch.empty_strided(b32.shape, b32.stride(), dtype=torch.float32, device=b32.device) if need_b else None
        if not (need_a or need_b):
            return None, None
        _lib.check(lib.stego_cosine_bwd(_lib.ptr(a32), *a32.stride(), _lib.ptr(b32), *b32.stride(), B, C, H, W, 1e-10,
                                        _lib.ptr(cosv), _lib.ptr(inva), _lib.ptr(invb), _lib.ptr(g.float().contiguous()),
                                        _lib.ptr(da), _lib.ptr(db), _lib.stream()), "stego_cosine_bwd")
        return da, db


def pixel_cosine(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """`(norm(a) * norm(b)).sum(1)` of the reference's optional alignment terms (train_segmentation.py:185,194-198) -> [B, h, w]."""
    return _PixelCosineFn.apply(a, b)


class _CrfLossFn(torch.autograd.Function):
    """Fused pairwise-kernel x Gram product of ContrastiveCRFLoss (csrc/crf_loss.cu); gradient w.r.t. `clusters` only
    (the reference's guidance is the resized input image: no gradient ever flows into it)."""

    @staticmethod
    def forward(ctx, guidance, clusters, coords, alpha, beta, gamma, w1, w2, shift):
        _lib.require_cuda(guidance, clusters, coords)
        lib = _lib.load()
        B, C, H, W = clusters.shape
        n = coords.shape[1]
        NP = _round_up(n, 64)
        g = guidance.detach().float()
        c = clusters.detach().float()
        coords = coords.contiguous()
        dev = c.device
        sel = torch.empty(B, C, NP, dtype=torch.float32, device=dev)
        gsel = torch.empty(B, NP, 4, dtype=torch.float32, device=dev)
        pos = torch.empty(NP, 2, dtype=torch.int32, device=dev)
        out = torch.empty(B, n, n, dtype=torch.float32, device=dev)
        _lib.check(lib.stego_crf_loss_fwd(_lib.ptr(g), *g.stride(), g.shape[1], _lib.ptr(c), *c.stride(), C, _lib.ptr(coords),
                                          B, n, H, W, float(alpha), float(beta), float(gamma), float(w1), float(w2),
                                          float(shift), _lib.ptr(sel), _lib.ptr(gsel), _lib.ptr(pos), _lib.ptr(out),
                                          _lib.stream()), "stego_crf_loss_fwd")
        ctx.save_for_backward(sel, gsel, pos, coords)
        ctx.meta = (B, C, H, W, n, float(alpha), float(beta), float(gamma), float(w1), float(w2), float(shift))
        return out

    @staticmethod
    def backward(ctx, grad_out):
        sel, gsel, pos, coords = ctx.saved_tensors
        B, C, H, W, n, alpha, beta, gamma, w1, w2, shift = ctx.meta
        lib = _lib.load()
        go = grad_out.float().contiguous()
        dsel = torch.empty_like(sel)
        dclusters = torch.zeros(B, C, H, W, dtype=torch.float32, device=sel.device)
        _lib.check(lib.stego_crf_loss_bwd(_lib.ptr(go), _lib.ptr(sel), _lib.ptr(gsel), _lib.ptr(pos), _lib.ptr(coords), B, C, n,
                                          alpha, beta, gamma, w1, w2, shift, _lib.ptr(dsel), _lib.ptr(dclusters),
                                          *dclusters.stride(), _lib.stream()), "stego_crf_loss_bwd")
        return None, dclusters, None, None, None, None, None, None, None


class ContrastiveCRFLoss(nn.Module):
    """modules.py:437-469: same constructor, same two `torch.randint` draws (row indices, then column indices) in the same
    order on the same device, same [B, n_samples, n_samples] result; the pairwise kernel, the Gram matrix of the selected
    code vectors and their product are one fused kernel (and one for the backward) instead of eight [B, n, n] temporaries."""

    def __init__(self, n_samples, alpha, beta, gamma, w1, w2, shift):
        super().__init__()
        self.alpha, self.beta, self.gamma = alpha, beta, gamma
        self.w1, self.w2 = w1, w2
        self.n_samples = n_samples
        self.shift = shift

    def draw_coords(self, h: int, w: int, device) -> torch.Tensor:
        return torch.cat([torch.randint(0, h, size=[1, self.n_samples], device=device),
                          torch.randint(0, w, size=[1, self.n_samples], device=device)], 0)

    def forward_with_coords(self, guidance, clusters, coords):
        """The loss for caller-supplied sample positions (int64 [2, n]: row indices, column indices).  The kernels index
        with them unchecked, so they are validated here (one device sync; `forward` draws them in range and skips this)."""
        h, w = guidance.shape[2], guidance.shape[3]
        if coords.dim() != 2 or coords.shape[0] != 2 or coords.dtype != torch.long:
            raise ValueError("ContrastiveCRFLoss: coords must be an int64 [2, n] tensor")
        if bool(((coords[0] < 0) | (coords[0] >= h) | (coords[1] < 0) | (coords[1] >= w)).any()):
            raise ValueError("ContrastiveCRFLoss: sample positions outside the feature map")
        return self._apply_kernel(guidance, clusters, coords)

    def _apply_kernel(self, guidance, clusters, coords):
        return _CrfLossFn.apply(guidance, clusters, coords, self.alpha, self.beta, self.gamma, self.w1, self.w2, self.shift)

    def forward(self, guidance, clusters):
        if not clusters.is_cuda:
            raise RuntimeError("stego_b200.ContrastiveCRFLoss: CUDA tensors required (no CPU fallback)")
        assert guidance.shape[0] == clusters.shape[0]
        assert guidance.shape[2:] == clusters.shape[2:]
        coords = self.draw_coords(guidance.shape[2], guidance.shape[3], clusters.device)
        return self._apply_kernel(guidance, clusters, coords)
