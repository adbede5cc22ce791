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
# segmentation head (cluster1 + cluster2): stage functions over caller-owned buffers (they allocate nothing, so the
# fused step captures them in its CUDA graph) and the autograd node.  Linear head: every cluster2 argument is None.
# ==================================================================================================
def pack_head_weights(w1, wa, wb, w1p, wab, wbp) -> None:
    """bf16 operand copies of the trainable head weights: w1 / wb into the first D rows of w1p / wbp [128, E] (rows
    >= D must be zero: the dgrad GEMM reads all 128), wa into wab [E, E]."""
    D = w1.shape[0]
    w1p[:D].copy_(w1.detach().reshape(D, -1))
    if wab is not None:
        wab.copy_(wa.detach().reshape(wab.shape))
        wbp[:D].copy_(wb.detach().reshape(D, -1))


def head_forward(feat_tok, m1, m2, B, hw, x1, x2, hid, code, w1p, b1, wab=None, ba=None, wbp=None, bb=None) -> None:
    """code = conv1x1(E->D)(f*m1) + conv1x1(E->D)(relu(conv1x1(E->E)(f*m2)))   (modules.py:108-111)

    feat_tok: [M = B*hw, E] bf16 tokens-major; m1 / m2: [B, E] fp32 Dropout2d noises (x1 / x2 receive f*m1 / f*m2), or
    None with x1 = x2 = feat_tok.  code: [M, P] fp32 with zero padding columns (P = D rounded up to 8)."""
    M, E = feat_tok.shape
    D = b1.shape[0]
    if m1 is not None:
        _lib.check(_lib.load().stego_head_dropout3(_lib.ptr(feat_tok), _lib.ptr(m1), _lib.ptr(m2), 0, _lib.ptr(x1),
                                                   _lib.ptr(x2), 0, B, hw, E, _lib.stream()), "stego_head_dropout3")
    ops.gemm(x1, w1p, code, M=M, N=D, K=E, bias=b1)
    if wab is not None:
        ops.gemm(x2, wab, hid, M=M, N=E, K=E, bias=ba, act=ops.ACT_RELU)
        ops.gemm(hid, wbp, code, M=M, N=D, K=E, bias=bb, residual=code)


def head_backward(dcode, x1, x2, hid, wbp, dyb, db_pad, dh, dhb, dw1, db1, dwa, dba, dwb, dbb) -> None:
    """The six parameter gradients (in the parameters' shapes) from d(code) [M, >= D] (columns contiguous).  Scratch:
    dyb [M, 128] bf16, d(code) padded for the GEMMs; db_pad [P], the column sum of d(code) (over its zero padding
    columns too when it has them: vector loads), copied into both D-wide bias gradients db1 and dbb; dh / dhb [M, E],
    d(hidden) before / after the ReLU.  db_pad, dw1, dwa, dba and dwb are accumulated into and must arrive zeroed."""
    M, E = x1.shape
    D, P, ld = db1.shape[0], db_pad.shape[0], dcode.stride(0)
    lib, st = _lib.load(), _lib.stream()
    sms = torch.cuda.get_device_properties(dcode.device).multi_processor_count
    wgrad = lambda a, b, out, rows: ops.gemm(a, b, out.view(rows, E), M=rows, N=E, K=M, a_mn=True, b_mn=True,
                                             splits=ops.wgrad_splits(M, rows, E, sms), atomic=True)
    _lib.check(lib.stego_cast_pad_bf16(_lib.ptr(dcode), ld, D, _lib.ptr(dyb), 128, M, st), "stego_cast_pad_bf16")
    _lib.check(lib.stego_colsum(_lib.ptr(dcode), 0, ld, P if dcode.shape[1] >= P else D, M, _lib.ptr(db_pad), st),
               "stego_colsum")
    db1.copy_(db_pad[:D])
    wgrad(dyb, x1, dw1, D)
    if hid is not None:
        dbb.copy_(db_pad[:D])
        wgrad(dyb, hid, dwb, D)
        # dH = dY . Wb  (B operand [K=c][N=E] is MN-major), then ReLU backward -> bf16 operand
        ops.gemm(dyb, wbp, dh, M=M, N=E, K=128, b_mn=True)
        _lib.check(lib.stego_relu_bwd_bf16(_lib.ptr(dh), _lib.ptr(hid), _lib.ptr(dhb), M * E, st), "stego_relu_bwd_bf16")
        _lib.check(lib.stego_colsum(_lib.ptr(dhb), 1, E, E, M, _lib.ptr(dba), st), "stego_colsum")
        wgrad(dhb, x2, dwa, E)


class _HeadFn(torch.autograd.Function):
    """head_forward / head_backward over per-call buffers.  feat_tok: [M, E] bf16 (no grad); masks: [B, E] fp32 or
    None.  Output: code storage [M, P] fp32 (columns >= D are padding)."""

    @staticmethod
    def forward(ctx, feat_tok, m1, m2, B, hw, w1, b1, wa, ba, wb, bb):
        M, E = feat_tok.shape
        nonlinear = wa is not None
        bf16 = dict(dtype=torch.bfloat16, device=feat_tok.device)
        w1p = torch.zeros(128, E, **bf16)
        wab, wbp, hid = (torch.empty(E, E, **bf16), torch.zeros(128, E, **bf16), torch.empty(M, E, **bf16)) \
            if nonlinear else (None, None, None)
        pack_head_weights(w1, wa, wb, w1p, wab, wbp)
        x1 = x2 = feat_tok
        if m1 is not None:
            x1, x2 = torch.empty_like(feat_tok), torch.empty_like(feat_tok) if nonlinear else None
        code = torch.zeros(M, _round_up(w1.shape[0], 8), dtype=torch.float32, device=feat_tok.device)
        f32 = lambda t: t.detach().float().contiguous() if t is not None else None
        head_forward(feat_tok, m1, m2, B, hw, x1, x2, hid, code, w1p, f32(b1), wab, f32(ba), wbp, f32(bb))
        ctx.save_for_backward(x1, x2 if nonlinear else None, hid, wbp)
        ctx.shapes = [p.shape if p is not None else None for p in (w1, b1, wa, ba, wb, bb)]
        return code

    @staticmethod
    def backward(ctx, dcode):
        x1, x2, hid, wbp = ctx.saved_tensors
        s1, sb1, sa, sba, sb, sbb = ctx.shapes
        f32 = dict(dtype=torch.float32, device=dcode.device)
        dcode = dcode.contiguous() if dcode.stride(1) != 1 else dcode
        dyb = torch.empty(x1.shape[0], 128, dtype=torch.bfloat16, device=dcode.device)
        db_pad = torch.zeros(_round_up(s1[0], 8), **f32)
        dw1, db1 = torch.zeros(s1, **f32), torch.empty(sb1, **f32)
        dwa = dba = dwb = dbb = dh = dhb = None
        if hid is not None:
            dwa, dba, dwb, dbb = torch.zeros(sa, **f32), torch.zeros(sba, **f32), torch.zeros(sb, **f32), torch.empty(sbb, **f32)
            dh, dhb = torch.empty(x1.shape, **f32), torch.empty_like(x1)
        head_backward(dcode, x1, x2, hid, wbp, dyb, db_pad, dh, dhb, dw1, db1, dwa, dba, dwb, dbb)
        return (None,) * 5 + (dw1, db1, dwa, dba, dwb, dbb)


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
    def backbone_tokens(self, img: torch.Tensor, use_graph: bool = False, mirror: bool = False) -> torch.Tensor:
        """Frozen ViT -> bf16 tokens-major teacher features [B, hw, E] (cls dropped): the final-norm tokens for
        dino_feat_type "feat", the last block's keys (head-major channels) for "KK" — the tensor forward() returns
        as image_feat, which both training paths feed to the head and the correspondence loss.  use_graph: replay the
        kernel sequence as one CUDA graph (result is a static buffer valid until the next call).  mirror: [2B, hw, E],
        the tokens of img and then of img.flip(3) from one pass (VisionTransformer.patch_features)."""
        self.model.eval()
        first = img[0] if isinstance(img, (list, tuple)) else img  # a list of batches is concatenated on the fly
        assert first.shape[2] % self.patch_size == 0
        assert first.shape[3] % self.patch_size == 0
        if self.feat_type == "feat":
            return self.model.patch_features(img, use_graph=use_graph, mirror=mirror)
        if self.feat_type == "KK":
            return self.model.key_features(img, use_graph=use_graph, mirror=mirror)
        raise ValueError("Unknown feat type:{}".format(self.feat_type))

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

    def head_params(self):
        """(w1, b1, wa, ba, wb, bb): cluster1 and the two convs of cluster2, whose entries are None for the linear head."""
        c1 = self.cluster1[0]
        if self.proj_type != "nonlinear":
            return c1.weight, c1.bias, None, None, None, None
        ca, cb = self.cluster2[0], self.cluster2[2]
        return c1.weight, c1.bias, ca.weight, ca.bias, cb.weight, cb.bias

    def head_code(self, feat_tok: torch.Tensor, m1, m2, fh: int, fw: int) -> torch.Tensor:
        """cluster1 (+ cluster2) on tokens-major features -> code [B, dim, h, w] (view of padded storage)."""
        B, hw, E = feat_tok.shape
        m2 = m2 if self.proj_type == "nonlinear" else None
        store = _HeadFn.apply(feat_tok.reshape(B * hw, E), m1, m2, B, hw, *self.head_params())
        return store.view(B, fh, fw, -1)[..., :self.dim].permute(0, 3, 1, 2)

    def eval_code(self, feat_tok: torch.Tensor, fh: int, fw: int) -> torch.Tensor:
        """The eval-mode code [B, C, h, w] of tokens-major features: the head's, or with projection_type None the
        features themselves (modules.py:108-113), as a bf16 view of feat_tok that the probe kernels read in place."""
        if self.proj_type is not None:
            return self.head_code(feat_tok, None, None, fh, fw)
        B, _, E = feat_tok.shape
        return feat_tok.view(B, fh, fw, E).permute(0, 3, 1, 2)

    # ---- reference entry point -------------------------------------------------------------------
    def forward(self, img, n=1, return_class_feat=False):
        self.model.eval()
        assert (img.shape[2] % self.patch_size == 0)
        assert (img.shape[3] % self.patch_size == 0)
        fh, fw = img.shape[2] // self.patch_size, img.shape[3] // self.patch_size
        B = img.shape[0]
        if n < 1:
            raise ValueError("DinoFeaturizer: n must be >= 1 (block depth - n is read)")
        with torch.no_grad():
            # n = 1 reads the last block; n > 1 block depth - n (block 0 once n >= depth), as feat[0] / qkv[0] of
            # get_intermediate_feat(img, n) do in the reference.  Attention matrices are never computed here.
            if return_class_feat:
                if n == 1:
                    return self.model(img).reshape(B, 1, 1, -1).permute(0, 3, 1, 2)
                x = self.model.block_taps(img, n).x[0]
                return self.model.final_norm(x, B)[:, 0].float().reshape(B, 1, 1, -1).permute(0, 3, 1, 2)
            if self.feat_type == "feat":
                if n == 1:
                    tok = self.model.patch_features(img)  # [B, hw, E] bf16
                else:
                    tok = self.model.final_norm(self.model.block_taps(img, n).x[0], B)[:, 1:].contiguous()
            elif self.feat_type == "KK":
                if n == 1:
                    tok = self.model.key_features(img)  # [B, hw, heads*64] bf16, head-major; the last block stops at k
                else:
                    qkv = self.model.block_taps(img, n).qkv[0]  # packed bf16 [B*N, 3E]: k is the middle third
                    tok = qkv.view(B, fh * fw + 1, 3, -1)[:, 1:, 1].contiguous()  # [B, hw, heads*64], head-major
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
        # any_teacher: like the reference, the teacher signal may be of any width and resolution, e.g. the one-hot label
        # maps of use_true_labels ([B, n_classes + 1, H, W] at label resolution, train_segmentation.py:135-137)
        losses, _cd_means, cd, elems = corr.corr_loss(orig_feats, orig_feats_pos, orig_code, orig_code_pos, coords1,
                                                      coords2, perms, spec, want_elems=True, any_teacher=True)
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
def cluster_lookup_forward(x, clusters, alpha, loss, scratch, probs=None, log_probs=None) -> None:
    """ClusterLookup.forward (modules.py:146-161) of x, an fp32 [B, C, H, W] view whose pixel y*W + x is ONE stride,
    into loss[0] (and the optional probs / log_probs [B, n, H, W]); alpha None is the one-hot argmax."""
    B, C, H, W = x.shape
    _lib.check(_lib.load().stego_cluster_lookup_fwd(
        _lib.ptr(x), x.stride(0), x.stride(1), x.stride(3), _lib.ptr(clusters), B, C, clusters.shape[0], H * W,
        int(alpha is not None), float(alpha) if alpha is not None else 0.0, 0, _lib.ptr(probs), _lib.ptr(log_probs),
        _lib.ptr(loss), _lib.ptr(scratch), _lib.stream()), "stego_cluster_lookup_fwd")


def cluster_lookup_backward(x, clusters, alpha, grad_loss, dnc, dclusters) -> None:
    """dclusters += grad_loss[0] * d(loss)/d(clusters); dclusters and the scratch dnc must arrive zeroed."""
    B, C, H, W = x.shape
    _lib.check(_lib.load().stego_cluster_lookup_bwd(
        _lib.ptr(x), x.stride(0), x.stride(1), x.stride(3), _lib.ptr(clusters), B, C, clusters.shape[0], H * W,
        int(alpha is not None), float(alpha) if alpha is not None else 0.0, _lib.ptr(grad_loss), _lib.ptr(dnc),
        _lib.ptr(dclusters), _lib.stream()), "stego_cluster_lookup_bwd")


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
        probs = torch.empty(B, n, H, W, dtype=torch.float32, device=dev) if want_probs else None
        logp = torch.empty(B, n, H, W, dtype=torch.float32, device=dev) if want_logp else None
        cluster_lookup_forward(xf, cl, alpha, loss, ops.probe_scratch(dev), probs, logp)
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
        dnc = torch.zeros(cl.shape, dtype=torch.float32, device=xf.device)
        dcl = torch.zeros(cl.shape, dtype=torch.float32, device=xf.device)
        g = (g_loss if g_loss is not None else torch.zeros((), device=xf.device)).to(torch.float32).reshape(1).contiguous()
        cluster_lookup_backward(xf, cl, ctx.alpha, g, dnc, dcl)
        return None, dcl.reshape(ctx.shape), None, None, None


class _ClusterLookupWideFn(torch.autograd.Function):
    """ClusterLookup's alpha None loss (the training step's cluster probe) on a wide code: the backbone's 384 / 768
    channels of projection_type None.  Loss and gradient come from one call of stego_cluster_lookup_wide (fixed-order
    reductions); backward scales the gradient by the upstream one."""

    @staticmethod
    def forward(ctx, x, clusters):
        B, C, H, W = x.shape
        n = clusters.shape[0]
        dev = x.device
        xt = ops.tokens_major(x)
        rows = B * H * W
        cl = clusters.detach().float().contiguous()
        loss = torch.empty(2, dtype=torch.float32, device=dev)
        dnc = torch.zeros(n, C, dtype=torch.float32, device=dev)
        dcl = torch.zeros(n, C, dtype=torch.float32, device=dev)
        assign = torch.empty(rows, dtype=torch.int32, device=dev)
        inv = torch.empty(rows, dtype=torch.float32, device=dev)
        _lib.check(_lib.load().stego_cluster_lookup_wide(
            _lib.ptr(xt), xt.stride(3), rows, C, _lib.ptr(cl), n, _lib.ptr(assign), _lib.ptr(inv),
            _lib.ptr(ops.probe_scratch(dev)), _lib.ptr(loss), _lib.ptr(dnc), _lib.ptr(dcl), _lib.stream()),
            "stego_cluster_lookup_wide")
        ctx.save_for_backward(dcl)
        ctx.shape = clusters.shape
        return loss[0]

    @staticmethod
    def backward(ctx, g):
        (dcl,) = ctx.saved_tensors
        return None, (dcl * g).reshape(ctx.shape)


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


def _overlapping(t: torch.Tensor) -> bool:
    """True unless t's strides provably give every element its own address (each stride, in increasing order, exceeds
    the span of the smaller ones).  Stride-0 broadcasts and other aliasing views are overlapping."""
    span = 0
    for st, sz in sorted((st, sz) for st, sz in zip(t.stride(), t.shape) if sz > 1):
        if st <= span:
            return True
        span += (sz - 1) * st
    return False


def cosine_forward(a, b, cosv, norma, normb) -> None:
    """cosv [B, H, W] = <normalize(a), normalize(b)> over the channels of fp32 [B, C, H, W] views a, b (any strides),
    and the unclamped norms the backward reads (csrc/cosine_loss.cu)."""
    B, C, H, W = a.shape
    _lib.check(_lib.load().stego_cosine_fwd(_lib.ptr(a), *a.stride(), _lib.ptr(b), *b.stride(), B, C, H, W, 1e-10,
                                            _lib.ptr(cosv), _lib.ptr(norma), _lib.ptr(normb), _lib.stream()),
               "stego_cosine_fwd")


def cosine_backward(a, b, cosv, norma, normb, grad_cos, da, db) -> None:
    """da / db (either may be None) = grad_cos [B, H, W] x d(cosv)/d(a) / d(b), written (not accumulated) with the
    strides of a / b."""
    B, C, H, W = a.shape
    _lib.check(_lib.load().stego_cosine_bwd(_lib.ptr(a), *a.stride(), _lib.ptr(b), *b.stride(), B, C, H, W, 1e-10,
                                            _lib.ptr(cosv), _lib.ptr(norma), _lib.ptr(normb), _lib.ptr(grad_cos),
                                            _lib.ptr(da), _lib.ptr(db), _lib.stream()), "stego_cosine_bwd")


def aug_sample_forward(coord_aug, code, grid, sampled) -> None:
    """The sampling half of the aug-alignment term (train_segmentation.py:189-199): grid [B, h, h, 2] = coord_aug
    [B, S, S, 2] (contiguous) resized to h x h as F.interpolate(bilinear, align_corners=False) does, and sampled
    [B, C, h, h] (contiguous) = sample(code, grid) (modules.py:287-288) of the fp32 code [B, C, h, h] (any strides)."""
    B, C, h, w = code.shape
    if h != w or coord_aug.shape[1] != coord_aug.shape[2] or not coord_aug.is_contiguous():
        raise ValueError(f"stego_b200.aug_sample_forward: square code and contiguous square coord_aug needed, got "
                         f"{tuple(code.shape)} and {tuple(coord_aug.shape)}")
    _lib.check(_lib.load().stego_aug_align_fwd(_lib.ptr(coord_aug), coord_aug.shape[1], _lib.ptr(code), *code.stride(),
                                               B, C, h, _lib.ptr(grid), _lib.ptr(sampled), _lib.stream()),
               "stego_aug_align_fwd")


def aug_sample_backward(grid, dsampled, dcode) -> None:
    """dcode [B, C, h, h] (the forward's code strides) += the grid_sample backward of dsampled at grid, by atomics."""
    B, C, h, _ = dcode.shape
    _lib.check(_lib.load().stego_aug_align_bwd(_lib.ptr(grid), _lib.ptr(dsampled), B, C, h, _lib.ptr(dcode),
                                               *dcode.stride(), _lib.stream()), "stego_aug_align_bwd")


def aug_loss(cosv, weight: float, loss, total=None) -> None:
    """loss[0] = -cosv.mean() in a fixed summation order; total[0] += weight * loss[0] when total is given."""
    _lib.check(_lib.load().stego_aug_align_loss(_lib.ptr(cosv), cosv.numel(), float(weight), _lib.ptr(loss),
                                                _lib.ptr(total), _lib.stream()), "stego_aug_align_loss")


def rec_scratch(M: int, E: int, D: int, device) -> torch.Tensor:
    """The per-CTA decoder-gradient partials rec_backward needs for M pixel rows on `device` (sized from its grid)."""
    with torch.cuda.device(device):
        nbytes = int(_lib.load().stego_rec_scratch_bytes(M, E, D))
    return torch.empty(-(-nbytes // 4), dtype=torch.float32, device=device)


def rec_forward(code, feat, m3, hw: int, weight, bias, cosv, nr, nf) -> None:
    """The reconstruction term (train_segmentation.py:183-187) over M pixel rows: cosv [M] = <normalize(decoder(code)),
    normalize(feat * m3)>, and the unclamped norms nr = |decoder(code)|, nf = |feat * m3| the backward reads
    (csrc/rec_loss.cu; the decoder output is never written).  code: fp32 [M, >= D] rows; feat: bf16 [M, E] rows;
    m3: fp32 [M / hw, E...] per-image channel scale or None; weight / bias: the decoder's [E, D, 1, 1] / [E]."""
    M, E, D = feat.shape[0], weight.shape[0], weight.shape[1]
    _lib.check(_lib.load().stego_rec_fwd(_lib.ptr(code), code.stride(0), _lib.ptr(feat), feat.stride(0), _lib.ptr(m3), hw,
                                         _lib.ptr(weight), _lib.ptr(bias), M, E, D, _lib.ptr(cosv), _lib.ptr(nr),
                                         _lib.ptr(nf), _lib.stream()), "stego_rec_fwd")


def rec_backward(code, feat, m3, hw: int, weight, bias, cosv, nr, nf, dcos, dcode, scratch, dweight, dbias) -> None:
    """dcode [M, >= D] rows += the term's code gradient for d loss / d cos = dcos[0]; dweight / dbias (the decoder's
    shapes) are written, summed over the rows in a fixed order."""
    M, E, D = feat.shape[0], weight.shape[0], weight.shape[1]
    _lib.check(_lib.load().stego_rec_bwd(_lib.ptr(code), code.stride(0), _lib.ptr(feat), feat.stride(0), _lib.ptr(m3), hw,
                                         _lib.ptr(weight), _lib.ptr(bias), M, E, D, _lib.ptr(cosv), _lib.ptr(nr),
                                         _lib.ptr(nf), _lib.ptr(dcos), _lib.ptr(dcode), dcode.stride(0),
                                         _lib.ptr(scratch), scratch.numel() * 4, _lib.ptr(dweight), _lib.ptr(dbias),
                                         _lib.stream()), "stego_rec_bwd")


CRF_SIDE = 56  # the CRF term works on resize(., 56) (train_segmentation.py:201-208)


def crf_params(fn) -> tuple:
    """(alpha, beta, gamma, w1, w2, shift) of a ContrastiveCRFLoss, as the kernels take them."""
    return tuple(float(v) for v in (fn.alpha, fn.beta, fn.gamma, fn.w1, fn.w2, fn.shift))


def crf_guidance(img, coords, gsel, pos) -> None:
    """The CRF term's guidance: gsel [B, NP, 4] = resize(img, 56) (fp32 [B, <= 3, H, W], any strides) at the samples
    coords [2, n], pos [NP, 2] their positions (csrc/crf_loss.cu)."""
    B, Cg, H, W = img.shape
    _lib.check(_lib.load().stego_crf_guidance(_lib.ptr(img), *img.stride(), Cg, H, W, _lib.ptr(coords), B,
                                              coords.shape[1], CRF_SIDE, _lib.ptr(gsel), _lib.ptr(pos), _lib.stream()),
               "stego_crf_guidance")


def crf_forward(code, coords, params, gsel, pos, raw, sel, nrm, tile_sum) -> None:
    """The CRF term's forward on the code (fp32 [B, C, h, w], any strides): raw [B, C, NP] = resize(code, 56) at the
    samples, sel = normalize(raw) over the channels, nrm [B, NP] the norms, tile_sum [B, NP/64, NP/64] the fp64 sums of
    -(Gram x pairwise kernel)."""
    B, C, h, w = code.shape
    _lib.check(_lib.load().stego_crf_mean_fwd(_lib.ptr(code), *code.stride(), C, h, w, _lib.ptr(coords), B,
                                              coords.shape[1], CRF_SIDE, *params, _lib.ptr(gsel), _lib.ptr(pos),
                                              _lib.ptr(raw), _lib.ptr(sel), _lib.ptr(nrm), _lib.ptr(tile_sum),
                                              _lib.stream()),
               "stego_crf_mean_fwd")


def crf_loss(tile_sum, n: int, weight: float, loss, total=None) -> None:
    """loss[0] = the mean of the B n^2 outputs from tile_sum, in a fixed order; total[0] += weight * loss[0] if given."""
    _lib.check(_lib.load().stego_crf_mean_loss(_lib.ptr(tile_sum), tile_sum.shape[0], n, float(weight), _lib.ptr(loss),
                                               _lib.ptr(total), _lib.stream()), "stego_crf_mean_loss")


def crf_backward(gscalar, sel, nrm, gsel, pos, coords, params, dsel, dcode) -> None:
    """dcode [B, C, h, w] (any strides) += the gradient of the mean for the upstream gradient gscalar[0] of every output,
    by atomics; dsel [B, C, NP] is scratch."""
    B, C, h, w = dcode.shape
    _lib.check(_lib.load().stego_crf_mean_bwd(_lib.ptr(gscalar), _lib.ptr(sel), _lib.ptr(nrm), _lib.ptr(gsel),
                                              _lib.ptr(pos), _lib.ptr(coords), B, C, coords.shape[1], h, w, CRF_SIDE,
                                              *params, _lib.ptr(dsel), _lib.ptr(dcode), *dcode.stride(), _lib.stream()),
               "stego_crf_mean_bwd")


class _PixelCosineFn(torch.autograd.Function):
    """cos[b, y, x] = <normalize(a)[b, :, y, x], normalize(b)[b, :, y, x]> (F.normalize eps 1e-10, modules.py:275-276): one
    read of each operand in the forward, one in the backward (csrc/cosine_loss.cu)."""

    @staticmethod
    def forward(ctx, a, b):
        _lib.require_cuda(a, b)
        # the backward writes each gradient with its operand's strides, so an operand whose elements share memory (a
        # broadcast prototype, stride 0) is made dense here: otherwise every pixel's gradient would land on the same floats
        a32, b32 = (t.contiguous() if _overlapping(t) else t for t in (a.detach().float(), b.detach().float()))
        B, C, H, W = a32.shape
        assert b32.shape == a32.shape
        cosv = torch.empty(B, H, W, dtype=torch.float32, device=a.device)
        norma, normb = torch.empty_like(cosv), torch.empty_like(cosv)
        cosine_forward(a32, b32, cosv, norma, normb)
        ctx.save_for_backward(a32, b32, cosv, norma, normb)
        return cosv

    @staticmethod
    def backward(ctx, g):
        a32, b32, cosv, norma, normb = ctx.saved_tensors
        need_a, need_b = ctx.needs_input_grad
        da = torch.empty_strided(a32.shape, a32.stride(), dtype=torch.float32, device=a32.device) if need_a else None
        db = torch.empty_strided(b32.shape, b32.stride(), dtype=torch.float32, device=b32.device) if need_b else None
        if not (need_a or need_b):
            return None, None
        cosine_backward(a32, b32, cosv, norma, normb, g.float().contiguous(), da, db)
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
