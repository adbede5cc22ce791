"""CPU oracle for the STEGO correspondence-distillation hot path.  TEST INFRASTRUCTURE ONLY.

This file is a plain-PyTorch fp32 restatement of the reference algorithm (mhamilton723/STEGO @
eb4d6b5).  It exists so that tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
`--impl reference` legs can check and time the CUDA path against it.  Nothing under stego_b200/
imports it, and it must never be used as (or behind) the product path.

Parity status: PINNED.  The reference has no tests or golden vectors of its own (SURVEY.md §4.1),
but it is importable without a GPU, so this restatement is checked function-by-function
against the real reference code by oracle/check_against_reference.py, and the golden fixtures under
tests/golden/ were produced by the reference itself (oracle/make_golden.py).

Every function cites the reference file:line it follows.  All random draws are explicit inputs
(coords, perms, dropout masks) so that the CUDA path and the oracle can be fed identical values.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F

Tensor = torch.Tensor


# --------------------------------------------------------------------------------------------------
# configuration (reference: src/configs/train_config.yml)
# --------------------------------------------------------------------------------------------------
@dataclass
class LossCfg:
    pointwise: bool = True
    zero_clamp: bool = True
    stabalize: bool = False  # (sic) spelling follows the reference config key
    feature_samples: int = 11
    neg_samples: int = 5
    pos_intra_shift: float = 0.18
    pos_inter_shift: float = 0.12
    neg_inter_shift: float = 0.46
    pos_intra_weight: float = 0.67
    pos_inter_weight: float = 0.25
    neg_inter_weight: float = 0.63
    use_salience: bool = False


# --------------------------------------------------------------------------------------------------
# src/modules.py:275-295 — norm, tensor_correlation, sample, super_perm
# --------------------------------------------------------------------------------------------------
def l2_normalize(t: Tensor, eps: float = 1e-10) -> Tensor:
    """modules.py:275-276 `norm`: x / max(||x||_2 over dim 1, eps)."""
    n = t.pow(2).sum(dim=1, keepdim=True).sqrt().clamp_min(eps)
    return t / n


def correlation(a: Tensor, b: Tensor) -> Tensor:
    """modules.py:283-284 `tensor_correlation` einsum nchw,ncij->nhwij as one GEMM per image."""
    n, c, h, w = a.shape
    _, _, i, j = b.shape
    out = torch.bmm(a.reshape(n, c, h * w).transpose(1, 2), b.reshape(n, c, i * j))
    return out.reshape(n, h, w, i, j)


def bilinear_sample(t: Tensor, coords: Tensor) -> Tensor:
    """modules.py:287-288 `sample`: grid_sample(t, coords.permute(0,2,1,3), border, align_corners=True).

    Written out as an explicit 4-tap gather (this is exactly what the CUDA sampling kernel does):
    out[b,:,i,j] = bilinear(t[b], x = coords[b,j,i,0], y = coords[b,j,i,1]).
    """
    B, C, H, W = t.shape
    grid = coords.permute(0, 2, 1, 3)  # [B, i, j, 2]
    x = ((grid[..., 0] + 1.0) / 2.0) * (W - 1)
    y = ((grid[..., 1] + 1.0) / 2.0) * (H - 1)
    x = x.clamp(0, W - 1)  # padding_mode='border' clips the source coordinate
    y = y.clamp(0, H - 1)
    x0 = x.floor()
    y0 = y.floor()
    x1 = x0 + 1
    y1 = y0 + 1
    w_nw = (x1 - x) * (y1 - y)
    w_ne = (x - x0) * (y1 - y)
    w_sw = (x1 - x) * (y - y0)
    w_se = (x - x0) * (y - y0)

    def tap(xi: Tensor, yi: Tensor) -> Tensor:
        inb = ((xi >= 0) & (xi <= W - 1) & (yi >= 0) & (yi <= H - 1)).to(t.dtype)
        xi_c = xi.clamp(0, W - 1).long()
        yi_c = yi.clamp(0, H - 1).long()
        flat = (yi_c * W + xi_c).reshape(B, 1, -1).expand(B, C, -1)
        v = t.reshape(B, C, H * W).gather(2, flat).reshape(B, C, *xi.shape[1:])
        return v * inb.unsqueeze(1)

    return (tap(x0, y0) * w_nw.unsqueeze(1) + tap(x1, y0) * w_ne.unsqueeze(1)
            + tap(x0, y1) * w_sw.unsqueeze(1) + tap(x1, y1) * w_se.unsqueeze(1))


def super_perm_from_randperm(perm: Tensor) -> Tensor:
    """modules.py:291-295 `super_perm` given the randperm draw: fixed points are bumped by +1,
    then everything is taken mod size (NOT a derangement: duplicates can occur)."""
    size = perm.shape[0]
    p = perm.clone()
    p[p == torch.arange(size, device=p.device)] += 1
    return p % size


def draw_loss_randomness(batch: int, cfg: LossCfg, device="cpu") -> Tuple[Tensor, Tensor, List[Tensor]]:
    """RNG order of ContrastiveCorrelationLoss.forward (modules.py:366-367, 383):
    rand(coords1), rand(coords2), then one randperm per negative sample."""
    shape = [batch, cfg.feature_samples, cfg.feature_samples, 2]
    coords1 = torch.rand(shape, device=device) * 2 - 1
    coords2 = torch.rand(shape, device=device) * 2 - 1
    perms = [super_perm_from_randperm(torch.randperm(batch, device=device, dtype=torch.long))
             for _ in range(cfg.neg_samples)]
    return coords1, coords2, perms


# --------------------------------------------------------------------------------------------------
# src/modules.py:325-398 — ContrastiveCorrelationLoss
# --------------------------------------------------------------------------------------------------
def corr_helper(f1: Tensor, f2: Tensor, c1: Tensor, c2: Tensor, shift: float, cfg: LossCfg) -> Tuple[Tensor, Tensor]:
    """modules.py:325-347 `helper`."""
    with torch.no_grad():
        fd = correlation(l2_normalize(f1), l2_normalize(f2))
        if cfg.pointwise:
            old_mean = fd.mean()
            fd = fd - fd.mean(dim=[3, 4], keepdim=True)
            fd = fd - fd.mean() + old_mean
    cd = correlation(l2_normalize(c1), l2_normalize(c2))
    lo = 0.0 if cfg.zero_clamp else -9999.0
    clamped = cd.clamp(lo, 0.8) if cfg.stabalize else cd.clamp(lo)
    return -clamped * (fd - shift), cd


def correlation_loss(feats: Tensor, feats_pos: Tensor, code: Tensor, code_pos: Tensor, coords1: Tensor,
                     coords2: Tensor, perms: Sequence[Tensor], cfg: LossCfg):
    """modules.py:349-398 `ContrastiveCorrelationLoss.forward` with the random draws injected.
    Returns the reference's 6-tuple."""
    f = bilinear_sample(feats, coords1)
    c = bilinear_sample(code, coords1)
    fp = bilinear_sample(feats_pos, coords2)
    cp = bilinear_sample(code_pos, coords2)
    intra_loss, intra_cd = corr_helper(f, f, c, c, cfg.pos_intra_shift, cfg)
    inter_loss, inter_cd = corr_helper(f, fp, c, cp, cfg.pos_inter_shift, cfg)
    neg_l, neg_c = [], []
    for perm in perms:
        fn = bilinear_sample(feats[perm], coords2)
        cn = bilinear_sample(code[perm], coords2)
        l, d = corr_helper(f, fn, c, cn, cfg.neg_inter_shift, cfg)
        neg_l.append(l)
        neg_c.append(d)
    return (intra_loss.mean(), intra_cd, inter_loss.mean(), inter_cd, torch.cat(neg_l, 0), torch.cat(neg_c, 0))


def weighted_correspondence_loss(out6, cfg: LossCfg) -> Tensor:
    """train_segmentation.py:169-181: means + weights (correspondence_weight = 1)."""
    intra, _, inter, _, neg, _ = out6
    return cfg.pos_inter_weight * inter.mean() + cfg.pos_intra_weight * intra.mean() + cfg.neg_inter_weight * neg.mean()


# --------------------------------------------------------------------------------------------------
# src/modules.py:134-161 — ClusterLookup
# --------------------------------------------------------------------------------------------------
def cluster_lookup(x: Tensor, clusters: Tensor, alpha: Optional[float], log_probs: bool = False):
    """modules.py:146-161. F.normalize default eps = 1e-12."""
    nc = clusters / clusters.pow(2).sum(1, keepdim=True).sqrt().clamp_min(1e-12)
    nx = x / x.pow(2).sum(1, keepdim=True).sqrt().clamp_min(1e-12)
    B, C, H, W = x.shape
    ip = torch.matmul(nc, nx.reshape(B, C, H * W)).reshape(B, -1, H, W)  # einsum bchw,nc->bnhw
    if alpha is None:
        probs = F.one_hot(ip.argmax(dim=1), clusters.shape[0]).permute(0, 3, 1, 2).to(torch.float32)
    else:
        probs = torch.softmax(ip * alpha, dim=1)
    loss = -(probs * ip).sum(1).mean()
    if log_probs:
        return torch.log_softmax(ip * alpha, dim=1)
    return loss, probs


# --------------------------------------------------------------------------------------------------
# src/dino/vision_transformer.py — frozen DINO ViT forward (functional, reference state-dict names)
# --------------------------------------------------------------------------------------------------
def contrastive_crf_loss(guidance: Tensor, clusters: Tensor, coords: Tensor, alpha: float, beta: float, gamma: float,
                         w1: float, w2: float, shift: float) -> Tensor:
    """ContrastiveCRFLoss.forward (src/modules.py:449-469) with the coordinate draw (`:456-458`, two torch.randint calls: row
    indices then column indices, shared by the batch) made an argument.  guidance [B, Cg, H, W], clusters [B, C, H, W],
    coords int64 [2, n] -> [B, n, n]."""
    ys, xs = coords[0], coords[1]
    g = guidance[:, :, ys, xs]  # [B, Cg, n]
    c = clusters[:, :, ys, xs]  # [B, C, n]
    dpos = ((ys[:, None] - ys[None, :]) ** 2 + (xs[:, None] - xs[None, :]) ** 2)[None]  # int64, like the reference
    dgui = (g[:, :, :, None] - g[:, :, None, :]).square().sum(1)
    kernel = w1 * torch.exp(-dpos / (2 * alpha) - dgui / (2 * beta)) + w2 * torch.exp(-dpos / (2 * gamma)) - shift
    gram = torch.einsum("bka,bkc->bac", c, c)
    return -(gram * kernel)


def vit_config(arch: str) -> Dict[str, int]:
    """vision_transformer.py:266-277 (vit_small / vit_base); depth 12, mlp_ratio 4, LN eps 1e-6."""
    if arch == "vit_small":
        return dict(embed_dim=384, heads=6, depth=12)
    if arch == "vit_base":
        return dict(embed_dim=768, heads=12, depth=12)
    raise ValueError(f"unknown arch {arch}")


def vit_random_state(arch: str, patch: int = 8, seed: int = 0, img_size: int = 224) -> Dict[str, Tensor]:
    """Random ViT weights with the reference's parameter names and init (vision_transformer.py:160-174):
    trunc_normal(std=.02) for Linear weights / pos_embed / cls_token, zeros for biases, LN = (1, 0).
    The patch-embed conv keeps PyTorch's default Conv2d init, like the reference."""
    cfg = vit_config(arch)
    E, depth = cfg["embed_dim"], cfg["depth"]
    g = torch.Generator().manual_seed(seed)

    def tn(*shape):
        t = torch.empty(*shape)
        torch.nn.init.trunc_normal_(t, std=0.02, generator=g)
        return t

    sd: Dict[str, Tensor] = {}
    npatch = (img_size // patch) ** 2
    sd["cls_token"] = tn(1, 1, E)
    sd["pos_embed"] = tn(1, npatch + 1, E)
    fan_in = 3 * patch * patch
    bound = 1.0 / math.sqrt(fan_in)
    sd["patch_embed.proj.weight"] = (torch.rand(E, 3, patch, patch, generator=g) * 2 - 1) * bound
    sd["patch_embed.proj.bias"] = (torch.rand(E, generator=g) * 2 - 1) * bound
    for i in range(depth):
        p = f"blocks.{i}."
        sd[p + "norm1.weight"] = torch.ones(E)
        sd[p + "norm1.bias"] = torch.zeros(E)
        sd[p + "attn.qkv.weight"] = tn(3 * E, E)
        sd[p + "attn.qkv.bias"] = torch.zeros(3 * E)
        sd[p + "attn.proj.weight"] = tn(E, E)
        sd[p + "attn.proj.bias"] = torch.zeros(E)
        sd[p + "norm2.weight"] = torch.ones(E)
        sd[p + "norm2.bias"] = torch.zeros(E)
        sd[p + "mlp.fc1.weight"] = tn(4 * E, E)
        sd[p + "mlp.fc1.bias"] = torch.zeros(4 * E)
        sd[p + "mlp.fc2.weight"] = tn(E, 4 * E)
        sd[p + "mlp.fc2.bias"] = torch.zeros(E)
    sd["norm.weight"] = torch.ones(E)
    sd["norm.bias"] = torch.zeros(E)
    return sd


def perturb_vit_state(sd: Dict[str, Tensor], seed: int = 1, scale: float = 0.05) -> Dict[str, Tensor]:
    """Make biases / LN affine non-trivial so parity tests exercise every term (the reference init
    leaves them at 0 / 1, which would hide indexing bugs)."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for k, v in sd.items():
        if k.endswith("bias") or "norm" in k:
            out[k] = v + scale * torch.randn(v.shape, generator=g)
        else:
            out[k] = v.clone()
    return out


def interpolate_pos_embed(pos_embed: Tensor, w_px: int, h_px: int, patch: int) -> Tensor:
    """vision_transformer.py:176-196 `interpolate_pos_encoding` (bicubic, with the +0.1 fudge).
    NB the reference calls it with (x, w, h) = (tokens, img.shape[2], img.shape[3])."""
    N = pos_embed.shape[1] - 1
    dim = pos_embed.shape[-1]
    w0 = w_px // patch
    h0 = h_px // patch
    if w0 * h0 == N and w_px == h_px:
        return pos_embed
    cls_pos = pos_embed[:, 0]
    patch_pos = pos_embed[:, 1:]
    s = int(math.sqrt(N))
    w0f, h0f = w0 + 0.1, h0 + 0.1
    patch_pos = F.interpolate(patch_pos.reshape(1, s, s, dim).permute(0, 3, 1, 2),
                              scale_factor=(w0f / math.sqrt(N), h0f / math.sqrt(N)), mode="bicubic")
    assert int(w0f) == patch_pos.shape[-2] and int(h0f) == patch_pos.shape[-1]
    patch_pos = patch_pos.permute(0, 2, 3, 1).reshape(1, -1, dim)
    return torch.cat((cls_pos.unsqueeze(0), patch_pos), dim=1)


def vit_forward(sd: Dict[str, Tensor], img: Tensor, arch: str, patch: int = 8) -> Tensor:
    """vision_transformer.py:198-209 prepare_tokens + :225-237 get_intermediate_feat(n=1):
    returns norm(x) of the last block, [B, N, E] (cls token first)."""
    cfg = vit_config(arch)
    E, heads, depth = cfg["embed_dim"], cfg["heads"], cfg["depth"]
    B = img.shape[0]
    x = F.conv2d(img, sd["patch_embed.proj.weight"], sd["patch_embed.proj.bias"], stride=patch)
    x = x.flatten(2).transpose(1, 2)  # [B, hw, E]
    x = torch.cat((sd["cls_token"].expand(B, -1, -1), x), dim=1)
    x = x + interpolate_pos_embed(sd["pos_embed"], img.shape[2], img.shape[3], patch)
    scale = (E // heads) ** -0.5
    for i in range(depth):
        p = f"blocks.{i}."
        y = F.layer_norm(x, (E,), sd[p + "norm1.weight"], sd[p + "norm1.bias"], eps=1e-6)
        qkv = F.linear(y, sd[p + "attn.qkv.weight"], sd[p + "attn.qkv.bias"])
        N = qkv.shape[1]
        qkv = qkv.reshape(B, N, 3, heads, E // heads).permute(2, 0, 3, 1, 4)
        q, k, v = qkv[0], qkv[1], qkv[2]
        attn = ((q @ k.transpose(-2, -1)) * scale).softmax(dim=-1)
        y = (attn @ v).transpose(1, 2).reshape(B, N, E)
        x = x + F.linear(y, sd[p + "attn.proj.weight"], sd[p + "attn.proj.bias"])
        y = F.layer_norm(x, (E,), sd[p + "norm2.weight"], sd[p + "norm2.bias"], eps=1e-6)
        y = F.gelu(F.linear(y, sd[p + "mlp.fc1.weight"], sd[p + "mlp.fc1.bias"]))
        x = x + F.linear(y, sd[p + "mlp.fc2.weight"], sd[p + "mlp.fc2.bias"])
    return F.layer_norm(x, (E,), sd["norm.weight"], sd["norm.bias"], eps=1e-6)


def vit_image_feat(sd: Dict[str, Tensor], img: Tensor, arch: str, patch: int = 8) -> Tensor:
    """modules.py:90-97: drop the cls token, view as NCHW [B, E, h, w]."""
    feat = vit_forward(sd, img, arch, patch)
    B = img.shape[0]
    fh, fw = img.shape[2] // patch, img.shape[3] // patch
    return feat[:, 1:, :].reshape(B, fh, fw, -1).permute(0, 3, 1, 2)


# --------------------------------------------------------------------------------------------------
# src/modules.py:73-81, 108-118 — segmentation head (cluster1 + cluster2) with Dropout2d masks injected
# --------------------------------------------------------------------------------------------------
def head_random_state(n_feats: int, dim: int, seed: int = 0) -> Dict[str, Tensor]:
    """Conv2d(·,·,1) default init, reference parameter names (net.cluster1.0 / net.cluster2.{0,2})."""
    g = torch.Generator().manual_seed(seed)

    def conv(o, i):
        b = 1.0 / math.sqrt(i)
        return (torch.rand(o, i, 1, 1, generator=g) * 2 - 1) * b, (torch.rand(o, generator=g) * 2 - 1) * b

    sd = {}
    sd["cluster1.0.weight"], sd["cluster1.0.bias"] = conv(dim, n_feats)
    sd["cluster2.0.weight"], sd["cluster2.0.bias"] = conv(n_feats, n_feats)
    sd["cluster2.2.weight"], sd["cluster2.2.bias"] = conv(dim, n_feats)
    return sd


def draw_dropout2d_mask(batch: int, channels: int, p: float = 0.1, device="cpu") -> Tensor:
    """The noise tensor F.dropout2d draws for a [B,C,H,W] input: bernoulli(1-p)/(1-p), shape [B,C,1,1]."""
    return torch.empty(batch, channels, 1, 1, device=device).bernoulli_(1 - p).div_(1 - p)


def _bf16_round(t: Tensor) -> Tensor:
    """Straight-through bf16 rounding (identity gradient): emulates where a bf16 autocast run of the
    reference would round GEMM operands, so the CUDA path can be compared at the 1e-3 bar."""
    return t + (t.detach().to(torch.bfloat16).to(t.dtype) - t.detach())


def head_forward(image_feat: Tensor, hp: Dict[str, Tensor], masks: Optional[Sequence[Tensor]],
                 round_bf16: bool = False):
    """modules.py:108-118 with proj_type='nonlinear': code = cluster1(drop(f)) + cluster2(drop(f));
    returns (drop(f) if dropout else f, code).  `masks` = the three Dropout2d noise tensors in call
    order (cluster1 input, cluster2 input, returned feats), or None for eval / dropout off.
    round_bf16=True rounds every GEMM operand (masked inputs, weights, hidden activation) to bf16 with
    fp32 accumulation — the reference under bf16 autocast."""
    m1, m2, m3 = masks if masks is not None else (1.0, 1.0, 1.0)
    r = _bf16_round if round_bf16 else (lambda t: t)
    code = F.conv2d(r(image_feat * m1), r(hp["cluster1.0.weight"]), hp["cluster1.0.bias"])
    h = torch.relu(F.conv2d(r(image_feat * m2), r(hp["cluster2.0.weight"]), hp["cluster2.0.bias"]))
    code = code + F.conv2d(r(h), r(hp["cluster2.2.weight"]), hp["cluster2.2.bias"])
    return image_feat * m3, code


# --------------------------------------------------------------------------------------------------
# src/train_segmentation.py:112-245, 373-383 — the training step
# --------------------------------------------------------------------------------------------------
def linear_probe_loss(code: Tensor, weight: Tensor, bias: Tensor, label: Tensor, n_classes: int) -> Tensor:
    """train_segmentation.py:210-219: 1x1 conv on detached code -> bilinear upsample (align_corners
    False) -> masked cross entropy."""
    logits = F.conv2d(code, weight, bias)
    logits = F.interpolate(logits, label.shape[-2:], mode="bilinear", align_corners=False)
    logits = logits.permute(0, 2, 3, 1).reshape(-1, n_classes)
    flat = label.reshape(-1)
    mask = (flat >= 0) & (flat < n_classes)
    return F.cross_entropy(logits[mask], flat[mask])


def adam_step(p: Tensor, g: Tensor, m: Tensor, v: Tensor, step: int, lr: float, b1=0.9, b2=0.999, eps=1e-8):
    """torch.optim.Adam (no weight decay, no amsgrad), one tensor, in place; `step` is 1-based."""
    m.mul_(b1).add_(g, alpha=1 - b1)
    v.mul_(b2).addcmul_(g, g, value=1 - b2)
    bc1 = 1 - b1 ** step
    bc2 = 1 - b2 ** step
    denom = (v.sqrt() / math.sqrt(bc2)).add_(eps)
    p.addcdiv_(m, denom, value=-lr / bc1)


def training_losses(image_feat: Tensor, image_feat_pos: Tensor, hp: Dict[str, Tensor], probes: Dict[str, Tensor],
                    label: Tensor, masks, masks_pos, coords1, coords2, perms, cfg: LossCfg, n_classes: int,
                    round_bf16: bool = False):
    """Loss assembly of training_step (train_segmentation.py:130-225) from frozen-backbone features.
    Returns dict of scalar losses; `total` is what manual_backward receives."""
    feats, code = head_forward(image_feat, hp, masks, round_bf16)
    feats_pos, code_pos = head_forward(image_feat_pos, hp, masks_pos, round_bf16)
    out6 = correlation_loss(feats, feats_pos, code, code_pos, coords1, coords2, perms, cfg)
    corr = weighted_correspondence_loss(out6, cfg)
    detached = code.detach().clone()
    lin = linear_probe_loss(detached, probes["linear_probe.weight"], probes["linear_probe.bias"], label, n_classes)
    clu, _ = cluster_lookup(detached, probes["cluster_probe.clusters"], None)
    return dict(total=corr + lin + clu, corr=corr, linear=lin, cluster=clu,
                pos_intra=out6[0], pos_inter=out6[2], neg_inter=out6[4].mean(),
                cd_intra=out6[1].mean(), cd_inter=out6[3].mean(), cd_neg=out6[5].mean(), code=code)


# --------------------------------------------------------------------------------------------------
# kNN descriptors (SURVEY.md §8(f) rank 1) — src/precompute_knns.py
# --------------------------------------------------------------------------------------------------
def knn_descriptors(image_feat: Tensor) -> Tensor:
    """precompute_knns.py:19 (get_feats): global-average-pool the [B,E,h,w] feature map, then L2-normalise."""
    return F.normalize(image_feat.mean([2, 3]), dim=1)


def knn_indices(normed_feats: Tensor, k: int = 30, n_batches: int = 16) -> Tuple[Tensor, Tensor]:
    """precompute_knns.py:83-92: similarities of every descriptor against all of them in n_batches slabs
    (`einsum("nf,mf->nm")`), `torch.topk(sims, k)` indices (each row contains itself).  Also returns the similarities
    (the reference discards them) so that tests can compare rankings up to floating-point ties."""
    n = normed_feats.shape[0]
    step = max(1, n // n_batches)
    idx, val = [], []
    for i in range(0, n, step):
        sims = torch.einsum("nf,mf->nm", normed_feats[i:i + step], normed_feats)
        v, ix = torch.topk(sims, k)
        idx.append(ix)
        val.append(v)
    return torch.cat(idx, 0), torch.cat(val, 0)
