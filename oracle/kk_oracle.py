"""dino_feat_type "KK" (src/modules.py:98-101): the keys of the ViT's last block as the teacher features, restated in plain
torch on top of oracle/stego_oracle.py.

The reference takes `qkv[1, :, :, 1:, :]` of get_intermediate_feat(img, n=1) — the key third of the last block's qkv,
cls token dropped — and lays the heads out head-major: channel = head * 64 + d.  (Its `reshape(B, 6, h, w, -1)` is written
for the 6 heads of ViT-S; this restatement keeps the head-major layout for every width, which is what stego_b200 computes.)
The step itself is stego_oracle.training_losses on these features: the choice of teacher changes nothing after the backbone.
"""
from __future__ import annotations

from typing import Dict

import torch
import torch.nn.functional as F
from torch import Tensor

import stego_oracle as O


def vit_last_keys(sd: Dict[str, Tensor], img: Tensor, arch: str, patch: int = 8) -> Tensor:
    """fp32 keys of the last block, [B, N, E] (cls token first), channels head-major: blocks 0 .. depth-2 as
    stego_oracle.vit_forward runs them, then LN1 and the key rows of the last block's qkv projection."""
    cfg = O.vit_config(arch)
    E, heads, depth = cfg["embed_dim"], cfg["heads"], cfg["depth"]
    B = img.shape[0]
    x = F.conv2d(img, sd["patch_embed.proj.weight"], sd["patch_embed.proj.bias"], stride=patch)
    x = x.flatten(2).transpose(1, 2)
    x = torch.cat((sd["cls_token"].expand(B, -1, -1), x), dim=1)
    x = x + O.interpolate_pos_embed(sd["pos_embed"], img.shape[2], img.shape[3], patch)
    scale = (E // heads) ** -0.5
    for i in range(depth - 1):
        p = f"blocks.{i}."
        y = F.layer_norm(x, (E,), sd[p + "norm1.weight"], sd[p + "norm1.bias"], eps=1e-6)
        qkv = F.linear(y, sd[p + "attn.qkv.weight"], sd[p + "attn.qkv.bias"])
        N = qkv.shape[1]
        qkv = qkv.reshape(B, N, 3, heads, E // heads).permute(2, 0, 3, 1, 4)
        attn = ((qkv[0] @ qkv[1].transpose(-2, -1)) * scale).softmax(dim=-1)
        y = (attn @ qkv[2]).transpose(1, 2).reshape(B, N, E)
        x = x + F.linear(y, sd[p + "attn.proj.weight"], sd[p + "attn.proj.bias"])
        y = F.layer_norm(x, (E,), sd[p + "norm2.weight"], sd[p + "norm2.bias"], eps=1e-6)
        x = x + F.linear(F.gelu(F.linear(y, sd[p + "mlp.fc1.weight"], sd[p + "mlp.fc1.bias"])),
                         sd[p + "mlp.fc2.weight"], sd[p + "mlp.fc2.bias"])
    p = f"blocks.{depth - 1}."
    y = F.layer_norm(x, (E,), sd[p + "norm1.weight"], sd[p + "norm1.bias"], eps=1e-6)
    return F.linear(y, sd[p + "attn.qkv.weight"][E:2 * E], sd[p + "attn.qkv.bias"][E:2 * E])


def vit_image_keys(sd: Dict[str, Tensor], img: Tensor, arch: str, patch: int = 8) -> Tensor:
    """The "KK" image_feat of modules.py:98-101: cls dropped, NCHW [B, E, h, w] (a view of tokens-major storage)."""
    k = vit_last_keys(sd, img, arch, patch)
    B = img.shape[0]
    fh, fw = img.shape[2] // patch, img.shape[3] // patch
    return k[:, 1:, :].reshape(B, fh, fw, -1).permute(0, 3, 1, 2)


def image_feat(sd: Dict[str, Tensor], img: Tensor, arch: str, feat_type: str, patch: int = 8) -> Tensor:
    """The teacher features DinoFeaturizer returns for `feat_type` ("feat" or "KK"), NCHW fp32."""
    if feat_type == "feat":
        return O.vit_image_feat(sd, img, arch, patch)
    if feat_type == "KK":
        return vit_image_keys(sd, img, arch, patch)
    raise ValueError("Unknown feat type:{}".format(feat_type))
