"""CPU oracle for the ViT's attention maps and last-n-block outputs.  TEST INFRASTRUCTURE ONLY.

A plain-PyTorch restatement of the reference's `VisionTransformer.get_intermediate_feat` (src/dino/vision_transformer.py:
225-237), `get_last_selfattention` (:239-246) and `get_intermediate_layers` (:248-256), on a reference-named state dict
like stego_oracle.vit_forward.  It is pinned to the reference by oracle/make_golden_vit_maps.py, which stores the
reference's own outputs in tests/golden/vit_small8_32px_maps.pt.  Nothing under stego_b200/ imports it.
"""
from __future__ import annotations

from typing import Dict, List, Tuple

import torch
import torch.nn.functional as F

import stego_oracle as O

Tensor = torch.Tensor


def vit_intermediate(sd: Dict[str, Tensor], img: Tensor, arch: str, patch: int = 8, n: int = 1
                     ) -> Tuple[List[Tensor], List[Tensor], List[Tensor]]:
    """get_intermediate_feat(img, n): for each of the last n blocks (every block for n >= depth, none for n <= 0),
    oldest first, feat = norm(block output) [B, N, E], attn = softmax(q k^T * 64^-0.5) [B, heads, N, N] and qkv
    [3, B, heads, N, 64].  The last block's attn is get_last_selfattention(img); the feats are
    get_intermediate_layers(img, n)."""
    cfg = O.vit_config(arch)
    E, heads, depth = cfg["embed_dim"], cfg["heads"], cfg["depth"]
    B = img.shape[0]
    x = F.conv2d(img, sd["patch_embed.proj.weight"], sd["patch_embed.proj.bias"], stride=patch)
    x = torch.cat((sd["cls_token"].expand(B, -1, -1), x.flatten(2).transpose(1, 2)), dim=1)
    x = x + O.interpolate_pos_embed(sd["pos_embed"], img.shape[2], img.shape[3], patch)
    scale = (E // heads) ** -0.5
    feats, attns, qkvs = [], [], []
    for i in range(depth):
        p = f"blocks.{i}."
        y = F.layer_norm(x, (E,), sd[p + "norm1.weight"], sd[p + "norm1.bias"], eps=1e-6)
        N = y.shape[1]
        qkv = F.linear(y, sd[p + "attn.qkv.weight"], sd[p + "attn.qkv.bias"])
        qkv = qkv.reshape(B, N, 3, heads, E // heads).permute(2, 0, 3, 1, 4)
        q, k, v = qkv[0], qkv[1], qkv[2]
        attn = ((q @ k.transpose(-2, -1)) * scale).softmax(dim=-1)
        y = (attn @ v).transpose(1, 2).reshape(B, N, E)
        x = x + F.linear(y, sd[p + "attn.proj.weight"], sd[p + "attn.proj.bias"])
        y = F.layer_norm(x, (E,), sd[p + "norm2.weight"], sd[p + "norm2.bias"], eps=1e-6)
        x = x + F.linear(F.gelu(F.linear(y, sd[p + "mlp.fc1.weight"], sd[p + "mlp.fc1.bias"])),
                         sd[p + "mlp.fc2.weight"], sd[p + "mlp.fc2.bias"])
        if depth - i <= n:
            feats.append(F.layer_norm(x, (E,), sd["norm.weight"], sd["norm.bias"], eps=1e-6))
            attns.append(attn)
            qkvs.append(qkv)
    return feats, attns, qkvs
