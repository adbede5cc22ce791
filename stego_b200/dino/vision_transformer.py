"""Frozen DINO ViT forward on H100: same constructor / parameter names / entry points as the reference
`src/dino/vision_transformer.py` (so DINO and STEGO checkpoints load unchanged), but the forward pass is
a fixed sequence of hand-written sm_90a kernels called through the C-ABI:

    patchify -> wgmma GEMM (+bias +pos-embed, cls rows) ->
    12 x [ LayerNorm -> qkv GEMM -> fused attention -> proj GEMM (+residual, in place) ->
           LayerNorm -> fc1 GEMM (+GELU) -> fc2 GEMM (+residual, in place) ] -> LayerNorm

Reference: vision_transformer.py:47-63 (Mlp), :66-90 (Attention), :94-114 (Block), :117-132 (PatchEmbed),
:135-256 (VisionTransformer), :266-277 (vit_small / vit_base).  The residual stream is fp32, GEMM
operands and activations between kernels are bf16.  The backbone is inference-only (STEGO freezes it:
src/modules.py:30-32), so there is no backward and dropout / drop-path are identities.
"""
from __future__ import annotations

import math
from functools import partial
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn as nn

from .. import ops


class Mlp(nn.Module):
    """Parameter holder for fc1 / fc2 (vision_transformer.py:47-63)."""

    def __init__(self, in_features, hidden_features=None, out_features=None, act_layer=nn.GELU, drop=0.):
        super().__init__()
        self.fc1 = nn.Linear(in_features, hidden_features or in_features)
        self.act = act_layer()
        self.fc2 = nn.Linear(hidden_features or in_features, out_features or in_features)
        self.drop = nn.Dropout(drop)


class Attention(nn.Module):
    """Parameter holder for qkv / proj (vision_transformer.py:66-90)."""

    def __init__(self, dim, num_heads=8, qkv_bias=False, qk_scale=None, attn_drop=0., proj_drop=0.):
        super().__init__()
        self.num_heads = num_heads
        self.scale = qk_scale or (dim // num_heads) ** -0.5
        self.qkv = nn.Linear(dim, dim * 3, bias=qkv_bias)
        self.attn_drop = nn.Dropout(attn_drop)
        self.proj = nn.Linear(dim, dim)
        self.proj_drop = nn.Dropout(proj_drop)


class Block(nn.Module):
    """Parameter holder for one pre-LN transformer block (vision_transformer.py:94-114)."""

    def __init__(self, dim, num_heads, mlp_ratio=4., qkv_bias=False, qk_scale=None, drop=0., attn_drop=0.,
                 drop_path=0., act_layer=nn.GELU, norm_layer=nn.LayerNorm):
        super().__init__()
        self.norm1 = norm_layer(dim)
        self.attn = Attention(dim, num_heads=num_heads, qkv_bias=qkv_bias, qk_scale=qk_scale, attn_drop=attn_drop,
                              proj_drop=drop)
        self.drop_path = nn.Identity()
        self.norm2 = norm_layer(dim)
        self.mlp = Mlp(in_features=dim, hidden_features=int(dim * mlp_ratio), act_layer=act_layer, drop=drop)


class PatchEmbed(nn.Module):
    """Parameter holder for the patch projection (vision_transformer.py:117-132)."""

    def __init__(self, img_size=224, patch_size=16, in_chans=3, embed_dim=768):
        super().__init__()
        self.img_size = img_size
        self.patch_size = patch_size
        self.num_patches = (img_size // patch_size) * (img_size // patch_size)
        self.proj = nn.Conv2d(in_chans, embed_dim, kernel_size=patch_size, stride=patch_size)


class VisionTransformer(nn.Module):
    """DINO ViT.  `get_intermediate_feat(x, n=1)` is the entry point STEGO uses (src/modules.py:90)."""

    def __init__(self, img_size=[224], patch_size=16, in_chans=3, num_classes=0, embed_dim=768, depth=12,
                 num_heads=12, mlp_ratio=4., qkv_bias=False, qk_scale=None, drop_rate=0., attn_drop_rate=0.,
                 drop_path_rate=0., norm_layer=nn.LayerNorm, **kwargs):
        super().__init__()
        if in_chans != 3:
            raise ValueError("stego_b200 ViT: in_chans must be 3")
        if embed_dim % num_heads != 0 or embed_dim // num_heads != 64:
            raise ValueError("stego_b200 ViT: head_dim must be 64 (vit_small / vit_base)")
        self.num_features = self.embed_dim = embed_dim
        self.num_heads = num_heads
        self.mlp_ratio = mlp_ratio
        self.patch_embed = PatchEmbed(img_size=img_size[0], patch_size=patch_size, in_chans=in_chans,
                                      embed_dim=embed_dim)
        self.cls_token = nn.Parameter(torch.zeros(1, 1, embed_dim))
        self.pos_embed = nn.Parameter(torch.zeros(1, self.patch_embed.num_patches + 1, embed_dim))
        self.pos_drop = nn.Dropout(p=drop_rate)
        self.blocks = nn.ModuleList([
            Block(dim=embed_dim, num_heads=num_heads, mlp_ratio=mlp_ratio, qkv_bias=qkv_bias, qk_scale=qk_scale,
                  drop=drop_rate, attn_drop=attn_drop_rate, norm_layer=norm_layer) for _ in range(depth)])
        self.norm = norm_layer(embed_dim)
        self.head = nn.Linear(embed_dim, num_classes) if num_classes > 0 else nn.Identity()
        nn.init.trunc_normal_(self.pos_embed, std=.02)
        nn.init.trunc_normal_(self.cls_token, std=.02)
        self.apply(self._init_weights)
        self._cache: Dict[str, object] = {}

    @staticmethod
    def _init_weights(m):
        if isinstance(m, nn.Linear):
            nn.init.trunc_normal_(m.weight, std=.02)
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)
        elif isinstance(m, nn.LayerNorm):
            nn.init.constant_(m.bias, 0)
            nn.init.constant_(m.weight, 1.0)

    # ------------------------------------------------------------------------------------------
    # host-side preparation (frozen weights -> bf16 GEMM operands, cached)
    # ------------------------------------------------------------------------------------------
    def _weights_key(self):
        return tuple((p.data_ptr(), p._version) for p in self.parameters())

    def _prepared(self):
        """bf16 copies of the GEMM weights and fp32 biases / LN params (cached while weights are unchanged)."""
        key = self._weights_key()
        if self._cache.get("key") != key:
            dev = self.cls_token.device
            E = self.embed_dim
            w = {}
            w["pe_w"] = self.patch_embed.proj.weight.detach().reshape(E, -1).to(torch.bfloat16).contiguous()
            w["pe_b"] = self.patch_embed.proj.bias.detach().float().contiguous()
            w["cls"] = self.cls_token.detach().float().reshape(E).contiguous()
            blocks = []
            for blk in self.blocks:
                def f32(t, n):
                    return t.detach().float().contiguous() if t is not None else torch.zeros(n, device=dev)
                blocks.append(dict(
                    n1w=f32(blk.norm1.weight, E), n1b=f32(blk.norm1.bias, E), eps1=blk.norm1.eps,
                    qkv_w=blk.attn.qkv.weight.detach().to(torch.bfloat16).contiguous(),
                    qkv_b=f32(blk.attn.qkv.bias, 3 * E),
                    proj_w=blk.attn.proj.weight.detach().to(torch.bfloat16).contiguous(),
                    proj_b=f32(blk.attn.proj.bias, E),
                    n2w=f32(blk.norm2.weight, E), n2b=f32(blk.norm2.bias, E), eps2=blk.norm2.eps,
                    fc1_w=blk.mlp.fc1.weight.detach().to(torch.bfloat16).contiguous(), fc1_b=f32(blk.mlp.fc1.bias, blk.mlp.fc1.out_features),
                    fc2_w=blk.mlp.fc2.weight.detach().to(torch.bfloat16).contiguous(), fc2_b=f32(blk.mlp.fc2.bias, E)))
            w["blocks"] = blocks
            w["nw"] = self.norm.weight.detach().float().contiguous()
            w["nb"] = self.norm.bias.detach().float().contiguous()
            self._cache = {"key": key, "w": w, "pos": {}}
        return self._cache["w"]

    def interpolate_pos_encoding(self, x, w, h):
        """vision_transformer.py:176-196: bicubic resize of the patch position embeddings (with the
        +0.1 fudge) when the token grid differs from the pre-training one.  Host-side torch, cached per
        resolution by `_pos_for` (the weights are frozen)."""
        npatch = x.shape[1] - 1
        N = self.pos_embed.shape[1] - 1
        if npatch == N and w == h:
            return self.pos_embed
        dim = x.shape[-1]
        p = self.patch_embed.patch_size
        w0, h0 = w // p + 0.1, h // p + 0.1
        side = int(math.sqrt(N))
        grid = self.pos_embed[:, 1:].reshape(1, side, side, dim).permute(0, 3, 1, 2)
        grid = nn.functional.interpolate(grid, scale_factor=(w0 / math.sqrt(N), h0 / math.sqrt(N)), mode='bicubic')
        assert int(w0) == grid.shape[-2] and int(h0) == grid.shape[-1]
        grid = grid.permute(0, 2, 3, 1).reshape(1, -1, dim)
        return torch.cat((self.pos_embed[:, :1], grid), dim=1)

    def _pos_for(self, H: int, W: int) -> torch.Tensor:
        self._prepared()
        cache = self._cache["pos"]
        if (H, W) not in cache:
            p = self.patch_embed.patch_size
            ntok = (H // p) * (W // p) + 1
            with torch.no_grad():
                dummy = torch.empty(1, ntok, self.embed_dim, device="meta")
                pos = self.interpolate_pos_encoding(dummy, H, W)
            cache[(H, W)] = pos.detach().float().reshape(ntok, self.embed_dim).contiguous()
        return cache[(H, W)]

    # ------------------------------------------------------------------------------------------
    # the kernel sequence
    # ------------------------------------------------------------------------------------------
    @torch.no_grad()
    def forward_tokens(self, img: torch.Tensor, want_qkv: bool = False
                       ) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
        """Returns (x, qkv_last): x = fp32 residual stream [B*N, E] after the last block (before the
        final norm); qkv_last = packed bf16 [B*N, 3E] of the last block if requested."""
        if not img.is_cuda:
            raise RuntimeError("stego_b200: the DINO ViT forward only exists as sm_90a kernels (no CPU fallback)")
        w = self._prepared()
        # bf16 images are taken as they are (patchify rounds fp32 images to bf16 anyway: same operand bits)
        img = (img if img.dtype == torch.bfloat16 else img.float()).contiguous()
        B, _, H, W = img.shape
        p = self.patch_embed.patch_size
        E, heads = self.embed_dim, self.num_heads
        hw = (H // p) * (W // p)
        N = hw + 1
        dev = img.device
        pos = self._pos_for(H, W)
        rows = ops.patchify(img, p)
        x = torch.empty(B * N, E, dtype=torch.float32, device=dev)
        ops.gemm(rows, w["pe_w"], x, M=B * hw, N=E, K=3 * p * p, bias=w["pe_b"], residual=pos, row_div=hw)
        ops.cls_rows(x, w["cls"], pos, B, N)
        y = torch.empty(B * N, E, dtype=torch.bfloat16, device=dev)
        qkv = torch.empty(B * N, 3 * E, dtype=torch.bfloat16, device=dev)
        ao = torch.empty(B * N, E, dtype=torch.bfloat16, device=dev)
        hid = torch.empty(B * N, w["blocks"][0]["fc1_w"].shape[0], dtype=torch.bfloat16, device=dev)
        Hd = hid.shape[1]
        blocks = w["blocks"]
        for bw in blocks:
            ops.layernorm(x, bw["n1w"], bw["n1b"], y, eps=bw["eps1"])
            ops.gemm(y, bw["qkv_w"], qkv, M=B * N, N=3 * E, K=E, bias=bw["qkv_b"])
            ops.attention(qkv, ao, B, N, E, heads)
            ops.gemm(ao, bw["proj_w"], x, M=B * N, N=E, K=E, bias=bw["proj_b"], residual=x)
            ops.layernorm(x, bw["n2w"], bw["n2b"], y, eps=bw["eps2"])
            ops.gemm(y, bw["fc1_w"], hid, M=B * N, N=Hd, K=E, bias=bw["fc1_b"], act=ops.ACT_GELU)
            ops.gemm(hid, bw["fc2_w"], x, M=B * N, N=E, K=Hd, bias=bw["fc2_b"], residual=x)
        return x, (qkv if want_qkv else None)

    @torch.no_grad()
    def patch_features(self, img: torch.Tensor, use_graph: bool = False) -> torch.Tensor:
        """norm(last block) with the cls token dropped, tokens-major bf16 [B, hw, E] — the tensor STEGO's
        DinoFeaturizer builds at src/modules.py:97, in the K-major layout the correlation GEMM wants.

        use_graph=True replays the whole kernel sequence (~110 launches) as ONE CUDA graph captured per input
        shape (the backbone is frozen and RNG-free).  The result then lives in a static buffer that the next
        replay overwrites: only for callers that consume it before calling again (the fused training step)."""
        if use_graph and (img[0] if isinstance(img, (list, tuple)) else img).is_cuda:
            return self._graphed_patch_features(img)
        if isinstance(img, (list, tuple)):
            img = torch.cat(list(img), 0)
        return self._patch_features_eager(img)

    def _graphed_patch_features(self, img) -> torch.Tensor:
        """`img` may be a list of image batches: they are copied into consecutive slices of the graph's static
        input (the fused step passes [img, img_pos] — no torch.cat of the two 19 MB batches)."""
        from .. import _lib
        self._prepared()
        graphs = self._cache.setdefault("graphs", {})
        parts = list(img) if isinstance(img, (list, tuple)) else [img]
        shape = (sum(p.shape[0] for p in parts),) + tuple(parts[0].shape[1:])
        dt = torch.bfloat16 if all(p.dtype == torch.bfloat16 for p in parts) else torch.float32
        key = (shape, parts[0].device.index, dt)
        if key not in graphs:
            img = torch.cat([p.to(dt) for p in parts], 0) if len(parts) > 1 else parts[0].to(dt)
            self._patch_features_eager(img)  # warm-up: kernel attributes, pos-embed cache, allocator
            torch.cuda.synchronize()
            static_in = img.detach().contiguous().clone()
            g = torch.cuda.CUDAGraph()
            n0 = _lib.load().stego_launch_count()
            with torch.cuda.graph(g):
                static_out = self._patch_features_eager(static_in)
            graphs[key] = (g, static_in, static_out, _lib.load().stego_launch_count() - n0)
        g, static_in, static_out, nlaunch = graphs[key]
        off = 0
        for part in parts:
            static_in[off:off + part.shape[0]].copy_(part)
            off += part.shape[0]
        g.replay()
        _lib.replayed_launches += nlaunch
        return static_out

    def _patch_features_eager(self, img: torch.Tensor) -> torch.Tensor:
        B = img.shape[0]
        x, _ = self.forward_tokens(img)
        w = self._prepared()
        N = x.shape[0] // B
        out = torch.empty(B * (N - 1), self.embed_dim, dtype=torch.bfloat16, device=x.device)
        ops.layernorm(x, w["nw"], w["nb"], out, eps=self.norm.eps, drop_cls_ntok=N)
        return out.view(B, N - 1, self.embed_dim)

    @torch.no_grad()
    def pooled_patch_features(self, img: torch.Tensor) -> torch.Tensor:
        """mean over the patch tokens of norm(last block) — `DinoFeaturizer(img)[0].mean([2, 3])` of
        src/precompute_knns.py:19 — fp32 [B, E], with the final LayerNorm and the pooling in one kernel (the [B, hw, E]
        feature map is never written)."""
        from .. import _lib
        B = img.shape[0]
        x, _ = self.forward_tokens(img)
        w = self._prepared()
        out = torch.zeros(B, self.embed_dim, dtype=torch.float32, device=x.device)
        _lib.check(_lib.load().stego_layernorm_gap(_lib.ptr(x), _lib.ptr(w["nw"]), _lib.ptr(w["nb"]), _lib.ptr(out), B,
                                                   x.shape[0] // B, self.embed_dim, float(self.norm.eps), _lib.stream()),
                   "stego_layernorm_gap")
        return out

    def _all_tokens(self, img: torch.Tensor, want_qkv: bool = False):
        B = img.shape[0]
        x, qkv = self.forward_tokens(img, want_qkv)
        w = self._prepared()
        out = torch.empty(x.shape[0], self.embed_dim, dtype=torch.bfloat16, device=x.device)
        ops.layernorm(x, w["nw"], w["nb"], out, eps=self.norm.eps)
        return out.view(B, -1, self.embed_dim), qkv

    # --- reference entry points ---------------------------------------------------------------
    def forward(self, x):
        """vision_transformer.py:211-216: cls token of the final norm."""
        tok, _ = self._all_tokens(x)
        return tok[:, 0].float()

    def forward_feats(self, x):
        tok, _ = self._all_tokens(x)
        return tok.float()

    def get_intermediate_feat(self, x, n=1):
        """vision_transformer.py:225-237.  Only n=1 (what STEGO uses) is provided.  Returns
        ([feat], [attn], [qkv]) like the reference: feat [B,N,E] fp32; qkv [3,B,heads,N,64];
        attn is None — the fused attention kernel never materialises the [B,heads,N,N] matrix and STEGO
        does not read it (src/modules.py:91-101)."""
        if n != 1:
            raise RuntimeError("stego_b200: get_intermediate_feat supports n=1 only")
        tok, qkv = self._all_tokens(x, want_qkv=True)
        B, N, E = tok.shape
        qkv = qkv.view(B, N, 3, self.num_heads, E // self.num_heads).permute(2, 0, 3, 1, 4).float()
        return [tok.float()], [None], [qkv]

    def get_intermediate_layers(self, x, n=1):
        if n != 1:
            raise RuntimeError("stego_b200: get_intermediate_layers supports n=1 only")
        tok, _ = self._all_tokens(x)
        return [tok.float()]


def vit_tiny(patch_size=16, **kwargs):
    raise ValueError("stego_b200: vit_tiny (head_dim 64, embed 192) is not built for this path")


def vit_small(patch_size=16, **kwargs):
    """vision_transformer.py:266-270."""
    return VisionTransformer(patch_size=patch_size, embed_dim=384, depth=12, num_heads=6, mlp_ratio=4,
                             qkv_bias=True, norm_layer=partial(nn.LayerNorm, eps=1e-6), **kwargs)


def vit_base(patch_size=16, **kwargs):
    """vision_transformer.py:273-277."""
    return VisionTransformer(patch_size=patch_size, embed_dim=768, depth=12, num_heads=12, mlp_ratio=4,
                             qkv_bias=True, norm_layer=partial(nn.LayerNorm, eps=1e-6), **kwargs)
