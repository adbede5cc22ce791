"""Thin Python wrappers over the C-ABI entry points of the GEMMs, the attention and the ViT glue.

These take torch CUDA tensors, pass raw device pointers + sizes + the current stream through
ctypes and return torch tensors.  They allocate outputs with torch (PyTorch owns all memory) and
never fall back to torch math.  The training step's other entry points are called from the stage functions in
modules.py, corr.py and segmenter.py, which share from here the probes' input formats (label dtypes, tokens-major
code view, partials scratch) and the split-K rule of the head's weight-gradient GEMMs.
"""
from __future__ import annotations

from typing import Optional

import torch

from . import _lib

ACT_NONE, ACT_GELU, ACT_RELU = 0, 1, 2


def gemm(a: torch.Tensor, b: torch.Tensor, out: torch.Tensor, *, M: int, N: int, K: int,
         a_mn: bool = False, b_mn: bool = False, bias: Optional[torch.Tensor] = None, act: int = ACT_NONE,
         residual: Optional[torch.Tensor] = None, row_div: int = 0, splits: int = 1,
         atomic: bool = False) -> torch.Tensor:
    """out[M,N] = act(A.B^T + bias) + residual on wgmma (see include/stego_b200.h: stego_gemm_bf16)."""
    _lib.require_cuda(a, b, out, bias, residual)
    assert a.dtype == torch.bfloat16 and b.dtype == torch.bfloat16
    assert a.dim() == 2 and b.dim() == 2 and out.dim() == 2
    assert a.stride(1) == 1 and b.stride(1) == 1 and out.stride(1) == 1
    assert out.dtype in (torch.bfloat16, torch.float32)
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.is_contiguous()
    if residual is not None:
        assert residual.dtype == torch.float32 and residual.stride(1) == 1
    rc = _lib.load().stego_gemm_bf16(
        _lib.ptr(a), a.stride(0), int(a_mn), _lib.ptr(b), b.stride(0), int(b_mn), M, N, K,
        _lib.ptr(out), out.stride(0), int(out.dtype == torch.bfloat16), _lib.ptr(bias), act,
        _lib.ptr(residual), residual.stride(0) if residual is not None else 0, row_div, splits, int(atomic),
        _lib.stream())
    _lib.check(rc, "stego_gemm_bf16")
    return out


def wgrad_splits(K: int, out_rows: int, out_cols: int, num_sms: int) -> int:
    """Split-K count of a weight-gradient GEMM (K = activation rows): tiles x splits fills ONE wave of the persistent
    GEMM grid (one CTA per SM; more splits would make a second round of the grid), each split at least 512 rows deep."""
    tiles = ((out_rows + 127) // 128) * ((out_cols + 127) // 128)
    return max(1, min(K // 512, num_sms // tiles))


def gemm_batched(a: torch.Tensor, b: torch.Tensor, out: torch.Tensor, *, a_mn: bool = False, b_mn: bool = False,
                 bias: Optional[torch.Tensor] = None, act: int = ACT_NONE) -> torch.Tensor:
    """out[n] = act(A[n] . B[n]^T + bias) for every n in ONE launch (stego_gemm_bf16_batched).
    a: [n, M, K] (or [n, K, M] if a_mn), b: [n, N, K] (or [n, K, N] if b_mn), bf16, inner dimension contiguous;
    out: [n, M, N] fp32 or bf16."""
    _lib.require_cuda(a, b, out, bias)
    assert a.dtype == torch.bfloat16 and b.dtype == torch.bfloat16 and a.dim() == 3 and b.dim() == 3 and out.dim() == 3
    assert a.stride(2) == 1 and b.stride(2) == 1 and out.stride(2) == 1 and out.dtype in (torch.bfloat16, torch.float32)
    n = a.shape[0]
    M, K = (a.shape[2], a.shape[1]) if a_mn else (a.shape[1], a.shape[2])
    N = b.shape[2] if b_mn else b.shape[1]
    assert b.shape[0] == n and out.shape == (n, M, N) and (b.shape[1] if b_mn else b.shape[2]) == K
    rc = _lib.load().stego_gemm_bf16_batched(
        _lib.ptr(a), a.stride(1), a.stride(0), int(a_mn), _lib.ptr(b), b.stride(1), b.stride(0), int(b_mn), n, M, N, K,
        _lib.ptr(out), out.stride(1), out.stride(0), int(out.dtype == torch.bfloat16), _lib.ptr(bias), act, _lib.stream())
    _lib.check(rc, "stego_gemm_bf16_batched")
    return out


def patchify(img: torch.Tensor, patch: int) -> torch.Tensor:
    """PatchEmbed im2col rows [B*hw, 3*p*p] bf16 (stego_vit_patchify / stego_vit_patchify_bf16)."""
    _lib.require_cuda(img)
    assert img.dtype in (torch.float32, torch.bfloat16) and img.is_contiguous() and img.shape[1] == 3
    B, _, H, W = img.shape
    out = torch.empty(B * (H // patch) * (W // patch), 3 * patch * patch, dtype=torch.bfloat16, device=img.device)
    lib = _lib.load()
    fn = lib.stego_vit_patchify if img.dtype == torch.float32 else lib.stego_vit_patchify_bf16
    _lib.check(fn(_lib.ptr(img), _lib.ptr(out), B, H, W, patch, _lib.stream()), "stego_vit_patchify")
    return out


def patchify_tta(img: torch.Tensor, patch: int) -> torch.Tensor:
    """Flip-TTA im2col rows [2B*hw, 3*p*p] bf16 of img [B, 3, H, W] (fp32 or bf16): the rows of img, then those of
    img.flip(3), which is never materialised (stego_vit_patchify_tta)."""
    _lib.require_cuda(img)
    assert img.dtype in (torch.float32, torch.bfloat16) and img.is_contiguous() and img.shape[1] == 3
    B, _, H, W = img.shape
    out = torch.empty(2 * B * (H // patch) * (W // patch), 3 * patch * patch, dtype=torch.bfloat16, device=img.device)
    _lib.check(_lib.load().stego_vit_patchify_tta(_lib.ptr(img), int(img.dtype == torch.bfloat16), _lib.ptr(out), B, H, W,
                                                  patch, _lib.stream()), "stego_vit_patchify_tta")
    return out


def cls_rows(x: torch.Tensor, cls_token: torch.Tensor, pos_embed: torch.Tensor, B: int, ntok: int) -> None:
    E = x.shape[-1]
    _lib.check(_lib.load().stego_vit_cls_rows(_lib.ptr(x), _lib.ptr(cls_token), _lib.ptr(pos_embed), B, ntok, E,
                                              _lib.stream()), "stego_vit_cls_rows")


def layernorm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, out: torch.Tensor, eps: float = 1e-6,
              drop_cls_ntok: int = 0) -> torch.Tensor:
    """fp32 [rows,E] -> bf16 LayerNorm (stego_layernorm_bf16)."""
    _lib.require_cuda(x, gamma, beta, out)
    assert x.dtype == torch.float32 and x.is_contiguous() and out.dtype == torch.bfloat16 and out.is_contiguous()
    rows, E = x.shape
    _lib.check(_lib.load().stego_layernorm_bf16(_lib.ptr(x), _lib.ptr(gamma), _lib.ptr(beta), _lib.ptr(out), rows, E,
                                                eps, drop_cls_ntok, _lib.stream()), "stego_layernorm_bf16")
    return out


def linear_rows_f32(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None) -> torch.Tensor:
    """fp32 [B, K] . bf16 [N, K]^T (+ fp32 bias [N]) -> new fp32 [B, N] (stego_linear_rows_f32).  w may be a row slice
    of a larger weight (inner dimension contiguous)."""
    _lib.require_cuda(x, w, bias)
    assert x.dtype == torch.float32 and x.dim() == 2 and x.is_contiguous()
    assert w.dtype == torch.bfloat16 and w.dim() == 2 and w.stride(1) == 1 and w.shape[1] == x.shape[1]
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.is_contiguous() and bias.numel() == w.shape[0]
    B, K = x.shape
    N = w.shape[0]
    out = torch.empty(B, N, dtype=torch.float32, device=x.device)
    _lib.check(_lib.load().stego_linear_rows_f32(_lib.ptr(x), _lib.ptr(w), w.stride(0), _lib.ptr(bias), _lib.ptr(out),
                                                 B, N, K, _lib.stream()), "stego_linear_rows_f32")
    return out


def attention(qkv: torch.Tensor, out: torch.Tensor, B: int, N: int, E: int, heads: int) -> torch.Tensor:
    """Fused softmax(q k^T / 8) v on wgmma (stego_attention_fwd). qkv [B*N, 3E] bf16, out [B*N, E] bf16."""
    _lib.require_cuda(qkv, out)
    assert qkv.dtype == torch.bfloat16 and qkv.is_contiguous() and out.dtype == torch.bfloat16 and out.is_contiguous()
    _lib.check(_lib.load().stego_attention_fwd(_lib.ptr(qkv), _lib.ptr(out), B, N, E, heads, _lib.stream()),
               "stego_attention_fwd")
    return out


def attention_probs(qkv: torch.Tensor, out: torch.Tensor, B: int, N: int, E: int, heads: int) -> torch.Tensor:
    """softmax(q k^T / 8) as fp32 [B, heads, N, N] (stego_attention_probs). qkv [B*N, 3E] bf16."""
    _lib.require_cuda(qkv, out)
    assert qkv.dtype == torch.bfloat16 and qkv.is_contiguous() and qkv.shape == (B * N, 3 * E)
    assert out.dtype == torch.float32 and out.is_contiguous() and out.numel() == B * heads * N * N
    _lib.check(_lib.load().stego_attention_probs(_lib.ptr(qkv), _lib.ptr(out), B, N, E, heads, _lib.stream()),
               "stego_attention_probs")
    return out


# label dtypes the probe kernels read directly, by element size (int64 is the reference's; uint8 uses 255 = ignore)
LABEL_BYTES = {torch.int64: 8, torch.int32: 4, torch.uint8: 1}


def probe_label(label: torch.Tensor, B: int, H: int, W: int):
    """(label, label_bytes) as the probe kernels read it: [B, H, W] contiguous int64 / int32 / uint8; any other dtype
    becomes int64."""
    lab = label.reshape(B, H, W)
    if lab.dtype not in LABEL_BYTES:
        lab = lab.to(torch.long)
    lab = lab.contiguous()
    return lab, LABEL_BYTES[lab.dtype]


def tokens_major(code: torch.Tensor) -> torch.Tensor:
    """Detached fp32 view of code [B, C, h, w] whose pixel (b, y, x) is row b*h*w + y*w + x at stride ld = stride(3),
    channels contiguous: the addressing of the probe kernels.  Other views (NCHW, code[::2], crops) are copied."""
    x = code.detach()
    B, _, h, w = x.shape
    if (x.dtype != torch.float32 or x.stride(1) != 1 or x.stride(2) != w * x.stride(3)
            or (B > 1 and x.stride(0) != h * w * x.stride(3))):
        x = x.float().permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
    return x


def probe_scratch(device) -> torch.Tensor:
    """The partials scratch of stego_cluster_lookup_fwd and stego_linear_probe_ce: 16 floats per SM."""
    sms = torch.cuda.get_device_properties(device).multi_processor_count
    return torch.empty(16 * sms, dtype=torch.float32, device=device)
