"""fp64 references of the frozen-ViT kernels, shared by the backbone tests.

Plain torch and device-agnostic: the GPU tests run these in float64 on the device, the CPU test pins them to the
oracle (oracle/stego_oracle.py).  `block_ref(..., rnd=True)` rounds to bf16 exactly where the kernel sequence stores
bf16 (LayerNorm output, qkv, attention output, GELU hidden) and keeps the residual stream fp32, so it is the
precision-faithful model of one block; `rnd=False` is the exact block.
"""
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if os.path.join(ROOT, "oracle") not in sys.path:
    sys.path.insert(0, os.path.join(ROOT, "oracle"))

BF16_U = 2.0 ** -8   # unit roundoff of bf16 (8-bit significand, round to nearest)
FP32_U = 2.0 ** -24  # unit roundoff of fp32
HEAD_DIM = 64
KEY_TILE = 64        # keys per tile of the fused attention kernel (csrc/attention.cu, ATT_BKV)

# The 2B backbone batches of the benchmark configurations: (arch, images, resolution, tokens, heads).
PROD = {"c1": ("vit_small", 64, 224, 785, 6), "c2": ("vit_base", 64, 320, 1601, 12), "c3": ("vit_base", 32, 448, 3137, 12)}

REGIMES = ("uniform", "sharp", "onehot", "allneg", "rising", "crossimage", "headtag")


def bf16(t):
    return t.to(torch.bfloat16).to(t.dtype)


def f32(t):
    return t.to(torch.float32).to(t.dtype)


def bf16_ulp(t):
    """Spacing of bf16 numbers at |t| (fp64 in, fp64 out); zeros get the spacing at the smallest normal."""
    m, e = torch.frexp(t.double().abs().clamp_min(2.0 ** -126))  # |t| = m 2^e, m in [0.5, 1)
    return torch.ldexp(torch.ones_like(m), e - 8)


def rel_l2(x, y):
    x, y = x.double(), y.double()
    return ((x - y).norm() / y.norm().clamp_min(1e-300)).item()


# ------------------------------------------------------------------------------------------------
# attention
# ------------------------------------------------------------------------------------------------
def _split(qkv, B, N, heads):
    """Packed [B*N, 3E] (q | k | v, head-major) -> q, k, v as [B, heads, N, 64] fp64."""
    return qkv.double().view(B, N, 3, heads, HEAD_DIM).permute(2, 0, 3, 1, 4).unbind(0)


def scaled_logits(qkv, B, N, heads):
    """q k^T / 8 for every image and head, [B, heads, N, N] fp64 (small shapes only)."""
    q, k, _ = _split(qkv, B, N, heads)
    return (q @ k.transpose(-2, -1)) * (HEAD_DIM ** -0.5)


def attention_ref(qkv, B, N, heads, max_bytes=4 << 30):
    """fp64 softmax(q k^T / 8) v of a packed [B*N, 3E] qkv, in chunks of images that keep the scores under
    `max_bytes`.  Returns [B*N, E] fp64 in the kernel's output layout (head-major columns)."""
    E = heads * HEAD_DIM
    per = max(1, int(max_bytes // (2 * heads * N * N * 8)))
    out = torch.empty(B, N, heads, HEAD_DIM, dtype=torch.float64, device=qkv.device)
    x = qkv.view(B, N, 3 * E)
    for b0 in range(0, B, per):
        b1 = min(B, b0 + per)
        q, k, v = _split(x[b0:b1], b1 - b0, N, heads)
        s = (q @ k.transpose(-2, -1)) * (HEAD_DIM ** -0.5)
        out[b0:b1] = (s.softmax(-1) @ v).transpose(1, 2)
        del q, k, v, s
    return out.view(B * N, E)


def onehot_targets(N):
    """Dominant key positions of the one-hot regime: the first key, both sides of the first tile boundary, the first
    key of the last (ragged) tile and the last key."""
    last_tile = KEY_TILE * ((N - 1) // KEY_TILE)
    return sorted({t for t in (0, KEY_TILE - 1, KEY_TILE, last_tile, N - 1) if t < N})


def attention_inputs(regime, B, N, heads, seed=0, device="cpu"):
    """bf16 packed qkv [B*N, 3E] for one input regime.  Each regime makes a specific kernel bug change the output by
    O(1) (scaled logit = q.k / 8; per-element std s of q and k gives a logit std of s^2):
      uniform    : logit std 0.15 (vit_random_state statistics): attention is nearly mean(v)
      sharp      : logit std 6 (trained DINO): softmax errors are no longer averaged away
      onehot     : every query has one key 72 logits above the rest, at onehot_targets(N): a dropped or shifted key
      allneg     : every real logit is about -40 and v is about 1: a zero-filled padding key (logit 0) let into the
                   softmax takes all the mass and drives the output to 0
      rising     : the row maximum rises tile after tile, alternately by about 8 and 3 (at least 1 into a ragged
                   last tile): a missing or wrong rescale of the running output reweights whole tiles
      crossimage : image b's queries point along channel b % 2, its first 64 keys along the other one, i.e. at the
                   queries of images b - 1 and b + 1 (logit 30 there): keys read from a neighbouring image dominate
      headtag    : sharp, with head h's v offset by 4 h: a head reading another head's v is off by 4 or more"""
    g = torch.Generator(device=device).manual_seed(seed)

    def rn(*shape):
        return torch.randn(*shape, generator=g, device=device)

    shp = (B, N, heads, HEAD_DIM)
    v = rn(*shp)
    if regime == "uniform":
        q, k = 0.387 * rn(*shp), 0.387 * rn(*shp)
    elif regime in ("sharp", "headtag"):
        q, k = 2.449 * rn(*shp), 2.449 * rn(*shp)
        if regime == "headtag":
            v = v + 4.0 * torch.arange(heads, device=device, dtype=v.dtype).view(1, 1, heads, 1)
    elif regime == "onehot":
        q, k = 0.3 * rn(*shp), 0.3 * rn(*shp)
        tgt = torch.tensor(onehot_targets(N), device=device)
        rows = torch.arange(N, device=device)
        k[:, tgt, :, torch.arange(len(tgt), device=device)] = 24.0  # target t_i carries channel i
        q[:, rows, :, rows % len(tgt)] = 24.0                      # query i wants target i % T
    elif regime == "allneg":
        q, k = 0.5 * rn(*shp), 0.5 * rn(*shp)
        q[..., 0] = 8.0
        k[..., 0] = -40.0 + 0.5 * rn(B, N, heads)
        v = 1.0 + 0.01 * v
    elif regime == "rising":
        q, k = 0.25 * rn(*shp), 0.25 * rn(*shp)
        j = torch.arange(N, device=device, dtype=torch.float32)
        t = j // KEY_TILE
        r = 5.5 * t + 2.5 * (t % 2) + (j % KEY_TILE) / 32.0  # tile maxima rise by 8, 3, 8, 3, ...
        hi = r.bfloat16().float()                            # logit r = hi + lo, both bf16-exact
        q[..., :2] = 8.0
        k[..., 0] = hi.view(1, N, 1)
        k[..., 1] = (r - hi).view(1, N, 1)
    elif regime == "crossimage":
        q, k = 0.5 * rn(*shp), 0.5 * rn(*shp)
        par = torch.arange(B, device=device) % 2
        for b in range(B):
            q[b, :, :, int(par[b])] += 6.0
            k[b, :KEY_TILE, :, 1 - int(par[b])] += 40.0
    else:
        raise ValueError(regime)
    E = heads * HEAD_DIM
    return torch.stack((q, k, v), 2).reshape(B * N, 3 * E).to(torch.bfloat16).contiguous()


# ------------------------------------------------------------------------------------------------
# LayerNorm and the block
# ------------------------------------------------------------------------------------------------
def layer_norm(x, w, b, eps):
    """fp64 LayerNorm over the last dimension (biased variance, like nn.LayerNorm)."""
    x = x.double()
    mean = x.mean(-1, keepdim=True)
    var = (x - mean).square().mean(-1, keepdim=True)
    return (x - mean) / torch.sqrt(var + eps) * w.double() + b.double()


def block_params(sd, i):
    """Block i of a reference-named state dict, fp64."""
    p = f"blocks.{i}."
    names = ("norm1.weight", "norm1.bias", "attn.qkv.weight", "attn.qkv.bias", "attn.proj.weight", "attn.proj.bias",
             "norm2.weight", "norm2.bias", "mlp.fc1.weight", "mlp.fc1.bias", "mlp.fc2.weight", "mlp.fc2.bias")
    return {n: sd[p + n].double() for n in names}


def block_ref(x, prm, B, N, heads, eps=1e-6, rnd=True):
    """One pre-LN block in fp64 from the residual stream x [B*N, E].  rnd=True: GEMM weights and the LayerNorm
    output, qkv, attention output and GELU hidden are rounded to bf16 and the residual to fp32, where the kernels
    store them.  Returns (x_out [B*N, E], qkv [B*N, 3E]), fp64."""
    r16 = bf16 if rnd else (lambda t: t)
    r32 = f32 if rnd else (lambda t: t)
    W = {n: (r16(t) if n.endswith("weight") and not n.startswith("norm") else t) for n, t in prm.items()}
    x = r32(x.double())
    y = r16(layer_norm(x, W["norm1.weight"], W["norm1.bias"], eps))
    qkv = r16(F.linear(y, W["attn.qkv.weight"], W["attn.qkv.bias"]))
    a = r16(attention_ref(qkv, B, N, heads))
    x = r32(x + F.linear(a, W["attn.proj.weight"], W["attn.proj.bias"]))
    y = r16(layer_norm(x, W["norm2.weight"], W["norm2.bias"], eps))
    h = r16(F.gelu(F.linear(y, W["mlp.fc1.weight"], W["mlp.fc1.bias"])))
    x = r32(x + F.linear(h, W["mlp.fc2.weight"], W["mlp.fc2.bias"]))
    return x, qkv


def embed_ref(sd, img, patch):
    """Patch embedding + cls token + (interpolated) position table, fp64, [B, N, E]."""
    import stego_oracle as O
    B = img.shape[0]
    x = F.conv2d(img.double(), sd["patch_embed.proj.weight"].double(), sd["patch_embed.proj.bias"].double(), stride=patch)
    x = torch.cat((sd["cls_token"].double().expand(B, -1, -1), x.flatten(2).transpose(1, 2)), 1)
    return x + O.interpolate_pos_embed(sd["pos_embed"].double(), img.shape[2], img.shape[3], patch)


def vit_tokens(sd, img, arch, patch=8):
    """The whole backbone in exact fp64 from the blocks above: (norm(last block) [B, N, E], last qkv [B*N, 3E])."""
    import stego_oracle as O
    cfg = O.vit_config(arch)
    E, heads = cfg["embed_dim"], cfg["heads"]
    x = embed_ref(sd, img, patch)
    B, N = x.shape[:2]
    x = x.reshape(B * N, E)
    qkv = None
    for i in range(cfg["depth"]):
        x, qkv = block_ref(x, block_params(sd, i), B, N, heads, rnd=False)
    return layer_norm(x, sd["norm.weight"], sd["norm.bias"], 1e-6).view(B, N, E), qkv


def logit_std(qkv, B, N, heads, max_images=2):
    """Mean over rows (and heads) of the std of the scaled logits along the keys, from the first images."""
    b = min(B, max_images)
    s = scaled_logits(qkv.view(B, N, -1)[:b].reshape(b * N, -1), b, N, heads)
    return s.std(-1).mean().item()
