"""The frozen-ViT kernels against float64 references at the production shapes, with sharp attention and adversarial
edges: fused attention, LayerNorm (+ drop_cls, + global average pool), patchify / cls_rows / patch embed, one block
against a precision-faithful fp64 block, CUDA-graph replay, patch 16 and the KK features.

The bars are derived from the arithmetic (see each test and DESIGN.md section 4) and the measured errors are written to
$STEGO_PARITY_DIR when it is set.
"""
import copy
import os
import sys
from functools import partial

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _vit_fp64 as R  # noqa: E402
from _parity_util import fp32_strict, record, rel  # noqa: E402

pytestmark = pytest.mark.gpu

SENTINEL = 0x7FC1  # a NaN bit pattern no kernel produces (they write canonical NaNs or finite values)
GUARD = 64


def _guarded(rows, cols, dev):
    """bf16 [rows + GUARD, cols] filled with the sentinel bits; the first `rows` rows are the output."""
    buf = torch.empty(rows + GUARD, cols, dtype=torch.bfloat16, device=dev)
    buf.view(torch.int16).fill_(SENTINEL)
    return buf


def _guard_intact(buf, rows):
    return bool((buf[rows:].view(torch.int16) == SENTINEL).all())


# ================================================================================================
# 1. fused attention
# ================================================================================================
# relative-L2 bars per regime, about 1.7x the largest value measured on an H100 over the production and ragged shapes
# (uniform 2.4e-3, sharp 1.7e-3, allneg 2.0e-3, rising 2.3e-3, crossimage 2.4e-3, headtag 1.7e-3; one-hot outputs are
# the dominant key's v exactly, 0).  The elementwise bar in _check_attention is the derived one.
ATT_REL_L2 = {"uniform": 4e-3, "sharp": 3e-3, "onehot": 1e-4, "allneg": 3.5e-3, "rising": 4e-3, "crossimage": 4e-3,
              "headtag": 3e-3}


def _check_attention(dev, B, N, heads, regime, seed):
    """Elementwise bar |out - ref| <= 2^-8 (|ref| + max_j |v[j, d]|): P is rounded to bf16 (relative error <= u = 2^-8)
    for the P V product while the row sum l adds the unrounded fp32 values, so sum_j dP_j v_j / l <= u max_j |v_j|;
    the output is rounded to bf16 once more (<= u |out|).  Scores, exponentials and sums in fp32 add O(1e-6)."""
    from stego_b200 import ops
    E = heads * 64
    qkv = R.attention_inputs(regime, B, N, heads, seed=seed, device=dev)
    buf = _guarded(B * N, E, dev)
    out = buf[:B * N]
    ops.attention(qkv, out, B, N, E, heads)
    again = torch.empty_like(out)
    ops.attention(qkv, again, B, N, E, heads)
    torch.cuda.synchronize()
    assert _guard_intact(buf, B * N), (regime, "wrote past the last row")
    assert torch.isfinite(out.float()).all(), (regime, "unwritten or non-finite rows")
    assert torch.equal(out.view(torch.int16), again.view(torch.int16)), (regime, "launches differ")
    ref = R.attention_ref(qkv, B, N, heads).view(B, N, E)
    vmax = qkv.view(B, N, 3, E)[:, :, 2].double().abs().amax(1, keepdim=True)  # [B, 1, E]: over that image's keys
    err = (out.double().view(B, N, E) - ref).abs()
    ratio = (err / (R.BF16_U * (ref.abs() + vmax))).max().item()
    r = R.rel_l2(out, ref.view(B * N, E))
    del ref, err, vmax, qkv
    return ratio, r


def _attention_case(dev, tag, B, N, heads, regimes=R.REGIMES):
    res = {}
    for i, regime in enumerate(regimes):
        ratio, r = _check_attention(dev, B, N, heads, regime, seed=100 + i)
        res[regime] = dict(max_err_over_bar=ratio, rel_l2=r, rel_l2_bar=ATT_REL_L2[regime])
    record(f"vit_fp64_attention_{tag}", dict(B=B, N=N, heads=heads, regimes=res))
    for regime, m in res.items():
        assert m["max_err_over_bar"] <= 1.0, (tag, regime, m)
        assert m["rel_l2"] < ATT_REL_L2[regime], (tag, regime, m)
    return res


@pytest.mark.parametrize("shape", ["c1", "c2", "c3"])
def test_attention_production_shapes(cuda_dev, shape):
    """Every row of the real 2B batches; at c3 (N = 3137) the second warpgroup of the last query tile owns one valid
    row and the last key tile holds one key."""
    _, B, _, N, heads = R.PROD[shape]
    _attention_case(cuda_dev, shape, B, N, heads)
    torch.cuda.empty_cache()


@pytest.mark.parametrize("heads", [1, 6, 12])
@pytest.mark.parametrize("N", [1, 2, 63, 64, 65, 127, 128, 129, 191, 192, 193, 257])
def test_attention_ragged(cuda_dev, N, heads):
    _attention_case(cuda_dev, f"ragged_N{N}_h{heads}", 3, N, heads)


# ================================================================================================
# 2. LayerNorm, drop_cls and LayerNorm + GAP
# ================================================================================================
LN_KINDS = ("normal", "offset", "outlier", "flat", "constant")


def _ln_rows(kind, rows, E, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn(rows, E, generator=g, device=dev)
    if kind == "offset":
        x = x + 1e3
    elif kind == "outlier":
        ch = torch.tensor([3, E // 3, E // 2 + 1, E - 5], device=dev)
        x[:, ch] = torch.tensor([300.0, -300.0, 300.0, -300.0], device=dev)
    elif kind == "flat":
        x = 0.25 + 1e-3 * x  # variance 1e-6, the size of eps
    elif kind == "constant":
        x = torch.full_like(x, 3.0)
    return x.contiguous()


def _ln_affine(E, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    return torch.randn(E, generator=g, device=dev), torch.randn(E, generator=g, device=dev)


def _ln_bar(x, gamma, beta, ref, eps):
    """1 bf16 ulp of ref + the fp32 statistics floor K u (|gamma| (|xhat| + |mean| rstd + 1) + |beta|): the fp32 sums
    err by a few ulps of |mean| (then scaled by rstd), rsqrtf and the affine by a few ulps of each term.  K = 32 keeps
    the floor at <= 1e-5 |gamma| for rows without an offset and |xhat| <= 4."""
    xd = x.double()
    mean = xd.mean(-1, keepdim=True)
    rstd = torch.rsqrt((xd - mean).square().mean(-1, keepdim=True) + eps)
    xhat = (xd - mean) * rstd
    floor = 32 * R.FP32_U * (gamma.double().abs() * (xhat.abs() + mean.abs() * rstd + 1) + beta.double().abs())
    return R.bf16_ulp(ref) + floor


@pytest.mark.parametrize("kind", LN_KINDS)
@pytest.mark.parametrize("E", [128, 384, 768])
def test_layernorm_fp64(cuda_dev, E, kind):
    from stego_b200 import ops
    eps = 1e-6
    gamma, beta = _ln_affine(E, cuda_dev, seed=E)
    prod = {128: [64 * 785], 384: [64 * 785], 768: [64 * 1601, 32 * 3137]}[E]
    worst = {}
    for rows in [1, 7, 8, 9] + prod:
        x = _ln_rows(kind, rows, E, cuda_dev, seed=rows)
        buf = _guarded(rows, E, cuda_dev)
        out = buf[:rows]
        ops.layernorm(x, gamma, beta, out, eps=eps)
        torch.cuda.synchronize()
        assert _guard_intact(buf, rows), (rows, "wrote past the last row")
        ref = R.layer_norm(x, gamma, beta, eps)
        err = (out.double() - ref).abs()
        ratio = (err / _ln_bar(x, gamma, beta, ref, eps)).max().item()
        worst[rows] = dict(max_err_over_bar=ratio, max_abs_err=err.max().item())
        assert ratio <= 1.0, (E, kind, rows, worst[rows])
        if kind == "constant":  # x - mean == 0 exactly: the output is beta rounded once
            assert torch.equal(out, beta.bfloat16().expand(rows, E))
    record(f"vit_fp64_layernorm_E{E}_{kind}", worst)


@pytest.mark.parametrize("shape", ["c1", "c2", "c3"])
def test_layernorm_drop_cls_rows(cuda_dev, shape):
    """drop_cls compacts token t >= 1 of image b to row b (N - 1) + t - 1, bit-identical to the plain LayerNorm of that
    row; nothing is written past B (N - 1) rows."""
    from stego_b200 import ops
    arch, B, _, N, _ = R.PROD[shape]
    E = 384 if arch == "vit_small" else 768
    gamma, beta = _ln_affine(E, cuda_dev, seed=1)
    x = _ln_rows("outlier", B * N, E, cuda_dev, seed=2)
    x += torch.arange(B * N, device=cuda_dev, dtype=torch.float32).view(-1, 1) % 97 * 0.01  # rows tell apart
    full = torch.empty(B * N, E, dtype=torch.bfloat16, device=cuda_dev)
    ops.layernorm(x, gamma, beta, full, eps=1e-6)
    buf = _guarded(B * (N - 1), E, cuda_dev)
    ops.layernorm(x, gamma, beta, buf[:B * (N - 1)], eps=1e-6, drop_cls_ntok=N)
    torch.cuda.synchronize()
    assert _guard_intact(buf, B * (N - 1))
    got = buf[:B * (N - 1)].view(B, N - 1, E)
    want = full.view(B, N, E)[:, 1:]
    bad = (got.view(torch.int16) != want.view(torch.int16)).any(-1).nonzero()
    assert bad.numel() == 0, f"{bad.shape[0]} misplaced rows, first (image, token-1) {bad[:4].tolist()}"
    ref = R.layer_norm(x.view(B, N, E)[:, 1:], gamma, beta, 1e-6)
    ratio = ((got.double() - ref).abs() / _ln_bar(x.view(B, N, E)[:, 1:], gamma, beta, ref, 1e-6)).max().item()
    record(f"vit_fp64_layernorm_drop_cls_{shape}", dict(max_err_over_bar=ratio))
    assert ratio <= 1.0


def _ln_gap(x, gamma, beta, out, B, ntok, E):
    from stego_b200 import _lib
    _lib.check(_lib.load().stego_layernorm_gap(_lib.ptr(x), _lib.ptr(gamma), _lib.ptr(beta), _lib.ptr(out), B, ntok, E,
                                               1e-6, _lib.stream()), "stego_layernorm_gap")


@pytest.mark.parametrize("E", [384, 768])
@pytest.mark.parametrize("ntok", [2, 65, 66, 785, 1601, 3137])
def test_layernorm_gap_fp64(cuda_dev, ntok, E):
    """Mean over the patch tokens of the fp64 LayerNorm, within 1e-5 of the terms' scale; the 64-token chunks end
    mid-chunk (66, 785) and on a boundary (65); the kernel accumulates into `out` (the caller zeroes it)."""
    B = 3
    gamma, beta = _ln_affine(E, cuda_dev, seed=7)
    x = _ln_rows("outlier", B * ntok, E, cuda_dev, seed=ntok)
    g = torch.Generator(device=cuda_dev).manual_seed(8)
    x += 2.0 * torch.randn(E, generator=g, device=cuda_dev)  # a per-channel pattern the pool keeps
    ref = R.layer_norm(x.view(B, ntok, E)[:, 1:], gamma, beta, 1e-6).mean(1)  # [B, E]
    scale = ref.abs() + beta.double().abs() + gamma.double().abs()
    out = torch.zeros(B, E, device=cuda_dev)
    _ln_gap(x, gamma, beta, out, B, ntok, E)
    pre = torch.randn(B, E, generator=g, device=cuda_dev)
    acc = pre.clone()
    _ln_gap(x, gamma, beta, acc, B, ntok, E)
    torch.cuda.synchronize()
    e0 = ((out.double() - ref).abs() / scale).max().item()
    e1 = ((acc.double() - (pre.double() + ref)).abs() / (scale + pre.double().abs())).max().item()
    r = R.rel_l2(out, ref)
    record(f"vit_fp64_layernorm_gap_ntok{ntok}_E{E}", dict(max_err_over_scale=e0, prefilled_max_err=e1, rel_l2=r))
    assert e0 < 1e-5 and r < 1e-5, (e0, r)
    assert e1 < 1e-5, e1


# ================================================================================================
# 3. embed stage
# ================================================================================================
EMBED_SIZES = [(224, 224), (320, 320), (448, 448), (224, 320), (96, 64)]


@pytest.mark.parametrize("H,W", [(224, 224), (224, 320), (96, 64)])
@pytest.mark.parametrize("p", [8, 16])
def test_patchify_exact(cuda_dev, p, H, W):
    from stego_b200 import ops
    torch.manual_seed(p * 1000 + H + W)
    img = torch.randn(3, 3, H, W, device=cuda_dev) * 3
    want = F.unfold(img, p, stride=p).transpose(1, 2).reshape(-1, 3 * p * p).bfloat16()
    assert torch.equal(ops.patchify(img, p), want)
    ib = img.bfloat16()
    want_b = F.unfold(ib.float(), p, stride=p).transpose(1, 2).reshape(-1, 3 * p * p).bfloat16()
    got_b = ops.patchify(ib, p)  # stego_vit_patchify_bf16
    assert torch.equal(got_b, want_b)
    assert torch.equal(got_b, ops.patchify(ib.float(), p))  # bit-identical to the fp32 entry on bf16 values


def _vit(E, heads, p, depth=1):
    from stego_b200.dino.vision_transformer import VisionTransformer
    return VisionTransformer(patch_size=p, embed_dim=E, depth=depth, num_heads=heads, qkv_bias=True,
                             norm_layer=partial(nn.LayerNorm, eps=1e-6))


def _zero_blocks(model):
    with torch.no_grad():
        for blk in model.blocks:
            for lin in (blk.attn.qkv, blk.attn.proj, blk.mlp.fc1, blk.mlp.fc2):
                lin.weight.zero_()
                lin.bias.zero_()


@pytest.mark.parametrize("p", [8, 16])
def test_embed_stage_fp64(cuda_dev, p):
    """A depth-1 ViT whose block adds exactly 0: forward_tokens is the embed output.  The cls rows are bit-equal to
    fp32 cls + pos[0]; the patch rows (bf16 conv operands, fp32 accumulation, + bias + interpolated position table)
    are within 1e-5 of the fp64 value relative to the sum of the magnitudes of its terms."""
    torch.manual_seed(20 + p)
    model = _vit(384, 6, p)
    with torch.no_grad():
        model.pos_embed.normal_(0, 0.5)
        model.cls_token.normal_(0, 0.5)
        model.patch_embed.proj.bias.normal_(0, 0.1)
    _zero_blocks(model)
    model = model.to(cuda_dev)
    sd = {k: v.detach() for k, v in model.state_dict().items()}
    res = {}
    for H, W in EMBED_SIZES:
        B = 3
        img = torch.randn(B, 3, H, W, device=cuda_dev)
        x, _ = model.forward_tokens(img)
        N = (H // p) * (W // p) + 1
        x = x.view(B, N, 384)
        cls_want = (sd["cls_token"].float() + sd["pos_embed"][:, 0].float()).view(1, 384).expand(B, 384)
        assert torch.equal(x[:, 0], cls_want), (p, H, W)
        sdq = dict(sd, **{"patch_embed.proj.weight": sd["patch_embed.proj.weight"].bfloat16().double()})
        ref = R.embed_ref(sdq, img.bfloat16().double(), p)
        mag = R.embed_ref({k: v.double().abs() for k, v in sdq.items()}, img.bfloat16().double().abs(), p)
        e = ((x[:, 1:].double() - ref[:, 1:]).abs() / mag[:, 1:]).max().item()
        r = R.rel_l2(x[:, 1:], ref[:, 1:])
        res[f"{H}x{W}"] = dict(max_err_over_magnitude=e, rel_l2=r)
        assert e < 1e-5 and r < 1e-5, (p, H, W, e, r)
    record(f"vit_fp64_embed_p{p}", res)


# ================================================================================================
# 4. one block at the production shapes, sharp attention, outlier residual channels
# ================================================================================================
# Measured on an H100 against the precision-faithful block: block output (x_out - x_in) 6.2e-4 (c1) to 7.5e-4 (c3),
# qkv 4.3e-5 to 6.7e-5.  Against the exact fp64 block (recorded only) the block output differs by 3.6e-3 to 5.3e-3.
BLOCK_REL_L2 = 1.5e-3
QKV_REL_L2 = 2e-4


def _sharp_block_model(arch, dev):
    import stego_oracle as O
    cfg = O.vit_config(arch)
    E, heads = cfg["embed_dim"], cfg["heads"]
    sd = O.perturb_vit_state(O.vit_random_state(arch, 8, seed=3))
    sd = {k: v for k, v in sd.items() if not k.startswith("blocks.") or k.startswith("blocks.0.")}
    model = _vit(E, heads, 8)
    model.load_state_dict(sd)
    with torch.no_grad():
        b = model.patch_embed.proj.bias  # outlier channels of the residual stream, as in trained DINO
        b[torch.tensor([5, E // 4, E // 2 + 3, E - 9])] = torch.tensor([40.0, -60.0, 80.0, -100.0])
    return model.to(dev), E, heads


@pytest.mark.parametrize("shape", ["c1", "c2", "c3"])
def test_block_vs_precision_faithful_fp64(cuda_dev, shape):
    arch, B, res, N, heads = R.PROD[shape]
    model, E, _ = _sharp_block_model(arch, cuda_dev)
    torch.manual_seed(30)
    img = torch.randn(B, 3, res, res, device=cuda_dev)
    twin = copy.deepcopy(model)
    _zero_blocks(twin)
    x0, _ = twin.forward_tokens(img)  # the embed output (pinned by test_embed_stage_fp64)
    del twin
    prm = {k: v.detach() for k, v in R.block_params(dict(model.state_dict()), 0).items()}
    # scale the q and k rows so the per-head logits have std 6
    _, qkv0 = R.block_ref(x0[:N], prm, 1, N, heads, rnd=False)
    f = (6.0 / R.logit_std(qkv0, 1, N, heads)) ** 0.5
    with torch.no_grad():
        model.blocks[0].attn.qkv.weight[:2 * E] *= f
        model.blocks[0].attn.qkv.bias[:2 * E] *= f
    prm = {k: v.detach() for k, v in R.block_params(dict(model.state_dict()), 0).items()}
    x1, qkv = model.forward_tokens(img, want_qkv=True)
    torch.cuda.synchronize()
    ref_x, ref_qkv = R.block_ref(x0, prm, B, N, heads, rnd=True)
    std = R.logit_std(ref_qkv, B, N, heads, max_images=1)
    d_got, d_ref = x1.double() - x0.double(), ref_x - x0.double()
    r_x = R.rel_l2(d_got, d_ref)
    r_qkv = R.rel_l2(qkv, ref_qkv)
    del ref_x, ref_qkv
    exact_x, exact_qkv = R.block_ref(x0, prm, B, N, heads, rnd=False)
    r_x_exact = R.rel_l2(d_got, exact_x - x0.double())
    r_qkv_exact = R.rel_l2(qkv, exact_qkv)
    m = dict(logit_std=std, rel_l2_block_delta=r_x, rel_l2_qkv=r_qkv, bar=BLOCK_REL_L2, qkv_bar=QKV_REL_L2,
             rel_l2_block_delta_vs_exact=r_x_exact, rel_l2_qkv_vs_exact=r_qkv_exact)
    record(f"vit_fp64_block_{shape}", m)
    assert 4.5 < std < 8.0, m
    assert r_x < BLOCK_REL_L2 and r_qkv < QKV_REL_L2, m
    del exact_x, exact_qkv
    torch.cuda.empty_cache()


# ================================================================================================
# 5. graph replay, patch 16, KK
# ================================================================================================
def _random_vit_small(dev, p=8):
    import stego_oracle as O
    from stego_b200.dino.vision_transformer import vit_small
    sd = O.perturb_vit_state(O.vit_random_state("vit_small", p, seed=3))
    model = vit_small(patch_size=p)
    model.load_state_dict(sd)
    return model.to(dev).eval(), sd


def test_graph_replay_equals_eager(cuda_dev):
    model, _ = _random_vit_small(cuda_dev)
    g = torch.Generator(device=cuda_dev).manual_seed(40)
    for (H, W) in [(96, 96), (64, 96), (96, 96)]:  # the last one replays the first graph after another was captured
        for _ in range(2):  # a second replay with new data
            img = torch.randn(2, 3, H, W, generator=g, device=cuda_dev)
            img_pos = torch.randn(2, 3, H, W, generator=g, device=cuda_dev)
            got = model.patch_features([img, img_pos], use_graph=True).clone()
            want = model.patch_features(torch.cat([img, img_pos]))
            assert torch.equal(got, want), (H, W)
    assert len(model._cache["graphs"]) == 2


@pytest.mark.parametrize("H,W", [(224, 224), (224, 320)])
def test_featurizer_patch16_vs_oracle(cuda_dev, H, W):
    import stego_oracle as O
    from stego_b200.config import make_cfg
    from stego_b200.modules import DinoFeaturizer
    fp32_strict()
    cfg = make_cfg(dino_patch_size=16, random_backbone_init=True)
    torch.manual_seed(0)
    net = DinoFeaturizer(70, cfg).to(cuda_dev).eval()
    sd = O.perturb_vit_state(O.vit_random_state("vit_small", 16, seed=3))
    net.model.load_state_dict(sd)
    img = torch.randn(2, 3, H, W, generator=torch.Generator().manual_seed(41)).to(cuda_dev)
    with torch.no_grad():
        feat, _ = net(img)
        want = O.vit_image_feat({k: v.to(cuda_dev) for k, v in sd.items()}, img, "vit_small", 16)
    assert feat.shape == want.shape == (2, 384, H // 16, W // 16)
    r = rel(feat, want)
    record(f"vit_fp64_patch16_{H}x{W}", dict(rel_l2=r))
    assert r < 1e-2, r


def test_featurizer_kk_nonsquare(cuda_dev):
    """dino_feat_type "KK": the last block's keys (heads concatenated) at a non-square image vs the fp64 backbone."""
    from stego_b200.config import make_cfg
    from stego_b200.modules import DinoFeaturizer
    import stego_oracle as O
    cfg = make_cfg(dino_feat_type="KK", random_backbone_init=True)
    torch.manual_seed(0)
    net = DinoFeaturizer(70, cfg).to(cuda_dev).eval()
    sd = O.perturb_vit_state(O.vit_random_state("vit_small", 8, seed=3))
    net.model.load_state_dict(sd)
    B, H, W = 2, 64, 96
    img = torch.randn(B, 3, H, W, generator=torch.Generator().manual_seed(42)).to(cuda_dev)
    with torch.no_grad():
        feat, _ = net(img)
        _, qkv = R.vit_tokens({k: v.to(cuda_dev).double() for k, v in sd.items()}, img.double(), "vit_small", 8)
    N = (H // 8) * (W // 8) + 1
    keys = qkv.view(B, N, 3, 384)[:, 1:, 1].reshape(B, H // 8, W // 8, 384).permute(0, 3, 1, 2)
    assert feat.shape == keys.shape
    r = rel(feat, keys)
    record("vit_fp64_kk_64x96", dict(rel_l2=r))
    assert r < 1e-2, r
