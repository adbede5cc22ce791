"""The attention-matrix kernel (stego_attention_probs) against float64 softmax of the same bf16 qkv at the production
shapes, its guard bands and determinism, its consistency with the fused attention, and the ViT / DinoFeaturizer entry
points built on it (get_last_selfattention, get_intermediate_feat / get_intermediate_layers for any n,
DinoFeaturizer.forward(img, n)) against the fp32 oracle.

Elementwise bar of the kernel.  Write the computed exponent of key j (log2 units) as t_j = (s_j - m) c with
c = log2(e) / 8, s_j = q.k_j and m the row maximum; P_j = 2^t_j / l.  Sources of error, u = 2^-24:
  * scores: q.k over 64 exact bf16 x bf16 products summed in fp32 by the tensor cores (not necessarily round to
    nearest, so 2u per addition): |ds_j| <= 128 u |q| |k_j|.  A shift common to all keys cancels in P, so the
    relative error of P_i is at most 2 max_j |ds_j| c ln 2 (softmax: dP_i / P_i = dz_i - sum_j P_j dz_j).
  * exponent: (s_j - m) rounded, times c (itself rounded): |dt_j| <= 3u |t_j|; the relative error of P_i from these
    is ln 2 (3u |t_i| + 3u sum_j P_j |t_j|).
  * ex2.approx: 2 ulp (2^-22) relative, once in P_i's numerator and once (weighted) in l.
  * l: per-thread fp32 partial sums over N/4 keys, two shuffle additions and, per key tile, one rescale by
    ex2((m_old - m_new) c): (N/4 + 4 + 3 T) u + T 2^-22 + 3u ln 2 R, with T key tiles and R the log2 rise of the row
    maximum after the first tile.
  * 1 / l and the product: 2u.
  * exponents below -126 flush to 0 (ftz): 2^-125 absolute.
so |P_i - P_ref,i| <= P_ref,i eps_i + 2^-125.  The row sums of P do not see the score error (it cancels in the
normalisation): |sum_i P_i - 1| <= (N/4 + 4 + 3 T) u + (T + 2) 2^-22 + ln 2 (6u sum_j P_j |t_j| + 3u R) + 2u.
The measured error / bar ratios are written to $STEGO_PARITY_DIR when it is set.
"""
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _vit_fp64 as R  # noqa: E402
from _parity_util import fp32_strict, record, rel  # noqa: E402

pytestmark = pytest.mark.gpu

U = R.FP32_U
EX2 = 2.0 ** -22
LOG2E = 1.0 / math.log(2.0)
LN2 = math.log(2.0)
SENTINEL = 0x7FA0DEAD  # a signalling-NaN bit pattern: the kernel writes finite values only
GUARD = 1024


def _guarded_probs(B, heads, N, dev):
    """fp32 output [B, heads, N, N] inside a buffer whose every float (output included) holds the sentinel."""
    n = B * heads * N * N
    buf = torch.empty(n + 2 * GUARD, dtype=torch.float32, device=dev)
    buf.view(torch.int32).fill_(SENTINEL)
    return buf, buf[GUARD:GUARD + n].view(B, heads, N, N)


def _guards_intact(buf):
    return bool((buf[:GUARD].view(torch.int32) == SENTINEL).all() and (buf[-GUARD:].view(torch.int32) == SENTINEL).all())


def _bits_checksum(P, chunk=1 << 27):
    """sum_i bits_i (i mod 65521 + 1) in int64, over chunks (no full-size temporary)."""
    flat = P.view(-1).view(torch.int32)
    total = 0
    for c0 in range(0, flat.numel(), chunk):
        part = flat[c0:c0 + chunk].to(torch.int64)
        w = torch.arange(c0, c0 + part.numel(), device=P.device, dtype=torch.int64) % 65521 + 1
        total += int((part * w).sum().item())
    return total


def _qk(qkv, B, N, heads, b):
    x = qkv.view(B, N, 3, heads, R.HEAD_DIM)[b]
    return x[:, 0].permute(1, 0, 2).double(), x[:, 1].permute(1, 0, 2).double()  # [heads, N, 64]


def _check_rows(P, qkv, B, N, heads, b, rows):
    """Max error / bar and max |row sum - 1| / bar over `rows` of image b (fp64, chunked by the caller's choice)."""
    q, k = _qk(qkv, B, N, heads, b)
    q = q[:, rows]
    s = q @ k.transpose(-2, -1)                                  # [heads, R, N] raw scores
    m = s.amax(-1, keepdim=True)
    t = (s - m) * (LOG2E / 8)                                    # log2 units, <= 0
    ref = torch.exp2(t)
    ref /= ref.sum(-1, keepdim=True)
    T = (N + R.KEY_TILE - 1) // R.KEY_TILE
    tbar = (ref * t.abs()).sum(-1, keepdim=True)
    rise = (m - s[..., :R.KEY_TILE].amax(-1, keepdim=True)) * (LOG2E / 8)
    kmax = k.norm(dim=-1).amax(-1).view(heads, 1, 1)
    es = 128 * U * q.norm(dim=-1, keepdim=True) * kmax * (LOG2E / 8)
    lsum = (N / 4 + 4 + 3 * T) * U + T * EX2 + 3 * U * LN2 * rise
    eps = LN2 * (2 * es + 3 * U * (t.abs() + tbar)) + 2 * EX2 + lsum + 2 * U
    got = P[b][:, rows].double()
    ratio = ((got - ref).abs() / (ref * eps + 2.0 ** -125)).max().item()
    sbar = (N / 4 + 4 + 3 * T) * U + (T + 2) * EX2 + LN2 * (6 * U * tbar + 3 * U * rise) + 2 * U
    sratio = ((got.sum(-1, keepdim=True) - 1).abs() / sbar).max().item()
    return ratio, sratio


def _check_probs(dev, B, N, heads, regime, seed, stride=None, repeat_exact=True):
    """Launch into a guarded buffer; check guards, that every element was written and finite, determinism, and every
    row of the first and last image (and every `stride`-th row of the others) against fp64."""
    from stego_b200 import ops
    E = heads * 64
    qkv = R.attention_inputs(regime, B, N, heads, seed=seed, device=dev)
    buf, P = _guarded_probs(B, heads, N, dev)
    ops.attention_probs(qkv, P, B, N, E, heads)
    torch.cuda.synchronize()
    assert _guards_intact(buf), (regime, "wrote outside the output")
    assert bool(torch.isfinite(P).all()), (regime, "unwritten or non-finite elements")
    if repeat_exact:
        again = torch.empty_like(P)
        ops.attention_probs(qkv, again, B, N, E, heads)
        assert torch.equal(P.view(torch.int32), again.view(torch.int32)), (regime, "launches differ")
        del again
    else:  # the c3 output is 15 GB: compare a position-weighted checksum of the bits of a second launch
        c0 = _bits_checksum(P)
        ops.attention_probs(qkv, P, B, N, E, heads)
        assert _bits_checksum(P) == c0, (regime, "launches differ")
    worst, worst_sum = 0.0, 0.0
    rows_per_chunk = max(1, (1 << 27) // (heads * N))  # ~1 GB of fp64 scores per chunk
    for b in range(B):
        if b in (0, B - 1) or stride is None:
            rows = torch.arange(N, device=dev)
        else:
            rows = torch.arange(b % stride, N, stride, device=dev)
        for r0 in range(0, rows.numel(), rows_per_chunk):
            a, s_ = _check_rows(P, qkv, B, N, heads, b, rows[r0:r0 + rows_per_chunk])
            worst, worst_sum = max(worst, a), max(worst_sum, s_)
    del P, buf, qkv
    return worst, worst_sum


def _probs_case(dev, tag, B, N, heads, regimes, stride=None, repeat_exact=True):
    res = {}
    for i, regime in enumerate(regimes):
        a, s_ = _check_probs(dev, B, N, heads, regime, seed=200 + i, stride=stride, repeat_exact=repeat_exact)
        res[regime] = dict(max_err_over_bar=a, max_rowsum_err_over_bar=s_)
    record(f"attention_probs_{tag}", dict(B=B, N=N, heads=heads, elements=B * heads * N * N, regimes=res))
    for regime, m in res.items():
        assert m["max_err_over_bar"] <= 1.0 and m["max_rowsum_err_over_bar"] <= 1.0, (tag, regime, m)


# ================================================================================================
# 1. kernel vs fp64 at the production batches and ragged sizes; 2. guard bands, row sums, determinism
# ================================================================================================
@pytest.mark.parametrize("shape", ["c1", "c2", "c3"])
def test_probs_production_shapes(cuda_dev, shape):
    """The 2B batches of c1 / c2 / c3; at c3 the output has 32 x 12 x 3137^2 = 3.78e9 > 2^31 elements (15 GB)."""
    _, B, _, N, heads = R.PROD[shape]
    regimes = R.REGIMES if shape == "c1" else ("uniform", "sharp", "onehot", "rising")
    if shape == "c3":
        assert B * heads * N * N > 2 ** 31
    _probs_case(cuda_dev, shape, B, N, heads, regimes, stride=97, repeat_exact=shape != "c3")
    torch.cuda.empty_cache()


@pytest.mark.parametrize("heads", [1, 6, 12])
@pytest.mark.parametrize("N", [1, 2, 63, 64, 65, 127, 128, 129, 191, 192, 193, 257])
def test_probs_ragged(cuda_dev, N, heads):
    _probs_case(cuda_dev, f"ragged_N{N}_h{heads}", 3, N, heads, R.REGIMES)


@pytest.mark.parametrize("N", [65, 785])
def test_probs_exact_onehot(cuda_dev, N):
    """Each query's target key scores 128 above every other key (channel value 32 in q and k): every other exponent
    is below -126 and flushes to 0, the target's is exactly 0, so each row of P is exactly one-hot."""
    from stego_b200 import ops
    import torch.nn.functional as F
    B, heads = 2, 6
    g = torch.Generator(device=cuda_dev).manual_seed(7)
    shp = (B, N, heads, 64)
    q, k, v = (0.3 * torch.randn(*shp, generator=g, device=cuda_dev) for _ in range(3))
    tgt = torch.tensor(R.onehot_targets(N), device=cuda_dev)
    rows = torch.arange(N, device=cuda_dev)
    k[:, tgt, :, torch.arange(len(tgt), device=cuda_dev)] = 32.0
    q[:, rows, :, rows % len(tgt)] = 32.0
    qkv = torch.stack((q, k, v), 2).reshape(B * N, 3 * heads * 64).to(torch.bfloat16).contiguous()
    P = torch.empty(B, heads, N, N, device=cuda_dev)
    ops.attention_probs(qkv, P, B, N, heads * 64, heads)
    want = F.one_hot(tgt[rows % len(tgt)], N).float().view(1, 1, N, N).expand(B, heads, N, N)
    assert torch.equal(P, want)


# ================================================================================================
# 3. consistency with the fused attention
# ================================================================================================
@pytest.mark.parametrize("B,N,heads", [(8, 785, 6), (3, 129, 12)])
def test_probs_times_v_matches_fused_attention(cuda_dev, B, N, heads):
    """fp64(P) @ v against ops.attention's output, with the elementwise bar of the fused-attention test
    (2^-8 (|ref| + max_j |v_j|): the fused kernel rounds P to bf16 and its output to bf16)."""
    from stego_b200 import ops
    E = heads * 64
    worst = {}
    for i, regime in enumerate(("uniform", "sharp", "rising")):
        qkv = R.attention_inputs(regime, B, N, heads, seed=300 + i, device=cuda_dev)
        P = torch.empty(B, heads, N, N, device=cuda_dev)
        ops.attention_probs(qkv, P, B, N, E, heads)
        out = torch.empty(B * N, E, dtype=torch.bfloat16, device=cuda_dev)
        ops.attention(qkv, out, B, N, E, heads)
        v = qkv.view(B, N, 3, heads, 64)[:, :, 2].permute(0, 2, 1, 3).double()   # [B, heads, N, 64]
        pv = (P.double() @ v).permute(0, 2, 1, 3).reshape(B, N, E)
        vmax = v.abs().amax(2).reshape(B, 1, E)
        worst[regime] = ((out.double().view(B, N, E) - pv).abs() / (R.BF16_U * (pv.abs() + vmax))).max().item()
    record(f"attention_probs_pv_B{B}_N{N}_h{heads}", worst)
    assert max(worst.values()) <= 1.0, worst


# ================================================================================================
# 4. model level against the fp32 oracle; 5. regressions
# ================================================================================================
MODELS = {"vit_small8_224": ("vit_small", 8, 224, 224), "vit_base16_224x320": ("vit_base", 16, 224, 320)}


def _model(arch, patch, dev):
    import stego_oracle as O
    from stego_b200.dino import vision_transformer as V
    sd = O.perturb_vit_state(O.vit_random_state(arch, patch, seed=3))
    model = getattr(V, arch)(patch_size=patch)
    model.load_state_dict(sd)
    return model.to(dev).eval(), {k: v.to(dev) for k, v in sd.items()}


def _logit_err(qkv_a, qkv_b):
    """Per-row max over keys of |z_a - z_b|, z = q.k / 8 in fp64, from two [3, B, heads, N, 64] qkv tensors."""
    za = qkv_a[0].double() @ qkv_a[1].double().transpose(-2, -1) / 8
    zb = qkv_b[0].double() @ qkv_b[1].double().transpose(-2, -1) / 8
    return (za - zb).abs().amax(-1)


def _map_ratio(P, P_ref, dz):
    """Row L1 distance of the maps over its bar.  ||softmax(z) - softmax(z')||_1 <= 2 ||z - z'||_inf (the softmax
    Jacobian diag(P) - P P^T has induced 1-norm <= 2 along the segment), so the bf16 backbone's maps may differ from
    the oracle's by at most twice the logit error its qkv carries; the kernel's own error (above) adds N 1e-5."""
    N = P.shape[-1]
    l1 = (P.double() - P_ref.double()).abs().sum(-1)
    return (l1 / (2 * dz + N * 1e-5)).max().item()


@pytest.mark.parametrize("name", list(MODELS))
def test_vit_maps_vs_oracle(cuda_dev, name):
    import vit_maps_oracle as VM
    fp32_strict()
    arch, patch, H, W = MODELS[name]
    model, sd = _model(arch, patch, cuda_dev)
    B = 2
    img = torch.randn(B, 3, H, W, generator=torch.Generator().manual_seed(43)).to(cuda_dev)
    depth = len(model.blocks)
    with torch.no_grad():
        ofeat, oattn, oqkv = VM.vit_intermediate(sd, img, arch, patch, n=depth)
        res = {}
        last = model.get_last_selfattention(img)
        for n in (1, 2, 12):
            feat, attn, qkv = model.get_intermediate_feat(img, n=n)
            assert len(feat) == len(attn) == len(qkv) == min(n, depth)
            if n == 1:  # the same qkv through the same kernel
                assert torch.equal(last, attn[0])
            for j, (f, a, q) in enumerate(zip(feat, attn, qkv)):
                blk = depth - len(feat) + j
                assert f.shape == ofeat[blk].shape and a.shape == oattn[blk].shape and q.shape == oqkv[blk].shape
                assert f.dtype == a.dtype == q.dtype == torch.float32
                r = dict(feat=rel(f, ofeat[blk]), qkv=rel(q, oqkv[blk]), attn=rel(a, oattn[blk]),
                         attn_l1_over_bar=_map_ratio(a, oattn[blk], _logit_err(q, oqkv[blk])))
                res[f"n{n}_block{blk}"] = r
                assert r["feat"] < 1e-2 and r["qkv"] < 1e-2 and r["attn_l1_over_bar"] <= 1.0, (n, blk, r)
        layers = model.get_intermediate_layers(img, n=3)
        assert len(layers) == 3
        for j, f in enumerate(layers):
            res[f"layers3_{j}"] = rel(f, ofeat[depth - 3 + j])
            assert res[f"layers3_{j}"] < 1e-2
        assert model.get_intermediate_feat(img, n=0) == ([], [], []) and model.get_intermediate_layers(img, n=0) == []
    record(f"vit_maps_{name}", res)


@pytest.mark.parametrize("name", list(MODELS))
def test_featurizer_n2_vs_oracle(cuda_dev, name):
    """DinoFeaturizer.forward(img, n=2) reads block depth - 2 for "feat", "KK" and the class feature (modules.py:90-106)."""
    import vit_maps_oracle as VM
    from stego_b200.config import make_cfg
    from stego_b200.modules import DinoFeaturizer
    fp32_strict()
    arch, patch, H, W = MODELS[name]
    _, sd = _model(arch, patch, cuda_dev)
    B, fh, fw = 2, H // patch, W // patch
    img = torch.randn(B, 3, H, W, generator=torch.Generator().manual_seed(44)).to(cuda_dev)
    with torch.no_grad():
        ofeat, _, oqkv = VM.vit_intermediate(sd, img, arch, patch, n=2)
    want = {"feat": ofeat[0][:, 1:].reshape(B, fh, fw, -1).permute(0, 3, 1, 2),
            "KK": oqkv[0][1][:, :, 1:].permute(0, 1, 3, 2).reshape(B, -1, fh, fw),
            "class": ofeat[0][:, :1].reshape(B, 1, 1, -1).permute(0, 3, 1, 2)}
    res = {}
    for feat_type in ("feat", "KK"):
        cfg = make_cfg(model_type=arch, dino_patch_size=patch, dino_feat_type=feat_type, random_backbone_init=True)
        torch.manual_seed(0)
        net = DinoFeaturizer(70, cfg).to(cuda_dev).eval()
        net.model.load_state_dict({k: v.cpu() for k, v in sd.items()})
        with torch.no_grad():
            got, _ = net(img, n=2)
            last, _ = net(img)
            if feat_type == "feat":
                cls = net(img, n=2, return_class_feat=True)
                res["class"] = rel(cls, want["class"])
                assert cls.shape == want["class"].shape
        assert got.shape == want[feat_type].shape
        res[feat_type] = rel(got, want[feat_type])
        res[feat_type + "_vs_last_block"] = rel(last, want[feat_type])
    record(f"featurizer_n2_{name}", res)
    assert res["feat"] < 1e-2 and res["KK"] < 1e-2 and res["class"] < 1e-2, res
    # n = 2 reads block depth - 2, not the last block (whose features are much further from that block's)
    assert res["feat_vs_last_block"] > 5 * res["feat"] and res["KK_vs_last_block"] > 5 * res["KK"], res


def test_n1_bit_identical_to_last_block_paths(cuda_dev):
    """get_intermediate_feat(x, 1) feat / qkv are the bits of the last-block computation (_all_tokens); the featurizer's
    default call is the bits of patch_features ("feat") and of the last block's keys ("KK")."""
    from stego_b200.config import make_cfg
    from stego_b200.modules import DinoFeaturizer
    model, sd = _model("vit_small", 8, cuda_dev)
    B, H, W = 2, 64, 96
    img = torch.randn(B, 3, H, W, generator=torch.Generator().manual_seed(45)).to(cuda_dev)
    with torch.no_grad():
        feat, attn, qkv = model.get_intermediate_feat(img, n=1)
        tok, qkv_last = model._all_tokens(img, want_qkv=True)
        N = tok.shape[1]
        assert torch.equal(feat[0], tok.float())
        assert torch.equal(qkv[0], qkv_last.view(B, N, 3, 6, 64).permute(2, 0, 3, 1, 4).float())
        assert attn[0].shape == (B, 6, N, N)
        for feat_type in ("feat", "KK"):
            cfg = make_cfg(dino_feat_type=feat_type, random_backbone_init=True)
            torch.manual_seed(0)
            net = DinoFeaturizer(70, cfg).to(cuda_dev).eval()
            net.model.load_state_dict({k: v.cpu() for k, v in sd.items()})
            got, _ = net(img)
            if feat_type == "feat":
                want = net.model.patch_features(img).float().view(B, H // 8, W // 8, -1).permute(0, 3, 1, 2)
            else:
                k = qkv[0][1, :, :, 1:, :]
                want = k.permute(0, 2, 1, 3).reshape(B, -1, 384).to(torch.bfloat16).float()
                want = want.view(B, H // 8, W // 8, -1).permute(0, 3, 1, 2)
            assert torch.equal(got, want), feat_type
