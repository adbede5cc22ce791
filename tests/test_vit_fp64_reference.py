"""CPU: the fp64 backbone references of tests/_vit_fp64.py against the oracle, and the attention input regimes
against what they claim to construct (the GPU tests' power rests on both)."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _vit_fp64 as R  # noqa: E402
import stego_oracle as O  # noqa: E402


def _sd64(arch, patch=8):
    return {k: v.double() for k, v in O.perturb_vit_state(O.vit_random_state(arch, patch, seed=3)).items()}


def test_vit_tokens_match_oracle_fp64():
    """With rounding off, 12 x block_ref + embed_ref + final norm is oracle.vit_forward (itself pinned to the
    reference by test_vit_tokens_golden), in fp64, at a non-square interpolated shape."""
    sd = _sd64("vit_small")
    torch.manual_seed(11)
    img = torch.randn(2, 3, 32, 48, dtype=torch.float64)
    with torch.no_grad():
        tok, qkv = R.vit_tokens(sd, img, "vit_small", 8)
        want = O.vit_forward(sd, img, "vit_small", 8)
    assert tok.shape == want.shape == (2, 25, 384) and qkv.shape == (50, 3 * 384)
    assert (tok - want).abs().max().item() < 1e-12


def test_block_rounding_points():
    """rnd=True stores qkv in bf16 and the residual in fp32 and stays within bf16 accuracy of the exact block."""
    sd = _sd64("vit_small")
    prm = R.block_params(sd, 0)
    torch.manual_seed(12)
    B, N = 2, 40
    x = torch.randn(B * N, 384, dtype=torch.float64)
    x_r, qkv_r = R.block_ref(x, prm, B, N, 6, rnd=True)
    x_e, qkv_e = R.block_ref(x, prm, B, N, 6, rnd=False)
    assert torch.equal(qkv_r, R.bf16(qkv_r)) and torch.equal(x_r, R.f32(x_r))
    d_r, d_e = x_r - R.f32(x), x_e - x
    assert 1e-5 < R.rel_l2(d_r, d_e) < 2e-2
    assert 1e-5 < R.rel_l2(qkv_r, qkv_e) < 1e-2


def test_attention_ref_chunking():
    torch.manual_seed(13)
    B, N, heads = 3, 70, 2
    qkv = torch.randn(B * N, 3 * heads * 64).bfloat16()
    whole = R.attention_ref(qkv, B, N, heads)
    chunked = R.attention_ref(qkv, B, N, heads, max_bytes=1)
    q, k, v = qkv.double().view(B, N, 3, heads, 64).permute(2, 0, 3, 1, 4)
    direct = ((q @ k.transpose(-2, -1)) / 8).softmax(-1) @ v
    assert torch.equal(whole, chunked)
    assert (whole - direct.transpose(1, 2).reshape(B * N, -1)).abs().max().item() < 1e-14


def test_bf16_ulp():
    t = torch.tensor([1.0, 1.5, 0.75, -3.0, 0.0, 256.0], dtype=torch.float64)
    assert R.bf16_ulp(t).tolist() == [2.0 ** -7, 2.0 ** -7, 2.0 ** -8, 2.0 ** -6, 2.0 ** -133, 2.0]


@pytest.mark.parametrize("N", [1, 2, 64, 65, 129, 193])
def test_attention_regimes(N):
    """Each input regime has the property the GPU test relies on, including at the ragged sizes."""
    B, heads = 3, 2
    mk = lambda r: R.attention_inputs(r, B, N, heads, seed=5)
    s = lambda qkv: R.scaled_logits(qkv, B, N, heads)
    if N >= 64:
        assert 0.1 < s(mk("uniform")).std(-1).mean().item() < 0.2
        assert 5.0 < s(mk("sharp")).std(-1).mean().item() < 7.0
    qkv = mk("onehot")
    lg = s(qkv)
    tg = torch.tensor(R.onehot_targets(N))
    want = tg[torch.arange(N) % len(tg)]
    assert torch.equal(lg.argmax(-1), want.view(1, 1, N).expand(B, heads, N))
    assert (lg.softmax(-1).amax(-1) > 1 - 1e-12).all()
    qkv = mk("allneg")
    assert s(qkv).max().item() < -30.0
    v = qkv.double().view(B, N, 3, -1)[:, :, 2]
    assert ((v - 1).abs() < 0.1).all()
    lg = s(mk("rising"))
    ntile = (N + 63) // 64
    if ntile > 1:
        tmax = torch.stack([lg[..., 64 * t:64 * (t + 1)].amax(-1) for t in range(ntile)], -1)
        steps = tmax[..., 1:] - tmax[..., :-1]
        assert (steps > 0.25).all()
        if ntile > 2:
            assert (steps.amax(-1) - steps.amin(-1) > 4.0).all()  # unequal steps: a per-tile factor cannot cancel
    qkv = mk("crossimage")
    q, k, _ = qkv.double().view(B, N, 3, heads, 64).permute(2, 0, 3, 1, 4)
    for b in range(B - 1):
        own = (q[b] @ k[b].transpose(-2, -1)).amax(-1) / 8
        nxt = (q[b] @ k[b + 1, :, :64].transpose(-2, -1)).amax(-1) / 8
        assert (nxt - own > 10.0).all()
    v = mk("headtag").double().view(B, N, 3, heads, 64)[:, :, 2]
    for h in range(heads):
        assert abs(v[:, :, h].mean().item() - 4.0 * h) < 0.5
