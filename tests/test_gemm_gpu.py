"""wgmma GEMM (stego_gemm_bf16) against a plain PyTorch fp32 reference on bf16-rounded operands."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _ref(a, b, bias=None, act=0, residual=None):
    y = a.float() @ b.float().t()
    if bias is not None:
        y = y + bias
    if act == 1:
        y = torch.nn.functional.gelu(y)
    elif act == 2:
        y = torch.relu(y)
    if residual is not None:
        y = y + residual
    return y


def _rel(x, y):
    return ((x.float() - y.float()).norm() / y.float().norm().clamp_min(1e-12)).item()


@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (300, 384, 192), (1000, 1152, 384), (785 * 2, 1536, 384),
                                   (257, 768, 3072)])
def test_gemm_tn_bias_bf16(cuda_dev, M, N, K):
    from stego_b200 import ops
    torch.manual_seed(0)
    a = torch.randn(M, K, device=cuda_dev).bfloat16()
    b = (torch.randn(N, K, device=cuda_dev) / K ** 0.5).bfloat16()
    bias = torch.randn(N, device=cuda_dev)
    out = torch.empty(M, N, device=cuda_dev, dtype=torch.bfloat16)
    ops.gemm(a, b, out, M=M, N=N, K=K, bias=bias)
    assert _rel(out, _ref(a, b, bias)) < 4e-3
    out32 = torch.empty(M, N, device=cuda_dev)
    ops.gemm(a, b, out32, M=M, N=N, K=K, bias=bias, act=ops.ACT_GELU)
    assert _rel(out32, _ref(a, b, bias, 1)) < 1e-5


def test_gemm_inplace_residual_and_relu(cuda_dev):
    from stego_b200 import ops
    torch.manual_seed(1)
    M, N, K = 900, 384, 1536
    a = torch.randn(M, K, device=cuda_dev).bfloat16()
    b = (torch.randn(N, K, device=cuda_dev) / K ** 0.5).bfloat16()
    bias = torch.randn(N, device=cuda_dev)
    x = torch.randn(M, N, device=cuda_dev)
    want = _ref(a, b, bias, 0, x)
    ops.gemm(a, b, x, M=M, N=N, K=K, bias=bias, residual=x)
    assert _rel(x, want) < 1e-5
    h = torch.empty(M, N, device=cuda_dev, dtype=torch.bfloat16)
    ops.gemm(a, b, h, M=M, N=N, K=K, bias=bias, act=ops.ACT_RELU)
    assert _rel(h, _ref(a, b, bias, 2)) < 4e-3


def test_gemm_ragged_n70(cuda_dev):
    from stego_b200 import ops
    torch.manual_seed(2)
    M, N, K = 1570, 70, 384
    a = torch.randn(M, K, device=cuda_dev).bfloat16()
    w = torch.zeros(128, K, device=cuda_dev, dtype=torch.bfloat16)
    w[:N] = (torch.randn(N, K, device=cuda_dev) / K ** 0.5).bfloat16()
    bias = torch.randn(N, device=cuda_dev)
    store = torch.full((M, 72), 7.0, device=cuda_dev)
    ops.gemm(a, w, store, M=M, N=N, K=K, bias=bias)
    assert _rel(store[:, :N], _ref(a, w[:N], bias)) < 1e-5
    assert torch.all(store[:, N:] == 7.0)  # padding columns untouched


def test_gemm_b_mn_major_dgrad(cuda_dev):
    from stego_b200 import ops
    torch.manual_seed(3)
    M, N, K = 700, 384, 128
    a = torch.randn(M, K, device=cuda_dev).bfloat16()
    bt = (torch.randn(K, N, device=cuda_dev) / K ** 0.5).bfloat16()  # stored [K][N]
    out = torch.empty(M, N, device=cuda_dev)
    ops.gemm(a, bt, out, M=M, N=N, K=K, b_mn=True)
    assert _rel(out, a.float() @ bt.float()) < 1e-5


def test_gemm_a_mn_major(cuda_dev):
    from stego_b200 import ops
    torch.manual_seed(4)
    M, N, K = 256, 384, 320
    at = torch.randn(K, M, device=cuda_dev).bfloat16()  # stored [K][M]
    b = (torch.randn(N, K, device=cuda_dev) / K ** 0.5).bfloat16()
    out = torch.empty(M, N, device=cuda_dev)
    ops.gemm(at, b, out, M=M, N=N, K=K, a_mn=True)
    assert _rel(out, at.float().t() @ b.float().t()) < 1e-5


@pytest.mark.parametrize("splits", [1, 7, 64])
def test_gemm_wgrad_splitk(cuda_dev, splits):
    from stego_b200 import ops
    torch.manual_seed(5)
    rows, n_out, k_in = 6400, 70, 384  # dW[n_out,k_in] = dY^T X
    dy = torch.zeros(rows, 128, device=cuda_dev, dtype=torch.bfloat16)
    dy[:, :n_out] = torch.randn(rows, n_out, device=cuda_dev).bfloat16()
    x = torch.randn(rows, k_in, device=cuda_dev).bfloat16()
    dw = torch.zeros(n_out, k_in, device=cuda_dev)
    ops.gemm(dy, x, dw, M=n_out, N=k_in, K=rows, a_mn=True, b_mn=True, splits=splits, atomic=True)
    want = dy[:, :n_out].float().t() @ x.float()
    assert _rel(dw, want) < 1e-5


def test_gemm_patch_embed_rows(cuda_dev):
    from stego_b200 import ops
    torch.manual_seed(6)
    B, hw, E, K = 3, 49, 384, 192
    a = torch.randn(B * hw, K, device=cuda_dev).bfloat16()
    w = (torch.randn(E, K, device=cuda_dev) / K ** 0.5).bfloat16()
    bias = torch.randn(E, device=cuda_dev)
    pos = torch.randn(hw + 1, E, device=cuda_dev)
    x = torch.zeros(B * (hw + 1), E, device=cuda_dev)
    ops.gemm(a, w, x, M=B * hw, N=E, K=K, bias=bias, residual=pos, row_div=hw)
    want = (_ref(a, w, bias).view(B, hw, E) + pos[1:]).reshape(B * hw, E)
    got = x.view(B, hw + 1, E)[:, 1:].reshape(B * hw, E)
    assert _rel(got, want) < 1e-5
    assert torch.all(x.view(B, hw + 1, E)[:, 0] == 0)


def test_gemm_bad_args_raise(cuda_dev):
    from stego_b200 import ops
    a = torch.zeros(128, 100, device=cuda_dev, dtype=torch.bfloat16)
    b = torch.zeros(128, 100, device=cuda_dev, dtype=torch.bfloat16)
    out = torch.zeros(128, 128, device=cuda_dev)
    with pytest.raises(RuntimeError):
        ops.gemm(a, b, out, M=128, N=128, K=100)


@pytest.mark.parametrize("mode", ["residual_other", "bf16_out_residual", "atomic", "bias_misaligned"])
def test_gemm_n1152_without_tma_epilogue(cuda_dev, mode):
    """N = 1152 (the ViT-B qkv width) is nine 128x128 column tiles; every epilogue variant that bypasses the TMA
    store (residual != out, bf16 output + residual, atomic output, misaligned bias) must write exactly the N columns
    through the register epilogue."""
    from stego_b200 import ops
    torch.manual_seed(11)
    M, N, K = 300, 1152, 384
    a = torch.randn(M, K, device=cuda_dev).bfloat16()
    w = (torch.randn(N, K, device=cuda_dev) / K ** 0.5).bfloat16()
    ref = a.float() @ w.float().t()
    if mode == "residual_other":
        r = torch.randn(M, N, device=cuda_dev)
        out = torch.empty(M, N, device=cuda_dev)
        ops.gemm(a, w, out, M=M, N=N, K=K, residual=r)
        assert _rel(out, ref + r) < 1e-5
    elif mode == "bf16_out_residual":
        r = torch.randn(M, N, device=cuda_dev)
        out = torch.empty(M, N, device=cuda_dev, dtype=torch.bfloat16)
        ops.gemm(a, w, out, M=M, N=N, K=K, residual=r)
        assert _rel(out, ref + r) < 4e-3
    elif mode == "atomic":
        out = torch.zeros(M, N, device=cuda_dev)
        ops.gemm(a, w, out, M=M, N=N, K=K, splits=1, atomic=True)
        assert _rel(out, ref) < 1e-5
    else:
        bias_store = torch.randn(N + 1, device=cuda_dev)
        bias = bias_store[1:]  # 4-byte aligned only
        out = torch.empty(M, N, device=cuda_dev)
        rc = _lib_gemm_raw(a, w, out, M, N, K, bias)
        assert rc == 0
        assert _rel(out, ref + bias) < 1e-5


def _lib_gemm_raw(a, w, out, M, N, K, bias):
    from stego_b200 import _lib
    return _lib.load().stego_gemm_bf16(_lib.ptr(a), a.stride(0), 0, _lib.ptr(w), w.stride(0), 0, M, N, K, _lib.ptr(out),
                                       out.stride(0), 0, _lib.ptr(bias), 0, 0, 0, 0, 1, 0, _lib.stream())


@pytest.mark.parametrize("n,M,N,K", [(3, 121, 121, 384), (2, 784, 784, 1152), (5, 50, 300, 72), (1, 128, 256, 64)])
def test_gemm_batched_ragged(cuda_dev, n, M, N, K):
    """stego_gemm_bf16_batched: independent GEMMs in one launch, M / N not tile multiples (TMA zero-fill / clipping per
    batch entry), fp32 output with a 16-byte-aligned row pitch."""
    from stego_b200 import ops
    torch.manual_seed(n * 7 + M)
    a = torch.randn(n, M, K, device=cuda_dev).bfloat16()
    b = (torch.randn(n, N, K, device=cuda_dev) / K ** 0.5).bfloat16()
    ld = (N + 3) // 4 * 4
    store = torch.full((n, M, ld), float("nan"), device=cuda_dev)
    ops.gemm_batched(a, b, store[:, :, :N])
    want = torch.einsum("nmk,npk->nmp", a.float(), b.float())
    assert torch.isfinite(store[:, :, :N]).all()
    assert _rel(store[:, :, :N], want) < 1e-5
    if ld > N:  # the row padding up to the 16-byte pitch holds either what was there or zeros, never part of a result
        pad = store[:, :, N:]
        assert (torch.isnan(pad) | (pad == 0)).all()
    out16 = torch.empty(n, M, (N + 7) // 8 * 8, device=cuda_dev, dtype=torch.bfloat16)
    ops.gemm_batched(a, b, out16[:, :, :N])
    assert _rel(out16[:, :, :N], want) < 4e-3
