"""Ping-pong GEMM schedule and its two epilogues (TMA store / TMA fp32 reduce-add, and the register epilogue kept for
split-K, the patch-embed row remap, a residual other than the output and unaligned outputs) against an fp32 PyTorch
reference on the bf16 operands."""
import pytest
import torch

pytestmark = pytest.mark.gpu

SENTINEL = 7.0
VIT_LINEARS = {  # name: (N, K, act, in-place residual), per embedding width E
    "qkv": lambda E: (3 * E, E, 0, False),
    "proj": lambda E: (E, E, 0, True),
    "fc1": lambda E: (4 * E, E, 1, False),
    "fc2": lambda E: (E, 4 * E, 0, True),
}


def _ref(a, b, bias=None, act=0):
    y = a.float() @ b.float().t()
    if bias is not None:
        y = y + bias
    if act == 1:
        y = torch.nn.functional.gelu(y)
    elif act == 2:
        y = torch.relu(y)
    return y


def _rel(x, y):
    return ((x.float() - y.float()).norm() / y.float().norm().clamp_min(1e-12)).item()


def _operands(M, N, K, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    a = torch.randn(M, K, device=dev, generator=g).bfloat16()
    b = (torch.randn(N, K, device=dev, generator=g) / K ** 0.5).bfloat16()
    bias = torch.randn(N, device=dev, generator=g)
    return a, b, bias


def _guarded(M, N, dtype, dev, fill=SENTINEL):
    """[M + 3, N + 8] store whose extra rows and columns must stay untouched; returns (store, out view)."""
    store = torch.full((M + 3, N + 8), fill, device=dev, dtype=dtype)
    return store, store[:M, :N]


def _guards_intact(store, M, N):
    return bool(torch.all(store[M:] == SENTINEL)) and bool(torch.all(store[:, N:] == SENTINEL))


@pytest.mark.parametrize("E", [384, 768])
@pytest.mark.parametrize("name", sorted(VIT_LINEARS))
@pytest.mark.parametrize("M", [100, 129, 785 * 3])
def test_vit_linear_shapes(cuda_dev, E, name, M):
    from stego_b200 import ops
    N, K, act, in_place = VIT_LINEARS[name](E)
    a, b, bias = _operands(M, N, K, cuda_dev, seed=E + M)
    want = _ref(a, b, bias, act)
    if in_place:  # x += proj / fc2: the TMA fp32 reduce-add epilogue
        store, x = _guarded(M, N, torch.float32, cuda_dev)
        x.copy_(torch.randn(M, N, device=cuda_dev))
        want = want + x
        ops.gemm(a, b, x, M=M, N=N, K=K, bias=bias, residual=x)
        assert _rel(x, want) < 1e-5
    else:  # bf16 activations: the TMA store epilogue
        store, out = _guarded(M, N, torch.bfloat16, cuda_dev)
        ops.gemm(a, b, out, M=M, N=N, K=K, bias=bias, act=act)
        assert _rel(out, want) < 4e-3
        store32, out32 = _guarded(M, N, torch.float32, cuda_dev)
        ops.gemm(a, b, out32, M=M, N=N, K=K, bias=bias, act=act)
        assert _rel(out32, want) < 1e-5
        assert _guards_intact(store32, M, N)
    assert _guards_intact(store, M, N)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("N", [8, 70, 200, 1000])
def test_ragged_n_guard_columns(cuda_dev, dtype, N):
    """N ending inside a 128-column tile: with whole 16-byte rows (TMA epilogue) or not (register epilogue), nothing
    past column N or row M is written."""
    from stego_b200 import ops
    M, K = 777, 384
    a, b, bias = _operands(M, N, K, cuda_dev, seed=N)
    for in_place in ([False, True] if dtype == torch.float32 else [False]):
        store, out = _guarded(M, N, dtype, cuda_dev)
        want = _ref(a, b, bias)
        if in_place:
            out.copy_(torch.randn(M, N, device=cuda_dev))
            want = want + out
            ops.gemm(a, b, out, M=M, N=N, K=K, bias=bias, residual=out)
        else:
            ops.gemm(a, b, out, M=M, N=N, K=K, bias=bias)
        assert _rel(out, want) < (4e-3 if dtype == torch.bfloat16 else 1e-5)
        assert _guards_intact(store, M, N)


def _tile_counts():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return [1, 3, sms - 1, sms + 1, 2 * sms + 1]


@pytest.mark.parametrize("which", range(5))
@pytest.mark.parametrize("in_place", [False, True])
def test_odd_and_small_tile_counts(cuda_dev, which, in_place):
    """Tile counts where a CTA's second MMA warpgroup has no tile, or one fewer than the first."""
    from stego_b200 import ops
    tiles = _tile_counts()[which]
    M, N, K = 128 * tiles - 5, 128, 256
    a, b, bias = _operands(M, N, K, cuda_dev, seed=tiles)
    store, out = _guarded(M, N, torch.float32, cuda_dev)
    want = _ref(a, b, bias)
    if in_place:
        out.zero_()
        ops.gemm(a, b, out, M=M, N=N, K=K, bias=bias, residual=out)
    else:
        ops.gemm(a, b, out, M=M, N=N, K=K, bias=bias)
    assert _rel(out, want) < 1e-5
    assert _guards_intact(store, M, N)


def test_register_epilogue_residual_not_out(cuda_dev):
    from stego_b200 import ops
    M, N, K = 1000, 384, 384
    a, b, bias = _operands(M, N, K, cuda_dev, seed=21)
    r = torch.randn(M, N, device=cuda_dev)
    store, out = _guarded(M, N, torch.float32, cuda_dev)
    ops.gemm(a, b, out, M=M, N=N, K=K, bias=bias, residual=r)
    assert _rel(out, _ref(a, b, bias) + r) < 1e-5
    assert _guards_intact(store, M, N)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_register_epilogue_unaligned_out(cuda_dev, dtype):
    """Output base 4 bytes past a 16-byte boundary, and an odd row pitch: no tensor map can describe it."""
    from stego_b200 import ops
    M, N, K = 517, 384, 384
    a, b, bias = _operands(M, N, K, cuda_dev, seed=22)
    want = _ref(a, b, bias)
    store = torch.full((M + 1, N + 5), SENTINEL, device=cuda_dev, dtype=dtype)
    out = store[:M, 2:N + 2] if dtype == torch.bfloat16 else store[:M, 1:N + 1]
    ops.gemm(a, b, out, M=M, N=N, K=K, bias=bias)
    assert _rel(out, want) < (4e-3 if dtype == torch.bfloat16 else 1e-5)
    lo = 2 if dtype == torch.bfloat16 else 1
    assert torch.all(store[:, :lo] == SENTINEL) and torch.all(store[:, N + lo:] == SENTINEL)
    assert torch.all(store[M:] == SENTINEL)


def test_register_epilogue_row_div(cuda_dev):
    from stego_b200 import ops
    B, hw, E, K = 5, 196, 768, 192
    a, w, bias = _operands(B * hw, E, K, cuda_dev, seed=23)
    pos = torch.randn(hw + 1, E, device=cuda_dev)
    x = torch.full((B * (hw + 1), E), SENTINEL, device=cuda_dev)
    ops.gemm(a, w, x, M=B * hw, N=E, K=K, bias=bias, residual=pos, row_div=hw)
    want = (_ref(a, w, bias).view(B, hw, E) + pos[1:]).reshape(B * hw, E)
    assert _rel(x.view(B, hw + 1, E)[:, 1:].reshape(B * hw, E), want) < 1e-5
    assert torch.all(x.view(B, hw + 1, E)[:, 0] == SENTINEL)


@pytest.mark.parametrize("splits", [3, 33])
def test_register_epilogue_split_k(cuda_dev, splits):
    from stego_b200 import ops
    rows, n_out, k_in = 50176 // 4, 70, 768
    g = torch.Generator(device=cuda_dev).manual_seed(24)
    dy = torch.zeros(rows, 128, device=cuda_dev, dtype=torch.bfloat16)
    dy[:, :n_out] = torch.randn(rows, n_out, device=cuda_dev, generator=g).bfloat16()
    x = torch.randn(rows, k_in, device=cuda_dev, generator=g).bfloat16()
    dw = torch.zeros(n_out, k_in, device=cuda_dev)
    ops.gemm(dy, x, dw, M=n_out, N=k_in, K=rows, a_mn=True, b_mn=True, splits=splits, atomic=True)
    assert _rel(dw, dy[:, :n_out].float().t() @ x.float()) < 1e-5


def test_two_launches_bit_identical(cuda_dev):
    from stego_b200 import ops
    M, N, K = 50240 // 4, 1536, 384
    a, b, bias = _operands(M, N, K, cuda_dev, seed=25)
    o1 = torch.empty(M, N, device=cuda_dev, dtype=torch.bfloat16)
    o2 = torch.empty_like(o1)
    ops.gemm(a, b, o1, M=M, N=N, K=K, bias=bias, act=ops.ACT_GELU)
    ops.gemm(a, b, o2, M=M, N=N, K=K, bias=bias, act=ops.ACT_GELU)
    assert torch.equal(o1, o2)
    a2, w2, b2 = _operands(M, 384, N, cuda_dev, seed=26)
    x0 = torch.randn(M, 384, device=cuda_dev)
    x1, x2 = x0.clone(), x0.clone()
    ops.gemm(a2, w2, x1, M=M, N=384, K=N, bias=b2, residual=x1)
    ops.gemm(a2, w2, x2, M=M, N=384, K=N, bias=b2, residual=x2)
    assert torch.equal(x1, x2)


def test_inplace_residual_in_cuda_graph(cuda_dev):
    """x += A.B^T + bias captured once and replayed twice gives x + 2 delta, where delta is the same GEMM stored
    (not added) by the TMA store epilogue: the fp32 reduce-add is the plain fp32 sum."""
    from stego_b200 import ops
    M, N, K = 3 * 785, 384, 1536
    a, b, bias = _operands(M, N, K, cuda_dev, seed=27)
    delta = torch.empty(M, N, device=cuda_dev)
    ops.gemm(a, b, delta, M=M, N=N, K=K, bias=bias)
    x0 = torch.randn(M, N, device=cuda_dev)
    x = x0.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):  # warm-up launch outside the capture (module load, function attributes)
        ops.gemm(a, b, x, M=M, N=N, K=K, bias=bias, residual=x)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.gemm(a, b, x, M=M, N=N, K=K, bias=bias, residual=x)
    x.copy_(x0)
    graph.replay()
    graph.replay()
    torch.cuda.synchronize()
    want = (x0 + delta) + delta
    assert torch.allclose(x, want, rtol=1e-6, atol=1e-6), (x - want).abs().max().item()
