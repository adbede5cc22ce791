"""The resident-weight GEMM (gemm_bf16_resident_kernel: K <= 384, K-major operands, TMA epilogue, >= 4 tiles per SM)
against gemm_bf16_kernel.  Each output element sees the same sequence of k16 wgmmas in both kernels, so the outputs
must be bit-identical.  The reference issues the same GEMM in row slices small enough (fewer than 4 tiles per SM) to
run gemm_bf16_kernel; test_intended_kernels_ran checks with torch.profiler, in a child process, which kernel each
case launches."""
import json
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

SENTINEL = 7.0
EPIS = {  # name: (output dtype, act, in-place fp32 residual)
    "bf16": (torch.bfloat16, 0, False),
    "gelu": (torch.bfloat16, 1, False),
    "relu": (torch.bfloat16, 2, False),
    "f32": (torch.float32, 0, False),
    "add": (torch.float32, 0, True),
}
# (M, N, K, epilogue): the ViT-S linears and the head's cluster2-a GEMM at c1 (64 images of 784 patches + cls), ragged
# M and N, short K with a K tail, and column / tile counts that do and do not divide 132 SMs
CASES = [
    (64 * 785, 1152, 384, "bf16"),   # qkv: 9 column blocks
    (64 * 785, 384, 384, "add"),     # proj: x += ...
    (64 * 785, 1536, 384, "gelu"),   # fc1
    (64 * 784, 384, 384, "relu"),    # head cluster2-a
    (64 * 785, 384, 384, "f32"),
    (64 * 785 - 57, 1152, 384, "bf16"),
    (64 * 785 - 57, 384, 384, "add"),
    (33001, 1000, 136, "gelu"),      # 8 column blocks, the last one ragged; K tail
    (70001, 200, 64, "add"),         # 2 column blocks, the last one 72 wide
    (40000, 1536, 64, "relu"),
    (176 * 128, 384, 384, "bf16"),   # 528 tiles: 4 per CTA on 132 SMs
    (176 * 128 + 1, 384, 384, "add"),
    (4 * 128, 16896, 64, "bf16"),    # 132 column blocks: one CTA per column
]
GRAPH_CASES = [CASES[0], CASES[1]]


def _ids(c):
    return f"M{c[0]}_N{c[1]}_K{c[2]}_{c[3]}"


def _operands(M, N, K, in_place, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    a = (torch.randn(M, K, device=dev, generator=g) * 0.5).bfloat16()
    b = (torch.randn(N, K, device=dev, generator=g) / K ** 0.5).bfloat16()
    bias = torch.randn(N, device=dev, generator=g)
    x0 = torch.randn(M, N, device=dev, generator=g) if in_place else None
    return a, b, bias, x0


def _guarded(M, N, dtype, dev):
    """[M + 3, N + 8] store whose extra rows and columns must stay untouched; returns (store, out view)."""
    store = torch.full((M + 3, N + 8), SENTINEL, device=dev, dtype=dtype)
    return store, store[:M, :N]


def _guards_intact(store, M, N):
    return bool(torch.all(store[M:] == SENTINEL)) and bool(torch.all(store[:, N:] == SENTINEL))


def _slice_rows(N, dev):
    """rows per reference slice: a multiple of 128 with fewer than 4 tiles per SM"""
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    tiles_n = (N + 127) // 128
    return 128 * max(1, (4 * sms - 1) // tiles_n)


def _setup(case, dev):
    """(launch(out), fresh output, reference output computed in row slices); the three share the operands"""
    from stego_b200 import ops
    M, N, K, epi = case
    dtype, act, in_place = EPIS[epi]
    a, b, bias, x0 = _operands(M, N, K, in_place, dev, seed=M + N + K)

    def launch(out, lo=0, hi=M):
        ops.gemm(a[lo:hi], b, out[lo:hi], M=hi - lo, N=N, K=K, bias=bias, act=act,
                 residual=out[lo:hi] if in_place else None)

    def fresh():
        store, out = _guarded(M, N, dtype, dev)
        if in_place:
            out.copy_(x0)
        return store, out

    ref_store, ref = fresh()
    step = _slice_rows(N, dev)
    for lo in range(0, M, step):
        launch(ref, lo, min(M, lo + step))
    return launch, fresh, ref_store


def _bit_equal(x, y):
    return torch.equal(x.view(torch.int16) if x.dtype == torch.bfloat16 else x.view(torch.int32),
                       y.view(torch.int16) if y.dtype == torch.bfloat16 else y.view(torch.int32))


@pytest.mark.parametrize("case", CASES, ids=_ids)
def test_bit_identical_to_sliced(cuda_dev, case):
    M, N = case[0], case[1]
    launch, fresh, ref_store = _setup(case, cuda_dev)
    store, out = fresh()
    launch(out)
    torch.cuda.synchronize()
    assert _guards_intact(ref_store, M, N)
    assert _guards_intact(store, M, N)
    assert _bit_equal(store, ref_store)
    assert torch.isfinite(out.float()).all()


@pytest.mark.parametrize("case", GRAPH_CASES, ids=_ids)
def test_repeat_and_graph_replay(cuda_dev, case):
    """two eager launches, and one replayed inside a CUDA graph, are bit-identical"""
    M, N = case[0], case[1]
    launch, fresh, ref_store = _setup(case, cuda_dev)
    runs = []
    for _ in range(2):
        store, out = fresh()
        launch(out)
        runs.append(store)
    store_g, out_g = fresh()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
        launch(out_g)
    torch.cuda.current_stream().wait_stream(s)
    graph.replay()
    torch.cuda.synchronize()
    for st in runs + [store_g]:
        assert _guards_intact(st, M, N)
        assert _bit_equal(st, ref_store)


def _kernel_cases(dev):
    """name -> (launch, whether the resident kernel must run); the M = 1000 cases stay on gemm_bf16_kernel"""
    cases = {}
    for case in CASES:
        launch, fresh, _ = _setup(case, dev)
        out = fresh()[1]
        cases[_ids(case)] = (lambda launch=launch, out=out: launch(out), True)
    for N, K, epi in ((1152, 384, "bf16"), (384, 384, "add"), (1536, 384, "gelu")):
        launch, fresh, _ = _setup((1000, N, K, epi), dev)
        out = fresh()[1]
        cases[_ids((1000, N, K, epi))] = (lambda launch=launch, out=out: launch(out), False)
    return cases


def test_intended_kernels_ran(cuda_dev):
    """every case above launches gemm_bf16_resident_kernel exactly once and no gemm_bf16_kernel; M = 1000 does not"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    res = subprocess.run([sys.executable, os.path.abspath(__file__), "--kernel-names"], cwd=root, capture_output=True,
                         text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-4000:]
    got = json.loads(res.stdout.strip().splitlines()[-1])
    assert len(got) == len(CASES) + 3
    for case, (resident, names) in got.items():
        gemms = [n for n in names if "gemm_bf16" in n]
        want = "gemm_bf16_resident_kernel" if resident else "gemm_bf16_kernel<"
        assert len(gemms) == 1 and want in gemms[0], (case, gemms)


if __name__ == "__main__" and sys.argv[1:] == ["--kernel-names"]:
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from torch.profiler import ProfilerActivity, profile
    dev = torch.device("cuda:0")
    for _ in range(2):  # the first sessions of a process can miss kernel records while the profiler initialises
        with profile(activities=[ProfilerActivity.CUDA]):
            torch.ones(1024, device=dev).sum().item()
    result = {}
    for case, (fn, resident) in _kernel_cases(dev).items():
        fn()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        result[case] = (resident, [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA])
    print(json.dumps(result))
