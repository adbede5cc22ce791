"""CPU: stego_gemm_bf16 / stego_gemm_bf16_batched refuse the calls their contract (include/stego_b200.h) rules out
before anything is launched, and say why.  atomic_out adds each split's partial sum into out, so a bias, an activation
or a residual cannot be applied there; a leading dimension shorter than its row would make rows overlap.
tests/test_gemm_fp64_gpu.py makes the same calls on device memory and checks that out is left untouched."""
import pytest
import torch

SENTINEL = -7.25

REFUSED = {  # name: (kwargs overrides, words the error names)
    "atomic_bias": (dict(atomic=1, bias=True), "atomic_out"),
    "atomic_act": (dict(atomic=1, act=1), "atomic_out"),
    "atomic_relu_split": (dict(atomic=1, act=2, splits=2), "atomic_out"),
    "atomic_residual": (dict(atomic=1, residual=True), "atomic_out"),
    "atomic_residual_in_place": (dict(atomic=1, residual="out"), "atomic_out"),
    "lda_short": (dict(lda=-8), "lda"),
    "lda_short_mn": (dict(a_mn=1, lda=-8), "lda"),
    "ldb_short": (dict(ldb=-8), "ldb"),
    "ldb_short_mn": (dict(b_mn=1, ldb=-8), "ldb"),
    "ldo_short": (dict(ldo=-2), "ldo"),
    "ldr_short": (dict(residual=True, ldr=-2), "ldr"),
    "batched_ldo_short": (dict(batched=True, ldo=-2), "ldo"),
}


def refused_call(name, dev):
    """Issue one call that must be refused; returns (rc, out before, out after the call, expected word).  Host tensors
    are used when dev is the CPU: the refusal comes before anything touches memory."""
    from stego_b200 import _lib as L
    dev = torch.device(dev)
    kw, word = REFUSED[name]
    M, N, K = 72, 80, 96
    a_mn, b_mn = kw.get("a_mn", 0), kw.get("b_mn", 0)
    lda = (M if a_mn else K) + kw.get("lda", 8)
    ldb = (N if b_mn else K) + kw.get("ldb", 8)
    ldo = N + kw.get("ldo", 8)
    a = torch.zeros((K if a_mn else M) * max(lda, 8) + 64, dtype=torch.bfloat16, device=dev)
    b = torch.zeros((K if b_mn else N) * max(ldb, 8) + 64, dtype=torch.bfloat16, device=dev)
    out = torch.full((M * N + M * 8 + 64,), SENTINEL, device=dev)
    bias = torch.ones(N, device=dev) if kw.get("bias") else None
    res = torch.ones(M * (N + 8), device=dev) if kw.get("residual") is True else None
    ldr = N + kw.get("ldr", 8) if res is not None else (ldo if kw.get("residual") == "out" else 0)
    rptr = out.data_ptr() if kw.get("residual") == "out" else L.ptr(res)
    before = out.clone()
    stream = L.stream() if dev.type == "cuda" else 0
    lib = L.load()
    if kw.get("batched"):
        rc = lib.stego_gemm_bf16_batched(a.data_ptr(), lda, 0, a_mn, b.data_ptr(), ldb, 0, b_mn, 1, M, N, K,
                                         out.data_ptr(), ldo, 0, 0, 0, 0, stream)
    else:
        rc = lib.stego_gemm_bf16(a.data_ptr(), lda, a_mn, b.data_ptr(), ldb, b_mn, M, N, K, out.data_ptr(), ldo, 0,
                                 L.ptr(bias), kw.get("act", 0), rptr, ldr, 0, kw.get("splits", 1), kw.get("atomic", 0),
                                 stream)
    if dev.type == "cuda":
        torch.cuda.synchronize()
    return rc, before, out, word


@pytest.mark.parametrize("name", sorted(REFUSED))
def test_refused_before_any_cuda_call(name):
    from stego_b200 import _lib
    rc, before, after, word = refused_call(name, "cpu")
    assert rc != 0, name
    assert word in _lib.last_error(), _lib.last_error()
    assert torch.equal(before, after)

