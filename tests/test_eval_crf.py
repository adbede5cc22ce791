"""Host-side checks of the CRF-refined evaluation (stego_b200.eval.fused_eval_crf) that need no GPU: every bad argument
is refused before anything is launched, and the new C-ABI entry points are declared, exported and validate their
arguments."""
import pytest
import torch

from stego_b200 import _lib
from stego_b200.eval import fused_eval_crf
from stego_b200.modules import ClusterLookup


def _args(B=2, C=8, h=3, w=4, H=12, W=16, n_lin=5, n_clu=5, label_dtype=torch.int64):
    lin = torch.nn.Conv2d(C, n_lin, (1, 1))
    clu = ClusterLookup(C, n_clu)
    code = torch.randn(B, C, h, w)
    img = torch.randn(B, 3, H, W)
    label = torch.randint(0, n_lin, (B, H, W)).to(label_dtype)
    return dict(code=code, linear_probe=lin, cluster_probe=clu, img=img, label=label,
                linear_confusion=torch.zeros(n_lin, n_lin, dtype=torch.int64),
                cluster_confusion=torch.zeros(n_clu, n_lin, dtype=torch.int64))


def _refused(exc, match, **kw):
    n0 = _lib.launch_count()
    a = _args(**{k: v for k, v in kw.items() if k in ("n_lin", "n_clu", "C", "label_dtype")})
    a.update({k: v for k, v in kw.items() if k not in ("n_lin", "n_clu", "C", "label_dtype")})
    with pytest.raises(exc, match=match):
        fused_eval_crf(**a)
    assert _lib.launch_count() == n0


def test_cpu_tensors_are_refused():
    _refused(RuntimeError, "CUDA")
    _refused(RuntimeError, "CUDA", label=None, linear_confusion=None, cluster_confusion=None)
    for dt in (torch.uint8, torch.int32):
        _refused(RuntimeError, "CUDA", label_dtype=dt)


def test_label_of_another_size_is_refused():
    _refused(ValueError, "label", label=torch.zeros(2, 12, 15, dtype=torch.int64))
    _refused(ValueError, "label", label=torch.zeros(3, 12, 16, dtype=torch.int64))
    _refused(ValueError, "label dtype", label=torch.zeros(2, 12, 16, dtype=torch.float32))


def test_more_than_32_classes_are_refused():
    _refused(ValueError, "unsupported", n_lin=33, linear_confusion=None, cluster_confusion=None, label=None)
    _refused(ValueError, "unsupported", n_clu=33, linear_confusion=None, cluster_confusion=None, label=None)
    _refused(ValueError, "unsupported", C=97)


def test_confusion_tensors_of_wrong_shape_or_dtype_are_refused():
    _refused(ValueError, "linear_confusion", linear_confusion=torch.zeros(5, 6, dtype=torch.int64))
    _refused(ValueError, "cluster_confusion", cluster_confusion=torch.zeros(6, 5, dtype=torch.int64))
    _refused(ValueError, "linear_confusion", linear_confusion=torch.zeros(5, 5, dtype=torch.int32))
    _refused(ValueError, "cluster_confusion", cluster_confusion=torch.zeros(5, 5, dtype=torch.float32))
    _refused(ValueError, "cluster_confusion", cluster_confusion=torch.zeros(5, 5, dtype=torch.int64).t())
    _refused(ValueError, "without a confusion", linear_confusion=None, cluster_confusion=None)
    _refused(ValueError, "without a label", label=None)


def test_other_shapes_are_refused():
    _refused(ValueError, "upsampling only", img=torch.randn(2, 3, 2, 16), label=None, linear_confusion=None,
             cluster_confusion=None)
    _refused(ValueError, "code_flipped", code_flipped=torch.randn(2, 8, 3, 5))
    _refused(ValueError, "img", img=torch.randn(2, 4, 12, 16))


def test_crf_entry_points_declared_and_checking_arguments():
    protos = _lib.header_prototypes()
    for name in ("stego_eval_crf_unary", "stego_crf_norm", "stego_crf_mean_field"):
        assert name in protos
    lib = _lib.load()
    n0 = _lib.launch_count()
    rc = lib.stego_eval_crf_unary(0, 0, 8, 8, 1, 2, 2, 4, 4, 0, 0, 5, 0, 5, 2.0, 0, 0, 0, 0)
    assert rc == -1 and "null pointer" in _lib.last_error()
    rc = lib.stego_crf_norm(3, 16, 4, *([0] * 9), 0)
    assert rc == -1 and "bad args" in _lib.last_error()
    for n_lin, n_clu in ((33, 5), (5, 33), (5, -1)):
        rc = lib.stego_crf_mean_field(1, 16, n_lin, n_clu, 10, *([0] * 9), 8, *([0] * 7), 8, 3.0, 4.0, *([0] * 9), 0, 0,
                                      0, 0, 0)
        assert rc == -1 and "unsupported" in _lib.last_error()
    # one probe (n_clu = 0) passes the limits and stops at the missing buffers
    rc = lib.stego_crf_mean_field(1, 16, 5, 0, 10, *([0] * 9), 8, *([0] * 7), 8, 3.0, 4.0, *([0] * 9), 0, 0, 0, 0, 0)
    assert rc == -1 and "null pointer" in _lib.last_error()
    assert _lib.launch_count() == n0
