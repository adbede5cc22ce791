"""Both training-step paths (the autograd-stitched one and the hand-scheduled fused_step.FusedStep) launch the head,
sampling and probe kernels through the same stage functions, so a change to a stage's arguments, layout or padding is
made once.

  * CPU: each of those entry points is referenced from exactly one function of the package.
  * GPU: the first step of a fused model and of an autograd twin from the same generator state gives bit-equal
    correspondence and cluster terms (both paths launch the same functions on the same inputs, and those reductions
    run in a fixed order).
"""
import ast
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "stego_b200")

SHARED_ENTRY_POINTS = [
    "stego_head_dropout3", "stego_cast_pad_bf16", "stego_relu_bwd_bf16", "stego_colsum", "stego_sample_norm_fwd",
    "stego_sample_norm_bwd", "stego_linear_probe_ce", "stego_cluster_lookup_fwd", "stego_cluster_lookup_bwd",
]


def _referencing_functions():
    """entry point -> set of 'module:qualified.function' names whose bodies reference it as an attribute."""
    refs = {name: set() for name in SHARED_ENTRY_POINTS}
    for dirpath, _, files in os.walk(PKG):
        for fn in files:
            if not fn.endswith(".py"):
                continue
            path = os.path.join(dirpath, fn)
            mod = os.path.relpath(path, ROOT)
            tree = ast.parse(open(path).read(), filename=path)

            def visit(node, scope):
                for child in ast.iter_child_nodes(node):
                    if isinstance(child, (ast.FunctionDef, ast.AsyncFunctionDef, ast.ClassDef)):
                        visit(child, scope + [child.name])
                        continue
                    if isinstance(child, ast.Attribute) and child.attr in refs:
                        refs[child.attr].add(f"{mod}:{'.'.join(scope) or '<module>'}")
                    visit(child, scope)
            visit(tree, [])
    return refs


def test_each_shared_entry_point_has_one_call_site():
    refs = _referencing_functions()
    for name, sites in refs.items():
        assert len(sites) == 1, f"{name} is called from {sorted(sites) or 'nowhere'}"


@pytest.mark.gpu
def test_first_step_fused_and_autograd_bit_equal(cuda_dev):
    import torch
    from _parity_util import make_batch, make_model
    fused, _ = make_model("vit_small", cuda_dev, fused=True)
    twin, _ = make_model("vit_small", cuda_dev, fused=False)
    batch = make_batch(4, 64, cuda_dev, seed=1)
    torch.manual_seed(777)
    gpu_state, cpu_state = torch.cuda.get_rng_state(cuda_dev), torch.get_rng_state()
    fused.training_step(batch, 0)
    torch.cuda.set_rng_state(gpu_state, cuda_dev)
    torch.set_rng_state(cpu_state)
    twin.training_step(batch, 0)
    assert fused._fused.step_idx == 1 and twin._fused is None
    torch.cuda.synchronize()
    got = {k: v.detach().clone() for k, v in fused.logged.items()}
    want = {k: v.detach().clone() for k, v in twin.logged.items()}
    for key in ("loss/pos_intra", "loss/pos_inter", "cd/pos_intra", "cd/pos_inter", "loss/cluster"):
        assert torch.equal(got[key], want[key]), (key, got[key].item(), want[key].item())
    # the linear-probe CE sums its pixels with fp64 atomics: equal up to their order
    lin_f, lin_t = got["loss/linear"].item(), want["loss/linear"].item()
    assert abs(lin_f - lin_t) <= 1e-6 * abs(lin_t), (lin_f, lin_t)
