"""The scripts under profiles/ time GPU work and identify the card through one module, profiles/_measure.py.

  * every profile imports without a GPU (its work is in main()), so a broken one fails here;
  * card() parses nvidia-smi's line, and card() and the timers refuse to run without a device rather than report a
    value that only looks measured;
  * no other profile creates CUDA events, reads a host clock or queries nvidia-smi on its own.
"""
import glob
import importlib.util
import os

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROFILES = os.path.join(ROOT, "profiles")
SCRIPTS = sorted(os.path.basename(p)[:-3] for p in glob.glob(os.path.join(PROFILES, "*.py")))
PRIVATE_MEASURING = ["torch.cuda.Event(", "elapsed_time", "perf_counter", "nvidia-smi"]


@pytest.fixture
def measure(monkeypatch):
    monkeypatch.syspath_prepend(PROFILES)
    import _measure
    return _measure


@pytest.mark.parametrize("name", SCRIPTS)
def test_profile_imports_without_gpu_and_has_main(name, measure):
    spec = importlib.util.spec_from_file_location(f"profiles_{name}", os.path.join(PROFILES, f"{name}.py"))
    module = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(module)
    if name != "_measure":
        assert callable(getattr(module, "main", None)), f"profiles/{name}.py has no main()"


def test_card_parses_nvidia_smi_line(measure):
    assert measure.parse_card("NVIDIA H100 80GB HBM3, 700.00, 1980\n") == dict(
        gpu="NVIDIA H100 80GB HBM3", power_limit_w=700.0, max_sm_clock_mhz=1980)
    assert measure.parse_card("NVIDIA H100 80GB HBM3, 400.00, 1980.0") == dict(
        gpu="NVIDIA H100 80GB HBM3", power_limit_w=400.0, max_sm_clock_mhz=1980)


def test_card_and_timers_need_a_device(measure, monkeypatch):
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)

    def never():
        raise AssertionError("timed without a device")

    with pytest.raises(RuntimeError, match="no CUDA device"):
        measure.card()
    with pytest.raises(RuntimeError, match="no CUDA device"):
        measure.window_ms(never, warmup=1, min_window_s=0.1, min_iters=1)
    with pytest.raises(RuntimeError, match="no CUDA device"):
        measure.call_ms(never)
    with pytest.raises(RuntimeError, match="no CUDA device"):
        measure.host_ms(never, 1)


@pytest.mark.parametrize("name", [s for s in SCRIPTS if s != "_measure"])
def test_profile_times_and_reads_the_card_through_measure(name):
    src = open(os.path.join(PROFILES, f"{name}.py")).read()
    found = [token for token in PRIVATE_MEASURING if token in src]
    assert not found, f"profiles/{name}.py measures on its own ({found}); use profiles/_measure.py"
