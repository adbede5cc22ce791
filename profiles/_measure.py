"""What every profile script shares: the card it runs on, three ways to time GPU work, and the JSON output.

The timers take their warm-up, window and bounds from the caller, so each script's numbers keep the meaning its
docstring and DESIGN.md give them.  card() only reads the device's settings; nothing here changes one.
"""
import json
import math
import os
import subprocess
import time

import torch

_QUERY = ["--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"]


def _require_device():
    if not torch.cuda.is_available():
        raise RuntimeError("no CUDA device: a profile measures a GPU and has nothing to report without one")


def parse_card(line):
    """One line of `nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv,noheader,nounits`."""
    name, power_limit, max_clock = [x.strip() for x in line.rsplit(",", 2)]
    return dict(gpu=name, power_limit_w=float(power_limit), max_sm_clock_mhz=int(float(max_clock)))


def card():
    """Name, power limit and max SM clock of the current CUDA device, read in the calling run."""
    _require_device()
    out = subprocess.run(["nvidia-smi", *_QUERY, "-i", str(torch.cuda.current_device())], capture_output=True,
                         text=True, check=True).stdout
    return parse_card(out.strip().splitlines()[0])


def call_ms(fn):
    """CUDA-event time of one call of fn on the current stream, and what the call returned."""
    _require_device()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    out = fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end), out


def window_ms(fn, *, warmup, min_window_s, min_iters, max_iters=None):
    """CUDA-event time per call over one back-to-back window: `warmup` calls, one call timed to size the window, then
    the fewest calls that fill min_window_s by that estimate, clamped to [min_iters, max_iters].
    Returns (ms per call, calls in the window)."""
    _require_device()
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    # the sizing call's result is dropped before the window: kept alive over it, validation_time's preview (copied to
    # the host by every call) made the ViT-S calls in the window a third to a half slower on an H100
    one = call_ms(fn)[0]
    n = math.ceil(min_window_s * 1e3 / max(one, 1e-3))
    if max_iters is not None:
        n = min(n, max_iters)
    n = max(n, min_iters)

    def window():
        for _ in range(n):
            fn()

    return call_ms(window)[0] / n, n


def enqueue_ms(fn, n):
    """Host-clock time per call of n calls of fn, from an idle device to the return of the last call (no wait for the
    device at the end): what the host spends issuing the work.  The device is synchronised afterwards."""
    _require_device()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n):
        fn()
    t = (time.perf_counter() - t0) * 1e3 / n
    torch.cuda.synchronize()
    return t


def host_ms(fn, n):
    """Host-clock time per call of n calls of fn, from an idle device to the synchronize after the last call; for
    work that ends on the host."""
    _require_device()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / n


def emit(result, out=None, indent=None):
    """Print result as JSON and, given a path, write the same text to it."""
    text = json.dumps(result, indent=indent)
    print(text)
    if out:
        os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
        with open(out, "w") as fh:
            fh.write(text + "\n")
