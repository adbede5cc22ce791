"""ctypes binding of libstego_b200.so — the C-ABI drop-in boundary (include/stego_b200.h).

There is deliberately NO fallback: if the shared library is missing or a call fails, a
RuntimeError is raised.  Nothing here imports the oracle.
"""
from __future__ import annotations

import ctypes
import gc
import os
import re
import threading
from typing import Dict, List, Tuple

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libstego_b200.so")
HEADER_PATH = os.path.join(_HERE, "..", "include", "stego_b200.h")

_lib = None
replayed_launches = 0  # kernels launched through CUDA-graph replays (not seen by stego_launch_count)

_CTYPES = {
    "int": ctypes.c_int,
    "float": ctypes.c_float,
    "double": ctypes.c_double,
    "long long": ctypes.c_longlong,
    "void*": ctypes.c_void_p,
    "const void*": ctypes.c_void_p,
    "const float*": ctypes.c_void_p,
    "float*": ctypes.c_void_p,
    "const long long*": ctypes.c_void_p,
    "long long*": ctypes.c_void_p,
    "const int*": ctypes.c_void_p,
    "int*": ctypes.c_void_p,
    "const char*": ctypes.c_char_p,
    "unsigned char*": ctypes.c_void_p,
    "const unsigned char*": ctypes.c_void_p,
    "const double*": ctypes.c_void_p,
    "double*": ctypes.c_void_p,
}


def header_prototypes() -> Dict[str, Tuple[str, List[str]]]:
    """Parse `STEGO_API <ret> name(args);` declarations from the public header."""
    text = open(HEADER_PATH).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    text = re.sub(r"//[^\n]*", "", text)
    text = re.sub(r"^\s*#[^\n]*", "", text, flags=re.M)  # preprocessor lines
    protos: Dict[str, Tuple[str, List[str]]] = {}
    for m in re.finditer(r"STEGO_API\s+([\w\s\*]+?)\s*\b(stego_\w+)\s*\(([^;]*?)\)\s*;", text, flags=re.S):
        ret, name, args = m.group(1).strip(), m.group(2), m.group(3).strip()
        arg_types: List[str] = []
        if args and args != "void":
            for a in args.split(","):
                a = " ".join(a.split())
                t = re.sub(r"\s*\b\w+$", "", a).strip()  # drop the parameter name
                t = t.replace(" *", "*")
                arg_types.append(t)
        protos[name] = (ret.replace(" *", "*"), arg_types)
    return protos


def load():
    """Load the shared library (once) and attach argtypes from the header."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"stego_b200: {LIB_PATH} is missing. Build it with `python -m stego_b200.build` "
            "(or __graft_entry__.build()). There is no CPU / eager fallback for the hot path.")
    lib = ctypes.CDLL(LIB_PATH)
    for name, (ret, args) in header_prototypes().items():
        fn = getattr(lib, name)  # AttributeError if the .so does not export a declared symbol
        fn.restype = _CTYPES[ret]
        fn.argtypes = [_CTYPES[a] for a in args]
    _lib = lib
    return lib


def launch_count() -> int:
    """Kernels this library launched in this process: direct launches + launches inside replayed CUDA graphs."""
    return int(load().stego_launch_count()) + replayed_launches


# One capture at a time in the process: a capture turns the garbage collector off process-wide (below), and a capture in
# torch's global error mode is invalidated by another thread's unsafe calls.  The multi-device paths capture from the
# calling thread, one device after another; nn.DataParallel replicas never capture (their forwards run eagerly).
_CAPTURE_LOCK = threading.Lock()


# One side stream per device to capture on.  torch.cuda.graph's default capture stream is one stream for the whole
# process, made on whichever device was current at the first capture, and entering it switches the current device to
# that one: a graph captured for another device would record its kernels in the first device's context.
_CAPTURE_STREAMS: Dict[int, torch.cuda.Stream] = {}


def capture_stream(device: torch.device) -> torch.cuda.Stream:
    """The side stream captures on `device` use (made on first use; callers hold _CAPTURE_LOCK)."""
    if device.index not in _CAPTURE_STREAMS:
        _CAPTURE_STREAMS[device.index] = torch.cuda.Stream(device=device)
    return _CAPTURE_STREAMS[device.index]


class Graph:
    """`fn()` captured as one CUDA graph on the current device (on that device's capture stream, ordered after its current
    stream), with its result; `replay` launches it on that device's current stream and counts the graph's launches of
    this library in replayed_launches (stego_launch_count does not see them)."""

    def __init__(self, fn):
        self.device = torch.device("cuda", torch.cuda.current_device())
        with _CAPTURE_LOCK, torch.cuda.device(self.device):
            self._capture(fn)

    def _capture(self, fn):
        torch.cuda.synchronize()
        # A dead graph in a reference cycle (a model's graphs hold closures over the model) is destroyed by whichever
        # garbage-collector pass finds it.  Destroying a graph is not permitted while a stream is capturing and
        # invalidates the capture, so collect first and let no automatic pass run inside the capture.
        gc.collect()
        enabled = gc.isenabled()
        gc.disable()
        try:
            self.graph = torch.cuda.CUDAGraph()
            n0 = load().stego_launch_count()
            with torch.cuda.graph(self.graph, stream=capture_stream(self.device)):
                self.result = fn()
            self.launches = load().stego_launch_count() - n0
        finally:
            if enabled:
                gc.enable()

    def replay(self) -> None:
        global replayed_launches
        if torch.cuda.current_device() == self.device.index:
            self.graph.replay()
        else:
            with torch.cuda.device(self.device):
                self.graph.replay()
        replayed_launches += self.launches


def last_error() -> str:
    return load().stego_last_error().decode("utf-8", "replace")


def check(rc: int, what: str) -> None:
    if rc != 0:
        raise RuntimeError(f"stego_b200.{what} failed with status {rc}: {last_error()}")


def ptr(t) -> int:
    """Raw device pointer of a tensor (0 for None)."""
    if t is None:
        return 0
    return t.data_ptr()


def stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def require_cuda(*tensors) -> None:
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise RuntimeError("stego_b200: hot-path tensors must live on a CUDA device (no CPU fallback)")
