"""Build libstego_b200.so (sm_90a) in-tree with nvcc.

The shared library is the drop-in boundary (C-ABI, see include/stego_b200.h). It is built in-tree so
the package imports straight from the source tree; the library is git-ignored.
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(CSRC, "_obj")
LIB = os.path.join(HERE, "libstego_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-I", os.path.join(HERE, "..", "include"),
] + os.environ.get("STEGO_NVCC_DEFS", "").split()  # extra -D flags for diagnostic builds


def _sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest(path: str) -> str:
    h = hashlib.sha256()
    for dep in [path] + [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith((".cuh", ".h"))]:
        with open(dep, "rb") as fh:
            h.update(fh.read())
    h.update(" ".join(FLAGS).encode())
    return h.hexdigest()


def _compile(src: str, verbose: bool) -> str:
    path = os.path.join(CSRC, src)
    obj = os.path.join(OBJ, src.replace(".cu", ".o"))
    stamp = obj + ".sha"
    dig = _digest(path)
    if os.path.exists(obj) and os.path.exists(stamp) and open(stamp).read() == dig:
        return obj
    cmd = [NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", path, "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
    if verbose:
        sys.stderr.write(r.stderr)
    with open(stamp, "w") as fh:
        fh.write(dig)
    return obj


def build(verbose: bool = False, force: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    if force:
        for f in os.listdir(OBJ):
            os.remove(os.path.join(OBJ, f))
    srcs = _sources()
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(lambda s: _compile(s, verbose), srcs))
    newest = max(os.path.getmtime(o) for o in objs)
    if force or not os.path.exists(LIB) or os.path.getmtime(LIB) < newest:
        cmd = [NVCC, "-shared", "-o", LIB] + objs + ["-cudart", "static"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    print(build(verbose="-v" in sys.argv, force="-f" in sys.argv))
