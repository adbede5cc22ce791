"""2-GPU data-parallel validation: each rank validates its own shard, validation_epoch_end sums the confusion counts
over the ranks, and every rank ends with the counts and metrics of one process that validated every shard (see
tests/ddp_validation_worker.py).  Needs two visible GPUs; skipped on a single-GPU machine."""
import json
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_ddp_validation_matches_one_process(cuda_dev):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    world = 2
    port = 29900 + os.getpid() % 90
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr",
           "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tests", "ddp_validation_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    lines = [json.loads(l.split(" ", 1)[1]) for l in r.stdout.splitlines() if l.startswith("DDP_VALIDATION_RESULT ")]
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert len(lines) == world and all(l["ok"] for l in lines)
    assert all(l["metrics"] == lines[0]["metrics"] for l in lines)
