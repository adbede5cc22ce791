"""2-GPU run of the data-parallel CUDA training step against shard-and-average (see tests/ddp_nccl_worker.py), once with the
fused peer-memory exchange (the default) and once with the NCCL fallback.
Needs two visible GPUs; skipped on a single-GPU machine.  With $STEGO_PARITY_DIR set, the workers' log is kept there."""
import json
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("exchange", ["p2p", "nccl"])
def test_ddp_step_matches_shard_and_average(cuda_dev, exchange):
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    world = 2
    port = 29600 + os.getpid() % 300 + (0 if exchange == "p2p" else 1)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr",
           "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tests", "ddp_nccl_worker.py")]
    env = dict(os.environ, STEGO_TEST_P2P="1" if exchange == "p2p" else "0")
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT, env=env)
    if os.environ.get("STEGO_PARITY_DIR"):
        os.makedirs(os.environ["STEGO_PARITY_DIR"], exist_ok=True)
        with open(os.path.join(os.environ["STEGO_PARITY_DIR"], f"ddp_{exchange}_parity.log"), "w") as fh:
            fh.write(r.stdout + "\n---- stderr ----\n" + r.stderr[-4000:])
    lines = [json.loads(l.split(" ", 1)[1]) for l in r.stdout.splitlines() if l.startswith("DDP_NCCL_RESULT ")]
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert len(lines) == world and all(l["ok"] and l["exchange"] == exchange for l in lines)
