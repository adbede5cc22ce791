"""Worker of tests/test_validation_ddp_gpu.py (launched by torchrun, one rank per GPU, NCCL).

Data-parallel validation (train_segmentation.py:476 validates each rank's shard of the val split; torchmetrics sums
the confusion counts over the ranks):
  1. BEFORE the process group exists, every rank validates ALL shards in one process -> the confusion counts and the
     metric dict of one process that saw every shard.
  2. Then the process group is initialised, rank r validates shard r, and validation_epoch_end sums the counts over
     the ranks.
  3. On every rank: the counts validation_epoch_end computed from equal those of step 1, and the metric dicts equal
     step 1's and each other's.
Prints one JSON line per rank; exit code 0 only if every check passed.
"""
import json
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))


def validate(model, shards):
    """validation_step over `shards`, then validation_epoch_end; returns (linear counts, cluster counts, metrics) with
    the counts as validation_epoch_end saw them just before its reset."""
    seen = {}
    for name in ("linear_metrics", "cluster_metrics"):
        m = getattr(model, name)
        reset = m.reset

        def snap(m=m, reset=reset, name=name):
            seen[name] = m.stats.clone()
            reset()
        m.reset = snap
    for i, s in enumerate(shards):
        model.validation_step(dict(img=s["img"], label=s["label"]), i)
    metrics = model.validation_epoch_end([])
    return seen["linear_metrics"], seen["cluster_metrics"], metrics


def main():
    from _parity_util import make_batch, make_model
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    shards = [make_batch(4, 96, dev, seed=200 + r) for r in range(world)]

    # ---- 1. one process validates every shard
    model, _ = make_model("vit_small", dev, fused=True, seed=0)
    lin1, clu1, met1 = validate(model, shards)
    lin0, _, _ = validate(model, shards[:1])
    del model

    # ---- 2. each rank validates its own shard
    dist.init_process_group("nccl", device_id=dev)
    model, _ = make_model("vit_small", dev, fused=True, seed=0)
    lin2, clu2, met2 = validate(model, [shards[rank]])
    ok = torch.equal(lin1, lin2) and torch.equal(clu1, clu2) and met1 == met2
    gathered = [None] * world
    dist.all_gather_object(gathered, met2)
    ok &= all(g == gathered[0] for g in gathered)
    ok &= not model.linear_metrics.stats.any() and not model.cluster_metrics.stats.any()
    ok &= not torch.equal(lin0, lin1)  # the other shards add counts (otherwise the sum proves nothing)
    res = dict(rank=rank, world=world, metrics=met2, counted=int(lin2.sum()), ok=bool(ok))
    print("DDP_VALIDATION_RESULT " + json.dumps(res), flush=True)
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
