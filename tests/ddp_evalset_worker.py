"""Worker of tests/test_evalset_gpu.py::test_ddp_validate_sums_to_one_process_counts (launched by torchrun with two
ranks; gloo, each rank on GPU local_rank % device_count, so one GPU serves both).

  1. BEFORE the process group exists, every rank runs validation_step over the batches of BOTH ranks' shards
     (EvalSet.frames(rank=r, world_size=2), DistributedSampler's padding included) and validation_epoch_end -> the
     confusion counts and metric dict of one process that saw every padded shard.
  2. Then the process group is initialised and rank r runs validate(store, B, r, 2), whose validation_epoch_end sums
     the counts over the ranks.
  3. On every rank: those counts and metrics equal step 1's.
Prints one JSON line per rank; exit code 0 only if every check passed.
"""
import json
import os
import sys
import tempfile

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))


def snapshot(model):
    seen = {}
    for name in ("linear_metrics", "cluster_metrics"):
        m = getattr(model, name)
        reset = m.reset

        def snap(m=m, reset=reset, name=name):
            seen[name] = m.stats.clone()
            reset()
        m.reset = snap
    return seen


def main():
    from _parity_util import make_model
    from stego_b200.evalset import EvalSet
    from test_evalset import load_gold, write_tree
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    dev = torch.device("cuda", local % torch.cuda.device_count())
    torch.cuda.set_device(dev)
    gold = load_gold()
    B = 2
    with tempfile.TemporaryDirectory() as root:
        write_tree(gold, root)
        store = EvalSet.coco(root, "cocostuff27", "val", 32, gold["fine_to_coarse"])  # 5 samples: shards pad to 6

    # ---- 1. one process validates every padded shard
    model, _ = make_model("vit_small", dev, fused=True, seed=0)
    seen1 = snapshot(model)
    i = 0
    for r in range(world):
        for batch in store.frames(B, mask=False, rank=r, world_size=world):
            model.validation_step(batch, i)
            i += 1
    met1 = model.validation_epoch_end([])
    del model

    # ---- 2. each rank validates its own shard
    dist.init_process_group("gloo")
    model, _ = make_model("vit_small", dev, fused=True, seed=0)
    seen2 = snapshot(model)
    met2 = model.validate(store, B, rank, world)
    ok = all(torch.equal(seen1[k], seen2[k]) for k in seen1) and met1 == met2
    gathered = [None] * world
    dist.all_gather_object(gathered, met2)
    ok &= all(g == gathered[0] for g in gathered)
    res = dict(rank=rank, world=world, metrics=met2, counted=int(seen2["linear_metrics"].sum()), ok=bool(ok))
    print("DDP_EVALSET_RESULT " + json.dumps(res), flush=True)
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
