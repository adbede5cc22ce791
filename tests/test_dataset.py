"""CPU: the resident training set's host draws (stego_b200.dataset.Sampler) against the reference loader's batches in
tests/golden/dataset.pt (oracle/make_golden_dataset.py), DistributedSampler's order, the global generators left
untouched, torch's worker seeding, and the refusals that happen before anything reaches the device."""
import os
import random
import sys

import numpy as np
import pytest
import torch
from torch.utils.data import DistributedSampler
from torch.utils.data._utils.worker import _generate_state as torch_generate_state

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from stego_b200 import dataset as D  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden", "dataset.pt")


def load_gold(path):
    """The fixture with each run expanded to its batches: dicts of CPU int64 ind, ind_pos and seed."""
    g = torch.load(path)
    for case in g["cases"].values():
        for w, run in case["runs"].items():
            parts = torch.split(run["draws"], run["sizes"])
            case["runs"][w] = [dict(ind=p[:, 0].clone(), ind_pos=p[:, 1].clone(), seed=p[:, 2].clone()) for p in parts]
    return g


@pytest.fixture(scope="module")
def gold():
    return load_gold(GOLD)


def draws(nns, B, num_neighbors, seed, workers, res, n_batches, **kw):
    out = []
    for epoch in D.Sampler(nns, B, num_neighbors, seed, workers, res=res, **kw):
        for b in epoch:
            out.append(b)
            if len(out) == n_batches:
                return out


@pytest.mark.parametrize("workers", [0, 1, 3])
@pytest.mark.parametrize("case", ["cropped_32", "cropped_30", "directory_32", "directory_30",
                                  "directory_unlabelled_32", "directory_unlabelled_30"])
def test_sampler_matches_reference_loader(gold, case, workers):
    run = gold["cases"][case]["runs"][workers]
    res = int(case.rsplit("_", 1)[1])
    got = draws(gold["nns"].numpy(), gold["batch_size"], gold["num_neighbors"], gold["seed"], workers, res, len(run))
    assert len(run) == 10  # 2.5 epochs of 13 samples in batches of 4: partial batches at each epoch's end
    for k, (want, (ind, pos, seeds)) in enumerate(zip(run, got)):
        assert ind.tolist() == want["ind"].tolist(), (k, "ind")
        assert pos.tolist() == want["ind_pos"].tolist(), (k, "ind_pos")
        assert seeds.tolist() == want["seed"].tolist(), (k, "seed")


def test_worker_streams_differ(gold):
    """The three golden runs differ from each other, so the W = 0 / 1 / 3 comparisons check three distinct streams."""
    runs = gold["cases"]["cropped_32"]["runs"]
    seeds = {w: torch.cat([b["seed"] for b in runs[w]]).tolist() for w in runs}
    assert seeds[0] != seeds[1] and seeds[1] != seeds[3] and seeds[0] != seeds[3]


@pytest.mark.parametrize("world_size", [2, 3])
def test_distributed_order_matches_distributed_sampler(world_size):
    n, B, seed = 13, 4, 7
    nns = np.stack([np.arange(n)] * 3, 1)
    for rank in range(world_size):
        sampler = D.Sampler(nns, B, 1, seed, 0, rank=rank, world_size=world_size, res=16)
        ref = DistributedSampler(list(range(n)), num_replicas=world_size, rank=rank, shuffle=True, seed=seed)
        for epoch, plan in zip(range(3), sampler):
            ref.set_epoch(epoch)
            want = list(iter(ref))
            got = [i for ind, _, _ in plan for i in ind.tolist()]
            assert got == want and len(got) == -(-n // world_size)


def test_global_generators_unchanged(gold):
    random.seed(123)
    np.random.seed(321)
    torch.manual_seed(99)
    states = random.getstate(), np.random.get_state(), torch.get_rng_state()
    for workers in (0, 2):
        draws(gold["nns"].numpy(), 4, 3, 11, workers, 32, 12)
    assert random.getstate() == states[0]
    after = np.random.get_state()
    assert all(np.array_equal(a, b) if isinstance(a, np.ndarray) else a == b for a, b in zip(after, states[1]))
    assert torch.equal(torch.get_rng_state(), states[2])


def test_generate_state_equals_torch():
    rng = np.random.default_rng(0)
    for base in [0, 1, (1 << 63) - 1, (1 << 32) - 1, 1 << 32] + [int(x) for x in rng.integers(0, 1 << 63, 200)]:
        for w in (0, 1, 2, 7, 63):
            assert D._generate_state(base, w) == torch_generate_state(base, w)


def test_abandoned_epoch_keeps_the_single_process_stream(gold):
    """Leaving an epoch early still draws its remaining samples, so the next epoch's stream is the reference's."""
    run = gold["cases"]["cropped_32"]["runs"][0]
    sampler = D.Sampler(gold["nns"].numpy(), 4, gold["num_neighbors"], gold["seed"], 0, res=32)
    next(next(sampler))
    second = next(sampler)
    assert next(second)[0].tolist() == run[4]["ind"].tolist()


# ---- refusals (before any device work) -------------------------------------------------------------------------------
class _Stub(D.ResidentDataset):
    """A store object without device memory, to reach the host-side checks of batches()."""

    def __init__(self, n, res, count=None, kind="cropped"):
        self.n, self.res, self.kind, self.has_labels = n, res, kind, True
        self.count = n if count is None else count


@pytest.mark.parametrize("kind", ["cocostuff27", "cityscapes", "potsdam", "cocostuff3"])
def test_refuses_non_training_classes(kind):
    with pytest.raises(ValueError, match="not a training set class"):
        D.ResidentDataset(4, 32, kind=kind)


@pytest.mark.parametrize("kw, match", [(dict(kind="voc"), "kind="), (dict(location="disk"), "location="),
                                       (dict(kind="cropped", has_labels=False), "always has labels")])
def test_refuses_bad_construction(kw, match):
    with pytest.raises(ValueError, match=match):
        D.ResidentDataset(4, 32, **kw)


@pytest.mark.parametrize("kw, match", [
    (dict(nns=np.zeros((5, 4), np.int64)), "5 rows for a 6-sample store"),
    (dict(num_neighbors=0), "num_neighbors=0"),
    (dict(num_neighbors=4), "num_neighbors=4"),
    (dict(nns=np.zeros((6, 1), np.int64)), "1 column"),
    (dict(nns=np.full((6, 4), 6, np.int64)), "outside 0..5"),
    (dict(nns=np.zeros((6, 4), np.float32)), "integer table"),
    (dict(res=64), "res=64"),
    (dict(dtype=torch.float16), "dtype="),
    (dict(batch_size=0), "batch_size=0"),
    (dict(world_size=2, rank=2), "rank=2"),
    (dict(loader_workers=-1), "loader_workers=-1"),
])
def test_batches_refusals(kw, match):
    args = dict(nns=np.zeros((6, 4), np.int64), batch_size=2, num_neighbors=3, seed=0)
    args.update(kw)
    with pytest.raises(ValueError, match=match):
        next(_Stub(6, 32).batches(**args))


def test_refuses_a_store_not_yet_full():
    with pytest.raises(ValueError, match="holds 3 of its 6"):
        next(_Stub(6, 32, count=3).batches(np.zeros((6, 4), np.int64), 2, 3, 0))
    with pytest.raises(ValueError, match="holds 3 of its 6"):
        next(_Stub(6, 32, count=3).frames(2))
