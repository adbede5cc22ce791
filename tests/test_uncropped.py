"""CPU: the random-crop loader's host draws (stego_b200.dataset.Sampler with row sizes) against the reference loader's
batches on the uncropped classes in tests/golden/uncropped.pt (oracle/make_golden_uncropped.py): shuffle order,
positives, aug seeds and every RandomCrop window; the global generators left untouched; DistributedSampler sharding
with windows; and the refusals that happen before anything reaches the device."""
import os
import random
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from stego_b200 import dataset as D  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden", "uncropped.pt")
CASES = [f"{layout}_{res}" for layout in ("cocostuff27", "cityscapes", "potsdam", "directory") for res in (32, 30)]


def load_gold(path):
    """The fixture with each case's rows expanded: full / squashed hold per index img (uint8 bytes of `values`),
    label (int64) and mask (its dtype and per-sample shape)."""
    g = torch.load(path)
    for name, case in g["cases"].items():
        res = int(name.rsplit("_", 1)[1])
        for part in ("full", "squashed"):
            rows = case[part]
            dtype = {"bool": torch.bool, "float32": torch.float32}[rows["mask_dtype"]]
            masks = []
            for bits, shape in zip(rows["mask"], rows["mask_shape"]):
                flat = np.unpackbits(bits.numpy())[:int(np.prod(shape))]
                masks.append(torch.from_numpy(flat.reshape(shape).copy()).to(dtype))
            case[part] = dict(img=[g["frames"][res][part][int(k)] for k in rows["img_index"]],
                              label=[lab.to(torch.int64) for lab in rows["label"]], mask=masks)
    return g


@pytest.fixture(scope="module")
def gold():
    return load_gold(GOLD)


def row_sizes(case) -> np.ndarray:
    """int64 [n, 4]: each index's Resize(res) image and label sizes, read off the reference's uncropped rows."""
    full = case["full"]
    return np.array([tuple(i.shape[-2:]) + tuple(lab.shape[-2:]) for i, lab in zip(full["img"], full["label"])],
                    dtype=np.int64)


def sampled(gold, case, crop, workers, n_batches, **kw):
    res = int(case.rsplit("_", 1)[1])
    sizes = row_sizes(gold["cases"][case]) if crop == "random" else None
    out = []
    for epoch in D.Sampler(gold["nns"].numpy(), gold["batch_size"], gold["num_neighbors"], gold["seed"], workers,
                           res=res, sizes=sizes, **kw):
        for b in epoch:
            out.append(b)
            if len(out) == n_batches:
                return out


@pytest.mark.parametrize("workers", [0, 2])
@pytest.mark.parametrize("crop", ["center", "random", None])
@pytest.mark.parametrize("case", CASES)
def test_sampler_matches_reference_loader(gold, case, crop, workers):
    run = gold["cases"][case]["runs"][(crop, workers)]
    parts = torch.split(run["draws"], run["sizes"])
    got = sampled(gold, case, crop, workers, len(parts))
    assert len(parts) == 5  # 2.5 epochs of 6 samples in batches of 4
    for k, (want, b) in enumerate(zip(parts, got)):
        ind, pos, seeds = b[:3]
        assert ind.tolist() == want[:, 0].tolist(), (k, "ind")
        assert pos.tolist() == want[:, 1].tolist(), (k, "ind_pos")
        assert seeds.tolist() == want[:, 2].tolist(), (k, "seed")
        if crop == "random":
            B = ind.size
            windows = b[3]
            assert windows[:B].tolist() == want[:, 3:7].tolist(), (k, "windows")
            assert windows[B:].tolist() == want[:, 7:11].tolist(), (k, "windows_pos")
        else:
            assert len(b) == 3 and not want[:, 3:].any()


def test_square_rows_draw_nothing(gold):
    """A row whose Resize(res) output is res x res draws no window (the fixture's 16 x 16 image at res 32), and its
    window is (0, 0): the draws after it follow the stream untouched, as the reference's."""
    sizes = row_sizes(gold["cases"]["cocostuff27_32"])
    assert tuple(sizes[0]) == (32, 32, 32, 32)
    g = torch.Generator()
    assert D._window(g, 123, sizes[0], 32) == (0, 0, 0, 0)
    after = torch.randint(0, 1000, (4,), generator=g)
    g2 = torch.Generator()
    g2.manual_seed(123)
    assert torch.equal(after, torch.randint(0, 1000, (4,), generator=g2))


def test_window_is_torchvision_random_crop():
    """_window restates RandomCrop.get_params under the class's manual_seed, for the image then the label."""
    import torchvision.transforms as T
    for seed, size in ((5, (32, 75, 32, 75)), (9, (70, 32, 40, 32)), (2 ** 31 - 2, (32, 33, 64, 32))):
        with torch.random.fork_rng(devices=[]):
            torch.manual_seed(seed)
            top, left, _, _ = T.RandomCrop.get_params(torch.empty(1, size[0], size[1]), (32, 32))
            torch.manual_seed(seed)
            ltop, lleft, _, _ = T.RandomCrop.get_params(torch.empty(1, size[2], size[3]), (32, 32))
        assert D._window(torch.Generator(), seed, size, 32) == (top, left, ltop, lleft)


def test_global_generators_do_not_move(gold):
    np.random.seed(3)
    random.seed(3)
    torch.manual_seed(3)
    states = (np.random.get_state()[1].copy(), random.getstate(), torch.get_rng_state().clone())
    sampled(gold, "cityscapes_30", "random", 0, 5)
    sampled(gold, "cityscapes_30", "random", 2, 5)
    assert (np.random.get_state()[1] == states[0]).all()
    assert random.getstate() == states[1]
    assert torch.equal(torch.get_rng_state(), states[2])


@pytest.mark.parametrize("world_size", [2, 3])
def test_distributed_windows(gold, world_size):
    """Each rank's share of DistributedSampler's order, every sample with its window: the windows of a sample depend on
    its seed and row alone, so the ranks' windows are those `_window` gives each (ind, seed) of their share."""
    from torch.utils.data import DistributedSampler
    case = gold["cases"]["directory_32"]
    sizes = row_sizes(case)
    nns = gold["nns"].numpy()
    for rank in range(world_size):
        sampler = D.Sampler(nns, 2, gold["num_neighbors"], gold["seed"], 0, rank=rank, world_size=world_size, res=32,
                            sizes=sizes)
        ref = DistributedSampler(list(range(nns.shape[0])), num_replicas=world_size, rank=rank, shuffle=True,
                                 seed=gold["seed"])
        for epoch in range(2):
            ref.set_epoch(epoch)
            batches = list(next(sampler))
            assert np.concatenate([b[0] for b in batches]).tolist() == list(ref)
            for ind, pos, _, windows in batches:
                B = ind.size
                for j, w in enumerate(windows):
                    row = ind[j] if j < B else pos[j - B]
                    sz = sizes[row]
                    assert 0 <= w[0] <= sz[0] - 32 and 0 <= w[1] <= sz[1] - 32
                    assert 0 <= w[2] <= sz[2] - 32 and 0 <= w[3] <= sz[3] - 32


def test_refusals_before_the_device():
    with pytest.raises(ValueError, match="not a training set class"):
        D.ResidentDataset(4, 32, kind="cityscapes")
    with pytest.raises(ValueError, match="EvalSet.potsdam"):
        D.ResidentDataset(4, 32, kind="potsdam")
    with pytest.raises(ValueError, match="crop"):
        D.ResidentDataset.crops("/nonexistent", "cityscapes", "five", 0.5, "train", 32, crop="random")


def test_bad_crop_is_refused_before_the_device():
    with pytest.raises(ValueError, match="crop"):
        D.ResidentDataset(4, 32, "directory", crop="left")
