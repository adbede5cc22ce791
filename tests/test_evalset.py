"""CPU: the resident evaluation sets (stego_b200.evalset) against the reference's classes in tests/golden/evalset.pt
(oracle/make_golden_evalset.py): each class's file listing and order, the label tables, DistributedSampler's shards
with their padding, and the refusals that happen before anything reaches the device."""
import os
import sys
import zlib

import numpy as np
import pytest
import torch
from scipy.io import savemat
from torch.utils.data import DistributedSampler

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from stego_b200 import evalset as E  # noqa: E402
from stego_b200.dataset import shard  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden", "evalset.pt")
KINDS = ("cocostuff27", "cocostuff15", "cocostuff3", "cityscapes", "potsdam", "potsdamraw")


def load_gold(path=GOLD):
    """The fixture with its compact fields expanded: PotsdamRaw's names, the tables as int64, each case's masks
    unpacked to bool rows and its img rows as the reference's fp32 values (values[c][byte])."""
    g = torch.load(path)
    g["raw"]["names"] = zlib.decompress(g["raw"]["names_zlib"]).decode()
    g["tables"] = {k: v.to(torch.int64) for k, v in g["tables"].items()}
    values = g["values"]
    for key, case in g["cases"].items():
        shape = case["mask_shape"]
        bits = np.unpackbits(case["mask"].numpy(), count=int(np.prod(shape)))
        case["mask"] = torch.from_numpy(bits.reshape(shape).astype(bool))
        frames = g["frames"][int(key.rsplit("_", 1)[1])][case["img_index"]].to(torch.int64)
        case["img"] = torch.stack([values[c][frames[:, c]] for c in range(3)], 1)
    return g


def write_tree(gold, root: str) -> None:
    """The fixture's file tree under `root`: Coco, Cityscapes and Potsdam as stored, PotsdamRaw's tiles from its pool."""
    for rel, data in gold["tree"].items():
        path = os.path.join(root, rel)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        with open(path, "wb") as f:
            f.write(data)
    raw = gold["raw"]
    base = os.path.join(root, "potsdamraw", "processed")
    for sub in ("imgs", "gt"):
        os.makedirs(os.path.join(base, sub), exist_ok=True)
    for name, e in zip(raw["names"].split("\n"), raw["tile_of"].tolist()):
        entry = raw["pool"][e]
        with open(os.path.join(base, "imgs", name), "wb") as f:
            f.write(entry["img"])
        if entry["gt"] is not None:
            with open(os.path.join(base, "gt", name), "wb") as f:
                f.write(entry["gt"])


def listing(root: str, kind: str) -> list:
    if kind.startswith("cocostuff"):
        images, labels = E.coco_files(root, kind, "val")
    elif kind == "cityscapes":
        images, labels = E.cityscapes_files(root, "val")
    elif kind == "potsdam":
        images, labels = E.potsdam_files(root, "val")
    else:
        images, labels = E.potsdamraw_files(root)
    assert len(images) == len(labels)
    return images, labels


def expected_rows(gold, kind: str, res: int, rel_paths: list) -> torch.Tensor:
    """The fixture row of each store index, matched by image path (CityscapesSeg's order is the file system's)."""
    case = gold["cases"][f"{kind}_{res}"]
    if kind == "potsdamraw":
        return gold["raw"]["tile_of"].to(torch.int64)
    where = {p: i for i, p in enumerate(case["paths"])}
    return case["row_of"][[where[p] for p in rel_paths]]


@pytest.fixture(scope="module")
def gold():
    return load_gold()


@pytest.fixture(scope="module")
def tree(gold, tmp_path_factory):
    root = str(tmp_path_factory.mktemp("evalset_tree"))
    write_tree(gold, root)
    return root


@pytest.mark.parametrize("kind", ["cocostuff27", "cocostuff15", "cocostuff3", "potsdam"])
def test_listing_order_matches_reference(gold, tree, kind):
    images, labels = listing(tree, kind)
    rel = [os.path.relpath(p, tree) for p in images]
    assert rel == gold["cases"][f"{kind}_32"]["paths"]
    if kind.startswith("cocostuff"):
        assert [os.path.relpath(p, tree) for p in labels] == [
            p.replace("images", "annotations").replace(".jpg", ".png") for p in rel]
    else:
        assert [os.path.relpath(p, tree) for p in labels] == [p.replace("/imgs/", "/gt/") for p in rel]


def test_coco_subsets():
    assert [E.coco_subset(k, "val") for k in ("cocostuff27", "cocostuff15", "cocostuff3")] == [7, 7, 6]
    assert [E.coco_subset(k, "train") for k in ("cocostuff27", "cocostuff15", "cocostuff3")] == [None, 7, 6]


def test_potsdamraw_listing(gold, tree):
    images, labels = listing(tree, "potsdamraw")
    names = gold["raw"]["names"].split("\n")
    assert len(names) == 38 * 15 * 15
    assert [os.path.basename(p) for p in images] == names
    assert [os.path.relpath(p, tree) for p in labels] == [os.path.join("potsdamraw", "processed", "gt", n)
                                                          for n in names]


def test_cityscapes_listing_is_torchvisions(gold, tree):
    from torchvision.datasets import Cityscapes
    images, labels = listing(tree, "cityscapes")
    tv = Cityscapes(os.path.join(tree, "cityscapes"), "val", mode="fine", target_type="semantic")
    assert images == tv.images
    assert labels == [t[0] for t in tv.targets]
    assert sorted(os.path.relpath(p, tree) for p in images) == sorted(gold["cases"]["cityscapes_32"]["paths"])


@pytest.mark.parametrize("kind", KINDS)
def test_label_tables_match_reference(gold, kind):
    got = E.label_table(kind, gold["fine_to_coarse"] if kind.startswith("cocostuff") else None)
    assert got.dtype == torch.int64 and torch.equal(got, gold["tables"][kind])


def test_fixture_values_are_the_loader_normalisation(gold):
    """The reference's transform of every byte is ToTensor's div then Normalize, in fp32 (frames.MEAN / STD)."""
    from stego_b200.frames import MEAN, STD
    x = torch.arange(256, dtype=torch.float32) / 255
    want = torch.stack([(x - m) / s for m, s in zip(MEAN, STD)])
    assert gold["values"].dtype == torch.float32 and torch.equal(gold["values"], want)


def test_fixture_covers_every_mask_rule(gold):
    dtypes = {k: (c["label_dtype"], c["mask_dtype"], tuple(c["mask"].shape[1:])) for k, c in gold["cases"].items()}
    assert dtypes["cocostuff27_32"] == ("int64", "bool", (32, 32))
    assert dtypes["cityscapes_30"] == ("int64", "bool", (1, 30, 30))
    assert dtypes["potsdam_32"] == ("int64", "float32", (32, 32))
    assert dtypes["potsdamraw_30"] == ("int64", "float32", (30, 30))


@pytest.mark.parametrize("world_size", [1, 2, 3, 4, 7])
@pytest.mark.parametrize("n", [1, 2, 5, 6, 13])
def test_shards_are_distributed_samplers(n, world_size):
    for rank in range(world_size):
        want = list(DistributedSampler(range(n), num_replicas=world_size, rank=rank, shuffle=False))
        assert shard(list(range(n)), rank, world_size) == want


def test_read_mat(tmp_path):
    rng = np.random.default_rng(0)
    img = rng.integers(0, 256, (9, 7, 4), dtype=np.uint8)
    gt = rng.integers(0, 256, (9, 7), dtype=np.uint8)
    savemat(tmp_path / "a.mat", {"img": img})
    savemat(tmp_path / "g.mat", {"gt": gt})
    got_img, got_gt = E.read_mat(str(tmp_path / "a.mat"), str(tmp_path / "g.mat"))
    assert got_img.flags["C_CONTIGUOUS"] and np.array_equal(got_img, img[..., :3]) and np.array_equal(got_gt, gt)
    _, missing = E.read_mat(str(tmp_path / "a.mat"), str(tmp_path / "none.mat"))
    assert missing.dtype == np.uint8 and missing.shape == (9, 7) and (missing == 255).all()


@pytest.mark.parametrize("what", ["float_img", "uint16_img", "two_channels", "int32_gt", "float_gt"])
def test_read_mat_refuses_other_dtypes(tmp_path, what):
    img = np.zeros((4, 5, 3), dtype=np.uint8)
    gt = np.zeros((4, 5), dtype=np.uint8)
    if what == "float_img":
        img = img.astype(np.float64)
    elif what == "uint16_img":
        img = img.astype(np.uint16)
    elif what == "two_channels":
        img = img[..., :2]
    elif what == "int32_gt":
        gt = gt.astype(np.int32)
    else:
        gt = gt.astype(np.float32)
    savemat(tmp_path / "a.mat", {"img": img})
    savemat(tmp_path / "g.mat", {"gt": gt})
    with pytest.raises(ValueError, match="uint8"):
        E.read_mat(str(tmp_path / "a.mat"), str(tmp_path / "g.mat"))


@pytest.mark.parametrize("kind,match", [("cropped", "kind='cropped'"), ("directory", "ResidentDataset"),
                                        ("voc", "one of"), ("cocostuff27", "fine_to_coarse")])
def test_refuses_bad_kind(kind, match):
    with pytest.raises(ValueError, match=match):
        E.EvalSet(4, 32, kind)


@pytest.mark.parametrize("args,match", [((4, 32, "cityscapes", "cpu"), "location"), ((0, 32, "potsdam"), "n=0"),
                                        ((4, 0, "potsdam"), "res=0"), ((4, 8193, "potsdam"), "res=8193"),
                                        ((4, 32.0, "potsdam"), "res=32.0"), ((True, 32, "potsdam"), "n=True")])
def test_refuses_bad_sizes_and_location(args, match):
    with pytest.raises(ValueError, match=match):
        E.EvalSet(*args)


def test_refuses_bad_tables():
    with pytest.raises(ValueError, match="0..254"):
        E.label_table("cocostuff15", {0: 300})
    with pytest.raises(ValueError, match="fine_to_coarse"):
        E.label_table("cocostuff3", [1, 2])


def test_refuses_bad_splits(tree):
    with pytest.raises(ValueError, match="image_set='test'"):
        E.coco_files(tree, "cocostuff27", "test")
    with pytest.raises(ValueError, match="kind='cityscapes'"):
        E.coco_files(tree, "cityscapes", "val")
    with pytest.raises(ValueError, match="image_set='train_extra'"):
        E.cityscapes_files(tree, "train_extra")
    with pytest.raises(ValueError, match="missing"):
        E.cityscapes_files(tree, "train")
    with pytest.raises(ValueError, match="image_set='test'"):
        E.potsdam_files(tree, "test")


def test_refuses_count_mismatch_and_empty_listing():
    with pytest.raises(ValueError, match="2 images but 1 label files"):
        E.EvalSet._from_files(["a", "b"], ["a"], "pil", 32, "cityscapes", "cuda", 4, 0)
    with pytest.raises(ValueError, match="names no files"):
        E.EvalSet._from_files([], [], "pil", 32, "cityscapes", "cuda", 4, 0)


def _unbuilt(n=5, count=5):
    """An EvalSet's bookkeeping without its memory: the argument checks of frames() run before any launch."""
    s = E.EvalSet.__new__(E.EvalSet)
    s.n, s.count, s.res, s.kind = n, count, 32, "potsdam"
    return s


@pytest.mark.parametrize("kw,match", [(dict(batch_size=0), "batch_size=0"), (dict(dtype=torch.float16), "dtype"),
                                      (dict(rank=2, world_size=2), "rank=2"), (dict(rank=-1), "rank=-1"),
                                      (dict(world_size=0), "world_size=0")])
def test_frames_refusals(kw, match):
    kw = dict(dict(batch_size=2), **kw)
    with pytest.raises(ValueError, match=match):
        next(_unbuilt().frames(**kw))


def test_frames_refuses_a_partial_store():
    with pytest.raises(ValueError, match="holds 3 of its 5"):
        next(_unbuilt(5, 3).frames(2))
