"""CPU: the host half of the loader frames and labels (stego_b200.frames) against Pillow, torchvision and the
reference's own loaders (tests/golden/frames.pt, oracle/make_golden_frames.py).

  * oracle/frames_oracle.py reproduces the fixture bit for bit: frames, and the labels of Coco (27 classes, 3 classes,
    exclude_things), CityscapesSeg and DirectoryDataset;
  * the index tables are Pillow's: pillow_nearest_index equals Pillow's NEAREST resize of an index image for thousands of
    size pairs up to 8000 px and ratios from 1:1000 to 1000:1, and the tables of every fixture case gather the
    fixture's frames;
  * output sizes and crop offsets are torchvision's;
  * label_lut tables give the fixture's remaps;
  * bad arguments are refused before anything is staged or launched, by the Python layer and by the C entries.
"""
import os
import sys

import numpy as np
import pytest
import torch
from PIL import Image
from torchvision.transforms import functional as TF

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import frames_oracle as FO  # noqa: E402

from stego_b200 import _lib, frames  # noqa: E402

GOLD = torch.load(os.path.join(ROOT, "tests", "golden", "frames.pt"))
CASES = GOLD["cases"]


def coco_luts():
    """The three Coco remaps as label_lut tables built from the data set's fine_to_coarse (fixture)."""
    coco = GOLD["coco"]
    t27 = frames.label_lut(coco["fine_to_coarse"])
    t3 = torch.full((256,), -1, dtype=torch.int64)
    for i, c in enumerate(coco["cocostuff3_coarse_classes"]):
        t3[t27 == c] = i
    return {"coco27": t27, "coco3": t3, "cocostuff": t27 - coco["first_stuff_index"]}


def all_luts():
    luts = coco_luts()
    luts["cityscapes"] = frames.label_lut({i: i - 7 for i in range(7, 256)}, ignore_from=256, default=-1)
    luts["directory"] = None
    return luts


def _want(case, key):
    """The fixture's label map as int64 [res, res] (DirectoryDataset keeps ToTargetTensor's leading 1)."""
    return case[key].numpy().astype(np.int64).reshape(case["res"], case["res"])


def _pillow_axis(n_in, n_out):
    a = np.arange(n_in, dtype=np.int32)[None, :]
    return np.asarray(Image.fromarray(a, mode="I").resize((n_out, 1), Image.NEAREST))[0].astype(np.int64)


def test_oracle_reproduces_reference_fixture():
    for c in CASES:
        img, lab, res, crop = c["image"].numpy(), c["label"].numpy(), c["res"], c["crop"]
        got = FO.frame(img, res, crop)
        assert got.dtype == np.float32 and np.array_equal(got.view(np.int32), c["frame"].numpy().view(np.int32))
        tables = dict(coco27=FO.coco_table(GOLD["coco"], "27"), coco3=FO.coco_table(GOLD["coco"], "3"),
                      cocostuff=FO.coco_table(GOLD["coco"], "stuff"), cityscapes=FO.cityscapes_table(), directory=None)
        for key, table in tables.items():
            assert np.array_equal(FO.label(lab, res, crop, table), _want(c, key)), (key, c["H"], c["W"])


def test_fixture_covers_the_edges():
    """The fixture holds a size where the closed form disagrees with Pillow and both round-half-even crops."""
    sides = {(c["res"], max(frames.output_size(c["H"], c["W"], c["res"], c["crop"]))) for c in CASES if c["crop"]}
    assert any(long == res + 1 for res, long in sides) and any(long == res + 3 for res, long in sides)
    closed = lambda n_in, n_out: np.minimum(np.floor((np.arange(n_out) + .5) * n_in / n_out), n_in - 1)
    disagree = 0
    for c in CASES:
        oh, ow = frames.output_size(c["H"], c["W"], c["res"], c["crop"])
        disagree += any(not np.array_equal(frames.pillow_nearest_index(n, o), closed(n, o))
                        for n, o in ((c["H"], oh), (c["W"], ow)))
    assert disagree >= 1


def test_tables_gather_the_fixture():
    for c in CASES:
        rows, cols = frames.index_tables(c["H"], c["W"], c["res"], c["crop"])
        assert rows.dtype == np.int32 and rows.shape == cols.shape == (c["res"],)
        img = c["image"].numpy()
        g = img[np.clip(rows, 0, None)][:, np.clip(cols, 0, None)].astype(np.float32)
        g[rows < 0] = 0
        g[:, cols < 0] = 0
        want = (g.transpose(2, 0, 1) / np.float32(255) - FO.MEAN[:, None, None]) / FO.STD[:, None, None]
        assert np.array_equal(want.view(np.int32), c["frame"].numpy().view(np.int32))


def _size_pairs():
    rng = np.random.default_rng(7)
    pairs = [(2, 7), (8, 7), (14, 3203), (1, 1), (1, 8000), (8000, 1), (8000, 8000), (7999, 8000), (8000, 7999),
             (8, 8000), (8000, 8), (3, 3000), (3000, 3), (320, 321), (321, 320), (4000, 320), (3000, 427)]
    for _ in range(2500):
        pairs.append(tuple(int(x) for x in rng.integers(1, 8001, 2)))
    for _ in range(500):  # extreme ratios, 1:1000 to 1000:1
        small = int(rng.integers(1, 9))
        big = int(min(8000, small * rng.integers(100, 1001)))
        pairs.append((small, big) if rng.random() < 0.5 else (big, small))
    return pairs


def test_pillow_nearest_index_equals_pillow():
    pairs = _size_pairs()
    assert len(pairs) >= 3000
    for n_in, n_out in pairs:
        got = frames.pillow_nearest_index(n_in, n_out)
        assert np.array_equal(got, _pillow_axis(n_in, n_out)), (n_in, n_out)
        assert got.min() >= 0  # no position reaches n_in at these sizes; the -1 branch is Pillow's fill


def test_pillow_rows_and_label_mode():
    """The same index along y, and on an 8-bit "L" image (the label maps' mode) along both axes."""
    rng = np.random.default_rng(8)
    for _ in range(40):
        h, w = (int(x) for x in rng.integers(1, 256, 2))
        oh, ow = (int(x) for x in rng.integers(1, 700, 2))
        ys, xs = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
        im = Image.fromarray(((ys * 7 + xs * 13) % 256).astype(np.uint8), mode="L").resize((ow, oh), Image.NEAREST)
        r, c = frames.pillow_nearest_index(h, oh), frames.pillow_nearest_index(w, ow)
        assert np.array_equal(np.asarray(im), ((r[:, None] * 7 + c[None, :] * 13) % 256).astype(np.uint8)), (h, w, oh, ow)


def test_output_size_and_crop_equal_torchvision():
    from torchvision.transforms.functional import _compute_resized_output_size
    rng = np.random.default_rng(9)
    sizes = [(1, 1), (320, 320), (321, 320), (323, 320), (480, 640), (640, 480), (1024, 2048), (3000, 4000), (1, 8000)]
    sizes += [tuple(int(x) for x in rng.integers(1, 5000, 2)) for _ in range(400)]
    for h, w in sizes:
        for res in (32, 224, 320):
            assert list(frames.output_size(h, w, res, "center")) == _compute_resized_output_size((h, w), [res])
            assert frames.output_size(h, w, res, None) == (res, res)
            oh, ow = frames.output_size(h, w, res, "center")
            if oh * ow > 4_000_000:
                continue
            grid = torch.arange(oh * ow, dtype=torch.int32).view(1, oh, ow)
            top_left = int(TF.center_crop(grid, [res])[0, 0, 0])
            assert frames.crop_offsets(oh, ow, res) == divmod(top_left, ow), (h, w, res)
    assert frames.crop_offsets(321, 320, 320) == (0, 0) and frames.crop_offsets(323, 320, 320) == (2, 0)


def test_label_lut_reproduces_fixture_remaps():
    luts = all_luts()
    for c in CASES:
        ids = FO.label(c["label"].numpy(), c["res"], c["crop"])
        for key, lut in luts.items():
            got = ids if lut is None else lut.numpy()[ids]
            assert np.array_equal(got, _want(c, key)), key
    t = frames.label_lut({0: 5, 3: 9}, ignore_from=200, default=-4)
    assert t.dtype == torch.int64 and t.shape == (256,)
    assert t[0] == 5 and t[3] == 9 and t[1] == -4 and t[199] == -4 and (t[200:] == -1).all()
    with pytest.raises(ValueError, match="ignore_from"):
        frames.label_lut({}, ignore_from=257)


@pytest.fixture
def no_launch(monkeypatch):
    """Fails the test if the library is reached or a pinned buffer is allocated."""
    def never(*a, **k):
        raise AssertionError("reached the library / staging for a call that should have been refused")
    monkeypatch.setattr(frames._lib, "load", never)
    monkeypatch.setattr(frames, "_stage", never)
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)


def test_bad_arguments_raise_before_any_launch(no_launch):
    rgb = np.zeros((8, 9, 3), np.uint8)
    lab = np.zeros((8, 9), np.uint8)
    bad_frames = [
        ((ValueError, "images"), dict(images=[], res=32)),
        ((ValueError, "float32"), dict(images=[rgb.astype(np.float32)], res=32)),
        ((ValueError, "torch.int64"), dict(images=[torch.zeros(8, 9, 3, dtype=torch.int64)], res=32)),
        ((ValueError, "shape"), dict(images=[np.zeros((8, 9, 4), np.uint8)], res=32)),
        ((ValueError, "shape"), dict(images=[lab], res=32)),
        ((ValueError, "0 x 9"), dict(images=[np.zeros((0, 9, 3), np.uint8)], res=32)),
        ((TypeError, "list"), dict(images=rgb, res=32)),
        ((TypeError, "not an array"), dict(images=[[1, 2, 3]], res=32)),
        ((ValueError, "res"), dict(images=[rgb], res=0)),
        ((ValueError, "res"), dict(images=[rgb], res=32.0)),
        ((ValueError, "crop"), dict(images=[rgb], res=32, crop="random")),
    ]
    for (exc, match), kw in bad_frames:
        with pytest.raises(exc, match=match):
            frames.load_frames(**kw)
    bad_labels = [
        ((ValueError, "images"), dict(labels=[], res=32)),
        ((ValueError, "shape"), dict(labels=[rgb], res=32)),
        ((ValueError, "int32"), dict(labels=[lab.astype(np.int32)], res=32)),
        ((ValueError, "256"), dict(labels=[lab], res=32, lut=torch.zeros(255, dtype=torch.int64))),
        ((ValueError, "256"), dict(labels=[lab], res=32, lut=np.zeros(256, np.float32))),
        ((ValueError, "256"), dict(labels=[lab], res=32, lut=np.zeros((2, 128), np.int64))),
    ]
    for (exc, match), kw in bad_labels:
        with pytest.raises(exc, match=match):
            frames.load_labels(**kw)


def test_cpu_only_calls_raise(monkeypatch, no_launch):
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(RuntimeError, match="CUDA"):
        frames.load_frames([np.zeros((4, 4, 3), np.uint8)], 8)
    with pytest.raises(RuntimeError, match="CUDA"):
        frames.load_labels([np.zeros((4, 4), np.uint8)], 8, lut=frames.label_lut({}))


def test_entries_declared_and_exported():
    protos = _lib.header_prototypes()
    assert protos["stego_frames_rgb8"][1] == ["const void*", "const void*", "long long", "long long", "int", "int",
                                             "float", "float", "float", "float", "float", "float", "float*", "void*"]
    assert protos["stego_labels_u8"][1] == ["const void*", "const void*", "long long", "long long", "int", "int",
                                           "const long long*", "long long*", "void*"]
    lib = _lib.load()
    lib.stego_frames_rgb8, lib.stego_labels_u8  # noqa: B018  (AttributeError if not exported)


def _staging(records, table, images_bytes):
    """A staging buffer laid out as the header describes: records, int32 tables, image bytes."""
    head = np.asarray(records, np.int64).reshape(-1).view(np.uint8)
    tab = np.asarray(table, np.int32).view(np.uint8)
    return np.concatenate([head, tab, np.zeros(images_bytes, np.uint8)])


def test_entries_refuse_bad_staging_without_a_launch():
    """Each bad record / table / size is refused by the C entry's host-side check (status -1, nothing launched).  The
    buffer's host address stands in for the device copy: no CUDA call is reached."""
    lib = _lib.load()
    res, H, W = 4, 3, 5
    table = [0, 1, 2, 2, 0, 1, 3, 4]  # rows then columns
    data = 32 + 4 * len(table)
    good = [data, H, W, 0]

    def call(records, tbl=table, nbytes=None, B=1, r=res, lut_entry=False, extra=H * W * 3):
        buf = _staging(records, tbl, extra)
        n = buf.size if nbytes is None else nbytes
        p = buf.ctypes.data
        launches = _lib.launch_count()
        if lut_entry:
            rc = lib.stego_labels_u8(p, p, n, len(tbl), B, r, 0, p, 0)
        else:
            rc = lib.stego_frames_rgb8(p, p, n, len(tbl), B, r, .5, .5, .5, .2, .2, .2, p, 0)
        assert _lib.launch_count() == launches
        return rc, _lib.last_error()

    bad = [
        (dict(records=[data + 1, H, W, 0]), "outside"),           # image runs past the buffer
        (dict(records=[8, H, W, 0]), "outside"),                  # image overlaps the records and tables
        (dict(records=[data, 0, W, 0]), "0 x 5"),
        (dict(records=[data, H, W, 1]), "tables start"),
        (dict(records=good, tbl=[0, 1, 2, 3, 0, 1, 3, 4]), "row 3"),   # row index H
        (dict(records=good, tbl=[0, 1, 2, 2, 0, 1, 3, 5]), "column 5"),
        (dict(records=good, tbl=[0, 1, 2, -2, 0, 1, 3, 4]), "row -2"),
        (dict(records=good, B=0), "B=0"),
        (dict(records=good, r=0), "res=0"),
        (dict(records=good, nbytes=20), "staging bytes"),
        (dict(records=[data, H, W, 0], lut_entry=True, extra=H * W - 1), "outside"),
    ]
    for kw, msg in bad:
        rc, err = call(**kw)
        assert rc == -1 and msg in err, (kw, rc, err)
    assert lib.stego_frames_rgb8(None, None, 100, 8, 1, 4, .5, .5, .5, .2, .2, .2, None, None) == -1
