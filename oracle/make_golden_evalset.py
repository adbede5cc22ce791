"""Generate tests/golden/evalset.pt from the REAL reference validation loader: ContrastiveSegDataset (src/data.py:419-565)
with crop_type=None over Coco (cocostuff27, cocostuff15, cocostuff3), CityscapesSeg, Potsdam and PotsdamRaw, read with
get_transform(res, ., "center") under DataLoader(batch_size=3, shuffle=False), at res 32 and 30, with mask=True and
mask=False, on the CPU.

    STEGO_REFERENCE_SRC=<reference checkout>/src python oracle/make_golden_evalset.py

The input is a seeded synthetic file tree in each class's layout: Coco's curated id lists (list 7 and list 6 in
different orders), images (some grayscale, the .jpg names holding PNG bytes: PIL decodes by content, losslessly) and
annotations (one palette PNG); Cityscapes leftImg8bit / gtFine labelIds in two cities; Potsdam's split file and .mat
tiles written with scipy.io.savemat (4-channel uint8 img, one tile without gt); PotsdamRaw's 38 x 15 x 15 processed
tiles, drawn from a pool of 4 tiles (one without gt) so that the tree stays small.  Sizes are mixed, label bytes are
uniform over 0..255 (outside every class's map), and every class has one 16 x 16 tile whose label is every byte once.

Stored:
  * tree: {relative path: file bytes} for Coco, Cityscapes and Potsdam; raw: PotsdamRaw's pool bytes, the pool entry
    of each tile (uint8, which is also the tile's row) and the reference's file names joined by newlines, zlib-
    compressed (names_zlib) (tests write the same tree);
  * values: fp32 [3, 256], the value the reference's image transform gives byte b in channel c (get_transform(16,
    False, "center") of a 16 x 16 image holding every byte once); frames[res]: uint8 [U, 3, res, res], the reference's
    img rows of every distinct image as the bytes whose values they are.  Each row is checked here to be exactly
    values[c][byte], so values[c][frames[res]] is the reference's fp32 row bit for bit, at a quarter of its size, and
    an image shared by several cases (Coco's kinds) is kept once;
  * fine_to_coarse: Coco's own table; tables: per kind the label the reference returns for each byte 0..255 (int16,
    read off the all-bytes tile at res 32);
  * cases[f"{kind}_{res}"]: paths (each index's image path relative to the root, the reference's order), row_of (index
    -> row; both None for potsdamraw, kept in raw), img_index (row -> frames[res] entry), and the reference's rows of
    label (int16, with label_dtype) and mask (bits packed by np.packbits, with mask_dtype and mask_shape, the rows'
    shape).  Every batch of every run (mask on / off) is checked here to equal the rows gathered at its
    ind, and the mask=False batches to carry no mask.
"""
from __future__ import annotations

import io
import os
import zlib
import sys
import tempfile
from types import SimpleNamespace

import numpy as np
import torch
from PIL import Image
from scipy.io import savemat

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import reference_shim  # noqa: E402
from make_golden_frames import _import_reference_loaders  # noqa: E402

OUT = os.path.join(HERE, "..", "tests", "golden", "evalset.pt")
RESOLUTIONS = (32, 30)
BATCH = 3
KINDS = ("cocostuff27", "cocostuff15", "cocostuff3", "cityscapes", "potsdam", "potsdamraw")
RAW_POOL = 4


def _png(arr, mode=None) -> bytes:
    buf = io.BytesIO()
    Image.fromarray(arr, mode=mode).save(buf, format="PNG")
    return buf.getvalue()


def _mat(key, arr) -> bytes:
    buf = io.BytesIO()
    savemat(buf, {key: arr})
    return buf.getvalue()


def _sample(rng, k):
    """Image H x W x 3 and label H x W; sample 0 is the 16 x 16 tile whose label is every byte once."""
    if k == 0:
        H = W = 16
        lab = np.arange(256, dtype=np.uint8).reshape(16, 16)
    else:
        H, W = int(rng.integers(12, 70)), int(rng.integers(12, 70))
        lab = rng.integers(0, 256, (H, W), dtype=np.uint8)
    return rng.integers(0, 256, (H, W, 3), dtype=np.uint8), lab


def tree():
    """{relative path: bytes} of the Coco, Cityscapes and Potsdam layouts, and the PotsdamRaw pool."""
    rng = np.random.default_rng(2025)
    files = {}
    # Coco: 6 ids; list 7 names 5 of them, list 6 four in another order
    ids = [f"00000000{k:04d}" for k in (139, 285, 632, 724, 776, 802)]
    for k, img_id in enumerate(ids):
        img, lab = _sample(rng, k)
        if k == 2:
            files[f"cocostuff/images/val2017/{img_id}.jpg"] = _png(img[..., 0], "L")  # grayscale, converted to RGB
        else:
            files[f"cocostuff/images/val2017/{img_id}.jpg"] = _png(img)
        if k == 3:  # a palette annotation: the indices are the label bytes
            pal = Image.frombytes("P", (lab.shape[1], lab.shape[0]), lab.tobytes())
            pal.putpalette([v for i in range(256) for v in (255 - i, i, i)])
            buf = io.BytesIO()
            pal.save(buf, format="PNG")
            files[f"cocostuff/annotations/val2017/{img_id}.png"] = buf.getvalue()
        else:
            files[f"cocostuff/annotations/val2017/{img_id}.png"] = _png(lab, "L")
    files["cocostuff/curated/val2017/Coco164kFull_Stuff_Coarse_7.txt"] = "\n".join(ids[:5]).encode() + b"\n"
    files["cocostuff/curated/val2017/Coco164kFew_Stuff_6.txt"] = "\n".join([ids[5], ids[0], ids[3], ids[1]]).encode()
    # Cityscapes: two cities
    for k, (city, num) in enumerate((("aachen", 19), ("bonn", 3), ("aachen", 7), ("bonn", 12), ("aachen", 1))):
        img, lab = _sample(rng, k)
        stem = f"{city}_{num:06d}_000019"
        files[f"cityscapes/leftImg8bit/val/{city}/{stem}_leftImg8bit.png"] = _png(img)
        files[f"cityscapes/gtFine/val/{city}/{stem}_gtFine_labelIds.png"] = _png(lab, "L")
    # Potsdam: the val split, one tile without gt
    pids = ["top_potsdam_2_10_RGBIR_7", "top_potsdam_2_10_RGBIR_12", "top_potsdam_3_11_RGBIR_0",
            "top_potsdam_7_8_RGBIR_3", "top_potsdam_6_9_RGBIR_21"]
    for k, pid in enumerate(pids):
        img, lab = _sample(rng, k)
        ir = rng.integers(0, 256, img.shape[:2] + (1,), dtype=np.uint8)
        files[f"potsdam/imgs/{pid}.mat"] = _mat("img", np.concatenate([img, ir], 2))
        if k != 3:
            files[f"potsdam/gt/{pid}.mat"] = _mat("gt", lab)
    files["potsdam/labelled_test.txt"] = "\n".join(pids).encode() + b"\n"
    pool = []
    for k in range(RAW_POOL):
        img, lab = _sample(rng, k)
        ir = rng.integers(0, 256, img.shape[:2] + (1,), dtype=np.uint8)
        pool.append(dict(img=_mat("img", np.concatenate([img, ir], 2)), gt=None if k == 2 else _mat("gt", lab)))
    n_raw = 38 * 15 * 15
    raw_of = [(7 * t + 3) % RAW_POOL for t in range(n_raw)]
    raw_of[0] = 0  # the first tile is the all-bytes one
    return files, dict(pool=pool, tile_of=raw_of)


def write_tree(root: str, files: dict, raw: dict) -> None:
    for rel, data in files.items():
        path = os.path.join(root, rel)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        with open(path, "wb") as f:
            f.write(data)
    base = os.path.join(root, "potsdamraw", "processed")
    os.makedirs(os.path.join(base, "imgs"), exist_ok=True)
    os.makedirs(os.path.join(base, "gt"), exist_ok=True)
    t = 0
    for i in range(38):
        for h in range(15):
            for w in range(15):
                entry = raw["pool"][raw["tile_of"][t]]
                with open(os.path.join(base, "imgs", f"{i}_{h}_{w}.mat"), "wb") as f:
                    f.write(entry["img"])
                if entry["gt"] is not None:
                    with open(os.path.join(base, "gt", f"{i}_{h}_{w}.mat"), "wb") as f:
                        f.write(entry["gt"])
                t += 1


def run(data, utils, root, kind, res, mask):
    from torch.utils.data import DataLoader
    cfg = SimpleNamespace(model_type="vit_small", res=res, dir_dataset_name=None, dir_dataset_n_classes=None,
                          crop_ratio=0.5, crop_type=None)
    ds = data.ContrastiveSegDataset(pytorch_data_dir=root, dataset_name=kind, crop_type=None, image_set="val",
                                    transform=utils.get_transform(res, False, "center"),
                                    target_transform=utils.get_transform(res, True, "center"), cfg=cfg, mask=mask)
    inner = ds.dataset
    if kind == "cityscapes":
        paths = list(inner.inner_loader.images)
    elif kind.startswith("cocostuff"):
        paths = list(inner.image_files)
    else:
        paths = [os.path.join(inner.root, "imgs", f if kind == "potsdamraw" else f + ".mat") for f in inner.files]
    return ds, [os.path.relpath(p, root) for p in paths], list(DataLoader(ds, BATCH, shuffle=False))


def value_table(utils) -> torch.Tensor:
    """fp32 [3, 256]: the reference's image transform of every byte in every channel, increasing in the byte."""
    every = np.repeat(np.arange(256, dtype=np.uint8).reshape(16, 16, 1), 3, axis=2)
    values = utils.get_transform(16, False, "center")(Image.fromarray(every)).reshape(3, 256).contiguous()
    assert (values[:, 1:] > values[:, :-1]).all()
    return values


def as_bytes(row: torch.Tensor, values: torch.Tensor) -> torch.Tensor:
    """The uint8 [3, res, res] whose values are the fp32 row exactly (asserted)."""
    idx = torch.stack([torch.searchsorted(values[c], row[c].contiguous()) for c in range(3)]).clamp(max=255)
    assert torch.equal(torch.stack([values[c][idx[c]] for c in range(3)]), row)
    return idx.to(torch.uint8)


def main():
    if not reference_shim.available():
        raise RuntimeError("set STEGO_REFERENCE_SRC to the reference's src directory")
    utils, data = _import_reference_loaders()
    files, raw = tree()
    cases, tables, fine_to_coarse = {}, {}, None
    values = value_table(utils)
    frames = {res: [] for res in RESOLUTIONS}
    frame_of = {res: {} for res in RESOLUTIONS}
    with tempfile.TemporaryDirectory() as root:
        write_tree(root, files, raw)
        for kind in KINDS:
            for res in RESOLUTIONS:
                ds, paths, batches = run(data, utils, root, kind, res, True)
                if kind.startswith("cocostuff"):
                    fine_to_coarse = dict(ds.dataset.fine_to_coarse)
                n = len(paths)
                rows = {k: [None] * n for k in ("img", "label", "mask")}
                for b in batches:
                    for j, i in enumerate(b["ind"].tolist()):
                        for k in rows:
                            rows[k][i] = b[k][j]
                R = {k: torch.stack(v) for k, v in rows.items()}
                # the same pass without the mask: no mask key, the same rows
                _, _, plain = run(data, utils, root, kind, res, False)
                for b in plain:
                    assert "mask" not in b and set(b) == {"ind", "img", "label"}, (kind, sorted(b))
                    assert torch.equal(b["img"], R["img"][b["ind"]]) and torch.equal(b["label"], R["label"][b["ind"]])
                for b in batches:
                    for k in rows:
                        assert b[k].dtype == R[k].dtype and torch.equal(b[k], R[k][b["ind"]]), (kind, res, k)
                if res == 32:  # the all-bytes tile (16 x 16, upsampled 2x): the label of every byte
                    first = paths.index(next(p for p in paths if _is_all_bytes(root, p)))
                    tables[kind] = R["label"][first][0::2, 0::2].reshape(256).to(torch.int16).clone()
                # PotsdamRaw keeps one row per pool entry
                if kind == "potsdamraw":
                    row_of = list(raw["tile_of"])
                    keep = [row_of.index(e) for e in range(RAW_POOL)]
                    for t, e in enumerate(row_of):
                        for k in rows:
                            assert torch.equal(R[k][t], R[k][keep[e]]), (t, k)
                    R = {k: v[keep] for k, v in R.items()}
                else:
                    row_of = list(range(n))
                assert R["label"].abs().max() < 1 << 15
                # img rows as bytes, one entry per distinct image and res
                keys = [f"potsdamraw/pool/{e}" for e in range(RAW_POOL)] if kind == "potsdamraw" else paths
                img_index = []
                for key, row in zip(keys, R["img"]):
                    b = as_bytes(row, values)
                    if key in frame_of[res]:
                        assert torch.equal(frames[res][frame_of[res][key]], b), (kind, res, key)
                    else:
                        frame_of[res][key] = len(frames[res])
                        frames[res].append(b)
                    img_index.append(frame_of[res][key])
                if kind == "potsdamraw":  # the 8550 paths and the pool entry of each are kept once, in `raw`
                    prefix = os.path.join("potsdamraw", "processed", "imgs") + os.sep
                    assert all(p.startswith(prefix) for p in paths)
                    raw["names_zlib"] = zlib.compress("\n".join(p[len(prefix):] for p in paths).encode(), 9)
                    paths = row_of = None
                case = dict(paths=paths, row_of=None if row_of is None else torch.tensor(row_of, dtype=torch.int64),
                            img_index=torch.tensor(img_index, dtype=torch.int64),
                            label_dtype=str(R["label"].dtype).replace("torch.", ""), label=R["label"].to(torch.int16),
                            mask_dtype=str(R["mask"].dtype).replace("torch.", ""), mask_shape=tuple(R["mask"].shape),
                            mask=torch.from_numpy(np.packbits(R["mask"].to(torch.bool).numpy().reshape(-1))))
                assert ((R["mask"] == 0) | (R["mask"] == 1)).all()
                cases[f"{kind}_{res}"] = case
                print(kind, res, n, "samples", case["label_dtype"], case["mask_dtype"], tuple(R["mask"].shape[1:]))
    raw["tile_of"] = torch.tensor(raw["tile_of"], dtype=torch.uint8)
    frames = {res: torch.stack(v) for res, v in frames.items()}
    torch.save(dict(tree=files, raw=raw, batch_size=BATCH, fine_to_coarse=fine_to_coarse, tables=tables,
                    values=values, frames=frames, cases=cases), OUT)
    print(f"wrote {OUT}: {os.path.getsize(OUT)} bytes")


def _is_all_bytes(root, rel):
    path = os.path.join(root, rel)
    if path.endswith(".mat"):
        from scipy.io import loadmat
        return loadmat(path)["img"].shape[:2] == (16, 16)
    with Image.open(path) as im:
        return im.size == (16, 16)


if __name__ == "__main__":
    main()
