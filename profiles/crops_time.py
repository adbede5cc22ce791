"""Cost of building a cropped training set (ResidentDataset.crops: the JPEG round trip of every crop on the GPU)
against the two-stage path it replaces (write_cropped's host JPEG / PNG files, then ResidentDataset.cropped).

    python profiles/crops_time.py [--out FILE]

Prints one JSON object with the card name and power limit read in the same run.  The source set is N_SRC seeded
synthetic COCO-like originals (640 x 480 and 480 x 640 JPEGs at quality 90, every eighth one grayscale) with PNG
annotations of bytes 0..181 and 255, in the cocostuff27 train layout, written to a temporary directory; crop_type
"five", crop_ratio 0.5 (320 x 240 crops), res 224, so the store holds 5 N_SRC rows.  The fine -> coarse table is a
stand-in of the real one's size.
  * `decode_ms_per_image`: the host decode of one original and its annotation (PIL open, convert("RGB")), one
    process.
  * `kernels`: for one build launch of B_SRC originals (5 B_SRC crops), the codec kernel (stego_jpeg_crops_codec) and
    the gather kernel (stego_jpeg_crops_store_rgb8), CUDA events over a window on staged inputs.
  * `build`: ResidentDataset.crops end to end (decode in WORKERS DataLoader workers, staging, kernels, label
    gather; the default batch_size 64 rows, i.e. 12 originals per launch), host clock to the synchronise after the
    last row, mean of two builds; ms per source image and crops/s.
  * `two_stage`: write_cropped (WORKERS workers) then ResidentDataset.cropped (WORKERS workers, batch_size 64) on
    the same sources, host clock, one run; and the speed-up of `build` over it.
"""
import argparse
import os
import shutil
import sys
import tempfile

import numpy as np
import torch
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from _measure import card, emit, host_ms, window_ms  # noqa: E402

N_SRC, B_SRC, RES, WORKERS, RATIO = 256, 64, 224, 8, 0.5
WINDOW = dict(warmup=3, min_window_s=0.5, min_iters=10)
FINE_TO_COARSE = {i: (i * 7) % 27 for i in range(182)}


def _write_coco(root):
    base = os.path.join(root, "cocostuff")
    for d in ("curated", "images", "annotations"):
        os.makedirs(os.path.join(base, d, "train2017"), exist_ok=True)
    rng = np.random.default_rng(0)
    ids = []
    for k in range(N_SRC):
        h, w = (480, 640) if k % 3 else (640, 480)
        img_id = f"{k:012d}"
        ids.append(img_id)
        yy, xx = np.mgrid[0:h, 0:w]
        smooth = np.stack([(xx // 3 + yy // 5) % 256, (yy // 2) % 256, (xx * yy // 97) % 256], -1)
        img = np.clip(smooth + rng.integers(-12, 13, (h, w, 3)), 0, 255).astype(np.uint8)
        pil = Image.fromarray(img).convert("L") if k % 8 == 0 else Image.fromarray(img)
        pil.save(os.path.join(base, "images", "train2017", img_id + ".jpg"), quality=90)
        label = rng.choice(np.r_[np.arange(182), 255], (h // 16, w // 16)).astype(np.uint8)
        Image.fromarray(np.kron(label, np.ones((16, 16), np.uint8))).save(
            os.path.join(base, "annotations", "train2017", img_id + ".png"))
    with open(os.path.join(base, "curated", "train2017", "Coco164kFull_Stuff_Coarse.txt"), "w") as f:
        f.write("".join(i + "\n" for i in ids))


def decode(root):
    from stego_b200.evalset import _EvalFiles, coco_files
    files = _EvalFiles(*coco_files(root, "cocostuff27", "train"), "pil")
    it = iter(range(32))
    return host_ms(lambda: files[next(it)], 32)


def kernels(root):
    from stego_b200 import _lib, crops, frames
    from stego_b200.evalset import _EvalFiles, coco_files
    files = _EvalFiles(*coco_files(root, "cocostuff27", "train"), "pil")
    arrays = [files[i][0] for i in range(B_SRC)]
    windows = [(i,) + w for i, x in enumerate(arrays) for w in crops.crop_windows(*x.shape[:2], "five", RATIO, i)]
    staging, words, ws_bytes = crops._stage(arrays, windows,
                                            lambda h, w: ((h, w), *frames.index_tables(h, w, RES, "center")))
    dev = torch.device("cuda:0")
    staged = staging.to(dev)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    store = torch.empty(len(windows), 3, RES, RES, dtype=torch.uint8, device=dev)
    lib = _lib.load()
    args = (staging.data_ptr(), _lib.ptr(staged), staging.numel(), words, len(windows))
    codec = lambda: lib.stego_jpeg_crops_codec(*args, _lib.ptr(ws), ws_bytes, _lib.stream())
    gather = lambda: lib.stego_jpeg_crops_store_rgb8(*args, RES, _lib.ptr(ws), ws_bytes, _lib.ptr(store),
                                                     len(windows), 0, _lib.stream())
    codec_ms = window_ms(codec, **WINDOW)[0]
    gather_ms = window_ms(gather, **WINDOW)[0]
    px = sum(h * w for _, _, _, h, w in windows)
    return dict(sources=B_SRC, crops=len(windows), crop_pixels=px, codec_ms=codec_ms, gather_ms=gather_ms,
                codec_mpix_per_s=px / codec_ms / 1e3, host_check_and_launch_included=True)


def build(root):
    from stego_b200.dataset import ResidentDataset
    ms = host_ms(lambda: ResidentDataset.crops(root, "cocostuff27", "five", RATIO, "train", RES, num_workers=WORKERS,
                                               fine_to_coarse=FINE_TO_COARSE), 2)
    return dict(ms_total=ms, ms_per_source=ms / N_SRC, crops_per_s=5 * N_SRC / ms * 1e3)


def two_stage(root):
    from stego_b200.crops import cropped_dir, write_cropped
    from stego_b200.dataset import ResidentDataset

    def run():
        shutil.rmtree(cropped_dir(root, "cocostuff27", "five", RATIO), ignore_errors=True)
        write_cropped(root, "cocostuff27", "five", RATIO, "train", num_workers=WORKERS, fine_to_coarse=FINE_TO_COARSE)
        ResidentDataset.cropped(root, "cocostuff27", "five", RATIO, "train", RES, num_workers=WORKERS)

    ms = host_ms(run, 1)
    return dict(ms_total=ms, ms_per_source=ms / N_SRC, crops_per_s=5 * N_SRC / ms * 1e3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from stego_b200 import _lib
    _lib.load()
    info = card()
    with tempfile.TemporaryDirectory() as root:
        _write_coco(root)
        result = dict(card=info, sources=N_SRC, res=RES, crop_ratio=RATIO, workers=WORKERS,
                      host_cores=os.cpu_count(), decode_ms_per_image=decode(root), kernels=kernels(root))
        result["build"] = build(root)
        result["two_stage"] = two_stage(root)
        result["speedup_over_two_stage"] = result["two_stage"]["ms_total"] / result["build"]["ms_total"]
        result["gpu_info_after"] = card()
    emit(result, args.out, indent=1)


if __name__ == "__main__":
    main()
