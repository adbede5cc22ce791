"""Cost of building a batch's loader frames and labels (src/utils.py:165-183 get_transform and COCO-Stuff's remap,
src/data.py:303-309) on the host, as the reference's loader workers do, and on the GPU with stego_b200.frames.

    python profiles/frames_time.py [--out FILE]

Prints one JSON object with the card name and power limit read in the same run.  For B = 32 decoded RGB images with
their uint8 label maps, COCO-sized (640 x 480) and Cityscapes-sized (2048 x 1024), both to res = 320:
  * `host_1core_ms` / `host_all_cores_ms`: per image, torchvision's Resize(NEAREST) / CenterCrop / ToTensor / Normalize
    on the PIL image, the same resize and crop of the label with ToTargetTensor, and COCO-Stuff's 182-assignment remap
    loop; host clock per batch, in this process on one thread, and in a pool of single-threaded worker processes, one
    per core (as loader workers run it; the decoded arrays are pickled to them).  Decoding is not included.
  * GPU path, load_frames + load_labels: `pack_ms` (host: index tables and the copy of the bytes into the pinned
    staging buffers, host clock), `upload_ms` (the two host-to-device copies, CUDA events over a window), `kernel_ms`
    (the two launches on staged buffers, CUDA events over a window) and `call_ms` (both public calls, host clock per
    batch from an idle device to the synchronise after them).
  * `kernel_bytes`: what the kernels must move at least (each gathered source byte read once, the fp32 frames and
    int64 labels written once); `kernel_bound_ms` = kernel_bytes / 3.35 TB/s, the H100 SXM's HBM3 bandwidth, and
    `kernel_vs_bound` = kernel_ms / kernel_bound_ms.
"""
import argparse
import multiprocessing as mp
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from _measure import card, emit, host_ms, window_ms  # noqa: E402

B, RES = 32, 320
SIZES = dict(coco=(480, 640), cityscapes=(1024, 2048))
HBM_BYTES_PER_S = 3.35e12
WINDOW = dict(warmup=3, min_window_s=0.5, min_iters=10)
FINE_TO_COARSE = {i: (i * 7) % 27 for i in range(182)}  # a stand-in with the real table's size: the loop's cost


def _worker_init():
    torch.set_num_threads(1)


def _host_one(args):
    """One sample of the reference's loader work after decoding."""
    import torchvision.transforms as T
    from PIL import Image
    from stego_b200.frames import MEAN, STD
    rgb, lab = args
    img = T.Compose([T.Resize(RES, Image.NEAREST), T.CenterCrop(RES), T.ToTensor(), T.Normalize(MEAN, STD)])(
        Image.fromarray(rgb))
    label = T.Compose([T.Resize(RES, Image.NEAREST), T.CenterCrop(RES)])(Image.fromarray(lab, mode="L"))
    label = torch.as_tensor(np.array(label), dtype=torch.int64)
    label[label == 255] = -1
    coarse = torch.zeros_like(label)
    for fine, c in FINE_TO_COARSE.items():
        coarse[label == fine] = c
    coarse[label == -1] = -1
    return img.shape[-1] + coarse.shape[-1]


def case(name, dev, pool):
    from stego_b200 import _lib, frames
    H, W = SIZES[name]
    rng = np.random.default_rng(H)
    rgbs = [rng.integers(0, 256, (H, W, 3), dtype=np.uint8) for _ in range(B)]
    labs = [rng.integers(0, 256, (H, W), dtype=np.uint8) for _ in range(B)]
    lut = frames.label_lut(FINE_TO_COARSE)
    lut_np = lut.numpy()
    jobs = list(zip(rgbs, labs))

    threads = torch.get_num_threads()
    torch.set_num_threads(1)
    _host_one(jobs[0])
    host1 = host_ms(lambda: [_host_one(j) for j in jobs], 2)
    torch.set_num_threads(threads)
    pool.map(_host_one, jobs)
    host_all = host_ms(lambda: pool.map(_host_one, jobs), 3)

    def pack():
        return frames._stage(rgbs, RES, "center"), frames._stage(labs, RES, "center", lut_np)

    (fs, fw, _), (ls, lw, lut_at) = pack()
    pack_ms = host_ms(pack, 10)
    fd, ld = fs.to(dev), ls.to(dev)
    upload_ms, _ = window_ms(lambda: (fd.copy_(fs, non_blocking=True), ld.copy_(ls, non_blocking=True)), **WINDOW)
    out_f = torch.empty(B, 3, RES, RES, device=dev)
    out_l = torch.empty(B, RES, RES, dtype=torch.int64, device=dev)
    lib = _lib.load()

    def kernels():
        _lib.check(lib.stego_frames_rgb8(fs.data_ptr(), fd.data_ptr(), fs.numel(), fw, B, RES, *frames.MEAN,
                                         *frames.STD, out_f.data_ptr(), _lib.stream()), "stego_frames_rgb8")
        _lib.check(lib.stego_labels_u8(ls.data_ptr(), ld.data_ptr(), ls.numel(), lw, B, RES, ld.data_ptr() + lut_at,
                                       out_l.data_ptr(), _lib.stream()), "stego_labels_u8")

    kernel_ms, calls = window_ms(kernels, **WINDOW)
    assert torch.equal(out_f, frames.load_frames(rgbs, RES)) and torch.equal(out_l, frames.load_labels(labs, RES, lut=lut))
    call = host_ms(lambda: (frames.load_frames(rgbs, RES), frames.load_labels(labs, RES, lut=lut)), 10)
    kernel_bytes = B * RES * RES * (3 + 12 + 1 + 8)
    bound_ms = kernel_bytes / HBM_BYTES_PER_S * 1e3
    return dict(name=name, B=B, size=[H, W], res=RES, host_1core_ms=round(host1, 2), host_all_cores_ms=round(host_all, 2),
                cpu_workers=pool._processes, pack_ms=round(pack_ms, 3), staging_bytes=fs.numel() + ls.numel(),
                upload_ms=round(upload_ms, 4), kernel_ms=round(kernel_ms, 4), kernel_calls=calls,
                call_ms=round(call, 3), kernel_bytes=kernel_bytes, kernel_bound_ms=round(bound_ms, 4),
                kernel_vs_bound=round(kernel_ms / bound_ms, 2))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from stego_b200 import _lib
    _lib.load()
    dev = torch.device("cuda:0")
    with mp.get_context("spawn").Pool(os.cpu_count(), initializer=_worker_init) as pool:
        cases = [case(n, dev, pool) for n in SIZES]
    emit(dict(card=card(), frames=cases, gpu_info_after=card()), args.out, indent=1)


if __name__ == "__main__":
    main()
