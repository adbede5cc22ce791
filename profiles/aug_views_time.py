"""Cost of building the aug-alignment views (img_aug, coord_aug; src/data.py:527-563) for one batch, on the card it runs on.

    python profiles/aug_views_time.py [--out FILE]

Prints one JSON object with the card name and power limit read in the same run.  For B = 32 frames at 224² and at
320² (output size = frame size), three implementations of the same views from the same seeds:
  * `kernel`: augment.aug_alignment_views, host draws and two launches.  `kernel_ms`: CUDA-event time per call over
    >= 0.5 s back to back (the device is busy for the whole window only if the host draws keep up);
    `kernel_host_ms`: host clock per call over 20 calls ending in a synchronise (draws, upload, launches, kernels).
  * `torchvision_cpu_1core_ms` / `torchvision_cpu_all_cores_ms`: the reference's per-sample composition
    (oracle/aug_oracle.reference_views: seed, img_aug, reseed, coord_aug) on fp32 CPU tensors, host clock per batch:
    one thread in this process, and a pool of single-threaded worker processes, one per core (as loader workers run it;
    the frames are pickled to them).
  * `torchvision_cuda_ms`: the same per-sample composition on CUDA tensors, host clock per batch.
"""
import argparse
import multiprocessing as mp
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
from _measure import card, emit, host_ms, window_ms  # noqa: E402

B = 32
SIZES = (224, 320)
WINDOW = dict(warmup=3, min_window_s=0.5, min_iters=10)


def _worker_init():
    torch.set_num_threads(1)


def _one(args):
    import aug_oracle
    frame, seed, size = args
    img_aug, coord_aug = aug_oracle.reference_views(frame, seed, size)
    return img_aug.shape[-1] + coord_aug.shape[0]


def case(size, dev, pool):
    import aug_oracle
    from stego_b200 import augment
    g = torch.Generator().manual_seed(size)
    frames = torch.randn(B, 3, size, size, generator=g) * 1.2 + 0.2
    seeds = [int(s) for s in torch.randint(0, 2147483647, (B,), generator=g)]
    img = frames.to(dev)
    kernel_ms, calls = window_ms(lambda: augment.aug_alignment_views(img, seeds, size), **WINDOW)
    kernel_host_ms = host_ms(lambda: augment.aug_alignment_views(img, seeds, size), 20)

    def per_sample(x):
        for b in range(B):
            aug_oracle.reference_views(x[b], seeds[b], size)

    threads = torch.get_num_threads()
    torch.set_num_threads(1)
    per_sample(frames)
    cpu1 = host_ms(lambda: per_sample(frames), 3)
    torch.set_num_threads(threads)
    jobs = [(frames[b], seeds[b], size) for b in range(B)]
    pool.map(_one, jobs)
    cpu_all = host_ms(lambda: pool.map(_one, jobs), 3)
    per_sample(img)
    cuda = host_ms(lambda: per_sample(img), 3)
    return dict(B=B, size=size, kernel_ms=round(kernel_ms, 4), kernel_calls=calls, kernel_host_ms=round(kernel_host_ms, 3),
                torchvision_cpu_1core_ms=round(cpu1, 2), torchvision_cpu_all_cores_ms=round(cpu_all, 2),
                cpu_workers=pool._processes, torchvision_cuda_ms=round(cuda, 2))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from stego_b200 import _lib
    _lib.load()
    dev = torch.device("cuda:0")
    with mp.get_context("spawn").Pool(os.cpu_count(), initializer=_worker_init) as pool:
        cases = [case(s, dev, pool) for s in SIZES]
    emit(dict(card=card(), views=cases, gpu_info_after=card()), args.out, indent=1)


if __name__ == "__main__":
    main()
