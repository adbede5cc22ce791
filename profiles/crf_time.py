"""Timing of the GPU dense CRF on a configs[4] frame (1024 x 2048, 27 classes): lattice construction and the ten
mean-field iterations.

    python profiles/crf_time.py

Prints one JSON object.  Each time is a host clock around 3 calls after one warm-up call, ending in a device
synchronise."""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from stego_b200 import crf  # noqa: E402
from _measure import card, emit, host_ms  # noqa: E402

H, W, C = 1024, 2048, 27


def main():
    argparse.ArgumentParser(description=__doc__).parse_args()
    dev = torch.device("cuda:0")
    res = dict(card=card(), pixels=H * W)
    torch.manual_seed(0)
    img = torch.randn(3, H, W, device=dev) * 0.5
    logp = torch.log_softmax(torch.randn(1, C, 128, 256, device=dev) * 3, 1)
    logp = torch.nn.functional.interpolate(logp, (H, W), mode="bilinear", align_corners=False)[0]
    image = crf.prepare_image(img)

    def build(d):
        lat = crf._lattice_points(H, W, d, 1 if d == 2 else 67, 0 if d == 2 else 3, None if d == 2 else image, dev)
        crf._norm(lat)
        return lat

    runs = {"lattice_build_position_ms": lambda: build(2), "lattice_build_bilateral_ms": lambda: build(5)}
    for it in (0, 1, 10):  # the mean field includes its bilateral lattice build
        runs[f"mean_field_{it}_iterations_ms"] = lambda it=it: crf.mean_field(logp, image, it)
    runs["dense_crf_per_frame_ms"] = lambda: crf.dense_crf(img, logp)
    for name, fn in runs.items():
        fn()
        res[name] = round(host_ms(fn, 3), 1)
    res.update(lattice_points_position=build(2).M, lattice_points_bilateral=build(5).M)
    emit(res)


if __name__ == "__main__":
    main()
