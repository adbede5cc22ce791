"""Timing of the GPU dense CRF on a configs[4] frame (1024 x 2048, 27 classes): lattice construction and the ten
mean-field iterations.  python profiles/crf_time.py"""
import os, sys, time, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from stego_b200 import crf
dev = torch.device("cuda:0")
torch.manual_seed(0)
H, W, C = 1024, 2048, 27
img = torch.randn(3, H, W, device=dev) * 0.5
logp = torch.log_softmax(torch.randn(1, C, 128, 256, device=dev) * 3, 1)
logp = torch.nn.functional.interpolate(logp, (H, W), mode="bilinear", align_corners=False)[0]
image = crf.prepare_image(img)


def timed(fn, n=3):
    fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / n * 1e3


def build(d):
    lat = crf._lattice_points(H, W, d, 1 if d == 2 else 67, 0 if d == 2 else 3, None if d == 2 else image, dev)
    crf._norm(lat)
    return lat


lat_g = timed(lambda: build(2))
lat_b = timed(lambda: build(5))
lg, lb = build(2), build(5)
print(f"lattice build: position {lat_g:.1f} ms (M = {lg.M}), bilateral {lat_b:.1f} ms (M = {lb.M}); pixels {H * W}")
for it in (0, 1, 10):
    ms = timed(lambda: crf.mean_field(logp, image, it))
    print(f"mean_field with {it:2d} iterations (incl. bilateral lattice build): {ms:.1f} ms")
print(f"whole dense_crf per frame: {timed(lambda: crf.dense_crf(img, logp)):.1f} ms")
