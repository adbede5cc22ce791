"""CPU: the aug-alignment views' parameter draws and their oracle (src/data.py:527-563, train_segmentation.py:408-416).

tests/golden/aug_views.pt holds what the reference's own ContrastiveSegDataset.__getitem__ returned
(oracle/make_golden_aug.py); oracle/aug_oracle.py must reproduce it bit for bit and its float64 restatement must lie
within fp32 rounding of it.  stego_b200.augment's host draws must be torchvision's, parameter for parameter, recorded
from inside the torchvision composition itself, and must leave the CPU generator as they found it.  The wrapper and the
C ABI reject bad arguments before anything is launched."""
import itertools
import math
import os
import re
import sys

import pytest
import torch
import torchvision.transforms.functional as TF

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import aug_oracle as AO  # noqa: E402
import make_golden_aug as MGA  # noqa: E402

from stego_b200 import augment  # noqa: E402

GOLDEN = torch.load(os.path.join(ROOT, "tests", "golden", "aug_views.pt"))
CASES = MGA.cases()


def test_golden_covers_the_cases():
    assert set(GOLDEN) == set(CASES)
    params = [augment.draw_params(GOLDEN[n]["seed"], f.shape[1], f.shape[2]) for n, (f, _, _) in CASES.items()]
    assert {p["flip"] for p in params} == {True, False} and {p["blur"] for p in params} == {True, False}
    assert any(f.shape[1] != f.shape[2] for f, _, _ in CASES.values())
    assert any(size > f.shape[1] for f, size, _ in CASES.values()) and any(size < f.shape[1] for f, size, _ in CASES.values())


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_reproduces_reference(name):
    """The oracle's composition is the reference's bit for bit; the float64 restatement on the drawn parameters is
    within 2^-18 of it (a few fp32 roundings of values below 8)."""
    frame, size, _ = CASES[name]
    want = GOLDEN[name]
    img_aug, coord_aug = AO.reference_views(frame, want["seed"], size)
    assert torch.equal(img_aug, want["img_aug"]) and torch.equal(coord_aug, want["coord_aug"])
    p = augment.draw_params(want["seed"], frame.shape[1], frame.shape[2])
    x, c = AO.views_fp64(frame, p, size, augment.blur_weights(p["sigma"]) if p["blur"] else None)
    assert (x - want["img_aug"].double()).abs().max() < 2 ** -18
    assert (c - want["coord_aug"].double()).abs().max() < 2 ** -20


def _record_torchvision(frame, seed, size, monkeypatch):
    """The parameters the torchvision composition passes to torchvision.transforms.functional, in call order."""
    calls = []

    def spy(name):
        fn = getattr(TF, name)

        def wrapped(*a, **k):
            calls.append((name, a[1:], k))
            return fn(*a, **k)
        monkeypatch.setattr(TF, name, wrapped)
    for name in ("hflip", "resized_crop", "adjust_brightness", "adjust_contrast", "adjust_saturation", "adjust_hue",
                 "rgb_to_grayscale", "gaussian_blur"):
        spy(name)
    with torch.random.fork_rng(devices=[]):
        AO.reference_views(frame, seed, size)
    monkeypatch.undo()
    return calls


def _expected_calls(p, size):
    """The calls the drawn parameters stand for (twice the geometric pair: img, then coord)."""
    geo = ([("hflip", (), {})] if p["flip"] else []) + [("resized_crop", tuple(p["crop"]) + ([size, size],), None)]
    names = {0: ("adjust_brightness", "brightness"), 1: ("adjust_contrast", "contrast"),
             2: ("adjust_saturation", "saturation"), 3: ("adjust_hue", "hue")}
    jit = [(names[k][0], (p[names[k][1]],), {}) for k in p["fn_idx"]]
    gray = [("rgb_to_grayscale", (), {"num_output_channels": 3})] if p["gray"] else []
    blur = [("gaussian_blur", ([5, 5], [p["sigma"], p["sigma"]]), {})] if p["blur"] else []
    return geo + jit + gray + blur + geo


def _same(calls, want):
    if len(calls) != len(want):
        return False
    for (n, a, k), (wn, wa, wk) in zip(calls, want):
        if n != wn:
            return False
        if n == "resized_crop":
            if tuple(a[:4]) != wa[:4] or list(a[4]) != wa[4]:
                return False
        elif n == "gaussian_blur":
            if list(a[0]) != wa[0] or [float(s) for s in a[1]] != wa[1]:  # exact: the same double
                return False
        elif tuple(a) != wa or (wk and k != wk):
            return False
    return True


def _fallback(seed, H, W):
    """True when RandomResizedCrop.get_params leaves its 10-try loop for the centre crop (a restatement of its loop
    on the same generator, used only to pick seeds)."""
    torch.default_generator.manual_seed(seed)
    torch.rand(1)
    log_ratio = torch.log(torch.tensor(augment.RATIO))
    for _ in range(10):
        area = H * W * torch.empty(1).uniform_(*augment.SCALE).item()
        ar = torch.exp(torch.empty(1).uniform_(log_ratio[0], log_ratio[1])).item()
        w, h = int(round(math.sqrt(area * ar))), int(round(math.sqrt(area / ar)))
        if 0 < w <= W and 0 < h <= H:
            return False
    return True


def _seed_search():
    """Seeds covering flip on / off, all 24 jitter orders, grayscale on / off, blur on / off (found by search)."""
    need = {("flip", True), ("flip", False), ("gray", True), ("gray", False), ("blur", True), ("blur", False)}
    need |= {("order", o) for o in itertools.permutations(range(4))}
    chosen = []
    with torch.random.fork_rng(devices=[]):
        for seed in range(5000):
            p = augment.draw_params(seed, 40, 40)
            have = {("flip", p["flip"]), ("gray", p["gray"]), ("blur", p["blur"]), ("order", tuple(p["fn_idx"]))}
            if have & need:
                need -= have
                chosen.append(seed)
            if not need:
                break
    assert not need, need
    return chosen


def test_draws_are_torchvision_draws(monkeypatch):
    """Every drawn parameter equals what the torchvision composition passes on, bit for bit, over a seed set that
    reaches every branch, including RandomResizedCrop's centre-crop fallback on square, wide and tall frames."""
    seeds = _seed_search()
    frames = [(40, 40)] * len(seeds)
    with torch.random.fork_rng(devices=[]):
        fb_square = next(s for s in range(20000) if _fallback(s, 40, 40))
    seeds += [fb_square, 3, 4]
    frames += [(40, 40), (8, 40), (40, 8)]  # the wide / tall frames always fall back (in_ratio outside [3/4, 4/3])
    g = torch.Generator().manual_seed(0)
    for seed, (H, W) in zip(seeds, frames):
        frame = torch.randn(3, H, W, generator=g)
        with torch.random.fork_rng(devices=[]):
            p = augment.draw_params(seed, H, W)
            assert _fallback(seed, H, W) == ((H, W) != (40, 40) or seed == fb_square)
        calls = _record_torchvision(frame, seed, 12, monkeypatch)
        assert _same(calls, _expected_calls(p, 12)), (seed, calls, p)


def test_records_and_generator_state():
    """draw_records leaves the CPU generator exactly as found; its records hold the parameters as the kernel reads
    them (fp32 words, fl(1 - factor) from the double, torchvision's fp32 Gaussian weights)."""
    torch.manual_seed(123)
    before = torch.get_rng_state()
    params, rec = augment.draw_records([7, 42, 2 ** 31 - 2, 2 ** 64 - 1], 30, 50)
    assert torch.equal(torch.get_rng_state(), before)
    assert rec.shape == (4, augment.RECORD_WORDS) and rec.dtype == torch.int32
    for p, r in zip(params, rec):
        assert r[0] == int(p["flip"]) and r[1:5].tolist() == list(p["crop"]) and r[5:9].tolist() == p["fn_idx"]
        assert r[9] == int(p["gray"]) and r[10] == int(p["blur"])
        f = r.view(torch.float32)
        for k, name in ((11, "brightness"), (13, "contrast"), (15, "saturation")):
            assert float(f[k]) == p[name]
            assert f[k + 1] == torch.tensor(1.0 - p[name], dtype=torch.float32)
        assert float(f[17]) == p["hue"]
        if p["blur"]:
            assert torch.equal(f[18:43], augment.blur_weights(p["sigma"]).reshape(-1))
        else:
            assert not r[18:].any()


def test_wrapper_rejects_bad_arguments():
    ok = torch.zeros(2, 3, 16, 16)
    with pytest.raises(RuntimeError, match="CUDA"):
        augment.aug_alignment_views(ok, [1, 2], 8)
    for bad in (torch.zeros(3, 16, 16), torch.zeros(2, 4, 16, 16), torch.zeros(2, 3, 0, 16), torch.zeros(0, 3, 16, 16)):
        with pytest.raises(ValueError, match="img"):
            augment.aug_alignment_views(bad, [1] * max(bad.shape[0], 1), 8)
    with pytest.raises(ValueError, match="float32"):
        augment.aug_alignment_views(ok.double(), [1, 2], 8)
    with pytest.raises(ValueError, match="seeds"):
        augment.aug_alignment_views(ok, [1], 8)
    for seed in (-1, 1 << 64, 1.5, True):
        with pytest.raises(ValueError, match="seed"):
            augment.aug_alignment_views(ok, [1, seed], 8)
    for size in (2, 8193, 8.0, True):
        with pytest.raises(ValueError, match="size"):
            augment.aug_alignment_views(ok, [1, 2], size)
    with pytest.raises(TypeError):
        augment.aug_alignment_views(None, [1], 8)


def test_c_abi_rejects_before_any_launch():
    from stego_b200 import _lib
    lib = _lib.load()
    P = 256  # never dereferenced: every call below fails its argument checks first
    n0 = lib.stego_launch_count()

    def call(img=P, rec=P, scratch=P, out=P, B=2, H=8, W=8, size=8):
        return lib.stego_aug_views(img, 3 * H * W, H * W, W, 1, B, H, W, size, rec, scratch, out, P, 0)

    cases = [(dict(img=0), "null pointer"), (dict(rec=0), "null pointer"), (dict(scratch=0), "null pointer"),
             (dict(out=0), "null pointer"), (dict(B=0), "B=0"), (dict(B=65536), "B=65536"), (dict(H=0), ">= 1"),
             (dict(W=0), ">= 1"), (dict(size=2), "size=2"), (dict(size=8193), "size=8193"),
             (dict(scratch=P + 4), "8-byte")]
    for kw, msg in cases:
        assert call(**kw) == -1, kw
        assert re.search(msg, _lib.last_error()), (kw, _lib.last_error())
    assert lib.stego_launch_count() == n0
    assert lib.stego_aug_record_words() == augment.RECORD_WORDS


def test_scratch_rule():
    from stego_b200 import _lib
    lib = _lib.load()
    tiles = math.ceil(224 / 32) * math.ceil(224 / 8)
    assert lib.stego_aug_scratch_bytes(32, 224) == (8 * 32 * tiles + 255) // 256 * 256 + 12 * 32 * 224 * 224
    assert lib.stego_aug_scratch_bytes(0, 224) == 0
