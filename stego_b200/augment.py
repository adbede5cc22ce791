"""The aug-alignment views `img_aug` / `coord_aug` of a batch on the GPU (reference src/data.py:527-563 with the
transforms of src/train_segmentation.py:408-416).

The reference's ContrastiveSegDataset.__getitem__ draws a seed per sample, seeds torch with it and runs

    img_aug   = ColorJitter(.3, .3, .3, .1) -> RandomGrayscale(.2) -> RandomApply([GaussianBlur((5, 5))])
                ( RandomResizedCrop(res, scale=(.8, 1)) ( RandomHorizontalFlip() (img) ) )
    coord_aug = the geometric pair again, re-seeded, on meshgrid(linspace(-1, 1, H), linspace(-1, 1, W)), as [H, W, 2]

on the CPU in its loader workers.  `aug_alignment_views` makes the same parameter draws on the host, from the same
seeds and through torchvision's own draw code, uploads them in one copy and builds both views of the whole batch in two
kernel launches (stego_aug_views).  The arithmetic is that of the installed torchvision's tensor path.
"""
from __future__ import annotations

import math
import struct

import torch
import torchvision.transforms as T
from torchvision.transforms._functional_tensor import _get_gaussian_kernel2d

from . import _lib

RECORD_WORDS = 48
SCALE, RATIO = (0.8, 1.0), (3.0 / 4.0, 4.0 / 3.0)          # RandomResizedCrop(size=res, scale=(0.8, 1.0))
JITTER = T.ColorJitter(brightness=.3, contrast=.3, saturation=.3, hue=.1)
GRAY_P, BLUR_P, BLUR_KERNEL, BLUR_SIGMA = 0.2, 0.5, (5, 5), (0.1, 2.0)


def _f32_bits(x: float) -> int:
    """The int32 word holding fl32(x) (struct rounds to nearest even, as a float32 tensor does)."""
    return struct.unpack("<i", struct.pack("<f", x))[0]


def draw_params(seed: int, H: int, W: int) -> dict:
    """The parameters one __getitem__ draws after `_set_seed(seed)`, in the reference's call order, for an [3, H, W]
    frame.  Uses (and leaves as found) the CPU default generator: the caller forks it."""
    torch.default_generator.manual_seed(seed)
    flip = bool(torch.rand(1) < 0.5)                                     # RandomHorizontalFlip.forward
    frame = torch.empty(1, 1, 1).expand(3, H, W)                         # only its size is read
    top, left, h, w = T.RandomResizedCrop.get_params(frame, list(SCALE), list(RATIO))
    fn_idx, b, c, s, hue = T.ColorJitter.get_params(JITTER.brightness, JITTER.contrast, JITTER.saturation, JITTER.hue)
    gray = bool(torch.rand(1) < GRAY_P)                                  # RandomGrayscale.forward
    blur = not (BLUR_P < torch.rand(1))                                  # RandomApply.forward
    sigma = T.GaussianBlur.get_params(*BLUR_SIGMA) if blur else None     # GaussianBlur.forward, only when applied
    return dict(flip=flip, crop=(int(top), int(left), int(h), int(w)), fn_idx=[int(k) for k in fn_idx],
                brightness=b, contrast=c, saturation=s, hue=hue, gray=gray, blur=blur, sigma=sigma)


def blur_weights(sigma: float) -> torch.Tensor:
    """The fp32 5x5 weights F.gaussian_blur convolves with: torchvision's own _get_gaussian_kernel2d."""
    return _get_gaussian_kernel2d(list(BLUR_KERNEL), [sigma, sigma], torch.float32, torch.device("cpu"))


def record(p: dict) -> list:
    """One sample's words of the stego_aug_views record (include/stego_b200.h)."""
    words = [0] * RECORD_WORDS
    words[0] = int(p["flip"])
    words[1:5] = p["crop"]
    words[5:9] = p["fn_idx"]
    words[9], words[10] = int(p["gray"]), int(p["blur"])
    for k, name in ((11, "brightness"), (13, "contrast"), (15, "saturation")):
        # _blend(img1, img2, ratio) multiplies by fl(ratio) and fl(1.0 - ratio), the latter formed in double
        words[k], words[k + 1] = _f32_bits(p[name]), _f32_bits(1.0 - p[name])
    words[17] = _f32_bits(p["hue"])
    if p["blur"]:
        words[18:43] = blur_weights(p["sigma"]).reshape(-1).view(torch.int32).tolist()
    return words


def draw_records(seeds, H: int, W: int):
    """(params, records): the draws of every seed and the int32 [B, 48] records, with the CPU and CUDA generators left
    exactly as they were (the CPU generator is forked; the CUDA generators are never touched)."""
    params = []
    with torch.random.fork_rng(devices=[]):
        for seed in seeds:
            params.append(draw_params(seed, H, W))
    return params, torch.tensor([record(p) for p in params], dtype=torch.int32)


def _check(img, seeds, size):
    if not isinstance(img, torch.Tensor):
        raise TypeError("stego_b200.augment: img must be a tensor")
    if img.dim() != 4 or img.shape[1] != 3:
        raise ValueError(f"stego_b200.augment: img must be [B, 3, H, W], got {tuple(img.shape)}")
    B, _, H, W = img.shape
    if not 1 <= B <= 65535 or H < 1 or W < 1:
        raise ValueError(f"stego_b200.augment: img shape {tuple(img.shape)}: 1 <= B <= 65535 and H, W >= 1")
    if img.dtype != torch.float32:
        raise ValueError(f"stego_b200.augment: img must be float32 (the normalised frames), got {img.dtype}")
    seeds = list(seeds)
    if len(seeds) != B:
        raise ValueError(f"stego_b200.augment: {len(seeds)} seeds for {B} images")
    for s in seeds:
        if isinstance(s, bool) or not isinstance(s, int) or not 0 <= s < 1 << 64:
            raise ValueError(f"stego_b200.augment: seed {s!r} must be an int in [0, 2^64)")
    if isinstance(size, bool) or not isinstance(size, int) or not 3 <= size <= 8192:
        raise ValueError(f"stego_b200.augment: size={size!r} (an int in 3..8192)")
    if not img.is_cuda:
        raise RuntimeError("stego_b200.augment: CUDA tensors required (no CPU fallback)")
    return seeds


def batch_seeds(seeds) -> list:
    """batch["seed"] as B Python ints: a list, or a CPU integer tensor as a DataLoader collates one.  A CUDA tensor
    raises, because reading it would synchronise with the device."""
    if isinstance(seeds, torch.Tensor):
        if seeds.is_cuda:
            raise ValueError("stego_b200.augment: batch['seed'] must be a list or a CPU tensor (reading a CUDA tensor "
                             "would synchronise with the device)")
        if seeds.dtype.is_floating_point or seeds.dtype.is_complex or seeds.dtype == torch.bool or seeds.dim() != 1:
            raise ValueError(f"stego_b200.augment: batch['seed'] must be a 1-d integer tensor, got {seeds.dtype} "
                             f"{tuple(seeds.shape)}")
        return seeds.tolist()
    return list(seeds)


def launch(img, records_dev, size, img_aug, coord_aug, scratch) -> None:
    """stego_aug_views on prepared operands: records int32 [B, 48] on the device, scratch of
    stego_aug_scratch_bytes bytes."""
    B, _, H, W = img.shape
    _lib.check(_lib.load().stego_aug_views(_lib.ptr(img), *img.stride(), B, H, W, size, _lib.ptr(records_dev),
                                           _lib.ptr(scratch), _lib.ptr(img_aug), _lib.ptr(coord_aug), _lib.stream()),
               "stego_aug_views")


def aug_alignment_views(img: torch.Tensor, seeds, size: int):
    """(img_aug [B, 3, size, size], coord_aug [B, size, size, 2]), fp32 on img's device: what the reference's
    __getitem__ returns as ret["img_aug"] / ret["coord_aug"] for frame img[b] after drawing seed seeds[b].

    img: normalised fp32 frames [B, 3, H, W] on CUDA, any strides; seeds: B ints (the reference draws
    np.random.randint(2147483647) per sample); size: cfg.res.  The draws run on the host on a forked CPU generator, so
    the caller's CPU and CUDA generator states are unchanged.  One host-to-device copy (the records), two launches on
    the current stream, no device-to-host copy and no synchronisation."""
    seeds = _check(img, seeds, size)
    B, _, H, W = img.shape
    dev = img.device
    _, records = draw_records(seeds, H, W)
    records = records.pin_memory().to(dev, non_blocking=True)
    img_aug = torch.empty(B, 3, size, size, dtype=torch.float32, device=dev)
    coord_aug = torch.empty(B, size, size, 2, dtype=torch.float32, device=dev)
    nbytes = int(_lib.load().stego_aug_scratch_bytes(B, size))
    scratch = torch.empty(math.ceil(nbytes / 8), dtype=torch.float64, device=dev)
    launch(img, records, size, img_aug, coord_aug, scratch)
    return img_aug, coord_aug
