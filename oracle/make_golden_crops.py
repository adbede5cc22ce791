"""Make tests/golden/crop_windows.pt: the crop windows of the reference's crop script (src/crop_datasets.py:14-74) on
a set of image sizes, items and ratios.  TEST INFRASTRUCTURE ONLY.

The reference module does not import here: it needs Hydra and Lightning and imports `_get_image_size`, which
torchvision 0.26 no longer has.  So its rule is restated on tensors, through torchvision itself:
  * "five": torchvision.transforms.functional.five_crop(img, [int(H * ratio), int(W * ratio)]) on a [1, H, W] tensor
    whose values are the pixel positions; each crop's top-left value and shape give its window.
  * "random": _random_crops(img, size, item, 5): top = hash((item, i, 0)) % (H - ch), left = hash((item, i, 1)) %
    (W - cw), then torchvision's crop(img, top, left, ch, cw), read back the same way.
Written independently of stego_b200.crops.crop_windows, which the tests compare against this table.  The fixture also
records the libjpeg-turbo version of the Pillow that judges the JPEG oracle (oracle/jpeg_oracle.py) on this machine.
"""
import os

import PIL
import PIL.features
import torch
import torchvision.transforms.functional as TF

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "crop_windows.pt")
SIZES = [(480, 640), (640, 427), (1024, 2048), (37, 50), (3, 5), (2, 2)]
ITEMS = [0, 1, 7, 4321, 49999]
RATIOS = [0.5, 0.7]


def window_of(crop: torch.Tensor, W: int) -> tuple:
    pos = int(crop[0, 0, 0])
    return (pos // W, pos % W, crop.shape[1], crop.shape[2])


def reference_windows(H: int, W: int, crop_type: str, ratio: float, item: int):
    img = torch.arange(H * W, dtype=torch.int64).view(1, H, W)
    size = [int(img.shape[1] * ratio), int(img.shape[2] * ratio)]
    if crop_type == "five":
        return [window_of(c, W) for c in TF.five_crop(img, size)]
    ch, cw = size
    if ch == H or cw == W or ch == 0 or cw == 0:
        return None  # the reference divides by zero (or cuts an empty crop)
    out = []
    for i in range(5):
        top, left = hash((item, i, 0)) % (H - ch), hash((item, i, 1)) % (W - cw)
        out.append(window_of(TF.crop(img, top, left, ch, cw), W))
    return out


def main():
    cases = []
    for H, W in SIZES:
        for ratio in RATIOS:
            for crop_type in ("five", "random"):
                for item in ITEMS if crop_type == "random" else [0]:
                    if int(H * ratio) == 0 or int(W * ratio) == 0:
                        continue
                    cases.append(dict(size=(H, W), ratio=ratio, crop_type=crop_type, item=item,
                                      windows=reference_windows(H, W, crop_type, ratio, item)))
    torch.save(dict(cases=cases, pillow=PIL.__version__, libjpeg_turbo=PIL.features.version("libjpeg_turbo"),
                    torchvision=__import__("torchvision").__version__), OUT)
    print(f"wrote {OUT}: {len(cases)} cases")


if __name__ == "__main__":
    main()
