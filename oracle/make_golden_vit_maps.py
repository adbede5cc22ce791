"""Generate tests/golden/vit_small8_32px_maps.pt from the REAL reference and check the oracle against it.

    STEGO_REFERENCE_SRC=<reference checkout>/src python oracle/make_golden_vit_maps.py

The reference's get_last_selfattention(img), get_intermediate_feat(img, n=3) and get_intermediate_layers(img, n=2), on
the seeded, perturbed ViT-S/8 and the 32 x 32 image of tests/golden/vit_small8_32px.pt (oracle/make_golden.py, item 4).
Only outputs are stored; the weights and the image are regenerated from their seeds.  Exit status 0 iff
oracle/vit_maps_oracle.vit_intermediate matches the reference.
"""
from __future__ import annotations

import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import reference_shim  # noqa: E402
import stego_oracle as O  # noqa: E402
import vit_maps_oracle as VM  # noqa: E402

OUT = os.path.join(HERE, "..", "tests", "golden", "vit_small8_32px_maps.pt")
RECIPE = ("sd = perturb_vit_state(vit_random_state('vit_small', 8, seed=3)); manual_seed(11); img = randn(2,3,32,32); "
          "reference get_last_selfattention(img), get_intermediate_feat(img, n=3), get_intermediate_layers(img, n=2)")


def inputs():
    sd = O.perturb_vit_state(O.vit_random_state("vit_small", 8, seed=3))
    torch.manual_seed(11)
    return sd, torch.randn(2, 3, 32, 32)


def reference_maps():
    _, vits = reference_shim.import_reference()
    sd, img = inputs()
    model = vits.vit_small(patch_size=8, num_classes=0)
    model.load_state_dict(sd)
    model.eval()
    with torch.no_grad():
        last = model.get_last_selfattention(img)
        feat, attn, qkv = model.get_intermediate_feat(img, n=3)
        layers = model.get_intermediate_layers(img, n=2)
    return dict(recipe=RECIPE, last_selfattention=last.clone(), feat3=[t.clone() for t in feat],
                attn3=[t.clone() for t in attn], qkv3=[t.clone() for t in qkv], layers2=[t.clone() for t in layers])


def check(g) -> float:
    """Largest absolute difference between the oracle and the stored reference outputs."""
    sd, img = inputs()
    with torch.no_grad():
        feat, attn, qkv = VM.vit_intermediate(sd, img, "vit_small", 8, n=3)
        layers, _, _ = VM.vit_intermediate(sd, img, "vit_small", 8, n=2)
        _, last, _ = VM.vit_intermediate(sd, img, "vit_small", 8, n=1)
    pairs = [(last[0], g["last_selfattention"])] + list(zip(feat, g["feat3"])) + list(zip(attn, g["attn3"])) \
        + list(zip(qkv, g["qkv3"])) + list(zip(layers, g["layers2"]))
    assert len(feat) == len(g["feat3"]) == 3 and len(layers) == len(g["layers2"]) == 2
    return max((a - b).abs().max().item() for a, b in pairs)


def main():
    torch.set_num_threads(1)
    g = reference_maps()
    err = check(g)
    print(f"oracle vs reference: max abs diff {err:.3e}")
    if err > 1e-5:
        sys.exit(1)
    torch.save(g, OUT)
    print(OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main()
