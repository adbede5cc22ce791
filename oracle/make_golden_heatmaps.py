"""Generate tests/golden/correspondence_heatmaps.pt from the REAL reference's correspondence heatmap lines.

    STEGO_REFERENCE_SRC=<reference checkout>/src python oracle/make_golden_heatmaps.py

src/plot_dino_correspondence.py cannot be imported (hydra, matplotlib, Lightning), so `get_heatmaps` (:39-58) is lifted
as TEXT and executed with the reference's own `sample` (src/modules.py:287-288), on the CPU: `net` is a callable that
returns fixed feature maps, and `Tensor.cuda` is the identity for the duration of the call.

Inputs: ViT-S width (E = 384) feature maps, low rank (4 components) plus noise so that each query correlates
positively with part of the map and negatively with the rest (the centring and the clamp both change values), rounded to
bf16 values (stored as bf16 without loss).  The self map is 12 x 16 and the KNN map 10 x 14, upsampled to the image
sizes 64 x 80 and 56 x 72.  Query points: the reference's three figure points, the corners +-1 and two beyond +-1.
heatmap_oracle restates the same lines in fp64; the tests compare both it and the kernels with the stored output.
"""
from __future__ import annotations

import ast
import os
import sys

import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import reference_shim  # noqa: E402

OUT = os.path.join(HERE, "..", "tests", "golden", "correspondence_heatmaps.pt")
E = 384
SELF_HW, KNN_HW = (12, 16), (10, 14)
IMG_HW, POS_HW = (64, 80), (56, 72)
POINTS = [[-.1, 0.0], [.5, .8], [-.7, -.7],      # the reference's figure points (:119-125)
          [1.0, 1.0], [-1.0, -1.0], [1.0, -1.0],  # corners
          [1.3, -1.2], [-2.0, 0.4]]               # beyond the border (clamped by grid_sample)


def inputs():
    """Seeded bf16-valued feature maps [1, E, h, w] of the image and its KNN image, and the query points."""
    g = torch.Generator().manual_seed(23)
    basis = torch.randn(4, E, generator=g)

    def fmap(hw):
        coef = torch.randn(hw[0] * hw[1], 4, generator=g)
        x = coef @ basis + 0.5 * torch.randn(hw[0] * hw[1], E, generator=g)
        return x.t().reshape(1, E, *hw).to(torch.bfloat16).float().contiguous()

    feats = fmap(SELF_HW)
    feats_pos = fmap(KNN_HW)
    query_points = torch.tensor(POINTS, dtype=torch.float32).reshape(1, len(POINTS), 1, 2)
    return dict(feats=feats, feats_pos=feats_pos, query_points=query_points)


def reference_get_heatmaps():
    """The reference's get_heatmaps function object, lifted from its source text."""
    modules, _ = reference_shim.import_reference()
    text = open(os.path.join(reference_shim.REFERENCE_SRC, "plot_dino_correspondence.py")).read()
    node = next(n for n in ast.walk(ast.parse(text)) if isinstance(n, ast.FunctionDef) and n.name == "get_heatmaps")
    env = dict(torch=torch, F=F, sample=modules.sample)
    exec(ast.get_source_segment(text, node), env)
    return env["get_heatmaps"]


def reference_lines(x):
    get_heatmaps = reference_get_heatmaps()
    img = torch.zeros(1, 3, *IMG_HW)
    img_pos = torch.zeros(1, 3, *POS_HW)
    maps = {id(img): x["feats"], id(img_pos): x["feats_pos"]}

    def net(t):
        return maps[id(t)], None

    cuda = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self
    try:
        with torch.no_grad():
            intra, inter = get_heatmaps(net, img, img_pos, x["query_points"])
    finally:
        torch.Tensor.cuda = cuda
    return intra, inter


def main():
    torch.set_num_threads(1)
    x = inputs()
    intra, inter = reference_lines(x)
    torch.save(dict(feats=x["feats"].to(torch.bfloat16), feats_pos=x["feats_pos"].to(torch.bfloat16),
                    query_points=x["query_points"], img_size=IMG_HW, pos_size=POS_HW,
                    heatmap_intra=intra.contiguous(), heatmap_inter=inter.contiguous()), OUT)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")
    for name, m in (("intra", intra), ("inter", inter)):
        print(name, tuple(m.shape), "max %.4f" % float(m.max()), "zero fraction %.3f" % float((m == 0).float().mean()))
    import heatmap_oracle as HO
    for name, tgt, size, ref in (("intra", x["feats"], IMG_HW, intra), ("inter", x["feats_pos"], POS_HW, inter)):
        o = HO.heatmaps(x["feats"], tgt, x["query_points"], size)[0]
        print(name, "oracle vs reference max |diff| %.3e" % float((o - ref.double()).abs().max()))


if __name__ == "__main__":
    main()
