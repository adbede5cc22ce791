"""Generate tests/golden/correspondence_pr.pt from the REAL reference's correspondence precision-recall lines.

    STEGO_REFERENCE_SRC=<reference checkout>/src python oracle/make_golden_correspondence.py

src/plot_pr_curves.py cannot be imported (hydra, seaborn, Lightning) nor run as written (`self.dino` and `self.crf`
are commented out but used).  So its statements are lifted as TEXT and executed: `LitRecalibrator.get_net_fd`
(:108-121) with the reference's own `sample`, `norm` and `tensor_correlation` (src/modules.py), `prep_fd` (:34-37) and
`plot_pr` (:160-167, nested in validation_epoch_end), whose `average_precision_score` call is recorded.

Inputs: a random-init ViT-S/8 (oracle/stego_oracle.py) on 2 seeded 56 x 56 images and the seeded segmentation head's
code (dim 70), both rounded to bf16 values before the reference sees them (so the file stores them as bf16 without
loss), piecewise-constant labels in -1 .. n_classes - 1 with n_classes = 5 (stored as int8), and the reference's
coordinate draws `torch.rand([B, fs, fs, 2]) * 2 - 1` at fs = 11, as validation_step (:134-136) makes them.
Stored: the inputs, fd of both methods ("code" = "STEGO (Ours)", "feats" = "DINO"), ld, and per method the AP with the
reference's targets (`ld.to(int64)`, after prep_fd) and with the exact rule (both samples pure with the same class, on
the raw fd).
correspondence_oracle.load_golden reads the file back as fp32 / int64.
"""
from __future__ import annotations

import ast
import os
import sys
import textwrap
import types

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import correspondence_oracle as CO  # noqa: E402
import reference_shim  # noqa: E402
import stego_oracle as O  # noqa: E402

OUT = os.path.join(HERE, "..", "tests", "golden", "correspondence_pr.pt")
B, RES, FS, N_CLASSES, DIM = 2, 56, 11, 5, 70


def inputs():
    """Seeded features, code, labels and coordinates (pure torch, no reference)."""
    g = torch.Generator().manual_seed(11)
    img = torch.randn(B, 3, RES, RES, generator=g)
    sd = O.vit_random_state("vit_small", 8, seed=0)
    with torch.no_grad():
        feats = O.vit_image_feat(sd, img, "vit_small", 8).contiguous()
        code = O.head_forward(feats, O.head_random_state(384, DIM, seed=0), None)[1].contiguous()
    feats, code = feats.to(torch.bfloat16).float(), code.to(torch.bfloat16).float()
    # piecewise-constant labels: a background class and 6 rectangles per image, labels -1 .. N_CLASSES - 1
    label = torch.randint(-1, N_CLASSES, (B, 1, 1), generator=g).expand(B, RES, RES).clone()
    for b in range(B):
        for _ in range(6):
            y0, x0 = torch.randint(0, RES - 8, (2,), generator=g).tolist()
            h, w = torch.randint(6, 28, (2,), generator=g).tolist()
            label[b, y0:y0 + h, x0:x0 + w] = int(torch.randint(-1, N_CLASSES, (1,), generator=g))
    coords1 = torch.rand([B, FS, FS, 2], generator=g) * 2 - 1
    coords2 = torch.rand([B, FS, FS, 2], generator=g) * 2 - 1
    return dict(feats=feats, code=code, label=label, coords1=coords1, coords2=coords2)


def _lift(text, tree, name, cls=None, parent=None):
    for node in ast.walk(tree):
        if cls and isinstance(node, ast.ClassDef) and node.name == cls:
            node = next(n for n in node.body if isinstance(n, ast.FunctionDef) and n.name == name)
            return textwrap.dedent(ast.get_source_segment(text, node, padded=True))
        if parent and isinstance(node, ast.FunctionDef) and node.name == parent:
            node = next(n for n in ast.walk(node) if isinstance(n, ast.FunctionDef) and n.name == name)
            return textwrap.dedent(ast.get_source_segment(text, node, padded=True))
        if not cls and not parent and isinstance(node, ast.FunctionDef) and node.name == name:
            return ast.get_source_segment(text, node)
    raise KeyError(name)


def reference_lines(x):
    from sklearn.metrics import average_precision_score, precision_recall_curve
    modules, _ = reference_shim.import_reference()
    text = open(os.path.join(reference_shim.REFERENCE_SRC, "plot_pr_curves.py")).read()
    tree = ast.parse(text)
    recorded = []

    def ap_score(targets, preds):
        v = average_precision_score(targets, preds)
        recorded.append(float(v))
        return v

    plt = types.SimpleNamespace(plot=lambda *a, **k: None)
    env = dict(torch=torch, F=F, sample=modules.sample, norm=modules.norm,
               tensor_correlation=modules.tensor_correlation, precision_recall_curve=precision_recall_curve,
               average_precision_score=ap_score, plt=plt)
    for src in (_lift(text, tree, "get_net_fd", cls="LitRecalibrator"), _lift(text, tree, "prep_fd"),
                _lift(text, tree, "plot_pr", parent="validation_epoch_end")):
        exec(src, env)
    me = types.SimpleNamespace(n_classes=N_CLASSES)
    out = {}
    lab, c1, c2 = x["label"], x["coords1"], x["coords2"]
    # validation_step :140-141
    ld, stego_fd, _, _ = env["get_net_fd"](me, x["code"], x["code"], lab, lab, c1, c2)
    ld, dino_fd, _, _ = env["get_net_fd"](me, x["feats"], x["feats"], lab, lab, c1, c2)
    out["ld"] = ld
    out["fd"] = {"code": stego_fd.clone(), "feats": dino_fd.clone()}
    # validation_epoch_end :208-209
    env["plot_pr"](env["prep_fd"](stego_fd.clone()), ld, "STEGO (Ours)")
    env["plot_pr"](env["prep_fd"](dino_fd.clone()), ld, "DINO")
    out["ap_reference"] = {"code": recorded[0], "feats": recorded[1]}
    return out


def main():
    torch.set_num_threads(1)
    x = inputs()
    ref = reference_lines(x)
    exact = CO.exact_targets(x["label"], N_CLASSES, x["coords1"], x["coords2"])
    ap_exact = {m: CO.average_precision(ref["fd"][m].numpy(), exact.numpy()) for m in ("code", "feats")}
    stored = dict(x, feats=x["feats"].to(torch.bfloat16), code=x["code"].to(torch.bfloat16),
                  label=x["label"].to(torch.int8))
    torch.save(dict(n_classes=N_CLASSES, **stored, fd=ref["fd"], ld=ref["ld"], ap_reference=ref["ap_reference"],
                    ap_exact=ap_exact), OUT)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")
    n_ref = int(ref["ld"].to(torch.int64).sum())
    print("positives: reference", n_ref, "exact", int(exact.sum()), "of", exact.numel())
    for m in ("code", "feats"):
        print(m, "AP reference %.6f exact %.6f diff %.3e" % (ref["ap_reference"][m], ap_exact[m],
                                                             ap_exact[m] - ref["ap_reference"][m]))


if __name__ == "__main__":
    main()
