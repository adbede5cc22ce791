"""Training-step time with the last block's keys as the teacher (dino_feat_type "KK") against the final-norm tokens
("feat"), on the card it runs on.

    python profiles/kk_step_time.py [--out FILE]

Prints one JSON line with the card name and power limit read in the same run.  For c1 (ViT-S/8 224², B = 32) and c2
(ViT-B/8 320², B = 32, one GPU): two models that differ only in dino_feat_type, each warmed up through eager step, graph
capture and replay, then timed alternately (rounds of `steps` fused training steps, inputs resident on the device,
CUDA events around each round, the overlapped parameter update flushed before the end event).  A "KK" step runs the
last block only to LN1 and the key third of its qkv GEMM; everything after the backbone is the same work.
"""
import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
from _measure import call_ms, card, emit  # noqa: E402

N_CLASSES = 27
SHAPES = {"c1": ("vit_small", 224, 32), "c2": ("vit_base", 320, 32)}


def step_case(name, dev, rounds=4, steps=20):
    import stego_oracle as O
    from stego_b200.config import make_cfg
    from stego_b200.segmenter import LitUnsupervisedSegmenter
    arch, res, B = SHAPES[name]
    g = torch.Generator().manual_seed(1)
    batch = dict(img=torch.randn(B, 3, res, res, generator=g).to(dev),
                 img_pos=torch.randn(B, 3, res, res, generator=g).to(dev),
                 label=torch.randint(-1, N_CLASSES, (B, res, res), generator=g).to(dev))
    sd = O.perturb_vit_state(O.vit_random_state(arch, 8, seed=3))
    kinds = ("feat", "KK")
    models = {}
    for kind in kinds:
        torch.manual_seed(0)
        m = LitUnsupervisedSegmenter(N_CLASSES, make_cfg(model_type=arch, random_backbone_init=True,
                                                         dino_feat_type=kind)).to(dev)
        m.net.model.load_state_dict(sd)
        m.train()
        m.configure_optimizers()
        for s in range(3):  # eager, capture, replay
            m.training_step(batch, s)
        assert m._fused is not None and m._fused.ws.graph is not None, kind
        models[kind] = m

    def run(m):
        for i in range(steps):
            m.training_step(batch, i)
        m.flush()

    ms = {k: [] for k in kinds}
    for _ in range(rounds):
        for kind in kinds:
            torch.cuda.synchronize()
            ms[kind].append(round(call_ms(lambda: run(models[kind]))[0] / steps, 3))
    best = {k: min(v) for k, v in ms.items()}
    out = dict(shape=name, arch=arch, res=res, B=B, steps_per_round=steps, ms_per_step_feat=ms["feat"],
               ms_per_step_kk=ms["KK"], best_ms_feat=best["feat"], best_ms_kk=best["KK"],
               kk_over_feat_best=round(best["KK"] / best["feat"], 4))
    del models
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from stego_b200 import _lib
    _lib.load()
    dev = torch.device("cuda:0")
    emit(dict(card=card(), steps=[step_case(n, dev) for n in SHAPES], gpu_info_after=card()), args.out)


if __name__ == "__main__":
    main()
