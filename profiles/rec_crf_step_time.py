"""Training-step time with the reconstruction and CRF terms (rec_weight, crf_weight > 0), on the card it runs on.

    python profiles/rec_crf_step_time.py [--out FILE]

Prints one JSON line with the card name and power limit read in the same run.  For c1 (ViT-S/8 224², B = 32) and c2
(ViT-B/8 320², B = 32, one GPU), seven models from one state, each warmed up through eager step, graph capture and
replay, then timed alternately (`rounds` rounds; per round and case a CUDA-event window of `steps` back-to-back
training steps, inputs resident on the device):

  * shipped         no optional term, the hand-scheduled step;
  * rec_fused       rec_weight 0.7 with fused_rec_crf: the hand-scheduled step;
  * rec_autograd    rec_weight 0.7, the switch off (the default): the autograd path;
  * crf_fused / crf_autograd           the same for crf_weight 0.5 (crf_samples 1000);
  * all_fused / all_autograd           rec 0.7, crf 0.5 and the aug-alignment term (0.6) fed by batch["seed"].

images/s counts the B frames of a step.  enqueue_ms is the host's time to issue one step (from an idle device to the
return of training_step, over `steps` steps).
"""
import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
from _measure import card, emit, enqueue_ms, window_ms  # noqa: E402

N_CLASSES = 27
SHAPES = {"c1": ("vit_small", 224, 32), "c2": ("vit_base", 320, 32)}
REC, CRF, AUG = dict(rec_weight=0.7), dict(crf_weight=0.5), dict(aug_alignment_weight=0.6)
ON = dict(fused_rec_crf=True)
CASES = {"shipped": dict(), "rec_fused": dict(REC, **ON), "rec_autograd": REC, "crf_fused": dict(CRF, **ON),
         "crf_autograd": CRF, "all_fused": dict(REC, **CRF, **AUG, **ON), "all_autograd": dict(REC, **CRF, **AUG)}


def step_case(name, dev, rounds=3, steps=10):
    import stego_oracle as O
    from stego_b200.config import make_cfg
    from stego_b200.segmenter import LitUnsupervisedSegmenter
    arch, res, B = SHAPES[name]
    g = torch.Generator().manual_seed(1)
    base = dict(img=torch.randn(B, 3, res, res, generator=g).to(dev),
                img_pos=torch.randn(B, 3, res, res, generator=g).to(dev),
                label=torch.randint(-1, N_CLASSES, (B, res, res), generator=g).to(dev))
    seeds = [int(s) for s in torch.randint(0, 2 ** 31 - 1, (B,), generator=g)]
    sd = O.perturb_vit_state(O.vit_random_state(arch, 8, seed=3))
    models, batches = {}, {}
    for case, over in CASES.items():
        torch.manual_seed(0)
        m = LitUnsupervisedSegmenter(N_CLASSES, make_cfg(model_type=arch, random_backbone_init=True, res=res,
                                                         **over)).to(dev)
        m.net.model.load_state_dict(sd)
        m.train()
        m.configure_optimizers()
        batches[case] = dict(base, seed=seeds) if case.startswith("all") else base
        for s in range(3):  # eager, capture, replay
            m.training_step(batches[case], s)
        fused = m._fused is not None and m._fused.ws is not None and m._fused.supported(batches[case])
        assert fused == (not case.endswith("autograd")), case
        models[case] = m

    def one(case):
        return lambda: models[case].training_step(batches[case], 0)

    ms = {c: [] for c in CASES}
    enq = {c: [] for c in CASES}
    for _ in range(rounds):
        for case in CASES:
            t, _ = window_ms(one(case), warmup=2, min_window_s=0.5, min_iters=steps)
            models[case].flush()
            ms[case].append(round(t, 3))
            enq[case].append(round(enqueue_ms(one(case), steps), 3))
            models[case].flush()
    best = {c: min(v) for c, v in ms.items()}
    out = dict(shape=name, arch=arch, res=res, B=B, ms_per_step=ms, enqueue_ms_per_step=enq, best_ms=best,
               images_per_s={c: round(B * 1e3 / v, 1) for c, v in best.items()},
               best_enqueue_ms={c: min(v) for c, v in enq.items()})
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
