"""Cost of the use_salience coordinate draws (src/modules.py:298-311, 357-364) on the card it runs on.

    python profiles/salience_time.py [--out FILE]

Prints one JSON object with the card name and power limit read in the same run.
  * `coords`: salience.salience_coords (one kernel + three torch.rand draws, no host synchronisation) against the
    autograd step's torch restatement (ContrastiveCorrelationLoss.draw_coords: torch.nonzero, then per image a boolean
    index and a randint, for both maps) on the same masks: c1 (B = 32, 224², fp32 and uint8 masks), c3 (B = 16, 448²),
    c1 with fs 64, and one 1024x2048 map (the bitmap in caller scratch).  Masks hold ~3 % salient pixels with one empty
    image per batch.  Kernel path: CUDA-event time over >= 0.5 s after a warm-up; torch path: host clock over 20 calls
    from an idle device (it waits for the device 2B + 2 times per call).
  * `step`: c1 training_step images/s (inputs resident on the device): the shipped configuration, use_salience on the
    fused step (graph replay), and use_salience with fused_step = False, alternated in one process.
"""
import argparse
import os
import sys
from types import SimpleNamespace

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
from _measure import call_ms, card, emit, host_ms, window_ms  # noqa: E402

N_CLASSES = 27
CASES = [("c1", 32, 224, 224, 11, torch.float32), ("c1_uint8", 32, 224, 224, 11, torch.uint8),
         ("c3", 16, 448, 448, 11, torch.float32), ("c1_fs64", 32, 224, 224, 64, torch.float32),
         ("map_1024x2048", 1, 1024, 2048, 11, torch.float32)]
WINDOW = dict(warmup=3, min_window_s=0.5, min_iters=10)


def masks(B, H, W, dtype, g):
    m = (torch.rand(B, 1, H, W, generator=g) < 0.03).float()
    m[0] = 0
    return m.to(dtype)


def coords_case(name, B, H, W, fs, dtype, dev):
    from stego_b200 import modules, salience
    g = torch.Generator().manual_seed(0)
    sal, sal_pos = masks(B, H, W, dtype, g).to(dev), masks(B, H, W, dtype, g).to(dev)
    lossfn = modules.ContrastiveCorrelationLoss(SimpleNamespace(use_salience=True, feature_samples=fs))
    feats = torch.empty(B, 1, device=dev)
    torch_draws = lambda: lossfn.draw_coords(feats, sal.to(torch.float32).squeeze(1),
                                             sal_pos.to(torch.float32).squeeze(1))
    ours_ms, ours_n = window_ms(lambda: salience.salience_coords(sal, sal_pos, fs), **WINDOW)
    torch_draws()
    torch_ms = host_ms(torch_draws, 20)
    return dict(case=name, B=B, H=H, W=W, fs=fs, mask_dtype=str(dtype).replace("torch.", ""),
                ours_ms=round(ours_ms, 4), ours_calls=ours_n, torch_ms=round(torch_ms, 3), torch_calls=20,
                speedup=round(torch_ms / ours_ms, 1))


def step_case(dev, rounds=4, steps=30):
    import stego_oracle as O
    from stego_b200.config import make_cfg
    from stego_b200.segmenter import LitUnsupervisedSegmenter
    B, res = 32, 224
    g = torch.Generator().manual_seed(1)
    batch = dict(img=torch.randn(B, 3, res, res, generator=g).to(dev),
                 img_pos=torch.randn(B, 3, res, res, generator=g).to(dev),
                 label=torch.randint(-1, N_CLASSES, (B, res, res), generator=g).to(dev),
                 mask=masks(B, res, res, torch.float32, g).to(dev), mask_pos=masks(B, res, res, torch.float32, g).to(dev))
    sd = O.perturb_vit_state(O.vit_random_state("vit_small", 8, seed=3))
    variants = {"shipped": dict(), "salience_fused": dict(use_salience=True),
                "salience_autograd": dict(use_salience=True, fused_step=False)}
    models = {}
    for name, over in variants.items():
        torch.manual_seed(0)
        m = LitUnsupervisedSegmenter(N_CLASSES, make_cfg(random_backbone_init=True, **over)).to(dev)
        m.net.model.load_state_dict(sd)
        m.train()
        m.configure_optimizers()
        for s in range(3):  # eager, capture, replay
            m.training_step(batch, s)
        models[name] = m

    def run(m):
        for i in range(steps):
            m.training_step(batch, i)
        m.flush()

    rates = {k: [] for k in variants}
    for _ in range(rounds):
        for name in variants:
            torch.cuda.synchronize()
            rates[name].append(round(B * steps / (call_ms(lambda: run(models[name]))[0] / 1e3), 1))
    assert models["salience_fused"]._fused.step_idx == 3 + rounds * steps
    assert models["salience_autograd"]._fused is None
    return dict(shape="c1", B=B, res=res, steps_per_round=steps,
                **{f"images_per_s_{k}": v for k, v in rates.items()})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from stego_b200 import _lib
    _lib.load()
    dev = torch.device("cuda:0")
    emit(dict(card=card(), coords=[coords_case(*c, dev) for c in CASES], step=step_case(dev), gpu_info_after=card()),
         args.out, indent=1)


if __name__ == "__main__":
    main()
