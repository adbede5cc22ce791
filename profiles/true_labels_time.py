"""Cost of the use_true_labels teacher signal (train_segmentation.py:135-140) on the card it runs on.

    python profiles/true_labels_time.py [--out FILE]

Prints one JSON line with the card name and power limit read in the same run.
  * `tiles`: corr.build_label_tiles (the label maps read directly, 7 slots) against the reference's op sequence in
    PyTorch eager: one_hot_feats(label + 1, n + 1) x2 (utils.py:65-66), then for the 7 slots the sampling and norm of
    modules.py:275-288, 372-386 (grid_sample on signal, signal_pos and five signal[perm] gathers, F.normalize), at the
    c1-c3 batch / label shapes (label resolution = image resolution), fs 11, 27 classes.  CUDA-event times over >= 0.5 s
    after a warm-up; bytes are the HBM writes of each side computed from the shapes.
  * `step`: c1 training_step images/s (fused step, graph replay, inputs resident on the device), use_true_labels off
    and on, alternated in one process.
"""
import argparse
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
from _measure import call_ms, card, emit, window_ms  # noqa: E402

N_CLASSES, FS, N_NEG = 27, 11, 5
SHAPES = {"c1": (32, 224), "c2": (32, 320), "c3": (16, 448)}  # batch, label / image resolution
WINDOW = dict(warmup=3, min_window_s=0.5, min_iters=10)


def eager_signal(label, label_pos, c1, c2, perms):
    """train_segmentation.py:135-137 + modules.py:372-386's sampling of the signal, and helper's norm (:332)."""
    sig = F.one_hot(label + 1, N_CLASSES + 1).permute(0, 3, 1, 2).to(torch.float32)
    sig_pos = F.one_hot(label_pos + 1, N_CLASSES + 1).permute(0, 3, 1, 2).to(torch.float32)
    sample = lambda t, c: F.grid_sample(t, c.permute(0, 2, 1, 3), padding_mode="border", align_corners=True)
    out = [F.normalize(sample(sig, c1), dim=1, eps=1e-10), F.normalize(sample(sig_pos, c2), dim=1, eps=1e-10)]
    for p in perms:
        out.append(F.normalize(sample(sig[p], c2), dim=1, eps=1e-10))
    return out


def tiles_case(name, dev):
    from stego_b200 import corr
    from stego_b200.config import make_cfg
    B, res = SHAPES[name]
    g = torch.Generator().manual_seed(0)
    label = torch.randint(-1, N_CLASSES, (B, res, res), generator=g).to(dev)
    label_pos = torch.randint(-1, N_CLASSES, (B, res, res), generator=g).to(dev)
    c1 = (torch.rand(B, FS, FS, 2, generator=g) * 2 - 1).to(dev)
    c2 = (torch.rand(B, FS, FS, 2, generator=g) * 2 - 1).to(dev)
    perms = torch.stack([torch.randperm(B, generator=g) for _ in range(N_NEG)]).to(dev)
    spec = corr.make_spec(make_cfg())
    out = torch.empty(2, spec.nslots, B, spec.rows, corr.teacher_width(N_CLASSES + 1), dtype=torch.bfloat16, device=dev)
    ours_ms, ours_n = window_ms(lambda: corr.build_label_tiles(label, label_pos, c1, c2, perms, spec, N_CLASSES,
                                                               raw_perms=True, out=out), **WINDOW)
    eager_ms, eager_n = window_ms(lambda: eager_signal(label, label_pos, c1, c2, perms), **WINDOW)
    C, S, px = N_CLASSES + 1, FS * FS, B * res * res
    eager_bytes = 2 * px * C * 8 + 2 * px * C * 4 + N_NEG * px * C * 4 + 2 * 7 * B * C * S * 4  # one_hot, float, gathers,
    ours_bytes = out.numel() * 2                                                             # samples + normalised
    return dict(shape=name, B=B, label_res=res, n_classes=N_CLASSES, fs=FS, ours_ms=round(ours_ms, 4), ours_calls=ours_n,
                eager_ms=round(eager_ms, 4), eager_calls=eager_n, speedup=round(eager_ms / ours_ms, 1),
                ours_hbm_write_mb=round(ours_bytes / 1e6, 3), eager_hbm_write_mb=round(eager_bytes / 1e6, 1))


def step_case(dev, rounds=4, steps=30):
    import stego_oracle as O
    from stego_b200.config import make_cfg
    from stego_b200.segmenter import LitUnsupervisedSegmenter
    B, res = SHAPES["c1"]
    g = torch.Generator().manual_seed(1)
    batch = dict(img=torch.randn(B, 3, res, res, generator=g).to(dev),
                 img_pos=torch.randn(B, 3, res, res, generator=g).to(dev),
                 label=torch.randint(-1, N_CLASSES, (B, res, res), generator=g).to(dev),
                 label_pos=torch.randint(-1, N_CLASSES, (B, res, res), generator=g).to(dev))
    sd = O.perturb_vit_state(O.vit_random_state("vit_small", 8, seed=3))
    models = {}
    for on in (False, True):
        torch.manual_seed(0)
        m = LitUnsupervisedSegmenter(N_CLASSES, make_cfg(random_backbone_init=True, use_true_labels=on)).to(dev)
        m.net.model.load_state_dict(sd)
        m.train()
        m.configure_optimizers()
        for s in range(3):  # eager, capture, replay
            m.training_step(batch, s)
        models[on] = m

    def run(m):
        for i in range(steps):
            m.training_step(batch, i)
        m.flush()

    rates = {False: [], True: []}
    for _ in range(rounds):
        for on in (False, True):
            torch.cuda.synchronize()
            rates[on].append(round(B * steps / (call_ms(lambda: run(models[on]))[0] / 1e3), 1))
    assert models[True]._fused.step_idx == 3 + rounds * steps
    return dict(shape="c1", B=B, res=res, steps_per_round=steps, images_per_s_true_labels_off=rates[False],
                images_per_s_true_labels_on=rates[True])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from stego_b200 import _lib
    _lib.load()
    dev = torch.device("cuda:0")
    emit(dict(card=card(), tiles=[tiles_case(n, dev) for n in SHAPES], step=step_case(dev), gpu_info_after=card()),
         args.out)


if __name__ == "__main__":
    main()
