"""Generate tests/golden/cd_histograms.pt from the REAL reference: the histograms its training step logs.

    STEGO_REFERENCE_SRC=<reference checkout>/src python oracle/make_golden_cd_hist.py

src/train_segmentation.py:112-245 (text unmodified, stub-Lightning base, oracle/lightning_harness.py) on the CPU at
ViT-S/8, B = 2, 64x64 images, with hist_freq = 1 at global_step = 1, so that should_log_hist holds (:142-144).  The
harness's no-op logger is replaced, for this run only, by one that records every `add_histogram(tag, values, step)`
call (:165-168).  Stored: the tags and steps, the value tensors (the cd of the three loss groups), what
torch.utils.tensorboard.summary.make_histogram makes of them with the writer's default bins, and those bins.
"""
from __future__ import annotations

import os
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import lightning_harness as H  # noqa: E402
import make_golden as MG  # noqa: E402

OUT = os.path.join(HERE, "..", "tests", "golden", "cd_histograms.pt")


def default_bins():
    """writer.py's SummaryWriter.default_bins, restated without creating a log directory."""
    v, pos, neg = 1e-12, [], []
    while v < 1e20:
        pos.append(v)
        neg.append(-v)
        v *= 1.1
    return neg[::-1] + [0] + pos


class _RecordingExperiment:
    def __init__(self):
        self.calls = []

    def add_histogram(self, tag, values, global_step=None, *a, **k):
        self.calls.append((tag, values.detach().clone(), global_step))


def main():
    from torch.utils.tensorboard.summary import make_histogram
    sys.path.insert(0, os.path.join(HERE, ".."))
    from stego_b200.config import make_cfg
    ts = H.load_reference_segmenter("reference")
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    with tempfile.TemporaryDirectory() as td:
        ck = os.path.join(td, "dino.pth")
        H.write_random_dino_checkpoint(ck, "vit_small")
        cfg = make_cfg(pretrained_weights=ck, hist_freq=1)
        torch.manual_seed(0)
        m = ts.LitUnsupervisedSegmenter(27, cfg)
    params = dict(m.named_parameters())
    with torch.no_grad():
        for k, v in MG.step_params().items():
            params[k].copy_(v)
    m.train()
    exp = _RecordingExperiment()
    m.logger = types.SimpleNamespace(experiment=exp)
    m.global_step = 1
    torch.manual_seed(777)
    m.training_step(H.make_batch(MG.STEP_B, MG.STEP_RES, "cpu"), 0)
    bins = default_bins()
    records = []
    for tag, values, step in exp.calls:
        h = make_histogram(values.numpy().astype(float), bins)
        records.append(dict(tag=tag, step=step, values=values, min=h.min, max=h.max, num=h.num, sum=h.sum,
                            sum_squares=h.sum_squares, bucket_limit=list(h.bucket_limit), bucket=list(h.bucket)))
    torch.save(dict(recipe="oracle/make_golden_cd_hist.py", default_bins=torch.tensor(np.array(bins, dtype=np.float64)),
                    records=records), OUT)
    print(OUT, os.path.getsize(OUT), [(r["tag"], tuple(r["values"].shape), r["num"]) for r in records])


if __name__ == "__main__":
    main()
