"""The hand-scheduled training step (fused_step.FusedStep) in its optional modes, alone and crossed with the
configurations of tests/test_step_configs_fp64_gpu.py (the MODE_ROWS table in tests/_step_fp64.py): feature_samples
12..64 (the multi-tile loss), use_true_labels (the one-hot label teacher of sample_labels_kernel), use_salience,
dino_feat_type "KK", the aug-alignment term (views, aug_align.cu and the cosine inside the step's graph) and the cd
histograms (the second tail graph, binning cd in the correlation epilogue), and all of them in one captured graph.

Every row runs test_step_configs_fp64_gpu.run_row: the fused path is taken; the autograd twin's first step from the same
generator states leaves both generators where the fused step left them, draws bit-equal coordinates and gives bit-equal
positive terms, cd means and cluster loss; NaN-filled code tiles have no effect; eager step, capture, replay, with the
replayed step checked stage by stage against the float64 composition of tests/_step_fp64.py and its Adam update
checked.  What the modes add to that check:

  fs 12..64   tiles of R = ceil(S / 128) 128 rows, rows >= S exactly zero; call stats and d(code) at CorrRef's bars.
  labels      the teacher tiles against the fp64 one-hot sample (gather_sample and the split bar), channels >= n + 1
              exactly zero; int64, int32 and uint8 labels.
  salience    ws.c1 / ws.c2 bit-equal to the coordinates the twin's draw_coords returned; an image whose mask is empty
              (the draw falls back to the CUDA generator) and one whose mask is full.
  "KK"        the tokens of the KK backbone graph the step replayed; the rest as for "feat".
  aug         ws.img_aug / ws.coord_aug bit-equal to augment.aug_alignment_views; grid (6 u m), sampled (at the kernel's
              grid), the cosines, d(sampled) and d(code) of the img_aug rows (test_loss_terms_fp64_gpu.cos_bars),
              loss/aug_alignment, d(code) of the img rows (the correspondence loss's bar plus the scatter's and their
              cross terms), the padding columns D..P of ws.code and ws.dall exactly zero, the head backward over 3B
              rows and loss/total with w * aug.
  hist        a logger and hist_freq = 1, so the compared step replays the histogram graph (step 0 is eager and logs
              nothing, step 1 captures the graph); the counts of intra_cd / inter_cd / neg_cd within the fp64 binning's
              per-edge brackets (only elements within their cd bar of an edge may move), the group sizes exact, min /
              max / sum / sum of squares within their bars; the step's losses and gradients at the bars without it.

Each row also asserts that it exercises what it names.  Largest error / bar ratios go to $STEGO_PARITY_DIR when it is
set.
"""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _step_fp64 as S  # noqa: E402
from test_step_configs_fp64_gpu import run_row  # noqa: E402

pytestmark = pytest.mark.gpu


def _claims(name, row, model, batches):
    """the row exercises what it names"""
    from stego_b200 import corr, salience
    cfg, ws, spec = model.cfg, model._fused.ws, model._spec
    B, E, D, P, fh, fw, hw, M, nonlinear = ws.dims
    fs = int(cfg.feature_samples)
    assert spec.fs == fs and spec.ncalls == 2 + cfg.neg_samples
    if fs >= 12:
        assert spec.tiled and spec.rows == -(-fs * fs // 128) * 128 and spec.rows > 128
    if cfg.use_true_labels:
        assert ws.label_pos is not None and ws.ET == corr.teacher_width(model.n_classes + 1)
        assert ws.label.dtype == ws.label_pos.dtype == getattr(torch, row["labels"])
    else:
        assert ws.label_pos is None and ws.ET == E
    if cfg.use_salience:
        assert ws.keep is not None
        if row["masks"] == "uint8_empty_full":
            mask = batches[0]["mask"]
            m, nbytes = salience.mask_view(mask, B)
            cnt = salience.counts(m, m, nbytes).cpu()
            assert cnt[0] == 0 and cnt[1] == mask[1].numel(), cnt
    else:
        assert ws.keep is None
    assert model.net.feat_type == cfg.dino_feat_type
    res = (ws.n_img * B, 3) + tuple(batches[0]["img"].shape[2:])
    assert model.net.model.graph_input(model.net.feat_type, res, batches[0]["img"].device) is not None
    if cfg.aug_alignment_weight > 0:
        assert ws.aug and ws.n_img == 3 and M == 3 * B * hw and ws.code.shape == (M, P)
        assert "loss/aug_alignment" in model.logged
    else:
        assert not ws.aug and ws.n_img == 2
    if row["hist"]:
        assert ws.hist is not None and ws.hist_graph is not None and ws.graph is None
        tags = [t for t, _ in model.logger.experiment.calls]
        assert tags == ["intra_cd", "inter_cd", "neg_cd"] * 2, tags  # steps 1 and 2
    else:
        assert ws.hist is None and ws.graph is not None
    assert (nonlinear, D) == (cfg.projection_type == "nonlinear", model.net.dim)


@pytest.mark.parametrize("name", list(S.MODE_CONFIGS))
def test_step_mode(cuda_dev, name, monkeypatch):
    row = S.MODE_CONFIGS[name]
    out = run_row(row, name, cuda_dev, monkeypatch)
    _claims(name, row, out["fused"], out["batches"])
    from _parity_util import record
    record(f"step_modes_{name}_twin", out["twin_rel"])
    out["ratios"].check(f"step_modes_fp64_{name}")
