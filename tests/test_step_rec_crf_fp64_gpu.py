"""The reconstruction and CRF terms (cfg.rec_weight, cfg.crf_weight with cfg.fused_rec_crf) inside the hand-scheduled
training step, against float64 stage by stage on the replayed CUDA graph, across the configurations and modes the step
accepts (the REC_CRF_ROWS table in tests/_step_fp64.py: each base row with the reconstruction term alone, the CRF term
alone and both).

Every row runs test_step_configs_fp64_gpu.run_row (fused path taken; the autograd twin's first step leaves both
generators where the fused step left them, with bit-equal positive terms, cd means and cluster loss and every gradient,
the decoder's included, within 3e-3 relative L2; eager step, capture, replay; the replayed step against
tests/_step_fp64.compose stage by stage; the Adam update of every group).  What the terms add to that check, on the
replayed step's own inputs (bars: tests/test_rec_crf_step_gpu.py):

  rec     ws.rec_dcos is autograd's fl(fl(-w) / (B hw)); rec_cos / rec_nr / rec_nf against
          _rec_crf_fp64.rec_term on ws.code's img rows, the img rows of the backbone tokens, ws.M3's img rows (None
          with dropout off) and the decoder snapshotted before the step, at rec_bars; loss/rec the kernel's fixed-order
          mean of its own cosines, against the fp64 mean within mean(cos bar) + u |loss|; the decoder's dW / db, read
          from the flat gradient buffer, at rec_bars' dW / db.
  crf     ws.crf_g is autograd's fl(fl(w) / (B n^2)); ws.crf_gsel bit-equal to F.interpolate(img, 56) at this step's
          ws.crf_coords (the guidance runs outside the graph, on the coordinates the replayed prologue drew); ws.crf_raw
          bit-equal to F.interpolate(code, 56) at the samples, with the step's channels-last code strides; sel and the
          norms at their bars; loss/crf at crf_loss_bars on the kernel's own sel / gsel, and end to end from the code.
  d(code) the img rows hold the correspondence loss's gather, the aug scatter (aug rows), the reconstruction
          backward's one add per 64-channel chunk and the CRF scatter's atomics: one bar of the sum of the stages'
          bars plus the cross terms of sharing the fp32 accumulators (each addition of one stage rounds against the
          other stages' sums of |contributions| too: u (A_all - A_own) per addition); the img_pos rows hold the
          correspondence loss's alone, at its bar.
  total   w_rec rec and w_crf crf at their fp64 bars, one product and one more rounding of the total per term.
  decoder the decoder's parameters sit in the net optimiser's group (the flat buffer's first group, at cfg.lr), as the
          reference puts them (train_segmentation.py:376-377), so they take the same Adam step count.

Each row also asserts that it runs what it names (test_step_modes_fp64_gpu._claims, plus the terms, M3, the frame
and the number of CRF samples).  Largest error / bar ratios go to $STEGO_PARITY_DIR when it is set.
"""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _step_fp64 as S  # noqa: E402
from _parity_util import fp32_strict, record  # noqa: E402
from test_step_configs_fp64_gpu import run_row  # noqa: E402
from test_step_modes_fp64_gpu import _claims  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture
def strict_fp32():
    """The autograd twin's decoder conv in fp32, not TF32; the previous settings are restored afterwards."""
    saved = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32, torch.get_float32_matmul_precision())
    fp32_strict()
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved[:2]
    torch.set_float32_matmul_precision(saved[2])


def _rec_crf_claims(row, model, batches):
    """the row runs the terms it names, with or without m3, at its frame and CRF sample count"""
    cfg, ws = model.cfg, model._fused.ws
    B, E, D, P, fh, fw, hw, M, nonlinear = ws.dims
    rec, crf = cfg.rec_weight > 0, cfg.crf_weight > 0
    assert (ws.rec, ws.crf) == (rec, crf) and (rec or crf)
    assert (ws.M3 is None) == (not cfg.dropout)
    H, W = row["frame"]
    assert tuple(batches[0]["img"].shape) == (row["B"], 3, H, W)
    assert (fh, fw) == (H // row["patch"], W // row["patch"])
    if crf:
        assert ws.crf_coords.shape == (2, cfg.crf_samples) and ws.crf_gsel.shape[1] == -(-cfg.crf_samples // 64) * 64
        assert "loss/crf" in model.logged
    else:
        assert not hasattr(ws, "crf_coords") and "loss/crf" not in model.logged
    if rec:
        assert "loss/rec" in model.logged
        flat = model._flat
        grp = flat.groups[0]
        assert grp.lr == cfg.lr and flat.optimizers[0].param_groups[0]["lr"] == cfg.lr
        for p in (model.decoder.weight, model.decoder.bias):
            assert any(p is q for q in grp.params), "decoder outside the net optimiser's group"
            off = (p.data_ptr() - flat.param.data_ptr()) // 4
            assert grp.start <= off and off + p.numel() <= grp.start + grp.numel
    else:
        assert "loss/rec" not in model.logged


@pytest.mark.parametrize("name", list(S.REC_CRF_CONFIGS))
def test_step_rec_crf(cuda_dev, strict_fp32, name, monkeypatch):
    row = S.REC_CRF_CONFIGS[name]
    out = run_row(row, name, cuda_dev, monkeypatch)
    _claims(name, row, out["fused"], out["batches"])
    _rec_crf_claims(row, out["fused"], out["batches"])
    record(f"step_rec_crf_{name}_twin", out["twin_rel"])
    out["ratios"].check(f"step_rec_crf_fp64_{name}")
