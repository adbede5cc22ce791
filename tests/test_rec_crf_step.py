"""CPU: the reconstruction and CRF terms on the hand-scheduled step (cfg.fused_rec_crf).

  * FusedStep.supported(): the switch off refuses both terms as before; on, each term alone and together, with the aug
    seeds, and the CRF term's limits (fp32 img, code dim <= 80);
  * the header declares the new entry points, the library exports them and refuses bad arguments;
  * each new entry point has one call site (as test_step_stages.py checks the others);
  * the fp64 restatements of tests/_rec_crf_fp64.py are pinned to the oracle, the golden file and float64 autograd.
"""
import os

import pytest
import torch
import torch.nn.functional as F

import _loss_terms_fp64 as R
import _rec_crf_fp64 as RC
import test_step_stages
from test_aug_step import _batch, _model

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def test_supported_truth_table():
    from stego_b200.fused_step import FusedStep
    off = dict(aug_alignment_weight=0.0)
    # the switch off (the default): either term sends the step to the autograd path, exactly as before
    for over in (dict(rec_weight=0.3), dict(crf_weight=0.3), dict(rec_weight=0.3, crf_weight=0.3)):
        assert not FusedStep(_model(**off, **over)).supported(_batch(seed=False))
        assert not FusedStep(_model(**over)).supported(_batch())
    on = dict(fused_rec_crf=True)
    for over in (dict(rec_weight=0.3), dict(crf_weight=0.3), dict(rec_weight=0.3, crf_weight=0.3)):
        assert FusedStep(_model(**off, **on, **over)).supported(_batch(seed=False))
        assert FusedStep(_model(**on, **over)).supported(_batch())                  # with the aug seeds
    # bf16 img: the CRF guidance is the fp32 image; the reconstruction term does not read it
    assert not FusedStep(_model(**off, **on, crf_weight=0.3)).supported(_batch(seed=False, dtype=torch.bfloat16))
    assert FusedStep(_model(**off, **on, rec_weight=0.3)).supported(_batch(seed=False, dtype=torch.bfloat16))
    # the CRF kernels take at most 80 code channels; the reconstruction term up to the step's 96
    assert not FusedStep(_model(**off, **on, crf_weight=0.3, dim=81)).supported(_batch(seed=False))
    assert FusedStep(_model(**off, **on, crf_weight=0.3, dim=80)).supported(_batch(seed=False))
    assert FusedStep(_model(**off, **on, rec_weight=0.3, dim=96)).supported(_batch(seed=False))
    # both terms off: the switch changes nothing
    for sw in (False, True):
        m = FusedStep(_model(**off, fused_rec_crf=sw))
        assert m.supported(_batch(seed=False)) and m.supported(_batch(seed=False, dtype=torch.bfloat16))


def test_rec_crf_rows_take_the_fused_step(monkeypatch):
    """Every batch of tests/_step_fp64.py's REC_CRF_ROWS goes to the fused step, so the GPU rows check the kernels they
    name; a configuration the step refuses belongs with the refusals above.  The salience rows' masks are CPU tensors
    here: their check stands in for salience.masks_supported (the mode rows test the real one on the GPU) and only
    asserts the [B, 1, H, W] frame-sized pair."""
    import _step_fp64 as S
    from stego_b200 import fused_step
    from stego_b200.config import make_cfg
    from stego_b200.segmenter import LitUnsupervisedSegmenter
    from test_aug_step import _CudaImg

    def masks_ok(mask, mask_pos, B, device):
        return tuple(mask.shape) == tuple(mask_pos.shape) == (B, 1) + tuple(frame)
    monkeypatch.setattr(fused_step.salience, "masks_supported", masks_ok)
    assert {n.rsplit("_", 1)[1] for n in S.REC_CRF_ROWS} == {"rec", "crf", "both"}
    for name, row in S.REC_CRF_CONFIGS.items():
        cfg = dict(row["cfg"])
        if cfg.get("aug_alignment_weight", 0) > 0:
            cfg["res"] = row["frame"][0]
        if row["hist"]:
            cfg["hist_freq"] = 1
        model = LitUnsupervisedSegmenter(row["n_classes"], make_cfg(model_type=row["arch"], random_backbone_init=True,
                                                                    dino_patch_size=row["patch"], **cfg))
        model.train()
        assert model.cfg.fused_rec_crf and (model.cfg.rec_weight > 0 or model.cfg.crf_weight > 0), name
        frame = row["frame"]
        for seed in (1, 2):
            b = S.make_batch(row, "cpu", seed=seed)
            b["img"] = _CudaImg(b["img"].shape)
            assert fused_step.FusedStep(model).supported(b), name


def test_default_is_off():
    from stego_b200.config import TRAIN_DEFAULTS
    assert TRAIN_DEFAULTS["fused_rec_crf"] is False


NEW_SYMBOLS = ["stego_rec_fwd", "stego_rec_bwd", "stego_rec_scratch_bytes", "stego_crf_guidance", "stego_crf_mean_fwd",
               "stego_crf_mean_loss", "stego_crf_mean_bwd"]


def test_header_declares_and_library_exports():
    from stego_b200 import _lib
    protos = _lib.header_prototypes()
    rec_in = ["const float*", "long long", "const void*", "long long", "const float*", "int", "const float*",
              "const float*", "long long", "int", "int"]
    assert protos["stego_rec_fwd"] == ("int", rec_in + ["float*"] * 3 + ["void*"])
    assert protos["stego_rec_scratch_bytes"] == ("long long", ["long long", "int", "int"])
    assert protos["stego_rec_bwd"] == ("int", rec_in + ["const float*"] * 4 + ["float*", "long long", "float*",
                                                                             "long long", "float*", "float*", "void*"])
    strides = ["long long"] * 4
    assert protos["stego_crf_guidance"] == ("int", ["const float*"] + strides + ["int"] * 3 +
                                            ["const long long*", "int", "int", "int", "float*", "int*", "void*"])
    assert protos["stego_crf_mean_fwd"] == ("int", ["const float*"] + strides + ["int"] * 3 +
                                            ["const long long*", "int", "int", "int"] + ["float"] * 6 +
                                            ["const float*", "const int*", "float*", "float*", "float*", "double*",
                                             "void*"])
    assert protos["stego_crf_mean_loss"] == ("int", ["const double*", "int", "int", "float", "float*", "float*",
                                                     "void*"])
    assert protos["stego_crf_mean_bwd"] == ("int", ["const float*"] * 4 + ["const int*", "const long long*"] +
                                            ["int"] * 6 + ["float"] * 6 + ["float*", "float*"] + strides + ["void*"])
    lib = _lib.load()
    for name in NEW_SYMBOLS:
        getattr(lib, name)


def test_library_refuses_bad_arguments():
    """Every check runs before any CUDA call, so these return errors on a machine without a GPU too."""
    from stego_b200 import _lib
    lib = _lib.load()
    p = 16  # a non-null stand-in: the argument checks fail before anything is dereferenced
    # null pointers, D > 96, ldc < D
    assert lib.stego_rec_fwd(None, 8, p, 8, None, 1, p, p, 4, 8, 8, p, p, p, None) != 0
    assert lib.stego_rec_fwd(p, 128, p, 8, None, 1, p, p, 4, 8, 97, p, p, p, None) != 0
    assert lib.stego_rec_fwd(p, 4, p, 8, None, 1, p, p, 4, 8, 8, p, p, p, None) != 0
    assert lib.stego_rec_scratch_bytes(0, 8, 8) == 0
    # scratch too small (checked before the launch)
    assert lib.stego_rec_bwd(p, 8, p, 8, None, 1, p, p, 4, 8, 8, p, p, p, p, p, 8, p, 0, p, p, None) != 0
    # C > 80, four guidance channels, n = 0
    assert lib.stego_crf_mean_fwd(p, 0, 0, 0, 0, 81, 28, 28, p, 2, 10, 56, .5, .15, .05, 10., 3., 0., p, p, p, p, p, p,
                                  None) != 0
    assert lib.stego_crf_guidance(p, 0, 0, 0, 0, 4, 224, 224, p, 2, 10, 56, p, p, None) != 0
    assert lib.stego_crf_guidance(p, 0, 0, 0, 0, 3, 224, 224, p, 2, 0, 56, p, p, None) != 0
    assert lib.stego_crf_mean_loss(None, 2, 10, 1.0, p, None, None) != 0
    assert lib.stego_crf_mean_bwd(p, p, p, p, p, p, 2, 81, 10, 28, 28, 56, .5, .15, .05, 10., 3., 0., p, p, 0, 0, 0, 0,
                                  None) != 0


def test_new_entry_points_have_one_call_site(monkeypatch):
    monkeypatch.setattr(test_step_stages, "SHARED_ENTRY_POINTS", NEW_SYMBOLS + ["stego_aug_align_loss"])
    refs = test_step_stages._referencing_functions()
    for name in NEW_SYMBOLS:
        assert len(refs[name]) == 1, f"{name} is called from {sorted(refs[name]) or 'nowhere'}"
    assert refs["stego_rec_fwd"] == {"stego_b200/modules.py:rec_forward"}
    assert refs["stego_rec_bwd"] == {"stego_b200/modules.py:rec_backward"}
    assert refs["stego_crf_guidance"] == {"stego_b200/modules.py:crf_guidance"}
    assert refs["stego_crf_mean_fwd"] == {"stego_b200/modules.py:crf_forward"}
    assert refs["stego_crf_mean_loss"] == {"stego_b200/modules.py:crf_loss"}
    assert refs["stego_crf_mean_bwd"] == {"stego_b200/modules.py:crf_backward"}
    # the reconstruction mean goes through the aug term's fixed-order stage
    assert refs["stego_aug_align_loss"] == {"stego_b200/modules.py:aug_loss"}


# ------------------------------------------------------------------------------------------------
# the fp64 restatements
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("E,D", [(24, 1), (40, 7), (64, 20)])
def test_rec_restatement_matches_float64_autograd(E, D):
    """rec_term against conv2d -> F.normalize -> sum -> mean in float64 autograd, with the step's m3 and a zero r pixel
    (zero weight rows and bias are not needed: a zero code row with zero bias gives r = 0) and a zero feature pixel."""
    g = torch.Generator().manual_seed(E * 100 + D)
    B, h = 2, 3
    code = torch.randn(B, D, h, h, generator=g, dtype=torch.float64)
    feat = torch.randn(B, E, h, h, generator=g, dtype=torch.float64)
    m3 = (torch.rand(B, E, 1, 1, generator=g) > 0.1).double() / 0.9
    W = torch.randn(E, D, 1, 1, generator=g, dtype=torch.float64)
    b = torch.randn(E, generator=g, dtype=torch.float64)
    code[0, :, 0, 0] = 0
    b_case = b.clone()
    feat[1, :, 2, 2] = 0
    wt = 0.7
    cr, Wr, br = (t.clone().requires_grad_(True) for t in (code, W, b_case))
    r = F.conv2d(cr, Wr, br)
    f = feat * m3
    cos = (F.normalize(r, dim=1, eps=R.EPS) * F.normalize(f, dim=1, eps=R.EPS)).sum(1)
    loss = -cos.mean()
    (wt * loss).backward()
    M = B * h * h
    rows = lambda t: t.permute(0, 2, 3, 1).reshape(M, -1)
    out = RC.rec_term(rows(code), rows(feat), rows(m3.expand(B, E, h, h)), W.view(E, D), b_case, -wt / M, eps=R.EPS)
    assert torch.allclose(out["cos"], cos.detach().reshape(M), rtol=0, atol=1e-13)
    assert torch.allclose(out["loss"], loss.detach(), rtol=1e-13, atol=0)
    assert torch.allclose(out["dcode"], rows(cr.grad), rtol=1e-11, atol=1e-14)
    assert torch.allclose(out["dW"], Wr.grad.view(E, D), rtol=1e-11, atol=1e-14)
    assert torch.allclose(out["db"], br.grad, rtol=1e-11, atol=1e-14)


@pytest.mark.parametrize("h,H", [(28, 224), (40, 320), (56, 448), (7, 13)])
def test_crf_restatement_matches_oracle_and_float64_autograd(h, H):
    """crf_term against oracle.contrastive_crf_loss(resize(img, 56), normalize(resize(code, 56)), coords).mean() in
    float64, with the gradient through F.interpolate / F.normalize by autograd; repeated, corner and edge samples."""
    import stego_oracle as O
    g = torch.Generator().manual_seed(h)
    B, C, n, S = 2, 5, 40, 56
    img = torch.randn(B, 3, H, H, generator=g, dtype=torch.float64)
    code = torch.randn(B, C, h, h, generator=g, dtype=torch.float64)
    coords = R.random_coords(n, S, S, g)
    coords[:, :4] = torch.tensor([[0, 0, S - 1, S - 1], [0, S - 1, 0, S - 1]])  # the four corners
    coords[:, 4:8] = coords[:, 8:12]                                            # repeats
    coords[0, 12], coords[1, 13] = 0, S - 1                                     # edges
    params = R.fp32_params(R.PARAMS)
    wt = 0.5
    cr = code.clone().requires_grad_(True)
    rs = lambda t: F.interpolate(t, S, mode="bilinear", align_corners=False)
    out = O.contrastive_crf_loss(rs(img), F.normalize(rs(cr), dim=1, eps=R.EPS), coords, *params)
    loss = out.mean()
    (wt * loss).backward()
    ref = RC.crf_term(img, code, coords, params, wt, eps=R.EPS)
    # the oracle, like the reference, divides the int64 position distances by a Python float, which promotes to fp32:
    # its position exponents carry one fp32 rounding (relative u |t| <= 2^-24 * 2 * 55^2 / (2 * 0.05) ~ 4e-3 absolute in
    # the exponent only where exp is below e^-60000), so the pin is at 1e-6 relative; everything else agrees to fp64
    assert torch.allclose(ref["out"], out.detach(), rtol=1e-6, atol=1e-300)
    assert torch.allclose(ref["loss"], loss.detach(), rtol=1e-6, atol=0)
    assert torch.allclose(ref["dcode"], cr.grad, rtol=1e-6, atol=1e-9 * cr.grad.abs().max().item())


def test_crf_restatement_matches_golden():
    """On the golden inputs (56 x 56 maps, so the resize is the identity, and unit code vectors, so the normalisation
    is too) out and the gradient w.r.t. the normalised code (the scattered d sel) are the reference's."""
    g = torch.load(os.path.join(GOLDEN, "contrastive_crf_loss.pt"))
    torch.manual_seed(51)
    gd = torch.rand(2, 3, 56, 56) * 4 - 2
    cl = F.normalize(torch.randn(2, 70, 56, 56), dim=1)
    torch.manual_seed(52)
    coords = torch.cat([torch.randint(0, 56, size=[1, 300]), torch.randint(0, 56, size=[1, 300])], 0)
    ref = RC.crf_term(gd, cl, coords, (.5, .15, .05, 10.0, 3.0, 0.00), 1.0)
    assert torch.allclose(ref["out"].float().reshape(-1)[::97], g["out_sub"], atol=1e-6)
    assert abs(ref["out_abs"].item() - g["out_abs_sum"].item()) < 1e-5 * g["out_abs_sum"].item()
    grad = R.scatter(ref["dsel"], coords, cl.shape)
    assert torch.allclose(grad.float().reshape(-1)[::53], g["grad_sub"], atol=1e-9, rtol=1e-5)
