"""CPU: the aug-alignment term on the hand-scheduled step, fed by per-sample seeds (batch["seed"]).

  * FusedStep.supported(): seeds without views only, fp32 img at cfg.res x cfg.res, no rec / crf term;
  * argument errors of both paths (the seeds, a bf16 img) are raised before anything is enqueued;
  * the header declares the sampling / loss entry points and the library exports them;
  * the cosine and aug-alignment entry points each have one call site (as test_step_stages.py checks the others).
"""
import pytest
import torch

import test_step_stages

RES = 32


class _CudaImg:
    """Stands for a CUDA img in supported(), which reads only metadata."""

    def __init__(self, shape, dtype=torch.float32):
        self.shape, self.dtype, self.is_cuda, self.device = torch.Size(shape), dtype, True, torch.device("cuda", 0)

    def dim(self):
        return len(self.shape)


def _model(**over):
    from stego_b200.config import make_cfg
    from stego_b200.segmenter import LitUnsupervisedSegmenter
    cfg = make_cfg(**{**dict(random_backbone_init=True, res=RES, aug_alignment_weight=0.5), **over})
    torch.manual_seed(0)
    m = LitUnsupervisedSegmenter(27, cfg)
    m.train()
    return m


def _batch(B=2, res=RES, dtype=torch.float32, seed=True, views=False, cuda_img=True):
    img = _CudaImg((B, 3, res, res), dtype) if cuda_img else torch.randn(B, 3, res, res).to(dtype)
    b = dict(img=img, img_pos=img, label=torch.zeros(B, res, res, dtype=torch.long))
    if seed is not False:
        b["seed"] = [11, 12][:B] if seed is True else seed
    if views:
        b["img_aug"] = torch.zeros(B, 3, res, res)
        b["coord_aug"] = torch.zeros(B, res, res, 2)
    return b


def test_supported_truth_table():
    from stego_b200.fused_step import FusedStep
    fs = FusedStep(_model())
    assert fs.supported(_batch())
    assert fs.supported(_batch(seed=torch.tensor([3, 4])))              # a collated CPU tensor
    assert not fs.supported(_batch(seed=False))                         # neither seeds nor views
    assert not fs.supported(_batch(seed=False, views=True))             # the caller's views: autograd path
    assert not fs.supported(_batch(views=True))                         # views and seeds: the views win
    assert not fs.supported(_batch(dtype=torch.bfloat16))               # the views are built from fp32 frames
    assert not fs.supported(_batch(res=2 * RES))                        # img not cfg.res x cfg.res
    assert not fs.supported(dict(_batch(), img=_CudaImg((2, 3, RES, 2 * RES))))
    for over in (dict(rec_weight=0.3), dict(crf_weight=0.3)):
        assert not FusedStep(_model(**over)).supported(_batch())
    # the term off: seeds in the batch change nothing
    off = FusedStep(_model(aug_alignment_weight=0.0))
    assert off.supported(_batch()) and off.supported(_batch(seed=False)) and off.supported(_batch(views=True))


def test_autograd_path_argument_errors():
    from stego_b200.segmenter import aug_views_of
    with pytest.raises(RuntimeError, match="batch\\['seed'\\]"):
        aug_views_of(_batch(seed=False, cuda_img=False), RES)
    with pytest.raises(ValueError, match="bfloat16"):
        aug_views_of(_batch(dtype=torch.bfloat16, cuda_img=False), RES)
    with pytest.raises(ValueError, match="3 seeds for 2 images"):
        aug_views_of(_batch(seed=[1, 2, 3], cuda_img=False), RES)
    with pytest.raises(ValueError, match="must be an int"):
        aug_views_of(_batch(seed=[1, -2], cuda_img=False), RES)
    with pytest.raises(ValueError, match="integer tensor"):
        aug_views_of(_batch(seed=torch.tensor([1.0, 2.0]), cuda_img=False), RES)
    # the caller's views are taken as they are
    b = _batch(views=True, cuda_img=False)
    assert aug_views_of(b, RES) == (b["img_aug"], b["coord_aug"])


def test_fused_path_argument_errors_before_any_work():
    """run() checks the seeds before it allocates, draws or enqueues anything."""
    from stego_b200.fused_step import FusedStep
    model = _model()
    fs = FusedStep(model)
    for seed, msg in (([1], "1 seeds for 2 images"), ([1, 1 << 64], "must be an int"), (torch.tensor([[1, 2]]), "1-d")):
        batch = _batch(seed=seed, cuda_img=False)
        state = torch.get_rng_state()
        with pytest.raises(ValueError, match=msg):
            fs.run(batch)
        assert torch.equal(torch.get_rng_state(), state) and fs.ws is None


NEW_SYMBOLS = ["stego_aug_align_fwd", "stego_aug_align_bwd", "stego_aug_align_loss"]


def test_header_declares_and_library_exports():
    from stego_b200 import _lib
    protos = _lib.header_prototypes()
    assert protos["stego_aug_align_fwd"] == ("int", ["const float*", "int", "const float*"] + ["long long"] * 4 +
                                             ["int", "int", "int", "float*", "float*", "void*"])
    assert protos["stego_aug_align_bwd"] == ("int", ["const float*", "const float*", "int", "int", "int", "float*"] +
                                             ["long long"] * 4 + ["void*"])
    assert protos["stego_aug_align_loss"] == ("int", ["const float*", "long long", "float", "float*", "float*", "void*"])
    lib = _lib.load()
    for name in NEW_SYMBOLS:
        getattr(lib, name)


def test_library_refuses_bad_arguments():
    from stego_b200 import _lib
    lib = _lib.load()
    assert lib.stego_aug_align_fwd(None, 8, None, 0, 0, 0, 0, 1, 1, 1, None, None, None) != 0
    assert lib.stego_aug_align_bwd(1, 1, 0, 1, 1, 1, 0, 0, 0, 0, None) != 0
    assert lib.stego_aug_align_loss(None, 1, 1.0, None, None, None) != 0


def test_cosine_and_aug_entry_points_have_one_call_site(monkeypatch):
    names = ["stego_cosine_fwd", "stego_cosine_bwd"] + NEW_SYMBOLS
    monkeypatch.setattr(test_step_stages, "SHARED_ENTRY_POINTS", names)
    refs = test_step_stages._referencing_functions()
    for name in names:
        assert len(refs[name]) == 1, f"{name} is called from {sorted(refs[name]) or 'nowhere'}"
    assert refs["stego_cosine_fwd"] == {"stego_b200/modules.py:cosine_forward"}
    assert refs["stego_aug_align_fwd"] == {"stego_b200/modules.py:aug_sample_forward"}
