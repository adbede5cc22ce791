"""CPU: the scene evaluation LitUnsupervisedSegmenter.eval_scene runs (plot_potsdam.py:44-83).

  * oracle/scene_oracle.py, the plain-torch restatement the GPU tests hold eval_scene to, reproduces the reference's own
    lines (tests/golden/scene.pt, written by oracle/make_golden_scene.py): the stitched image and label exactly (the
    tile order of the reference's permutes), the cluster log-probabilities to 1e-5, the confusion counts, the
    Hungarian assignment and the mapped predictions exactly;
  * eval_scene refuses bad arguments before anything is enqueued, and leaves the metrics and the net's modes alone;
  * the header declares the two mosaic entries, the library exports them, and they refuse bad mosaics without a GPU.
"""
import ctypes
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
GOLD = os.path.join(ROOT, "tests", "golden", "scene.pt")


# ================================================================================================
# the oracle against the reference's own lines
# ================================================================================================
def test_oracle_scene_matches_reference_golden():
    import eval_step_oracle as EO
    import make_golden_scene as MG
    import scene_oracle as SO
    import stego_oracle as O
    g = torch.load(GOLD, weights_only=False)
    assert (g["n_classes"], tuple(g["grid"]), g["tile"], g["batch"]) == (MG.N_CLASSES, (MG.R, MG.C), MG.T, MG.BATCH)
    p = MG.params()
    vit = O.perturb_vit_state(O.vit_random_state("vit_small", 8, seed=3))
    head = {k[len("net."):]: v for k, v in p.items() if k.startswith("net.")}
    tiles, label = MG.inputs()
    with torch.no_grad():
        got = SO.scene_loop(lambda im: EO.net_code(vit, head, im), p["linear_probe.weight"], p["linear_probe.bias"],
                            p["cluster_probe.clusters"], tiles, label, (MG.R, MG.C), MG.N_CLASSES, batch=MG.BATCH)
    assert torch.equal(got["image"], g["image"]) and torch.equal(got["label"], g["label"])
    assert got["cluster_probs"].shape == g["cluster_probs"].shape == (MG.N_CLASSES, MG.R * MG.T, MG.C * MG.T)
    assert float((got["cluster_probs"] - g["cluster_probs"]).abs().max()) < 1e-5
    assert torch.equal(got["cluster_stats"], g["cluster_stats"]) and int(g["cluster_stats"].sum()) > 0
    lut = SO.hungarian(got["cluster_stats"], MG.N_CLASSES, 0)
    assert torch.equal(lut, g["assignments"][1].long())
    assert torch.equal(lut[got["cluster_preds"]], g["mapped_preds"].long())


def test_stitch_places_tile_i_at_row_i_div_C_column_i_mod_C():
    import scene_oracle as SO
    R, C, h, w = 3, 5, 4, 6
    tiles = torch.arange(R * C).view(-1, 1, 1, 1).expand(R * C, 2, h, w) * 10 + torch.arange(2).view(1, 2, 1, 1)
    m = SO.stitch(tiles, R, C)
    assert m.shape == (2, R * h, C * w)
    for i in range(R * C):
        blk = m[:, (i // C) * h:(i // C + 1) * h, (i % C) * w:(i % C + 1) * w]
        assert torch.equal(blk, tiles[i])
    # the reference's own permutes (plot_potsdam.py:65-81) at this size
    ref_img = tiles.reshape(R, C, 2, h, w).permute(2, 0, 3, 1, 4).reshape(2, h * R, w * C)
    ref_lab = tiles[:, 0].reshape(R, C, h, w).permute(0, 2, 1, 3).reshape(h * R, w * C)
    assert torch.equal(m, ref_img) and torch.equal(SO.stitch(tiles[:, 0], R, C), ref_lab)


def test_hungarian_with_extra_clusters_matches_unsupervised_metrics():
    import scene_oracle as SO
    from stego_b200.eval import UnsupervisedMetrics
    g = torch.Generator().manual_seed(0)
    m = UnsupervisedMetrics("x/", 4, 3, True)
    m.stats += torch.randint(0, 50, (7, 4), generator=g)
    m.compute()
    clusters = torch.arange(7)
    assert torch.equal(SO.hungarian(m.stats, 4, 3), m.map_clusters(clusters))


# ================================================================================================
# argument errors, before anything is enqueued
# ================================================================================================
def _model(n_classes=5, **over):
    from stego_b200.config import make_cfg
    from stego_b200.segmenter import LitUnsupervisedSegmenter
    torch.manual_seed(0)
    return LitUnsupervisedSegmenter(n_classes, make_cfg(random_backbone_init=True, **over))


def _scene(R=2, C=3, t=32, dtype=torch.int64):
    g = torch.Generator().manual_seed(3)
    return torch.randn(R * C, 3, t, t, generator=g), torch.randint(0, 5, (R * C, t, t), generator=g).to(dtype)


def _refused(model, exc, words, tiles, grid, **kw):
    from stego_b200 import _lib
    stats = (model.test_linear_metrics.stats.clone(), model.test_cluster_metrics.stats.clone())
    modes = [m.training for m in model.modules()]
    launches = _lib.launch_count()
    with pytest.raises(exc) as e:
        model.eval_scene(tiles, grid, **kw)
    for w in words:
        assert w in str(e.value), (w, str(e.value))
    assert _lib.launch_count() == launches
    assert torch.equal(stats[0], model.test_linear_metrics.stats)
    assert torch.equal(stats[1], model.test_cluster_metrics.stats)
    assert modes == [m.training for m in model.modules()]


@pytest.mark.parametrize("run_crf", [False, True])
def test_cpu_tensors_refused(run_crf):
    model = _model()
    tiles, label = _scene()
    _refused(model, RuntimeError, ["CUDA"], tiles, (2, 3), label=label, run_crf=run_crf)
    _refused(model, RuntimeError, ["CUDA"], tiles, (2, 3), run_crf=run_crf, probes=("cluster",))


@pytest.mark.parametrize("grid", [(2, 2), (3, 2, 1), (0, 6), "ab", None])
def test_bad_grid_refused(grid):
    tiles, _ = _scene()
    _refused(_model(), ValueError, ["eval_scene", "grid"], tiles, grid)


@pytest.mark.parametrize("probes", [(), ("cluster", "cluster"), ("linear", "kmeans"), "cluster"])
def test_bad_probes_refused(probes):
    tiles, _ = _scene()
    _refused(_model(), ValueError, ["eval_scene", "probes"], tiles, (2, 3), probes=probes)


@pytest.mark.parametrize("chunk", [0, -1, 2.5, True])
def test_bad_chunk_refused(chunk):
    tiles, _ = _scene()
    _refused(_model(), ValueError, ["chunk"], tiles, (2, 3), chunk=chunk)


def test_tiles_and_labels_refused():
    model = _model()
    tiles, label = _scene()
    for run_crf in (False, True):
        _refused(model, ValueError, ["eval_scene", "patches"], torch.randn(6, 3, 36, 36), (2, 3), run_crf=run_crf)
        _refused(model, ValueError, ["fp32 or bf16"], tiles.double(), (2, 3), run_crf=run_crf)
        _refused(model, ValueError, ["[R*C, 3, H, W]"], tiles[0], (2, 3), run_crf=run_crf)
        _refused(model, ValueError, ["label", "per tile"], tiles, (2, 3), label=label[:, :16], run_crf=run_crf)
        _refused(model, ValueError, ["label", "per tile"], tiles, (2, 3), label=label[:5], run_crf=run_crf)
        _refused(model, ValueError, ["label dtype"], tiles, (2, 3), label=label.float(), run_crf=run_crf)


def test_probe_limits_refused():
    tiles, _ = _scene()
    _refused(_model(projection_type=None), ValueError, ["projection_type None"], tiles, (2, 3))
    _refused(_model(n_classes=30, extra_clusters=3), ValueError, ["33 cluster-probe rows"], tiles, (2, 3),
             run_crf=True, probes=("cluster",))


def test_mosaic_beyond_the_crf_slot_ids_refused():
    """6 lattice slots per pixel must fit the int32 slot ids: a 19000 x 19000 mosaic does not (without the CRF it is
    only refused for being on the CPU)."""
    tiles = torch.empty(1, 3, 8, 8).expand(19000 // 8 * 19000 // 8, 3, 8, 8)  # no storage behind the tiles
    grid = (19000 // 8, 19000 // 8)
    _refused(_model(), ValueError, ["int32 slot ids"], tiles, grid, run_crf=True)
    _refused(_model(), RuntimeError, ["CUDA"], tiles, grid)


@pytest.mark.parametrize("R,C", [(1, 17), (17, 1), (17, 17)])
def test_mosaic_beyond_the_bilateral_key_width_refused(R, C):
    """The bilateral lattice's 12-bit key coordinates bound the mosaic's longer side at about 5380 pixels: 17 tiles of
    320 are refused up front (stego_crf_lattice would refuse them only after the backbone ran), 16 are not."""
    from stego_b200 import crf
    tiles = torch.empty(1, 3, 320, 320).expand(R * C, 3, 320, 320)
    _refused(_model(), ValueError, ["bilateral lattice", "2048"], tiles, (R, C), run_crf=True)
    _refused(_model(), RuntimeError, ["CUDA"], tiles, (R, C))
    bound, limit = crf.lattice_key_bound(16 * 320, 320, 5, crf.Bi_XY_STD, crf.Bi_RGB_STD)
    assert bound < limit and crf.lattice_key_bound(17 * 320, 320, 5, crf.Bi_XY_STD, crf.Bi_RGB_STD)[0] >= limit
    _refused(_model(), RuntimeError, ["CUDA"], tiles[:16], (1, 16), run_crf=True)
    # the kernel's own check refuses the same frame (before any CUDA call; host addresses stand in for the buffers)
    from stego_b200 import _lib
    buf = torch.zeros(16, dtype=torch.int64)
    rc = _lib.load().stego_crf_lattice(320, 17 * 320, 5, crf.Bi_XY_STD, crf.Bi_RGB_STD, buf.data_ptr(), buf.data_ptr(),
                                       buf.data_ptr(), 0)
    assert rc != 0 and "do not fit" in _lib.last_error()


def test_map_clusters_needs_compute_and_the_cluster_probe():
    model = _model()
    tiles, _ = _scene()
    _refused(model, ValueError, ["compute()"], tiles, (2, 3), map_clusters=True)
    model.test_cluster_metrics.stats += 1
    model.test_cluster_metrics.compute()
    _refused(model, ValueError, ["cluster probe"], tiles, (2, 3), map_clusters=True, probes=("linear",))
    _refused(model, RuntimeError, ["CUDA"], tiles, (2, 3), map_clusters=True)


# ================================================================================================
# the C-ABI entries
# ================================================================================================
def test_header_declares_and_library_exports_mosaic_entries():
    from stego_b200 import _lib
    protos = _lib.header_prototypes()
    probes = protos["stego_eval_probes"][1]
    assert protos["stego_eval_probes_mosaic"] == ("int", probes[:-1] + ["int", "int", "int", "long long", "void*"])
    unary = protos["stego_eval_crf_unary"][1]
    assert protos["stego_eval_crf_unary_mosaic"] == ("int", unary[:-1] + ["int", "int", "int", "int", "long long",
                                                                          "void*"])
    lib = ctypes.CDLL(_lib.LIB_PATH)
    assert hasattr(lib, "stego_eval_probes_mosaic") and hasattr(lib, "stego_eval_crf_unary_mosaic")


@pytest.mark.parametrize("mosaic,words", [
    (dict(tile0=5), "do not fit"),          # tiles [5, 7) of a 2 x 3 grid
    (dict(tile0=-1), "do not fit"),
    (dict(rows=0), "do not fit"),
    (dict(pitch=3 * 32 - 1), "pitch"),
    (dict(probes=0), "probes = 0"),
    (dict(probes=4), "probes = 4"),
])
def test_mosaic_entries_refuse_bad_arguments(mosaic, words):
    """Refused before any CUDA call (host addresses stand in for the buffers)."""
    from stego_b200 import _lib
    lib = _lib.load()
    buf = torch.zeros(4096, dtype=torch.float32)
    a = dict(tile0=0, rows=2, cols=3, pitch=3 * 32, probes=3)
    a.update(mosaic)
    P = buf.data_ptr()
    B, C, h, w, H, W = 2, 70, 4, 4, 32, 32
    for name in ("stego_eval_probes_mosaic", "stego_eval_crf_unary_mosaic"):
        if name == "stego_eval_probes_mosaic":
            if "probes" in mosaic:
                continue
            rc = lib.stego_eval_probes_mosaic(P, 0, C, C, B, h, w, H, W, P, P, 5, P, 5, 2.0, P, 0, 0, P, P, 0, 0, 0, 0, 0,
                                              a["tile0"], a["rows"], a["cols"], a["pitch"], 0)
        else:
            rc = lib.stego_eval_crf_unary_mosaic(P, 0, C, C, B, h, w, H, W, P, P, 5, P, 5, 2.0, P, P, P, a["probes"],
                                                 a["tile0"], a["rows"], a["cols"], a["pitch"], 0)
        assert rc != 0 and words in _lib.last_error() and name in _lib.last_error(), _lib.last_error()
