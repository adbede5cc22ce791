"""LitUnsupervisedSegmenter.eval_scene (plot_potsdam.py:44-83) on the GPU.

  * without the CRF, its predictions, log-probabilities and both confusion matrices are bit-equal to eval_step run per
    chunk and stitched with torch (chunk 1, 7 and 64, grids that are not square, fp32 and bf16 tiles, ViT-S/8 and
    ViT-B/8, the four-pixel and the generic probe kernels);
  * with the CRF on a 1 x 1 grid it is bit-equal to eval_step(run_crf=True) on the tile;
  * with the CRF on a mosaic its marginals are within 1e-4 of dense_crf on the stitched image and log-probabilities,
    with equal labels off near-ties, two calls are bit-identical, and pixels beside the seams differ from the per-tile
    CRF (the CRF crosses the seams);
  * with the CRF on a small mosaic its marginals are within the bars of the float64 mean field (tests/_crf_fp64.py);
  * the one-probe rows (cluster or linear) match that probe's half of the two-probe rows; map_clusters equals the
    host's map_clusters;
  * a full Potsdam scene (15 x 15 tiles of 320², ViT-B/8, cluster-only CRF at 4800²) completes without caching its
    position lattice, and a mean field whose value buffers do not fit is refused before it is enqueued.
"""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu


def _model(dev, n_classes=27, seed=0, **over):
    import stego_oracle as O
    from stego_b200.config import make_cfg
    from stego_b200.segmenter import LitUnsupervisedSegmenter
    arch = over.get("model_type", "vit_small")
    torch.manual_seed(seed)
    model = LitUnsupervisedSegmenter(n_classes, make_cfg(random_backbone_init=True, **over)).to(dev)
    model.net.model.load_state_dict(O.perturb_vit_state(O.vit_random_state(arch, 8, seed=3)))
    with torch.no_grad():
        model.cluster_probe.clusters.normal_(generator=torch.Generator(device=dev).manual_seed(4))
    return model


def _scene(dev, R, C, t, n_classes, label_dtype=torch.int64, dtype=torch.float32, seed=9, smooth=False):
    g = torch.Generator(device=dev).manual_seed(seed)
    tiles = torch.randn(R * C, 3, t, t, device=dev, generator=g)
    if smooth:  # a scene with large regions: colour ramps across the whole mosaic plus a little noise
        m = torch.linspace(-1.5, 1.5, C * t, device=dev).view(1, 1, -1).expand(3, R * t, C * t).clone()
        m[1] = torch.linspace(-1.5, 1.5, R * t, device=dev).view(-1, 1)
        tiles = m.view(3, R, t, C, t).permute(1, 3, 0, 2, 4).reshape(R * C, 3, t, t) + 0.1 * tiles
    label = torch.randint(0, n_classes, (R * C, t, t), device=dev, generator=g)
    r = torch.rand(R * C, t, t, device=dev, generator=g)
    label[r < 0.05] = 255 if label_dtype == torch.uint8 else -1
    return tiles.to(dtype), label.to(label_dtype)


def _stats(model):
    return model.test_linear_metrics.stats.clone(), model.test_cluster_metrics.stats.clone()


def _reset(model):
    model.test_linear_metrics.reset()
    model.test_cluster_metrics.reset()


# ================================================================================================
# without the CRF: eval_step per chunk, stitched
# ================================================================================================
CASES = {
    # name: model overrides, n_classes, R, C, t, chunk, tile dtype, label dtype
    "s8_3x5_64_chunk1": (dict(), 27, 3, 5, 64, 1, torch.float32, torch.int64),
    "s8_3x5_64_chunk7_bf16_u8": (dict(), 27, 3, 5, 64, 7, torch.bfloat16, torch.uint8),
    "s8_2x7_48_chunk64_3cls_extra2_i32": (dict(extra_clusters=2), 3, 2, 7, 48, 64, torch.float32, torch.int32),
    "s8_4x2_64_chunk7_kk": (dict(dino_feat_type="KK"), 27, 4, 2, 64, 7, torch.float32, torch.int64),
    "b8_2x3_320_chunk4": (dict(model_type="vit_base"), 27, 2, 3, 320, 4, torch.float32, torch.int64),
}


@pytest.mark.parametrize("case", list(CASES))
def test_no_crf_bit_equal_to_eval_step_per_chunk(cuda_dev, case):
    import scene_oracle as SO
    over, n, R, C, t, chunk, dt, ldt = CASES[case]
    model = _model(cuda_dev, n, **over)
    tiles, label = _scene(cuda_dev, R, C, t, n, ldt, dt)
    got = model.eval_scene(tiles, (R, C), label=label, want_probs=True, chunk=chunk)
    got_stats = _stats(model)
    _reset(model)
    parts = {k: [] for k in ("linear_preds", "cluster_preds", "linear_probs", "cluster_probs")}
    for t0 in range(0, R * C, chunk):
        out = model.eval_step(dict(img=tiles[t0:t0 + chunk], label=label[t0:t0 + chunk]), want_probs=True)
        for k in parts:
            parts[k].append(out[k])
    for k, v in parts.items():
        want = SO.stitch(torch.cat(v, 0), R, C)
        assert got[k].shape == want.shape and got[k].dtype == want.dtype, k
        assert torch.equal(got[k], want), (case, k)
    want_stats = _stats(model)
    assert torch.equal(got_stats[0], want_stats[0]) and torch.equal(got_stats[1], want_stats[1])
    assert int(got_stats[1].sum()) > 0


def test_no_crf_one_probe_and_no_label(cuda_dev):
    model = _model(cuda_dev)
    tiles, label = _scene(cuda_dev, 2, 3, 64, 27)
    both = model.eval_scene(tiles, (2, 3), want_probs=True)
    assert int(model.test_cluster_metrics.stats.sum()) == 0
    clu = model.eval_scene(tiles, (2, 3), label=label, probes=("cluster",), want_probs=True)
    assert sorted(clu) == ["cluster_preds", "cluster_probs"]
    assert torch.equal(clu["cluster_preds"], both["cluster_preds"]) and torch.equal(clu["cluster_probs"], both["cluster_probs"])
    assert int(model.test_linear_metrics.stats.sum()) == 0 and int(model.test_cluster_metrics.stats.sum()) > 0
    lin = model.eval_scene(tiles, (2, 3), probes=("linear",))
    assert sorted(lin) == ["linear_preds"] and torch.equal(lin["linear_preds"], both["linear_preds"])


# ================================================================================================
# with the CRF
# ================================================================================================
@pytest.mark.parametrize("n_classes,ldt", [(27, torch.int64), (3, torch.uint8)])
def test_crf_1x1_bit_equal_to_eval_step(cuda_dev, n_classes, ldt):
    model = _model(cuda_dev, n_classes)
    tiles, label = _scene(cuda_dev, 1, 1, 64, n_classes, ldt)
    got = model.eval_scene(tiles, (1, 1), label=label, run_crf=True, want_probs=True)
    got_stats = _stats(model)
    _reset(model)
    want = model.eval_step(dict(img=tiles, label=label), run_crf=True, want_probs=True)
    for k in ("linear_preds", "cluster_preds", "linear_probs", "cluster_probs"):
        assert torch.equal(got[k], want[k][0]), k
    want_stats = _stats(model)
    assert torch.equal(got_stats[0], want_stats[0]) and torch.equal(got_stats[1], want_stats[1])


def _crf_scene(dev, R=2, C=3, t=64, n=27):
    model = _model(dev, n)
    tiles, label = _scene(dev, R, C, t, n, smooth=True)
    return model, tiles, label


def test_crf_mosaic_against_dense_crf_on_the_stitched_scene(cuda_dev):
    import scene_oracle as SO
    from stego_b200 import crf
    R, C, t = 2, 3, 64
    model, tiles, label = _crf_scene(cuda_dev, R, C, t)
    logp = model.eval_scene(tiles, (R, C), want_probs=True)
    got = model.eval_scene(tiles, (R, C), label=label, run_crf=True, want_probs=True)
    image = SO.stitch(tiles, R, C)
    for probe in ("linear", "cluster"):
        want = crf.dense_crf(image, logp[f"{probe}_probs"])
        q = got[f"{probe}_probs"]
        assert q.shape == want.shape == (logp[f"{probe}_probs"].shape[0], R * t, C * t)
        assert float((q - want).abs().max()) < 1e-4, probe
        top2 = want.topk(2, 0).values
        clear = (top2[0] - top2[1]) > 2e-4
        assert torch.equal(got[f"{probe}_preds"][clear], want.argmax(0).to(torch.uint8)[clear]), probe
        assert float(clear.float().mean()) > 0.9
    # the confusion counts: the CRF predictions against the stitched label
    from stego_b200.eval import UnsupervisedMetrics
    lin, clu = _stats(model)
    for preds, stats, rows in ((got["linear_preds"], lin, 27), (got["cluster_preds"], clu, 27)):
        m = UnsupervisedMetrics("x/", 27, rows - 27, False, device=cuda_dev)
        m.update(preds, SO.stitch(label, R, C))
        assert torch.equal(m.stats, stats)


def test_crf_mosaic_repeats_and_crosses_the_seams(cuda_dev):
    import scene_oracle as SO
    R, C, t = 2, 3, 64
    model, tiles, label = _crf_scene(cuda_dev, R, C, t)
    a = model.eval_scene(tiles, (R, C), run_crf=True, want_probs=True)
    b = model.eval_scene(tiles, (R, C), run_crf=True, want_probs=True)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    per_tile = SO.stitch(model.eval_step(dict(img=tiles), run_crf=True, want_probs=True)["cluster_probs"], R, C)
    diff = (a["cluster_probs"] - per_tile).abs().amax(0)
    seams_x = torch.cat([diff[:, c * t - 1:c * t + 1] for c in range(1, C)], 1)
    seams_y = torch.cat([diff[r * t - 1:r * t + 1, :] for r in range(1, R)], 0)
    assert float(seams_x.max()) > 1e-3 and float(seams_y.max()) > 1e-3
    assert float(seams_x.mean()) > float(diff[8:t - 8, 8:t - 8].mean())


@pytest.mark.parametrize("probe", ["cluster", "linear"])
def test_one_probe_rows_match_the_two_probe_run(cuda_dev, probe):
    R, C, t = 2, 3, 64
    model, tiles, label = _crf_scene(cuda_dev, R, C, t)
    both = model.eval_scene(tiles, (R, C), label=label, run_crf=True, want_probs=True)
    stats2 = dict(zip(("linear", "cluster"), _stats(model)))
    _reset(model)
    one = model.eval_scene(tiles, (R, C), label=label, run_crf=True, want_probs=True, probes=(probe,))
    assert sorted(one) == [f"{probe}_preds", f"{probe}_probs"]
    q1, q2 = one[f"{probe}_probs"], both[f"{probe}_probs"]
    assert float((q1 - q2).abs().max()) < 1e-6
    top2 = q2.topk(2, 0).values
    clear = (top2[0] - top2[1]) > 2e-6
    assert torch.equal(one[f"{probe}_preds"][clear], both[f"{probe}_preds"][clear])
    stats1 = dict(zip(("linear", "cluster"), _stats(model)))
    other = "linear" if probe == "cluster" else "cluster"
    assert int(stats1[other].sum()) == 0 and int(stats1[probe].sum()) > 0
    assert int((stats1[probe] - stats2[probe]).abs().sum()) <= 2 * int((~clear).sum())


def test_crf_mosaic_against_the_fp64_mean_field(cuda_dev):
    """The mosaic's marginals against tests/_crf_fp64.py's float64 mean field on the same unary rows and lattices (a
    2 x 3 mosaic of 16² tiles): the bars of test_crf_fp64_gpu.py's ten-iteration chain, |dQ| < 2e-3 and equal labels
    wherever the fp64 top-2 gap exceeds twice the largest error."""
    import _crf_fp64 as F64
    import scene_oracle as SO
    from stego_b200 import _lib as L, crf
    from stego_b200.eval import _probe_codes, _probe_tables
    R, C, t = 2, 3, 16
    model = _model(cuda_dev, 5, extra_clusters=2)
    tiles, label = _scene(cuda_dev, R, C, t, 5, smooth=True)
    got = model.eval_scene(tiles, (R, C), run_crf=True, want_probs=True)
    # the unary rows eval_scene builds, from the same eval-mode code (one chunk)
    net, HH, WW, h = model.net, R * t, C * t, t // 8
    with model._net_in_eval_mode(), torch.no_grad():
        code = net.head_code(net.backbone_tokens(tiles, mirror=True), None, None, h, h)
    x, xf, ld = _probe_codes(code[:R * C], code[R * C:])
    wl, bl, cl = _probe_tables(model.linear_probe, model.cluster_probe, net.dim)
    n_lin, n_clu = wl.shape[0], cl.shape[0]
    scratch = torch.empty(R * C * h * h, 80, device=cuda_dev)
    unary = torch.empty(HH * WW, 64, device=cuda_dev)
    Q = torch.empty(HH * WW, 64, device=cuda_dev)
    L.check(L.load().stego_eval_crf_unary_mosaic(
        L.ptr(x), L.ptr(xf), ld, net.dim, R * C, h, h, t, t, L.ptr(wl), L.ptr(bl), n_lin, L.ptr(cl), n_clu, 2.0,
        L.ptr(scratch), L.ptr(unary), L.ptr(Q), 3, 0, R, C, WW, L.stream()), "stego_eval_crf_unary_mosaic")
    lat64 = lambda lat: F64.lattice(lat.offset, lat.bary, lat.n1, lat.n2, lat.M)
    g64 = lat64(crf._position_lattice(HH, WW, cuda_dev, cache=False))
    image = crf.prepare_image(SO.stitch(tiles, R, C))
    b64 = lat64(crf._lattice_points(HH, WW, 5, F64.BI_XY_STD, F64.BI_RGB_STD, image, cuda_dev))
    for lo, n, probe in ((0, n_lin, "linear"), (32, n_clu, "cluster")):
        want = F64.mean_field(unary[:, lo:lo + n], g64, b64)
        q = got[f"{probe}_probs"].reshape(n, HH * WW).t()
        err = (q.double() - want).abs().max().item()
        top = want.topk(2, 1).values
        clear = (top[:, 0] - top[:, 1]) > 2 * err
        print(f"\n{probe}: max |dQ| {err:.2e} against fp64, {int((~clear).sum())} near-tie pixels")
        assert err < 2e-3, (probe, err)
        assert torch.equal(got[f"{probe}_preds"].reshape(-1).long()[clear], want.argmax(1)[clear]), probe


@pytest.mark.parametrize("run_crf,extra", [(False, 0), (False, 2), (True, 2)])
def test_map_clusters_equals_the_host_mapping(cuda_dev, run_crf, extra):
    model = _model(cuda_dev, 3, extra_clusters=extra)
    tiles, label = _scene(cuda_dev, 2, 3, 64, 3)
    model.eval_scene(tiles, (2, 3), label=label)
    model.test_cluster_metrics.compute()
    raw = model.eval_scene(tiles, (2, 3), run_crf=run_crf)["cluster_preds"]
    got = model.eval_scene(tiles, (2, 3), run_crf=run_crf, map_clusters=True)["cluster_preds"]
    want = model.test_cluster_metrics.map_clusters(raw.long().cpu())
    assert got.dtype == torch.uint8
    assert torch.equal(torch.where(got == 255, -1, got.long()).cpu(), want.cpu())


def test_over_budget_mean_field_refused_before_it_is_enqueued(cuda_dev, monkeypatch):
    from stego_b200 import crf
    model, tiles, label = _crf_scene(cuda_dev)
    crf._POSITION_LATTICES.pop((128, 192, cuda_dev.index), None)  # dense_crf on a 128 x 192 frame caches it
    monkeypatch.setattr(crf, "_free_device_memory", lambda dev: 1 << 20)
    with pytest.raises(RuntimeError) as e:
        model.eval_scene(tiles, (2, 3), label=label, run_crf=True, probes=("cluster",))
    assert "eval_scene" in str(e.value) and "value buffers need" in str(e.value) and "bilateral lattice" in str(e.value)
    torch.cuda.synchronize()
    assert int(model.test_cluster_metrics.stats.sum()) == 0  # the mean field's counts never ran
    assert (128, 192, cuda_dev.index) not in crf._POSITION_LATTICES


# ================================================================================================
# a full Potsdam scene, once
# ================================================================================================
def test_full_potsdam_scene_4800(cuda_dev, monkeypatch):
    """15 x 15 tiles of 320² (plot_potsdam.py's scene), ViT-B/8, 3 classes, cluster-only CRF over the 4800² mosaic."""
    from stego_b200 import crf
    R = C = 15
    t = 320
    model = _model(cuda_dev, 3, model_type="vit_base")
    tiles, label = _scene(cuda_dev, R, C, t, 3, torch.uint8, smooth=True)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(cuda_dev)
    base = torch.cuda.memory_allocated(cuda_dev)
    out = model.eval_scene(tiles, (R, C), label=label, run_crf=True, probes=("cluster",))
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated(cuda_dev)
    print(f"\neval_scene 15x15 x 320^2 cluster-only CRF: peak {peak / 2**30:.2f} GiB allocated "
          f"({(peak - base) / 2**30:.2f} GiB above the inputs)")
    assert out["cluster_preds"].shape == (R * t, C * t)
    assert int(out["cluster_preds"].max()) < 3
    assert int(model.test_cluster_metrics.stats.sum()) > 0
    assert not any(k[:2] == (R * t, C * t) for k in crf._POSITION_LATTICES)
    # the over-budget path at this size: refused after the lattices are built, before the mean field
    stats = model.test_cluster_metrics.stats.clone()
    monkeypatch.setattr(crf, "_free_device_memory", lambda dev: 1 << 30)
    with pytest.raises(RuntimeError, match="value buffers need"):
        model.eval_scene(tiles, (R, C), label=label, run_crf=True, probes=("cluster",))
    torch.cuda.synchronize()
    assert torch.equal(model.test_cluster_metrics.stats, stats)
