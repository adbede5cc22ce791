"""Multi-device inference on the GPU: the library from several devices and host threads, nn.DataParallel over the
DinoFeaturizer, and the `devices=` paths of eval_step, eval_scene, knn_topk and precompute_knns.

On any GPU count:
  * the library from two host threads at once on one device: the backbone (GEMM with TMA and register epilogues,
    attention), the kNN search and the probes give the same bits in every thread, 20 rounds;
  * stego_knn_topk_rows over splits into 128-row-block ranges, concatenated, is torch.equal to stego_knn_topk
    (n = 1, 127, 128, 129, 2975, 2 * 128 * SMs + 77 and 118 287; E = 384 and 768; a single block, the ragged last block);
  * the sharded paths behind `devices=` (frame slices of eval_step, tile-row bands of eval_scene, row ranges of
    knn_topk) with every slice on one device are bit-equal to the single-device calls: the staging, gathering and
    count-summing logic without a second device;
  * a DataParallel replica (torch.nn.parallel.replicate + parallel_apply, one device) equals the module, reads the
    module's prepared weights, and sees an in-place change of a backbone weight;
  * a CUDA graph is captured on its own device's capture stream and replays there.

With two or more visible GPUs (at 2 devices and at every visible device, up to 8): the same calls with `devices=` and
nn.DataParallel(model.net) bit-equal to one device; a graph captured for device 1 records and replays on device 1; every
opt-in kernel (the backbone GEMMs and attention, attention probabilities, correlation forward / backward at
feature_samples 11 and 28, head, probes, eval probe and CRF unary kernels, kNN, rec, salience coordinates) on device 1
equal to device 0 before and after it; and devices 0 and 1 driven from two host threads at once, 20 rounds.
"""
import os
import sys
import threading

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu

N_GPUS = torch.cuda.device_count() if torch.cuda.is_available() else 0
multi = pytest.mark.skipif(N_GPUS < 2, reason="needs at least 2 visible GPUs")
DEVICE_SETS = [2, min(N_GPUS, 8)] if N_GPUS > 2 else [2]


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


def _frames(dev, B, res, n_classes=27, label_dtype=torch.int64, dtype=torch.float32, seed=5):
    g = torch.Generator(device=dev).manual_seed(seed)
    img = torch.randn(B, 3, res, res, device=dev, generator=g)
    label = torch.randint(0, n_classes, (B, res, res), device=dev, generator=g)
    label[torch.rand(B, res, res, device=dev, generator=g) < 0.05] = 255 if label_dtype == torch.uint8 else -1
    return img.to(dtype), label.to(label_dtype)


def _stats(model):
    return model.test_linear_metrics.stats.clone(), model.test_cluster_metrics.stats.clone()


def _reset(model):
    model.test_linear_metrics.reset()
    model.test_cluster_metrics.reset()


def _equal_dicts(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert a[k].device == b[k].device and torch.equal(a[k], b[k]), k


# ================================================================================================
# the library from several host threads
# ================================================================================================
def _library_round(model, img, feats):
    from stego_b200.knn import knn_topk
    from stego_b200.eval import fused_probe_log_probs
    tok = model.net.backbone_tokens(img)  # eager: GEMM (TMA and register epilogues), attention, LayerNorm
    idx, vals = knn_topk(feats, 8, return_values=True)
    code = model.net.eval_code(tok, img.shape[2] // 8, img.shape[3] // 8)
    lp = fused_probe_log_probs(code, model.linear_probe, model.cluster_probe, img.shape[-2:], 2.0)
    return [tok, idx, vals, *lp]


def test_library_from_two_host_threads():
    dev = torch.device("cuda", 0)
    model = _model(dev)
    model.eval()
    img, _ = _frames(dev, 2, 64)
    feats = torch.randn(700, 384, device=dev, generator=torch.Generator(device=dev).manual_seed(1))
    with torch.no_grad():
        want = _library_round(model, img, feats)
        torch.cuda.synchronize()
        for _ in range(20):
            got, errors = [None, None], []

            def run(i):
                try:
                    with torch.cuda.device(dev), torch.cuda.stream(torch.cuda.Stream(dev)):
                        got[i] = _library_round(model, img, feats)
                        torch.cuda.current_stream().synchronize()
                except Exception as e:  # surfaced below
                    errors.append(e)
            threads = [threading.Thread(target=run, args=(i,)) for i in range(2)]
            for t in threads:
                t.start()
            for t in threads:
                t.join()
            assert not errors, errors
            for res in got:
                assert all(torch.equal(a, b) for a, b in zip(res, want))


# ================================================================================================
# kNN row ranges
# ================================================================================================
def _knn_planes(feats):
    from stego_b200 import _lib
    n, E = feats.shape
    planes = torch.empty(2, n, E, dtype=torch.bfloat16, device=feats.device)
    _lib.check(_lib.load().stego_knn_prep(_lib.ptr(feats), n, E, _lib.ptr(planes), _lib.stream()), "stego_knn_prep")
    return planes


def _knn_rows(planes, k, r0, r1):
    from stego_b200 import _lib
    _, n, E = planes.shape
    idx = torch.empty(r1 - r0, k, dtype=torch.long, device=planes.device)
    vals = torch.empty(r1 - r0, k, dtype=torch.float32, device=planes.device)
    _lib.check(_lib.load().stego_knn_topk_rows(_lib.ptr(planes), n, E, k, r0, r1 - r0, _lib.ptr(idx), _lib.ptr(vals),
                                               _lib.stream()), "stego_knn_topk_rows")
    return idx, vals


def _knn_splits(n):
    """Splits of [0, n) into ranges starting on multiples of 128: the whole set, a single block first, the ragged last
    block alone, and a mixed split."""
    blocks = (n + 127) // 128
    cuts = [[0, n]]
    if blocks > 1:
        cuts.append([0, 128, n])
        cuts.append([0, (blocks - 1) * 128, n])
        cuts.append(sorted({0, 128 * (blocks // 3), 128 * (2 * blocks // 3), n}))
    return cuts


@pytest.mark.parametrize("E", [384, 768])
@pytest.mark.parametrize("n", [1, 127, 128, 129, 2975, "2*128*SMs+77", 118287])
def test_knn_topk_rows_concatenated_equal_knn_topk(n, E):
    from stego_b200.knn import knn_topk
    dev = torch.device("cuda", 0)
    if n == "2*128*SMs+77":
        n = 2 * 128 * torch.cuda.get_device_properties(dev).multi_processor_count + 77
    k = min(30, n)
    g = torch.Generator(device=dev).manual_seed(n + E)
    feats = torch.randn(n, E, device=dev, generator=g)
    if n > 10:
        feats[5] = feats[3]  # an exact duplicate: the self-first rule on absolute rows
    want_i, want_v = knn_topk(feats, k, return_values=True)
    planes = _knn_planes(feats)
    for cuts in _knn_splits(n):
        parts = [_knn_rows(planes, k, a, b) for a, b in zip(cuts[:-1], cuts[1:]) if b > a]
        assert torch.equal(torch.cat([p[0] for p in parts]), want_i), cuts
        assert torch.equal(torch.cat([p[1] for p in parts]), want_v), cuts
    del planes
    torch.cuda.empty_cache()


def test_knn_sharded_on_one_device_equals_knn_topk():
    from stego_b200.knn import _knn_topk_sharded, knn_topk
    dev = torch.device("cuda", 0)
    feats = torch.randn(2975, 384, device=dev, generator=torch.Generator(device=dev).manual_seed(2))
    want = knn_topk(feats, 30, return_values=True)
    for shards in ([(dev, 0, 1024), (dev, 1024, 2975)], [(dev, 0, 0), (dev, 0, 128), (dev, 128, 2975)]):
        got = _knn_topk_sharded(feats, 30, True, shards)
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])


# ================================================================================================
# the sharded eval_step / eval_scene on one device
# ================================================================================================
EVAL_CASES = {
    # name: model overrides, B, res, run_crf, want_probs, label dtype (None: no label), frame dtype
    "probs_i64": (dict(), 5, 64, False, True, torch.int64, torch.float32),
    "u8_bf16": (dict(), 5, 64, False, False, torch.uint8, torch.bfloat16),
    "nolabel": (dict(), 3, 64, False, True, None, torch.float32),
    "crf_i32": (dict(), 3, 32, True, True, torch.int32, torch.float32),
    "crf_nolabel": (dict(), 3, 32, True, False, None, torch.float32),
    "kk_linear_head": (dict(dino_feat_type="KK", projection_type="linear"), 4, 64, False, True, torch.int64,
                       torch.float32),
    "baseline_vitb": (dict(model_type="vit_base", projection_type=None, dim=768), 3, 64, False, True, torch.int64,
                      torch.float32),
}


@pytest.mark.parametrize("case", list(EVAL_CASES))
def test_eval_step_slices_on_one_device_equal_eval_step(case):
    over, B, res, run_crf, want_probs, label_dtype, dtype = EVAL_CASES[case]
    dev = torch.device("cuda", 0)
    model = _model(dev, **over)
    img, label = _frames(dev, B, res, label_dtype=label_dtype or torch.int64, dtype=dtype)
    batch = dict(img=img) if label_dtype is None else dict(img=img, label=label)
    want = model.eval_step(batch, run_crf=run_crf, want_probs=want_probs)
    want_stats = _stats(model)
    _reset(model)
    shards = [(dev, 0, 0), (dev, 0, 2), (dev, 2, B)]  # an idle device, then two slices of different sizes
    got = model._eval_step_sharded(img, batch.get("label"), run_crf, want_probs, shards)
    _equal_dicts(got, want)
    for a, b in zip(_stats(model), want_stats):
        assert torch.equal(a, b)


SCENE_CASES = {
    # name: R, C, t, chunk, run_crf, probes, map_clusters, bands (tile-row ranges)
    "3x4_chunk1": (3, 4, 64, 1, False, ("linear", "cluster"), False, [(0, 1), (1, 3)]),
    "3x4_chunk7_cluster": (3, 4, 64, 7, False, ("cluster",), False, [(0, 2), (2, 3)]),
    "4x3_chunk64_linear_idle": (4, 3, 64, 64, False, ("linear",), False, [(0, 0), (0, 1), (1, 4)]),
    "3x4_crf": (3, 4, 64, 5, True, ("linear", "cluster"), False, [(0, 1), (1, 3)]),
    "3x4_crf_cluster_map": (3, 4, 64, 64, True, ("cluster",), True, [(0, 2), (2, 3)]),
}


@pytest.mark.parametrize("case", list(SCENE_CASES))
def test_eval_scene_bands_on_one_device_equal_eval_scene(case):
    R, C, t, chunk, run_crf, probes, map_clusters, bands = SCENE_CASES[case]
    dev = torch.device("cuda", 0)
    model = _model(dev)
    tiles, label = _frames(dev, R * C, t, seed=11)
    if map_clusters:
        model.eval_step(dict(img=tiles[:2], label=label[:2]))
        model.test_cluster_metrics.compute()
        _reset(model)
    kw = dict(run_crf=run_crf, probes=probes, want_probs=True, map_clusters=map_clusters, chunk=chunk)
    want = model.eval_scene(tiles, (R, C), label, **kw)
    want_stats = _stats(model)
    _reset(model)
    got = model._eval_scene_bands(tiles, label, run_crf, probes, True, map_clusters, chunk, R, C, R * C, t, t,
                                  [(dev, r0, r1) for r0, r1 in bands])
    _equal_dicts(got, want)
    for a, b in zip(_stats(model), want_stats):
        assert torch.equal(a, b)


def test_eval_step_devices_of_one_is_the_single_device_call():
    dev = torch.device("cuda", 0)
    model = _model(dev)
    img, label = _frames(dev, 3, 64)
    want = model.eval_step(dict(img=img, label=label), want_probs=True)
    want_stats = _stats(model)
    _reset(model)
    got = model.eval_step(dict(img=img, label=label), want_probs=True, devices=[0])
    _equal_dicts(got, want)
    assert all(torch.equal(a, b) for a, b in zip(_stats(model), want_stats))


# ================================================================================================
# DataParallel replicas (one device)
# ================================================================================================
def test_replica_reads_the_module_cache_and_sees_weight_changes():
    from torch.nn.parallel import parallel_apply, replicate
    dev = torch.device("cuda", 0)
    model = _model(dev)
    net = model.net
    net.eval()
    img, _ = _frames(dev, 2, 64)
    with torch.no_grad():
        want = net(img)
        cache = net.model._cache
        replica = replicate(net, [0], detach=True)[0]
        got = parallel_apply([replica], [(img,)], devices=[0])[0]
        assert all(torch.equal(a, b) for a, b in zip(got, want))
        assert net.model._cache is cache and list(cache["w"]) == [dev]  # the module's one entry, reused
        net.model.blocks[3].mlp.fc1.weight.mul_(1.01)
        want2 = net(img)
        assert not torch.equal(want2[1], want[1])
        replica = replicate(net, [0], detach=True)[0]
        got2 = parallel_apply([replica], [(img,)], devices=[0])[0]
        assert all(torch.equal(a, b) for a, b in zip(got2, want2))


# ================================================================================================
# two or more devices
# ================================================================================================
@multi
@pytest.mark.parametrize("nd", DEVICE_SETS)
@pytest.mark.parametrize("arch,res,over", [("vit_small", 224, dict()), ("vit_base", 320, dict()),
                                           ("vit_small", 224, dict(dino_feat_type="KK")),
                                           ("vit_small", 224, dict(projection_type="linear")),
                                           ("vit_small", 224, dict(projection_type=None, dim=384))])
def test_data_parallel_forward_equals_the_module(nd, arch, res, over):
    dev = torch.device("cuda", 0)
    model = _model(dev, model_type=arch, **over)
    net = model.net
    net.eval()
    par = torch.nn.DataParallel(net, device_ids=list(range(nd)))
    with torch.no_grad():
        for B in (1, nd - 1, 3 * nd + 1):
            if B < 1:
                continue
            img, _ = _frames(dev, B, res, seed=B)
            want = net(img)
            got = par(img)
            assert all(torch.equal(a, b) for a, b in zip(got, want)), B
        net.model.blocks[0].attn.qkv.weight.add_(0.01)
        img, _ = _frames(dev, nd + 1, res)
        assert all(torch.equal(a, b) for a, b in zip(par(img), net(img)))


@multi
@pytest.mark.parametrize("nd", DEVICE_SETS)
def test_reference_eval_loop_with_data_parallel(nd):
    """eval_segmentation.py:119-138 with par_model = DataParallel(model.net): the same predictions as model.net."""
    import torch.nn.functional as F
    dev = torch.device("cuda", 0)
    model = _model(dev)
    model.eval()
    img, label = _frames(dev, 2 * nd + 1, 64)
    par_model = torch.nn.DataParallel(model.net, device_ids=list(range(nd)))

    def body(m):
        with torch.no_grad():
            feats, code1 = m(img)
            feats, code2 = m(img.flip(dims=[3]))
            code = (code1 + code2.flip(dims=[3])) / 2
            code = F.interpolate(code, label.shape[-2:], mode='bilinear', align_corners=False)
            linear_probs = torch.log_softmax(model.linear_probe(code), dim=1)
            cluster_probs = model.cluster_probe(code, 2, log_probs=True)
            return linear_probs.argmax(1), cluster_probs.argmax(1)

    want, got = body(model.net), body(par_model)
    assert all(torch.equal(a, b) for a, b in zip(got, want))


@multi
@pytest.mark.parametrize("nd", DEVICE_SETS)
@pytest.mark.parametrize("case", list(EVAL_CASES))
def test_eval_step_devices_equal_one_device(nd, case):
    over, B, res, run_crf, want_probs, label_dtype, dtype = EVAL_CASES[case]
    dev = torch.device("cuda", 0)
    model = _model(dev, **over)
    for B in (B, nd - 1, 3 * nd + 1):
        if B < 1:
            continue
        img, label = _frames(dev, B, res, label_dtype=label_dtype or torch.int64, dtype=dtype, seed=B)
        batch = dict(img=img) if label_dtype is None else dict(img=img, label=label)
        _reset(model)
        want = model.eval_step(batch, run_crf=run_crf, want_probs=want_probs)
        want_stats = _stats(model)
        _reset(model)
        got = model.eval_step(batch, run_crf=run_crf, want_probs=want_probs, devices=list(range(nd)))
        _equal_dicts(got, want)
        assert all(torch.equal(a, b) for a, b in zip(_stats(model), want_stats))


@multi
def test_eval_step_devices_sees_a_training_step_and_leaves_training_state():
    dev = torch.device("cuda", 0)
    model = _model(dev)
    model.train()
    model.configure_optimizers()
    g = torch.Generator(device=dev).manual_seed(3)
    tb = dict(img=torch.randn(2, 3, 64, 64, device=dev, generator=g),
              img_pos=torch.randn(2, 3, 64, 64, device=dev, generator=g),
              label=torch.randint(0, 27, (2, 64, 64), device=dev, generator=g))
    img, label = _frames(dev, 5, 64)
    model.training_step(tb, 0)
    model.eval_step(dict(img=img, label=label), devices=[0, 1])
    model.training_step(tb, 1)
    model.flush()
    params = [p.detach().clone() for p in model.parameters()]
    flat = [t.clone() for t in (model._flat.param, model._flat.exp_avg, model._flat.exp_avg_sq)]
    rng = (torch.get_rng_state(), torch.cuda.get_rng_state(dev))
    _reset(model)
    got = model.eval_step(dict(img=img, label=label), devices=[0, 1])
    got_stats = _stats(model)
    _reset(model)
    want = model.eval_step(dict(img=img, label=label))
    _equal_dicts(got, want)
    assert all(torch.equal(a, b) for a, b in zip(got_stats, _stats(model)))
    assert all(torch.equal(a, b.detach()) for a, b in zip(params, model.parameters()))
    assert all(torch.equal(a, b) for a, b in zip(flat, (model._flat.param, model._flat.exp_avg,
                                                        model._flat.exp_avg_sq)))
    assert torch.equal(rng[0], torch.get_rng_state()) and torch.equal(rng[1], torch.cuda.get_rng_state(dev))


@multi
@pytest.mark.parametrize("nd", DEVICE_SETS)
@pytest.mark.parametrize("case", list(SCENE_CASES))
def test_eval_scene_devices_equal_one_device(nd, case):
    R, C, t, chunk, run_crf, probes, map_clusters, _ = SCENE_CASES[case]
    dev = torch.device("cuda", 0)
    model = _model(dev)
    tiles, label = _frames(dev, R * C, t, seed=11)
    if map_clusters:
        model.eval_step(dict(img=tiles[:2], label=label[:2]))
        model.test_cluster_metrics.compute()
        _reset(model)
    kw = dict(run_crf=run_crf, probes=probes, want_probs=True, map_clusters=map_clusters, chunk=chunk)
    want = model.eval_scene(tiles, (R, C), label, **kw)
    want_stats = _stats(model)
    _reset(model)
    got = model.eval_scene(tiles, (R, C), label, devices=list(range(nd)), **kw)
    _equal_dicts(got, want)
    assert all(torch.equal(a, b) for a, b in zip(_stats(model), want_stats))


@multi
def test_eval_scene_devices_full_potsdam_scene_without_crf():
    dev = torch.device("cuda", 0)
    model = _model(dev, model_type="vit_base")
    tiles, label = _frames(dev, 225, 320, seed=12)
    want = model.eval_scene(tiles, (15, 15), label, probes=("cluster",))
    want_stats = _stats(model)
    _reset(model)
    got = model.eval_scene(tiles, (15, 15), label, probes=("cluster",), devices=list(range(min(N_GPUS, 8))))
    _equal_dicts(got, want)
    assert all(torch.equal(a, b) for a, b in zip(_stats(model), want_stats))


@multi
@pytest.mark.parametrize("nd", DEVICE_SETS)
@pytest.mark.parametrize("n,E", [(1, 384), (129, 384), (2975, 768), (118287, 384)])
def test_knn_devices_equal_one_device(nd, n, E):
    from stego_b200.knn import knn_topk
    dev = torch.device("cuda", 0)
    feats = torch.randn(n, E, device=dev, generator=torch.Generator(device=dev).manual_seed(n))
    k = min(30, n)
    want = knn_topk(feats, k, return_values=True)
    got = knn_topk(feats, k, return_values=True, devices=list(range(nd)))
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])


@multi
@pytest.mark.parametrize("nd", DEVICE_SETS)
@pytest.mark.parametrize("feat_type", ["feat", "KK"])
def test_precompute_knns_devices_equal_one_device(nd, feat_type):
    from stego_b200.knn import precompute_knns
    dev = torch.device("cuda", 0)
    model = _model(dev, dino_feat_type=feat_type)
    model.net.eval()
    g = torch.Generator().manual_seed(7)
    batches = [dict(img=torch.randn(b, 3, 64, 64, generator=g)) for b in (4, 3, 4, 1, 4)]
    want = precompute_knns(model.net, batches, 5)
    got = precompute_knns(model.net, batches, 5, devices=list(range(nd)))
    assert torch.equal(got, want)


@multi
def test_library_on_a_second_device_and_back():
    """device 0, then device 1, then device 0 again: every opt-in kernel gives device 0's bits on device 1."""
    import copy
    from stego_b200.knn import knn_topk
    d0, d1 = torch.device("cuda", 0), torch.device("cuda", 1)
    model = _model(d0)
    models = {d0: model, d1: copy.deepcopy(model).to(d1)}
    img, label = _frames(d0, 3, 64)
    feats = torch.randn(700, 384, device=d0, generator=torch.Generator(device=d0).manual_seed(1))

    def run(dev):
        with torch.cuda.device(dev):
            m = models[dev]
            x, lab, f = img.to(dev), label.to(dev), feats.to(dev)
            out = m.eval_step(dict(img=x, label=lab), want_probs=True)
            crf = m.eval_step(dict(img=x[:, :, :32, :32], label=lab[:, :32, :32].contiguous()), run_crf=True)
            idx = knn_topk(f, 8, return_values=True)
            res = [t.to(d0) for t in list(out.values()) + list(crf.values()) + list(idx)]
            return res + [t.to(d0) for t in _stats(m)]

    a = run(d0)
    b = run(d1)
    c = run(d0)
    assert all(torch.equal(x, y) for x, y in zip(a[:-2], b[:-2]))
    assert all(torch.equal(x, y) for x, y in zip(a[:-2], c[:-2]))


def test_graph_captures_on_its_own_device_stream():
    """A graph is captured on the capture stream of the device current at its creation (not torch.cuda.graph's one
    process-wide default stream, which belongs to whichever device captured first) and replays there."""
    from stego_b200 import _lib
    dev = torch.device("cuda", 0)
    x = torch.ones(8, device=dev)
    g = _lib.Graph(lambda: x * 2)
    assert g.device == dev and _lib.capture_stream(dev).device == dev
    x.fill_(3)
    g.replay()
    assert torch.equal(g.result, torch.full((8,), 6.0, device=dev))


@multi
def test_graph_captured_for_a_second_device_runs_there():
    from stego_b200 import _lib
    d0, d1 = torch.device("cuda", 0), torch.device("cuda", 1)
    with torch.cuda.device(d0):
        a = torch.ones(8, device=d0)
        g0 = _lib.Graph(lambda: a * 2)
    with torch.cuda.device(d1):
        b = torch.ones(8, device=d1)
        g1 = _lib.Graph(lambda: b * 5)
    assert g1.device == d1 and g1.result.device == d1 and _lib.capture_stream(d1).device == d1
    b.fill_(2)
    a.fill_(4)
    g1.replay()  # replayed from device 0's context: the graph still runs on device 1's current stream
    g0.replay()
    with torch.cuda.device(d1):
        assert torch.equal(g1.result, torch.full((8,), 10.0, device=d1))
    assert torch.equal(g0.result, torch.full((8,), 8.0, device=d0))


@multi
def test_library_on_two_devices_from_two_host_threads():
    """Device 0 and device 1 from two host threads at once, 20 rounds: each thread's results are the bits of one thread
    alone on device 0 (the per-device opt-in of every kernel raced from both threads)."""
    import copy
    d0, d1 = torch.device("cuda", 0), torch.device("cuda", 1)
    model = _model(d0)
    model.eval()
    models = {d0: model, d1: copy.deepcopy(model).to(d1)}
    img, _ = _frames(d0, 2, 64)
    feats = torch.randn(700, 384, device=d0, generator=torch.Generator(device=d0).manual_seed(1))
    inputs = {d: (img.to(d), feats.to(d)) for d in (d0, d1)}
    with torch.no_grad():
        want = _library_round(model, img, feats)
        torch.cuda.synchronize(d0)
        for _ in range(20):
            got, errors = {}, []

            def run(d):
                try:
                    with torch.cuda.device(d), torch.cuda.stream(torch.cuda.Stream(d)):
                        res = _library_round(models[d], *inputs[d])
                        torch.cuda.current_stream().synchronize()
                        got[d] = [t.to(d0) for t in res]
                except Exception as e:  # surfaced below
                    errors.append(e)
            threads = [threading.Thread(target=run, args=(d,)) for d in (d0, d1)]
            for t in threads:
                t.start()
            for t in threads:
                t.join()
            assert not errors, errors
            for d in (d0, d1):
                assert all(torch.equal(a, b) for a, b in zip(got[d], want)), d


@multi
@pytest.mark.parametrize("fs", [11, 28])
def test_training_kernels_on_a_second_device_and_back(fs):
    """device 0, then device 1, then device 0 again, each a fresh model from the same seed: the hand-scheduled training
    step with the reconstruction term and salience draws (correlation forward / backward at feature_samples fs, head,
    probes, rec, salience coordinates, Adam) and the attention probabilities give device 0's bits on device 1."""
    from _parity_util import make_batch, make_model
    d0, d1 = torch.device("cuda", 0), torch.device("cuda", 1)

    def run(dev):
        with torch.cuda.device(dev):
            model, _ = make_model("vit_small", dev, fused=True, fused_rec_crf=True, rec_weight=0.7, use_salience=True,
                                  feature_samples=fs, res=64)
            batch = make_batch(4, 64, dev)
            g = torch.Generator().manual_seed(5)
            batch["mask"] = (torch.rand(4, 1, 64, 64, generator=g) > 0.6).float().to(dev)
            batch["mask_pos"] = (torch.rand(4, 1, 64, 64, generator=g) > 0.3).float().to(dev)
            torch.manual_seed(777)
            losses = [model.training_step(batch, i).detach() for i in range(2)]
            model.flush()
            with torch.no_grad():
                attn = model.net.model.get_last_selfattention(batch["img"])
            out = losses + [attn] + [p.detach() for p in model.parameters() if p.requires_grad]
            torch.cuda.synchronize(dev)
            return [t.to(d0) for t in out]

    a, b, c = run(d0), run(d1), run(d0)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    assert all(torch.equal(x, y) for x, y in zip(a, c))
