"""GPU: the aug-alignment term (train_segmentation.py:189-199) on the hand-scheduled step.

Kernels (stego_aug_align_fwd / _bwd / _loss through modules.aug_sample_forward / aug_sample_backward / aug_loss, with
the cosine of modules.cosine_forward / cosine_backward) at the c1 / c2 / c3 code shapes (h = 28 / 40 / 56, S = 8h,
D = 70), on views from real seeds (flipped and unflipped, crops touching the frame edge) and on hand-made coordinates
(grid at +-1 and beyond, so the border clamp acts; grid points on integer taps, whose presence is asserted), for NCHW
and channels-last code:

  * grid and sampled are bit-equal to torch CUDA's F.interpolate / F.grid_sample on the same inputs (ATen's arithmetic;
    the four taps accumulated in ATen's order: the nw product rounded, then ne, sw, se fused onto the sum), and within
    the bars below of an fp64 restatement;
  * d(code) from the scatter and d(code_aug) are within the bars below of fp64 autograd.

Bars (u = 2^-24).  grid: ATen's lambdas are exact here (scale = 8), so each value is four products and three sums of
numbers of magnitude <= m = max|coord_aug|: 6 u m.  sampled, restated in fp64 at the kernel's own grid: the source
position ((g + 1) / 2) (h - 1) is formed with three roundings, |dx| <= 3 u h; the weights (x1 - x)(y1 - y) then move by
<= 2 (3 u h) + 3 u, and the sum of four products adds 4 u; with c = max|code| the bar is c (4 (6 u h + 3 u) + 4 u).
d(code): each element is a sum of k contributions w g (k counted from the grid: _step_fp64.tap_counts) made in any order by the
atomics; with A the fp64 sum of |w g| (grid_sample's backward of |g|) the sum costs (k + 1) u A.  The weights are
formed in fp32 from the fp32 position: each factor is off by <= 3 u h + 2 u, the product by <= (6 h + 8) u absolute
(a weight near 0 has no relative bound), which adds k (6 h + 8) u max|g|.  d(code_aug) is the cosine
backward, whose bars test_loss_terms_fp64_gpu.py derives; here it is checked through the same relative bar as d(code).

Step (c1: ViT-S/8 224², and ViT-B/8 320²): from one model state, generator state and seeded batch, one fused step and
one autograd step leave both generators in the same state and log bit-equal positive correspondence terms and cluster
loss (neg_inter is the mean of the negative calls' losses, formed in another order on each path).  The fused step's
cosines are bit-equal to the autograd step's: torch's own mean of them reproduces the autograd step's
loss/aug_alignment bit for bit.  The logged loss/aug_alignment is the fixed-order fp64 mean of those cosines, rounded
once; the autograd step's fp32 torch mean is within n u mean|cos| of it.  loss/linear is summed with fp64 atomics (as in
test_step_stages.py) and loss/total adds the terms in another order, so both get derived bars.  Parameter gradients
agree within test_salience_gpu.py's relative bar (the scatter, the grid_sample backward and the split-K weight
gradients all use fp32 atomics).  Because the aug term's share of the head gradients could hide under that bar, its
contribution is isolated (the step with the term minus the same step without it, whose draws up to the term are the
same) and compared between the two paths at 1e-3: d(code_aug) sent to the wrong rows, or d(sampled) scattered into
the wrong image, moves that difference by its whole size.
"""
import pytest
import torch
import torch.nn.functional as F

from _parity_util import NAMES, grads_of, make_batch, make_model, rel
from _step_fp64 import aug_grid_bar, aug_sampled_bar, aug_scatter_bar

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
D = 70


def _views(B, S, seed0, dev):
    """Views of B seeds picked (on the host draws alone) to hold an unflipped view, a flipped view and a crop touching
    the frame edge."""
    from stego_b200.augment import aug_alignment_views, draw_params, draw_records
    edge = lambda p: p["crop"][0] == 0 or p["crop"][1] == 0 or p["crop"][0] + p["crop"][2] == S or \
        p["crop"][1] + p["crop"][3] == S
    wanted = [lambda p: not p["flip"], lambda p: p["flip"], edge]
    seeds, s = [], seed0
    with torch.random.fork_rng(devices=[]):
        while wanted:
            p = draw_params(s, S, S)
            hit = [f for f in wanted if f(p)]
            if hit:
                seeds.append(s)
                wanted = [f for f in wanted if f not in hit]
            s += 1
    seeds += list(range(s, s + B - len(seeds)))
    g = torch.Generator().manual_seed(seed0)
    img = torch.randn(B, 3, S, S, generator=g).to(dev)
    params, _ = draw_records(seeds, S, S)
    _, coord = aug_alignment_views(img, seeds, S)
    return coord, params


def _handmade(B, S, h, dev):
    """Coordinates whose resized grid reaches +-1 and beyond (border clamp) and lands on integer taps.  The last kind is
    constant on each 8 x 8 block with the values 2k / (h - 1) - 1: the resize reads two pixels of one block with
    lambda = 0.5, so the grid gets the block's value exactly, and its source position is the integer k wherever
    ((g + 1) / 2) (h - 1) rounds back to k in fp32 (test_kernels_vs_torch_and_fp64 asserts that such points exist)."""
    lin = torch.linspace(-1.0, 1.0, S)
    yy, xx = torch.meshgrid(lin, lin, indexing="ij")
    base = torch.stack([xx, yy], -1)
    k = torch.arange(S) // (S // h)
    taps = torch.stack(torch.meshgrid(k * 2.0 / (h - 1) - 1, k * 2.0 / (h - 1) - 1, indexing="ij")[::-1], -1)
    out = [base, -base, base * 1.3, taps]
    return torch.stack([out[b % 4] for b in range(B)]).to(dev).contiguous()


def _code(B, h, layout, dev, seed):
    g = torch.Generator().manual_seed(seed)
    c = torch.randn(B, D, h, h, generator=g).to(dev)
    if layout == "nchw":
        return c
    store = torch.zeros(B, h, h, 72, device=dev)  # tokens-major, pitch 72: the step's code storage
    store[..., :D] = c.permute(0, 2, 3, 1)
    return store[..., :D].permute(0, 3, 1, 2)


def _stage_fwd(coord, code):
    from stego_b200 import modules
    B, _, h, _ = code.shape
    grid = torch.empty(B, h, h, 2, device=code.device)
    sampled = torch.empty(B, D, h, h, device=code.device)
    modules.aug_sample_forward(coord, code, grid, sampled)
    return grid, sampled


def _torch_ref(coord, code):
    grid = F.interpolate(coord.permute(0, 3, 1, 2), code.shape[2], mode="bilinear", align_corners=False).permute(0, 2, 3, 1)
    return grid, F.grid_sample(code, grid.permute(0, 2, 1, 3), padding_mode="border", align_corners=True)


def _bits(t):
    return t.contiguous().view(torch.int32)


@pytest.mark.parametrize("h", [28, 40, 56])
@pytest.mark.parametrize("layout", ["nchw", "channels_last"])
@pytest.mark.parametrize("coords", ["views", "handmade"])
def test_kernels_vs_torch_and_fp64(cuda_dev, h, layout, coords):
    from stego_b200 import modules
    B, S = 8, 8 * h
    if coords == "views":
        coord, params = _views(B, S, 100 + h, cuda_dev)
        flips = {p["flip"] for p in params}
        edges = any(p["crop"][0] == 0 or p["crop"][1] == 0 or p["crop"][0] + p["crop"][2] == S
                    or p["crop"][1] + p["crop"][3] == S for p in params)
        assert flips == {True, False} and edges, "the seeds must cover both flips and a crop at the frame edge"
    else:
        coord = _handmade(B, S, h, cuda_dev)
    code = _code(B, h, layout, cuda_dev, seed=h)
    grid, sampled = _stage_fwd(coord, code)
    if coords == "handmade":  # the case holds what it claims: interior integer taps and border-clamped points
        pos = ((grid + 1) / 2) * (h - 1)  # fp32, grid_taps' arithmetic before the clamp
        assert int(((pos == pos.floor()) & (pos > 0) & (pos < h - 1)).sum()) >= B // 4 * h * h
        assert bool((grid > 1).any()) and bool((grid < -1).any())
    tgrid, tsampled = _torch_ref(coord, code)
    assert torch.equal(_bits(grid), _bits(tgrid)), int((_bits(grid) != _bits(tgrid)).sum())
    assert torch.equal(_bits(sampled), _bits(tsampled)), int((_bits(sampled) != _bits(tsampled)).sum())
    sbar = aug_sampled_bar(code, h)

    # fp64 restatement
    g64 = F.interpolate(coord.double().permute(0, 3, 1, 2), h, mode="bilinear", align_corners=False).permute(0, 2, 3, 1)
    assert (grid.double() - g64).abs().max().item() <= aug_grid_bar(coord)
    code64 = code.double().requires_grad_(True)
    s64 = F.grid_sample(code64, grid.double().permute(0, 2, 1, 3), padding_mode="border", align_corners=True)
    assert (sampled.double() - s64).abs().max().item() <= sbar

    # backward: d(sampled) from the cosine against a code_aug, scattered into d(code)
    code_aug = _code(B, h, "channels_last", cuda_dev, seed=h + 1)
    cosv, na, nb = (torch.empty(B, h, h, device=cuda_dev) for _ in range(3))
    modules.cosine_forward(sampled, code_aug, cosv, na, nb)
    w = 0.6
    dcos = torch.full((B, h, h), -w, device=cuda_dev).div_(B * h * h)
    dsampled = torch.empty_like(sampled)
    dcode_aug = torch.empty_strided(code_aug.shape, code_aug.stride(), device=cuda_dev)  # written with code_aug's strides
    modules.cosine_backward(sampled, code_aug, cosv, na, nb, dcos, dsampled, dcode_aug)
    dcode = torch.zeros_like(code)
    modules.aug_sample_backward(grid, dsampled, dcode)
    loss, total = torch.empty(1, device=cuda_dev), torch.full((1,), 2.0, device=cuda_dev)
    modules.aug_loss(cosv, w, loss, total)

    ca64 = code_aug.double().requires_grad_(True)
    s64 = F.grid_sample(code64, g64.permute(0, 2, 1, 3), padding_mode="border", align_corners=True)
    cos64 = (F.normalize(s64, dim=1, eps=1e-10) * F.normalize(ca64, dim=1, eps=1e-10)).sum(1)
    l64 = -cos64.mean()
    (w * l64).backward()
    # the fixed-order fp64 mean of the kernel's cosines, rounded once
    assert loss.item() == float(torch.tensor(-cosv.double().mean().item(), dtype=torch.float32))
    assert abs(loss.item() - l64.item()) <= 64 * U * cosv.abs().mean().item() + 1e-6
    assert total.item() == float(torch.tensor(2.0) + torch.tensor(w, dtype=torch.float32) * loss.cpu())

    # d(code) at the kernel's own grid and d(sampled): the scatter alone
    code64b = code.double().requires_grad_(True)
    sb = F.grid_sample(code64b, grid.double().permute(0, 2, 1, 3), padding_mode="border", align_corners=True)
    (sb * dsampled.double()).sum().backward()
    code64c = code.double().requires_grad_(True)
    sa = F.grid_sample(code64c, grid.double().permute(0, 2, 1, 3), padding_mode="border", align_corners=True)
    (sa * dsampled.double().abs()).sum().backward()
    bar = aug_scatter_bar(grid, code64c.grad, dsampled, h)
    err = (dcode.double() - code64b.grad).abs()
    assert bool((err <= bar).all()), float((err / bar).max())
    # and against torch's fp32 grid_sample backward (atomics in another order): the same bar
    ct = code.detach().clone().requires_grad_(True)
    F.grid_sample(ct, tgrid.permute(0, 2, 1, 3), padding_mode="border", align_corners=True).backward(dsampled)
    assert bool(((dcode.double() - ct.grad.double()).abs() <= 2 * bar).all())
    # the whole chain against fp64: d(code) and d(code_aug), relative to their norms
    assert rel(dcode, code64.grad) < 1e-5, rel(dcode, code64.grad)
    assert rel(dcode_aug, ca64.grad) < 1e-5, rel(dcode_aug, ca64.grad)


def _aug_batch(B, res, dev, seed):
    b = make_batch(B, res, dev, seed=seed)
    b["seed"] = [1000 * seed + i for i in range(B)]
    return b


def _one_step_each(fused, twin, batch, dev):
    torch.manual_seed(777)
    gpu_state, cpu_state = torch.cuda.get_rng_state(dev), torch.get_rng_state()
    loss_f = fused.training_step(batch, 0)
    after, after_cpu = torch.cuda.get_rng_state(dev), torch.get_rng_state()
    torch.cuda.set_rng_state(gpu_state, dev)
    torch.set_rng_state(cpu_state)
    loss_t = twin.training_step(batch, 0)
    assert fused._fused.step_idx == 1 and twin._fused is None
    assert torch.equal(torch.cuda.get_rng_state(dev), after), "CUDA generator consumption differs"
    assert torch.equal(torch.get_rng_state(), after_cpu), "CPU generator consumption differs"
    torch.cuda.synchronize()
    return loss_f, loss_t


def _check_logged(fused, twin, B, hw):
    got, want = fused.logged, twin.logged
    for key in ("loss/pos_intra", "loss/pos_inter", "cd/pos_intra", "cd/pos_inter", "loss/cluster"):
        assert torch.equal(got[key], want[key]), (key, got[key].item(), want[key].item())
    # the negative terms' mean: stego_step_losses on one path, a torch mean on the other (as without the aug term)
    nf, nt = got["loss/neg_inter"].item(), want["loss/neg_inter"].item()
    assert abs(nf - nt) <= 8 * U * abs(nt), (nf, nt)
    ws = fused._fused.ws
    ref = -ws.cosv.double().mean().item()
    n = B * hw
    a_f, a_t = got["loss/aug_alignment"].item(), want["loss/aug_alignment"].item()
    assert a_f == float(torch.tensor(ref, dtype=torch.float32)), (a_f, ref)
    assert torch.equal(want["loss/aug_alignment"], -ws.cosv.mean()), "the two paths' cosines differ"
    # torch's fp32 mean: at most n - 1 roundings of partial sums bounded by sum|cos|, and the division
    assert abs(a_t - ref) <= (n * U) * ws.cosv.abs().double().mean().item() + U * abs(ref), (a_t, ref)
    lin_f, lin_t = got["loss/linear"].item(), want["loss/linear"].item()
    assert abs(lin_f - lin_t) <= 1e-6 * abs(lin_t), (lin_f, lin_t)
    w = fused.cfg.aug_alignment_weight
    terms = [got[k].item() for k in ("loss/pos_intra", "loss/pos_inter", "loss/neg_inter", "loss/linear", "loss/cluster")]
    bar = abs(w) * abs(a_f - a_t) + abs(lin_f - lin_t) + 8 * U * (sum(abs(t) for t in terms) + abs(w * a_f))
    assert abs(got["loss/total"].item() - want["loss/total"].item()) <= bar


@pytest.mark.parametrize("shape,variant", [(("vit_small", 224, 8), "feat"), (("vit_base", 320, 4), "feat"),
                                           (("vit_small", 224, 8), "salience"), (("vit_small", 224, 8), "KK")])
def test_first_step_fused_vs_autograd(cuda_dev, shape, variant):
    arch, res, B = shape
    over = dict(aug_alignment_weight=0.6, res=res)
    if variant == "KK":
        over["dino_feat_type"] = "KK"
    if variant == "salience":
        over["use_salience"] = True
    fused, _ = make_model(arch, cuda_dev, fused=True, **over)
    twin, _ = make_model(arch, cuda_dev, fused=False, **over)
    batch = _aug_batch(B, res, cuda_dev, seed=1)
    if variant == "salience":
        g = torch.Generator().manual_seed(5)
        batch["mask"] = (torch.rand(B, 1, res, res, generator=g) > 0.6).float().to(cuda_dev)
        batch["mask_pos"] = (torch.rand(B, 1, res, res, generator=g) > 0.3).float().to(cuda_dev)
    _one_step_each(fused, twin, batch, cuda_dev)
    assert fused._fused.ws.aug and fused._fused.ws.n_img == 3
    _check_logged(fused, twin, B, (res // 8) ** 2)
    g_f, g_t = grads_of(fused), grads_of(twin)
    for k in NAMES:
        assert rel(g_f[k], g_t[k]) < 3e-3, (k, rel(g_f[k], g_t[k]))


def test_aug_term_gradient_wiring(cuda_dev):
    """The aug term's own contribution to the head gradients (step with the term minus step without it) agrees between
    the fused and the autograd path."""
    arch, res, B = "vit_small", 224, 8
    batch = _aug_batch(B, res, cuda_dev, seed=4)
    diffs = {}
    for fused in (True, False):
        g = {}
        for w in (0.6, 0.0):
            m, _ = make_model(arch, cuda_dev, fused=fused, aug_alignment_weight=w, res=res)
            torch.manual_seed(777)
            m.training_step(batch, 0)
            assert (m._fused is not None and m._fused.ws is not None) == fused
            g[w] = grads_of(m)
            del m
        diffs[fused] = {k: g[0.6][k] - g[0.0][k] for k in NAMES if k.startswith("net.")}
    for k in diffs[True]:
        d_f, d_t = diffs[True][k], diffs[False][k]
        assert d_t.abs().max().item() > 0, k
        assert rel(d_f, d_t) < 1e-3, (k, rel(d_f, d_t))


def test_cuda_seed_tensor_raises(cuda_dev):
    model, _ = make_model("vit_small", cuda_dev, fused=True, aug_alignment_weight=0.6, res=64)
    batch = _aug_batch(2, 64, cuda_dev, seed=2)
    batch["seed"] = torch.tensor(batch["seed"], device=cuda_dev)
    from stego_b200.fused_step import FusedStep
    assert not FusedStep(model).supported(batch)
    with pytest.raises(ValueError, match="CUDA tensor"):
        model.training_step(batch, 0)
    batch["seed"] = batch["seed"].cpu()
    assert FusedStep(model).supported(batch)
    with pytest.raises(ValueError, match="bfloat16"):
        model.training_step(dict(batch, img=batch["img"].bfloat16()), 0)


def test_histogram_step(cuda_dev):
    from types import SimpleNamespace
    models = []
    for fused in (True, False):
        m, _ = make_model("vit_small", cuda_dev, fused=fused, aug_alignment_weight=0.6, res=64, hist_freq=1)
        m.logger = SimpleNamespace(experiment=SimpleNamespace(add_histogram_raw=lambda *a, **k: None))
        models.append(m)
    batch = _aug_batch(4, 64, cuda_dev, seed=3)
    torch.manual_seed(5)
    for s in range(2):  # step 1 logs histograms
        st, st_cpu = torch.cuda.get_rng_state(cuda_dev), torch.get_rng_state()
        models[0].training_step(batch, s)
        after = torch.cuda.get_rng_state(cuda_dev)
        torch.cuda.set_rng_state(st, cuda_dev)
        torch.set_rng_state(st_cpu)
        models[1].training_step(batch, s)
        assert torch.equal(torch.cuda.get_rng_state(cuda_dev), after)
        torch.cuda.synchronize()
        g_f, g_t = grads_of(models[0]), grads_of(models[1])
        for k in NAMES:
            assert rel(g_f[k], g_t[k]) < 3e-3, (s, k, rel(g_f[k], g_t[k]))
        if s == 0:
            for key in ("loss/pos_intra", "loss/pos_inter", "cd/pos_intra", "cd/pos_inter", "loss/cluster"):
                assert torch.equal(models[0].logged[key], models[1].logged[key]), (s, key)
        else:  # the parameters differ in the last bits after one update (atomics): compare at a relative bar
            assert models[0]._fused.ws.hist is not None
            for key in ("loss/pos_intra", "loss/pos_inter", "loss/aug_alignment", "loss/cluster"):
                a, b = models[0].logged[key].item(), models[1].logged[key].item()
                assert abs(a - b) <= 1e-4 * abs(b) + 1e-6, (key, a, b)


def test_graph_capture_and_replay_match_eager(cuda_dev):
    """Three steps with cuda_graph=True (eager, capture, replay) log what three steps with cuda_graph=False log; the
    second step captures the tail graph and the views go straight into the backbone graph's input."""
    runs = {}
    for use_graph in (True, False):
        m, _ = make_model("vit_small", cuda_dev, fused=True, aug_alignment_weight=0.6, res=64, cuda_graph=use_graph)
        batches = [_aug_batch(4, 64, cuda_dev, seed=s) for s in (1, 2, 1)]
        torch.manual_seed(9)
        logs = []
        for s, b in enumerate(batches):
            m.training_step(b, s)
            torch.cuda.synchronize()
            logs.append({k: v.item() for k, v in m.logged.items()})
            ws = m._fused.ws
            assert (ws.graph is not None) == (use_graph and s >= 1), s
        runs[use_graph] = logs
    for s in range(3):
        for k, v in runs[False][s].items():
            g = runs[True][s][k]
            if s == 0:
                assert g == v, (s, k, g, v)  # same kernels on the same inputs
            else:
                assert abs(g - v) <= 1e-4 * abs(v) + 1e-6, (s, k, g, v)


def test_shipped_configuration_unchanged(cuda_dev):
    """aug_alignment_weight = 0: seeds in the batch change nothing, and the workspace has no aug buffers."""
    a, _ = make_model("vit_small", cuda_dev, fused=True)
    b, _ = make_model("vit_small", cuda_dev, fused=True)
    batch = make_batch(4, 64, cuda_dev, seed=1)
    torch.manual_seed(777)
    a.training_step(batch, 0)
    torch.manual_seed(777)
    b.training_step(dict(batch, seed=[1, 2, 3, 4]), 0)
    torch.cuda.synchronize()
    assert not a._fused.ws.aug and a._fused.ws.n_img == 2 and "loss/aug_alignment" not in a.logged
    for k in a.logged:
        assert torch.equal(a.logged[k], b.logged[k]), k
