"""The probe kernels (csrc/probes.cu) and the eval-frame kernels (csrc/eval_probes.cu) against float64 references at
the production shapes, with the edges where they go wrong: saturated softmax, exact ties, zero pixels and centroids,
ignored labels down to a whole batch, logit spreads of +-100, batch-strided views and nearly cancelling neighbours.

Every bar is derived from the arithmetic (u = 2^-24, fp32 FMA chains, fast exponentials, atomic accumulation; see each
test and DESIGN.md section 4) from the per-element sums of |terms| the fp64 references in tests/_probes_fp64.py
return.  The largest error / bar ratios are written to $STEGO_PARITY_DIR when it is set.  test_intended_kernels_ran
checks with torch.profiler, in a child process (CUPTI state must not leak into the CUDA-graph captures of later tests),
that each kind of case launches the kernel it means to test.
"""
import json
import os
import subprocess
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _probes_fp64 as R  # noqa: E402
from _parity_util import grads_of, make_batch, make_model, params_of, record, rel  # noqa: E402

pytestmark = pytest.mark.gpu
U = R.U


_PROFILER_READY = False


def _kernels(fn):
    """Run fn under torch.profiler; return its result and the names of the CUDA kernels it launched.  The first
    sessions of a process can miss kernel records while the profiler initialises, so two throw-away sessions come first."""
    global _PROFILER_READY
    from torch.profiler import ProfilerActivity, profile
    if not _PROFILER_READY:
        for _ in range(2):
            with profile(activities=[ProfilerActivity.CUDA]):
                torch.ones(1024, device="cuda").sum().item()
        _PROFILER_READY = True
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
    return out, names


def _ran(names, want, not_want=()):
    assert any(want in n for n in names), (want, sorted(names))
    for w in not_want:
        assert not any(w in n for n in names), (w, sorted(names))


def _ratio(err, bar):
    """max err / bar over elements (0 / 0 counts as 0)"""
    return float(torch.where(err == 0, torch.zeros_like(err), err / bar).max())


# ================================================================================================
# 1. ClusterLookup
# ================================================================================================
def _cluster_run(x4, cl, alpha, grad):
    from stego_b200 import _lib
    lib = _lib.load()
    B, C, H, W = x4.shape
    n, dev = cl.shape[0], x4.device
    assert x4.stride(2) == W * x4.stride(3)
    P = H * W
    assign = torch.full((B, P), -1, dtype=torch.long, device=dev)
    probs = torch.empty(B, n, P, device=dev)
    logp = torch.empty(B, n, P, device=dev) if alpha is not None else None
    loss = torch.empty(2, device=dev)
    scratch = torch.empty(16 * torch.cuda.get_device_properties(dev).multi_processor_count, device=dev)
    g = torch.tensor([grad], device=dev)
    dnc = torch.zeros(n, C, device=dev)
    dcl = torch.zeros(n, C, device=dev)
    a = (int(alpha is not None), float(alpha or 0.0))
    _lib.check(lib.stego_cluster_lookup_fwd(_lib.ptr(x4), x4.stride(0), x4.stride(1), x4.stride(3), _lib.ptr(cl), B, C, n, P,
                                            *a, _lib.ptr(assign), _lib.ptr(probs), _lib.ptr(logp), _lib.ptr(loss),
                                            _lib.ptr(scratch), _lib.stream()), "cluster fwd")
    _lib.check(lib.stego_cluster_lookup_bwd(_lib.ptr(x4), x4.stride(0), x4.stride(1), x4.stride(3), _lib.ptr(cl), B, C, n, P,
                                            *a, _lib.ptr(g), _lib.ptr(dnc), _lib.ptr(dcl), _lib.stream()), "cluster bwd")
    return dict(assign=assign, probs=probs, logp=logp, loss=loss[0], dnc=dnc, dcl=dcl)


def _chain(total, dev, channels_last_bwd):
    """Longest fp32 accumulation chain of one dnc element: pixels per CTA (shared-memory atomics) + CTAs (global
    atomics), for the launch geometry of stego_cluster_lookup_bwd."""
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    per, cap = (8, 4 * sms) if channels_last_bwd else (128, 8 * sms)
    grid = min((total + per - 1) // per, cap)
    return -(-total // (grid * per)) * per + grid


def _cluster_check(x4, cl, alpha, grad, tag, regime):
    """Bars (C channels, n centroids, S = sum_c |x_hat_c c_hat_kc| <= 1 from the reference):
      inner product   E_ip = (2C + 16) u S: C-term FMA chain, plus two fp32 normalisations ((C/2 + 3) u each: sum of
                      squares, sqrt, reciprocal) and the rounding of x * inv.
      assignment      equal to the fp64 argmax wherever the fp64 top-2 margin exceeds 2 max_k E_ip; the rest counted.
      log-probs       alpha (E_ip_k + max_j E_ip_j) + (n + 8) u (1 + alpha) + u |logp|: the logits' error moves the
                      log-sum-exp by at most max_j; expf / logf (2 ulp) over n terms.  probs: p (bar_logp + 4 u).
      loss            mean of the per-pixel bar (max ip, or sum_k |dp_k ip_k| + p_k E_ip_k) + 32 u mean |term|: each
                      partial sums at most 16 fp32 terms before the fp64 reduction.
      dnc (d loss / d normalised centroids)  |gs| [sum_p ddip_k |x_hat_c| + (L + C/2 + 6) u sum_p |dip_k x_hat_c|],
                      L = pixels per CTA + CTAs (the two atomic levels); ddip from dp and E_ip; pixels off the safe
                      margin may go to either candidate centroid, so their |gs x_hat| is added to both rows.
      dclusters       normalise backward of dnc: (D + c_hat sum|c_hat| D) / |c| + (C + 8) u (|dnc| + |c_hat| |c_hat . dnc|) / |c|,
                      and (D + u |dnc|) 1e12 for an all-zero row."""
    dev = x4.device
    B, C, H, W = x4.shape
    n, P = cl.shape[0], H * W
    got = _cluster_run(x4, cl, alpha, grad)
    ref = R.cluster_ref(x4.reshape(B, C, P), cl, alpha, grad)
    ip, S = ref["ip"], ref["S"]
    E_ip = (2 * C + 16) * U * S
    Emax = E_ip.amax(1)
    top2 = ip.topk(2, 1).values
    margin = top2[:, 0] - top2[:, 1]
    safe = margin > 2 * Emax
    arg = got["assign"]
    m = {}
    assert (arg >= 0).all() and (arg < n).all()
    assert torch.equal(arg[safe], ref["arg"][safe]), (tag, int((arg[safe] != ref["arg"][safe]).sum()))
    near = ~safe
    m["near_ties"], m["pixels"] = int(near.sum()), B * P
    if regime == "ties":  # exact fp32 ties by construction: the first maximum wins, as in torch.argmax
        assert not (arg == 1).any(), tag
        assert not (arg[:, P // 2:] == 3).any(), tag
    elif regime == "zeros":
        zero = (x4.reshape(B, C, P) == 0).all(1)
        assert zero.any() and (arg[zero] == 0).all(), tag
    else:
        assert m["near_ties"] <= max(4, 2e-3 * B * P), (tag, m)
    L = _chain(B * P, dev, x4.stride(1) == 1 and n <= 32 and alpha is None)
    xh, gs = ref["xh"], abs(ref["gs"])
    if alpha is None:
        assert torch.equal(got["probs"], torch.nn.functional.one_hot(arg, n).permute(0, 2, 1).float())
        term = top2[:, 0]
        loss_bar = (Emax.mean() + 32 * U * term.abs().mean()).item()
        ddip = torch.zeros_like(ip)
        mix = torch.zeros(n, C, dtype=torch.float64, device=dev)
        nb, npix = near.nonzero(as_tuple=True)
        if len(nb):
            xa = xh[nb, :, npix].abs() * gs
            mix.index_add_(0, ref["arg"][nb, npix], xa)
            mix.index_add_(0, arg[nb, npix], xa)
    else:
        lp, p = ref["logp"], ref["probs"]
        bar_lp = alpha * (E_ip + Emax[:, None]) + (n + 8) * U * (1 + alpha) + U * lp.abs()
        m["logp"] = _ratio((got["logp"].double() - lp).abs(), bar_lp)
        bar_p = p * (bar_lp + 4 * U)
        m["probs"] = _ratio((got["probs"].double() - p).abs(), bar_p)
        dotp = (p * ip).sum(1, keepdim=True)
        ddot = (bar_p * ip.abs() + p * E_ip).sum(1, keepdim=True)
        loss_bar = (ddot.mean() + 32 * U * dotp.abs().mean()).item()
        ddip = bar_p * (1 + alpha * (ip - dotp).abs()) + alpha * p * (E_ip + ddot)
        mix = torch.zeros(n, C, dtype=torch.float64, device=dev)
    m["loss"] = abs(got["loss"].item() - ref["loss"].item()) / loss_bar
    D = gs * (torch.einsum("bkp,bcp->kc", ddip, xh.abs()) +
              (L + C / 2 + 6) * U * torch.einsum("bkp,bcp->kc", ref["dip"].abs(), xh.abs())) + mix
    m["dnc"] = _ratio((got["dnc"].double() - ref["dnc"]).abs(), D + 1e-300)
    cd, dnc, ch = cl.double(), ref["dnc"], ref["ch"]
    nrm = cd.norm(dim=1, keepdim=True)
    full = (D + ch.abs() * (ch.abs() * D).sum(1, keepdim=True)) / nrm.clamp_min(1e-12) + \
        (C + 8) * U * (dnc.abs() + ch.abs() * (ch * dnc).sum(1, keepdim=True).abs()) / nrm.clamp_min(1e-12)
    zero_row = (D + U * dnc.abs()) / 1e-12
    bar_dcl = torch.where(nrm > 1e-12, full, zero_row)
    m["dcl"] = _ratio((got["dcl"].double() - ref["dcl"]).abs(), bar_dcl + 1e-300)
    assert torch.isfinite(got["dcl"]).all(), tag
    record(f"probes_fp64_cluster_{tag}", m)
    for k, v in m.items():
        if k not in ("near_ties", "pixels"):
            assert v <= 1.0, (tag, k, m)
    return m


CLUSTER_REGIMES = ("random", "sharp", "ties", "zeros", "zerorow")


def _code_view(x, dev, ld=72):
    """The training step's code layout: [B, h*w, 72] fp32 storage, [B, C, h, w] channels-last view"""
    B, C, P = x.shape
    side = int(round(P ** 0.5))
    buf = torch.full((B, P, ld), float("nan"), device=dev)
    buf[..., :C] = x.permute(0, 2, 1)
    return buf.view(B, side, side, ld)[..., :C].permute(0, 3, 1, 2)


@pytest.mark.parametrize("regime", CLUSTER_REGIMES)
@pytest.mark.parametrize("shape", ["c1", "c2", "c3"])
def test_cluster_lookup_fp64(cuda_dev, shape, regime):
    """ClusterLookup on the step's channels-last code at c1 / c2 / c3 (C = 70, n = 27): alpha=None forward and backward
    (the training configuration) and alpha forward + backward (2, or 50 for the saturated regime)."""
    B, h, _ = R.TRAIN[shape]
    x, cl = R.cluster_inputs(regime, B, R.DIM, h * h, R.NCLS, seed=hash((shape, regime)) % 1000, device=cuda_dev)
    x4 = _code_view(x, cuda_dev)
    _cluster_check(x4, cl, None, 1.0, f"{shape}_{regime}_argmax", regime)
    alpha = 50.0 if regime == "sharp" else 2.0
    _cluster_check(x4, cl, alpha, 0.7, f"{shape}_{regime}_softmax", regime)


@pytest.mark.parametrize("n", [33, 48, 64])
@pytest.mark.parametrize("regime", ["random", "ties", "zerorow"])
def test_cluster_lookup_generic_kernel_fp64(cuda_dev, n, regime):
    """The per-thread kernel at its limits: NCHW input, n = 33..64 centroids, C = 96, both modes."""
    x, cl = R.cluster_inputs(regime, 4, 96, 24 * 24, n, seed=n, device=cuda_dev)
    x4 = x.view(4, 96, 24, 24)
    for alpha in (None, 3.0):
        _cluster_check(x4, cl, alpha, 1.3, f"generic_n{n}_{regime}_{'argmax' if alpha is None else 'softmax'}", regime)


# ================================================================================================
# 2. linear probe + bilinear upsample + masked cross entropy
# ================================================================================================
def _lce_run(code4, W, b, label, n, grad, dW0, db0):
    from stego_b200 import _lib
    lib = _lib.load()
    B, C, h, w = code4.shape
    H, Wd = label.shape[-2:]
    assert code4.stride(1) == 1 and code4.stride(2) == w * code4.stride(3) and code4.stride(0) == h * w * code4.stride(3)
    dev = code4.device
    rows = B * h * w
    logits = torch.empty(rows, 32, device=dev)
    dlogits = torch.zeros(rows, 32, device=dev)
    partials = torch.empty(64, device=dev)
    loss = torch.empty(2, device=dev)
    dW, db = dW0.clone(), db0.clone()
    lb = {torch.int64: 8, torch.int32: 4, torch.uint8: 1}[label.dtype]
    _lib.check(lib.stego_linear_probe_ce(_lib.ptr(code4), code4.stride(3), C, _lib.ptr(W), _lib.ptr(b), n, _lib.ptr(label), lb,
                                         B, h, w, H, Wd, _lib.ptr(logits), _lib.ptr(dlogits), _lib.ptr(partials),
                                         _lib.ptr(loss), float(grad), _lib.ptr(dW), _lib.ptr(db), _lib.stream()),
               "stego_linear_probe_ce")
    return dict(loss=loss[0], count=loss[1], dW=dW, db=db)


def _lce_bars(code4, ref, n, H, W):
    """Bars (C channels, n classes; Ml = |b| + sum_c |W_kc x_c| per low-res logit, from the reference):
      low-res logit   E_l = (C + 1) u Ml (FMA chain from the bias)
      upsampled       E_z = sum_t w_t E_l + 6 u sum_t w_t |l_t| (x then y interpolation, 3 roundings each)
                      + e_y |l_bottom - l_top| + e_x |l_right - l_left|, e = the fp32 weight's distance from the fp64
                      one (0 at power-of-two ratios; ~1e-7 of the logit step otherwise)
      CE per pixel    E_z[label] + max_k E_z + (2 + 1.5 n) u + 2^-20.4 + 2 u (|z_lab - max| + |ce|): __expf is
                      (2 + 1.17 |z - max|) ulp and sum_k e^(z_k - max) |z_k - max| <= n / e; __logf absolute error
      loss            sum of the CE bars / count + 8 u mean |ce| (warp sums) + u |loss|
      softmax         rho_k = E_z,k + max E_z + (4 + 1.2 |z_k - max| + 1.5 n) u relative, + u |g| for the -1
      logit grad      interp^T(rho p) + (34 + A) u interp^T |g| + (e_y + e_x) per-corner |g|: 16 + 16 FMAs of the
                      separable reduction, A tiles' atomics per cell
      dW, db          s [dDl |x| + (128 + R / 128 + 4) u |dl| |x|] + u |result|: 128-row FMA chain per CTA, one atomic
                      per CTA and output, s = grad / count; each of the R / 128 atomics rounds the running value, so
                      accumulating into a non-zero dW0 adds (R / 128) u |dW0| (in _lce_case)."""
    B, C, h, w = code4.shape
    cr = ref["corners"]
    A = ((2 * H // h + 2) // 16 + 2) * ((2 * W // w + 2) // 16 + 2)
    s = abs(ref["s"])
    ddl = torch.zeros_like(ref["dl"])
    adl = torch.zeros_like(ref["dl"])
    num, ce_abs = 0.0, 0.0
    for b, pi in enumerate(ref["per"]):
        E_l = (C + 1) * U * pi["Ml"]
        E_z = cr.interp(E_l) + 6 * U * cr.wabs(pi["l"]) + cr.lam_term(pi["l"])
        Emax = E_z.amax(0)
        z, p, lab, v = pi["z"], pi["p"], pi["lab"], pi["valid"]
        mx = z.amax(0)
        zl = z.gather(0, lab[None])[0]
        E_ce = E_z.gather(0, lab[None])[0] + Emax + (2 + 1.5 * n) * U + R.LOGF_ABS + 2 * U * ((zl - mx).abs() + pi["ce"].abs())
        num += float((E_ce + 8 * U * pi["ce"].abs())[v].sum())
        ce_abs += float(pi["ce"].abs()[v].sum())
        rho = E_z + Emax + (4 + 1.2 * (z - mx).abs() + 1.5 * n) * U
        dg = (rho * p + U * pi["g"].abs()) * v[None].double()
        R.adjoint_into(ddl[b], cr, dg)
        R.adjoint_into(ddl[b], cr, pi["g"].abs(), [cr.ey + cr.ex] * 4)
        R.adjoint_into(adl[b], cr, pi["g"].abs())
    ddl += (34 + A) * U * adl
    rows = B * h * w
    K = 128 + rows / 128 + 4
    X = code4.double().reshape(B, C, h * w).abs()
    cnt = max(ref["count"], 1)
    loss_bar = num / cnt + (abs(ref["loss"].item()) * U if ref["count"] else 0.0)
    dW_bar = s * (torch.einsum("bkr,bcr->kc", ddl, X) + K * U * torch.einsum("bkr,bcr->kc", ref["dl"].abs(), X))
    db_bar = s * (ddl.sum((0, 2)) + K * U * ref["dl"].abs().sum((0, 2)))
    return loss_bar, dW_bar, db_bar


def _lce_case(dev, tag, B, h, w, H, W, n, label_dtype=torch.int64, ignore="random", spread=4.0, grad=1.0,
              accumulate=False, view=None):
    code, Wt, b, label = R.linear_inputs(B, R.DIM, h, w, H, W, n, spread, label_dtype, ignore, seed=h * 7 + W + n,
                                         device=dev)
    code4 = code.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
    g = torch.Generator(device=dev).manual_seed(5)
    dW0 = torch.randn(n, R.DIM, device=dev, generator=g) if accumulate else torch.zeros(n, R.DIM, device=dev)
    db0 = torch.randn(n, device=dev, generator=g) if accumulate else torch.zeros(n, device=dev)
    got = _lce_run(code4, Wt, b, label, n, grad, dW0, db0)
    ref = R.linear_ce_ref(code4, Wt, b, label, n, grad)
    loss_bar, dW_bar, db_bar = _lce_bars(code4, ref, n, H, W)
    dW_want, db_want = dW0.double() + ref["dW"], db0.double() + ref["db"]
    G = -(-B * h * w // 128)  # atomics per output element (linear_wgrad_kernel CTAs)
    dW_bar = dW_bar + U * dW_want.abs() + G * U * dW0.double().abs()
    db_bar = db_bar + U * db_want.abs() + G * U * db0.double().abs()
    m = dict(count=ref["count"])
    assert int(got["count"].item()) == ref["count"], (tag, got["count"].item(), ref["count"])
    assert torch.isfinite(got["dW"]).all() and torch.isfinite(got["db"]).all(), tag
    if ref["count"] == 0:  # the reference: NaN loss, zero gradient
        assert torch.isnan(got["loss"]).item(), tag
        assert torch.equal(got["dW"], dW0) and torch.equal(got["db"], db0), tag
    else:
        m["loss"] = abs(got["loss"].item() - ref["loss"].item()) / loss_bar
    m["dW"] = _ratio((got["dW"].double() - dW_want).abs(), dW_bar)
    m["db"] = _ratio((got["db"].double() - db_want).abs(), db_bar)
    record(f"probes_fp64_linear_{tag}", m)
    for k in ("loss", "dW", "db"):
        if k in m:
            assert m[k] <= 1.0, (tag, k, m)
    return m


@pytest.mark.parametrize("shape", ["c1", "c2", "c3"])
def test_linear_probe_ce_production_fp64(cuda_dev, shape):
    """28 -> 224, 40 -> 320, 56 -> 448 at the training batch, n = 27, int64 labels with -1 / n ignored."""
    B, h, H = R.TRAIN[shape]
    _lce_case(cuda_dev, shape, B, h, h, H, H, 27)


@pytest.mark.parametrize("n", [5, 27, 32])
@pytest.mark.parametrize("ratio", ["7x9to50x61", "identity", "down_y", "down_x"])
def test_linear_probe_ce_ratios_fp64(cuda_dev, ratio, n):
    """Non-integer upsampling, identity, and downsampling: 40 -> 12 rows (the box clamped to h) and 40 -> 12
    columns (box clamped to w; bw * n > 256 for n >= 27 takes the strided branch of the transpose-reduction)."""
    B, h, w, H, W = {"7x9to50x61": (3, 7, 9, 50, 61), "identity": (2, 28, 28, 28, 28), "down_y": (2, 40, 8, 12, 64),
                     "down_x": (2, 8, 40, 64, 12)}[ratio]
    dt = {5: torch.int32, 27: torch.uint8, 32: torch.int64}[n]
    _lce_case(cuda_dev, f"{ratio}_n{n}", B, h, w, H, W, n, label_dtype=dt)


@pytest.mark.parametrize("ignore", ["tiles", "image", "all"])
@pytest.mark.parametrize("label_dtype", [torch.int64, torch.int32, torch.uint8])
def test_linear_probe_ce_ignored_fp64(cuda_dev, ignore, label_dtype):
    """Whole 16 x 16 tiles, one whole image, and every pixel of the batch ignored.  With no valid pixel the loss is NaN
    (0 / 0, as the reference's CrossEntropyLoss over an empty selection) and dW, db stay exactly as they were."""
    _lce_case(cuda_dev, f"ignore_{ignore}_{str(label_dtype)[6:]}", 4, 28, 28, 224, 224, 27, label_dtype=label_dtype,
              ignore=ignore, grad=0.37, accumulate=True)


@pytest.mark.parametrize("spread", [30.0, 100.0])
def test_linear_probe_ce_spread_and_accumulate_fp64(cuda_dev, spread):
    """Logits spread over +-spread (saturated softmax, __expf far from 0), upstream gradient 0.37 accumulated into
    non-zero dW, db."""
    _lce_case(cuda_dev, f"spread{int(spread)}", 8, 40, 40, 320, 320, 27, spread=spread, grad=0.37, accumulate=True)


@pytest.mark.parametrize("view", ["batch_step", "row_crop"])
def test_linear_probe_ce_strided_views(cuda_dev, view):
    """segmenter.linear_probe_ce on channels-last code views whose batch stride is not h*w*ld: code[::2] and
    code[:, :, 1:].  Image b > 0 must be read from its own pixels (the loss and the gradients against fp64)."""
    from stego_b200.segmenter import linear_probe_ce
    dev = cuda_dev
    B, h, H, n = 6, 28, 224, 27
    code, Wt, b, label = R.linear_inputs(B, R.DIM, h + 1, h, H, H, n, seed=3, device=dev)
    store = torch.zeros(B, h + 1, h, 72, device=dev)
    store[..., :R.DIM] = code.permute(0, 2, 3, 1)
    full = store[..., :R.DIM].permute(0, 3, 1, 2)
    x = full[::2, :, :h] if view == "batch_step" else full[:3, :, 1:]
    lab = label[:3]
    assert x.stride(0) != h * h * 72
    Wp = torch.nn.Parameter(Wt.view(n, R.DIM, 1, 1).clone())
    bp = torch.nn.Parameter(b.clone())
    loss = linear_probe_ce(x, Wp, bp, lab)
    loss.backward()
    xc = x.contiguous()
    ref = R.linear_ce_ref(xc, Wt, b, lab, n)
    loss_bar, dW_bar, db_bar = _lce_bars(xc, ref, n, H, H)
    m = dict(loss=abs(loss.item() - ref["loss"].item()) / loss_bar,
             dW=_ratio((Wp.grad.view(n, R.DIM).double() - ref["dW"]).abs(), dW_bar + U * ref["dW"].abs()),
             db=_ratio((bp.grad.double() - ref["db"]).abs(), db_bar + U * ref["db"].abs()))
    record(f"probes_fp64_linear_view_{view}", m)
    for k, v in m.items():
        assert v <= 1.0, (view, k, m)


# ================================================================================================
# 3. the c4 eval frame: flip-TTA + upsample + both probes + confusion counts
# ================================================================================================
def _eval_modules(dev, n_lin, n_clu, seed):
    from stego_b200.modules import ClusterLookup
    g = torch.Generator(device=dev).manual_seed(seed)
    lin = torch.nn.Conv2d(R.DIM, n_lin, (1, 1)).to(dev)
    clu = ClusterLookup(R.DIM, n_clu).to(dev)
    with torch.no_grad():
        lin.weight.copy_(torch.randn(n_lin, R.DIM, 1, 1, generator=g, device=dev) * 0.3)
        lin.bias.copy_(torch.randn(n_lin, generator=g, device=dev) * 0.1)
        clu.clusters.copy_(torch.randn(n_clu, R.DIM, generator=g, device=dev))
    return lin, clu


def _lse_bar(z):
    """log-sum-exp of fp32 logits z [n, pix] with __expf / ex2.approx and __logf: each exponential's argument carries
    ~2 u (|z| + |max|) of rounding (x log2 e and the max shift), ex2.approx 2^-22; n-term sum; __logf absolute."""
    n = z.shape[0]
    return (6 + n + 5 * z.abs().amax(0)) * U + R.LOGF_ABS


def _eval_case(dev, tag, code, lin, clu, H, W, flip=None, anticorr=False, alpha=2.0, n_cls=27):
    """Bars per output pixel (C channels; M sums from the reference):
      linear logit    E_z = sum_t w_t (C + 3) u Ml_t + 8 u sum_t |l_t| + lambda term: the low-res FMA chain (the TTA
                      average rounds once), and the interpolation, whose vertical / horizontal differences (vec4
                      kernel) round relative to the corners, not to the weighted sum
      cluster dots    E_dv = sum_t w_t (1.5 C + 8) u Mdc_t + 8 u sum_t |dc_t| + lambda term (centroid normalisation)
      norm            |v|^2 = sum_tt' w_t w_t' <x_t, x_t'> from fp64 Gram entries of the fp32 code, combined in fp64 with
                      the fp32 weights (rounded by <= 3 u): relative error of 1 / |v|
                      eta = 3 u A / |v| + (C + 18) 2^-53 A^2 / (2 |v|^2) + lambda + 4 u, A = sum_t w_t |x_t|: first order
                      in the conditioning A / |v| (in fp32 the second term would be (C + 18) u A^2 / (2 |v|^2))
      cosine          E_cos = E_dv / |v| + |cos| eta;  logits alpha cos
      log-probs       E_k + max_j E_j + lse bar (_lse_bar) + u (|logp| + |lse|)
    anticorr: the bar is 4 x the error bound of the fp32 reference sequence (upsample, normalise, dot) at that pixel,
      [sum_c |c_hat_c| 3 u sum_t w_t |x_tc| + (C + 2) u |c_hat| . |v|] / |v| + |cos| (3 u |sum_t w_t |x_t|| / |v| + (C/2 + 3) u),
      which is first order in the conditioning: the fused kernel must not be much worse than upsampling first.
    argmax: equal to the fp64 argmax where the top-2 log-prob margin exceeds twice the bar; confusion counts exactly
    those of the kernel's own argmax maps, and within 2 x the near-tie count of the fp64 argmax's counts."""
    from stego_b200.eval import fused_probe_log_probs
    B, C, h, w = code.shape
    n_lin, n_clu = lin.weight.shape[0], clu.clusters.shape[0]
    g = torch.Generator(device=dev).manual_seed(17)
    label = torch.randint(-1, n_cls + 2, (B, H, W), generator=g, device=dev)
    lc = torch.zeros(n_lin, n_cls, dtype=torch.int64, device=dev)
    cc = torch.zeros(n_clu, n_cls, dtype=torch.int64, device=dev)
    ll, cl_, la, ca = fused_probe_log_probs(code, lin, clu, (H, W), alpha, want_argmax=True, code_flipped=flip,
                                            label=label, linear_confusion=lc, cluster_confusion=cc)
    assert torch.equal(lc, R.confusion(la, label, n_lin, n_cls)), tag
    assert torch.equal(cc, R.confusion(ca, label, n_clu, n_cls)), tag
    Wl, bl, cls = lin.weight.detach().view(n_lin, C), lin.bias.detach(), clu.clusters.detach()
    m = dict(lin_logp=0.0, clu_logp=0.0, lin_near=0, clu_near=0)
    ref_la = torch.empty(B, H, W, dtype=torch.long, device=dev)
    ref_ca = torch.empty_like(ref_la)
    band = 128
    for b in range(B):
        xbar = R.tta_code(code[b:b + 1], None if flip is None else flip[b:b + 1])[0]
        for y0 in range(0, H, band):
            rows = (y0, min(H, y0 + band))
            e = R.eval_band(xbar, Wl, bl, cls, alpha, H, W, rows)
            cr = e["corners"]
            sl = (b, slice(None), slice(*rows))
            # linear probe
            z = e["z"]
            E_z = cr.interp((C + 3) * U * e["Ml"]) + 8 * U * sum(t.abs() for t in cr.gather(e["l"])) + cr.lam_term(e["l"])
            lse = torch.logsumexp(z, 0)
            bar = E_z + E_z.amax(0) + _lse_bar(z) + U * (e["lin_logp"].abs() + lse.abs())
            got = ll[sl].reshape(n_lin, -1).double()
            m["lin_logp"] = max(m["lin_logp"], _ratio((got - e["lin_logp"]).abs(), bar))
            m["lin_near"] += _argmax_check(la[b, rows[0]:rows[1]].reshape(-1), e["lin_logp"], bar, ref_la[b, rows[0]:rows[1]], tag)
            # cluster probe
            vn, cos = e["vnorm"], e["cos"]
            E_dv = cr.interp((1.5 * C + 8) * U * e["Mdc"]) + 8 * U * sum(t.abs() for t in cr.gather(e["dc"])) + \
                cr.lam_term(e["dc"])
            xn = xbar.reshape(C, -1).norm(dim=0, keepdim=True)
            lam_n = 2 * (cr.ey + cr.ex) * torch.stack(cr.gather(xn)).amax(0)[0]
            if anticorr:
                ch = e["ch"]
                wabs_norm = e["wabs_x"].norm(dim=0)
                v_abs = (cr.interp(xbar.reshape(C, -1))).abs()
                E_cos = (ch.abs() @ (3 * U * e["wabs_x"]) + (C + 2) * U * (ch.abs() @ v_abs)) / vn + \
                    cos.abs() * (3 * U * wabs_norm / vn + (C / 2 + 3) * U + lam_n / vn)
                E_cos = 4 * E_cos
            else:
                A = e["wxn"]
                eta = 3 * U * A / vn + (C + 18) * 2.0 ** -53 * A ** 2 / (2 * vn ** 2) + lam_n / vn + 4 * U
                eta = torch.where(eta < 0.5, eta, torch.full_like(eta, float("inf")))
                E_cos = E_dv / vn + cos.abs() * eta
            zero = vn == 0
            E_s = alpha * E_cos + 2 * U * alpha * cos.abs()
            E_s = torch.where(zero[None], torch.zeros_like(E_s), E_s)
            s = alpha * cos
            lse = torch.logsumexp(s, 0)
            bar = E_s + E_s.amax(0) + _lse_bar(s) + U * (e["clu_logp"].abs() + lse.abs())
            got = cl_[sl].reshape(n_clu, -1).double()
            m["clu_logp"] = max(m["clu_logp"], _ratio((got - e["clu_logp"]).abs(), bar))
            m["clu_near"] += _argmax_check(ca[b, rows[0]:rows[1]].reshape(-1), e["clu_logp"], bar, ref_ca[b, rows[0]:rows[1]], tag)
            if zero.any():
                assert (ca[b, rows[0]:rows[1]].reshape(-1)[zero] == 0).all(), tag
            del e
    for pred, ref_pred, cm, near, n_pred in ((la, ref_la, lc, m["lin_near"], n_lin), (ca, ref_ca, cc, m["clu_near"], n_clu)):
        diff = int((cm - R.confusion(ref_pred, label, n_pred, n_cls)).abs().sum())
        assert diff <= 2 * near, (tag, diff, near)
    m["pixels"] = B * H * W
    record(f"probes_fp64_eval_{tag}", m)
    assert m["lin_logp"] <= 1.0 and m["clu_logp"] <= 1.0, (tag, m)
    # near-ties are where the two top log-probs are within twice the (worst-case) bar of each other
    assert m["lin_near"] <= 2e-2 * B * H * W and m["clu_near"] <= 2e-2 * B * H * W, (tag, m)
    return m


def _argmax_check(got, logp, bar, ref_out, tag):
    """kernel argmax == fp64 argmax off near-ties (top-2 margin <= 2 x the larger bar); returns the near-tie count"""
    top2 = logp.topk(2, 0)
    margin = top2.values[0] - top2.values[1]
    safe = margin > 2 * bar.amax(0)
    ref_out.copy_(top2.indices[0].view(ref_out.shape))
    assert torch.equal(got.long()[safe], top2.indices[0][safe]), (tag, int((got.long()[safe] != top2.indices[0][safe]).sum()))
    return int((~safe).sum())


def _c4_code(dev, regime, seed=0):
    B, h, w, _, _ = R.EVAL_C4
    g = torch.Generator(device=dev).manual_seed(seed)
    if regime.startswith("anticorr"):
        return R.anticorrelated_code(B, R.DIM, h, w, float(regime[len("anticorr"):]), seed=seed, device=dev)
    code = torch.randn(B, R.DIM, h, w, generator=g, device=dev)
    if regime == "zeros":
        code[:, :, 10:13, 20:23] = 0.0   # output pixels whose four corners are all zero: v = 0
        code[:, :, ::9, ::11] = 0.0
    return code


def _cl(t):
    return t.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)


@pytest.mark.parametrize("regime", ["random", "flip", "zeros", "anticorr1e-1", "anticorr1e-2", "anticorr1e-3"])
def test_eval_frame_vec4_fp64(cuda_dev, regime):
    """The c4 frame (4 x 128 x 256 -> 1024 x 2048, 27 / 27 classes): eval_probe_vec4_kernel<27, 27>."""
    _, _, _, H, W = R.EVAL_C4
    code = _cl(_c4_code(cuda_dev, regime))
    flip = _cl(_c4_code(cuda_dev, "random", seed=1)) if regime == "flip" else None
    lin, clu = _eval_modules(cuda_dev, 27, 27, seed=2)
    _eval_case(cuda_dev, f"vec4_{regime}", code, lin, clu, H, W, flip=flip, anticorr=regime.startswith("anticorr"))


@pytest.mark.parametrize("variant", ["factor6", "factor6_flip", "nclu30", "nclu30_flip"])
def test_eval_frame_generic_fp64(cuda_dev, variant):
    """eval_probe_kernel at the c4 size: a horizontal factor of 6 (not a multiple of 8: 256 -> 1536), and 30 cluster
    centroids for 27 linear classes (extra clusters, dropped from the confusion counts as in utils.py:222)."""
    B, h, w, H, W = R.EVAL_C4
    if variant.startswith("factor6"):
        W = 6 * w
    code = _cl(_c4_code(cuda_dev, "random", seed=3))
    flip = _cl(_c4_code(cuda_dev, "random", seed=4)) if variant.endswith("flip") else None
    lin, clu = _eval_modules(cuda_dev, 27, 30 if variant.startswith("nclu30") else 27, seed=5)
    _eval_case(cuda_dev, f"generic_{variant}", code, lin, clu, H, W, flip=flip)


@pytest.mark.parametrize("view", ["batch_step", "row_crop"])
def test_eval_frame_strided_views_fp64(cuda_dev, view):
    """Channels-last code views whose batch stride is not h*w*ld, without flip-TTA: image b > 0 must be read from its
    own pixels."""
    B, h, w, H, W = R.EVAL_C4
    store = torch.randn(2 * B, h + 1, w, 72, device=cuda_dev)
    full = store[..., :R.DIM].permute(0, 3, 1, 2)
    code = full[::2, :, :h] if view == "batch_step" else full[:B, :, 1:]
    assert code.stride(0) != h * w * 72
    lin, clu = _eval_modules(cuda_dev, 27, 27, seed=6)
    _eval_case(cuda_dev, f"view_{view}", code, lin, clu, H, W)


# ================================================================================================
# 4. a fused training step whose labels are all ignored
# ================================================================================================
def test_fused_step_all_labels_ignored(cuda_dev):
    """train_segmentation.py:210-218 with no valid label pixel: the linear loss is NaN (as the reference's), its
    gradients are exactly 0, every parameter stays finite after the Adam update, and every other gradient is the one
    the same step computes with normal labels."""
    dev = cuda_dev
    batch = make_batch(2, 64, dev)
    ign = dict(batch, label=torch.full_like(batch["label"], -1))
    out = {}
    for name, bt in (("normal", batch), ("ignored", ign)):
        model, _ = make_model("vit_small", dev, fused=True)
        torch.manual_seed(123)
        model.training_step(bt, 0)
        torch.cuda.synchronize()
        out[name] = (model, grads_of(model), params_of(model), float(model.logged["loss/linear"]))
    _, g_n, _, lin_n = out["normal"]
    model, g_i, p_i, lin_i = out["ignored"]
    assert model._fused is not None
    assert lin_n == lin_n and lin_i != lin_i  # finite vs NaN
    assert torch.equal(g_i["linear_probe.weight"], torch.zeros_like(g_i["linear_probe.weight"]))
    assert torch.equal(g_i["linear_probe.bias"], torch.zeros_like(g_i["linear_probe.bias"]))
    for k, p in p_i.items():
        assert torch.isfinite(p).all(), k
    worst = 0.0
    for k in g_n:
        if not k.startswith("linear_probe"):
            worst = max(worst, rel(g_i[k], g_n[k]))
            assert rel(g_i[k], g_n[k]) < 1e-5, (k, rel(g_i[k], g_n[k]))
    record("probes_fp64_step_all_ignored", dict(worst_other_grad_rel=worst))


# ================================================================================================
# 5. which kernel each kind of case runs (torch.profiler in a child process)
# ================================================================================================
def _kernel_cases(dev):
    """name -> (launch, kernels that must run, kernels that must not): the same inputs and entry points as above."""
    B, h, _ = R.TRAIN["c1"]
    x, cl = R.cluster_inputs("random", B, R.DIM, h * h, R.NCLS, device=dev)
    x4 = _code_view(x, dev)
    xg, clg = R.cluster_inputs("random", 4, 96, 24 * 24, 64, device=dev)
    xg4 = xg.view(4, 96, 24, 24)

    def lce(b_, h_, w_, H_, W_):
        code, Wt, bb, label = R.linear_inputs(b_, R.DIM, h_, w_, H_, W_, 27, device=dev)
        code4 = _cl(code)
        z = torch.zeros(27, R.DIM, device=dev)
        return lambda: _lce_run(code4, Wt, bb, label, 27, 1.0, z, z[:, 0].clone())

    def ev(variant):
        from stego_b200.eval import fused_probe_log_probs
        Be, he, we, He, We = R.EVAL_C4
        if variant == "factor6":
            We = 6 * we
        if variant == "view":
            code = torch.randn(2 * Be, he + 1, we, 72, device=dev)[..., :R.DIM].permute(0, 3, 1, 2)[::2, :, :he]
        else:
            code = _cl(_c4_code(dev, "random"))
        flip = _cl(_c4_code(dev, "random", seed=1)) if variant == "flip" else None
        lin, clu = _eval_modules(dev, 27, 30 if variant == "nclu30" else 27, seed=2)
        label = torch.zeros(Be, He, We, dtype=torch.long, device=dev)
        lc = torch.zeros(27, 27, dtype=torch.int64, device=dev)
        cc = torch.zeros(clu.clusters.shape[0], 27, dtype=torch.int64, device=dev)
        return lambda: fused_probe_log_probs(code, lin, clu, (He, We), 2.0, want_argmax=True, code_flipped=flip,
                                             label=label, linear_confusion=lc, cluster_confusion=cc)

    lin4 = ("linear_logits_kernel", "linear_ce_kernel", "linear_ce_finish_kernel", "linear_wgrad_kernel")
    vec4, gen = "eval_probe_vec4_kernel", "eval_probe_kernel"
    return {
        "cluster_cl_argmax": (lambda: _cluster_run(x4, cl, None, 1.0),
                              ("cluster_lookup_cl_kernel<false>", "cluster_lookup_cl_kernel<true>", "cluster_norm_bwd_kernel"),
                              ("cluster_lookup_kernel<",)),
        "cluster_cl_softmax": (lambda: _cluster_run(x4, cl, 2.0, 1.0),
                               ("cluster_lookup_cl_kernel<false>", "cluster_lookup_kernel<true>"), ()),
        "cluster_generic_n64": (lambda: _cluster_run(xg4, clg, 3.0, 1.0),
                                ("cluster_lookup_kernel<false>", "cluster_lookup_kernel<true>"), ("cluster_lookup_cl_kernel",)),
        "linear_c1": (lce(B, h, h, 224, 224), lin4, ()),
        "linear_down_x": (lce(2, 8, 40, 64, 12), lin4, ()),
        "eval_vec4": (ev("random"), ("eval_prep_kernel", vec4), (gen,)),
        "eval_vec4_flip": (ev("flip"), ("eval_prep_kernel", vec4), (gen,)),
        "eval_vec4_view": (ev("view"), ("eval_prep_kernel", vec4), (gen,)),
        "eval_generic_factor6": (ev("factor6"), ("eval_prep_kernel", gen), (vec4,)),
        "eval_generic_nclu30": (ev("nclu30"), ("eval_prep_kernel", gen), (vec4,)),
    }


def test_intended_kernels_ran(cuda_dev):
    """Shape alone does not pick a kernel (the vec4 eval kernel also needs aligned buffers, the channels-last cluster
    kernel a unit channel stride and n <= 32): profile one launch of each kind and check the kernel names."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--kernel-names"], cwd=root, capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
    for case, (want, not_want) in got["expect"].items():
        for k in want:
            _ran(got["names"][case], k)
        for k in not_want:
            assert not any(k in n for n in got["names"][case]), (case, k, got["names"][case])


if __name__ == "__main__" and sys.argv[1:] == ["--kernel-names"]:
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    cases = _kernel_cases(torch.device("cuda:0"))
    names, expect = {}, {}
    for case, (fn, want, not_want) in cases.items():
        _, names[case] = _kernels(fn)
        names[case] = sorted(names[case])
        expect[case] = (list(want), list(not_want))
    print(json.dumps(dict(names=names, expect=expect)))
