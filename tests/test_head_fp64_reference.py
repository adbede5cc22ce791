"""CPU: pins the float64 references of tests/_head_fp64.py (used by test_head_fp64_gpu.py) to independent
restatements: the head forward to oracle/stego_oracle.py::head_forward, the backward to torch autograd through
Conv2d(1x1) -> ReLU -> Conv2d(1x1), Adam to torch.optim.Adam; and checks that the input builders make the edges they
claim (exact zero pre-activations, bf16 ties, dropped channels)."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _head_fp64 as R  # noqa: E402
import stego_oracle as O  # noqa: E402

B, H, W, E = 2, 5, 7, 64


def _inputs(regime, nonlinear=True, d=R.D):
    return R.head_inputs(regime, B, H * W, E, d=d, nonlinear=nonlinear, seed=3)


def _nchw(f):
    return f.double().reshape(B, H, W, -1).permute(0, 3, 1, 2)


def test_forward_matches_oracle_head_forward():
    for regime in ("uniform", "outliers", "zero_pre", "dropped"):
        x = _inputs(regime)
        hp = {"cluster1.0.weight": x["w1"].double().reshape(R.D, E, 1, 1), "cluster1.0.bias": x["b1"].double(),
              "cluster2.0.weight": x["wa"].double().reshape(E, E, 1, 1), "cluster2.0.bias": x["ba"].double(),
              "cluster2.2.weight": x["wb"].double().reshape(R.D, E, 1, 1), "cluster2.2.bias": x["bb"].double()}
        # the kernel (and the reference) form f * m in fp32 before rounding to bf16; the oracle rounds its own product.
        # So the masks are checked here, and the convs in eval mode on each fp32 product (the oracle in float64)
        f32m = [(x["f"].float().reshape(B, H * W, E) * x[k].reshape(B, 1, E)).reshape(B * H * W, E) for k in ("m1", "m2")]
        ref = R.head_forward(x["f"], x["m1"], x["m2"], B, x["w1"], x["b1"], x["wa"], x["ba"], x["wb"], x["bb"])
        assert torch.equal(ref["x1"], R.bf16(f32m[0].double())) and torch.equal(ref["x2"], R.bf16(f32m[1].double()))
        for xm in f32m:
            _, c = O.head_forward(_nchw(xm), hp, None, round_bf16=True)
            c = c.permute(0, 2, 3, 1).reshape(B * H * W, R.D)
            r = R.head_forward(xm.bfloat16(), None, None, B, x["w1"], x["b1"], x["wa"], x["ba"], x["wb"], x["bb"])
            assert torch.allclose(r["code"], c, rtol=0, atol=1e-12 * float(r["code_abs"].max())), regime


def test_forward_linear_and_eval_and_stagewise():
    x = _inputs("uniform", nonlinear=False)
    r = R.head_forward(x["f"], x["m1"], None, B, x["w1"], x["b1"])
    want = R.bf16(R.masked(x["f"], x["m1"], B, rnd=False)) @ R.bf16(x["w1"].double()).T + x["b1"].double()
    assert torch.allclose(r["code"], want, rtol=1e-14, atol=1e-14) and "hid" not in r
    x = _inputs("uniform")
    ev = R.head_forward(x["f"], None, None, B, x["w1"], x["b1"], x["wa"], x["ba"], x["wb"], x["bb"])
    assert torch.equal(ev["x1"], x["f"].double()) and torch.equal(ev["x2"], x["f"].double())
    # stage-wise: the given hidden activation replaces the computed one
    hid = torch.zeros_like(ev["hid"])
    st = R.head_forward(x["f"], None, None, B, x["w1"], x["b1"], x["wa"], x["ba"], x["wb"], x["bb"], hid=hid)
    assert torch.allclose(st["code"], ev["x1"] @ R.bf16(x["w1"].double()).T + x["b1"].double() + x["bb"].double(),
                          rtol=1e-14, atol=1e-14)


def test_backward_matches_autograd():
    for regime in ("uniform", "zero_pre", "dropped"):
        x = _inputs(regime)
        f = R.masked(x["f"], x["m1"], B, rnd=False)
        c1 = torch.nn.Conv2d(E, R.D, 1).double()
        ca, cb = torch.nn.Conv2d(E, E, 1).double(), torch.nn.Conv2d(E, R.D, 1).double()
        with torch.no_grad():
            for conv, w, b in ((c1, "w1", "b1"), (ca, "wa", "ba"), (cb, "wb", "bb")):
                conv.weight.copy_(x[w].double().reshape(conv.weight.shape))
                conv.bias.copy_(x[b].double())
        inp = _nchw(f)
        code = c1(inp) + cb(torch.relu(ca(inp)))
        dc = R.dcode_inputs("dense", B, H, W, 72, seed=4)
        code.backward(dc[:, :R.D].double().reshape(B, H, W, R.D).permute(0, 3, 1, 2))
        hid = torch.relu(f @ x["wa"].double().T + x["ba"].double())
        r = R.head_backward(dc, f, f, hid, x["wb"], rnd=False)
        tol = lambda t: dict(rtol=0, atol=1e-12 * float(t.abs().max()) + 1e-300)
        assert torch.allclose(r["dw1"], c1.weight.grad.reshape(R.D, E), **tol(r["dw1_abs"]))
        assert torch.allclose(r["db"][:R.D], c1.bias.grad, **tol(r["db_abs"]))
        assert torch.allclose(r["dwb"], cb.weight.grad.reshape(R.D, E), **tol(r["dwb_abs"]))
        assert torch.allclose(r["dwa"], ca.weight.grad.reshape(E, E), **tol(r["dwa_abs"]))
        assert torch.allclose(r["dba"], ca.bias.grad, **tol(r["dba_abs"]))
        assert torch.equal(r["dba"], r["dba_unrounded"])  # rnd=False: no storage point between them
        assert (r["db"][R.D:] == 0).all()  # padding columns of d(code) are zero


def test_backward_rounding_points():
    x = _inputs("uniform")
    f = x["f"].double()
    hid = R.bf16(torch.relu(f @ R.bf16(x["wa"].double()).T + x["ba"].double()))
    dc = R.dcode_inputs("dense", B, H, W, 72, seed=5)
    wb = R.bf16(x["wb"].double())
    r = R.head_backward(dc, f, f, hid, wb)
    assert torch.equal(r["dyb"][:, :R.D], dc[:, :R.D].bfloat16().double()) and (r["dyb"][:, R.D:] == 0).all()
    dh = r["dyb"][:, :R.D] @ wb
    assert torch.allclose(r["dh"], dh, rtol=1e-14, atol=0)
    assert torch.equal(r["dhb"], torch.where(hid > 0, dh, 0.0).bfloat16().double())
    # stage-wise: a given dh is used as is
    r2 = R.head_backward(dc, f, f, hid, wb, dh=torch.ones_like(dh))
    assert torch.equal(r2["dhb"], (hid > 0).double())


def test_input_builders_make_their_edges():
    x = _inputs("zero_pre")
    band = slice(E // 4, E // 4 + 32)
    r = R.head_forward(x["f"], x["m1"], x["m2"], B, x["w1"], x["b1"], x["wa"], x["ba"], x["wb"], x["bb"])
    assert (r["pre"][:, band] == 0).all() and (r["hid"][:, band] == 0).all()
    assert (r["pre"][:, :E // 4] != 0).all()
    x = _inputs("dropped")
    assert (x["m1"][1] == 0).all() and (x["m2"][1] == 0).all()
    assert ((x["m1"][0] == 0).sum() > 0) and set(x["m1"].unique().tolist()) == {0.0, float(torch.tensor(R.DROPPED).float())}
    r = R.head_forward(x["f"], x["m1"], x["m2"], B, x["w1"], x["b1"])
    assert (r["x1"][H * W:] == 0).all()
    x = _inputs("outliers")
    assert (x["f"].float().abs() == 300).sum() == 8 * B * H * W
    dc = R.dcode_inputs("dense", B, H, W, 72, seed=1)
    b = dc.bfloat16().float()
    up = (dc.bfloat16().view(torch.int16) + 1).view(torch.bfloat16).float()
    dn = (dc.bfloat16().view(torch.int16) - 1).view(torch.bfloat16).float()
    ties = ((dc - b).abs() == (up - b).abs() / 2) | ((dc - b).abs() == (dn - b).abs() / 2)
    assert ties[:, :R.D][dc[:, :R.D] != 0].float().mean() > 0.1
    assert (dc[:, R.D:] == 0).all()
    sp = R.dcode_inputs("sparse", B, H, W, 72, seed=1)
    nz = (sp[:, :R.D] != 0).any(1)
    assert 0 < int(nz.sum()) <= B * H * W
    rg = R.dcode_inputs("range", B, H, W, 72, seed=1)[:, :R.D].abs()
    assert float(rg.max() / rg[rg > 0].min()) > 1e8


def test_adam_matches_torch_optim_adam_over_50_steps():
    g = torch.Generator().manual_seed(0)
    p0 = torch.randn(1000, generator=g, dtype=torch.float64)
    tp = p0.clone().requires_grad_(True)
    opt = torch.optim.Adam([tp], lr=5e-4, foreach=False)
    p, m, v = p0.clone(), torch.zeros_like(p0), torch.zeros_like(p0)
    for t in range(1, 51):
        if t == 20:
            for pg in opt.param_groups:
                pg["lr"] = 5e-3
        lr = opt.param_groups[0]["lr"]
        grad = torch.randn(1000, generator=g, dtype=torch.float64) * 10 ** (torch.rand(1000, generator=g) * 8 - 6)
        tp.grad = grad.clone()
        opt.step()
        r = R.adam(p, grad, m, v, t, lr)
        p, m, v = r["p"], r["m"], r["v"]
        st = opt.state[tp]
        # float64 both: only their rounding (and cancellation in m) separates them
        close = lambda a, b: torch.allclose(a, b, rtol=1e-12, atol=1e-12 * float(b.abs().max()))
        assert close(st["exp_avg"], m) and close(st["exp_avg_sq"], v) and close(tp.detach(), p)
        assert close(tp.detach() - p0, p - p0)  # the accumulated updates, not only the parameters
    # grad_scale multiplies the gradient first
    a = R.adam(p, grad, m, v, 3, 1e-3, grad_scale=0.125)
    b = R.adam(p, grad * 0.125, m, v, 3, 1e-3)
    assert torch.equal(a["p"], b["p"]) and torch.equal(a["v"], b["v"])


def test_rank_sum_is_fp32_in_rank_order():
    e = [torch.tensor([1.0, -0.0]), torch.tensor([2.0 ** -24, -0.0]), torch.tensor([2.0 ** -24, 0.0])]
    s = R.rank_sum_fp32(e)
    assert s[0] == 1.0  # (1 + u) rounds to 1 twice: the fp32 order, not the exact sum 1 + 2^-23
    assert s[1] == 0 and not torch.signbit(s[1])  # the sum starts from +0
