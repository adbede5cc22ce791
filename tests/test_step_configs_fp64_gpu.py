"""The hand-scheduled training step (fused_step.FusedStep) in the configurations it accepts beyond the shipped one:
code widths 1..96, the linear head, dropout off, 3..32 classes with up to 64 cluster rows, patch 16, non-square frames,
labels at another resolution, batches of 1 and 3, 1 and 14 negatives, and the loss's clamp / centring switches (the
table in tests/_step_fp64.py).  Per row:

  1. fused path   FusedStep.supported(batch), and _fused.step_idx advances on each step.
  2. twin         the first step of an autograd twin (cfg.fused_step=False) from the same generator states leaves both
                  generators where the fused step left them; the positive correspondence terms, their cd means and the
                  cluster loss are bit-equal (both paths launch the same kernels on the same inputs, and those
                  reductions run in a fixed order); the linear loss within 1e-6 (fp64 atomics in either order); every
                  gradient within 3e-3 relative L2 (test_step_parity_gpu.py's bar: atomics in another order, the twin's
                  own kink sides), except d(clusters) at D = 1, which is exactly 0 (a one-channel centroid normalises
                  to +-1) and so is held to its absolute fp64 bar in check 3 only.
  3. fp64         three steps (eager, capture, replay); the replayed step's own tensors against tests/_step_fp64.compose
                  on the same backbone tokens, noises ws.M1 / M2 / M3, coordinates ws.c1 / c2, permutations ws.perms and
                  the parameters snapshotted before the step, stage-wise (each stage from what the kernels before it
                  computed), with the bars the stage tests derive:
                    head forward   test_head_fp64_gpu._check_forward: x1 / x2 bit-exact, hid within gamma_{E+2} pre_abs
                                   and one bf16 rounding, code within gamma_{E+3} code_abs, against the exact head within
                                   6 * 2^-8 prop_abs;
                    operand tiles  |hi + lo - n| <= E_n + 2^-16 (|n| + E_n) (test_corr_fp64_gpu.py), rows >= S and code
                                   channels >= D exactly zero;
                    call stats     E_loss and E_cd_mean of CorrRef;
                    d(code)        CorrRef's backward bar on ws.dall, whose columns D..P stay exactly zero;
                    logged terms   neg_inter: sum of the negatives' E_loss / n_neg + gamma_{ncalls} mean |loss_k|
                                   (stego_step_losses, test_head_fp64_gpu.py section 7); total: sum_k w_k E_loss_k +
                                   E_lin + E_clu + gamma_{ncalls+3} (sum |w_k loss_k| + |lin| + |clu|);
                    linear probe   test_probes_fp64_gpu._lce_bars (loss, dW, db) + u |dW| for the final atomic;
                    cluster probe  test_probes_fp64_gpu._cluster_check's argmax bars: E_ip = (2C + 16) u S, loss within
                                   mean max_k E_ip + 32 u mean |max ip|, plus 2 max_k E_ip on the pixels whose fp64 top-2
                                   margin is under 2 max_k E_ip (near ties); dnc within |gs| (L + C/2 + 6) u sum_p |x_hat|,
                                   L the kernel's atomic chain, plus |gs x_hat| into every candidate row of a near tie;
                                   dclusters through the normalise backward;
                    head backward  from the step's d(code): test_fused_step_head_fp64's bars (colsum gamma_{40+blocks},
                                   split-K wgrad gamma_{64 kbps + splits}, dh gamma_130), dyb and dhb bit-exact.
                    rec / crf      with the reconstruction and CRF terms, their stages and their share of the img
                                   rows' d(code) (_rec_crf_stages, _cross_bar; tests/test_step_rec_crf_fp64_gpu.py).
  4. padding      ws.ctiles (torch.empty) is NaN-filled when the workspace is made: after the first step nothing logged
                  or in the flat gradient buffer is NaN and channels D..128 of every code tile are zero; ws.code is
                  allocated zero-filled and its columns D..P are still exactly zero after the replayed step.
  5. update       the replayed step's Adam update of every group against _head_fp64.adam from the step's gradients
                  and the moments before it (test_head_fp64_gpu._adam_ratios).

Largest error / bar ratios go to $STEGO_PARITY_DIR when it is set.
"""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _corr_fp64 as RC  # noqa: E402
import _head_fp64 as RH  # noqa: E402
import _loss_terms_fp64 as RL  # noqa: E402
import _probes_fp64 as RP  # noqa: E402
import _rec_crf_fp64 as RRC  # noqa: E402
import _step_fp64 as S  # noqa: E402
from _parity_util import rel  # noqa: E402
from stego_b200 import hist as hist_mod  # noqa: E402
from test_loss_terms_fp64_gpu import cos_bars, crf_bars  # noqa: E402
from test_rec_crf_step_gpu import crf_dcode_bar, crf_loss_bars, dcode_from_raw, rec_bars, scatter_box, scatter_taps  # noqa: E402,E501
from test_head_fp64_gpu import Ratios, _adam_ratios, _check_forward, _colsum_bar, _same_bits, _wgrad_bar  # noqa: E402
from test_probes_fp64_gpu import _chain, _lce_bars  # noqa: E402

pytestmark = pytest.mark.gpu
U, G = RH.U, RH.gamma
NAN = float("nan")


def _snapshot(model, which):
    model.flush()
    sd = dict(model.named_parameters())
    return {k: (sd[k].grad if which == "grad" else sd[k]).detach().clone() for k in S.names_of(model)}


def _cluster_bars(r, loss, dcl, x, cl, dev):
    """the step's cluster loss and d(clusters) (argmax mode, upstream gradient 1) against cluster_ref"""
    B, C, P = x.shape
    n = cl.shape[0]
    ref = RP.cluster_ref(x, cl, None, 1.0)
    ip, Sabs = ref["ip"], ref["S"]
    E_ip = (2 * C + 16) * U * Sabs
    Emax = E_ip.amax(1)
    top = ip.amax(1)
    near = (ip.topk(2, 1).values[:, 0] - ip.topk(2, 1).values[:, 1]) <= 2 * Emax
    r["cluster_near_ties"] = int(near.sum())  # recorded, not a ratio
    loss_bar = (Emax.mean() + 32 * U * top.abs().mean() + (2 * Emax * near.double()).mean()).item()
    r.add("loss_cluster", loss, torch.tensor(ref["loss"].item()), torch.tensor(loss_bar))
    xh, gs = ref["xh"], abs(ref["gs"])
    L = _chain(B * P, dev, x.stride(1) == 1 and n <= 32)
    cand = ((ip >= top[:, None] - 2 * Emax[:, None]) & near[:, None]).double()
    D = gs * ((L + C / 2 + 6) * U * torch.einsum("bkp,bcp->kc", ref["dip"].abs(), xh.abs()) +
              torch.einsum("bkp,bcp->kc", cand, xh.abs()))
    cd, dnc, ch = cl.double(), ref["dnc"], ref["ch"]
    nrm = cd.norm(dim=1, keepdim=True)
    full = (D + ch.abs() * (ch.abs() * D).sum(1, keepdim=True)) / nrm.clamp_min(1e-12) + \
        (C + 8) * U * (dnc.abs() + ch.abs() * (ch * dnc).sum(1, keepdim=True).abs()) / nrm.clamp_min(1e-12)
    r.add("dclusters", dcl, ref["dcl"], torch.where(nrm > 1e-12, full, (D + U * dnc.abs()) / 1e-12) + 1e-300)


def _rec_crf_stages(r, model, batch, before, grads, tok, M3):
    """The reconstruction and CRF terms of the replayed step, stage-wise on its own inputs (see
    tests/test_step_rec_crf_fp64_gpu.py).  Returns the terms' fp64 d(code) of the img rows [B hw, D], its bar, the
    (roundings, sum of |contributions|) each term adds to those rows' fp32 accumulators, and per term (weight, fp64
    loss, its bar, the step's loss)."""
    from stego_b200 import modules
    ws, cfg = model._fused.ws, model.cfg
    B, E, D, P, fh, fw, hw, M, nonlinear = ws.dims
    dev = ws.code.device
    N = B * hw
    rm = lambda t: t.permute(0, 2, 3, 1).reshape(N, -1)
    want = torch.zeros(N, D, dtype=torch.float64, device=dev)
    bar = torch.zeros_like(want)
    acc, losses = [], {}
    if ws.rec:  # -cosine(decoder(code), feats * m3) on the img rows, with the decoder the step ran with
        W, b = before["decoder.weight"], before["decoder.bias"]
        code = ws.code[:N]
        m3 = M3[:B].repeat_interleave(hw, 0) if M3 is not None else None
        # d loss / d cos = -w / (B hw): fl(-w) times an fp32 reciprocal on the device, three roundings
        dcos = ws.rec_dcos.item()
        assert abs(dcos + float(cfg.rec_weight) / N) <= G(3) * float(cfg.rec_weight) / N, "d loss / d cos of rec"
        ref = RRC.rec_term(code[:, :D], tok[:N], m3, W.view(E, D), b, dcos)
        bars = rec_bars(ref, code, W, N, D, E, dcos)
        for k in ("cos", "nr", "nf"):
            r.add("rec_" + k, getattr(ws, "rec_" + k), ref[k], bars[k])
        loss = float(ws.rec_loss[0])
        assert loss == float(torch.tensor(-ws.rec_cos.double().mean().item(), dtype=torch.float32))
        assert float(model.logged["loss/rec"]) == loss
        e = bars["cos"].mean().item() + U * abs(loss)
        r.add("loss_rec", torch.tensor(loss), torch.tensor(ref["loss"].item()), torch.tensor(e))
        r.add("dW_decoder", grads["decoder.weight"].view(E, D), ref["dW"], bars["dW"])
        r.add("db_decoder", grads["decoder.bias"], ref["db"], bars["db"])
        want += ref["dcode"]
        bar += bars["dcode"]
        # one fp32 add of each 64-channel chunk's partial onto the row's accumulator
        acc.append((-(-E // 64), ref["dr"].abs() @ W.double().view(E, D).abs() + bars["dcode"]))
        losses["rec"] = (float(cfg.rec_weight), ref["loss"].item(), e, loss)
    if ws.crf:  # crf_loss_fn(resize(img, 56), normalize(resize(code, 56))) at this step's samples
        coords = ws.crf_coords
        n = coords.shape[1]
        ys, xs = coords[0], coords[1]
        img = batch["img"]
        code = ws.code.view(ws.n_img * B, fh, fw, P)[:B, ..., :D].permute(0, 3, 1, 2)  # the step's strides
        rs = lambda t: F.interpolate(t, modules.CRF_SIDE, mode="bilinear", align_corners=False)
        w = float(cfg.crf_weight)
        # d loss / d out = w / (B n^2) of the mean: fl(w) times an fp32 reciprocal on the device, three roundings
        g = ws.crf_g
        assert abs(g.item() - w / (B * n * n)) <= G(3) * w / (B * n * n), "d loss / d out of the CRF term"
        run = dict(gsel=ws.crf_gsel[:, :n, :3], raw=ws.crf_raw[:, :, :n], sel=ws.crf_sel[:, :, :n],
                   nrm=ws.crf_nrm[:, :n], g=g)
        # the guidance ran outside the graph, on the coordinates the replayed prologue drew
        assert torch.equal(run["gsel"], rs(img)[:, :, ys, xs].permute(0, 2, 1)), "crf_gsel differs from F.interpolate"
        assert torch.equal(run["raw"], rs(code)[:, :, ys, xs]), "crf_raw differs from F.interpolate"
        assert torch.equal(ws.crf_pos[:n].long(), coords.t())
        p32 = RL.fp32_params(modules.crf_params(model.crf_loss_fn))
        raw64 = run["raw"].double()
        nv = raw64.norm(dim=1)
        sel64 = raw64 / nv.clamp_min(RL.EPS32)[:, None]
        eS = G(-(-D // 32) + 5)
        eN = eS / 2 + eS ** 2 + G(2)
        r.add("crf_sel", run["sel"], sel64, sel64.abs() * (eN + U) + 2.0 ** -149)
        r.add("crf_nrm", run["nrm"], nv, nv * eS)
        cbar, loss64, e2e, _, _ = crf_loss_bars(run, coords, p32, D, code, fh, fw)
        loss = float(ws.crf_loss[0])
        assert float(model.logged["loss/crf"]) == loss
        r.add("loss_crf", torch.tensor(loss), loss64.cpu(), cbar.cpu())
        full = RRC.crf_term(img, code, coords, p32, w)
        r.add("loss_crf_e2e", torch.tensor(loss), full["loss"].cpu(), (cbar + e2e).cpu())
        dc, ref_raw = dcode_from_raw(raw64, run, coords, p32, code.shape)
        _, ds_raw = crf_bars(ref_raw, D, p32)
        cb = crf_dcode_bar(run, ref_raw, ds_raw, coords, code, n, fh, fw)
        want += rm(dc)
        bar += rm(cb)
        # at most one atomic per sample whose fp32 taps can land on the element (crf_dcode_bar's box)
        cnt = scatter_box(torch.ones_like(ref_raw["dv"]), coords, fh, fw)
        acc.append((rm(cnt), rm(scatter_taps(ref_raw["dv"].abs(), coords, fh, fw) + cb)))
        losses["crf"] = (w, loss64.item(), cbar.item(), loss)
    return want, bar, acc, losses


def _cross_bar(old, new):
    """The cross terms of several stages accumulating into the same fp32 d(code) elements: each stage's bar covers the
    roundings of its own additions against its own sum of |contributions|; each of its k additions onto the shared
    accumulator rounds against the others' sums too, u (A_all - A_own) per addition.  old: the (k, A) of the stages
    whose cross terms are already in the bar (among themselves), new: those added here."""
    A_new = sum(A for _, A in new)
    A_all = A_new + sum(A for _, A in old)
    return sum(k * U * A_new for k, _ in old) + sum(k * U * (A_all - A) for k, A in new)


def _fp64_replayed_step(r, model, batch, before, grads, dev, hist=False):
    """check 3 (and the ws.code / d(code) padding of check 4) on the replayed step's workspace; with the modes (see
    tests/test_step_modes_fp64_gpu.py) also the label teacher tiles, the aug-alignment term over 3B rows and (hist) the
    cd histograms the replayed histogram graph binned"""
    from stego_b200 import augment, ops
    ws, cfg = model._fused.ws, model.cfg
    B, E, D, P, fh, fw, hw, M, nonlinear = ws.dims
    nI = ws.n_img
    n = model.n_classes
    parts = [batch["img"], batch["img_pos"]]
    aug = None
    if ws.aug:  # the views the step built from the seeds, bit for bit; the backbone graph read img_aug as its input
        img_aug, coord_aug = augment.aug_alignment_views(batch["img"], augment.batch_seeds(batch["seed"]), cfg.res)
        assert _same_bits(ws.coord_aug, coord_aug), "coord_aug"
        static_in = model.net.model.graph_input(model.net.feat_type, (3 * B,) + tuple(batch["img"].shape[1:]), dev)
        assert static_in is not None and _same_bits(static_in[2 * B:], img_aug), "img_aug"
        parts.append(img_aug)
        aug = dict(coord=ws.coord_aug, w=float(cfg.aug_alignment_weight), grid=ws.grid, dsampled=ws.dsampled)
    with torch.no_grad():  # the same backbone graph the step replayed, on the same images
        tok = model.net.backbone_tokens(parts, use_graph=True).reshape(M, E).clone()
    w = {k: before.get(k) for k in S.HEAD}
    assert _same_bits(ws.w1p[:D], w["net.cluster1.0.weight"].reshape(D, E).bfloat16())
    assert (ws.w1p[D:] == 0).all()
    if nonlinear:
        assert _same_bits(ws.wab, w["net.cluster2.0.weight"].reshape(E, E).bfloat16())
        assert _same_bits(ws.wbp[:D], w["net.cluster2.2.weight"].reshape(D, E).bfloat16())
    M1 = ws.M1.view(nI * B, E)
    M2 = ws.M2.view(nI * B, E) if nonlinear else None
    M3 = ws.M3.view(nI * B, E) if ws.M3 is not None else None
    assert (M3 is not None) == bool(cfg.dropout)
    x = dict(f=tok, m1=M1, m2=M2, w1=w["net.cluster1.0.weight"], b1=w["net.cluster1.0.bias"],
             wa=w["net.cluster2.0.weight"], ba=w["net.cluster2.0.bias"], wb=w["net.cluster2.2.weight"],
             bb=w["net.cluster2.2.bias"])
    # head forward stage-wise; also: ws.code's columns D..P are still exactly zero (pad=0)
    _check_forward(r, dict(x1=ws.x1, x2=ws.x2, hid=ws.hid, code=ws.code), x, nI * B, D, nonlinear, True, pad=0.0)

    edges = torch.from_numpy(hist_mod.default_bins().copy()) if hist else None
    ref = S.compose(tok, B, fh, fw, M1, M2, M3, ws.c1, ws.c2, ws.perms, before, ws.label, cfg, n, hid=ws.hid,
                    code=ws.code, label_pos=ws.label_pos, aug=aug, hist_edges=edges)
    corr, stats = ref["corr"], ref["stats"]
    Sn = corr.S
    assert ws.ftiles.shape[-1] == ws.ET and corr.E == ws.ET
    if ws.label_pos is not None:  # the one-hot teacher: channels n + 1 .. ET are exactly zero
        assert torch.equal(ws.ftiles[..., n + 1:], torch.zeros_like(ws.ftiles[..., n + 1:])), "label tile channels"
    # operand tiles (the teacher tiles from the features or labels, the code tiles from the step's code)
    for name, tiles, vals, bars, C in (("ftiles", ws.ftiles, corr.fn, corr.fE, ws.ET), ("ctiles", ws.ctiles, corr.cn,
                                                                                         corr.cE, D)):
        assert torch.equal(tiles[:, :, :, Sn:], torch.zeros_like(tiles[:, :, :, Sn:])), (name, "rows >= S")
        assert torch.equal(tiles[..., C:], torch.zeros_like(tiles[..., C:])), (name, "pad channels")
        hl = tiles.double()[0] + tiles.double()[1]
        for s in range(corr.nslots):
            r.add(name, hl[s, :, :Sn, :C], vals[s], bars[s] + RC.SPLIT * (vals[s].abs() + bars[s]))
    st = ws.stats.double().cpu()
    for k, s in enumerate(stats):
        r.add("call_loss", st[k, 0], torch.tensor(s["loss"]), torch.tensor(s["E_loss"]))
        r.add("call_cd_mean", st[k, 1], torch.tensor(s["cd_mean"]), torch.tensor(s["E_cd_mean"]))
    # d(code): the correspondence loss's into the img and img_pos rows (plus the aug term's scatter into the img rows,
    # and its cosine backward into the img_aug rows); the padding columns stay zero
    dall = ws.dall.view(M, P)
    assert (dall[:, D:] == 0).all(), "d(code) padding columns"
    rows = slice(0, 2 * B * hw)
    bar = ref["dcode_bar"][rows]
    want = ref["dcode"][rows]
    rm = lambda t: t.permute(0, 2, 3, 1).reshape(B * hw, -1)
    old = [(rm(corr.hits[0]), rm(corr.Ao[0]))]  # the correspondence loss's gather into the img rows
    if ws.aug:
        a = ref["aug"]
        code_img = ws.code.view(nI * B, fh, fw, P)[:B, ..., :D].permute(0, 3, 1, 2)
        code_aug = ws.code.view(nI * B, fh, fw, P)[2 * B:, ..., :D].permute(0, 3, 1, 2)
        r.add("aug_grid", ws.grid, a["grid"], torch.tensor(S.aug_grid_bar(ws.coord_aug), device=dev))
        r.add("aug_sampled", ws.sampled, a["sampled"], torch.tensor(S.aug_sampled_bar(code_img, fh), device=dev))
        cref = RL.pixel_cosine(ws.sampled, code_aug, ga=ws.dcos)
        dcos_bar, cbars = cos_bars(cref, D, False, ws.dcos)
        r.add("aug_cos", ws.cosv, cref["cos"], dcos_bar)
        r.add("aug_dsampled", ws.dsampled, cref["da"], cbars["da"])
        r.add("dcode_aug_rows", dall[2 * B * hw:, :D], rm(cref["db"]), rm(cbars["db"]))
        aug_loss = float(ws.aug_loss[0])
        assert aug_loss == float(torch.tensor(-ws.cosv.double().mean().item(), dtype=torch.float32))
        e_aug = dcos_bar.mean().item() + U * abs(aug_loss)
        r.add("loss_aug_alignment", torch.tensor(aug_loss), torch.tensor(-cref["cos"].mean().item()),
              torch.tensor(e_aug))
        assert float(model.logged["loss/aug_alignment"]) == aug_loss
        # the scatter's bar, and the cross terms of sharing the img rows' fp32 accumulators with the correspondence
        # loss's gather (k more additions onto its sum of |terms|, its hits more onto the scatter's)
        k = S.tap_counts(ws.grid, fh)
        sc = S.aug_scatter_bar(ws.grid, a["A"], ws.dsampled, fh) + k * U * corr.Ao[0] + corr.hits[0] * U * a["A"]
        bar = torch.cat([rm(sc) + bar[:B * hw], bar[B * hw:]])
        old.append((rm(k), rm(a["A"])))
    rc_losses = {}
    if ws.rec or ws.crf:  # their d(code) joins the img rows' accumulators, with the cross terms of sharing them
        rc_want, rc_bar, new, rc_losses = _rec_crf_stages(r, model, batch, before, grads, tok, M3)
        img = slice(0, B * hw)
        want = torch.cat([want[img] + rc_want, want[B * hw:]])
        bar = torch.cat([bar[img] + rc_bar + _cross_bar(old, new), bar[B * hw:]])
    r.add("dcode", dall[rows, :D], want, bar)
    # linear probe (upstream gradient 1, accumulated from zero)
    code4 = ws.code.view(nI * B, fh, fw, P)[..., :D].permute(0, 3, 1, 2)[:B]
    LH, LW = ws.label.shape[-2:]
    lin = ref["lin"]
    lbar, dW_bar, db_bar = _lce_bars(code4, lin, n, LH, LW)
    r.add("loss_linear", ws.lin_loss[0].cpu(), lin["loss"].cpu(), torch.tensor(lbar))
    assert int(ws.lin_loss[1].item()) == lin["count"]
    r.add("dW_linear", grads["linear_probe.weight"].reshape(n, D), lin["dW"], dW_bar + U * lin["dW"].abs())
    r.add("db_linear", grads["linear_probe.bias"], lin["db"], db_bar + U * lin["db"].abs())
    # cluster probe
    _cluster_bars(r, ws.clu_loss[0].cpu(), grads["cluster_probe.clusters"], code4.reshape(B, D, hw),
                  before["cluster_probe.clusters"], dev)
    # the logged terms the step assembles (stego_step_losses, then w * aug onto the total)
    logged = {k: float(v) for k, v in model.logged.items()}
    cw, nn = S.call_weights(cfg), len(stats) - 2
    L = ref["losses"]
    neg_bar = sum(s["E_loss"] for s in stats[2:]) / nn + G(len(stats)) * sum(abs(s["loss"]) for s in stats[2:]) / nn
    r.add("loss_neg_inter", torch.tensor(logged["loss/neg_inter"]), torch.tensor(L["neg_inter"]), torch.tensor(neg_bar))
    for key, kk in (("loss/pos_intra", 0), ("loss/pos_inter", 1)):
        assert logged[key] == float(st[kk, 0])
    e_lin, e_clu = lbar, r.bars["loss_cluster"]
    # w * rec and w * crf: each fl(w l) added onto the running total, one more rounding of it per term (the sum
    # below then also counts the terms' and the aug term's sizes), and the fp64 loss off by its bar
    extra = len(rc_losses)
    terms_abs = sum(abs(c * s["loss"]) for c, s in zip(cw, stats)) + abs(L["linear"]) + abs(L["cluster"])
    if extra:
        terms_abs += sum(abs(wt * got) for wt, _, _, got in rc_losses.values())
        terms_abs += abs(float(cfg.aug_alignment_weight) * aug_loss) if ws.aug else 0.0
    tot_bar = sum(c * s["E_loss"] for c, s in zip(cw, stats)) + e_lin + e_clu + G(len(stats) + 5 + extra) * terms_abs
    want_total = L["total"]
    for wt, l64, e, got in rc_losses.values():
        want_total += wt * l64
        tot_bar += abs(wt) * e + U * abs(wt * got)
    if ws.aug:  # stage-wise: the step's own aug loss, weighted in fp32
        wa = float(cfg.aug_alignment_weight)
        want_total += wa * (aug_loss - L["aug_alignment"])
        tot_bar += abs(wa) * e_aug + G(3) * abs(wa * aug_loss)
    r.add("loss_total", torch.tensor(logged["loss/total"]), torch.tensor(want_total), torch.tensor(tot_bar))
    if hist:
        _hist_checks(r, ws.hist, ref["hist"])
    # head backward from the step's own d(code), over all nB rows
    hb = RH.head_backward(dall, ws.x1, ws.x2, ws.hid, ws.wbp, d=D, dh=ws.dh)
    dyb = torch.zeros(M, 128, dtype=torch.bfloat16, device=dev)
    dyb[:, :D] = dall[:, :D].bfloat16()
    assert _same_bits(ws.dyb, dyb), "dyb"
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    wg_d, cs = _wgrad_bar(M, ops.wgrad_splits(M, D, E, sms)), _colsum_bar(M, True)
    g = {k: grads[k].reshape(grads[k].shape[0], -1).squeeze(1) for k in S.HEAD if k in grads}
    r.add("db_pad", ws.db_pad, hb["db"], cs * hb["db_abs"])
    r.add("db1", g["net.cluster1.0.bias"], hb["db"][:D], cs * hb["db_abs"][:D])
    r.add("dw1", g["net.cluster1.0.weight"], hb["dw1"], wg_d * hb["dw1_abs"])
    if nonlinear:
        assert _same_bits(ws.dhb, torch.where(ws.hid.float() > 0, ws.dh, 0.0).bfloat16()), "dhb"
        wg_e = _wgrad_bar(M, ops.wgrad_splits(M, E, E, sms))
        r.add("dbb", g["net.cluster2.2.bias"], hb["db"][:D], cs * hb["db_abs"][:D])
        r.add("dwb", g["net.cluster2.2.weight"], hb["dwb"], wg_d * hb["dwb_abs"])
        r.add("dh", ws.dh, hb["dh"], G(130) * hb["dh_abs"])
        r.add("dba", g["net.cluster2.0.bias"], hb["dba"], cs * hb["dba_abs"])
        r.add("dwa", g["net.cluster2.0.weight"], hb["dwa"], wg_e * hb["dwa_abs"])


def _hist_checks(r, h, want):
    """the counts the histogram graph binned against the fp64 binning: at every bucket edge, the number of elements
    below it lies between those certainly below (cd + E_cd under the edge) and those possibly below (cd - E_cd under
    it), so only elements within their cd bar of an edge may move; the group sizes exactly; min / max within max E_cd,
    sum within sum E_cd, the sum of squares within sum E_cd (2 |cd| + E_cd), each plus fp64 summation slack"""
    counts, stats = h.counts.cpu(), h.stats.cpu()
    r["hist_ambiguous_near_ties"] = sum(g["ambiguous"] for g in want)
    for gi, g in enumerate(want):
        got = counts[gi]
        assert int(got.sum()) == g["num"] == h.num[gi], (gi, int(got.sum()), g["num"])
        cum = got.cumsum(0)
        lo_ok = bool((g["hi"].cpu().cumsum(0) <= cum).all())
        hi_ok = bool((cum <= g["lo"].cpu().cumsum(0)).all())
        assert lo_ok and hi_ok, (gi, "histogram counts outside the fp64 edge brackets")
        if g["ambiguous"] == 0:
            assert torch.equal(got, g["counts"].cpu()), gi
        slack = 1e-12 * g["abs_sum"]
        r.add("hist_min", stats[gi, 0], torch.tensor(g["min"]), torch.tensor(g["E_minmax"]))
        r.add("hist_max", stats[gi, 1], torch.tensor(g["max"]), torch.tensor(g["E_minmax"]))
        r.add("hist_sum", stats[gi, 2], torch.tensor(g["sum"]), torch.tensor(g["E_sum"] + slack))
        r.add("hist_sumsq", stats[gi, 3], torch.tensor(g["sumsq"]), torch.tensor(g["E_sumsq"] + 1e-12 * g["sumsq"]))


class StepRatios(Ratios):
    """Ratios that also keep each scalar bar (the total's bar is built from the parts' bars) and counters"""

    def __init__(self):
        super().__init__()
        self.bars = {}

    def add(self, name, got, ref, bar):
        if bar.numel() == 1:
            self.bars[name] = float(bar)
        return super().add(name, got, ref, bar)

    def check(self, tag):
        counts = {k: self.pop(k) for k in [k for k in self if k.endswith("_near_ties")]}
        super().check(tag)
        from _parity_util import record
        record(tag + "_counts", counts)


class _Recorder:
    def __init__(self):
        self.calls = []

    def add_histogram_raw(self, tag, **kw):
        self.calls.append((tag, kw))


def run_row(row, tag, dev, monkeypatch):
    """checks 1-5 on one row of tests/_step_fp64.py (CONFIGS or MODE_CONFIGS); returns the fused model, its batches and
    the ratios.  hist rows get a logger: step 0 is eager, step 1 captures the histogram graph, step 2 replays it."""
    from types import SimpleNamespace
    from stego_b200 import augment
    from stego_b200.fused_step import FusedStep
    fused = S.make_model(row, dev, fused=True)
    twin = S.make_model(row, dev, fused=False)
    hist = bool(row.get("hist"))
    if hist:
        for m in (fused, twin):
            m.logger = SimpleNamespace(experiment=_Recorder())
    names = S.names_of(fused)
    p0, p0t = _snapshot(fused, "param"), _snapshot(twin, "param")
    for k in names:
        assert torch.equal(p0[k], p0t[k]), k
    batches = [S.make_batch(row, dev, seed=1), S.make_batch(row, dev, seed=2)]
    # 1. the fused path takes every batch of the row
    for b in batches:
        assert FusedStep(fused).supported(b), tag
    # 4. the code tiles come from torch.empty: NaN in them must not survive the step
    alloc = FusedStep._alloc

    def nan_alloc(self, *a, **k):
        ws = alloc(self, *a, **k)
        ws.ctiles.fill_(NAN)
        return ws
    monkeypatch.setattr(FusedStep, "_alloc", nan_alloc)

    torch.manual_seed(777)
    gpu_state, cpu_state = torch.cuda.get_rng_state(dev), torch.get_rng_state()
    fused.training_step(batches[0], 0)
    g_f = _snapshot(fused, "grad")
    torch.cuda.synchronize()
    assert fused._fused.step_idx == 1
    after_gpu, after_cpu = torch.cuda.get_rng_state(dev), torch.get_rng_state()
    got = {k: v.detach().clone() for k, v in fused.logged.items()}
    ws = fused._fused.ws
    D = ws.dims[2]
    coords = (ws.c1.clone(), ws.c2.clone())
    assert all(torch.isfinite(v).all() for v in got.values()), got
    assert torch.isfinite(fused._flat.grad).all() and torch.isfinite(fused._flat.param).all()
    assert (ws.ctiles[..., D:] == 0).all(), "code tile channels D..128"
    if ws.aug:  # before the backbone graph exists the views are built into ws.img_aug
        img_aug, coord_aug = augment.aug_alignment_views(batches[0]["img"], batches[0]["seed"], fused.cfg.res)
        assert _same_bits(ws.img_aug, img_aug) and _same_bits(ws.coord_aug, coord_aug), "aug views"

    # 2. the autograd twin from the same generator states, its coordinates recorded where it draws them
    drawn = []
    lossfn = twin.contrastive_corr_loss_fn
    orig_draw = lossfn.draw_coords
    monkeypatch.setattr(lossfn, "draw_coords", lambda *a: drawn.append(orig_draw(*a)) or drawn[-1])
    torch.cuda.set_rng_state(gpu_state, dev)
    torch.set_rng_state(cpu_state)
    twin.training_step(batches[0], 0)
    g_t = _snapshot(twin, "grad")
    torch.cuda.synchronize()
    assert twin._fused is None
    assert torch.equal(torch.cuda.get_rng_state(dev), after_gpu), "CUDA generator consumption differs"
    assert torch.equal(torch.get_rng_state(), after_cpu), "CPU generator consumption differs"
    assert len(drawn) == 1 and all(_same_bits(a, b) for a, b in zip(coords, drawn[0])), "coordinates differ"
    want = {k: v.detach().clone() for k, v in twin.logged.items()}
    for key in ("loss/pos_intra", "loss/pos_inter", "cd/pos_intra", "cd/pos_inter", "loss/cluster"):
        assert torch.equal(got[key], want[key]), (key, got[key].item(), want[key].item())
    lin_f, lin_t = got["loss/linear"].item(), want["loss/linear"].item()
    assert abs(lin_f - lin_t) <= 1e-6 * abs(lin_t), (lin_f, lin_t)
    twin_rel = {k: rel(g_f[k], g_t[k]) for k in names}
    for k in names:
        if k == "cluster_probe.clusters" and D == 1:
            # a one-channel centroid normalises to +-1 whatever its value: the exact gradient is 0 and both paths hold
            # rounding noise, which the fp64 check below bounds absolutely
            continue
        if k.startswith("net.") and D == 1 and fused.cfg.crf_weight > 0:
            # likewise each CRF sample normalises to +-1: the exact d(code) of the CRF term is 0, which the fused
            # backward gives exactly (sel dsel sel = dsel), while autograd's F.normalize backward leaves a rounding of
            # dsel / |v| (6e-3 relative L2 of the head gradients); the fp64 check below holds the fused step's
            continue
        assert twin_rel[k] < 3e-3, (k, twin_rel)

    # 3. + 5. eager, capture, replay; the replayed step against fp64
    fused.training_step(batches[1], 1)
    assert fused._fused.step_idx == 2
    ws = fused._fused.ws
    graphs = (ws.graph, ws.hist_graph)
    assert (graphs[1] if hist else graphs[0]) is not None and (graphs[0] if hist else graphs[1]) is None
    before = _snapshot(fused, "param")  # flushes: the parameters the replayed step runs with
    flat = fused._flat
    state0 = [t.clone() for t in (flat.param, flat.exp_avg, flat.exp_avg_sq)]
    steps0 = [o.steps for o in flat.optimizers]
    fused.training_step(batches[0], 2)
    grads = _snapshot(fused, "grad")  # flushes
    torch.cuda.synchronize()
    assert fused._fused.step_idx == 3
    assert fused._fused.ws is ws and (ws.graph, ws.hist_graph) == graphs and ws.eager_steps == 1, \
        "the compared step must replay the graph the step before captured"
    r = StepRatios()
    _fp64_replayed_step(r, fused, batches[0], before, grads, dev, hist=hist)
    g_all = flat.grad.clone()
    for grp, opt, s0 in zip(flat.groups, flat.optimizers, steps0):
        sl = slice(grp.start, grp.start + grp.numel)
        assert opt.steps == s0 + 1
        _adam_ratios(r, [t[sl] for t in (state0[0], g_all, state0[1], state0[2])],
                     [t[sl] for t in (flat.param, flat.exp_avg, flat.exp_avg_sq)], opt.steps, grp.lr, flat.grad_scale)
    return dict(fused=fused, batches=batches, ratios=r, twin_rel=twin_rel)


@pytest.mark.parametrize("name", list(S.CONFIGS))
def test_step_config(cuda_dev, name, monkeypatch):
    out = run_row(S.CONFIGS[name], name, cuda_dev, monkeypatch)
    from _parity_util import record
    record(f"step_configs_{name}_twin", out["twin_rel"])
    out["ratios"].check(f"step_configs_fp64_{name}")
