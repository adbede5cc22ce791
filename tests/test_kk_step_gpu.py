"""dino_feat_type "KK" (src/modules.py:98-101: the last block's keys as the teacher features) on the GPU.

  1. VisionTransformer.key_features is, bit for bit, the K third of the full last block's packed qkv with the cls rows
     dropped (ViT-S/8 and ViT-B/8; 224², 320², 64x96; eager and graph-replayed; a "feat" graph and a "KK" graph of the
     same shape side by side; list-of-batches input);
  2. DinoFeaturizer.backbone_tokens with "KK" has the bits of forward(img)[0], and the head on those tokens the bits of
     forward(img)[1]: training and validation feed the head the same tensor;
  3. the six-step procedure of test_step_parity_gpu.py (eager, capture, replays; fused step vs autograd twin vs oracle)
     and 4. its full-size c1-c3 comparison, run unchanged on "KK" models (the oracle steps on the keys);
  5. the reference's own "KK" training step (tests/golden/kk_step.pt) through the fused CUDA step, with the reference's
     draws injected;
  6. knn_descriptors for "KK" (LN1 + pooling, then stego_linear_rows_f32) vs fp64 and vs the reference's get_feats;
  7. stego_linear_rows_f32 vs fp64, and its argument checks.
"""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

from _parity_util import ROOT, record, rel

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.join(ROOT, "oracle"))


def _featurizer(arch, dev, feat_type="KK", **over):
    import stego_oracle as O
    from stego_b200.config import make_cfg
    from stego_b200.modules import DinoFeaturizer
    torch.manual_seed(0)
    net = DinoFeaturizer(70, make_cfg(model_type=arch, dino_feat_type=feat_type, random_backbone_init=True, **over))
    sd = O.perturb_vit_state(O.vit_random_state(arch, 8, seed=3))
    net.model.load_state_dict(sd)
    return net.to(dev), sd


def _full_block_keys(vit, img):
    """K third of the full last block's packed qkv, cls rows dropped: [B, hw, E] bf16."""
    B, E = img.shape[0], vit.embed_dim
    _, qkv = vit.forward_tokens(img, want_qkv=True)
    return qkv.view(B, -1, 3, E)[:, 1:, 1]


# ---------------------------------------------------------------------------------------------------------------------
# 1. key_features bits
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("arch", ["vit_small", "vit_base"])
def test_key_features_bit_identical_to_full_block(cuda_dev, arch):
    net, _ = _featurizer(arch, cuda_dev)
    vit = net.model.eval()
    g = torch.Generator().manual_seed(50)
    for (H, W) in [(224, 224), (320, 320), (64, 96)]:
        B = 2
        for rep in range(2):  # a second graph replay with new data
            img = torch.randn(B, 3, H, W, generator=g).to(cuda_dev)
            img_pos = torch.randn(B, 3, H, W, generator=g).to(cuda_dev)
            both = torch.cat([img, img_pos], 0)
            with torch.no_grad():
                want = _full_block_keys(vit, both)
                eager = vit.key_features(both)
                assert eager.shape == (2 * B, (H // 8) * (W // 8), vit.embed_dim)
                assert torch.equal(eager, want), (arch, H, W, "eager")
                graphed = vit.key_features([img, img_pos], use_graph=True).clone()
                assert torch.equal(graphed, want), (arch, H, W, "graph", rep)
                # a "feat" graph of the same shape lives beside the "KK" one and replays its own sequence
                feat_g = vit.patch_features([img, img_pos], use_graph=True).clone()
                assert torch.equal(feat_g, vit.patch_features(both)), (arch, H, W, "feat graph")
                assert torch.equal(vit.key_features([img, img_pos], use_graph=True), want), (arch, H, W, "graph again")
    kinds = sorted(k[0] for k in vit._cache["graphs"])
    assert kinds == ["KK"] * 3 + ["feat"] * 3, kinds


# ---------------------------------------------------------------------------------------------------------------------
# 2. training and validation feed the head the same tensor
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("arch", ["vit_small", "vit_base"])
def test_backbone_tokens_match_forward(cuda_dev, arch):
    net, _ = _featurizer(arch, cuda_dev)
    net.eval()
    B, H, W = 2, 64, 96
    fh, fw = H // 8, W // 8
    img = torch.randn(B, 3, H, W, generator=torch.Generator().manual_seed(51)).to(cuda_dev)
    with torch.no_grad():
        feat, code = net(img)
        tok = net.backbone_tokens(img)
        assert torch.equal(tok.float().view(B, fh, fw, -1).permute(0, 3, 1, 2), feat)
        assert torch.equal(net.backbone_tokens(img, use_graph=True), tok)
        assert torch.equal(net.head_code(tok, None, None, fh, fw), code)
        # and they are the keys, not the final-norm tokens
        assert not torch.equal(tok, net.model.patch_features(img))


# ---------------------------------------------------------------------------------------------------------------------
# 3 / 4. the parity procedures of test_step_parity_gpu.py on "KK" models
# ---------------------------------------------------------------------------------------------------------------------
def _kk_parity(monkeypatch):
    """test_step_parity_gpu's module with every model it builds set to dino_feat_type "KK" (and, for the image-to-loss
    half of the full-size test, the oracle's fp32 ViT returning the last block's keys)."""
    import kk_oracle as KK
    import _parity_util as PU
    import test_step_parity_gpu as SP
    built = []

    def make_model(arch, dev, fused=True, **over):
        model, sd = PU.make_model(arch, dev, fused=fused, dino_feat_type="KK", **over)
        built.append(model)
        return model, sd

    def oracle_keys(sd, imgs, arch, odev, chunk=8):
        sdd = {k: v.to(odev) for k, v in sd.items()}
        with torch.no_grad():
            return torch.cat([KK.vit_image_keys(sdd, imgs[i:i + chunk].to(odev).float(), arch, 8)
                              for i in range(0, imgs.shape[0], chunk)], 0)

    monkeypatch.setattr(SP, "make_model", make_model)
    monkeypatch.setattr(SP, "oracle_vit_feats", oracle_keys)
    monkeypatch.setattr(SP, "record", lambda name, payload: record("kk_" + name, payload))
    return SP, built


# Oracle-gradient bar of the hidden-layer weight (cluster2.0, E x E behind the ReLU) on keys.  Its weight gradient is
# computed from the bf16-rounded hidden-layer gradient (dgrad operand), which the oracle does not round; on the final-norm
# tokens that puts it ~2e-4 from the oracle, on the keys (not normalised per token) the same rounding measured 1.01e-3
# and 1.07e-3 at step 4 of this procedure on an H100 (every other gradient stays under 1e-3, the fused-vs-autograd and
# parameter bars are unchanged).
HIDDEN_W_BAR = 2e-3


@pytest.mark.parametrize("reset_at", [None, 2], ids=["plain", "reset_probe_steps=2"])
def test_multistep_graph_replay_vs_autograd_vs_oracle(cuda_dev, reset_at):
    """test_step_parity_gpu.py's six steps (eager, capture, 4 replays) on "KK" models: the fused step is taken, and it
    is compared with the autograd twin and with the oracle stepping on the CUDA backbone's keys after every step."""
    from _parity_util import NAMES, OracleStepper, feats_from_tokens, grads_of, make_batch, make_model, params_of, \
        peek_draws
    from test_step_parity_gpu import _check_losses
    arch, res, B, nsteps = "vit_small", 64, 4, 6
    fused, _ = make_model(arch, cuda_dev, fused=True, reset_probe_steps=reset_at, dino_feat_type="KK")
    twin, _ = make_model(arch, cuda_dev, fused=False, reset_probe_steps=reset_at, dino_feat_type="KK")
    for k, v in params_of(fused).items():
        assert torch.equal(v, params_of(twin)[k])
    batches = [make_batch(B, res, cuda_dev, seed=1), make_batch(B, res, cuda_dev, seed=2)]
    orc = OracleStepper(params_of(fused), "cpu")
    h = res // 8
    torch.manual_seed(777)
    worst = dict(grad=0.0, param=0.0, twin_param=0.0)
    for s in range(nsteps):
        batch = batches[s % 2]
        assert fused._fused is None or fused._fused.supported(batch)
        draws = peek_draws(fused, B, cuda_dev)
        gpu_state, cpu_state = torch.cuda.get_rng_state(cuda_dev), torch.get_rng_state()
        p_before = params_of(fused)
        loss = fused.training_step(batch, s)
        g_f, p_f = grads_of(fused), params_of(fused)
        after_state = torch.cuda.get_rng_state(cuda_dev)
        torch.cuda.set_rng_state(gpu_state, cuda_dev)
        torch.set_rng_state(cpu_state)
        loss_t = twin.training_step(batch, s)
        g_t, p_t = grads_of(twin), params_of(twin)
        assert torch.equal(torch.cuda.get_rng_state(cuda_dev), after_state), f"step {s}: RNG consumption differs"
        assert fused._fused.step_idx == s + 1 and twin._fused is None
        if s >= 2:
            assert fused._fused.ws.graph is not None  # replay regime
        assert abs(float(loss) - float(loss_t)) < 2e-5 * abs(float(loss_t)), (s, float(loss), float(loss_t))
        for k in NAMES:
            worst["twin_grad"] = max(worst.get("twin_grad", 0.0), rel(g_f[k], g_t[k]))
            assert rel(g_f[k], g_t[k]) < 3e-3, (s, k, rel(g_f[k], g_t[k]))
            worst["twin_param"] = max(worst["twin_param"], rel(p_f[k], p_t[k]))
            assert rel(p_f[k], p_t[k]) < 2e-4, (s, k, rel(p_f[k], p_t[k]))
        with torch.no_grad():
            tok = fused.net.backbone_tokens(torch.cat([batch["img"], batch["img_pos"]], 0)).float().cpu()
        out = orc.losses(feats_from_tokens(tok, 2 * B, h, h), B, batch["label"].cpu(), draws)
        _check_losses(fused, loss, out)
        g_o = orc.grads()
        for k in NAMES:
            worst["grad"] = max(worst["grad"], rel(g_f[k], g_o[k]))
            assert rel(g_f[k], g_o[k]) < (HIDDEN_W_BAR if k == "net.cluster2.0.weight" else 1e-3), (s, k, rel(g_f[k], g_o[k]))
        orc.adam(g_f)
        resetting = reset_at is not None and s == reset_at
        if resetting:
            for k in ("linear_probe.weight", "linear_probe.bias", "cluster_probe.clusters"):
                assert torch.equal(p_f[k], p_t[k]), k
                assert not torch.allclose(p_f[k], p_before[k]), k
                orc.adopt(k, p_f[k])
        for k in NAMES:
            if resetting and not k.startswith("net."):
                continue
            d_f = p_f[k].cpu() - p_before[k].cpu()
            d_o = orc.p[k].detach() - p_before[k].cpu()
            worst["param"] = max(worst["param"], rel(d_f, d_o))
            assert rel(d_f, d_o) < 1e-4, (s, k, rel(d_f, d_o))
            assert rel(p_f[k], orc.p[k]) < 1e-5, (s, k)
    if reset_at is not None:
        assert fused.optimizers()[1].steps == nsteps - reset_at - 1 and fused.optimizers()[0].steps == nsteps
    assert fused.net.feat_type == twin.net.feat_type == "KK"
    # the keys graph served the fused steps; no "feat" graph was ever captured
    assert {k[0] for k in fused.net.model._cache["graphs"]} == {"KK"}
    record(f"kk_multistep_{'reset' if reset_at is not None else 'plain'}", dict(steps=nsteps, worst=worst))


@pytest.mark.parametrize("cfg_name", ["c1", "c2", "c3"])
def test_fullsize_step_vs_gpu_fp32_oracle(cuda_dev, monkeypatch, cfg_name):
    SP, built = _kk_parity(monkeypatch)
    SP.test_fullsize_step_vs_gpu_fp32_oracle(cuda_dev, cfg_name)
    (model,) = built
    assert model.net.feat_type == "KK" and model._fused.ws.graph is not None
    del built[:]
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------------
# 5. the reference's "KK" step through the fused CUDA step
# ---------------------------------------------------------------------------------------------------------------------
def _golden():
    return torch.load(os.path.join(ROOT, "tests", "golden", "kk_step.pt"))


def _reference_draws(B, E, n_neg, fs):
    """The reference step's draws under manual_seed(777) on the CPU generator, in its order (net(img) x3 Dropout2d
    noises, net(img_pos) x3, rand x2, randperm x n_neg), with the randperms raw (the fused step applies super_perm's
    fix-up in the sampling kernel)."""
    import make_golden as MG
    import stego_oracle as O
    torch.manual_seed(777)
    masks = [O.draw_dropout2d_mask(B, E) for _ in range(6)]
    c1 = torch.rand(B, fs, fs, 2) * 2 - 1
    c2 = torch.rand(B, fs, fs, 2) * 2 - 1
    raw = torch.stack([torch.randperm(B) for _ in range(n_neg)])
    m_ref, mp_ref, c1_ref, c2_ref, p_ref = MG.step_draws()
    assert all(torch.equal(a, b) for a, b in zip(masks, m_ref + mp_ref))
    assert torch.equal(c1, c1_ref) and torch.equal(c2, c2_ref)
    assert all(torch.equal(O.super_perm_from_randperm(r), p) for r, p in zip(raw, p_ref))
    return masks, c1, c2, raw


def test_reference_kk_step_through_cuda(cuda_dev, monkeypatch):
    import make_golden as MG
    import make_golden_kk_step as MK
    import stego_oracle as O
    from stego_b200.fused_step import FusedStep
    want = _golden()["training_step"]
    B, E = MG.STEP_B, MG.STEP_E
    model, _ = _make_step_model(cuda_dev)
    masks, c1, c2, raw = _reference_draws(B, E, model.cfg.neg_samples, model.cfg.feature_samples)
    dev_draws = [t.to(cuda_dev) for t in (torch.cat([masks[0], masks[3]]), torch.cat([masks[1], masks[4]]),
                                           torch.cat([masks[2], masks[5]]), c1, c2, raw)]
    prologue = FusedStep._prologue

    def injected(self, ws):
        prologue(self, ws)  # the step's own draws (and the rest of the prologue), then the reference's values on top
        for dst, src in zip((ws.M1, ws.M2, ws.M3, ws.c1, ws.c2, ws.perms), dev_draws):
            dst.copy_(src.view_as(dst))

    monkeypatch.setattr(FusedStep, "_prologue", injected)
    p0 = MG.step_params()
    batch = {k: v.to(cuda_dev) for k, v in MK.step_batch().items() if k in ("img", "img_pos", "label")}
    loss = model.training_step(batch, 0)
    assert model._fused is not None and model._fused.ws.graph is None and model._fused.step_idx == 1
    model.flush()
    named = dict(model.named_parameters())
    logged = {k: float(v) for k, v in model.logged.items()}
    m = dict(loss_rel=abs(float(loss) - want["loss"]) / abs(want["loss"]))
    for k in ("loss/linear", "loss/cluster", "cd/pos_intra", "cd/pos_inter", "cd/neg_inter"):
        m[k] = abs(logged[k] - want["logged"][k]) / abs(want["logged"][k])
    for k in ("loss/pos_intra", "loss/pos_inter", "loss/neg_inter"):
        m[k] = abs(logged[k] - want["logged"][k])
    grad_rel, delta_rel = {}, {}
    for k in MG.STEP_NAMES:
        g = want["grads"][k]
        idx = g["idx"].long()
        mine = named[k].grad.detach().cpu().reshape(-1)
        grad_rel[k] = ((mine[idx] - g["values"]).norm() / g["values"].norm()).item()
        d_got = named[k].detach().cpu().reshape(-1)[idx] - p0[k].reshape(-1)[idx]
        d_want = want["params_after"][k] - p0[k].reshape(-1)[idx]
        delta_rel[k] = ((d_got - d_want).norm() / d_want.norm()).item()
        # the update the kernels made is torch-Adam on the gradients they computed
        p = p0[k].reshape(-1)[idx].clone()
        O.adam_step(p, mine[idx], torch.zeros_like(p), torch.zeros_like(p), 1, 5e-4 if k.startswith("net.") else 5e-3)
        assert rel(named[k].detach().cpu().reshape(-1)[idx], p) < 1e-5, k
    record("kk_reference_step", dict(terms=m, grad_rel=grad_rel, post_adam_delta_rel=delta_rel))
    print("reference KK step through CUDA:", m, grad_rel, delta_rel)
    # the reference computes in fp32 end to end, the CUDA step on bf16 operands (backbone included): the bars of the
    # image -> loss half of test_fullsize_step_vs_gpu_fp32_oracle
    assert m["loss_rel"] < 5e-3, m
    for k in ("loss/linear", "loss/cluster", "cd/pos_intra", "cd/pos_inter", "cd/neg_inter"):
        assert m[k] < 5e-3, (k, m)
    for k in ("loss/pos_intra", "loss/pos_inter", "loss/neg_inter"):
        assert m[k] < 5e-3 * abs(want["logged"][k]) + 1e-3, (k, m)
    for k in MG.STEP_NAMES:
        assert grad_rel[k] < 0.2, (k, grad_rel[k])
        # Adam's first step is lr * g / |g| elementwise: sign-like, so it flips only where a gradient is near zero
        assert delta_rel[k] < 0.5, (k, delta_rel[k])


def _make_step_model(dev):
    import lightning_harness as H
    import make_golden as MG
    import tempfile
    from stego_b200.config import make_cfg
    from stego_b200.segmenter import LitUnsupervisedSegmenter
    with tempfile.TemporaryDirectory() as td:
        sd = H.write_random_dino_checkpoint(os.path.join(td, "dino.pth"), "vit_small")
    torch.manual_seed(0)
    model = LitUnsupervisedSegmenter(27, make_cfg(dino_feat_type="KK", random_backbone_init=True)).to(dev)
    model.net.model.load_state_dict(sd)
    named = dict(model.named_parameters())
    with torch.no_grad():
        for k, v in MG.step_params().items():
            named[k].copy_(v.to(dev))
    model.train()
    model.configure_optimizers()
    return model, sd


# ---------------------------------------------------------------------------------------------------------------------
# 6. kNN descriptors
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("arch,H,W", [("vit_small", 64, 96), ("vit_base", 224, 224)])
def test_knn_descriptors_kk_vs_fp64(cuda_dev, arch, H, W):
    """Mean over patches of the keys, in fp64 from the same residual stream and the same bf16 key weights."""
    from stego_b200.knn import knn_descriptors
    net, _ = _featurizer(arch, cuda_dev)
    net.eval()
    vit = net.model
    E = vit.embed_dim
    img = torch.randn(3, 3, H, W, generator=torch.Generator().manual_seed(52)).to(cuda_dev)
    with torch.no_grad():
        got = knn_descriptors(net, img)
        x, _ = vit.forward_tokens(img, stop_before_last=True)
        bw = vit._prepared()["blocks"][-1]
        xs = x.double().view(3, -1, E)[:, 1:]
        y = F.layer_norm(xs, (E,), bw["n1w"].double(), bw["n1b"].double(), eps=bw["eps1"])
        want = y.mean(1) @ bw["qkv_w"][E:2 * E].double().t() + bw["qkv_b"][E:2 * E].double()
        # and the same quantity through the [B, hw, E] key map the training step uses
        via_map = vit.key_features(img).float().mean(1)
    r, r_map = rel(got, want), rel(via_map, want)
    record(f"kk_knn_fp64_{arch}_{H}x{W}", dict(rel_l2=r, key_map_rel_l2=r_map))
    assert got.shape == (3, E) and got.dtype == torch.float32
    assert r < 1e-4, r
    assert r_map < 2e-3, r_map  # the map rounds every key to bf16


def test_knn_descriptors_kk_vs_reference_get_feats(cuda_dev):
    import make_golden_kk_step as MK
    from stego_b200.knn import knn_descriptors
    want = _golden()["descriptors"]
    model, _ = _make_step_model(cuda_dev)
    net = model.net.eval()
    batch = MK.step_batch()
    with torch.no_grad():
        got = F.normalize(knn_descriptors(net, torch.cat([batch["img"], batch["img_pos"]], 0).to(cuda_dev)), dim=1)
    r = rel(got, want)
    record("kk_knn_vs_reference_get_feats", dict(rel_l2=r))
    # the reference runs its ViT in fp32, this package on bf16 GEMM operands: the keys themselves sit within the 1e-2 of
    # test_vit_backbone_fp64_gpu.py::test_featurizer_kk_nonsquare (measured 2.9e-3 here on an H100); the descriptor
    # arithmetic after the backbone is checked against fp64 at 1e-4 above
    assert r < 1e-2, r


def test_knn_descriptors_kk_dropout_and_precompute(cuda_dev):
    from stego_b200.knn import knn_descriptors, precompute_knns
    net, _ = _featurizer("vit_small", cuda_dev)
    img = torch.randn(5, 3, 64, 96, generator=torch.Generator().manual_seed(53)).to(cuda_dev)
    net.train()
    torch.manual_seed(11)
    with torch.no_grad():
        want_t = net(img)[0].mean([2, 3])
    st = torch.cuda.get_rng_state(cuda_dev)
    torch.manual_seed(11)
    with torch.no_grad():
        got_t = knn_descriptors(net, img)
    assert torch.equal(torch.cuda.get_rng_state(cuda_dev), st)  # the draws of net(img), no more, no fewer
    assert rel(got_t, want_t) < 2e-3
    assert (got_t == 0).float().mean().item() > 0.05  # ~10 % of the channels dropped
    net.eval()
    batches = [dict(img=torch.randn(4, 3, 64, 64)) for _ in range(3)]
    idx = precompute_knns(net, batches, k=5)
    assert idx.shape == (12, 5) and torch.equal(idx[:, 0].cpu(), torch.arange(12))


# ---------------------------------------------------------------------------------------------------------------------
# 7. stego_linear_rows_f32
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,N,K,ldw", [(3, 384, 384, 1152), (5, 768, 768, 768), (1, 7, 8, 16), (40, 130, 1000, 1000)])
def test_linear_rows_vs_fp64(cuda_dev, B, N, K, ldw):
    from stego_b200 import ops
    g = torch.Generator().manual_seed(B * N + K)
    x = torch.randn(B, K, generator=g).to(cuda_dev)
    w_all = torch.randn(N, ldw, generator=g).to(torch.bfloat16).to(cuda_dev)
    w = w_all[:, :K]
    bias = torch.randn(N, generator=g).to(cuda_dev)
    got = ops.linear_rows_f32(x, w, bias)
    want = x.double() @ w.double().t() + bias.double()
    assert rel(got, want) < 1e-6
    assert rel(ops.linear_rows_f32(x, w), x.double() @ w.double().t()) < 1e-6


def test_linear_rows_rejects_bad_arguments(cuda_dev):
    from stego_b200 import _lib, ops
    x = torch.zeros(2, 64, device=cuda_dev)
    w = torch.zeros(32, 64, dtype=torch.bfloat16, device=cuda_dev)
    lib = _lib.load()
    assert lib.stego_linear_rows_f32(_lib.ptr(x), _lib.ptr(w), 60, 0, _lib.ptr(x), 2, 32, 64, _lib.stream()) == -1
    assert "ldw" in _lib.last_error()
    assert lib.stego_linear_rows_f32(_lib.ptr(x) + 4, _lib.ptr(w), 64, 0, _lib.ptr(x), 2, 32, 60, _lib.stream()) == -1
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.linear_rows_f32(x.cpu(), w)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.linear_rows_f32(x, w.cpu())
