"""Shared helpers of the GPU parity tests: the oracle stepping the same trainable parameters as the CUDA path.

The oracle (oracle/stego_oracle.py) is plain torch and device-agnostic: `odev="cuda"` runs the very same functions in
fp32 on the GPU with TF32 disabled (cuBLAS / cuDNN fp32 kernels — "the reference PyTorch path" on the GPU), which makes
the BASELINE.json full-size configurations a seconds-long check; `odev="cpu"` is the CPU oracle.
"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))

NAMES = ["net.cluster1.0.weight", "net.cluster1.0.bias", "net.cluster2.0.weight", "net.cluster2.0.bias",
         "net.cluster2.2.weight", "net.cluster2.2.bias", "linear_probe.weight", "linear_probe.bias",
         "cluster_probe.clusters"]


def fp32_strict():
    """No TF32 anywhere: the GPU oracle must be an fp32 computation."""
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    torch.set_float32_matmul_precision("highest")


def rel(x, y):
    x, y = x.detach().double().cpu(), y.detach().double().cpu()
    return ((x - y).norm() / y.norm().clamp_min(1e-30)).item()


def lr_of(name):
    return 5e-4 if name.startswith("net.") else 5e-3  # train_segmentation.py:379-381


def make_model(arch, dev, fused=True, seed=0, n_classes=27, patch=8, **cfg_over):
    import stego_oracle as O
    from stego_b200.config import make_cfg
    from stego_b200.segmenter import LitUnsupervisedSegmenter
    cfg = make_cfg(model_type=arch, random_backbone_init=True, fused_step=fused, dino_patch_size=patch, **cfg_over)
    torch.manual_seed(seed)
    model = LitUnsupervisedSegmenter(n_classes, cfg).to(dev)
    sd = O.perturb_vit_state(O.vit_random_state(arch, patch, seed=3))
    model.net.model.load_state_dict(sd)
    model.train()
    model.configure_optimizers()
    return model, sd


def make_batch(B, res, dev, seed=1):
    g = torch.Generator().manual_seed(seed)
    img = torch.randn(B, 3, res, res, generator=g)
    img_pos = img + 0.3 * torch.randn(B, 3, res, res, generator=g)
    label = torch.randint(-1, 27, (B, res, res), generator=g)
    return dict(img=img.to(dev), img_pos=img_pos.to(dev), label=label.to(dev))


def params_of(model):
    model.flush()
    sd = dict(model.named_parameters())
    return {k: sd[k].detach().clone() for k in NAMES}


def grads_of(model):
    model.flush()
    sd = dict(model.named_parameters())
    return {k: sd[k].grad.detach().clone() for k in NAMES}


def peek_draws(model, B, dev):
    """The random draws the NEXT training step will make (Dropout2d noises of net(img) and net(img_pos), the two
    coordinate grids, the negative permutations), learnt by consuming the generator and putting its state back."""
    from stego_b200.modules import super_perm
    st = torch.cuda.get_rng_state(dev)
    m = model.net.draw_masks(B, dev)
    mp = model.net.draw_masks(B, dev)
    c1, c2 = model.contrastive_corr_loss_fn.draw_coords(torch.empty(B, 1, device=dev), None, None)
    perms = [super_perm(B, dev) for _ in range(model.cfg.neg_samples)]
    torch.cuda.set_rng_state(st, dev)
    return m, mp, c1, c2, perms


class OracleStepper:
    """The oracle's copy of the trainable state: parameters, Adam moments, per-optimiser step counts."""

    def __init__(self, params0, odev):
        self.odev = odev
        self.p = {k: v.detach().to(odev, torch.float32).clone().requires_grad_(True) for k, v in params0.items()}
        self.m = {k: torch.zeros_like(v) for k, v in self.p.items()}
        self.v = {k: torch.zeros_like(v) for k, v in self.p.items()}
        self.steps = {k: 0 for k in self.p}

    def losses(self, f_all, B, label, draws, round_bf16=True):
        import stego_oracle as O
        m, mp, c1, c2, perms = draws
        od = self.odev
        for t in self.p.values():
            t.grad = None
        hp = {k[len("net."):]: v for k, v in self.p.items() if k.startswith("net.")}
        probes = {k: v for k, v in self.p.items() if not k.startswith("net.")}
        to4 = lambda t: t.to(od).view(B, -1, 1, 1)
        out = O.training_losses(f_all[:B], f_all[B:], hp, probes, label.to(od), [to4(x) for x in m], [to4(x) for x in mp],
                                c1.to(od), c2.to(od), [p.to(od) for p in perms], O.LossCfg(), 27, round_bf16=round_bf16)
        out["total"].backward()
        return out

    def grads(self):
        return {k: v.grad.detach().clone() for k, v in self.p.items()}

    def adam(self, grads=None):
        import stego_oracle as O
        with torch.no_grad():
            for k, p in self.p.items():
                self.steps[k] += 1
                g = (grads[k].to(self.odev) if grads is not None else p.grad)
                O.adam_step(p, g, self.m[k], self.v[k], self.steps[k], lr_of(k))

    def adopt(self, name, value):
        """A re-initialised parameter (reset_probe_steps): take the new value, fresh Adam state."""
        with torch.no_grad():
            self.p[name].copy_(value.to(self.odev))
        self.m[name].zero_()
        self.v[name].zero_()
        self.steps[name] = 0


def feats_from_tokens(tok, B2, h, w):
    """[2B, hw, E] tokens-major -> NCHW view [2B, E, h, w] (what DinoFeaturizer returns, src/modules.py:97)."""
    return tok.view(B2, h, w, -1).permute(0, 3, 1, 2)


def oracle_vit_feats(sd, imgs, arch, odev, chunk=8):
    """fp32 oracle ViT features of `imgs` on `odev`, in chunks (the reference materialises [B,heads,N,N])."""
    import stego_oracle as O
    sdd = {k: v.to(odev) for k, v in sd.items()}
    outs = []
    with torch.no_grad():
        for i in range(0, imgs.shape[0], chunk):
            outs.append(O.vit_image_feat(sdd, imgs[i:i + chunk].to(odev).float(), arch, 8))
    return torch.cat(outs, 0)


def record(name, payload):
    """Keep a machine-readable copy of what a parity test measured, in $STEGO_PARITY_DIR when that is set."""
    d = os.environ.get("STEGO_PARITY_DIR")
    if not d:
        return
    os.makedirs(d, exist_ok=True)
    with open(os.path.join(d, f"parity_{name}.json"), "w") as fh:
        json.dump(payload, fh, indent=1, sort_keys=True)
