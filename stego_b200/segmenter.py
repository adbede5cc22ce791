"""`LitUnsupervisedSegmenter` — the training-step orchestration of the reference
(src/train_segmentation.py:53-383) re-hosted on the fused sm_90a path, without a Lightning dependency.

Same constructor `(n_classes, cfg)`, attribute names (`net`, `linear_probe`, `cluster_probe`,
`train_cluster_probe`, `decoder`, `contrastive_corr_loss_fn`, ...), `forward`, `training_step(batch,
batch_idx)` and `configure_optimizers()`; state-dict keys match the reference checkpoints
(SURVEY.md §5).  What changes is HOW a step runs:

  * img and img_pos go through the frozen ViT as ONE batch of 2B (one kernel sequence instead of two);
  * the head, the correspondence loss, both probes and their backward are the fused kernels of
    modules.py / corr.py (autograd only stitches ~10 custom nodes together);
  * all trainable parameters (and their .grad) are views into ONE flat fp32 buffer, so data-parallel
    training needs exactly one exchange per step (reference: Lightning-DDP bucketed all-reduce,
    train_segmentation.py:476,227): the sum over ranks is read from the peers' HBM over NVLink inside the Adam
    kernel itself (p2p.py / csrc/p2p_update.cu), with one NCCL all-reduce + three Adam launches as the fallback.

Per-rank semantics follow the reference: negatives, `old_mean` and every mean are computed over the LOCAL
shard; only gradients cross ranks (averaged).
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib, corr
from .modules import ClusterLookup, ContrastiveCorrelationLoss, ContrastiveCRFLoss, DinoFeaturizer, \
    FeaturePyramidNet, _ClusterLookupFn, norm, pixel_cosine, sample


# --------------------------------------------------------------------------------------------------
# flat parameter / gradient storage + fused Adam
# --------------------------------------------------------------------------------------------------
class FlatGroup:
    """A contiguous slice of the flat parameter buffer updated with one learning rate."""

    def __init__(self, params: Sequence[nn.Parameter], lr: float, start: int):
        self.params = list(params)
        self.lr = lr
        self.start = start
        self.numel = sum(p.numel() for p in self.params)


class FusedAdam:
    """torch.optim.Adam-compatible update (betas .9/.999, eps 1e-8, no weight decay) on a flat slice,
    one kernel launch (stego_adam_step).  Mirrors the optimizer objects `configure_optimizers` returns
    (train_segmentation.py:373-383): `.zero_grad()`, `.step()`, `.param_groups`."""

    def __init__(self, owner: "FlatParams", group: FlatGroup):
        self.owner, self.group = owner, group
        self.param_groups = [dict(params=group.params, lr=group.lr, betas=(0.9, 0.999), eps=1e-8)]
        self.steps = 0

    def zero_grad(self, set_to_none: bool = False):
        g = self.group
        self.owner.grad[g.start:g.start + g.numel].zero_()

    def reset_state(self):
        """Fresh optimiser state for this group (what constructing a new torch.optim.Adam does)."""
        g = self.group
        self.owner.exp_avg[g.start:g.start + g.numel].zero_()
        self.owner.exp_avg_sq[g.start:g.start + g.numel].zero_()
        self.steps = 0

    def state_dict(self):
        """torch.optim.Adam layout (per-parameter `step`, `exp_avg`, `exp_avg_sq`), so a checkpoint written here resumes
        under torch.optim.Adam and vice versa."""
        g, o = self.group, self.owner
        state, off = {}, g.start
        for i, p in enumerate(g.params):
            n = p.numel()
            if self.steps > 0:
                state[i] = dict(step=torch.tensor(float(self.steps)),
                                exp_avg=o.exp_avg[off:off + n].view(p.shape).clone(),
                                exp_avg_sq=o.exp_avg_sq[off:off + n].view(p.shape).clone())
            off += n
        pg = self.param_groups[0]
        return dict(state=state, param_groups=[dict(lr=pg["lr"], betas=pg["betas"], eps=pg["eps"], weight_decay=0,
                                                    amsgrad=False, params=list(range(len(g.params))))])

    def load_state_dict(self, sd):
        g, o = self.group, self.owner
        pg = sd["param_groups"][0]
        self.param_groups[0].update(lr=pg["lr"], betas=tuple(pg["betas"]), eps=pg["eps"])
        off, steps = g.start, 0
        for i, p in enumerate(g.params):
            n = p.numel()
            st = sd["state"].get(i, sd["state"].get(str(i)))
            if st is None:
                o.exp_avg[off:off + n].zero_()
                o.exp_avg_sq[off:off + n].zero_()
            else:
                o.exp_avg[off:off + n].copy_(st["exp_avg"].reshape(-1))
                o.exp_avg_sq[off:off + n].copy_(st["exp_avg_sq"].reshape(-1))
                steps = max(steps, int(float(st["step"])))
            off += n
        self.steps = steps

    def step(self):
        g, o = self.group, self.owner
        self.steps += 1
        pg = self.param_groups[0]
        sl = slice(g.start, g.start + g.numel)
        rc = _lib.load().stego_adam_step(_lib.ptr(o.param[sl]), _lib.ptr(o.grad[sl]), _lib.ptr(o.exp_avg[sl]),
                                         _lib.ptr(o.exp_avg_sq[sl]), g.numel, float(pg["lr"]), pg["betas"][0],
                                         pg["betas"][1], pg["eps"], self.steps, o.grad_scale, _lib.stream())
        _lib.check(rc, "stego_adam_step")


class FlatParams:
    """Re-homes the given parameters (and their .grad) as views into flat fp32 buffers."""

    def __init__(self, groups: Sequence[Sequence[nn.Parameter]], lrs: Sequence[float]):
        params = [p for g in groups for p in g]
        dev = params[0].device
        total = sum(p.numel() for p in params)
        self.param = torch.empty(total, dtype=torch.float32, device=dev)
        self.grad = torch.zeros(total, dtype=torch.float32, device=dev)
        self.exp_avg = torch.zeros(total, dtype=torch.float32, device=dev)
        self.exp_avg_sq = torch.zeros(total, dtype=torch.float32, device=dev)
        self.grad_scale = 1.0  # 1/world_size after a sum all-reduce
        self.groups: List[FlatGroup] = []
        off = 0
        for g, lr in zip(groups, lrs):
            fg = FlatGroup(g, lr, off)
            for p in g:
                n = p.numel()
                self.param[off:off + n].copy_(p.detach().reshape(-1))
                p.data = self.param[off:off + n].view(p.shape)
                p.grad = self.grad[off:off + n].view(p.shape)
                off += n
            self.groups.append(fg)
        self.optimizers = [FusedAdam(self, g) for g in self.groups]

    def ensure_bound(self):
        """The fused kernels write through raw pointers into the flat buffers: every parameter (and its .grad) must
        still be the view made at construction.  `.grad = None` (zero_grad(set_to_none=True)) is repaired here; a
        parameter whose storage moved (model.to() / .cuda() after configure_optimizers) cannot be, and raises."""
        for g in self.groups:
            off = g.start
            for p in g.params:
                n = p.numel()
                if p.data_ptr() != self.param.data_ptr() + 4 * off:
                    raise RuntimeError("stego_b200: a trainable parameter no longer lives in the flat parameter buffer "
                                       "(model moved after configure_optimizers()?); call configure_optimizers() again")
                if p.grad is None or p.grad.data_ptr() != self.grad.data_ptr() + 4 * off:
                    p.grad = self.grad[off:off + n].view(p.shape)
                off += n

    def rebind(self):
        """Autograd may replace .grad objects; point them back at the flat buffer (values are accumulated
        in place when .grad is already set, so this is only a safety net)."""
        for g in self.groups:
            off = g.start
            for p in g.params:
                n = p.numel()
                view = self.grad[off:off + n].view(p.shape)
                if p.grad is None or p.grad.data_ptr() != view.data_ptr():
                    if p.grad is not None:
                        view.add_(p.grad)
                    p.grad = view
                off += n


def allreduce_gradients(flat: FlatParams) -> None:
    """The ONE collective of the data-parallel step: sum all-reduce of the flat gradient buffer over NCCL
    (NVLink 5 / NVSwitch; <= 2.8 MB, latency-bound); the 1/world scale is folded into the Adam kernel."""
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(flat.grad, op=dist.ReduceOp.SUM)
        flat.grad_scale = 1.0 / dist.get_world_size()
    else:
        flat.grad_scale = 1.0


# --------------------------------------------------------------------------------------------------
# linear probe: 1x1 conv -> bilinear upsample -> masked CE, forward + backward in one fused call
# --------------------------------------------------------------------------------------------------
class _LinearProbeCEFn(torch.autograd.Function):

    @staticmethod
    def forward(ctx, code_nchw, weight, bias, label):
        # code_nchw: detached [B, C, h, w] view whose channel stride is 1 (tokens-major storage)
        B, C, h, w = code_nchw.shape
        n = weight.shape[0]
        dev = code_nchw.device
        if n > 32 or C > 96:
            raise RuntimeError(f"stego_b200 linear probe: n_classes={n} (<=32) / dim={C} (<=96) unsupported")
        x = code_nchw.detach()
        if x.dtype != torch.float32 or x.stride(1) != 1 or x.stride(2) != w * x.stride(3):
            x = x.float().permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
        ld = x.stride(3)
        rows = B * h * w
        H, W = label.shape[-2], label.shape[-1]
        lab = label.reshape(B, H, W)
        if lab.dtype not in (torch.int64, torch.int32, torch.uint8):
            lab = lab.to(torch.long)
        lab = lab.contiguous()
        label_bytes = {torch.int64: 8, torch.int32: 4, torch.uint8: 1}[lab.dtype]
        logits = torch.empty(rows, 32, dtype=torch.float32, device=dev)
        dlogits = torch.zeros(rows, 32, dtype=torch.float32, device=dev)
        partials = torch.empty(16 * torch.cuda.get_device_properties(dev).multi_processor_count * 2,
                               dtype=torch.float32, device=dev)
        loss = torch.empty(2, dtype=torch.float32, device=dev)
        dW = torch.zeros(n, C, dtype=torch.float32, device=dev)
        db = torch.zeros(n, dtype=torch.float32, device=dev)
        wf = weight.detach().float().reshape(n, C).contiguous()
        bf = bias.detach().float().contiguous()
        rc = _lib.load().stego_linear_probe_ce(_lib.ptr(x), ld, C, _lib.ptr(wf), _lib.ptr(bf), n, _lib.ptr(lab), label_bytes, B,
                                               h, w,
                                               H, W, _lib.ptr(logits), _lib.ptr(dlogits), _lib.ptr(partials),
                                               _lib.ptr(loss), 1.0, _lib.ptr(dW), _lib.ptr(db), _lib.stream())
        _lib.check(rc, "stego_linear_probe_ce")
        ctx.save_for_backward(dW, db)
        ctx.wshape = weight.shape
        return loss[0]

    @staticmethod
    def backward(ctx, g):
        dW, db = ctx.saved_tensors
        return None, (dW * g).reshape(ctx.wshape), db * g, None


def linear_probe_ce(code_nchw, weight, bias, label):
    return _LinearProbeCEFn.apply(code_nchw, weight, bias, label)


# --------------------------------------------------------------------------------------------------
# the module
# --------------------------------------------------------------------------------------------------
class LitUnsupervisedSegmenter(nn.Module):
    """train_segmentation.py:53-383 (the parts on the training hot path)."""

    def __init__(self, n_classes, cfg):
        super().__init__()
        self.cfg = cfg
        self.n_classes = n_classes
        dim = cfg.dim if cfg.continuous else n_classes
        if cfg.arch == "dino":
            self.net = DinoFeaturizer(dim, cfg)
        elif cfg.arch == "feature-pyramid":
            raise RuntimeError("stego_b200: arch 'feature-pyramid' needs the caller's cut model; construct "
                               "FeaturePyramidNet directly (API-surface only, not on the fused path)")
        else:
            raise ValueError("Unknown arch {}".format(cfg.arch))
        self.train_cluster_probe = ClusterLookup(dim, n_classes)
        self.cluster_probe = ClusterLookup(dim, n_classes + cfg.extra_clusters)
        self.linear_probe = nn.Conv2d(dim, n_classes, (1, 1))
        self.decoder = nn.Conv2d(dim, self.net.n_feats, (1, 1))
        # train_segmentation.py:80-88: the validation / test metric objects the eval script reads (`test_*_metrics`,
        # eval_segmentation.py:137-141).  Their `stats` histograms are what the fused eval kernel accumulates into.
        from .eval import UnsupervisedMetrics
        self.cluster_metrics = UnsupervisedMetrics("test/cluster/", n_classes, cfg.extra_clusters, True)
        self.linear_metrics = UnsupervisedMetrics("test/linear/", n_classes, 0, False)
        self.test_cluster_metrics = UnsupervisedMetrics("final/cluster/", n_classes, cfg.extra_clusters, True)
        self.test_linear_metrics = UnsupervisedMetrics("final/linear/", n_classes, 0, False)
        self.linear_probe_loss_fn = torch.nn.CrossEntropyLoss()
        self.crf_loss_fn = ContrastiveCRFLoss(cfg.crf_samples, cfg.alpha, cfg.beta, cfg.gamma, cfg.w1, cfg.w2, cfg.shift)
        self.contrastive_corr_loss_fn = ContrastiveCorrelationLoss(cfg)
        self.automatic_optimization = False
        self.val_steps = 0
        self.global_step = 0
        self.logged: Dict[str, torch.Tensor] = {}
        self._flat: Optional[FlatParams] = None
        self._spec = corr.make_spec(cfg)
        self._fused = None
        self.profile_marks = None  # optional list: bench.py --breakdown collects (name, cuda event) pairs here

    # ---- Lightning-shaped surface ----------------------------------------------------------------
    def forward(self, x):
        self.flush()
        return self.net(x)[1]

    def _apply(self, fn, *args, **kwargs):
        """`.to()` / `.cuda()`: the metric histograms are plain tensors (the reference's are torchmetrics states) and follow
        the module to its device."""
        out = super()._apply(fn, *args, **kwargs)
        for name in ("cluster_metrics", "linear_metrics", "test_cluster_metrics", "test_linear_metrics"):
            m = getattr(self, name, None)
            if m is not None:
                m.stats = fn(m.stats)
        return out

    def flush(self):
        """The hand-scheduled step leaves its parameter update (all-reduce + Adam) on a side stream so that the next
        step's frozen backbone overlaps it; this makes the CURRENT stream wait for it.  Call it before reading
        parameters / gradients / optimiser state outside training_step (forward and state_dict do)."""
        if self._fused is not None:
            self._fused.flush()

    def state_dict(self, *args, **kwargs):
        self.check_update_health()
        return super().state_dict(*args, **kwargs)

    def reset_probes(self):
        """train_segmentation.py:232-237: re-initialise both probes and give them fresh Adam state (runs on the
        current stream; the parameters stay views of the flat buffer, so captured graphs remain valid)."""
        print("RESETTING PROBES")
        with torch.no_grad():
            self.linear_probe.reset_parameters()
            self.cluster_probe.reset_parameters()
        _, linear_probe_optim, cluster_probe_optim = self.optimizers()
        linear_probe_optim.reset_state()
        cluster_probe_optim.reset_state()

    def log(self, name, value, **_kwargs):
        self.logged[name] = value.detach() if torch.is_tensor(value) else value

    def configure_optimizers(self):
        """train_segmentation.py:373-383: Adam(net [+decoder], lr=cfg.lr), Adam(linear_probe, 5e-3),
        Adam(cluster_probe, 5e-3) — here three fused-Adam views over one flat buffer."""
        main = [p for p in self.net.parameters() if p.requires_grad]
        if self.cfg.rec_weight > 0:
            main.extend(self.decoder.parameters())
        groups = [main, list(self.linear_probe.parameters()), list(self.cluster_probe.parameters())]
        self.flush()
        self._flat = FlatParams(groups, [self.cfg.lr, 5e-3, 5e-3])
        import torch.distributed as dist
        self._peer = None
        if self._flat.param.is_cuda and dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            # Lightning-DDP broadcasts module state from rank 0 when it wraps the model (train_segmentation.py:476)
            dist.broadcast(self._flat.param, src=0)
            if getattr(self.cfg, "p2p_update", True):
                # the per-step exchange: all-reduce fused into Adam over NVLink peer memory (csrc/p2p_update.cu); NCCL is
                # the fallback when the ranks cannot map each other's memory (not one node, no P2P, IPC unavailable)
                from .p2p import PeerUpdate
                try:
                    self._peer = PeerUpdate(self._flat)
                except RuntimeError as e:
                    if dist.get_rank() == 0:
                        print(f"stego_b200: peer-memory update unavailable, using NCCL all-reduce ({e})")
        return tuple(self._flat.optimizers)

    def apply_update(self):
        """manual_backward's DDP all-reduce + the three optimizer.step() calls (train_segmentation.py:227-230) on the
        current stream: one fused exchange-and-Adam over peer memory, or NCCL all-reduce + three Adam launches."""
        net_optim, linear_probe_optim, cluster_probe_optim = self.optimizers()
        if getattr(self, "_peer", None) is not None:
            self._peer.step((net_optim, linear_probe_optim, cluster_probe_optim))
        else:
            allreduce_gradients(self._flat)
            net_optim.step()
            cluster_probe_optim.step()
            linear_probe_optim.step()

    def check_update_health(self):
        """Raises if a rank missed the peer-memory rendezvous (synchronises the device)."""
        self.flush()
        if getattr(self, "_peer", None) is not None:
            self._peer.check()

    def optimizers(self):
        if self._flat is None:
            self.configure_optimizers()
        return tuple(self._flat.optimizers)

    def _mark(self, name):
        if self.profile_marks is not None:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            self.profile_marks.append((name, ev))

    # ---- the step ---------------------------------------------------------------------------------
    def training_step(self, batch, batch_idx):
        """train_segmentation.py:112-245.  The shipped configuration (dino arch, correspondence loss, no salience /
        rec / aug / crf terms) runs as the hand-scheduled kernel sequence of fused_step.FusedStep; anything else
        (or cfg.fused_step = False) takes the autograd-stitched path below.  Both compute the same step."""
        if getattr(self.cfg, "fused_step", True):
            if self._fused is None:
                from .fused_step import FusedStep
                self._fused = FusedStep(self)
            if self._fused.supported(batch):
                return self._fused.run(batch)
        return self._training_step_autograd(batch, batch_idx)

    def _training_step_autograd(self, batch, batch_idx):
        cfg = self.cfg
        self.flush()
        net_optim, linear_probe_optim, cluster_probe_optim = self.optimizers()
        net_optim.zero_grad()
        linear_probe_optim.zero_grad()
        cluster_probe_optim.zero_grad()

        self._mark("start")
        img, img_pos, label = batch["img"], batch["img_pos"], batch["label"]
        B = img.shape[0]
        net = self.net
        fh, fw = img.shape[2] // net.patch_size, img.shape[3] // net.patch_size
        use_pos = cfg.correspondence_weight > 0

        # frozen backbone on img ++ img_pos in one pass (reference: two net() calls, :130,:132)
        with torch.no_grad():
            tok_all = net.backbone_tokens(torch.cat([img, img_pos], 0) if use_pos else img,
                                          use_graph=getattr(cfg, "cuda_graph", True))  # [2B, hw, E] bf16
        self._mark("vit_forward")
        # Dropout2d noises in the reference's RNG order: net(img) draws three, then net(img_pos) draws three
        m1, m2, m3 = net.draw_masks(B, img.device)
        if use_pos:
            p1, p2, p3 = net.draw_masks(B, img.device)
            cat = lambda a, b: torch.cat([a, b], 0) if a is not None else None
            M1, M2 = cat(m1, p1), cat(m2, p2)
        else:
            M1, M2, p3 = m1, m2, None
        code_all = net.head_code(tok_all, M1, M2, fh, fw)  # [2B, dim, h, w]
        code = code_all[:B]
        E = tok_all.shape[-1]
        feats = tok_all[:B].view(B, fh, fw, E).permute(0, 3, 1, 2)  # NCHW view, bf16, channel stride 1

        self._mark("head_forward")
        loss = 0
        if use_pos:
            code_pos = code_all[B:]
            feats_pos = tok_all[B:].view(B, fh, fw, E).permute(0, 3, 1, 2)
            if cfg.use_true_labels:
                raise RuntimeError("stego_b200: use_true_labels is not part of the fused path")
            salience = batch["mask"].to(torch.float32).squeeze(1) if cfg.use_salience else None
            salience_pos = batch["mask_pos"].to(torch.float32).squeeze(1) if cfg.use_salience else None
            lossfn = self.contrastive_corr_loss_fn
            coords1, coords2 = lossfn.draw_coords(feats, salience, salience_pos)
            # same RNG calls as modules.super_perm (randperm per negative); its fix-up runs inside the sampling kernel
            perms = torch.empty(cfg.neg_samples, B, dtype=torch.long, device=img.device)
            for i in range(cfg.neg_samples):
                torch.randperm(B, device=img.device, dtype=torch.long, out=perms[i])
            # the returned-feature dropout (modules.py:116) is folded into the sampling kernel (chan_scale)
            losses, cd_means, _, _ = corr.corr_loss(feats, feats_pos, code_all, None, coords1, coords2, perms, self._spec,
                                                    want_elems=False, chan_scale=m3 if cfg.dropout else None,
                                                    chan_scale_pos=p3 if cfg.dropout else None, raw_perms=True,
                                                    pair=True)
            pos_intra_loss, pos_inter_loss = losses[0], losses[1]
            neg_inter_loss = losses[2:].mean()
            self.log('loss/pos_intra', pos_intra_loss)
            self.log('loss/pos_inter', pos_inter_loss)
            self.log('loss/neg_inter', neg_inter_loss)
            self.log('cd/pos_intra', cd_means[0])
            self.log('cd/pos_inter', cd_means[1])
            self.log('cd/neg_inter', cd_means[2:].mean())
            loss = loss + (cfg.pos_inter_weight * pos_inter_loss + cfg.pos_intra_weight * pos_intra_loss +
                           cfg.neg_inter_weight * neg_inter_loss) * cfg.correspondence_weight

        # optional terms, off in the shipped config (train_config.yml: rec/aug_alignment/crf weights 0): fused kernels for the
        # pairwise CRF term and the two cosine alignments; resize / grid_sample / the decoder conv stay torch ops
        if cfg.rec_weight > 0 or cfg.aug_alignment_weight > 0 or cfg.crf_weight > 0:
            feats_f = feats.float() * (m3.view(B, E, 1, 1) if (cfg.dropout and m3 is not None) else 1.0)
            if cfg.rec_weight > 0:
                rec_loss = -pixel_cosine(self.decoder(code), feats_f).mean()
                self.log('loss/rec', rec_loss)
                loss = loss + cfg.rec_weight * rec_loss
            if cfg.aug_alignment_weight > 0:
                _, code_aug = net(batch["img_aug"])
                coord = F.interpolate(batch["coord_aug"].permute(0, 3, 1, 2), code_aug.shape[2], mode="bilinear",
                                      align_corners=False).permute(0, 2, 3, 1)
                aug = -pixel_cosine(sample(code, coord), code_aug).mean()
                self.log('loss/aug_alignment', aug)
                loss = loss + cfg.aug_alignment_weight * aug
            if cfg.crf_weight > 0:
                rs = lambda t: F.interpolate(t, 56, mode="bilinear", align_corners=False)
                crf = self.crf_loss_fn(rs(img), norm(rs(code))).mean()
                self.log('loss/crf', crf)
                loss = loss + cfg.crf_weight * crf

        self._mark("corr_loss_forward")
        detached_code = code.detach()
        linear_loss = linear_probe_ce(detached_code, self.linear_probe.weight, self.linear_probe.bias, label)
        loss = loss + linear_loss
        self.log('loss/linear', linear_loss)
        cluster_loss, _, _ = _ClusterLookupFn.apply(detached_code, self.cluster_probe.clusters, None, False, False)
        loss = loss + cluster_loss
        self.log('loss/cluster', cluster_loss)
        self.log('loss/total', loss)

        self._mark("probes_forward")
        loss.backward()  # manual_backward (:227)
        self._flat.rebind()
        self._mark("backward")
        self.apply_update()
        self._mark("allreduce_adam")

        if cfg.reset_probe_steps is not None and self.global_step == cfg.reset_probe_steps:
            self.reset_probes()
        self.global_step += 1
        return loss
