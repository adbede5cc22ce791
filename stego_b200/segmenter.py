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

import contextlib
from typing import Dict, List, Optional, Sequence

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib, corr, ops
from .modules import ClusterLookup, ContrastiveCorrelationLoss, ContrastiveCRFLoss, DinoFeaturizer, \
    FeaturePyramidNet, _ClusterLookupFn, _ClusterLookupWideFn, norm, pixel_cosine, sample


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
        # the hyper-parameters go over as doubles: the kernel's coefficients (1 - beta2 above all) are formed from them
        rc = _lib.load().stego_adam_step(_lib.ptr(o.param[sl]), _lib.ptr(o.grad[sl]), _lib.ptr(o.exp_avg[sl]),
                                         _lib.ptr(o.exp_avg_sq[sl]), g.numel, float(pg["lr"]), float(pg["betas"][0]),
                                         float(pg["betas"][1]), float(pg["eps"]), self.steps, o.grad_scale, _lib.stream())
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


def true_label_pos(batch) -> torch.Tensor:
    """batch["label_pos"], the labels of img_pos that cfg.use_true_labels takes as the positive teacher signal
    (train_segmentation.py:128, 136-137)."""
    if batch.get("label_pos") is None:
        raise RuntimeError("stego_b200: cfg.use_true_labels needs batch['label_pos'] (the labels of img_pos) next to "
                           "batch['label']")
    return batch["label_pos"]


def aug_views_of(batch, res: int):
    """(img_aug, coord_aug) of the aug-alignment term (train_segmentation.py:189-199): the caller's views when the batch
    carries them, else built from batch["img"] (fp32, normalised) and the per-sample seeds batch["seed"] at res."""
    if batch.get("img_aug") is not None or batch.get("coord_aug") is not None:
        return batch["img_aug"], batch["coord_aug"]
    if batch.get("seed") is None:
        raise RuntimeError("stego_b200: cfg.aug_alignment_weight > 0 needs batch['seed'] (one seed per sample) or the "
                           "views batch['img_aug'] / batch['coord_aug']")
    from .augment import aug_alignment_views, batch_seeds
    return aug_alignment_views(batch["img"], batch_seeds(batch["seed"]), res)


# --------------------------------------------------------------------------------------------------
# linear probe: 1x1 conv -> bilinear upsample -> masked CE, forward + backward in one fused call
# --------------------------------------------------------------------------------------------------
def linear_probe_ce_step(x, weight, bias, label, logits, dlogits, partials, loss, dW, db, grad_scale: float) -> None:
    """Linear probe forward + backward (train_segmentation.py:213-218) of x, a tokens-major [B, C, h, w] view
    (ops.tokens_major), against label [B, H, W] (an ops.LABEL_BYTES dtype): loss [2] = (mean CE, valid pixels), dW / db
    += grad_scale * gradient.  dlogits, dW and db are accumulated into and must arrive zeroed."""
    B, C, h, w = x.shape
    H, W = label.shape[-2], label.shape[-1]
    lib = _lib.load()
    if C > 96:  # the backbone's width (projection_type None): exact fixed-point logit gradient, bit-reproducible dW / db
        dfix = torch.zeros(B * h * w, 32, dtype=torch.int64, device=x.device) if dlogits is not None else None
        _lib.check(lib.stego_linear_probe_ce_wide(
            _lib.ptr(x), x.stride(3), C, _lib.ptr(weight), _lib.ptr(bias), weight.shape[0], _lib.ptr(label),
            ops.LABEL_BYTES[label.dtype], B, h, w, H, W, _lib.ptr(logits), _lib.ptr(dlogits), _lib.ptr(dfix),
            _lib.ptr(partials), _lib.ptr(loss), grad_scale, _lib.ptr(dW), _lib.ptr(db), _lib.stream()),
            "stego_linear_probe_ce_wide")
        return
    _lib.check(lib.stego_linear_probe_ce(
        _lib.ptr(x), x.stride(3), C, _lib.ptr(weight), _lib.ptr(bias), weight.shape[0], _lib.ptr(label),
        ops.LABEL_BYTES[label.dtype], B, h, w, H, W, _lib.ptr(logits), _lib.ptr(dlogits), _lib.ptr(partials),
        _lib.ptr(loss), grad_scale, _lib.ptr(dW), _lib.ptr(db), _lib.stream()), "stego_linear_probe_ce")


class _LinearProbeCEFn(torch.autograd.Function):

    @staticmethod
    def forward(ctx, code_nchw, weight, bias, label):
        # code_nchw: detached [B, C, h, w] view whose channel stride is 1 (tokens-major storage)
        B, C, h, w = code_nchw.shape
        n = weight.shape[0]
        dev = code_nchw.device
        if n > 32 or not (C <= 96 or C in (384, 768)):
            raise RuntimeError(f"stego_b200 linear probe: n_classes={n} (<=32) / dim={C} (<=96, or 384 / 768) "
                               f"unsupported")
        rows = B * h * w
        lab, _ = ops.probe_label(label, B, label.shape[-2], label.shape[-1])
        logits = torch.empty(rows, 32, dtype=torch.float32, device=dev)
        dlogits = torch.zeros(rows, 32, dtype=torch.float32, device=dev)
        loss = torch.empty(2, dtype=torch.float32, device=dev)
        dW = torch.zeros(n, C, dtype=torch.float32, device=dev)
        db = torch.zeros(n, dtype=torch.float32, device=dev)
        wf = weight.detach().float().reshape(n, C).contiguous()
        bf = bias.detach().float().contiguous()
        linear_probe_ce_step(ops.tokens_major(code_nchw), wf, bf, lab, logits, dlogits, ops.probe_scratch(dev), loss,
                             dW, db, 1.0)
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
        dim = cfg.dim if cfg.continuous else n_classes
        # the limits of the probe and correspondence-loss kernels, checked before anything is drawn or built, so that an
        # unsupported configuration fails here rather than part-way through its first training step.  The one wider
        # code is the DINO baseline's: projection_type None, where the code is the backbone's features
        # (modules.py:108-113) and dim their width
        n_feats = 384 if cfg.model_type == "vit_small" else 768
        baseline = cfg.arch == "dino" and cfg.projection_type is None and cfg.continuous and dim == n_feats
        if not (1 <= dim <= 96 or baseline):
            raise RuntimeError(f"stego_b200: code dim {dim} unsupported (1..96, or the backbone's {n_feats} with "
                               f"projection_type None)")
        if not 1 <= n_classes <= 32:
            raise RuntimeError(f"stego_b200: n_classes={n_classes} unsupported by the linear probe (1..32)")
        if not 0 <= cfg.extra_clusters <= 64 - n_classes:
            raise RuntimeError(f"stego_b200: n_classes + extra_clusters = {n_classes + cfg.extra_clusters} cluster "
                               f"probe rows unsupported (<= 64)")
        spec = corr.make_spec(cfg)
        super().__init__()
        self.cfg = cfg
        self.n_classes = n_classes
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
        self._spec = spec
        self._fused = None
        self.profile_marks = None  # optional list: bench.py --breakdown collects (name, cuda event) pairs here
        # cd histograms every cfg.hist_freq steps (train_segmentation.py:144-146, 165-168) go to
        # logger.experiment.add_histogram_raw: anything with that, e.g. a Lightning TensorBoardLogger or
        # SimpleNamespace(experiment=SummaryWriter(...)).  None: no histograms, and the step launches nothing extra.
        # Under torch.distributed each rank bins its own shard; set the logger on rank 0 only, as the reference writes
        # from rank 0's experiment.
        self.logger = None
        self.logged_histograms: Dict[str, dict] = {}  # tag -> the add_histogram_raw fields last passed to the logger
        self._hist_pending = None  # (hist.CdHistogram, global_step) staged by a step, delivered by the next one

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
        self._deliver_histograms()

    def should_log_hist(self) -> bool:
        """train_segmentation.py:142-144 (should_log_hist), for a step that has a logger and a correspondence loss."""
        f = getattr(self.cfg, "hist_freq", None)
        return (self.logger is not None and f is not None and self.global_step % f == 0 and self.global_step > 0
                and self.cfg.correspondence_weight > 0)

    def _stage_histograms(self, h) -> None:
        """Queue the copies of a step's histograms to the host; the next training_step or flush() logs them."""
        h.stage()
        self._hist_pending = (h, self.global_step)

    def _deliver_histograms(self) -> None:
        if self._hist_pending is None:
            return
        h, step = self._hist_pending
        self._hist_pending = None
        for tag, f in h.results().items():
            self.logged_histograms[tag] = f
            if self.logger is not None:
                self.logger.experiment.add_histogram_raw(tag, global_step=step, **f)

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
        """train_segmentation.py:112-245.  The shipped configuration (dino arch, correspondence loss, no rec / crf
        terms; use_salience, use_true_labels, "KK" and the aug-alignment term fed by batch["seed"] included, and the rec /
        crf terms with cfg.fused_rec_crf) runs as the hand-scheduled kernel sequence of fused_step.FusedStep; anything
        else (or cfg.fused_step = False) takes the autograd-stitched path below.  Both compute the same step.

        With cfg.aug_alignment_weight > 0 the batch carries either the views batch["img_aug"] / batch["coord_aug"]
        (the autograd path, with them) or batch["seed"]: B ints, a list or a CPU tensor, from which the step builds
        the views itself (augment.aug_alignment_views at cfg.res, from the fp32 batch["img"]).

        projection_type None (the DINO baseline, dim = the backbone's width, correspondence_weight 0) trains the probes
        alone on the autograd path: the backbone on img, its features as the code, the wide probe kernels, Adam."""
        if self.net.proj_type is None:
            self._check_baseline_step()
            self._deliver_histograms()
            return self._training_step_autograd(batch, batch_idx)
        self._deliver_histograms()
        if getattr(self.cfg, "fused_step", True):
            if self._fused is None:
                from .fused_step import FusedStep
                self._fused = FusedStep(self)
            if self._fused.supported(batch):
                return self._fused.run(batch)
        return self._training_step_autograd(batch, batch_idx)

    def _check_baseline_step(self) -> None:
        """The DINO baseline's step (projection_type None): the probes on the backbone's features, dim its width, with
        no term that needs a code-side gradient or a code-side kernel beyond 96 channels.  Checked before anything is
        enqueued."""
        cfg, net = self.cfg, self.net
        if net.dim != net.n_feats:
            raise ValueError(f"stego_b200: projection_type None makes the code the backbone's {net.n_feats} channels, "
                             f"but dim is {net.dim}: the reference cannot run this configuration")
        if cfg.correspondence_weight > 0:
            raise ValueError("stego_b200: projection_type None trains the probes alone; correspondence_weight > 0 has "
                             "no parameter to train (set it to 0, as the DINO baseline does)")
        for name in ("rec_weight", "aug_alignment_weight", "crf_weight"):
            if getattr(cfg, name) > 0:
                raise ValueError(f"stego_b200: {name} > 0 with projection_type None is unsupported (its kernels take "
                                 f"codes of at most 96 channels)")

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
        if cfg.aug_alignment_weight > 0:
            img_aug, coord_aug = aug_views_of(batch, cfg.res)
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
        if net.proj_type is None:  # the DINO baseline: the code is the features (modules.py:108-113)
            code_all = tok_all.float().view(-1, fh, fw, tok_all.shape[-1]).permute(0, 3, 1, 2)
        else:
            code_all = net.head_code(tok_all, M1, M2, fh, fw)  # [2B, dim, h, w]
        code = code_all[:B]
        E = tok_all.shape[-1]
        feats = tok_all[:B].view(B, fh, fw, E).permute(0, 3, 1, 2)  # NCHW view, bf16, channel stride 1

        self._mark("head_forward")
        loss = 0
        hist = None
        if use_pos:
            code_pos = code_all[B:]
            feats_pos = tok_all[B:].view(B, fh, fw, E).permute(0, 3, 1, 2)
            label_pos = true_label_pos(batch) if cfg.use_true_labels else None
            salience = batch["mask"].to(torch.float32).squeeze(1) if cfg.use_salience else None
            salience_pos = batch["mask_pos"].to(torch.float32).squeeze(1) if cfg.use_salience else None
            lossfn = self.contrastive_corr_loss_fn
            if self.should_log_hist():
                from .hist import CdHistogram
                hist = CdHistogram(self._spec, B, img.device)
            coords1, coords2 = lossfn.draw_coords(feats, salience, salience_pos)
            # same RNG calls as modules.super_perm (randperm per negative); its fix-up runs inside the sampling kernel
            perms = torch.empty(cfg.neg_samples, B, dtype=torch.long, device=img.device)
            for i in range(cfg.neg_samples):
                torch.randperm(B, device=img.device, dtype=torch.long, out=perms[i])
            if cfg.use_true_labels:
                # train_segmentation.py:135-137: the teacher signal is the one-hot ground truth, sampled straight from
                # the label maps (m3 / p3 were drawn, as the reference's net() calls draw them, and scale nothing)
                ftiles = corr.build_label_tiles(label, label_pos, coords1, coords2, perms, self._spec, self.n_classes,
                                                raw_perms=True)
                losses, cd_means, _, _ = corr.corr_loss(None, None, code_all, None, coords1, coords2, perms, self._spec,
                                                        want_elems=False, raw_perms=True, pair=True, ftiles=ftiles,
                                                        hist=hist)
            else:
                # the returned-feature dropout (modules.py:116) is folded into the sampling kernel (chan_scale)
                losses, cd_means, _, _ = corr.corr_loss(feats, feats_pos, code_all, None, coords1, coords2, perms,
                                                        self._spec, want_elems=False,
                                                        chan_scale=m3 if cfg.dropout else None,
                                                        chan_scale_pos=p3 if cfg.dropout else None, raw_perms=True,
                                                        pair=True, hist=hist)
            if hist is not None:
                self._stage_histograms(hist)
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
                _, code_aug = net(img_aug)
                coord = F.interpolate(coord_aug.permute(0, 3, 1, 2), code_aug.shape[2], mode="bilinear",
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
        if net.dim > 96:
            cluster_loss = _ClusterLookupWideFn.apply(detached_code, self.cluster_probe.clusters)
        else:
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

    # ---- validation -------------------------------------------------------------------------------
    @contextlib.contextmanager
    def _net_in_eval_mode(self):
        """The net in eval mode inside the block, every module's train / eval mode restored on exit (also on an error):
        there is no Trainer to call `.train()` afterwards, and the hand-scheduled step only runs on a net in training
        mode."""
        modes = [(m, m.training) for m in self.net.modules()]
        self.net.eval()
        try:
            yield
        finally:
            for m, mode in modes:
                m.training = mode

    def validation_step(self, batch, batch_idx):
        """train_segmentation.py:254-275: the eval-mode net, then upsampling to the label size, both probes, both
        argmaxes and both `UnsupervisedMetrics.update` calls as ONE fused_probe_log_probs pass (the upsampled code is
        never materialised).  `cluster_probe(code, None)[1].argmax(1)` is the argmax of the inner products, which is
        the argmax of the kernel's alpha = 2 logits.

        Waits for the previous step's parameter update, draws no random numbers and leaves the training step's CUDA
        graphs and workspace alone.  The net's train / eval modes are restored on exit: there is no Trainer to call
        `.train()` afterwards, and the hand-scheduled step only runs on a net in training mode.  Returns the
        reference's preview dict on the CPU (first cfg.n_images entries, int64 predictions)."""
        from .eval import fused_probe_log_probs
        self.flush()
        img, label = batch["img"], batch["label"]
        n_images = getattr(self.cfg, "n_images", 5)
        with self._net_in_eval_mode(), torch.no_grad():
            _, code = self.net(img)
            out = fused_probe_log_probs(code, self.linear_probe, self.cluster_probe, label.shape[-2:], 2.0,
                                        want_log_probs=False, want_argmax=n_images > 0, label=label,
                                        linear_confusion=self.linear_metrics.stats,
                                        cluster_confusion=self.cluster_metrics.stats)
        none = torch.empty(0, *label.shape[-2:], dtype=torch.long)
        return {"img": img[:n_images].detach().cpu(),
                "linear_preds": out[2][:n_images].long().cpu() if n_images > 0 else none,
                "cluster_preds": out[3][:n_images].long().cpu() if n_images > 0 else none,
                "label": label[:n_images].detach().cpu()}

    def correspondence_pr_step(self, batch, metric) -> None:
        """plot_pr_curves.py:126-142 (LitRecalibrator.validation_step) for the two methods this package has: the head's
        code ("STEGO (Ours)", :140) and the backbone features ("DINO", :141) of the eval-mode net, scored against
        the labels by `metric`, a correspondence.CorrespondencePR.  Draws coords1 then coords2 with the reference's two
        `torch.rand([B, fs, fs, 2]) * 2 - 1` calls (:134-136) at cfg.feature_samples, on the image's device.

        Like validation_step it waits for the previous step's parameter update, leaves the training step's CUDA graphs
        and workspace alone and restores the net's train / eval modes on exit.  Nothing is copied to the host."""
        self.flush()
        img, label = batch["img"], batch["label"]
        with self._net_in_eval_mode(), torch.no_grad():
            feats, code = self.net(img)
            fs = int(self.cfg.feature_samples)
            coord_shape = [img.shape[0], fs, fs, 2]
            coords1 = torch.rand(coord_shape, device=img.device) * 2 - 1
            coords2 = torch.rand(coord_shape, device=img.device) * 2 - 1
            metric.update(feats, code, label, coords1, coords2)

    def eval_step(self, batch, run_crf: bool = False, want_probs: bool = False) -> Dict[str, torch.Tensor]:
        """The evaluation loop body of eval_segmentation.py:122-141 (also demo_segmentation.py:57-78, plot_potsdam.py:44-57)
        for one batch of frames:

            code = (net(img)[1] + net(img.flip(3))[1].flip(3)) / 2
            code = F.interpolate(code, size, mode='bilinear', align_corners=False)
            linear_probs  = torch.log_softmax(linear_probe(code), dim=1)
            cluster_probs = cluster_probe(code, 2, log_probs=True)
            preds = batched_crf(img, probs).argmax(1) if run_crf else probs.argmax(1)     # for both probes
            test_linear_metrics.update(linear_preds, label); test_cluster_metrics.update(cluster_preds, label)

        batch["img"]: the normalised frames [B, 3, H, W], fp32 or bf16, CUDA.  batch["label"] (optional): [B, H', W'],
        uint8 with 255 = ignore, int32 or int64; with it both `final/` confusion matrices (test_linear_metrics.stats,
        test_cluster_metrics.stats) are accumulated in the same pass, and `compute()` stays the caller's call.  The output
        size is the label's (eval_segmentation, plot_potsdam), or the frames' without a label (demo_segmentation); with
        run_crf the label must have the frames' size (the dense CRF runs at image resolution, fused_eval_crf).

        The frame and its mirror go through the frozen ViT as one batch of 2B, the mirrored frames read in place by the
        patchify kernel and the whole backbone replayed as one CUDA graph per frame shape (cached beside the training
        step's graphs, never replacing them).  The eval-mode head (no dropout noise) runs once over the 2B rows, then
        fused_probe_log_probs (or fused_eval_crf with run_crf) takes the two halves of the code as code / code_flipped.

        Returns dict(linear_preds, cluster_preds), uint8 [B, H', W'] on the device; with want_probs also
        linear_probs / cluster_probs fp32 [B, n, H', W']: the log-probabilities without CRF, the CRF marginals with it.
        Like validation_step it waits for the previous step's parameter update, draws no random numbers, leaves the
        training step's workspace, graphs and parameters alone and restores the net's train / eval modes on exit.
        With projection_type None (the DINO baseline, dim = the backbone's width) the code is the mirrored bf16 tokens
        themselves, read in place by the probe kernels.  Configurations the fused eval kernels do not take
        (projection_type None with another dim; more than 32 cluster-probe rows) and CPU tensors are refused before
        anything is enqueued."""
        from .eval import fused_eval_crf, fused_probe_log_probs
        img, label = batch["img"], batch.get("label")
        self._check_eval_args(img, label, run_crf)
        self.flush()
        net = self.net
        B, fh, fw = img.shape[0], img.shape[2] // net.patch_size, img.shape[3] // net.patch_size
        stats = dict(linear_confusion=self.test_linear_metrics.stats, cluster_confusion=self.test_cluster_metrics.stats) \
            if label is not None else {}
        with self._net_in_eval_mode(), torch.no_grad():
            tok = net.backbone_tokens(img, use_graph=getattr(self.cfg, "cuda_graph", True), mirror=True)  # [2B, hw, E]
            code_all = net.eval_code(tok, fh, fw)  # [2B, dim, h, w]
            code, code_flipped = code_all[:B], code_all[B:]
            if run_crf:
                out = fused_eval_crf(code, self.linear_probe, self.cluster_probe, img, 2.0, code_flipped=code_flipped,
                                     label=label, want_marginals=want_probs, **stats)
                preds, probs = out[:2], out[2:]
            else:
                size = label.shape[-2:] if label is not None else img.shape[-2:]
                out = fused_probe_log_probs(code, self.linear_probe, self.cluster_probe, size, 2.0,
                                            want_log_probs=want_probs, want_argmax=True, code_flipped=code_flipped,
                                            label=label, **stats)
                preds, probs = out[2:], out[:2]
        result = dict(linear_preds=preds[0], cluster_preds=preds[1])
        if want_probs:
            result.update(linear_probs=probs[0], cluster_probs=probs[1])
        return result

    def eval_scene(self, tiles: torch.Tensor, grid: Sequence[int], label: Optional[torch.Tensor] = None,
                   run_crf: bool = False, probes: Sequence[str] = ("linear", "cluster"), want_probs: bool = False,
                   map_clusters: bool = False, chunk: int = 64) -> Dict[str, torch.Tensor]:
        """A scene evaluated from its tiles and stitched into one mosaic (plot_potsdam.py:44-83):

            for each chunk of tiles: eval_step's loop body (flip-TTA code, upsampling, probes, metric updates)
            stitch: tile i goes to tile row i // C, tile column i % C of an R t x C t mosaic
            probs = dense_crf(mosaic image, mosaic probs) if run_crf          # one CRF across the tile seams
            preds = test_cluster_metrics.map_clusters(probs.argmax(0)) if map_clusters

        tiles: the normalised frames [R*C, 3, t, t'], fp32 or bf16, CUDA, in row-major tile order; grid = (R, C).  label
        (optional): [R*C, t, t'], uint8 with 255 = ignore, int32 or int64.  probes: the probes to evaluate, "linear"
        and / or "cluster".  Returns `<probe>_preds` uint8 [R t, C t'] per probe and, with want_probs,
        `<probe>_probs` fp32 [n, R t, C t']: the log-probabilities without the CRF, the CRF marginals with it.

        The tiles go through the backbone `chunk` at a time, each frame with its mirror in one pass as in eval_step
        (two graph shapes at most: the full chunk and the tail), and the probe kernels write straight into the mosaic.
        Without run_crf the confusion matrices (test_linear_metrics / test_cluster_metrics.stats) are updated per tile
        and the outputs are bit-equal to eval_step per chunk, stitched.  With run_crf the chunks write the CRF's unary
        rows of the mosaic, the stitched image is embedded once and one mean field runs over the whole mosaic; the
        confusion counts are those of its predictions against the stitched label.  One probe (plot_potsdam's
        probes=("cluster",), or the linear probe alone) runs rows of that probe only: 32 floats a pixel instead of 64,
        half the CRF's memory and filtering work.  The mosaic's position lattice is built for the call, not cached,
        unless the grid is a single tile.  A CRF mosaic must fit the lattice's packed keys (a longer side of at most
        about 5380 pixels: Potsdam's 4800² scene fits, its native 6000² does not) and its int32 slot ids.

        map_clusters: the cluster predictions mapped to classes by test_cluster_metrics' Hungarian assignment
        (UnsupervisedMetrics.map_clusters; unmatched extra clusters become 255); the metric's compute() must have run.
        Every argument is checked before the first launch (ValueError for shapes and limits, RuntimeError for CPU
        tensors), and the mean field's value buffers are checked against the free device memory before it is
        enqueued (RuntimeError naming the sizes)."""
        from . import crf
        from .eval import _eval_codes, _probe_tables
        R, C, n_tiles, H, W, probes = self._check_scene_args(tiles, grid, label, run_crf, probes, map_clusters, chunk)
        self.flush()
        tiles = tiles.detach().contiguous()
        lib = _lib.load()
        net = self.net
        dev = tiles.device
        p = net.patch_size
        h, w = H // p, W // p
        HH, WW = R * H, C * W
        lin_on, clu_on = "linear" in probes, "cluster" in probes
        n_lin, n_clu = self.linear_probe.weight.shape[0], self.cluster_probe.clusters.shape[0]
        wl, bl, cl = _probe_tables(self.linear_probe, self.cluster_probe, net.dim)
        scratch = torch.empty(min(chunk, n_tiles) * h * w, 80, dtype=torch.float32, device=dev)  # eval_probes.cu EV_LD
        lin_stats = self.test_linear_metrics.stats if label is not None and lin_on else None
        clu_stats = self.test_cluster_metrics.stats if label is not None and clu_on else None
        out = {}
        if run_crf:
            row = 32 * len(probes)  # rows of both probes (linear, then cluster), or of the one requested
            unary = torch.empty(HH * WW, row, dtype=torch.float32, device=dev)
            Q = torch.empty(HH * WW, row, dtype=torch.float32, device=dev)
        else:
            lab, lab_bytes = ops.probe_label(label, n_tiles, H, W) if label is not None else (None, 0)
            preds = {k: torch.empty(HH, WW, dtype=torch.uint8, device=dev) for k in probes}
            probs = {k: torch.empty(n, HH, WW, dtype=torch.float32, device=dev)
                     for k, n in (("linear", n_lin), ("cluster", n_clu)) if k in probes} if want_probs else {}
        with self._net_in_eval_mode(), torch.no_grad():
            for t0 in range(0, n_tiles, chunk):
                img = tiles[t0:t0 + chunk]
                B = img.shape[0]
                tok = net.backbone_tokens(img, use_graph=getattr(self.cfg, "cuda_graph", True), mirror=True)
                code_all = net.eval_code(tok, h, w)  # [2B, dim, h, w]
                x, xf, ld, bf16 = _eval_codes(code_all[:B], code_all[B:])
                sfx = "_bf16" if bf16 else ""
                if run_crf:
                    _lib.check(getattr(lib, "stego_eval_crf_unary_mosaic" + sfx)(
                        _lib.ptr(x), _lib.ptr(xf), ld, net.dim, B, h, w, H, W, _lib.ptr(wl), _lib.ptr(bl), n_lin,
                        _lib.ptr(cl), n_clu, 2.0, _lib.ptr(scratch), _lib.ptr(unary), _lib.ptr(Q), int(lin_on) + 2 * int(clu_on), t0, R, C, WW,
                        _lib.stream()), "stego_eval_crf_unary_mosaic" + sfx)
                else:
                    _lib.check(getattr(lib, "stego_eval_probes_mosaic" + sfx)(
                        _lib.ptr(x), _lib.ptr(xf), ld, net.dim, B, h, w, H, W, _lib.ptr(wl), _lib.ptr(bl), n_lin,
                        _lib.ptr(cl), n_clu, 2.0, _lib.ptr(scratch), _lib.ptr(probs.get("linear")),
                        _lib.ptr(probs.get("cluster")), _lib.ptr(preds.get("linear")), _lib.ptr(preds.get("cluster")),
                        _lib.ptr(lab[t0:] if lab is not None else None), lab_bytes, n_lin if lab is not None else 0,
                        _lib.ptr(lin_stats), _lib.ptr(clu_stats), t0, R, C, WW, _lib.stream()),
                        "stego_eval_probes_mosaic" + sfx)
        if run_crf:
            image = crf.prepare_image(tiles.view(R, C, 3, H, W).permute(2, 0, 3, 1, 4).reshape(3, HH, WW))
            lg = crf._position_lattice(HH, WW, dev, cache=n_tiles == 1)
            lb = crf._bilateral_lattice([image])
            crf.check_value_buffers(lg.M, lb.M, row, dev, "eval_scene")
            val_g = torch.empty(2, lg.M, row, dtype=torch.float32, device=dev)
            val_b = torch.empty(2, lb.M, row, dtype=torch.float32, device=dev)
            lab, lab_bytes = (None, 0)
            if label is not None:
                lab, lab_bytes = ops.probe_label(label.reshape(R, C, H, W).permute(0, 2, 1, 3), 1, HH, WW)
            preds = {k: torch.empty(HH, WW, dtype=torch.uint8, device=dev) for k in probes}
            probs = {k: torch.empty(n, HH, WW, dtype=torch.float32, device=dev)
                     for k, n in (("linear", n_lin), ("cluster", n_clu)) if k in probes} if want_probs else {}
            # the mean field's two probe slots in row order; one probe (either) takes the first slot
            slots = [(k, n, st) for k, n, st in (("linear", n_lin, lin_stats), ("cluster", n_clu, clu_stats)) if k in probes]
            (first, n0, conf0), (second, n1, conf1) = slots[0], (slots[1] if len(slots) == 2 else (None, 0, None))
            _lib.check(lib.stego_crf_mean_field(
                1, HH * WW, n0, n1, crf.MAX_ITER, _lib.ptr(unary), _lib.ptr(Q),
                _lib.ptr(lg.offset), _lib.ptr(lg.bary), _lib.ptr(lg.rowptr), _lib.ptr(lg.slots), _lib.ptr(lg.n1),
                _lib.ptr(lg.n2), _lib.ptr(lg.norm), lg.M,
                _lib.ptr(lb.offset), _lib.ptr(lb.bary), _lib.ptr(lb.rowptr), _lib.ptr(lb.slots), _lib.ptr(lb.n1),
                _lib.ptr(lb.n2), _lib.ptr(lb.norm), lb.M, float(crf.POS_W), float(crf.Bi_W),
                _lib.ptr(val_g[0]), _lib.ptr(val_g[1]), _lib.ptr(val_b[0]), _lib.ptr(val_b[1]),
                _lib.ptr(probs.get(first)), _lib.ptr(probs.get(second)), _lib.ptr(preds[first]),
                _lib.ptr(preds.get(second)), _lib.ptr(lab), lab_bytes, n_lin if lab is not None else 0,
                _lib.ptr(conf0), _lib.ptr(conf1), _lib.stream()), "stego_crf_mean_field")
        for k in probes:
            out[f"{k}_preds"] = preds[k]
            if want_probs:
                out[f"{k}_probs"] = probs[k]
        if map_clusters:
            lut = self.test_cluster_metrics.map_clusters(torch.arange(n_clu, device=dev)).to(torch.uint8)
            out["cluster_preds"] = lut[out["cluster_preds"].int()]
        return out

    def _check_scene_args(self, tiles, grid, label, run_crf, probes, map_clusters, chunk):
        """eval_scene's own rules, then eval_step's on the tiles as one batch (shapes and limits: ValueError; CPU
        tensors last: RuntimeError).  Returns (R, C, n_tiles, H, W, probes as a tuple)."""
        if tiles.dim() != 4:
            raise ValueError(f"eval_scene: tiles must be [R*C, 3, H, W], got {tuple(tiles.shape)}")
        n_tiles, _, H, W = tiles.shape
        try:
            R, C = (int(g) for g in grid)
        except (TypeError, ValueError):
            raise ValueError(f"eval_scene: grid must be (rows, columns), got {grid!r}") from None
        if R < 1 or C < 1 or R * C != n_tiles:
            raise ValueError(f"eval_scene: a {R} x {C} grid does not hold the {n_tiles} tiles")
        probes = tuple(probes)
        if not probes or len(set(probes)) != len(probes) or not set(probes) <= {"linear", "cluster"}:
            raise ValueError(f"eval_scene: probes must be \"linear\" and / or \"cluster\", got {probes!r}")
        if isinstance(chunk, bool) or not isinstance(chunk, int) or chunk < 1:
            raise ValueError(f"eval_scene: chunk must be a positive int, got {chunk!r}")
        if label is not None and tuple(label.shape) != (n_tiles, H, W):
            raise ValueError(f"eval_scene: label {tuple(label.shape)} is not one {H}x{W} map per tile of {n_tiles}")
        if run_crf:
            from . import crf
            if 6 * R * H * C * W >= 1 << 31:
                raise ValueError(f"eval_scene: a {R * H}x{C * W} mosaic has more lattice slots than the CRF's int32 "
                                 f"slot ids hold (6 per pixel, < 2^31)")
            bound, limit = crf.lattice_key_bound(R * H, C * W, 5, crf.Bi_XY_STD, crf.Bi_RGB_STD)
            if bound >= limit:
                raise ValueError(f"eval_scene: a {R * H}x{C * W} mosaic's bilateral lattice coordinates reach "
                                 f"{bound:.0f}, beyond the {limit} its packed keys hold (a longer side of at most "
                                 f"about 5380 pixels)")
        if map_clusters:
            if "cluster" not in probes:
                raise ValueError("eval_scene: map_clusters needs the cluster probe")
            if not hasattr(self.test_cluster_metrics, "assignments"):
                raise ValueError("eval_scene: map_clusters needs test_cluster_metrics.compute() to have run (its "
                                 "Hungarian assignment)")
        self._check_eval_args(tiles, label, run_crf, who="eval_scene")
        return R, C, n_tiles, H, W, probes

    def _check_eval_args(self, img, label, run_crf: bool, who: str = "eval_step") -> None:
        """eval_step's arguments against the rules of the kernels it calls, shapes and limits first (ValueError), the
        device last (RuntimeError), so that nothing is enqueued for a call that would fail part-way."""
        from .eval import _check_crf_args
        net = self.net
        p = net.patch_size
        if img.dim() != 4 or img.shape[1] != 3 or img.shape[0] < 1 or img.dtype not in (torch.float32, torch.bfloat16):
            raise ValueError(f"{who}: img must be fp32 or bf16 [B, 3, H, W], got {img.dtype} {tuple(img.shape)}")
        B, _, H, W = img.shape
        # the patchify rules (stego_vit_patchify_tta): patch 8 or 16, whole patches, rows of a multiple of 8 pixels
        if p not in (8, 16) or H % p or W % p or W % 8:
            raise ValueError(f"{who}: a {H}x{W} frame is not whole {p}x{p} patches with W a multiple of 8 "
                             f"(patch 8 or 16)")
        if net.proj_type is None and net.dim != net.n_feats:
            raise ValueError(f"{who}: projection_type None gives a code of {net.n_feats} channels, and the probes were "
                             f"built for dim={net.dim}: the DINO baseline needs dim={net.n_feats}")
        n_lin, n_clu = self.linear_probe.weight.shape[0], self.cluster_probe.clusters.shape[0]
        if n_lin > 32 or n_clu > 32:
            raise ValueError(f"{who}: {n_lin} linear-probe classes / {n_clu} cluster-probe rows unsupported by the "
                             f"fused evaluation probes (at most 32 each)")
        if label is not None:
            if label.dtype not in ops.LABEL_BYTES:
                raise ValueError(f"{who}: label dtype {label.dtype} unsupported (uint8, int32 or int64)")
            Hl, Wl = label.shape[-2:]
            if label.dim() < 2 or label.numel() != B * Hl * Wl:
                raise ValueError(f"{who}: label {tuple(label.shape)} is not one [H, W] map per frame of {B}")
            if Hl < H // p or Wl < W // p:
                raise ValueError(f"{who}: label {Hl}x{Wl} is smaller than the code {H // p}x{W // p} "
                                 f"(upsampling only)")
        if run_crf:
            # fused_eval_crf's own checks (label at the frames' size, ...), on a stand-in of the code's shape
            stub = torch.empty(1, device=img.device).expand(B, net.dim, H // p, W // p)
            stats = (self.test_linear_metrics.stats, self.test_cluster_metrics.stats) if label is not None else (None, None)
            _check_crf_args(stub, self.linear_probe, self.cluster_probe, img, stub, label, *stats)
        _lib.require_cuda(img, label, self.linear_probe.weight, self.cluster_probe.clusters,
                          self.test_linear_metrics.stats, self.test_cluster_metrics.stats, net.cluster1[0].weight)

    def validation_epoch_end(self, outputs=None) -> Dict[str, float]:
        """train_segmentation.py:277-283, 361-371 without the figures: sum both confusion matrices over the ranks (what
        torchmetrics' dist_reduce_fx="sum" does; once per epoch gives the same sums as once per step), compute mIoU /
        accuracy, log them once global_step > 2, reset both metrics.  Returns the metric dict (keys `test/linear/mIoU`,
        `test/linear/Accuracy`, `test/cluster/mIoU`, `test/cluster/Accuracy`) for callers that pick checkpoints
        themselves.  The Hungarian assignment stays on `cluster_metrics` for `map_clusters`."""
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            for m in (self.linear_metrics, self.cluster_metrics):
                dist.all_reduce(m.stats, op=dist.ReduceOp.SUM)
        tb_metrics = {**self.linear_metrics.compute(), **self.cluster_metrics.compute()}
        if self.global_step > 2:
            for k, v in tb_metrics.items():
                self.log(k, v)
        self.linear_metrics.reset()
        self.cluster_metrics.reset()
        return tb_metrics
