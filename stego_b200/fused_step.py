"""Hand-scheduled training step: the kernel sequence of `LitUnsupervisedSegmenter.training_step`
(src/train_segmentation.py:112-245) issued directly through the C-ABI, without autograd.

The autograd path (segmenter._training_step_autograd) stitches ~10 custom nodes together and leaves ~110 tiny
torch kernels (zero fills, RNG post-processing, gradient accumulation, scalar loss arithmetic) on the critical
path, each costing ~4 us of launch latency behind the frozen ViT.  Here

  * every buffer of the step lives in a workspace allocated once per input shape;
  * the *prologue* — everything that does not depend on the ViT output: the Dropout2d / coordinate / permutation
    draws (same torch RNG calls in the same order as the reference: net(img) x3 noises, net(img_pos) x3,
    rand x2, randperm x neg_samples), the bf16 operand copies of the trainable head weights, and ONE memset of
    all accumulate-into buffers (+ the flat gradient buffer) — runs on a side stream concurrently with the ViT graph;
  * forward and backward kernels are called in order, weight gradients are accumulated straight into the flat
    gradient buffer (no per-parameter AccumulateGrad kernels), and the scalar loss arithmetic is one launch.

Numerically this is the same kernel sequence as the autograd path (tests/test_modules_gpu.py checks both against the
oracle and against each other).
"""
from __future__ import annotations

import ctypes

import torch

from . import _lib, corr, ops


# label dtypes the linear-probe CE kernel reads directly (int64 is the reference's; uint8 uses 255 = ignore)
_LABEL_BYTES = {torch.int64: 8, torch.int32: 4, torch.uint8: 1}


def _round_up(a: int, b: int) -> int:
    return (a + b - 1) // b * b


class _Workspace:
    pass


class FusedStep:

    def __init__(self, seg):
        self.seg = seg
        self.ws = None
        self.key = None
        self.side = None
        self.step_idx = 0
        self.update_done = None

    # ------------------------------------------------------------------------------------------
    def supported(self, batch) -> bool:
        seg, cfg = self.seg, self.seg.cfg
        img = batch["img"]
        return (img.is_cuda and seg.training and seg.net.training and cfg.correspondence_weight > 0
                and not cfg.use_salience and not cfg.use_true_labels and seg.net.proj_type is not None
                and cfg.rec_weight == 0 and cfg.aug_alignment_weight == 0 and cfg.crf_weight == 0
                and cfg.neg_samples >= 1 and cfg.dino_feat_type == "feat"
                and seg.linear_probe.weight.shape[0] <= 32 and seg.net.dim <= 96
                and batch["label"].dtype in _LABEL_BYTES)

    # ------------------------------------------------------------------------------------------
    def _alloc(self, B, H, W, LH, LW, dev, label_dtype):
        seg, cfg, net = self.seg, self.seg.cfg, self.seg.net
        ws = _Workspace()
        E, D = net.n_feats, net.dim
        fh, fw = H // net.patch_size, W // net.patch_size
        hw = fh * fw
        M = 2 * B * hw
        P = _round_up(D, 8)
        spec = seg._spec
        f32, bf = torch.float32, torch.bfloat16
        nonlinear = net.proj_type == "nonlinear"
        ws.dims = (B, E, D, P, fh, fw, hw, M, nonlinear)
        ws.num_sms = torch.cuda.get_device_properties(dev).multi_processor_count
        # RNG outputs
        ws.M1 = torch.empty(2 * B, E, 1, 1, dtype=f32, device=dev)
        ws.M2 = torch.empty(2 * B, E, 1, 1, dtype=f32, device=dev) if nonlinear else None
        ws.M3 = torch.empty(2 * B, E, 1, 1, dtype=f32, device=dev) if cfg.dropout else None
        ws.c1 = torch.empty(B, spec.fs, spec.fs, 2, dtype=f32, device=dev)
        ws.c2 = torch.empty(B, spec.fs, spec.fs, 2, dtype=f32, device=dev)
        ws.perms = torch.empty(spec.n_neg, B, dtype=torch.long, device=dev)
        # head
        ws.x1 = torch.empty(M, E, dtype=bf, device=dev)
        ws.x2 = torch.empty(M, E, dtype=bf, device=dev) if nonlinear else None
        ws.hid = torch.empty(M, E, dtype=bf, device=dev) if nonlinear else None
        ws.code = torch.zeros(M, P, dtype=f32, device=dev)  # padding columns stay zero (the GEMMs write D columns)
        ws.w1p = torch.zeros(128, E, dtype=bf, device=dev)   # rows >= D stay zero
        ws.wbp = torch.zeros(128, E, dtype=bf, device=dev) if nonlinear else None
        ws.wab = torch.empty(E, E, dtype=bf, device=dev) if nonlinear else None
        ws.dyb = torch.empty(M, 128, dtype=bf, device=dev)
        ws.dh = torch.empty(M, E, dtype=f32, device=dev) if nonlinear else None
        ws.dhb = torch.empty(M, E, dtype=bf, device=dev) if nonlinear else None
        # correspondence loss
        ws.ftiles = torch.empty(2, spec.nslots, B, spec.rows, E, dtype=bf, device=dev)
        ws.ctiles = torch.empty(2, spec.nslots, B, spec.rows, corr.CODE_PAD, dtype=bf, device=dev)
        ws.partials, ws.row_means = spec.scratch(B, dev)
        ws.stats = torch.empty(spec.ncalls, 4, dtype=f32, device=dev)
        cw = float(cfg.correspondence_weight)
        wts = [cfg.pos_intra_weight * cw, cfg.pos_inter_weight * cw] + [cfg.neg_inter_weight * cw / spec.n_neg] * spec.n_neg
        ws.call_w = (ctypes.c_float * len(wts))(*[float(v) for v in wts])
        ws.gscale = torch.tensor([float(v) for v in wts], dtype=f32, device=dev)
        # probes
        n_lin = seg.linear_probe.weight.shape[0]
        n_clu = seg.cluster_probe.clusters.shape[0]
        ws.n_lin, ws.n_clu = n_lin, n_clu
        ws.logits = torch.empty(B * hw, 32, dtype=f32, device=dev)
        ws.ce_partials = torch.empty(16 * ws.num_sms * 2, dtype=f32, device=dev)
        ws.lin_loss = torch.empty(2, dtype=f32, device=dev)
        ws.clu_loss = torch.empty(2, dtype=f32, device=dev)
        ws.clu_scratch = torch.empty(16 * ws.num_sms, dtype=f32, device=dev)
        ws.one = torch.ones(1, dtype=f32, device=dev)
        ws.out4 = torch.empty(4, dtype=f32, device=dev)
        ws.label = torch.empty(B, LH, LW, dtype=label_dtype, device=dev)  # static copy: the tail graph bakes pointers
        ws.label_bytes = _LABEL_BYTES[label_dtype]
        ws.graph = None
        ws.eager_steps = 0
        # everything the kernels accumulate into: ONE buffer, ONE memset per step
        sizes = dict(dlogits=B * hw * 32, dtiles=spec.nslots * B * spec.rows * corr.DT_LD, dall=M * P,
                     dnc=n_clu * D, db_pad=P)
        total = sum(_round_up(v, 64) for v in sizes.values())
        ws.zbuf = torch.zeros(total, dtype=f32, device=dev)
        off = 0
        for name, n in sizes.items():
            setattr(ws, name, ws.zbuf[off:off + n])
            off += _round_up(n, 64)
        ws.label_shape = (LH, LW)
        return ws

    # ------------------------------------------------------------------------------------------
    def _prologue(self, ws):
        """Side stream: RNG draws (reference order), operand copies of the trainable weights, accumulator memset."""
        seg, cfg, net = self.seg, self.seg.cfg, self.seg.net
        B, E, D, P, fh, fw, hw, M, nonlinear = ws.dims
        keep = 0.9  # Dropout2d(p=.1), modules.py:41
        for half in (0, 1):  # net(img) then net(img_pos): cluster1 noise, cluster2 noise, returned-feature noise
            sl = slice(half * B, (half + 1) * B)
            ws.M1[sl].bernoulli_(keep).div_(keep)
            if nonlinear:
                ws.M2[sl].bernoulli_(keep).div_(keep)
            if ws.M3 is not None:
                ws.M3[sl].bernoulli_(keep).div_(keep)
        torch.rand(ws.c1.shape, out=ws.c1).mul_(2).sub_(1)  # modules.py:366-367
        torch.rand(ws.c2.shape, out=ws.c2).mul_(2).sub_(1)
        for i in range(ws.perms.shape[0]):                  # super_perm's randperm (modules.py:291-295)
            torch.randperm(B, device=ws.perms.device, dtype=torch.long, out=ws.perms[i])
        c1 = net.cluster1[0]
        ws.w1p[:D].copy_(c1.weight.detach().view(D, E))
        if nonlinear:
            ws.wab.copy_(net.cluster2[0].weight.detach().view(E, E))
            ws.wbp[:D].copy_(net.cluster2[2].weight.detach().view(D, E))
        ws.zbuf.zero_()
        seg._flat.grad.zero_()

    # ------------------------------------------------------------------------------------------
    def _tail(self, ws, tok_all):
        """Head forward .. head backward on the current stream: static workspace, no allocation, no RNG, no host
        synchronisation — captured as one CUDA graph after the first (eager) step."""
        seg, cfg, net = self.seg, self.seg.cfg, self.seg.net
        lib = _lib.load()
        B, E, D, P, fh, fw, hw, M, nonlinear = ws.dims
        spec = seg._spec
        st = _lib.stream()
        feat_tok = tok_all.reshape(M, E)

        # ---- head forward (modules.py:108-111)
        _lib.check(lib.stego_head_dropout3(_lib.ptr(feat_tok), _lib.ptr(ws.M1), _lib.ptr(ws.M2), 0, _lib.ptr(ws.x1),
                                           _lib.ptr(ws.x2), 0, 2 * B, hw, E, st), "stego_head_dropout3")
        c1 = net.cluster1[0]
        ops.gemm(ws.x1, ws.w1p, ws.code, M=M, N=D, K=E, bias=c1.bias.detach())
        if nonlinear:
            ca, cb = net.cluster2[0], net.cluster2[2]
            ops.gemm(ws.x2, ws.wab, ws.hid, M=M, N=E, K=E, bias=ca.bias.detach(), act=ops.ACT_RELU)
            ops.gemm(ws.hid, ws.wbp, ws.code, M=M, N=D, K=E, bias=cb.bias.detach(), residual=ws.code)
        seg._mark("head_forward")

        # ---- correspondence loss forward (modules.py:349-398)
        tok_pos = tok_all[B:]
        m3 = ws.M3[:B] if ws.M3 is not None else None
        p3 = ws.M3[B:] if ws.M3 is not None else None
        _lib.check(lib.stego_sample_norm_fwd(
            _lib.ptr(tok_all), _lib.ptr(tok_pos), 1, hw * E, 1, fw * E, E, _lib.ptr(m3), _lib.ptr(p3),
            _lib.ptr(ws.c1), _lib.ptr(ws.c2), _lib.ptr(ws.perms), _lib.ptr(ws.ftiles), B, E, E, fh, fw, spec.fs,
            spec.nslots, 1, st), "stego_sample_norm_fwd")
        code_pos = ws.code[B * hw:]
        _lib.check(lib.stego_sample_norm_fwd(
            _lib.ptr(ws.code), _lib.ptr(code_pos), 0, hw * P, 1, fw * P, P, 0, 0, _lib.ptr(ws.c1), _lib.ptr(ws.c2),
            _lib.ptr(ws.perms), _lib.ptr(ws.ctiles), B, D, corr.CODE_PAD, fh, fw, spec.fs, spec.nslots, 1, st),
            "stego_sample_norm_fwd")
        spec.forward(ws.ftiles, ws.ctiles, B, E, D, ws.partials, ws.row_means, ws.stats)
        seg._mark("corr_loss_forward")

        # ---- probes on the detached code (train_segmentation.py:213-225): forward + backward in place
        lp = seg.linear_probe
        lab = ws.label
        LH, LW = ws.label_shape
        _lib.check(lib.stego_linear_probe_ce(
            _lib.ptr(ws.code), P, D, _lib.ptr(lp.weight), _lib.ptr(lp.bias), ws.n_lin, _lib.ptr(lab), ws.label_bytes, B, fh, fw,
            LH, LW,
            _lib.ptr(ws.logits), _lib.ptr(ws.dlogits), _lib.ptr(ws.ce_partials), _lib.ptr(ws.lin_loss), 1.0,
            _lib.ptr(lp.weight.grad), _lib.ptr(lp.bias.grad), st), "stego_linear_probe_ce")
        cl = seg.cluster_probe.clusters
        _lib.check(lib.stego_cluster_lookup_fwd(
            _lib.ptr(ws.code), hw * P, 1, P, _lib.ptr(cl), B, D, ws.n_clu, hw, 0, 0.0, 0, 0, 0, _lib.ptr(ws.clu_loss),
            _lib.ptr(ws.clu_scratch), st), "stego_cluster_lookup_fwd")
        out4 = ws.out4
        _lib.check(lib.stego_step_losses(_lib.ptr(ws.stats), spec.ncalls, ws.call_w, _lib.ptr(ws.lin_loss),
                                         _lib.ptr(ws.clu_loss), _lib.ptr(out4), st), "stego_step_losses")
        seg._mark("probes_forward")

        # ---- backward (manual_backward, :227)
        _lib.check(lib.stego_cluster_lookup_bwd(
            _lib.ptr(ws.code), hw * P, 1, P, _lib.ptr(cl), B, D, ws.n_clu, hw, 0, 0.0, _lib.ptr(ws.one),
            _lib.ptr(ws.dnc), _lib.ptr(cl.grad), st), "stego_cluster_lookup_bwd")
        spec.backward(ws.ftiles, ws.ctiles, B, E, D, ws.stats, ws.row_means, ws.gscale, None, None, ws.dtiles)
        dall_pos = ws.dall[B * hw * P:]
        _lib.check(lib.stego_sample_norm_bwd(
            _lib.ptr(ws.code), _lib.ptr(code_pos), hw * P, 1, fw * P, P, _lib.ptr(ws.c1), _lib.ptr(ws.c2),
            _lib.ptr(ws.perms), _lib.ptr(ws.dtiles), _lib.ptr(ws.dall), _lib.ptr(dall_pos), B, D, fh, fw, spec.fs,
            spec.nslots, 1, st), "stego_sample_norm_bwd")
        # head backward: d(code) [M, P] -> bias / weight gradients straight into the flat gradient buffer
        _lib.check(lib.stego_cast_pad_bf16(_lib.ptr(ws.dall), P, D, _lib.ptr(ws.dyb), 128, M, st), "stego_cast_pad_bf16")
        _lib.check(lib.stego_colsum(_lib.ptr(ws.dall), 0, P, P, M, _lib.ptr(ws.db_pad), st), "stego_colsum")
        c1.bias.grad.copy_(ws.db_pad[:D])

        def splits_for(out_rows, out_cols):
            # split-K so that tiles x splits fills ONE wave of the persistent GEMM (one CTA per SM): at most num_sms
            # CTAs (more splits would make a second round of the grid)
            tiles = ((out_rows + 127) // 128) * ((out_cols + 127) // 128)
            return max(1, min(M // 512, ws.num_sms // tiles))
        ops.gemm(ws.dyb, ws.x1, c1.weight.grad.view(D, E), M=D, N=E, K=M, a_mn=True, b_mn=True,
                 splits=splits_for(D, E), atomic=True)
        if nonlinear:
            cb.bias.grad.copy_(ws.db_pad[:D])
            ops.gemm(ws.dyb, ws.hid, cb.weight.grad.view(D, E), M=D, N=E, K=M, a_mn=True, b_mn=True,
                     splits=splits_for(D, E), atomic=True)
            ops.gemm(ws.dyb, ws.wbp, ws.dh, M=M, N=E, K=128, b_mn=True)
            _lib.check(lib.stego_relu_bwd_bf16(_lib.ptr(ws.dh), _lib.ptr(ws.hid), _lib.ptr(ws.dhb), M * E, st),
                       "stego_relu_bwd_bf16")
            _lib.check(lib.stego_colsum(_lib.ptr(ws.dhb), 1, E, E, M, _lib.ptr(ca.bias.grad), st), "stego_colsum")
            ops.gemm(ws.dhb, ws.x2, ca.weight.grad.view(E, E), M=E, N=E, K=M, a_mn=True, b_mn=True,
                     splits=splits_for(E, E), atomic=True)

    # ------------------------------------------------------------------------------------------
    def run(self, batch):
        seg, cfg, net = self.seg, self.seg.cfg, self.seg.net
        lib = _lib.load()
        img, img_pos, label = batch["img"], batch["img_pos"], batch["label"]
        dev = img.device
        B, _, H, W = img.shape
        LH, LW = label.shape[-2], label.shape[-1]
        if seg._flat is None:
            seg.configure_optimizers()
        seg._flat.ensure_bound()  # parameters / .grad still are the views into the flat buffers the kernels write
        net_optim, linear_probe_optim, cluster_probe_optim = seg.optimizers()
        # a new flat parameter buffer (or another label dtype) invalidates the captured graph
        key = (B, H, W, LH, LW, dev.index, id(seg._flat), label.dtype)
        if self.key != key:
            self.flush()
            self.ws = self._alloc(B, H, W, LH, LW, dev, label.dtype)
            self.key = key
            self.side = torch.cuda.Stream(device=dev)
        ws = self.ws
        B, E, D, P, fh, fw, hw, M, nonlinear = ws.dims
        main = torch.cuda.current_stream()
        seg._mark("start")

        # ---- side stream: [gradient all-reduce + Adam of the PREVIOUS step, enqueued at the end of that step] ->
        #      prologue of this step.  The frozen ViT on the main stream depends on neither, so the whole update
        #      (the one collective of the data-parallel step included) is hidden under the next step's backbone.
        self.side.wait_stream(main)
        with torch.cuda.stream(self.side):
            self._prologue(ws)
            ready = torch.cuda.Event()
            ready.record(self.side)

        use_graph = bool(getattr(cfg, "cuda_graph", True)) and seg.profile_marks is None
        overlap = bool(getattr(cfg, "overlap_update", True)) and seg.profile_marks is None
        with torch.no_grad():
            tok_all = net.backbone_tokens([img, img_pos], use_graph=getattr(cfg, "cuda_graph", True))  # [2B,hw,E] bf16
            ws.label.copy_(label.reshape(B, LH, LW))
            main.wait_event(ready)
            seg._mark("vit_forward")
            if use_graph and ws.graph is not None and ws.graph[1] == tok_all.data_ptr():
                ws.graph[0].replay()
                _lib.replayed_launches += ws.graph[2]
            elif use_graph and ws.eager_steps >= 1:
                # second step on this shape: capture head fwd .. head bwd (static workspace, no allocation, no RNG) as ONE
                # CUDA graph; the eager first step has already set kernel attributes and warmed the allocator
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                n0 = lib.stego_launch_count()
                with torch.cuda.graph(g):
                    self._tail(ws, tok_all)
                ws.graph = (g, tok_all.data_ptr(), lib.stego_launch_count() - n0)
                g.replay()
                _lib.replayed_launches += ws.graph[2]
            else:
                self._tail(ws, tok_all)
                ws.eager_steps += 1
            seg._mark("backward")
            out4 = ws.out4
            loss = out4[0].clone()  # the workspace is overwritten by the next step; the returned loss is not

            # ---- update: all-reduce (N > 1) + three fused Adam launches (+ the probe reset of
            #      train_segmentation.py:232-237) on the side stream, behind the tail
            tail_done = torch.cuda.Event()
            tail_done.record(main)
            self.side.wait_event(tail_done)
            with torch.cuda.stream(self.side):
                seg.apply_update()
                if cfg.reset_probe_steps is not None and seg.global_step == cfg.reset_probe_steps:
                    seg.reset_probes()
                self.update_done = torch.cuda.Event()
                self.update_done.record(self.side)
            if not overlap:
                main.wait_event(self.update_done)
            seg._mark("allreduce_adam")

        # logging (views of the workspace: valid until the next step overwrites them)
        seg.log('loss/pos_intra', ws.stats[0, 0])
        seg.log('loss/pos_inter', ws.stats[1, 0])
        seg.log('loss/neg_inter', out4[2])
        seg.log('cd/pos_intra', ws.stats[0, 1])
        seg.log('cd/pos_inter', ws.stats[1, 1])
        seg.log('cd/neg_inter', out4[3])
        seg.log('loss/linear', ws.lin_loss[0])
        seg.log('loss/cluster', ws.clu_loss[0])
        seg.log('loss/total', out4[0])
        self.step_idx += 1
        seg.global_step += 1
        return loss

    def flush(self):
        """Make the current stream wait for the parameter update of the last step (it runs on the side stream so that
        the next step's frozen backbone can overlap it).  Anything that reads parameters, gradients or optimiser
        state outside training_step — validation forward, checkpointing, tests — goes through here
        (LitUnsupervisedSegmenter.flush / forward / state_dict call it)."""
        if self.update_done is not None:
            torch.cuda.current_stream().wait_event(self.update_done)
