"""Hand-scheduled training step: the kernel sequence of `LitUnsupervisedSegmenter.training_step`
(src/train_segmentation.py:112-245) without autograd.

The autograd path (segmenter._training_step_autograd) stitches ~10 custom nodes together and leaves ~110 tiny
torch kernels (zero fills, RNG post-processing, gradient accumulation, scalar loss arithmetic) on the critical
path, each costing ~4 us of launch latency behind the frozen ViT.  Here

  * every buffer of the step lives in a workspace allocated once per input shape;
  * the *prologue* — everything that does not depend on the ViT output: the Dropout2d / coordinate / permutation
    draws (same torch RNG calls in the same order as the reference: net(img) x3 noises, net(img_pos) x3,
    rand x2 (with use_salience: the draws of salience.draw_into), randperm x neg_samples, and with the aug-alignment
    term net(img_aug) x3), the bf16 operand copies
    of the trainable head weights, and ONE memset of all accumulate-into buffers (+ the flat gradient buffer) — runs on a side stream concurrently with the ViT graph;
  * forward and backward stages are called in order, weight gradients are accumulated straight into the flat
    gradient buffer (no per-parameter AccumulateGrad kernels), and the scalar loss arithmetic is one launch.

The stages are the functions the autograd nodes call (modules.pack_head_weights / head_forward / head_backward /
cluster_lookup_forward / cluster_lookup_backward, corr.build_tiles / build_label_tiles / sample_norm_backward / LossSpec,
segmenter.linear_probe_ce_step), given the workspace instead of per-call buffers: both paths launch the same kernels
with the same arguments.  Only stego_step_losses is called from here alone.

With cfg.aug_alignment_weight > 0 and batch["seed"] (train_segmentation.py:189-199) the step builds img_aug / coord_aug
itself (augment: host draws on a forked CPU generator, one pinned upload, two launches, all before the backbone is
enqueued), runs img, img_pos and img_aug through the backbone as ONE batch of 3B and the head over 3B rows; the term is
modules.aug_sample_forward / cosine_forward / aug_loss and their backward, inside the tail graph.

With cfg.fused_rec_crf the reconstruction term (cfg.rec_weight, train_segmentation.py:183-187) and the CRF term
(cfg.crf_weight, :201-208) run here too: modules.rec_forward / rec_backward (the decoder output never leaves the
kernel) and modules.crf_forward / crf_loss / crf_backward (only the n sampled points of the 56 x 56 maps), inside the
tail graph.  The CRF coordinates are drawn by the prologue after everything else, as the term's two randint calls come
last in the reference; its image guidance is sampled by one eager launch per step, so the graph bakes no caller pointer.
"""
from __future__ import annotations

import ctypes

import torch

from . import _lib, augment, corr, modules, ops, salience, segmenter


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
        self._masks = None  # use_salience: this step's (mask, mask_pos), read by the prologue

    # ------------------------------------------------------------------------------------------
    def supported(self, batch) -> bool:
        seg, cfg = self.seg, self.seg.cfg
        img = batch["img"]
        return (img.is_cuda and seg.training and seg.net.training and cfg.correspondence_weight > 0
                and seg.net.proj_type is not None
                and self._rec_crf_supported(batch)
                and (cfg.aug_alignment_weight == 0 or self._aug_supported(batch))
                and cfg.neg_samples >= 1 and cfg.dino_feat_type in ("feat", "KK")
                and seg.linear_probe.weight.shape[0] <= 32 and seg.net.dim <= 96
                and batch["label"].dtype in ops.LABEL_BYTES
                and (not cfg.use_true_labels or (batch.get("label_pos") is not None and seg.n_classes <= 255
                                                 and batch["label_pos"].dtype in ops.LABEL_BYTES))
                and (not cfg.use_salience or salience.masks_supported(batch.get("mask"), batch.get("mask_pos"),
                                                                      img.shape[0], img.device)))

    def _aug_supported(self, batch) -> bool:
        """The aug-alignment term runs here when the step builds the views itself: seeds and no views, fp32 img at
        cfg.res x cfg.res, seeds readable without a device synchronisation."""
        img, seeds, res = batch["img"], batch.get("seed"), self.seg.cfg.res
        return (seeds is not None and batch.get("img_aug") is None and batch.get("coord_aug") is None
                and not (isinstance(seeds, torch.Tensor) and seeds.is_cuda)
                and img.dtype == torch.float32 and img.dim() == 4 and tuple(img.shape[1:]) == (3, res, res))

    def _rec_crf_supported(self, batch) -> bool:
        """The reconstruction / CRF terms run here only with cfg.fused_rec_crf; the CRF term needs the fp32 image (its
        guidance) and a code of at most 80 channels (stego_crf_loss_*)."""
        cfg = self.seg.cfg
        if cfg.rec_weight == 0 and cfg.crf_weight == 0:
            return True
        return bool(getattr(cfg, "fused_rec_crf", False)) and (
            cfg.crf_weight == 0 or (batch["img"].dtype == torch.float32 and self.seg.net.dim <= 80))

    # ------------------------------------------------------------------------------------------
    def _alloc(self, B, H, W, LH, LW, dev, label_dtype, label_pos_dtype, mask_shape, aug, rec, crf):
        seg, cfg, net = self.seg, self.seg.cfg, self.seg.net
        ws = _Workspace()
        E, D = net.n_feats, net.dim
        fh, fw = H // net.patch_size, W // net.patch_size
        hw = fh * fw
        n_img = 3 if aug else 2  # backbone / head rows: img, img_pos (, img_aug)
        M = n_img * B * hw
        P = _round_up(D, 8)
        spec = seg._spec
        f32, bf = torch.float32, torch.bfloat16
        nonlinear = net.proj_type == "nonlinear"
        ws.dims = (B, E, D, P, fh, fw, hw, M, nonlinear)
        ws.n_img = n_img
        # RNG outputs (img_aug's third noise is drawn, as net(img_aug) draws it, and scales nothing)
        ws.M1 = torch.empty(n_img * B, E, 1, 1, dtype=f32, device=dev)
        ws.M2 = torch.empty(n_img * B, E, 1, 1, dtype=f32, device=dev) if nonlinear else None
        ws.M3 = torch.empty(n_img * B, E, 1, 1, dtype=f32, device=dev) if cfg.dropout else None
        ws.c1 = torch.empty(B, spec.fs, spec.fs, 2, dtype=f32, device=dev)
        ws.c2 = torch.empty(B, spec.fs, spec.fs, 2, dtype=f32, device=dev)
        ws.perms = torch.empty(spec.n_neg, B, dtype=torch.long, device=dev)
        # use_salience: the keep uniforms and, for maps too large for shared memory, the kernel's bitmap scratch
        ws.keep = torch.empty(B, spec.fs, spec.fs, dtype=f32, device=dev) if mask_shape is not None else None
        ws.sal_scratch = salience.scratch_for(B, *mask_shape[-2:], dev) if mask_shape is not None else None
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
        # correspondence loss; the teacher operand is the features, or with use_true_labels the one-hot labels
        ws.ET = corr.teacher_width(seg.n_classes + 1) if cfg.use_true_labels else E
        ws.ftiles = torch.empty(2, spec.nslots, B, spec.rows, ws.ET, dtype=bf, device=dev)
        ws.ctiles = torch.empty(2, spec.nslots, B, spec.rows, corr.CODE_PAD, dtype=bf, device=dev)
        ws.partials, ws.row_means = spec.scratch(B, dev)
        ws.stats = torch.empty(spec.ncalls, 4, dtype=f32, device=dev)
        cw = float(cfg.correspondence_weight)
        wts = [cfg.pos_intra_weight * cw, cfg.pos_inter_weight * cw] + [cfg.neg_inter_weight * cw / spec.n_neg] * spec.n_neg
        ws.call_w = (ctypes.c_float * len(wts))(*[float(v) for v in wts])
        ws.gscale = torch.tensor([float(v) for v in wts], dtype=f32, device=dev)
        # probes
        n_clu = seg.cluster_probe.clusters.shape[0]
        ws.logits = torch.empty(B * hw, 32, dtype=f32, device=dev)
        ws.ce_partials = ops.probe_scratch(dev)
        ws.lin_loss = torch.empty(2, dtype=f32, device=dev)
        ws.clu_loss = torch.empty(2, dtype=f32, device=dev)
        ws.clu_scratch = ops.probe_scratch(dev)
        ws.one = torch.ones(1, dtype=f32, device=dev)
        ws.out4 = torch.empty(4, dtype=f32, device=dev)
        ws.label = torch.empty(B, LH, LW, dtype=label_dtype, device=dev)  # static copy: the tail graph bakes pointers
        ws.label_pos = torch.empty(B, LH, LW, dtype=label_pos_dtype, device=dev) if cfg.use_true_labels else None
        ws.graph = None
        ws.eager_steps = 0
        ws.hist = None        # hist.CdHistogram and the tail graph that fills it, made on the first histogram step
        ws.hist_graph = None
        ws.aug = aug
        if aug:  # the aug-alignment term: the views, the sampled code of img, the cosine and its gradients
            ws.img_aug = torch.empty(B, 3, H, W, dtype=f32, device=dev)  # used until the backbone graph exists
            ws.coord_aug = torch.empty(B, H, W, 2, dtype=f32, device=dev)
            # the view records go up through two pinned host buffers used in turn: one is refilled once the copy made
            # from it two steps earlier has run (enqueued ahead of that step's backbone, so the wait is for work long
            # done), and no pinned block is allocated per step
            ws.rec_host = [torch.empty(B, augment.RECORD_WORDS, dtype=torch.int32).pin_memory() for _ in range(2)]
            ws.rec_copied = [None, None]
            ws.rec_dev = torch.empty(B, augment.RECORD_WORDS, dtype=torch.int32, device=dev)
            ws.aug_scratch = torch.empty(-(-int(_lib.load().stego_aug_scratch_bytes(B, H)) // 8), dtype=torch.float64,
                                         device=dev)
            ws.grid = torch.empty(B, fh, fw, 2, dtype=f32, device=dev)
            ws.sampled = torch.empty(B, D, fh, fw, dtype=f32, device=dev)
            ws.dsampled = torch.empty(B, D, fh, fw, dtype=f32, device=dev)
            ws.cosv, ws.norma, ws.normb = (torch.empty(B, fh, fw, dtype=f32, device=dev) for _ in range(3))
            # d(loss)/d(cos) of loss += w * -(cos.mean()): autograd's fl(fl(-w) / N), one value per pixel
            ws.dcos = torch.full((B, fh, fw), -float(cfg.aug_alignment_weight), dtype=f32, device=dev).div_(B * hw)
            ws.aug_loss = torch.empty(1, dtype=f32, device=dev)
        ws.rec, ws.crf = rec, crf
        if rec:  # the reconstruction term: per-pixel cosine and norms, its gradient, the decoder-gradient partials
            ws.rec_cos, ws.rec_nr, ws.rec_nf = (torch.empty(B * hw, dtype=f32, device=dev) for _ in range(3))
            ws.rec_dcos = torch.full((1,), -float(cfg.rec_weight), dtype=f32, device=dev).div_(B * hw)  # as ws.dcos
            ws.rec_loss = torch.empty(1, dtype=f32, device=dev)
            ws.rec_scratch = modules.rec_scratch(B * hw, E, D, dev)
        if crf:  # the CRF term: the coordinates, the sampled guidance and code, the tile sums
            n = seg.crf_loss_fn.n_samples
            NP = _round_up(n, 64)
            ws.crf_coords = torch.empty(2, n, dtype=torch.long, device=dev)
            ws.crf_gsel = torch.empty(B, NP, 4, dtype=f32, device=dev)
            ws.crf_pos = torch.empty(NP, 2, dtype=torch.int32, device=dev)
            ws.crf_raw = torch.empty(B, D, NP, dtype=f32, device=dev)
            ws.crf_sel = torch.empty(B, D, NP, dtype=f32, device=dev)
            ws.crf_dsel = torch.empty(B, D, NP, dtype=f32, device=dev)
            ws.crf_nrm = torch.empty(B, NP, dtype=f32, device=dev)
            ws.crf_tiles = torch.empty(B, NP // 64, NP // 64, dtype=torch.float64, device=dev)
            # d(loss)/d(out) of loss += w * out.mean(): autograd's fl(fl(w) / (B n^2)), the same for every output
            ws.crf_g = torch.full((1,), float(cfg.crf_weight), dtype=f32, device=dev).div_(B * n * n)
            ws.crf_loss = torch.empty(1, dtype=f32, device=dev)
        # everything the kernels accumulate into: ONE buffer, ONE memset per step
        sizes = dict(dlogits=B * hw * 32, dtiles=spec.nslots * B * spec.rows * corr.DT_LD, dall=M * P,
                     dnc=n_clu * D, db_pad=P)
        total = sum(_round_up(v, 64) for v in sizes.values())
        ws.zbuf = torch.zeros(total, dtype=f32, device=dev)
        off = 0
        for name, n in sizes.items():
            setattr(ws, name, ws.zbuf[off:off + n])
            off += _round_up(n, 64)
        return ws

    # ------------------------------------------------------------------------------------------
    def _prologue(self, ws):
        """Side stream: RNG draws (reference order), operand copies of the trainable weights, accumulator memset."""
        seg, cfg, net = self.seg, self.seg.cfg, self.seg.net
        B, E, D, P, fh, fw, hw, M, nonlinear = ws.dims
        keep = 0.9  # Dropout2d(p=.1), modules.py:41

        def noises(i):  # the i-th net() call of the step: cluster1 noise, cluster2 noise, returned-feature noise
            sl = slice(i * B, (i + 1) * B)
            ws.M1[sl].bernoulli_(keep).div_(keep)
            if nonlinear:
                ws.M2[sl].bernoulli_(keep).div_(keep)
            if ws.M3 is not None:
                ws.M3[sl].bernoulli_(keep).div_(keep)

        noises(0)  # net(img)
        noises(1)  # net(img_pos)
        if ws.keep is not None:  # use_salience (modules.py:357-364): 2B randint calls, reg1, reg2, keep; one kernel
            salience.draw_into(*self._masks, seg._spec.fs, ws.c1, ws.c2, ws.keep, ws.sal_scratch)
        else:
            torch.rand(ws.c1.shape, out=ws.c1).mul_(2).sub_(1)  # modules.py:366-367
            torch.rand(ws.c2.shape, out=ws.c2).mul_(2).sub_(1)
        for i in range(ws.perms.shape[0]):                  # super_perm's randperm (modules.py:291-295)
            torch.randperm(B, device=ws.perms.device, dtype=torch.long, out=ws.perms[i])
        if ws.aug:
            noises(2)  # net(img_aug), after the correspondence loss (train_segmentation.py:189-190)
        if ws.crf:  # ContrastiveCRFLoss.draw_coords on the 56 x 56 maps: rows, then columns (train_segmentation.py:201-208)
            for i in range(2):
                torch.randint(0, modules.CRF_SIDE, (1, ws.crf_coords.shape[1]), out=ws.crf_coords[i:i + 1])
        w1, _, wa, _, wb, _ = net.head_params()
        modules.pack_head_weights(w1, wa, wb, ws.w1p, ws.wab, ws.wbp)
        ws.zbuf.zero_()
        seg._flat.grad.zero_()

    # ------------------------------------------------------------------------------------------
    def _tail(self, ws, tok_all, hist=None):
        """Head forward .. head backward on the current stream: static workspace, no allocation, no RNG, no host
        synchronisation — captured as one CUDA graph after the first (eager) step.  hist: the correlation forward also
        bins the cd histograms into it (a second graph, for the steps that log them)."""
        seg, net = self.seg, self.seg.net
        B, E, D, P, fh, fw, hw, M, nonlinear = ws.dims
        spec = seg._spec
        params = net.head_params()
        _, b1, _, ba, _, bb = params
        # [nB, C, h, w] views of the tokens-major features and of the padded code storage: img rows, then img_pos rows
        # (, then img_aug rows)
        n = ws.n_img
        feats = tok_all.view(n * B, fh, fw, E).permute(0, 3, 1, 2)
        code = ws.code.view(n * B, fh, fw, P)[..., :D].permute(0, 3, 1, 2)
        img_rows, pos_rows, aug_rows = slice(0, B), slice(B, 2 * B), slice(2 * B, 3 * B)

        # ---- head forward (modules.py:108-111)
        modules.head_forward(tok_all.reshape(M, E), ws.M1, ws.M2, n * B, hw, ws.x1, ws.x2, ws.hid, ws.code, ws.w1p, b1,
                             ws.wab, ba, ws.wbp, bb)
        seg._mark("head_forward")

        # ---- correspondence loss forward (modules.py:349-398)
        if ws.label_pos is not None:  # use_true_labels (train_segmentation.py:135-137)
            corr.build_label_tiles(ws.label, ws.label_pos, ws.c1, ws.c2, ws.perms, spec, seg.n_classes, raw_perms=True,
                                   out=ws.ftiles)
        else:
            m3, p3 = (ws.M3[img_rows], ws.M3[pos_rows]) if ws.M3 is not None else (None, None)
            corr.build_tiles(feats[img_rows], feats[pos_rows], ws.c1, ws.c2, ws.perms, spec, E, m3, p3, raw_perms=True,
                             out=ws.ftiles)
        corr.build_tiles(code[img_rows], code[pos_rows], ws.c1, ws.c2, ws.perms, spec, corr.CODE_PAD, raw_perms=True,
                         out=ws.ctiles)
        spec.forward(ws.ftiles, ws.ctiles, B, ws.ET, D, ws.partials, ws.row_means, ws.stats, hist=hist)
        if ws.aug:  # -cosine(sample(code, coord), code_aug) (train_segmentation.py:189-199)
            modules.aug_sample_forward(ws.coord_aug, code[img_rows], ws.grid, ws.sampled)
            modules.cosine_forward(ws.sampled, code[aug_rows], ws.cosv, ws.norma, ws.normb)
        m3_img = ws.M3[img_rows] if ws.M3 is not None else None
        dec = seg.decoder
        if ws.rec:  # -cosine(decoder(code), feats * m3) (train_segmentation.py:183-187)
            modules.rec_forward(ws.code[:B * hw], tok_all[:B].reshape(B * hw, E), m3_img, hw, dec.weight, dec.bias,
                                ws.rec_cos, ws.rec_nr, ws.rec_nf)
        if ws.crf:  # crf_loss_fn(resize(img, 56), norm(resize(code, 56))) at the samples (train_segmentation.py:201-208)
            crf_p = modules.crf_params(seg.crf_loss_fn)
            modules.crf_forward(code[img_rows], ws.crf_coords, crf_p, ws.crf_gsel, ws.crf_pos, ws.crf_raw, ws.crf_sel,
                                ws.crf_nrm, ws.crf_tiles)
        seg._mark("corr_loss_forward")

        # ---- probes on the detached code (train_segmentation.py:213-225): forward + backward in place
        lp, cl = seg.linear_probe, seg.cluster_probe.clusters
        segmenter.linear_probe_ce_step(code[:B], lp.weight, lp.bias, ws.label, ws.logits, ws.dlogits, ws.ce_partials,
                                       ws.lin_loss, lp.weight.grad, lp.bias.grad, 1.0)
        modules.cluster_lookup_forward(code[:B], cl, None, ws.clu_loss, ws.clu_scratch)
        _lib.check(_lib.load().stego_step_losses(_lib.ptr(ws.stats), spec.ncalls, ws.call_w, _lib.ptr(ws.lin_loss),
                                                 _lib.ptr(ws.clu_loss), _lib.ptr(ws.out4), _lib.stream()),
                   "stego_step_losses")
        if ws.rec:  # loss/rec, and its weighted value onto the total
            modules.aug_loss(ws.rec_cos, seg.cfg.rec_weight, ws.rec_loss, ws.out4)
        if ws.aug:  # loss/aug_alignment, and its weighted value onto the total
            modules.aug_loss(ws.cosv, seg.cfg.aug_alignment_weight, ws.aug_loss, ws.out4)
        if ws.crf:  # loss/crf, and its weighted value onto the total
            modules.crf_loss(ws.crf_tiles, ws.crf_coords.shape[1], seg.cfg.crf_weight, ws.crf_loss, ws.out4)
        seg._mark("probes_forward")

        # ---- backward (manual_backward, :227)
        modules.cluster_lookup_backward(code[:B], cl, None, ws.one, ws.dnc, cl.grad)
        spec.backward(ws.ftiles, ws.ctiles, B, ws.ET, D, ws.stats, ws.row_means, ws.gscale, None, None, ws.dtiles)
        dall = ws.dall.view(M, P)
        corr.sample_norm_backward(code[img_rows], code[pos_rows], ws.c1, ws.c2, ws.perms, spec, ws.dtiles,
                                  dall[:B * hw], dall[B * hw:2 * B * hw], raw_perms=True)
        dcode = dall.view(n * B, fh, fw, P)[..., :D].permute(0, 3, 1, 2)
        if ws.aug:  # d(code_aug) into the img_aug rows, d(sampled) scattered into the img rows
            modules.cosine_backward(ws.sampled, code[aug_rows], ws.cosv, ws.norma, ws.normb, ws.dcos, ws.dsampled,
                                    dcode[aug_rows])
            modules.aug_sample_backward(ws.grid, ws.dsampled, dcode[img_rows])
        if ws.rec:  # d(code) into the img rows; the decoder's gradient straight into the flat gradient buffer
            modules.rec_backward(ws.code[:B * hw], tok_all[:B].reshape(B * hw, E), m3_img, hw, dec.weight, dec.bias,
                                 ws.rec_cos, ws.rec_nr, ws.rec_nf, ws.rec_dcos, dall[:B * hw], ws.rec_scratch,
                                 dec.weight.grad, dec.bias.grad)
        if ws.crf:  # d(code) scattered into the img rows
            modules.crf_backward(ws.crf_g, ws.crf_sel, ws.crf_nrm, ws.crf_gsel, ws.crf_pos, ws.crf_coords, crf_p,
                                 ws.crf_dsel, dcode[img_rows])
        # head backward: d(code) [M, P] -> bias / weight gradients straight into the flat gradient buffer
        modules.head_backward(dall, ws.x1, ws.x2, ws.hid, ws.wbp, ws.dyb, ws.db_pad, ws.dh, ws.dhb,
                              *[p.grad if p is not None else None for p in params])

    # ------------------------------------------------------------------------------------------
    def run(self, batch):
        seg, cfg, net = self.seg, self.seg.cfg, self.seg.net
        img, img_pos, label = batch["img"], batch["img_pos"], batch["label"]
        dev = img.device
        B, _, H, W = img.shape
        LH, LW = label.shape[-2], label.shape[-1]
        if seg._flat is None:
            seg.configure_optimizers()
        seg._flat.ensure_bound()  # parameters / .grad still are the views into the flat buffers the kernels write
        net_optim, linear_probe_optim, cluster_probe_optim = seg.optimizers()
        label_pos = batch["label_pos"] if cfg.use_true_labels else None
        mask = batch["mask"] if cfg.use_salience else None
        aug = cfg.aug_alignment_weight > 0
        rec, crf = cfg.rec_weight > 0, cfg.crf_weight > 0  # supported() admitted them only with cfg.fused_rec_crf
        if aug:  # the host draws of the views come first: they overlap the previous step's work on the device
            seeds = augment._check(img, augment.batch_seeds(batch["seed"]), cfg.res)
            _, records = augment.draw_records(seeds, H, W)
        # a new flat parameter buffer (or another label dtype) invalidates the captured graph
        key = (B, H, W, LH, LW, dev.index, id(seg._flat), label.dtype,
               label_pos.dtype if label_pos is not None else None,
               (tuple(mask.shape), mask.dtype, batch["mask_pos"].dtype) if mask is not None else None, aug, rec, crf)
        if self.key != key:
            self.flush()
            self.ws = self._alloc(B, H, W, LH, LW, dev, label.dtype, key[-5], key[-4][0] if mask is not None else None,
                                  aug, rec, crf)
            self.key = key
            self.side = torch.cuda.Stream(device=dev)
        ws = self.ws
        B, E, D, P, fh, fw, hw, M, nonlinear = ws.dims
        spec = seg._spec
        main = torch.cuda.current_stream()
        seg._mark("start")

        # ---- side stream: [gradient all-reduce + Adam of the PREVIOUS step, enqueued at the end of that step] ->
        #      prologue of this step.  The frozen ViT on the main stream depends on neither, so the whole update
        #      (the one collective of the data-parallel step included) is hidden under the next step's backbone.
        self.side.wait_stream(main)
        self._masks = (batch["mask"], batch["mask_pos"]) if ws.keep is not None else None
        ready = torch.cuda.Event()

        def prologue():
            with torch.cuda.stream(self.side):
                self._prologue(ws)
                ready.record(self.side)

        # with use_salience the prologue waits on the host for the mask counts (salience.draw_into): it goes after the
        # backbone is enqueued, so that wait overlaps the ViT (which draws nothing from the generators)
        if ws.keep is None:
            prologue()

        use_graph = bool(getattr(cfg, "cuda_graph", True)) and seg.profile_marks is None
        overlap = bool(getattr(cfg, "overlap_update", True)) and seg.profile_marks is None
        with torch.no_grad():
            parts = [img, img_pos]
            if aug:
                # the views go straight into the backbone graph's input once that graph exists (no copy)
                img_aug = ws.img_aug
                if getattr(cfg, "cuda_graph", True):
                    static_in = net.model.graph_input(net.feat_type, (3 * B, 3, H, W), dev)
                    img_aug = static_in[2 * B:] if static_in is not None else img_aug
                i = self.step_idx % 2
                if ws.rec_copied[i] is not None:
                    ws.rec_copied[i].synchronize()
                ws.rec_host[i].copy_(records)
                ws.rec_dev.copy_(ws.rec_host[i], non_blocking=True)
                ws.rec_copied[i] = torch.cuda.Event()
                ws.rec_copied[i].record(main)
                augment.launch(img, ws.rec_dev, H, img_aug, ws.coord_aug, ws.aug_scratch)
                parts.append(img_aug)
            tok_all = net.backbone_tokens(parts, use_graph=getattr(cfg, "cuda_graph", True))  # [nB, hw, E] bf16
            if ws.keep is not None:
                prologue()
            ws.label.copy_(label.reshape(B, LH, LW))
            if label_pos is not None:
                ws.label_pos.copy_(label_pos.reshape(B, LH, LW))
            main.wait_event(ready)
            if ws.crf:  # the guidance from this step's img, outside the tail graph (which bakes no caller pointer)
                modules.crf_guidance(img, ws.crf_coords, ws.crf_gsel, ws.crf_pos)
            seg._mark("vit_forward")
            if seg.should_log_hist():
                # histogram steps replay a tail graph of their own (captured the first time one is needed), so the
                # graph of every other step stays what it is
                if ws.hist is None:
                    from .hist import CdHistogram
                    ws.hist = CdHistogram(spec, B, dev)
                if use_graph and ws.hist_graph is not None and ws.hist_graph[1] == tok_all.data_ptr():
                    ws.hist_graph[0].replay()
                elif use_graph and ws.eager_steps >= 1:
                    ws.hist_graph = (_lib.Graph(lambda: self._tail(ws, tok_all, ws.hist)), tok_all.data_ptr())
                    ws.hist_graph[0].replay()
                else:
                    self._tail(ws, tok_all, ws.hist)
                seg._stage_histograms(ws.hist)
            elif use_graph and ws.graph is not None and ws.graph[1] == tok_all.data_ptr():
                ws.graph[0].replay()
            elif use_graph and ws.eager_steps >= 1:
                # second step on this shape: capture head fwd .. head bwd (static workspace, no allocation, no RNG) as ONE
                # CUDA graph; the eager first step has already set kernel attributes and warmed the allocator
                ws.graph = (_lib.Graph(lambda: self._tail(ws, tok_all)), tok_all.data_ptr())
                ws.graph[0].replay()
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
        if ws.rec:
            seg.log('loss/rec', ws.rec_loss[0])
        if ws.aug:
            seg.log('loss/aug_alignment', ws.aug_loss[0])
        if ws.crf:
            seg.log('loss/crf', ws.crf_loss[0])
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
