"""fp64 references of the correspondence-loss kernels (csrc/corr_loss.cu, driven by stego_b200/corr.py), shared by the
correspondence-loss tests.

Plain torch and device-agnostic: the GPU tests run these in float64 on the device, one (call, image) block of [S, S]
at a time (at feature_samples = 64 one fp64 block is 134 MB), and the CPU test pins them to the oracle
(oracle/stego_oracle.py) and to fp64 autograd through it.  Every value comes with the bar the GPU test holds the kernel
to, built from per-element sums of |terms|; the constants are derived in tests/test_corr_fp64_gpu.py.

The bilinear taps are computed with the kernels' own fp32 coordinate arithmetic (make_taps: ((c + 1) / 2) (W - 1),
clamp, floor, four weight products, a clamped last row / column with zero weights), emulated in torch fp32, which is
IEEE round-to-nearest, so reference and kernel use the same taps and the same weights.  Everything after the taps is
float64.  The backward is written out analytically: the autograd graph of [ncalls, B, S, S] fp64 tensors at
feature_samples = 64 does not fit sensibly.
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if os.path.join(ROOT, "oracle") not in sys.path:
    sys.path.insert(0, os.path.join(ROOT, "oracle"))

U = 2.0 ** -24           # unit roundoff of fp32
SPLIT = 2.0 ** -16       # |x - hi - lo| <= SPLIT |x| for the bf16 hi/lo split, and |lo_a lo_b| <= SPLIT |a b|
EPS = 1e-10              # l2 normalisation floor (modules.py:275-276; SampleParams.eps)
HI = float(torch.tensor(0.8, dtype=torch.float32))  # the stabalize bound as the kernels hold it: 0.8 rounded to fp32
TILE = 128               # rows of a tile and padded code channels


def taps(coords, H, W):
    """coords [B, fs, fs, 2] -> (idx [B, S, 4] long, w [B, S, 4] float64) for sample s = i fs + j, which reads
    coords[b, j, i] (modules.py:288 permutes the grid).  Taps in the order nw, ne, sw, se as make_taps."""
    B, fs = coords.shape[0], coords.shape[1]
    c = coords.detach().float().permute(0, 2, 1, 3).reshape(B, fs * fs, 2)
    x = ((c[..., 0] + 1.0) / 2.0) * float(W - 1)
    y = ((c[..., 1] + 1.0) / 2.0) * float(H - 1)
    x = x.clamp(0.0, float(W - 1))
    y = y.clamp(0.0, float(H - 1))
    x0, y0 = x.floor(), y.floor()
    x1, y1 = x0 + 1.0, y0 + 1.0
    w00, w01 = (x1 - x) * (y1 - y), (x - x0) * (y1 - y)
    w10, w11 = (x1 - x) * (y - y0), (x - x0) * (y - y0)
    ix0, iy0 = x0.long(), y0.long()
    ix1, iy1 = ix0 + 1, iy0 + 1
    cx, cy = ix1 > W - 1, iy1 > H - 1
    ix1, iy1 = torch.where(cx, W - 1, ix1), torch.where(cy, H - 1, iy1)
    zero = torch.zeros_like(w00)
    w01, w11 = torch.where(cx, zero, w01), torch.where(cx, zero, w11)
    w10, w11 = torch.where(cy, zero, w10), torch.where(cy, zero, w11)
    idx = torch.stack([iy0 * W + ix0, iy0 * W + ix1, iy1 * W + ix0, iy1 * W + ix1], -1)
    return idx, torch.stack([w00, w01, w10, w11], -1).double()


def gather_sample(src, img, idx, w, cs=None):
    """Bilinear sample of src[img[b]] ([B, C, H, W], any float dtype) at the taps of image b: (v [B, S, C] float64,
    A [B, S, C] = sum_t |src_t| w_t |cs|, the magnitude the fp32 4-tap sum rounds against)."""
    B, C = img.shape[0], src.shape[1]
    flat = src.detach().double().reshape(src.shape[0], C, -1)[img]
    S = idx.shape[1]
    v = torch.zeros(B, C, S, dtype=torch.float64, device=src.device)
    A = torch.zeros_like(v)
    for t in range(4):
        vt = flat.gather(2, idx[:, None, :, t].expand(B, C, S))
        v += vt * w[:, None, :, t]
        A += vt.abs() * w[:, None, :, t]
    if cs is not None:
        s = cs.detach().double()[img][..., None]
        v, A = v * s, A * s.abs()
    return v.transpose(1, 2), A.transpose(1, 2)


def chain_norm(C, vec8=False):
    """fp32 chain length of the sum of squares in the sampling kernels: the per-lane terms, the warp butterfly, +1"""
    cpad = -(-C // 64) * 64
    per_lane = 8 * (-(-C // 256)) if vec8 else cpad // 32
    return max(per_lane, cpad // 32) + 6


def normalise(v, A, L):
    """v / max(|v|, eps) and its bar.  The fp32 4-tap sum (and the chan_scale product) is off by <= 5 u A per channel
    (delta); the sum of squares is an L-term chain, then sqrt and the reciprocal round once each and x * inv once:
      |v| > eps : E_n = delta / |v| + |n| eta, eta = sum_c |v_c| delta_c / |v|^2 + (L / 2 + 3) u
      otherwise : E_n = delta / eps + u |n|
    Returns (n, E_n, |v|)."""
    nrm = v.norm(dim=-1, keepdim=True)
    den = nrm.clamp_min(EPS)
    n = v / den
    delta = 5 * U * A
    eta = (v.abs() * delta).sum(-1, keepdim=True) / den ** 2 + (L / 2 + 3) * U
    E = torch.where(nrm > EPS, delta / den + n.abs() * eta, delta / EPS + U * n.abs())
    return n, E, nrm


def resolve_perms(perms, B, raw):
    """[n_neg, B] image index of each negative slot; raw randperm draws get super_perm's fix-up (modules.py:291-295)"""
    if perms is None:
        return None
    p = perms if torch.is_tensor(perms) else torch.stack(list(perms))
    p = p.long().clone()
    if raw:
        ar = torch.arange(B, device=p.device)
        p = torch.where(p == ar, (p + 1) % B, p)
    return p


class CorrRef:
    """fp64 ContrastiveCorrelationLoss of the kernels' call layout: call 0 intra (slot 0 vs slot 0), call 1 inter (slot 0
    vs slot 1), call 2 + k negative k (slot 0 vs slot 2 + k).  Slot 0 samples img / code at coords1, slot 1 img_pos /
    code_pos at coords2, slot 2 + k img[perm_k] / code[perm_k] at coords2; chan_scale multiplies the feature samples.

    cfg: anything with pointwise, zero_clamp, stabalize, feature_samples, neg_samples and the three shifts.
    vec8: the feature tiles come from sample_norm_vec8_kernel (only the sum-of-squares chain length differs).
    hi: the stabalize clamp bound, 0.8 in fp32 as the kernels hold it (the fp64 oracle clamps at 0.8 in fp64).
    The teacher feats may lie on another grid than the code (the one-hot label maps of use_true_labels, at label
    resolution): each is sampled with the taps of its own size, at the same normalised coordinates."""

    def __init__(self, feats, feats_pos, code, code_pos, coords1, coords2, perms, cfg, chan_scale=None,
                 chan_scale_pos=None, raw_perms=False, vec8=False, hi=HI):
        self.cfg = cfg
        self.B, self.E = feats.shape[:2]
        self.D, self.H, self.W = code.shape[1:]
        FH, FW = feats.shape[2:]
        self.fs = int(cfg.feature_samples)
        self.S = self.fs * self.fs
        self.n_neg = int(cfg.neg_samples)
        self.nslots = self.ncalls = 2 + self.n_neg
        self.slot_of_call = list(range(self.ncalls))
        self.shifts = [cfg.pos_intra_shift, cfg.pos_inter_shift] + [cfg.neg_inter_shift] * self.n_neg
        self.lo = 0.0 if cfg.zero_clamp else -9999.0
        self.hi = hi if cfg.stabalize else float("inf")
        self.pointwise = bool(cfg.pointwise)
        self.tiled = self.S > TILE
        self.nT = -(-self.S // TILE) if self.tiled else 1
        self.dev = feats.device
        B = self.B
        ar = torch.arange(B, device=self.dev)
        pr = resolve_perms(perms, B, raw_perms) if self.n_neg else None
        t1, t2 = taps(coords1, self.H, self.W), taps(coords2, self.H, self.W)
        f1, f2 = (t1, t2) if (FH, FW) == (self.H, self.W) else (taps(coords1, FH, FW), taps(coords2, FH, FW))
        self.code, self.code_pos = code, code_pos
        # per slot: (image of each b, code taps, feature source, code source, chan_scale, feature taps)
        self.slots = [(ar, t1, feats, code, chan_scale, f1), (ar, t2, feats_pos, code_pos, chan_scale_pos, f2)]
        for k in range(self.n_neg):
            self.slots.append((pr[k].to(self.dev), t2, feats, code, chan_scale, f2))
        Lf, Lc = chain_norm(self.E, vec8), chain_norm(self.D)
        self.fn, self.fE, self.cn, self.cE, self.cv, self.cA, self.cnrm = [], [], [], [], [], [], []
        for img, (idx, w), fsrc, csrc, cs, (fidx, fw) in self.slots:
            v, A = gather_sample(fsrc, img, fidx, fw, cs)
            n, E, _ = normalise(v, A, Lf)
            self.fn.append(n)
            self.fE.append(E)
            v, A = gather_sample(csrc, img, idx, w)
            n, E, nrm = normalise(v, A, Lc)
            self.cn.append(n)
            self.cE.append(E)
            self.cv.append(v)
            self.cA.append(A)
            self.cnrm.append(nrm)
        # chain lengths: fp32 partial sums of the forward reductions (single tile: 64 elements per thread + warp + 8
        # warps; multi-tile: 32 per thread + 2 shuffles per row of a tile), the row sum of fd
        self.L_red = 40 if self.tiled else 80
        self.L_row = 34

    # --------------------------------------------------------------------------------------------
    def _einsum(self, a, Ea, b, Eb, K):
        """a . b^T of normalised samples and its bar: operand bars plus the split (E + SPLIT |x| per operand), the dropped
        lo . lo term (SPLIT), and a (K + 2)-term fp32 accumulation chain over the three split passes."""
        val = a @ b.T
        M = a.abs() @ b.abs().T
        E = (Ea + SPLIT * a.abs()) @ b.abs().T + a.abs() @ (Eb + SPLIT * b.abs()).T + (SPLIT + (K + 2) * U) * M
        return val, E

    def block(self, k, b):
        """fd, cd and their bars for call k, image b; centred fd and the row means (0 when not pointwise)."""
        sB = self.slot_of_call[k]
        fd, Efd = self._einsum(self.fn[0][b], self.fE[0][b], self.fn[sB][b], self.fE[sB][b], 3 * self.E)
        cd, Ecd = self._einsum(self.cn[0][b], self.cE[0][b], self.cn[sB][b], self.cE[sB][b], 3 * TILE)
        S = self.S
        if self.pointwise:
            m = fd.mean(1, keepdim=True)
            Em = Efd.mean(1, keepdim=True) + self.L_row * U * fd.abs().mean(1, keepdim=True) + 2 * U * m.abs()
        else:
            m = torch.zeros(S, 1, dtype=fd.dtype, device=fd.device)
            Em = torch.zeros_like(m)
        fdc = fd - m
        Efdc = Efd + Em + U * fdc.abs()
        cl = cd.clamp(self.lo, self.hi)
        return dict(fd=fd, Efd=Efd, cd=cd, Ecd=Ecd, m=m, Em=Em, fdc=fdc, Efdc=Efdc, cl=cl)

    def forward(self):
        """Per-call stats.  offset = old_mean - mean(centred fd), batch-global per call; loss = mean of
        -cl (fdc + offset - shift).  Bars: cl is 1-Lipschitz in cd, so |cl - cl_ref| <= E_cd with no kink rule."""
        n = self.B * self.S * self.S
        L = self.L_red
        self.stats = []
        for k in range(self.ncalls):
            sh = self.shifts[k]
            acc = dict.fromkeys(("fd", "fdc", "cl_fdcs", "cl", "cd", "Efd", "Efdc", "afd", "afdm", "Ecd", "acd",
                                 "E0", "Lcl", "acl"), 0.0)
            for b in range(self.B):
                x = self.block(k, b)
                fd, fdc, cl, cd = x["fd"], x["fdc"], x["cl"], x["cd"]
                acc["fd"] += fd.sum().item()
                acc["fdc"] += fdc.sum().item()
                acc["cl_fdcs"] += (cl * (fdc - sh)).sum().item()
                acc["cl"] += cl.sum().item()
                acc["cd"] += cd.sum().item()
                acc["Efd"] += x["Efd"].sum().item()
                acc["Efdc"] += x["Efdc"].sum().item()
                acc["afd"] += fd.abs().sum().item()
                afdm = fd.abs() + x["m"].abs()
                acc["afdm"] += afdm.sum().item()
                acc["Ecd"] += x["Ecd"].sum().item()
                acc["acd"] += cd.abs().sum().item()
                acc["E0"] += ((fdc - sh).abs() * x["Ecd"] + cl.abs() * x["Efdc"]).sum().item()
                acc["Lcl"] += (cl.abs() * (afdm + abs(sh))).sum().item()
                acc["acl"] += cl.abs().sum().item()
                del x
            old, mc = acc["fd"] / n, acc["fdc"] / n
            off = (old - mc) if self.pointwise else 0.0
            E_old = acc["Efd"] / n + L * U * acc["afd"] / n
            E_mc = acc["Efdc"] / n + L * U * acc["afdm"] / n
            E_off = (E_old + E_mc + 2 * U * (abs(old) + abs(mc))) if self.pointwise else 0.0
            loss = -(acc["cl_fdcs"] + off * acc["cl"]) / n
            E0 = acc["E0"] + L * U * acc["Lcl"]
            E1 = acc["Ecd"] + L * U * acc["acl"]
            E_loss = (E0 + abs(off) * E1 + abs(acc["cl"]) * E_off) / n + U * abs(loss)
            cdm = acc["cd"] / n
            E_cdm = acc["Ecd"] / n + L * U * acc["acd"] / n + U * abs(cdm)
            self.stats.append(dict(loss=loss, E_loss=E_loss, cd_mean=cdm, E_cd_mean=E_cdm, old_mean=old, mean_c=mc,
                                   offset=off, E_off=E_off, loss_abs=acc["Lcl"] / n))
        return self.stats

    def elems(self, k, x):
        """Loss elements -cl (fdc + offset - shift) of a block and their bar (two fp32 adds and a product)."""
        st, sh = self.stats[k], self.shifts[k]
        t = x["fdc"] + st["offset"] - sh
        e = -x["cl"] * t
        E = t.abs() * x["Ecd"] + x["cl"].abs() * (x["Efdc"] + st["E_off"]) + \
            3 * U * x["cl"].abs() * (x["fdc"].abs() + abs(st["offset"]) + abs(sh))
        return e, E

    def backward(self, glosses, gelem=None, gcd=None, visit=None):
        """d code, d code_pos for upstream weights glosses [ncalls] on the call means, gelem / gcd [ncalls, B, S, S]
        (any device / dtype) on the loss elements and on cd.  visit(k, b, block) sees every block with its loss elements
        (block["elem"], block["Eelem"]) before it is dropped.

          G    = -up (fdc + offset - shift) 1[lo <= cd <= hi] + gcd,  up = glosses[k] / (B S S) + gelem
          dA   = G . B_c (slot 0), dB = G^T . A_c (the call's slot; slot 0 again for the intra call)
        Bars: E_G from fdc, offset and up (five fp32 roundings), G's own split (SPLIT |G|) and its final add; inside the
        band |cd - bound| < E_cd the kernel may take either side of the clamp, so |up (fdc + offset - shift)| is added to
        E_G there, and through E_G to the bar of every row the element touches.  The gradient tiles sum
        3 * 128-term wgmma chains and 2 ncalls nT fp32 read-modify-writes: L_b = 384 + 2 ncalls nT + 2."""
        n = self.B * self.S * self.S
        D, S = self.D, self.S
        g = [torch.zeros(self.B, S, D, dtype=torch.float64, device=self.dev) for _ in range(self.nslots)]
        Eg = [torch.zeros_like(t) for t in g]
        Lb = 3 * TILE + 2 * self.ncalls * self.nT + 2
        self.band_count = 0
        for k in range(self.ncalls):
            st, sh, sB = self.stats[k], self.shifts[k], self.slot_of_call[k]
            gs = float(glosses[k]) / n
            for b in range(self.B):
                x = self.block(k, b)
                up = torch.full_like(x["fd"], gs)
                if gelem is not None:
                    up = up + gelem[k, b].to(self.dev).double()
                cd, fdc = x["cd"], x["fdc"]
                t = fdc + st["offset"] - sh
                pas = (cd >= self.lo) & (cd <= self.hi)
                band = ((cd - self.lo).abs() < x["Ecd"]) | ((cd - self.hi).abs() < x["Ecd"])
                self.band_count += int(band.sum())
                Gk = -up * t
                G = torch.where(pas, Gk, torch.zeros_like(Gk))
                EG = torch.where(pas, up.abs() * (x["Efdc"] + st["E_off"]) + 2 * U * (up.abs() + abs(gs)) * t.abs() +
                                 5 * U * up.abs() * (x["fd"].abs() + x["m"].abs() + abs(st["offset"]) + abs(sh)),
                                 torch.zeros_like(Gk))
                EG = EG + torch.where(band, Gk.abs(), torch.zeros_like(Gk))
                if gcd is not None:
                    gc = gcd[k, b].to(self.dev).double()
                    G = G + gc
                    EG = EG + U * gc.abs()
                EG = EG + (2 * U + SPLIT) * G.abs()
                if visit is not None:
                    x["elem"], x["Eelem"] = self.elems(k, x)
                    x["G"], x["EG"], x["band"] = G, EG, band
                    visit(k, b, x)
                del x
                for (dst, other, sa) in ((0, sB, False), (sB, 0, True)):
                    Gm = G.T if sa else G
                    EGm = EG.T if sa else EG
                    c, Ec = self.cn[other][b], self.cE[other][b]
                    g[dst][b] += Gm @ c
                    Eg[dst][b] += EGm @ c.abs() + Gm.abs() @ (Ec + SPLIT * c.abs()) + \
                        (SPLIT + Lb * U) * (Gm.abs() @ c.abs())
        self.g, self.Eg = g, Eg
        return self._sample_backward(g, Eg)

    def _sample_backward(self, g, Eg):
        """normalise backward (fp32, sample_dv) and the bilinear gather into d code / d code_pos.
          |v| > eps : dv = (g - v (v . g) / |v|^2) / |v|, bar from E_g, the tap error delta = 5 u A of v, the L-term
                      dot and norm chains (L = 10: three channels per lane + warp butterfly);
          otherwise : dv = g / eps, bar E_g / eps + u |dv|.
        d code[pixel] sums w dv over the samples whose non-zero tap hits the pixel, in a chain of hits + 2 roundings."""
        L = 10
        B, D, HW = self.B, self.D, self.H * self.W
        z = lambda c: torch.zeros(B * HW, c, dtype=torch.float64, device=self.dev)  # pixel-major accumulators
        out, Eo, Ao, hits = ({False: z(c), True: z(c)} for c in (D, D, D, 1))
        self.dv, self.Edv = [], []
        for s, (img, (idx, w), _, _, _, _) in enumerate(self.slots):
            v, A, nrm, gg, Eg_ = self.cv[s], self.cA[s], self.cnrm[s], g[s], Eg[s]
            delta = 5 * U * A
            den = nrm.clamp_min(EPS)
            dot = (v * gg).sum(-1, keepdim=True)
            p = v * dot / den ** 2
            dv_n = (gg - p) / den
            E_dot = (v.abs() * Eg_).sum(-1, keepdim=True) + (gg.abs() * delta).sum(-1, keepdim=True) + \
                (L + 1) * U * (v * gg).abs().sum(-1, keepdim=True)
            en = (v.abs() * delta).sum(-1, keepdim=True) / den ** 2 + (L / 2 + 2) * U
            Ep = delta * dot.abs() / den ** 2 + v.abs() * E_dot / den ** 2 + p.abs() * (2 * en + 4 * U)
            Edv_n = (Eg_ + Ep + U * (gg.abs() + p.abs())) / den + dv_n.abs() * (en + 2 * U)
            dv_e = gg / EPS
            big = nrm > EPS
            dv = torch.where(big, dv_n, dv_e)
            Edv = torch.where(big, Edv_n, Eg_ / EPS + U * dv_e.abs())
            self.dv.append(dv)
            self.Edv.append(Edv)
            pos = s == 1
            for t in range(4):
                wt = w[:, :, t]
                ix = (img[:, None] * HW + idx[:, :, t]).reshape(-1)
                for tgt, val in ((out, dv * wt[..., None]), (Eo, Edv * wt[..., None]), (Ao, (dv * wt[..., None]).abs()),
                                 (hits, (wt != 0).double()[..., None])):
                    tgt[pos].index_add_(0, ix, val.reshape(ix.shape[0], -1))
        nchw = lambda t: t.view(B, self.H, self.W, -1).permute(0, 3, 1, 2)
        res = []
        for pos in (False, True):
            bar = Eo[pos] + (hits[pos] + 2) * U * Ao[pos]
            res.append((nchw(out[pos]), nchw(bar)))
        self.hits = (nchw(hits[False]), nchw(hits[True]))
        self.Ao = (nchw(Ao[False]), nchw(Ao[True]))  # sum |w dv| per element: what its fp32 accumulator rounds against
        return res


# ------------------------------------------------------------------------------------------------
# input builders: each regime makes one kind of kernel bug move the outputs by O(1)
# ------------------------------------------------------------------------------------------------
def lowrank_maps(B, C, h, w, g, rank=16, noise=0.1):
    """production-like maps: correlated low-rank channels plus noise (NCHW fp32)"""
    basis = torch.randn(rank, C, generator=g)
    mix = torch.randn(B, h, w, rank, generator=g)
    return (mix @ basis + noise * torch.randn(B, h, w, C, generator=g)).permute(0, 3, 1, 2).contiguous()


def centre_coord(k, n):
    """an fp32 grid coordinate whose make_taps source coordinate is exactly pixel k of an axis of n pixels"""
    c0 = torch.tensor(2.0 * k / (n - 1) - 1.0, dtype=torch.float32)
    cands = [c0]
    for d in (float("inf"), float("-inf")):
        c = c0
        for _ in range(256):
            c = torch.nextafter(c, torch.tensor(d))
            cands.append(c)
    for c in sorted(cands, key=lambda t: abs(t.item() - c0.item())):
        if (((c + 1.0) / 2.0) * float(n - 1)).item() == k:
            return float(c)
    return None  # no fp32 coordinate lands exactly on this pixel


def centres(n):
    """(pixels, coordinates) of the pixels of an n-pixel axis that an fp32 coordinate hits exactly (always 0 and n - 1)"""
    ks = [k for k in range(n) if centre_coord(k, n) is not None]
    return torch.tensor(ks), torch.tensor([centre_coord(k, n) for k in ks])


def centre_grid(B, fs, H, W, g, last=False):
    """[B, fs, fs, 2] coordinates on pixel centres (all bilinear weights 0 or 1); last=True puts every sample of the
    first row of samples on the last column and of the first column on the last row"""
    (_, tx), (_, ty) = centres(W), centres(H)
    xs = torch.randint(0, len(tx), (B, fs, fs), generator=g)
    ys = torch.randint(0, len(ty), (B, fs, fs), generator=g)
    if last:
        xs[:, :, 0] = len(tx) - 1
        ys[:, 0, :] = len(ty) - 1
    return torch.stack([tx[xs], ty[ys]], -1)


def make_inputs(regime, B, E, D, H, W, fs, n_neg, seed=0):
    """CPU fp32 inputs of one regime: feats, feats_pos [B, E, H, W], code, code_pos [B, D, H, W], coords1, coords2
    [B, fs, fs, 2], raw randperm draws [n_neg, B] (with fixed points), chan_scale / chan_scale_pos [B, E] or None.

      corr   production-like correlated low-rank maps, uniform coordinates x 1.2 (some beyond +-1)
      flat   every image's features one shared direction plus 1e-2 noise: fd ~ 1, centred fd ~ 1e-4
      kinks  one-hot codes in channels 0 / 1 and the code (0.8, 0.6) / 5 at pixel centres: cd exactly 0 or 1
             (bf16-exact) or within fp32 rounding of 0.8
      border coordinates exactly +-1, beyond +-1, on pixel centres, on the last row / column, and a quarter of all
             samples of an image on one pixel (a long gather chain in sample_norm_bwd)
      zeros  all-zero code and feature pixels under pixel-centre samples (zero norms: the eps branches), chan_scale
             zeroing random channels and every channel of image 0
      tagged every image and each of feats / feats_pos / code / code_pos carries its own offset direction, so a wrong
             image, slot or coordinate set is an O(1) error; the raw permutations include fixed points
      scale1e3 / scale1e-3   corr scaled by 1e3 / 1e-3"""
    g = torch.Generator().manual_seed(seed)
    base = regime[len("scale"):] if regime.startswith("scale") else None
    feats, feats_pos = lowrank_maps(B, E, H, W, g), lowrank_maps(B, E, H, W, g)
    code, code_pos = lowrank_maps(B, D, H, W, g), lowrank_maps(B, D, H, W, g)
    c1 = (torch.rand(B, fs, fs, 2, generator=g) * 2 - 1) * 1.2
    c2 = (torch.rand(B, fs, fs, 2, generator=g) * 2 - 1) * 1.2
    perms = torch.stack([torch.randperm(B, generator=g) for _ in range(n_neg)]) if n_neg else None
    cs = csp = None
    if regime == "flat":
        d0 = torch.randn(1, E, 1, 1, generator=g)
        a = d0.abs().mean()
        d = d0 + 1e-2 * a * torch.randn(B, E, 1, 1, generator=g)
        feats = d + 1e-2 * a * torch.randn(B, E, H, W, generator=g)
        feats_pos = d + 1e-2 * a * torch.randn(B, E, H, W, generator=g)
    elif regime == "kinks":
        kind = torch.randint(0, 3, (2, B, H, W), generator=g)
        proto = torch.zeros(3, D)
        proto[0, 0], proto[1, 1] = 1.0, 1.0
        proto[2, 0], proto[2, 1] = 0.8 / 5, 0.6 / 5
        code = proto[kind[0]].permute(0, 3, 1, 2).contiguous()
        code_pos = proto[kind[1]].permute(0, 3, 1, 2).contiguous()
        c1, c2 = centre_grid(B, fs, H, W, g), centre_grid(B, fs, H, W, g)
    elif regime == "border":
        for c in (c1, c2):
            flat = c.view(B, -1, 2)
            n = flat.shape[1]
            sel = torch.randint(0, 6, (B, n), generator=g)
            flat[sel == 0] = torch.tensor([1.0, 1.0])
            flat[sel == 1] = torch.tensor([-1.0, 1.0])
            flat[sel == 2] = torch.tensor([1.5, -1.7])
            cg = centre_grid(B, fs, H, W, g, last=True).view(B, -1, 2)
            flat[sel == 3] = cg[sel == 3]
            flat[:, : n // 4] = torch.tensor([centres(W)[1][-2], centres(H)[1][1]])
    elif regime == "zeros":
        (kx, tx), (ky, ty) = centres(W), centres(H)
        tx, ty = tx[kx % 2 == 0], ty[ky % 3 == 0]
        for t in (feats, feats_pos, code, code_pos):
            t[:, :, ::3, ::2] = 0.0
        grid = centre_grid(B, fs, H, W, g)
        on = torch.stack([tx[torch.randint(0, len(tx), (B, fs, fs), generator=g)],
                          ty[torch.randint(0, len(ty), (B, fs, fs), generator=g)]], -1)
        half = torch.rand(B, fs, fs, 1, generator=g) < 0.5
        c1 = torch.where(half, on, grid)
        c2 = torch.where(~half, on, c1 * 0.9)
        cs = (torch.rand(B, E, generator=g) > 0.1).float() / 0.9
        csp = (torch.rand(B, E, generator=g) > 0.1).float() / 0.9
        cs[0] = 0.0
    elif regime == "tagged":
        for t in (feats, feats_pos, code, code_pos):
            C = t.shape[1]
            t += 3.0 * torch.randn(B, C, 1, 1, generator=g)
        if n_neg:
            perms[0] = torch.arange(B)  # every negative image a fixed point: the fix-up picks b + 1 mod B
    elif base is not None:
        s = float(base)
        feats, feats_pos, code, code_pos = feats * s, feats_pos * s, code * s, code_pos * s
    if regime == "corr" or regime == "tagged":
        cs = (torch.rand(B, E, generator=g) > 0.1).float() / 0.9
        csp = (torch.rand(B, E, generator=g) > 0.1).float() / 0.9
    return dict(feats=feats, feats_pos=feats_pos, code=code, code_pos=code_pos, coords1=c1, coords2=c2, perms=perms,
                chan_scale=cs, chan_scale_pos=csp)
