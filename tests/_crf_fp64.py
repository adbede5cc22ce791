"""fp64 references of the dense CRF (csrc/crf.cu through stego_b200/crf.py and stego_b200/eval.py::fused_eval_crf),
shared by the CRF tests.

Plain, vectorised torch (no Python loop over pixels or lattice points), device-agnostic: the GPU tests run these in
float64 on the device at the c4 frame, the CPU test pins them to the fp32 restatement oracle/crf_oracle.py.  The
conventions are those of the restatement (the published permutohedral lattice of Adams et al. 2010 with densecrf's
blur stencil, slice scale and NORMALIZE_SYMMETRIC kernels, Potts mean field):

  embed           elevated, rem0, rank, barycentric weights and the d+1 vertices (full (d+1)-coordinate tuples) of
                  every pixel, plus its decision margin: the smallest distance to a rounding midpoint (where up != down)
                  and the smallest |residual_i - residual_j|.  In exact arithmetic sum_r bary_r vertex_r = elevated,
                  bary >= 0 and sum_r bary_r = 1.
  lattice_tables  unique points, offsets, the 2(d+1) neighbour tables and the stable-sorted CSR list, from full vertex
                  tuples packed in a mixed radix over the observed coordinate range (not crf._pack's fixed-width fields);
                  `concat` is the B-frame concatenation of crf._bilateral_lattice.
  filter          splat, d+1 blur passes and slice on a given lattice, with the magnitude and error-propagation
                  vectors of the fp32 bars (derived in tests/test_crf_fp64_gpu.py).
  norm, unary_from_logits, update, mean_field.
"""
import math

import torch

U = 2.0 ** -24  # unit roundoff of fp32
MAX_ITER = 10
POS_W, POS_XY_STD, BI_W, BI_XY_STD, BI_RGB_STD = 3.0, 1.0, 4.0, 67.0, 3.0
CLIP = 1e-5


def gamma(k):
    """gamma_k = k u / (1 - k u): the bound on k fp32 roundings in a chain (Higham, Lemma 3.1)."""
    return k * U / (1 - k * U)


def alpha(d):
    """densecrf's slice scale 1 / (1 + 2^-d)"""
    return 1.0 / (1.0 + 2.0 ** -d)


# ------------------------------------------------------------------------------------------------
# embedding
# ------------------------------------------------------------------------------------------------
def features(H, W, d, sxy, srgb=None, image=None, device="cpu"):
    """The exact features [N, d] in float64, pixels row-major: (x / sxy, y / sxy[, c0 / srgb, c1 / srgb, c2 / srgb]);
    image [H, W, 3] uint8 in the channel order the kernel reads (crf.prepare_image's BGR)."""
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float64, device=device),
                            torch.arange(W, dtype=torch.float64, device=device), indexing="ij")
    cols = [xs.reshape(-1) / sxy, ys.reshape(-1) / sxy]
    if d == 5:
        im = image.reshape(-1, 3).to(device=device, dtype=torch.float64)
        cols += [im[:, c] / srgb for c in range(3)]
    return torch.stack(cols, 1)


def canonical(d, device="cpu"):
    """canonical[r][k] = r if k <= d - r else r - (d + 1): vertex r of the canonical simplex, by rank"""
    r = torch.arange(d + 1, device=device)[:, None]
    k = torch.arange(d + 1, device=device)[None, :]
    return torch.where(k <= d - r, r, r - (d + 1))


def embed(f):
    """f [N, d] float64 -> dict(elevated, elev_abs (sum of |terms| of elevated), rem0, rank, bary [N, d+1],
    vertices [N, d+1 (vertex r), d+1 (coordinate)] int64, margin [N])."""
    f = f.double()
    N, d = f.shape
    dev = f.device
    j = torch.arange(d, dtype=torch.float64, device=dev)
    scale = math.sqrt(2.0 / 3.0) * (d + 1) / torch.sqrt((j + 1) * (j + 2))
    cf = f * scale
    zero = torch.zeros(N, 1, dtype=torch.float64, device=dev)
    # elevated[j] = sum_{k >= j} cf[k] - j cf[j - 1]   (permutohedral.cpp's running sum from the last feature down)
    suffix = torch.cat([cf.flip(1).cumsum(1).flip(1), zero], 1)
    suffix_abs = torch.cat([cf.abs().flip(1).cumsum(1).flip(1), zero], 1)
    prev = torch.cat([zero, cf], 1)
    jj = torch.arange(d + 1, dtype=torch.float64, device=dev)
    el = suffix - jj * prev
    el_abs = suffix_abs + jj * prev.abs()
    # nearest remainder-0 point
    up = torch.ceil(el / (d + 1)) * (d + 1)
    down = torch.floor(el / (d + 1)) * (d + 1)
    rem0 = torch.where(up - el < el - down, up, down)
    inf = torch.full_like(el, math.inf)
    round_margin = torch.where(up != down, ((up - el) - (el - down)).abs(), inf).amin(1)
    s = torch.round(rem0.sum(1) / (d + 1)).long()
    # ranks of the residuals, ties as the kernel breaks them: for i < j, diff_i < diff_j ranks i up, else j
    diff = el - rem0
    upper = torch.ones(d + 1, d + 1, dtype=torch.bool, device=dev).triu(1)
    lt = diff[:, :, None] < diff[:, None, :]
    rank = (lt & upper).sum(2) + (~lt & upper).sum(1)
    rank_margin = (diff[:, :, None] - diff[:, None, :]).abs().masked_fill(~upper, math.inf).amin((1, 2))
    rank = rank + s[:, None]
    lo, hi = (rank < 0).long(), (rank > d).long()
    rank = rank + (d + 1) * (lo - hi)
    rem0 = rem0 + (d + 1) * (lo - hi).double()
    # barycentric weights
    v = (el - rem0) / (d + 1)
    bary = torch.zeros(N, d + 2, dtype=torch.float64, device=dev)
    bary.scatter_add_(1, d - rank, v)
    bary.scatter_add_(1, d - rank + 1, -v)
    bary[:, 0] += 1.0 + bary[:, d + 1]
    can = canonical(d, dev)
    verts = rem0.round().long()[:, None, :] + can[:, rank].permute(1, 0, 2)
    return dict(elevated=el, elev_abs=el_abs, rem0=rem0, rank=rank, bary=bary[:, :d + 1], vertices=verts,
                margin=torch.minimum(round_margin, rank_margin))


def unpack(keys, d, bits):
    """the kernel's packed keys [N, d+1] (d fields of `bits` bits, biased, first coordinate in the top field) ->
    full vertex tuples [N, d+1, d+1]: the last coordinate is minus the sum of the others (lattice points lie in the
    hyperplane sum = 0)."""
    fields = [((keys >> (bits * (d - 1 - i))) & ((1 << bits) - 1)) - (1 << (bits - 1)) for i in range(d)]
    c = torch.stack(fields, -1)
    return torch.cat([c, -c.sum(-1, keepdim=True)], -1)


def is_simplex(verts):
    """[N] bool: the d+1 vertices form a simplex of the permutohedral triangulation: vertex 0 is a remainder-0 point
    (coordinates multiples of d+1), every vertex sums to 0, and each step v_r - v_{r-1} is (1, ..., 1) minus d+1 in
    one coordinate, a different coordinate for every step."""
    N, R, D1 = verts.shape
    d = D1 - 1
    ok = (verts[:, 0] % (d + 1) == 0).all(1) & (verts.sum(2) == 0).all(1)
    step = verts[:, 1:] - verts[:, :-1] - 1                                   # [N, d, d+1]: 0 or -(d+1)
    ok &= ((step == 0) | (step == -(d + 1))).all(2).all(1) & ((step != 0).sum(2) == 1).all(1)
    ok &= ((step != 0).sum(1) <= 1).all(1)                                    # distinct coordinates
    return ok


# ------------------------------------------------------------------------------------------------
# lattice tables
# ------------------------------------------------------------------------------------------------
def lattice_tables(verts):
    """verts [N, d+1, d+1] int64 -> dict(M, points [M, d+1], offset [N, d+1], n1, n2 [d+1, M] (-1: missing),
    rowptr [M+1], slots [N (d+1)], counts [M]).  Points are numbered in lexicographic order of their coordinates
    (what sorting crf.cu's fixed-width keys gives when nothing wraps); neighbours along axis j are the point - 1 with
    coordinate j moved by +d (n1) and + 1 with coordinate j moved by -d (n2); slots are (pixel, vertex) = pixel (d+1)
    + vertex, sorted by point and by slot within a point."""
    N, R, D1 = verts.shape
    d = D1 - 1
    dev = verts.device
    c = verts[..., :d].reshape(-1, d)
    lo = c.amin(0) - (d + 1)
    span = c.amax(0) - lo + (d + 2)             # room for the +-d / +-1 moves of the neighbours
    assert float(span.double().log2().sum()) < 62, "mixed radix overflow"
    w = torch.ones(d, dtype=torch.long, device=dev)
    for i in range(d - 2, -1, -1):
        w[i] = w[i + 1] * span[i + 1]
    pack = lambda x: ((x - lo) * w).sum(-1)
    uniq, inv = torch.unique(pack(c), return_inverse=True)
    M = int(uniq.numel())
    pts = torch.stack([(uniq // w[i]) % span[i] + lo[i] for i in range(d)], 1)
    n1 = torch.empty(d + 1, M, dtype=torch.long, device=dev)
    n2 = torch.empty_like(n1)
    for j in range(d + 1):
        for dst, step, move in ((n1, -1, d), (n2, 1, -d)):
            k = pts + step
            if j < d:
                k[:, j] = pts[:, j] + move
            q = pack(k)
            pos = torch.searchsorted(uniq, q).clamp_(max=M - 1)
            dst[j] = torch.where(uniq[pos] == q, pos, torch.full_like(pos, -1))
    ids = inv.reshape(-1)
    S = ids.numel()
    slots = torch.argsort(ids * S + torch.arange(S, device=dev))      # unique keys: any sort is the stable one
    counts = torch.bincount(ids, minlength=M)
    rowptr = torch.cat([torch.zeros(1, dtype=torch.long, device=dev), counts.cumsum(0)])
    full = torch.cat([pts, -pts.sum(1, keepdim=True)], 1)
    return dict(d=d, N=N, M=M, points=full, offset=inv.reshape(N, d + 1), n1=n1, n2=n2, rowptr=rowptr, slots=slots,
                counts=counts)


def concat(tables):
    """crf._bilateral_lattice's concatenation of B frames' tables: point ids, neighbours (-1 kept) and slots offset
    by each frame's base.  Returns the concatenated dict and the bases [B]."""
    Ms = torch.tensor([t["M"] for t in tables])
    bases = torch.cat([torch.zeros(1, dtype=torch.long), Ms.cumsum(0)[:-1]])
    d, N = tables[0]["d"], tables[0]["N"]
    out = dict(d=d, N=N * len(tables), M=int(Ms.sum()))
    out["offset"] = torch.cat([t["offset"] + int(b) for t, b in zip(tables, bases)])
    for k in ("n1", "n2"):
        out[k] = torch.cat([t[k] + int(b) * (t[k] >= 0) for t, b in zip(tables, bases)], 1)
    out["slots"] = torch.cat([t["slots"] + i * N * (d + 1) for i, t in enumerate(tables)])
    out["rowptr"] = torch.cat([t["rowptr"][:-1] + i * N * (d + 1) for i, t in enumerate(tables)] +
                              [torch.full((1,), len(tables) * N * (d + 1), dtype=torch.long,
                                          device=tables[0]["rowptr"].device)])
    out["counts"] = torch.cat([t["counts"] for t in tables])
    return out, bases


# ------------------------------------------------------------------------------------------------
# filtering
# ------------------------------------------------------------------------------------------------
def lattice(offset, bary, n1, n2, M=None):
    """a lattice as the filters take it: int64 ids, bary cast to float64, slot counts per point"""
    offset, n1, n2 = offset.long(), n1.long(), n2.long()
    M = int(n1.shape[1]) if M is None else M
    return dict(d=offset.shape[1] - 1, N=offset.shape[0], M=M, offset=offset, bary=bary.double(), n1=n1, n2=n2,
                counts=torch.bincount(offset.reshape(-1), minlength=M))


def splat(lat, inp):
    """values [M, C] = sum over slots of point i of bary * inp[pixel], and the sum of |terms|"""
    M, C = lat["M"], inp.shape[1]
    vals = torch.zeros(M, C, dtype=torch.float64, device=inp.device)
    mag = torch.zeros_like(vals)
    for r in range(lat["d"] + 1):
        t = lat["bary"][:, r:r + 1] * inp
        vals.index_add_(0, lat["offset"][:, r], t)
        mag.index_add_(0, lat["offset"][:, r], t.abs())
    return vals, mag


def blur(v, n1j, n2j):
    """one pass: v + 0.5 (v[n1] + v[n2]), missing neighbours (-1) read as 0"""
    pad = torch.cat([v, torch.zeros_like(v[:1])])
    return v + 0.5 * (pad[n1j] + pad[n2j])


def slice_(lat, vals):
    """sum_r bary_r vals[offset_r] (without the alpha scale), and the same with |bary|"""
    out = sum(lat["bary"][:, r:r + 1] * vals[lat["offset"][:, r]] for r in range(lat["d"] + 1))
    out_abs = sum(lat["bary"][:, r:r + 1].abs() * vals[lat["offset"][:, r]].abs() for r in range(lat["d"] + 1))
    return out, out_abs


def filter(lat, inp, reverse=False, bars=False, keep=False):
    """splat, the d+1 blur passes (axes 0..d, or d..0 with reverse) and the slice scaled by alpha(d).
    Returns dict(passes: the values after the splat and after each pass (with keep; otherwise the last two, or with
    bars=False only the last), out [N, C]); with bars also
      mag[j]  the fp64 magnitudes: sum of |splat terms|, then each pass applied to the previous magnitudes;
      err[j]  the fp32 error bound: gamma_{m_i + 1} mag_0 (product of norm and Q, product with bary, m_i - 1 additions
              in any order), then per pass blur(err) (1 + gamma_2) + gamma_2 mag (two roundings of old + 0.5 (a + b)
              on values bounded by the magnitudes)."""
    d = lat["d"]
    vals, mag = splat(lat, inp)
    passes = [vals]
    out = dict(passes=passes)
    if not bars and not keep:
        for j in (range(d, -1, -1) if reverse else range(d + 1)):
            passes[0] = blur(passes[0], lat["n1"][j], lat["n2"][j])
        out["out"] = alpha(d) * slice_(lat, passes[0])[0]
        return out
    if bars:
        err = (lat["counts"] + 1).double()[:, None] * U / (1 - (lat["counts"] + 1).double()[:, None] * U) * mag
        out["mag"], out["err"] = [mag], [err]
    axes = range(d, -1, -1) if reverse else range(d + 1)
    for j in axes:
        passes.append(blur(passes[-1], lat["n1"][j], lat["n2"][j]))
        if bars:
            m = blur(out["mag"][-1], lat["n1"][j], lat["n2"][j])
            out["mag"].append(m)
            out["err"].append(blur(out["err"][-1], lat["n1"][j], lat["n2"][j]) * (1 + gamma(2)) + gamma(2) * m)
        if not keep and len(passes) > 2:  # the last two passes are all the tests read back
            for k in ("passes", "mag", "err"):
                if k in out:
                    out[k].pop(0)
    s, _ = slice_(lat, passes[-1])
    out["out"] = alpha(d) * s
    return out


def norm(lat, bars=False):
    """NORMALIZE_SYMMETRIC: 1 / sqrt(K 1 + 1e-20), K 1 = alpha slice(blur(splat(1))).  With bars, the fp32 bound:
    the slice chain carries sum |b| err alpha + gamma_{d+4} alpha sum |b| (mag + err) (two products per term, d
    additions, alpha's own rounding, the + 1e-20), and 1 / sqrtf halves its relative error and adds two correct
    roundings."""
    ones = torch.ones(lat["N"], 1, dtype=torch.float64, device=lat["bary"].device)
    f = filter(lat, ones, bars=bars)
    k1 = f["out"][:, 0]
    n = 1.0 / torch.sqrt(k1 + 1e-20)
    if not bars:
        return n
    a = alpha(lat["d"])
    e_prop, _ = slice_(dict(lat, bary=lat["bary"].abs()), f["err"][-1])
    _, m = slice_(lat, f["mag"][-1] + f["err"][-1])
    err_s = a * e_prop[:, 0] + gamma(lat["d"] + 4) * a * m[:, 0]
    rel = err_s / k1
    return n, dict(filter=f, k1=k1, k1_err=err_s, bar=n * (0.5 * rel * (1 + rel) + gamma(2)))


def softmax(t):
    return torch.softmax(t.double(), 1)


def unary_from_logits(logits, clip=CLIP):
    """logits [N, C] -> (U = -log(clip(softmax(logits), clip, 1)) [N, C], the probabilities)"""
    p = torch.softmax(logits.double(), 1)
    return -torch.log(p.clamp(clip, 1.0)), p


def update(U, Q, lat_g, lat_b, norm_g, norm_b, w_g=POS_W, w_b=BI_W, bars=False):
    """One mean-field step: Q' = softmax(-U + w_g n_g K_g(n_g Q) + w_b n_b K_b(n_b Q)).  Returns dict(q, t, and with
    bars: dt, the fp32 bound on t).  The slice of the update carries gamma_{d+6} on the |terms| (d+1 products and
    additions, alpha and its rounding, the norm, the weight) plus the propagated blur error, and the sum
    -U + t_g + t_b two more roundings."""
    U, Q = U.double(), Q.double()
    ng, nb = norm_g.double()[:, None], norm_b.double()[:, None]
    t = -U
    dt = gamma(2) * U.abs() if bars else None
    for lat, n, w in ((lat_g, ng, w_g), (lat_b, nb, w_b)):
        f = filter(lat, Q * n, bars=bars)
        t = t + w * n * f["out"]
        if bars:
            a, d = alpha(lat["d"]), lat["d"]
            e_prop, _ = slice_(dict(lat, bary=lat["bary"].abs()), f["err"][-1])
            _, m = slice_(lat, f["mag"][-1] + f["err"][-1])
            mag_t = w * a * n * m
            dt = dt + w * a * n * e_prop + gamma(d + 6) * mag_t + gamma(2) * mag_t
    out = dict(q=softmax(t), t=t)
    if bars:
        out["dt"] = dt
    return out


def softmax_bar(q, z, n, dz=None):
    """bound on |q_fp32 - q| for q = softmax over n lanes computed as __expf(z) / sum (z = t - max t <= 0):
    each __expf is within 2 + floor(1.173 |z|) ulp (2^-23 relative), the sum and the divide (n + 2) u, an input error
    dz on t moves log q by at most 2 max dz.  Relative to q: 2 max dz + eps_i + sum_j q_j eps_j + (n + 2) u; plus
    2^-126, the flush-to-zero of __expf's result."""
    eps = (2 + torch.floor(1.173 * z.abs())) * 2.0 ** -23
    rel = eps + (q * eps).sum(1, keepdim=True) + (n + 2) * U
    if dz is not None:
        rel = rel + 2 * dz.amax(1, keepdim=True)
    return q * rel + 2.0 ** -126


def mean_field(U, lat_g, lat_b, n_iter=MAX_ITER, norm_g=None, norm_b=None, record=False):
    """densecrf's inference: Q_0 = softmax(-U), n_iter updates.  norm_*: None computes the fp64 normalisation of the
    lattice.  Returns the last Q, or with record every Q_k (k = 0 .. n_iter)."""
    norm_g = norm(lat_g) if norm_g is None else norm_g.double()
    norm_b = norm(lat_b) if norm_b is None else norm_b.double()
    Q = softmax(-U)
    seq = [Q] if record else None
    for _ in range(n_iter):
        Q = update(U, Q, lat_g, lat_b, norm_g, norm_b)["q"]
        if record:
            seq.append(Q)
    return seq if record else Q


# ------------------------------------------------------------------------------------------------
# input builders
# ------------------------------------------------------------------------------------------------
IMAGES = ("piecewise", "constant", "noise", "black", "saturated")


def image(kind, H, W, seed=0):
    """[H, W, 3] uint8 frames in the kernel's channel order:
    piecewise   a 4 x 4 grid of constant colours plus +-12 of noise (edges for the bilateral kernel)
    constant    one colour everywhere (the bilateral lattice degenerates to the position one: largest slot counts)
    noise       uniform in [0, 255] per channel (M_b tends to 6 N)
    black       all channels 0 (exactly zero colour coordinates: rank ties)
    saturated   all channels 255"""
    g = torch.Generator().manual_seed(seed)
    if kind == "piecewise":
        base = torch.randint(20, 236, (1, 3, 4, 4), generator=g).float()
        x = torch.nn.functional.interpolate(base, (H, W), mode="nearest")[0].permute(1, 2, 0)
        return (x + torch.randint(-12, 13, (H, W, 3), generator=g)).clamp(0, 255).to(torch.uint8).contiguous()
    if kind == "constant":
        return torch.randint(0, 256, (1, 1, 3), generator=g).to(torch.uint8).expand(H, W, 3).contiguous()
    if kind == "noise":
        return torch.randint(0, 256, (H, W, 3), generator=g).to(torch.uint8)
    if kind == "black":
        return torch.zeros(H, W, 3, dtype=torch.uint8)
    if kind == "saturated":
        return torch.full((H, W, 3), 255, dtype=torch.uint8)
    raise ValueError(kind)


def normalised(img_u8):
    """the normalised frames [B, 3, H, W] whose crf.prepare_image is img_u8 [B, H, W, 3] (kernel channel order):
    channel-reversed, centred on the uint8 value so that the x255-and-truncate lands on it exactly."""
    mean = torch.tensor([0.485, 0.456, 0.406]).view(1, 3, 1, 1)
    std = torch.tensor([0.229, 0.224, 0.225]).view(1, 3, 1, 1)
    x = (img_u8.flip(-1).permute(0, 3, 1, 2).double() + 0.5) / 255.0
    return ((x - mean.double()) / std.double()).float()


UNARIES = ("random", "onehot", "straddle", "uniform")


def logits(kind, N, C, seed=0):
    """class scores [N, C] float32:
    random    N(0, 3^2)
    onehot    +50 on one class, -50 on the others (probabilities at the clip, U = -log 1e-5 off the winner)
    straddle  the winner at 0, the others at log(1e-5 S) (1 + 10^-3 U(-1, 1)) with S the softmax denominator: the
              probabilities straddle the clip at 1e-5
    uniform   all equal (bit-identical lanes, ties everywhere)"""
    g = torch.Generator().manual_seed(seed)
    if kind == "random":
        return torch.randn(N, C, generator=g) * 3
    if kind == "onehot":
        z = torch.full((N, C), -50.0)
        z[torch.arange(N), torch.randint(0, C, (N,), generator=g)] = 50.0
        return z
    if kind == "straddle":
        S = 1.0 + (C - 1) * 1e-5
        z = math.log(1e-5 * S) + 1e-3 * (torch.rand(N, C, generator=g, dtype=torch.float64) * 2 - 1)
        z[torch.arange(N), torch.randint(0, C, (N,), generator=g)] = 0.0
        return z.float()
    if kind == "uniform":
        return torch.full((N, C), 0.75)
    raise ValueError(kind)
