"""fp64 reference of the fused kNN search (stego_knn_topk: csrc/knn.cu, stego_b200/knn.py) and the inputs its tests
run on, shared by tests/test_knn_fp64_reference.py (CPU) and tests/test_knn_fp64_gpu.py.

Plain torch and device-agnostic: the GPU tests run `knn_reference` in float64 on the device (the n x n similarity
matrix of the COCO-Stuff size is 10^13 fp64 flop and is formed 4096 rows at a time), the CPU test pins it to the oracle
(oracle/stego_oracle.py::knn_indices) and to a brute-force loop.

The order the kernel promises and the reference applies: a row's own index first, whatever its similarity to itself
comes out as, then (similarity descending, index ascending).
"""
import torch

U = 2.0 ** -24        # unit roundoff of fp32
TILE = 128            # query rows per row block and key columns per tile (KNN_BM, KNN_BN)
HALF = 64             # key columns per scan thread
MAXK = 32             # KNN_MAXK
EPS_LEVELS = (0.0, 1e-7, 1e-5, 1e-3)


def sim_error_bar(E):
    """Bound on |kernel similarity - fp64 similarity| for fp32 descriptors of width E.  With a, b the exactly
    normalised rows (sum |a_c b_c| <= |a| |b| = 1 by Cauchy-Schwarz) and u = 2^-24:

      normalisation  knn_prep_kernel sums x^2 in fp32 (E / 32 fmaf per lane, 5 shuffle adds: relative gamma_{E/32+5}
                     of a sum of positive terms), then sqrtf, 1 / x and x * inv, each correctly rounded: every element
                     of a row carries the same factor 1 + d, |d| <= (E / 64 + 6) u.  Two rows: 2 (E / 64 + 6) u |sim|.
      hi / lo split  hi = bf16(v), lo = bf16(v - hi); v - hi is exact in fp32 and bf16 rounding is 2^-8 relative, so
                     |lo| <= 2^-8 |v| and the residual |v - hi - lo| <= 2^-16 |v|.  The two residuals cost
                     2 * 2^-16 sum |a b| and the lo x lo pass the kernel drops another 2^-16 sum |a b|: 3 * 2^-16.
      accumulation   the three passes are one chain of 3 E exact bf16 x bf16 products in the tensor core's fp32
                     accumulator, whose rounding is not documented as IEEE round-to-nearest; like the other suites
                     (tests/test_head_fp64_gpu.py) it is treated as a 3 E-term fp32 chain, an assumption:
                     gamma_{3E} (1 + 2^-7) sum |a b|, the second factor for |hi| |lo| terms on top of |hi| |hi|.

    The split term is a worst case over the rounding of every element; measured errors sit an order of magnitude below
    (they are recorded beside the bar)."""
    k = 3 * E
    gamma = k * U / (1 - k * U)
    return 2 * (E / 64 + 6) * U + 3 * 2.0 ** -16 + gamma * (1 + 2.0 ** -7)


def normalize64(feats):
    """x / max(|x|, 1e-12) in float64: F.normalize's rule (a zero row stays zero)."""
    x = feats.double()
    return x / x.norm(dim=1, keepdim=True).clamp_min(1e-12)


def knn_reference(feats, k, device="cpu", chunk=4096, gather=None):
    """The k + 1 best neighbours of every row of feats [n, E] by cosine similarity in float64 on `device` (k + 1 so
    that the runner-up of the k-th is known; min(k + 1, n) columns).  Order: the row itself first, then (similarity
    descending, index ascending), exactly — ties are not left to topk.  Similarities are formed `chunk` rows at a
    time, never as the whole n x n matrix.
    gather: optional int64 [n, m] column indices; the fp64 similarities at those columns are returned too.
    Returns dict(idx int64 [n, kk], val float64 [n, kk] (column 0 is the row's similarity to itself), gathered)."""
    xn = normalize64(feats.to(device))
    n = xn.shape[0]
    kk = min(k + 1, n)
    ar = torch.arange(kk, device=xn.device)
    idx, val, got = [], [], []
    for i in range(0, n, chunk):
        s = xn[i:i + chunk] @ xn.T
        r_ = s.shape[0]
        rows = torch.arange(r_, device=xn.device)
        if gather is not None:
            got.append(s.gather(1, gather[i:i + r_].to(xn.device)))
        diag = s[rows, rows + i].clone()
        s[rows, rows + i] = float("inf")                      # the row itself sorts first
        kth = torch.topk(s, kk, dim=1).values[:, -1:]          # values only: which of several ties topk picks is moot
        cand = s >= kth                                        # everything that can be among the kk best
        r, c = cand.nonzero(as_tuple=True)                     # row-major: index ascending within a row
        v = s[r, c]
        o = torch.sort(v, descending=True, stable=True).indices
        o = o[torch.sort(r[o], stable=True).indices]           # grouped by row; inside a row (value desc, index asc)
        cnt = cand.sum(1)
        first = torch.cumsum(cnt, 0) - cnt
        sel = o[(first[:, None] + ar[None, :]).reshape(-1)]
        vv = v[sel].view(r_, kk)
        vv[:, 0] = diag
        idx.append(c[sel].view(r_, kk))
        val.append(vv)
        del s, cand, r, c, v, o
    out = dict(idx=torch.cat(idx, 0), val=torch.cat(val, 0))
    if gather is not None:
        out["gathered"] = torch.cat(got, 0)
    return out


# ------------------------------------------------------------------------------------------------
# input builders: fp32 [n, E] on the CPU, seeded
# ------------------------------------------------------------------------------------------------
def lattice_plants(n):
    """(source, copy) row pairs exact_lattice plants on top of its random duplicates: copies 64 columns away (the other
    half of a key tile, or half 0 of the next tile against half 1 of this one), 128 and more away (another tile), and
    in the last row block."""
    pairs = [(0, 64), (70, 6), (63, 128), (1, 129), (100, 164), (130, 2), (3, n - 1), (n - 2, 4), (127, n - 3)]
    seen, out = set(), []
    for a, b in pairs:
        if 0 <= a < n and 0 <= b < n and a != b and b not in seen and a not in seen:
            out.append((a, b))
            seen.update((a, b))
    return out


def exact_lattice(n, E, seed, nnz=16, scale=True):
    """Rows with exactly nnz = 16 entries of +-1 and zeros elsewhere, drawn with replacement from a pool of about n / 3
    patterns (so exact duplicates are common), with the pairs of lattice_plants(n) copied on top, each row times a
    power of two.  Then |x| = 4 * 2^p exactly, the normalised entries +-1/4 are exact in bf16, the lo plane is zero and
    every similarity is a multiple of 1/16 in [-1, 1] that fp32 sums exactly in any order: the kernel's values must equal
    the fp64 values bit for bit, and with 33 possible values almost every position is a tie."""
    g = torch.Generator().manual_seed(seed)
    pool_n = max(2, n // 3)
    pos = torch.rand(pool_n, E, generator=g).argsort(1)[:, :nnz]
    sign = torch.randint(0, 2, (pool_n, nnz), generator=g).float() * 2 - 1
    pool = torch.zeros(pool_n, E).scatter_(1, pos, sign)
    x = pool[torch.randint(0, pool_n, (n,), generator=g)]
    for a, b in lattice_plants(n):
        x[b] = x[a]
    if scale:
        x = x * 2.0 ** torch.randint(-3, 4, (n, 1), generator=g).float()
    return x


def clustered(n, E, seed):
    """Cluster centres + 0.35 sigma noise, ~20 rows per cluster, random row scales: descriptors with a realistic
    neighbourhood structure (what tests/test_knn_gpu.py has always used)."""
    g = torch.Generator().manual_seed(seed)
    base = torch.randn(max(8, n // 20), E, generator=g)
    x = base[torch.randint(0, base.shape[0], (n,), generator=g)] + 0.35 * torch.randn(n, E, generator=g)
    return x * (0.5 + torch.rand(n, 1, generator=g))


def near_duplicates(n, E, seed, pairs=64):
    """clustered(n, E) with (original, copy) row pairs planted: copy = original + eps |original| / sqrt(E) * noise for
    eps cycling through EPS_LEVELS (0: a bitwise copy).  The copy sits before its original in half the pairs; the
    first pairs straddle a half tile (63 | 64), a key tile and row block (127 | 128) and, when n allows, the first and
    the last row block; the rest are drawn at random.  Consecutive video frames are the realistic case.
    Returns feats, pairs int64 [m, 2] (original, copy), eps float64 [m]."""
    g = torch.Generator().manual_seed(seed + 1)
    x = clustered(n, E, seed)
    fixed = [(63, 64), (128, 127), (10, n - 5), (n - 6, 11), (190, 200), (300, 40)]
    used, kept = set(), []
    for a, b in fixed:
        if 0 <= a < n and 0 <= b < n and not {a, b} & used:
            kept.append((a, b))
            used.update((a, b))
    fixed = kept
    free = [i for i in torch.randperm(n, generator=g).tolist() if i not in used]
    m = max(0, min(pairs, n // 4) - len(fixed))
    rand = [(free[2 * j], free[2 * j + 1]) for j in range(m)]
    rand = [(a, b) if (a < b) == (j // 4 % 2 == 0) else (b, a) for j, (a, b) in enumerate(rand)]  # both ways per eps
    pr = torch.tensor(fixed + rand, dtype=torch.long)
    eps = torch.tensor([EPS_LEVELS[j % len(EPS_LEVELS)] for j in range(pr.shape[0])], dtype=torch.float64)
    orig = x[pr[:, 0]]
    noise = torch.randn(pr.shape[0], E, generator=g)
    x[pr[:, 1]] = orig + (eps[:, None] * orig.double().norm(dim=1, keepdim=True) / E ** 0.5).float() * noise
    return x, pr, eps


def scaled_rows(n, E, seed):
    """clustered(n, E) with row norms spread over 1e-6 .. 1e6 (normalisation must remove them) and row n // 2 all
    zero (the eps clamp of the normalisation: every similarity of that row is exactly 0).  Returns feats, zero row."""
    g = torch.Generator().manual_seed(seed + 2)
    x = clustered(n, E, seed)
    x = x / x.norm(dim=1, keepdim=True) * 10.0 ** (torch.rand(n, 1, generator=g) * 12 - 6)
    z = n // 2
    x[z] = 0.0
    return x, z
