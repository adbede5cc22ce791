"""Oracle of the JPEG round trip a crop goes through in the reference's crop script: Pillow's default save (baseline,
quality 75, 4:2:0, islow DCT) followed by Pillow's decode.  TEST INFRASTRUCTURE ONLY.

Restated from the published algorithm, in numpy integer arithmetic, on a uint8 H x W x 3 image; no bitstream is
written (the entropy coding is lossless and changes nothing the decoder returns).  The stages:

  * RGB -> YCbCr: the IJG fixed-point formulae with 16 fraction bits (ITU-R BT.601 coefficients, FIX(x) =
    round(x 2^16)); Y rounds half up, Cb / Cr round with ONE_HALF - 1.
  * Edge replication to the 16 x 16 MCU grid (luma blocks past ceil(W / 8) and ceil(H / 8) are dummies the decoder
    never shows).  Columns are replicated at full resolution before downsampling; rows only to an even count, and
    the rows below that are copies of the last downsampled (and last luma) row.
  * h2v2 chroma downsampling: (a + b + c + d + bias) >> 2, bias 1, 2, 1, 2, ... along each output row.
  * Per 8 x 8 block: the islow forward DCT (13-bit constants, 2 pass-1 bits) of the samples - 128; quantisation by
    8 q rounded half away from zero, q the ITU T.81 Annex K tables scaled for quality 75 ((q * 50 + 50) // 100,
    clamped to 1..255); dequantisation by q; the islow inverse DCT, + 128 and clamped to 0..255.
  * Chroma upsampling: h2v2 "fancy" (triangle filter: 3/4 nearer and 1/4 farther sample along each axis, rounding
    bias 8 on even and 7 on odd output columns, edges replicated) when the subsampled width exceeds 2; a chroma plane
    of width 1 or 2 (images up to 4 columns wide) is replicated 2 x 2 instead, as libjpeg picks the plain upsampler
    there.
  * YCbCr -> RGB: the IJG fixed-point tables (16 fraction bits), clamped to 0..255.

Its judge is Pillow itself: np.asarray(Image.open(BytesIO(saved)).convert("RGB")) of the image saved with
Image.save(f, "JPEG") (tests/test_crops.py).
"""
from __future__ import annotations

import numpy as np

QUALITY = 75
LUMA_BASE = np.array([
    16, 11, 10, 16, 24, 40, 51, 61,
    12, 12, 14, 19, 26, 58, 60, 55,
    14, 13, 16, 24, 40, 57, 69, 56,
    14, 17, 22, 29, 51, 87, 80, 62,
    18, 22, 37, 56, 68, 109, 103, 77,
    24, 35, 55, 64, 81, 104, 113, 92,
    49, 64, 78, 87, 103, 121, 120, 101,
    72, 92, 95, 98, 112, 100, 103, 99], dtype=np.int64).reshape(8, 8)
CHROMA_BASE = np.full((8, 8), 99, dtype=np.int64)
CHROMA_BASE[:4, :4] = np.array([[17, 18, 24, 47], [18, 21, 26, 66], [24, 26, 56, 99], [47, 66, 99, 99]])


def quant_table(base: np.ndarray, quality: int = QUALITY) -> np.ndarray:
    """IJG jpeg_quality_scaling + jpeg_add_quant_table with force_baseline: int64 [8, 8], natural order."""
    scale = 5000 // quality if quality < 50 else 200 - 2 * quality
    return np.clip((base * scale + 50) // 100, 1, 255)


LUMA_Q, CHROMA_Q = quant_table(LUMA_BASE), quant_table(CHROMA_BASE)

# islow DCT constants: FIX(x) = round(x * 2^13)
CONST_BITS, PASS1_BITS = 13, 2
F0298, F0390, F0541, F0765 = 2446, 3196, 4433, 6270
F0899, F1175, F1501, F1847 = 7373, 9633, 12299, 15137
F1961, F2053, F2562, F3072 = 16069, 16819, 20995, 25172


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def _odd(t4, t5, t6, t7):
    """The shared odd-part rotation of the islow forward and inverse DCTs (t4..t7 in the forward naming)."""
    z1, z2, z3, z4 = t4 + t7, t5 + t6, t4 + t6, t5 + t7
    z5 = (z3 + z4) * F1175
    t4, t5, t6, t7 = t4 * F0298, t5 * F2053, t6 * F3072, t7 * F1501
    z1, z2, z3, z4 = z1 * -F0899, z2 * -F2562, z3 * -F1961 + z5, z4 * -F0390 + z5
    return t4 + z1 + z3, t5 + z2 + z4, t6 + z2 + z3, t7 + z1 + z4


def _fdct_1d(d, pass1: bool):
    """jpeg_fdct_islow on 8 int64 arrays (one transform per element): the 8 outputs of that pass."""
    tmp0, tmp7 = d[0] + d[7], d[0] - d[7]
    tmp1, tmp6 = d[1] + d[6], d[1] - d[6]
    tmp2, tmp5 = d[2] + d[5], d[2] - d[5]
    tmp3, tmp4 = d[3] + d[4], d[3] - d[4]
    tmp10, tmp13, tmp11, tmp12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    out = [None] * 8
    sh = CONST_BITS - PASS1_BITS if pass1 else CONST_BITS + PASS1_BITS
    if pass1:
        out[0], out[4] = (tmp10 + tmp11) << PASS1_BITS, (tmp10 - tmp11) << PASS1_BITS
    else:
        out[0], out[4] = _descale(tmp10 + tmp11, PASS1_BITS), _descale(tmp10 - tmp11, PASS1_BITS)
    z1 = (tmp12 + tmp13) * F0541
    out[2] = _descale(z1 + tmp13 * F0765, sh)
    out[6] = _descale(z1 + tmp12 * -F1847, sh)
    o7, o5, o3, o1 = _odd(tmp4, tmp5, tmp6, tmp7)
    out[7], out[5], out[3], out[1] = (_descale(o, sh) for o in (o7, o5, o3, o1))
    return out


def _idct_1d(c, pass1: bool):
    """jpeg_idct_islow on 8 dequantised int64 arrays: the 8 outputs of that pass (pass 2 before the + 128)."""
    z1 = (c[2] + c[6]) * F0541
    tmp2, tmp3 = z1 + c[6] * -F1847, z1 + c[2] * F0765
    tmp0, tmp1 = (c[0] + c[4]) << CONST_BITS, (c[0] - c[4]) << CONST_BITS
    tmp10, tmp13, tmp11, tmp12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    t0, t1, t2, t3 = _odd(c[7], c[5], c[3], c[1])
    sh = CONST_BITS - PASS1_BITS if pass1 else CONST_BITS + PASS1_BITS + 3
    return [_descale(v, sh) for v in (tmp10 + t3, tmp11 + t2, tmp12 + t1, tmp13 + t0,
                                      tmp13 - t0, tmp12 - t1, tmp11 - t2, tmp10 - t3)]


def quantize(coef: np.ndarray, q: np.ndarray) -> np.ndarray:
    """coef / (8 q) rounded half away from zero (libjpeg's division; its reciprocal form gives the same integers)."""
    d = 8 * q
    mag = (np.abs(coef) + d // 2) // d
    return np.where(coef < 0, -mag, mag)


def codec_blocks(samples: np.ndarray, q: np.ndarray) -> np.ndarray:
    """FDCT -> quantise -> dequantise -> IDCT of uint8 blocks [n, 8, 8]: the decoded blocks, uint8."""
    x = samples.astype(np.int64) - 128
    rows = _fdct_1d([x[:, :, k] for k in range(8)], True)       # along each row
    x = np.stack(rows, axis=2)
    cols = _fdct_1d([x[:, k, :] for k in range(8)], False)      # along each column
    coef = np.stack(cols, axis=1)
    deq = quantize(coef, q) * q
    cols = _idct_1d([deq[:, k, :] for k in range(8)], True)     # pass 1: columns
    x = np.stack(cols, axis=1)
    rows = _idct_1d([x[:, :, k] for k in range(8)], False)      # pass 2: rows
    return np.clip(np.stack(rows, axis=2) + 128, 0, 255).astype(np.uint8)


def _codec_plane(plane: np.ndarray, q: np.ndarray) -> np.ndarray:
    h, w = plane.shape
    blocks = plane.reshape(h // 8, 8, w // 8, 8).transpose(0, 2, 1, 3).reshape(-1, 8, 8)
    return codec_blocks(blocks, q).reshape(h // 8, w // 8, 8, 8).transpose(0, 2, 1, 3).reshape(h, w)


def rgb_to_ycc(rgb: np.ndarray):
    r, g, b = (rgb[..., c].astype(np.int64) for c in range(3))
    half, offset = 1 << 15, 128 << 16
    y = (19595 * r + 38470 * g + 7471 * b + half) >> 16
    cb = (-11059 * r - 21709 * g + 32768 * b + offset + half - 1) >> 16
    cr = (32768 * r - 27439 * g - 5329 * b + offset + half - 1) >> 16
    return y, cb, cr


def ycc_to_rgb(y, cb, cr) -> np.ndarray:
    cb, cr = cb.astype(np.int64) - 128, cr.astype(np.int64) - 128
    half = 1 << 15
    r = y + ((91881 * cr + half) >> 16)
    g = y + ((-22554 * cb - 46802 * cr + half) >> 16)
    b = y + ((116130 * cb + half) >> 16)
    return np.clip(np.stack([r, g, b], axis=-1), 0, 255).astype(np.uint8)


def downsample_h2v2(plane: np.ndarray) -> np.ndarray:
    """2 x 2 averages of an even-sized plane with the alternating bias 1, 2 along each output row."""
    s = plane[0::2, 0::2] + plane[0::2, 1::2] + plane[1::2, 0::2] + plane[1::2, 1::2]
    bias = np.where(np.arange(s.shape[1]) % 2 == 0, 1, 2)
    return (s + bias) >> 2


def upsample_h2v2(c: np.ndarray, out_h: int, out_w: int) -> np.ndarray:
    """The decoder's chroma upsampling of the ceil(H / 2) x ceil(W / 2) plane `c` to out_h x out_w."""
    ch, cw = c.shape
    c = c.astype(np.int64)
    if cw <= 2:  # plain 2 x 2 replication
        return np.repeat(np.repeat(c, 2, 0), 2, 1)[:out_h, :out_w]
    i = np.arange(ch)
    above, below = c[np.maximum(i - 1, 0)], c[np.minimum(i + 1, ch - 1)]
    out = np.empty((2 * ch, 2 * cw), dtype=np.int64)
    for v, near in ((0, above), (1, below)):
        s = 3 * c + near                                   # column sums
        left = s[:, np.maximum(np.arange(cw) - 1, 0)]
        right = s[:, np.minimum(np.arange(cw) + 1, cw - 1)]
        out[v::2, 0::2] = (3 * s + left + 8) >> 4
        out[v::2, 1::2] = (3 * s + right + 7) >> 4
    return out[:out_h, :out_w]


def roundtrip(rgb: np.ndarray) -> np.ndarray:
    """np.asarray(Image.open(BytesIO(jpeg)).convert("RGB")) of Image.fromarray(rgb).save(jpeg, "JPEG"): uint8
    H x W x 3."""
    rgb = np.asarray(rgb)
    if rgb.dtype != np.uint8 or rgb.ndim != 3 or rgb.shape[2] != 3 or rgb.shape[0] < 1 or rgb.shape[1] < 1:
        raise ValueError(f"jpeg_oracle.roundtrip: a uint8 H x W x 3 image, got {rgb.dtype} {rgb.shape}")
    H, W = rgb.shape[:2]
    Hp, Wp = -(-H // 16) * 16, -(-W // 16) * 16
    ch, cw = -(-H // 2), -(-W // 2)
    # columns: the full-resolution rows are replicated to the MCU width before downsampling; rows: only to the
    # 2-row group, then the downsampled rows are replicated to the MCU height (so for an even H the padding
    # chroma rows repeat the average of rows H - 2 and H - 1, not of row H - 1 with itself)
    padded = np.pad(rgb, ((0, 2 * ch - H), (0, Wp - W), (0, 0)), mode="edge")
    y, cb, cr = rgb_to_ycc(padded)
    y = np.pad(y, ((0, Hp - 2 * ch), (0, 0)), mode="edge")
    y_dec = _codec_plane(y, LUMA_Q)[:H, :W].astype(np.int64)

    def chroma(c):
        return _codec_plane(np.pad(downsample_h2v2(c), ((0, Hp // 2 - ch), (0, 0)), mode="edge"), CHROMA_Q)[:ch, :cw]

    cb_dec, cr_dec = chroma(cb), chroma(cr)
    return ycc_to_rgb(y_dec, upsample_h2v2(cb_dec, H, W), upsample_h2v2(cr_dec, H, W))
