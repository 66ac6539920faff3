"""The pixels of Pillow's JPEG save and reload, img.save(f, "JPEG", quality=q) then Image.open(f).convert("RGB"), in
NumPy int64, one function per step of libjpeg-turbo's integer chain (baseline, 4:2:0, ISLOW DCT both ways, fancy
upsampling).  Huffman coding is lossless, so no bitstream is needed: the round trip's bytes depend on this chain alone.

    roundtrip(rgb, quality)   (H, W, 3) uint8 -> (H, W, 3) uint8, any H, W >= 1

Two rules pin the edges, and the tests check that breaking either one loses Pillow's bytes:
  (a) the encoder pads the DOWNSAMPLED chroma plane to the iMCU by repeating its last real row, ceil(H / 2) - 1; the
      image itself is padded on the right by repeating its last column before downsampling;
  (b) the decoder upsamples fancily only when the chroma plane is more than 2 samples wide; a plane 1 or 2 samples
      wide is replicated 2 x 2.
Also the seeded test images (content()) and the grid of cases (grid()) the CPU and GPU tests and the golden share.
"""
from __future__ import annotations

import numpy as np

# ITU-T T.81 Annex K, tables K.1 and K.2, natural (row-major) order
LUMA = np.array([
    16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55,
    14, 13, 16, 24, 40, 57, 69, 56, 14, 17, 22, 29, 51, 87, 80, 62,
    18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
    49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99], dtype=np.int64)
CHROMA = np.array([
    17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99,
    24, 26, 56, 99, 99, 99, 99, 99, 47, 66, 99, 99, 99, 99, 99, 99] + [99] * 32, dtype=np.int64)

SCALEBITS, HALF = 16, 1 << 15
CONST_BITS, PASS1_BITS = 13, 2


def FIX(x: float) -> int:
    return int(x * (1 << SCALEBITS) + 0.5)


def FIX13(x: float) -> int:
    return int(x * (1 << CONST_BITS) + 0.5)


def descale(x, n: int):
    return (x + (1 << (n - 1))) >> n


# ------------------------------------------------------------------------------------------------------------ 1. tables
def quant_tables(quality: int) -> np.ndarray:
    """int64 [2, 64] natural order: Annex K scaled to the quality (jpeg_quality_scaling) and clamped to [1, 255]
    (baseline)."""
    q = int(quality)
    if not 1 <= q <= 100:
        raise ValueError(f"JPEG quality {quality!r} outside 1..100")
    s = 5000 // q if q < 50 else 200 - 2 * q
    return np.clip((np.stack([LUMA, CHROMA]) * s + 50) // 100, 1, 255)


# ------------------------------------------------------------------------------------------------------------ 2. colour
def rgb_to_ycc(rgb: np.ndarray) -> np.ndarray:
    """(H, W, 3) uint8 -> (3, H, W) int64 Y, Cb, Cr."""
    r, g, b = (rgb[..., i].astype(np.int64) for i in range(3))
    y = (FIX(0.299) * r + FIX(0.587) * g + FIX(0.114) * b + HALF) >> 16
    cb = (-FIX(0.16874) * r - FIX(0.33126) * g + FIX(0.5) * b + (128 << 16) + HALF - 1) >> 16
    cr = (FIX(0.5) * r - FIX(0.41869) * g - FIX(0.08131) * b + (128 << 16) + HALF - 1) >> 16
    return np.stack([y, cb, cr])


# ------------------------------------------------------------------------------------------------------------ 3. padding
def padded_size(H: int, W: int):
    """The image padded to whole 16 x 16 MCUs."""
    return -(-H // 16) * 16, -(-W // 16) * 16


def pad_mcu(plane: np.ndarray) -> np.ndarray:
    """(H, W) -> (Hp, Wp), the last row and the last column repeated."""
    H, W = plane.shape
    Hp, Wp = padded_size(H, W)
    return np.pad(plane, ((0, Hp - H), (0, Wp - W)), mode="edge")


# ------------------------------------------------------------------------------------------------------------ 4. chroma
def downsample_chroma(padded: np.ndarray, H: int) -> np.ndarray:
    """(Hp, Wp) padded chroma -> (Hp / 2, Wp / 2): (a + b + c + d + bias) >> 2 with the bias 1, 2, 1, 2 along the row, on
    the ceil(H / 2) rows the image reaches; the rest repeat the last of them (rule (a))."""
    s = padded[0::2, 0::2] + padded[0::2, 1::2] + padded[1::2, 0::2] + padded[1::2, 1::2]
    bias = np.where(np.arange(s.shape[1]) % 2 == 0, 1, 2)
    out = (s + bias) >> 2
    ch = -(-H // 2)
    out[ch:] = out[ch - 1]
    return out


# ------------------------------------------------------------------------------------------------------------ blocks
def to_blocks(plane: np.ndarray) -> np.ndarray:
    h, w = plane.shape
    return plane.reshape(h // 8, 8, w // 8, 8).swapaxes(1, 2)


def from_blocks(blocks: np.ndarray) -> np.ndarray:
    bh, bw = blocks.shape[:2]
    return blocks.swapaxes(1, 2).reshape(bh * 8, bw * 8)


# ------------------------------------------------------------------------------------------------------------ 5. FDCT
def _fdct_1d(d, first: bool):
    """One pass of jpeg_fdct_islow along the last axis; first: the row pass (outputs scaled up by 2^PASS1_BITS)."""
    x = [d[..., i] for i in range(8)]
    tmp0, tmp7 = x[0] + x[7], x[0] - x[7]
    tmp1, tmp6 = x[1] + x[6], x[1] - x[6]
    tmp2, tmp5 = x[2] + x[5], x[2] - x[5]
    tmp3, tmp4 = x[3] + x[4], x[3] - x[4]
    tmp10, tmp13 = tmp0 + tmp3, tmp0 - tmp3
    tmp11, tmp12 = tmp1 + tmp2, tmp1 - tmp2
    n = CONST_BITS - PASS1_BITS if first else CONST_BITS + PASS1_BITS
    out = [None] * 8
    if first:
        out[0], out[4] = (tmp10 + tmp11) << PASS1_BITS, (tmp10 - tmp11) << PASS1_BITS
    else:
        out[0], out[4] = descale(tmp10 + tmp11, PASS1_BITS), descale(tmp10 - tmp11, PASS1_BITS)
    z1 = (tmp12 + tmp13) * FIX13(0.541196100)
    out[2] = descale(z1 + tmp13 * FIX13(0.765366865), n)
    out[6] = descale(z1 - tmp12 * FIX13(1.847759065), n)
    z1, z2, z3, z4 = tmp4 + tmp7, tmp5 + tmp6, tmp4 + tmp6, tmp5 + tmp7
    z5 = (z3 + z4) * FIX13(1.175875602)
    tmp4, tmp5 = tmp4 * FIX13(0.298631336), tmp5 * FIX13(2.053119869)
    tmp6, tmp7 = tmp6 * FIX13(3.072711026), tmp7 * FIX13(1.501321110)
    z1, z2 = z1 * -FIX13(0.899976223), z2 * -FIX13(2.562915447)
    z3, z4 = z3 * -FIX13(1.961570560) + z5, z4 * -FIX13(0.390180644) + z5
    out[7] = descale(tmp4 + z1 + z3, n)
    out[5] = descale(tmp5 + z2 + z4, n)
    out[3] = descale(tmp6 + z2 + z3, n)
    out[1] = descale(tmp7 + z1 + z4, n)
    return np.stack(out, axis=-1)


def fdct_islow(samples: np.ndarray) -> np.ndarray:
    """(..., 8, 8) samples (0..255) -> coefficients scaled by 8: rows, then columns, of sample - 128."""
    d = _fdct_1d(samples - 128, True)
    return _fdct_1d(d.swapaxes(-1, -2), False).swapaxes(-1, -2)


# ------------------------------------------------------------------------------------------------------------ 6. quantise
def quantize(coef: np.ndarray, qt: np.ndarray) -> np.ndarray:
    """sign(x) ((|x| + d / 2) / d), d = 8 qval (the FDCT's outputs carry a factor 8)."""
    d = (8 * qt).reshape(8, 8)
    return np.sign(coef) * ((np.abs(coef) + d // 2) // d)


# ------------------------------------------------------------------------------------------------------------ 7. IDCT
def _idct_1d(d, first: bool):
    """One pass of jpeg_idct_islow along the last axis; first: the column pass on dequantised coefficients."""
    x = [d[..., i] for i in range(8)]
    z2, z3 = x[2], x[6]
    z1 = (z2 + z3) * FIX13(0.541196100)
    tmp2 = z1 - z3 * FIX13(1.847759065)
    tmp3 = z1 + z2 * FIX13(0.765366865)
    tmp0, tmp1 = (x[0] + x[4]) << CONST_BITS, (x[0] - x[4]) << CONST_BITS
    tmp10, tmp13 = tmp0 + tmp3, tmp0 - tmp3
    tmp11, tmp12 = tmp1 + tmp2, tmp1 - tmp2
    tmp0, tmp1, tmp2, tmp3 = x[7], x[5], x[3], x[1]
    z1, z2, z3, z4 = tmp0 + tmp3, tmp1 + tmp2, tmp0 + tmp2, tmp1 + tmp3
    z5 = (z3 + z4) * FIX13(1.175875602)
    tmp0, tmp1 = tmp0 * FIX13(0.298631336), tmp1 * FIX13(2.053119869)
    tmp2, tmp3 = tmp2 * FIX13(3.072711026), tmp3 * FIX13(1.501321110)
    z1, z2 = z1 * -FIX13(0.899976223), z2 * -FIX13(2.562915447)
    z3, z4 = z3 * -FIX13(1.961570560) + z5, z4 * -FIX13(0.390180644) + z5
    tmp0, tmp1, tmp2, tmp3 = tmp0 + z1 + z3, tmp1 + z2 + z4, tmp2 + z2 + z3, tmp3 + z1 + z4
    n = CONST_BITS - PASS1_BITS if first else CONST_BITS + PASS1_BITS + 3
    return np.stack([descale(v, n) for v in (tmp10 + tmp3, tmp11 + tmp2, tmp12 + tmp1, tmp13 + tmp0,
                                             tmp13 - tmp0, tmp12 - tmp1, tmp11 - tmp2, tmp10 - tmp3)], axis=-1)


def idct_islow(q: np.ndarray, qt: np.ndarray) -> np.ndarray:
    """(..., 8, 8) quantised coefficients -> samples: dequantise, columns, then rows, clamp(v + 128, 0, 255)."""
    d = _idct_1d((q * qt.reshape(8, 8)).swapaxes(-1, -2), True).swapaxes(-1, -2)
    return np.clip(_idct_1d(d, False) + 128, 0, 255)


def code_plane(plane: np.ndarray, qt: np.ndarray) -> np.ndarray:
    """Steps 5 to 7 on a plane of whole blocks."""
    return from_blocks(idct_islow(quantize(fdct_islow(to_blocks(plane)), qt), qt))


# ------------------------------------------------------------------------------------------------------------ 8. upsample
EVEN_BIAS, ODD_BIAS = 8, 7


def fancy_upsample(c: np.ndarray, above: np.ndarray, below: np.ndarray) -> np.ndarray:
    """h2v2_fancy_upsample of c (ch, cw), with the context rows above and below each row -> (2 ch, 2 cw): column sums
    3 this + other, then even outputs (3 sum + left + 8) >> 4 and odd ones (3 sum + right + 7) >> 4, the first even and
    the last odd output (4 sum + 8) >> 4 and (4 sum + 7) >> 4."""
    out = np.empty((2 * c.shape[0], 2 * c.shape[1]), dtype=np.int64)
    for r0, other in ((0, above), (1, below)):
        s = 3 * c + other
        left = np.concatenate([s[:, :1], s[:, :-1]], axis=1)
        right = np.concatenate([s[:, 1:], s[:, -1:]], axis=1)
        even, odd = (3 * s + left + EVEN_BIAS) >> 4, (3 * s + right + ODD_BIAS) >> 4
        even[:, 0] = (4 * s[:, 0] + EVEN_BIAS) >> 4
        odd[:, -1] = (4 * s[:, -1] + ODD_BIAS) >> 4
        out[r0::2, 0::2], out[r0::2, 1::2] = even, odd
    return out


def upsample_chroma(plane: np.ndarray, H: int, W: int) -> np.ndarray:
    """A decoded chroma plane -> (H, W), from its ceil(H / 2) x ceil(W / 2) real samples: fancy_upsample with the row
    above for the upper output row and the row below for the lower one, the edge row itself at the top and the bottom;
    a plane at most 2 samples wide is replicated 2 x 2 instead (rule (b))."""
    ch, cw = -(-H // 2), -(-W // 2)
    c = plane[:ch, :cw]
    if cw <= 2:
        return np.repeat(np.repeat(c, 2, axis=0), 2, axis=1)[:H, :W]
    above = np.concatenate([c[:1], c[:-1]])
    below = np.concatenate([c[1:], c[-1:]])
    return fancy_upsample(c, above, below)[:H, :W]


# ------------------------------------------------------------------------------------------------------------ 9. colour
def ycc_to_rgb(y: np.ndarray, cb: np.ndarray, cr: np.ndarray) -> np.ndarray:
    cb, cr = cb - 128, cr - 128
    r = y + ((FIX(1.402) * cr + HALF) >> 16)
    g = y + ((-FIX(0.34414) * cb - FIX(0.71414) * cr + HALF) >> 16)
    b = y + ((FIX(1.772) * cb + HALF) >> 16)
    return np.clip(np.stack([r, g, b], axis=-1), 0, 255).astype(np.uint8)


# ------------------------------------------------------------------------------------------------------------ the chain
def roundtrip(rgb: np.ndarray, quality: int = 75) -> np.ndarray:
    """Pillow's save(f, "JPEG", quality=quality) then Image.open(f).convert("RGB"): (H, W, 3) uint8 -> (H, W, 3) uint8."""
    rgb = np.asarray(rgb)
    if rgb.dtype != np.uint8 or rgb.ndim != 3 or rgb.shape[2] != 3 or min(rgb.shape[:2]) < 1:
        raise ValueError(f"expected (H, W, 3) uint8 with H, W >= 1, got {rgb.dtype} {rgb.shape}")
    H, W = rgb.shape[:2]
    qt = quant_tables(quality)
    y, cb, cr = (pad_mcu(p) for p in rgb_to_ycc(rgb))
    y = code_plane(y, qt[0])
    cb, cr = (code_plane(downsample_chroma(p, H), qt[1]) for p in (cb, cr))
    return ycc_to_rgb(y[:H, :W], upsample_chroma(cb, H, W), upsample_chroma(cr, H, W))


# ------------------------------------------------------------------------------------------------------------ test images
KINDS = ("noise", "zeros", "full", "checker", "blocky", "smooth")


def content(kind: str, H: int, W: int, seed: int) -> np.ndarray:
    """A seeded (H, W, 3) uint8 image: uniform noise, constant 0 or 255, a 0 / 255 pixel checkerboard, random 4 x 4
    blocks with noise on top, or a smooth gradient with a little noise."""
    rng = np.random.default_rng(seed)
    if kind == "noise":
        return rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    if kind in ("zeros", "full"):
        return np.full((H, W, 3), 0 if kind == "zeros" else 255, dtype=np.uint8)
    if kind == "checker":
        c = ((np.arange(H)[:, None] + np.arange(W)[None, :]) % 2 * 255).astype(np.uint8)
        return np.repeat(c[..., None], 3, axis=2)
    if kind == "blocky":
        base = rng.integers(0, 256, (-(-H // 4), -(-W // 4), 3))
        base = np.repeat(np.repeat(base, 4, axis=0), 4, axis=1)[:H, :W]
        return np.clip(base + rng.integers(-12, 13, (H, W, 3)), 0, 255).astype(np.uint8)
    if kind == "smooth":
        yy, xx = np.meshgrid(np.linspace(0, 1, H), np.linspace(0, 1, W), indexing="ij")
        ph = rng.uniform(0, 2 * np.pi, 3)
        v = 127.5 + 110 * np.sin(np.stack([3 * yy + 2 * xx, 2 * yy - 3 * xx, 4 * xx * yy], axis=-1) + ph)
        return np.clip(v + rng.normal(0, 2, (H, W, 3)), 0, 255).astype(np.uint8)
    raise ValueError(f"unknown content kind {kind!r}")


def grid(n: int = 240, seed: int = 2026):
    """(H, W, quality, kind, seed) cases: n random ones with H, W in 1..99 and quality in 1..100 over every kind, then
    every H, W in 1..5 against a few widths, odd x even shapes, and 85^2, 255 x 257 and 256^2."""
    rng = np.random.default_rng(seed)
    cases = []
    for i in range(n):
        H, W = (int(v) for v in rng.integers(1, 100, 2))
        cases.append((H, W, int(rng.integers(1, 101)), KINDS[i % len(KINDS)], 1000 + i))
    for i, (H, W) in enumerate([(h, w) for h in range(1, 6) for w in (1, 2, 3, 4, 5, 17, 32)]
                               + [(w, h) for h in range(1, 6) for w in (17, 32)]):
        cases.append((H, W, (7, 50, 75, 100)[i % 4], KINDS[i % len(KINDS)], 2000 + i))
    for i, (H, W) in enumerate([(15, 16), (16, 15), (17, 18), (33, 48), (47, 31), (63, 64), (65, 2)]):
        cases.append((H, W, 75, KINDS[i % len(KINDS)], 3000 + i))
    for i, (H, W) in enumerate([(85, 85), (255, 257), (256, 256)]):
        for j, kind in enumerate(("noise", "smooth", "blocky")):
            cases.append((H, W, (75, 30, 95)[j], kind, 4000 + 3 * i + j))
    return cases
