"""Image content and quant tables that the synthetic generator (jpegqs_b200.synth) never makes.

`synth.make_image` draws pixels in about [24, 232], so no value the smoothing kernel, the IDCT
or the forward DCTs clamp ever reaches a clamp.  Real JPEGs are full of such content: black
letterbox bars (DC -1024, which must come out as -1023), clipped highlights, black-on-white
strokes.  `saturated_pixels` draws it, with the same deterministic integer arithmetic as synth
(counter hashes, no floating point before the exact integer DCT of `synth.quantize_blocks`):

  * letterbox bars of 0 at the top and bottom, a 255 pillar at the right,
  * 1-pixel strokes at full contrast (0 on 255),
  * a Nyquist checker of 0 / 255,
  * ramps that wrap from 255 to 0,
  * flat 8x8 blocks at 0, 255 or mid-grey,
  * patches of the synthetic content in between.

`with_dequant_edge` adds coefficients whose de-quantized value sits exactly at the ends of the
reference's legal range [-2048, 2047] (quantsmooth.h:2602), or one past it (`stop`).
"""
from __future__ import annotations

import numpy as np

from jpegqs_b200 import synth
from jpegqs_b200.image import CoefImage, Component, JCS_GRAYSCALE, JCS_YCbCr, blocks_for

SAMPLINGS = ("gray", "444", "422", "420", "440")
_SAMP = {"444": (1, 1), "422": (2, 1), "420": (2, 2), "440": (1, 2)}

# Every other sampling libjpeg codes with integral ratios, as (h, v) factors of Y / Cb / Cr: factors
# of 3 (box up-sampling by 3, the clipped last cell of the JOINT_YUV down-sample), of 4 on either
# axis (10 blocks per MCU at 4x2, MCU rows of 4 block rows), more than 10 blocks per MCU (33, 44),
# a 16x8 MCU whose ratios are all 1, chroma sampled above luma, and two chroma of different factors;
# and grey files whose SOF gives the one component factors other than 1x1 (a scan of one component
# has 1-block MCUs, but the picture is still the component's sample grid).
FACTORS = {"411": ((4, 1), (1, 1), (1, 1)),
           "31": ((3, 1), (1, 1), (1, 1)), "13": ((1, 3), (1, 1), (1, 1)),
           "32": ((3, 2), (1, 1), (1, 1)), "23": ((2, 3), (1, 1), (1, 1)),
           "410": ((4, 2), (1, 1), (1, 1)), "14": ((1, 4), (1, 1), (1, 1)), "24": ((2, 4), (1, 1), (1, 1)),
           "33": ((3, 3), (1, 1), (1, 1)), "44": ((4, 4), (1, 1), (1, 1)),
           "21_21_21": ((2, 1), (2, 1), (2, 1)), "11_22_22": ((1, 1), (2, 2), (2, 2)),
           "22_21_12": ((2, 2), (2, 1), (1, 2)), "41_21_21": ((4, 1), (2, 1), (2, 1)),
           "g22": ((2, 2),), "g31": ((3, 1),), "g14": ((1, 4),), "g44": ((4, 4),)}
GEOMETRIES = tuple(k for k in FACTORS if k != "411")


def factors(subsampling: str):
    """(h, v) per component of a sampling name of SAMPLINGS or FACTORS."""
    if subsampling == "gray":
        return ((1, 1),)
    if subsampling in _SAMP:
        return (_SAMP[subsampling], (1, 1), (1, 1))
    return FACTORS[subsampling]


def saturated_pixels(c: int, y0: int, y1: int, width: int, sx: int, sy: int, seed: int,
                     height: int, full_width: int) -> np.ndarray:
    """Pixels of component c, rows [y0, y1) x [0, width), int64 in [0, 255]; (sx, sy) the
    sub-sampling relative to luma, (full_width, height) the image size in luma pixels."""
    Y = (np.arange(y0, y1, dtype=np.int64) * sy)[:, None]
    X = (np.arange(width, dtype=np.int64) * sx)[None, :]
    Y, X = np.broadcast_arrays(Y, X)
    # 48x48 luma-pixel cells, each of one kind; the kind comes from a hash of the cell
    kind = (synth._hash_noise(X // 48, Y // 48, c, seed) % np.uint32(6)).astype(np.int64)
    strokes = np.where(((X % 7) == 3) | ((Y % 9) == 4), 0, 255)
    checker = ((X + Y) & 1) * 255
    ramp = (X * 5 + Y * 3 + 37 * c + seed) % 256                     # wraps 255 -> 0
    h8 = synth._hash_noise(X // 8, Y // 8, c + 7, seed)
    flat = np.choose((h8 % np.uint32(3)).astype(np.int64), [0, 255, 128])
    smooth = synth.pixels(c, y0, y1, width, sx, sy, seed)
    v = np.choose(kind, [strokes, checker, ramp, flat, smooth, 255 - strokes])
    bar = max(8, height // 12)
    v = np.where((Y < bar) | (Y >= height - bar), 0 if c == 0 else 128, v)   # letterbox
    v = np.where(X >= full_width - 24, 255 if c == 0 else 0, v)               # pillar
    return v.astype(np.int64)


def make_image(width: int, height: int, subsampling: str, tables, content: str = "synth",
               seed: int = 12345, chunk_rows: int = 64) -> CoefImage:
    """An image of either content ('synth': synth.pixels; 'saturated': saturated_pixels),
    quantized with tables = (luma table, chroma table); subsampling is a name of SAMPLINGS or
    FACTORS, or a sequence of (h, v) per component."""
    samp = factors(subsampling) if isinstance(subsampling, str) else tuple(subsampling)
    cs = JCS_GRAYSCALE if len(samp) == 1 else JCS_YCbCr
    mh, mv = max(s[0] for s in samp), max(s[1] for s in samp)
    comps = []
    for c, (hs, vs) in enumerate(samp):
        wb, hb = blocks_for(width, hs, mh), blocks_for(height, vs, mv)
        q = np.asarray(tables[0 if c == 0 else 1], dtype=np.uint16).copy()
        coef = np.empty((hb, wb, 64), dtype=np.int16)
        for r0 in range(0, hb, chunk_rows):
            r1 = min(hb, r0 + chunk_rows)
            if content == "saturated":
                px = saturated_pixels(c, r0 * 8, r1 * 8, wb * 8, mh // hs, mv // vs, seed, height, width)
            else:
                px = synth.pixels(c, r0 * 8, r1 * 8, wb * 8, mh // hs, mv // vs, seed)
            coef[r0:r1] = synth.quantize_blocks(px, q)
        comps.append(Component(coef=coef, quant=q, h_samp=hs, v_samp=vs, quant_tbl_no=0 if c == 0 else 1))
    return CoefImage(width=width, height=height, colorspace=cs, comps=comps)


# ---- quant tables ---------------------------------------------------------------------------

def annex_k(quality: int):
    return synth.quality_table(synth.ANNEX_K_LUMA, quality), synth.quality_table(synth.ANNEX_K_CHROMA, quality)


def flat(value: int):
    """Every anti-diagonal uniform: the schedule is uniform chunks only."""
    t = np.full(64, value, dtype=np.uint16)
    return t, t.copy()


def random_tables(seed: int):
    """Seeded values 1..2047 (legal in 16-bit DQT tables; the OR stays below 0x800)."""
    rng = np.random.RandomState(seed)
    return tuple(rng.randint(1, 2048, size=64).astype(np.uint16) for _ in range(2))


def part_uniform():
    """Equal on anti-diagonals 2, 5, 8, 11 and 13 only, distinct values elsewhere: uniform
    and plain chunks in one schedule."""
    u, v = np.meshgrid(np.arange(8), np.arange(8))
    s = (u + v).reshape(64)
    t = (20 + 3 * np.arange(64)).astype(np.uint16)
    for d in (2, 5, 8, 11, 13):
        t[s == d] = 16 + 6 * d
    c = t.copy()
    c[s == 5] = 7
    return t, c


TABLES = {"k10": annex_k(10), "k50": annex_k(50), "k90": annex_k(90), "k97": annex_k(97),
          "flat": flat(12), "rand": random_tables(2047), "diag": part_uniform()}


def with_dequant_edge(im: CoefImage, stop: bool, comp: int = 1) -> CoefImage:
    """A copy of im whose component `comp` carries coefficients de-quantized to exactly 2047
    and -2048 (the ends of the legal range) in a few blocks; stop=True puts +2048 (one past
    the end) in one of them, which makes the reference stop at that component."""
    out = im.clone()
    c = out.comps[comp]
    c.quant = c.quant.copy()
    c.quant[9], c.quant[17] = 23, 32                     # 23 * 89 = 2047, 32 * 64 = 2048
    if comp > 0:
        c.quant_tbl_no = 2                               # a table slot of its own
    # every other block stays inside the legal range with the new quant values
    c.coef = c.coef.copy()
    c.coef[..., 9] = np.clip(c.coef[..., 9], -89, 89)
    c.coef[..., 17] = np.clip(c.coef[..., 17], -64, 63)
    hb, wb = c.hblk, c.wblk
    for k, (by, bx) in enumerate([(0, 0), (hb // 2, wb // 3), (hb - 1, wb - 1), (hb // 3, wb // 2)]):
        c.coef[by, bx, 9] = 89 if k % 2 == 0 else -89
        c.coef[by, bx, 17] = -64
    if stop:
        c.coef[hb // 2, wb // 3, 17] = 64
    return out
