"""JPEG files for the decoder tests (parse_jpeg / read_jpeg / decode_model / decode_async).

Every file is written by libjpeg-turbo: Pillow's encoder for the usual flavours (samplings,
qualities, optimised tables, restart markers, CMYK, untransformed RGB, progressive), and
jpeg_write_coefficients through tests/libjpeg_pixels.py for 4:1:1, 4:4:0 and the saturated
coefficient sets of hard_content.py.  The content is deterministic integer arithmetic."""
from __future__ import annotations

import io
import os
import tempfile

import numpy as np

import libjpeg_pixels as lp
from render_images import make


def pixels(w: int, h: int, channels: int = 3, seed: int = 0) -> np.ndarray:
    """Ramps, a checker and pseudo-random texture: busy enough for long codes and FF bytes."""
    yy, xx = np.mgrid[0:h, 0:w].astype(np.int64)
    rnd = (xx * 7919 + yy * 104729 + seed * 31337) % 9973 % 97
    base = (xx * 3 + yy * 5 + rnd) % 256
    chans = [base, (base // 2 + 3 * rnd) % 256, 255 - base, ((xx ^ yy) * 13 + seed) % 256]
    return np.stack(chans[:channels], -1).astype(np.uint8)


def pillow_jpeg(w: int, h: int, mode: str = "RGB", seed: int = 0, **save) -> bytes:
    from PIL import Image
    if mode == "CMYK":
        im = Image.frombytes("CMYK", (w, h), pixels(w, h, 4, seed).tobytes())
    elif mode == "L":
        im = Image.fromarray(np.ascontiguousarray(pixels(w, h, 3, seed)[..., 0]))
    else:
        im = Image.fromarray(pixels(w, h, 3, seed))
    b = io.BytesIO()
    im.save(b, "JPEG", **save)
    return b.getvalue()


def coef_writer_jpeg(image) -> bytes:
    """The file jpeg_write_coefficients makes of a coefficient set (raises lp.LibjpegError for sets
    8-bit JPEG cannot code)."""
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "w.jpg")
        lp.decode(image, p)
        with open(p, "rb") as f:
            return f.read()


def libjpeg_coefficients(data: bytes):
    """jpeg_read_coefficients of a file (the oracle)."""
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "f.jpg")
        with open(p, "wb") as f:
            f.write(data)
        return lp.read_coefficients(p)


def flavours():
    """(name, bytes) of every sequential flavour the tests decode."""
    out = []
    for ss, sub in (("420", 2), ("422", 1), ("444", 0)):
        for q in (30, 75, 100):
            out.append((f"{ss}_q{q}", pillow_jpeg(250, 190, subsampling=sub, quality=q, seed=q)))
        out.append((f"{ss}_opt", pillow_jpeg(203, 149, subsampling=sub, quality=85, optimize=True)))
    for q in (30, 75, 100):
        out.append((f"gray_q{q}", pillow_jpeg(250, 190, "L", quality=q)))
    out.append(("gray_opt", pillow_jpeg(203, 149, "L", quality=85, optimize=True)))
    for w, h in ((1, 1), (17, 9), (33, 47), (250, 190)):
        out.append((f"size_{w}x{h}", pillow_jpeg(w, h, quality=80, seed=w)))
    out.append(("rst_rows1", pillow_jpeg(250, 190, quality=75, restart_marker_rows=1)))
    out.append(("rst_blocks7", pillow_jpeg(250, 190, quality=75, restart_marker_blocks=7)))
    out.append(("rst_gray", pillow_jpeg(97, 61, "L", quality=90, restart_marker_blocks=3)))
    out.append(("cmyk", pillow_jpeg(120, 80, "CMYK", quality=90)))
    out.append(("cmyk_rst", pillow_jpeg(120, 80, "CMYK", quality=60, restart_marker_blocks=5)))
    out.append(("keep_rgb", pillow_jpeg(120, 80, quality=90, keep_rgb=True, subsampling=0)))
    for ss in ("411", "440"):
        out.append((f"writer_{ss}", coef_writer_jpeg(make(75, 53, ss, "k50", "synth", 2))))
    return out + geometry_files()


# sizes of 24k +- 1 and 32k +- 1 and below 8, none a multiple of an MCU
GEOMETRY_SIZES = ((73, 49), (95, 31), (5, 7), (47, 65))


def geometry_files():
    """(name, bytes) of jpeg_write_coefficients files of every geometry of render_images.GEOMETRIES
    (at most 10 blocks per MCU, one interleaved scan), without restart markers, with one every 7
    MCUs and with one every MCU row."""
    import scan_files as sf
    from render_images import GEOMETRIES
    out = []
    for k, ss in enumerate(GEOMETRIES):
        w, h = GEOMETRY_SIZES[k % len(GEOMETRY_SIZES)]
        data = coef_writer_jpeg(make(w, h, ss, ("k50", "k90", "rand")[k % 3], ("synth", "saturated")[k % 2], 2 + k))
        out += [(f"writer_{ss}", data), (f"writer_{ss}_rst7", sf.rescan(data, restart_interval=7)),
                (f"writer_{ss}_rows1", sf.rescan(data, restart_rows=1))]
    return out


def per_component_files():
    """(name, bytes) of 3x3 and 4x4 luma (11 and 18 blocks per MCU), which libjpeg writes as one scan
    per component: the device decoders take single interleaved scans only, so these take the host
    route."""
    return [(f"writer_{ss}", coef_writer_jpeg(make(w, h, ss, "k50", c, 4))) for ss, w, h, c in
            (("33", 73, 47, "synth"), ("44", 95, 65, "saturated"))]


def hard_sets():
    """(name, coefficient set, bytes) of the hard_content sets the writer can code."""
    out = []
    for ss in ("420", "444", "gray", "411", "440"):
        for table, content in (("k90", "saturated"), ("k10", "saturated"), ("rand", "saturated"), ("k50", "synth")):
            im = make(61, 43, ss, table, content, 5)
            try:
                out.append((f"{ss}_{table}_{content}", im, coef_writer_jpeg(im)))
            except lp.LibjpegError:
                continue
    return out


def progressive():
    return [("prog_420", pillow_jpeg(250, 190, quality=75, progressive=True)),
            ("prog_gray", pillow_jpeg(97, 61, "L", quality=75, progressive=True))]
