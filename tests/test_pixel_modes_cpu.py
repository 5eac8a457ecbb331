"""Colour modes of the render (include/jpegqs_cuda.h JPEGQS_PIXELS_*) on the CPU: the render model with
mode "RGB" / "L" against Pillow's decode-then-convert, for CMYK, YCCK, grey, YCbCr and untransformed RGB
files at every scale; a numpy restatement of Pillow's conversions; the reader's colour space against
libjpeg's jpeg_read_header; the tool's Adobe marker for a transform-1 file; argument checks.  Nothing here
needs a GPU."""
import io
import os
import subprocess

import numpy as np
import pytest
from PIL import Image

import jpegqs_b200 as qs
from jpegqs_b200 import cuda
from jpegqs_b200.image import CoefImage, Component, JCS_CMYK, JCS_YCCK, JCS_YCbCr, JCS_RGB, JCS_GRAYSCALE

import decode_files as df
import libjpeg_cmyk as lc
import libjpeg_pixels as lp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "jpeg-quantsmooth_b200", "csrc", "jpegqs")


# ---- Pillow's conversions, restated in numpy -------------------------------------------------------
def muldiv255(a, b):
    t = a.astype(np.int64) * b + 128
    return ((t >> 8) + t) >> 8


def cmyk_to_rgb(cmyk):
    """Pillow's cmyk2rgb of a Pillow CMYK picture [..., 4]"""
    c = cmyk.astype(np.int64)
    nk = 255 - c[..., 3:4]
    return np.clip(nk - muldiv255(c[..., :3], nk), 0, 255).astype(np.uint8)


def rgb_to_l(rgb):
    """Pillow's rgb2l"""
    v = rgb.astype(np.int64)
    return ((v[..., 0] * 19595 + v[..., 1] * 38470 + v[..., 2] * 7471 + 0x8000) >> 16).astype(np.uint8)


def libjpeg_cmyk_to_pillow(px):
    """Pillow's CMYK picture from libjpeg's JCS_CMYK output (raw mode CMYK;I: inverted); libjpeg has
    already run ycck_cmyk_convert on a YCCK file's samples"""
    return (255 - px.astype(np.int64)).astype(np.uint8)


def pillow_reference(data, d, mode):
    """Image.open, draft at d > 1, convert(mode), as a numpy [H, W, C] array; None when Pillow's draft
    does not give libjpeg's 1/d size"""
    im = Image.open(io.BytesIO(data))
    w, h = im.size
    if d > 1:
        if w < d or h < d:
            return None
        im.draft(None, (w // d, h // d))
        if im.size != (-(-w // d), -(-h // d)):
            return None
    out = np.asarray(im.convert(mode))
    return out if out.ndim == 3 else out[..., None]


def libjpeg_reference(data, d, mode):
    """the same from libjpeg's scaled decode and the numpy conversions (any size)"""
    px = lc.decode_bytes(data, d)
    nc = px.shape[2]
    if nc == 4:
        rgb = cmyk_to_rgb(libjpeg_cmyk_to_pillow(px))
    elif nc == 1:
        rgb = np.repeat(px, 3, 2)
    else:
        rgb = px
    return rgb if mode == "RGB" else rgb_to_l(rgb)[..., None]


def model(data, d, mode, layout="hwc"):
    out = cuda.render_model(cuda.read_jpeg(data), layout=layout, scale_denom=d, mode=mode)
    return out if layout == "hwc" else np.moveaxis(out, 0, -1)


# ---- files ------------------------------------------------------------------------------------------
def segments(data):
    """(marker, payload) of the segments between SOI and the first SOS, and the rest from SOS"""
    i, out = 2, []
    while data[i + 1] != 0xDA:
        n = int.from_bytes(data[i + 2:i + 4], "big")
        out.append((data[i + 1], data[i + 4:i + 2 + n]))
        i += 2 + n
    return out, data[i:]


def rebuild(segs, rest):
    return b"\xff\xd8" + b"".join(b"\xff" + bytes([c]) + (len(p) + 2).to_bytes(2, "big") + p for c, p in segs) + rest


def with_markers(data, jfif=None, adobe=None):
    """the file with its APP0 and APP14 segments dropped, then a JFIF APP0 when jfif, and an Adobe APP14
    with transform `adobe` when it is an int"""
    segs, rest = segments(data)
    segs = [(c, p) for c, p in segs if c not in (0xE0, 0xEE)]
    head = []
    if jfif:
        head.append((0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00"))
    if adobe is not None:
        head.append((0xEE, b"Adobe" + b"\x00\x64\x00\x00\x00\x00" + bytes([adobe])))
    return rebuild(head + segs, rest)


def cmyk_file(w=67, h=45, seed=0, **save):
    return df.pillow_jpeg(w, h, "CMYK", seed, **save)


def _blocks(n, f, fmax):
    return -(-(-(-n * f // fmax)) // 8)


def ycck_file(w, h, factors, seed=0, colorspace=JCS_YCCK):
    """a 4-component file written by jpeg_write_coefficients in colorspace (libjpeg's Adobe marker:
    transform 2 for YCCK, 0 for CMYK) from seeded coefficients with these (h, v) factors"""
    rng = np.random.default_rng(seed)
    mh, mv = max(f[0] for f in factors), max(f[1] for f in factors)
    comps = []
    for c, (hs, vs) in enumerate(factors):
        wb, hb = _blocks(w, hs, mh), _blocks(h, vs, mv)
        coef = np.zeros((hb, wb, 64), np.int16)
        coef[..., 0] = rng.integers(-50, 50, (hb, wb))
        coef[..., 1:10] = rng.integers(-4, 5, (hb, wb, 9))
        quant = np.full(64, 6 + 2 * c, np.uint16)
        comps.append(Component(coef=coef, quant=quant, h_samp=hs, v_samp=vs, quant_tbl_no=c))
    return lc.write_coefficients(CoefImage(width=w, height=h, colorspace=colorspace, comps=comps))


YCCK_FACTORS = {"444": [(1, 1)] * 4, "y2k2": [(2, 2), (1, 1), (1, 1), (2, 2)], "k_alone": [(1, 1), (1, 1), (1, 1), (1, 2)]}


def cmyk_files():
    yield "q90", cmyk_file(quality=90)
    yield "q50", cmyk_file(71, 39, 1, quality=50)
    yield "q20_progressive", cmyk_file(64, 50, 2, quality=20, progressive=True)
    yield "restart", cmyk_file(90, 33, 3, quality=75, restart_marker_blocks=1) if _restart_ok() else cmyk_file(90, 33, 3)


def _restart_ok():
    try:
        df.pillow_jpeg(8, 8, "CMYK", 0, restart_marker_blocks=1)
        return True
    except TypeError:
        return False


def mode_files():
    """(name, file) pairs covering every colour space"""
    yield from cmyk_files()
    for name, fac in YCCK_FACTORS.items():
        yield "ycck_" + name, ycck_file(53, 37, fac, seed=len(name))
    base = cmyk_file(61, 29, 5, quality=80)
    yield "adobe1", with_markers(base, adobe=1)
    yield "adobe7", with_markers(base, adobe=7)
    yield "no_app14", with_markers(base)
    yield "grey", df.pillow_jpeg(45, 31, "L", 1, quality=70)
    yield "ycbcr420", df.pillow_jpeg(45, 31, "RGB", 2, quality=70)
    yield "ycbcr444", df.pillow_jpeg(37, 23, "RGB", 3, quality=90, subsampling=0)
    try:
        yield "keep_rgb", df.pillow_jpeg(37, 23, "RGB", 4, quality=90, keep_rgb=True)
    except TypeError:
        pass


FILES = dict(mode_files())


# ---- tests ------------------------------------------------------------------------------------------
def test_numpy_conversions_are_pillows():
    c, k = np.meshgrid(np.arange(256), np.arange(256), indexing="ij")
    cmyk = np.stack([c, (c * 7) % 256, 255 - c, k], -1).astype(np.uint8).reshape(256, 256, 4)
    want = np.asarray(Image.frombytes("CMYK", (256, 256), cmyk.tobytes()).convert("RGB"))
    assert np.array_equal(cmyk_to_rgb(cmyk), want)
    rgb = np.random.default_rng(1).integers(0, 256, (200, 300, 3), dtype=np.uint8)
    assert np.array_equal(rgb_to_l(rgb), np.asarray(Image.fromarray(rgb).convert("L")))
    # CMYK -> L is CMYK -> RGB -> L
    assert np.array_equal(np.asarray(Image.frombytes("CMYK", (256, 256), cmyk.tobytes()).convert("L")),
                          rgb_to_l(want))


@pytest.mark.parametrize("name", sorted(FILES))
@pytest.mark.parametrize("d", [1, 2, 4, 8])
@pytest.mark.parametrize("mode", ["RGB", "L"])
def test_render_model_mode_is_pillows_convert(name, d, mode):
    data = FILES[name]
    got = model(data, d, mode)
    want = pillow_reference(data, d, mode)
    if want is not None:
        assert got.shape == want.shape and np.array_equal(got, want), name
    assert np.array_equal(got, libjpeg_reference(data, d, mode)), name
    if d == 2:
        assert np.array_equal(model(data, d, mode, "chw"), got)


@pytest.mark.parametrize("d", [2, 4, 8])
def test_pictures_smaller_than_the_scale(d):
    """Pillow's draft divides by zero below d pixels; libjpeg's scaled decode is the reference"""
    for data in (cmyk_file(5, 3, 7, quality=80), ycck_file(3, 6, YCCK_FACTORS["y2k2"], seed=8)):
        for mode in ("RGB", "L"):
            assert np.array_equal(model(data, d, mode), libjpeg_reference(data, d, mode))


@pytest.mark.parametrize("ncomp", [3, 4])
@pytest.mark.parametrize("marker", ["none", "jfif", 0, 1, 2, 7])
def test_reader_colour_space_is_libjpegs(tmp_path, ncomp, marker):
    base = cmyk_file(24, 16, 9) if ncomp == 4 else df.pillow_jpeg(24, 16, "RGB", 9, subsampling=0)
    data = with_markers(base, jfif=marker == "jfif", adobe=marker if isinstance(marker, int) else None)
    p = tmp_path / "f.jpg"
    p.write_bytes(data)
    want = lp.read_coefficients(str(p)).colorspace
    assert cuda.read_jpeg(data).colorspace == want
    assert cuda.parse_jpeg(data)[0].colorspace == want
    expect = {3: {"none": JCS_YCbCr, "jfif": JCS_YCbCr, 0: JCS_RGB}, 4: {"none": JCS_CMYK, "jfif": JCS_CMYK, 0: JCS_CMYK}}
    assert want == expect[ncomp].get(marker, JCS_YCbCr if ncomp == 3 else JCS_YCCK)


@pytest.mark.skipif(not os.path.exists(EXE), reason="the tool is not built")
def test_tool_writes_transform_2_for_a_transform_1_file(tmp_path):
    """libjpeg reads Adobe transform 1 on 4 components as YCCK, and its writer then marks the file
    with transform 2; the tool does the same, and the pixels do not change"""
    src, out = tmp_path / "src.jpg", tmp_path / "out.jpg"
    src.write_bytes(with_markers(cmyk_file(40, 24, 11, quality=85), adobe=1))
    assert subprocess.run([EXE, "-n", "0", "-i", "0", str(src), str(out)]).returncode == 0
    segs, _ = segments(out.read_bytes())
    adobe = [p for c, p in segs if c == 0xEE and p[:5] == b"Adobe"]
    assert len(adobe) == 1 and adobe[0][11] == 2
    assert np.array_equal(np.asarray(Image.open(out).convert("RGB")), np.asarray(Image.open(src).convert("RGB")))


def test_mode_none_is_the_existing_model():
    for name in ("grey", "ycbcr420", "ycbcr444"):
        im = cuda.read_jpeg(FILES[name])
        for d in (1, 4):
            a = cuda.render_model(im, scale_denom=d)
            assert np.array_equal(a, cuda.render_model(im, scale_denom=d, mode=None))
            assert np.array_equal(a, cuda.render_model(im, scale_denom=d, mode="RGB"))
    with pytest.raises(cuda.QsError):
        cuda.render_model(cuda.read_jpeg(FILES["q90"]))              # 4 components: the file's own colour only


def test_argument_checks():
    im = cuda.read_jpeg(FILES["q90"])
    for bad in ("CMYK", "rgb", "YCbCr", 1, b"RGB"):
        with pytest.raises(ValueError):
            cuda.render_model(im, mode=bad)
    lib = cuda.load()
    arrays = [np.ascontiguousarray(c.coef) for c in im.comps]
    ci = cuda._Image()
    cuda._fill_image(ci, im, [a.ctypes.data for a in arrays], [])
    out = np.zeros(im.width * im.height * 3, np.uint8)
    assert lib.jpegqs_cuda_render_model_mode(ci, JCS_YCCK, 0, 0, 1, 1, out.ctypes.data) == 0
    for cs in (JCS_YCbCr, JCS_RGB, JCS_GRAYSCALE, 0, 9):        # not a 4-component colour space
        assert lib.jpegqs_cuda_render_model_mode(ci, cs, 0, 0, 1, 1, out.ctypes.data) == -2
    for mode in (-1, 3):
        assert lib.jpegqs_cuda_render_model_mode(ci, JCS_CMYK, 0, 0, 1, mode, out.ctypes.data) == -2
    assert lib.jpegqs_cuda_render_model_mode(ci, JCS_CMYK, 0, 0, 1, 0, out.ctypes.data) == -3
    assert qs.cuda._mode(None, "x") == 0 and qs.cuda._mode("RGB", "x") == 1 and qs.cuda._mode("L", "x") == 2
