"""The compressor of jpegqs_cuda_compress_async, without a GPU: compress_model (the device's per-block
functions and the encoder on one CPU thread) writes exactly the bytes of Pillow's
Image.fromarray(P).save(f, "JPEG", quality=q, subsampling=s, optimize=o), over a seeded sweep of grey
and RGB pictures from 1 x 1 to about 300 a side, every sampling, quality and optimize setting, on
random, gradient, saturated and hard content; also with libjpeg-turbo's SIMD code switched off.  A
numpy restatement of libjpeg's compressor equals the model, and five plausible mistakes in it each give
a file Pillow does not write.  The model's files read back with their own coefficients and tables.
Also the argument checks of the Python keywords and of the C calls without a context."""
import ctypes as C
import io
import os
import subprocess
import sys

import numpy as np
import pytest

Image = pytest.importorskip("PIL.Image")
ImageFile = pytest.importorskip("PIL.ImageFile")
# with optimize, Pillow gives libjpeg one output buffer of max(MAXBLOCK, about W * H) bytes and
# fails on files larger than that (noise at high quality); a larger buffer changes no byte
ImageFile.MAXBLOCK = 1 << 28

import hard_content as hc
import libjpeg_pixels as lp
from jpegqs_b200 import cuda
from jpegqs_b200.image import CoefImage, Component, JCS_GRAYSCALE, JCS_YCbCr

QUALITIES = (1, 5, 10, 24, 25, 50, 75, 85, 95, 100)
SUBS = ("4:4:4", "4:2:2", "4:2:0")
EDGE = (1, 2, 7, 8, 9, 15, 16, 17, 18, 22, 23, 24, 31, 32, 33)


def pillow(a, quality, subsampling, optimize):
    b = io.BytesIO()
    Image.fromarray(a if a.shape[2] == 3 else a[:, :, 0]).save(b, "JPEG", quality=quality, subsampling=subsampling,
                                                               optimize=optimize)
    return b.getvalue()


def content(rng, h, w, c, kind, seed=0):
    if kind == "random":
        return rng.randint(0, 256, (h, w, c)).astype(np.uint8)
    if kind == "gradient":
        yy, xx = np.indices((h, w))
        g = [(xx * 255 // max(w - 1, 1) + k * 40) % 256 for k in range(c)]
        g = [(g[k] + yy * (k + 1) * 3) % 256 for k in range(c)]
        return np.stack(g, 2).astype(np.uint8)
    if kind == "saturated":
        return (rng.randint(0, 2, (h, w, c)) * 255).astype(np.uint8)
    if kind == "normal":
        return np.clip(rng.normal(128, 90, (h, w, c)), 0, 255).astype(np.uint8)
    # hard_content's letterbox bars, strokes, checkers, wrapping ramps and flat blocks
    return np.stack([hc.saturated_pixels(k, 0, h, w, 1, 1, seed, h, w) for k in range(c)], 2).astype(np.uint8)


KINDS = ("random", "gradient", "saturated", "normal", "hard")


def cases():
    """(picture, quality, subsampling, optimize): a seeded sweep"""
    rng = np.random.RandomState(2026)
    out = []
    for i in range(420):
        if i < 120:                                   # both sides of the 8 and 16 boundaries
            h, w = EDGE[rng.randint(len(EDGE))], EDGE[rng.randint(len(EDGE))]
        elif i % 12 == 0:
            h, w = rng.randint(150, 301, 2)
        else:
            h, w = rng.randint(1, 100, 2)
        c = 1 if i % 4 == 0 else 3
        a = content(rng, int(h), int(w), c, KINDS[i % len(KINDS)], seed=i)
        out.append((a, QUALITIES[i % len(QUALITIES)], SUBS[(i // 2) % 3], bool((i // 6) % 2)))
    # fact of the edges: at 18 x 22 4:2:0 the bottom chroma rows repeat the last down-sampled row
    a = content(np.random.RandomState(18), 22, 18, 3, "random")
    out += [(a, q, "4:2:0", o) for q in (50, 95) for o in (False, True)]
    return out


CASES = cases()


@pytest.mark.parametrize("i", range(0, len(CASES), 20))
def test_model_equals_pillow(i):
    for a, q, s, o in CASES[i:i + 20]:
        assert cuda.compress_model(a, q, s, o) == pillow(a, q, s, o), (a.shape, q, s, o)


def test_numeric_subsampling_and_grey_2d():
    a = content(np.random.RandomState(3), 37, 41, 3, "random")
    for k, s in enumerate(SUBS):
        assert cuda.compress_model(a, 80, k) == cuda.compress_model(a, 80, s) == pillow(a, 80, s, False)
    g = a[:, :, 0]
    assert cuda.compress_model(g, 60, "4:2:2") == pillow(g[:, :, None], 60, "4:2:2", False)


_SIMD_OFF = r'''
import io, sys
import numpy as np
from PIL import Image, ImageFile
ImageFile.MAXBLOCK = 1 << 28
d = np.load(sys.argv[1])
out = []
for k in range(int(d["n"])):
    a = d[f"a{k}"]
    b = io.BytesIO()
    Image.fromarray(a if a.shape[2] == 3 else a[:, :, 0]).save(b, "JPEG", quality=int(d[f"q{k}"]),
        subsampling=str(d[f"s{k}"]), optimize=bool(d[f"o{k}"]))
    out.append(b.getvalue())
open(sys.argv[2], "wb").write(b"".join(len(x).to_bytes(8, "little") + x for x in out))
'''


def test_model_equals_pillow_without_simd(tmp_path):
    """libjpeg-turbo's C code is the contract: its SIMD paths switched off give the same files"""
    sub = CASES[::7]
    arrays = {"n": len(sub)}
    for k, (a, q, s, o) in enumerate(sub):
        arrays.update({f"a{k}": a, f"q{k}": q, f"s{k}": s, f"o{k}": int(o)})
    np.savez(tmp_path / "in.npz", **arrays)
    script = tmp_path / "save.py"
    script.write_text(_SIMD_OFF)
    env = dict(os.environ, JSIMD_FORCENONE="1")
    subprocess.run([sys.executable, str(script), str(tmp_path / "in.npz"), str(tmp_path / "out.bin")], check=True, env=env)
    raw, pos = (tmp_path / "out.bin").read_bytes(), 0
    for a, q, s, o in sub:
        n = int.from_bytes(raw[pos:pos + 8], "little")
        assert cuda.compress_model(a, q, s, o) == raw[pos + 8:pos + 8 + n], (a.shape, q, s, o)
        pos += 8 + n


# ---- a numpy restatement of libjpeg's compressor, and mistakes it could make ----
LUMA = np.array([16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
                 14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
                 49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99], np.int64)
CHROMA = np.full(64, 99, np.int64)
CHROMA[[0, 1, 2, 3, 8, 9, 10, 11, 16, 17, 18, 24, 25]] = [17, 18, 24, 47, 18, 21, 26, 66, 24, 26, 56, 47, 66]


def fix(x):
    return int(x * 65536 + 0.5)


def quant_table(base, q, baseline=True):
    scale = 5000 // q if q < 50 else 200 - 2 * q
    return np.clip((base * scale + 50) // 100, 1, 255 if baseline else 32767)


def fdct_1d(d, pass1):
    """jfdctint.c's jpeg_fdct_islow along the last axis"""
    t0, t7 = d[..., 0] + d[..., 7], d[..., 0] - d[..., 7]
    t1, t6 = d[..., 1] + d[..., 6], d[..., 1] - d[..., 6]
    t2, t5 = d[..., 2] + d[..., 5], d[..., 2] - d[..., 5]
    t3, t4 = d[..., 3] + d[..., 4], d[..., 3] - d[..., 4]
    t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
    sh = 11 if pass1 else 15

    def ds(x, n):
        return (x + (1 << (n - 1))) >> n
    o = [None] * 8
    o[0], o[4] = ((t10 + t11) << 2, (t10 - t11) << 2) if pass1 else (ds(t10 + t11, 2), ds(t10 - t11, 2))
    z1 = (t12 + t13) * 4433
    o[2], o[6] = ds(z1 + t13 * 6270, sh), ds(z1 - t12 * 15137, sh)
    z5 = (t4 + t5 + t6 + t7) * 9633
    z1, z2 = -(t4 + t7) * 7373, -(t5 + t6) * 20995
    z3, z4 = -(t4 + t6) * 16069 + z5, -(t5 + t7) * 3196 + z5
    o[7], o[5] = ds(t4 * 2446 + z1 + z3, sh), ds(t5 * 16819 + z2 + z4, sh)
    o[3], o[1] = ds(t6 * 25172 + z2 + z3, sh), ds(t7 * 12299 + z1 + z4, sh)
    return np.stack(o, -1)


def restated(a, q, s, o, mutant=None):
    """(file bytes, coefficient arrays, tables) of libjpeg's compressor restated in numpy; mutant names a
    mistake: 'bottom_clamp' (bottom chroma from clamped full-resolution rows), 'right_repeat' (right
    chroma from a repeated down-sampled column), 'const_bias', 'no_baseline', 'truncate'"""
    h, w, c = a.shape
    p = a.astype(np.int64)
    if c == 3:
        r, g, b = p[..., 0], p[..., 1], p[..., 2]
        planes = [(fix(0.299) * r + fix(0.587) * g + fix(0.114) * b + 32768) >> 16,
                  (-fix(0.16874) * r - fix(0.33126) * g + fix(0.5) * b + (128 << 16) + 32767) >> 16,
                  (fix(0.5) * r - fix(0.41869) * g - fix(0.08131) * b + (128 << 16) + 32767) >> 16]
    else:
        planes = [p[..., 0]]
    si = SUBS.index(s) if isinstance(s, str) else s
    lh, lv = (1, 1) if c == 1 or si == 0 else (2, 1) if si == 1 else (2, 2)
    tabs = [quant_table(LUMA, q, mutant != "no_baseline"), quant_table(CHROMA, q, mutant != "no_baseline")]
    arrays, comps = [], []
    for k, pl in enumerate(planes):
        hs, vs = (lh, lv) if k == 0 else (1, 1)
        sx, sy = lh // hs, lv // vs
        dw, dh = -(-w * hs // lh), -(-h * vs // lv)
        wb, hb = -(-dw // 8), -(-dh // 8)
        cx, cy = np.arange(wb * 8), np.arange(hb * 8)
        if mutant != "bottom_clamp":
            cy = np.minimum(cy, dh - 1)
        if mutant == "right_repeat":
            cx = np.minimum(cx, dw - 1)
        x0, x1 = np.minimum(cx * sx, w - 1), np.minimum(cx * sx + 1, w - 1)
        y0, y1 = np.minimum(cy * sy, h - 1), np.minimum(cy * sy + 1, h - 1)
        if sx == 1:
            v = pl[np.ix_(y0, x0)]
        elif sy == 1:
            bias = 0 if mutant == "const_bias" else cx & 1
            v = (pl[np.ix_(y0, x0)] + pl[np.ix_(y0, x1)] + bias) >> 1
        else:
            bias = 1 if mutant == "const_bias" else 1 + (cx & 1)
            v = (pl[np.ix_(y0, x0)] + pl[np.ix_(y0, x1)] + pl[np.ix_(y1, x0)] + pl[np.ix_(y1, x1)] + bias) >> 2
        blk = (v - 128).reshape(hb, 8, wb, 8).transpose(0, 2, 1, 3)
        blk = fdct_1d(blk, True)
        blk = fdct_1d(blk.swapaxes(-1, -2), False).swapaxes(-1, -2)
        t = blk.reshape(hb, wb, 64)
        qq = tabs[min(k, 1)] * 8
        mag = np.abs(t) // qq if mutant == "truncate" else (np.abs(t) + qq // 2) // qq
        arrays.append((np.sign(t) * mag).astype(np.int16))
        comps.append(Component(coef=arrays[-1], quant=tabs[min(k, 1)].astype(np.uint16), h_samp=hs if c == 3 else 1,
                               v_samp=vs if c == 3 else 1, quant_tbl_no=min(k, 1)))
    image = CoefImage(width=w, height=h, colorspace=JCS_YCbCr if c == 3 else JCS_GRAYSCALE, comps=comps)
    prefix = b"\xff\xd8\xff\xe0\x00\x10JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00"
    data, st = cuda.encode_model(image, arrays, prefix, list(range(1, c + 1)), [min(k, 1) for k in range(c)], o)
    assert st == 0
    if c == 1 and si:                                 # Pillow's luma sampling in a grey file's SOF
        i = 2
        while data[i + 1] not in (0xC0, 0xC1):
            i += 2 + int.from_bytes(data[i + 2:i + 4], "big")
        data = data[:i + 11] + bytes([0x21 if si == 1 else 0x22]) + data[i + 12:]
    return data, arrays, tabs


@pytest.mark.parametrize("i", range(0, len(CASES), 60))
def test_restatement_equals_model(i):
    for a, q, s, o in CASES[i:i + 60:3]:
        assert restated(a, q, s, o)[0] == cuda.compress_model(a, q, s, o), (a.shape, q, s, o)


MUTANT_CASES = [(content(np.random.RandomState(18), 22, 18, 3, "random"), 50, "4:2:0", False),
                (content(np.random.RandomState(5), 24, 30, 3, "normal"), 85, "4:2:2", False),
                (content(np.random.RandomState(6), 17, 33, 3, "random"), 1, "4:4:4", True),
                (content(np.random.RandomState(7), 40, 40, 1, "gradient"), 75, "4:2:0", False)]


@pytest.mark.parametrize("mutant", ["bottom_clamp", "right_repeat", "const_bias", "no_baseline", "truncate"])
def test_each_mutant_differs_from_pillow(mutant):
    for a, q, s, o in MUTANT_CASES:
        assert restated(a, q, s, o)[0] == pillow(a, q, s, o)
    assert any(restated(a, q, s, o, mutant)[0] != pillow(a, q, s, o) for a, q, s, o in MUTANT_CASES), mutant


@pytest.mark.skipif(lp.JPEG_SO is None, reason="no libjpeg inside Pillow")
def test_files_hold_the_coefficients_and_tables(tmp_path):
    for k, (a, q, s, o) in enumerate(CASES[::40]):
        path = tmp_path / f"{k}.jpg"
        path.write_bytes(cuda.compress_model(a, q, s, o))
        back = lp.read_coefficients(str(path))
        _, arrays, tabs = restated(a, q, s, o)
        assert len(back.comps) == len(arrays)
        for c, (comp, arr) in enumerate(zip(back.comps, arrays)):
            assert np.array_equal(comp.coef, arr), (a.shape, q, s, c)
            assert np.array_equal(comp.quant.astype(np.int64), tabs[min(c, 1)]), (q, c)


# ---- argument checks ----
def test_python_keywords():
    a = np.zeros((8, 8, 3), np.uint8)
    for q in (0, 101, 50.0, True, "75"):
        with pytest.raises(ValueError, match="quality"):
            cuda.compress_model(a, q)
    for s in (3, -1, "4:1:1", True, None):
        with pytest.raises(ValueError, match="subsampling"):
            cuda.compress_model(a, 75, s)
    for bad in (np.zeros((8, 8, 2), np.uint8), np.zeros((8, 8, 4), np.uint8), np.zeros((8, 8, 3), np.int16)):
        with pytest.raises(ValueError):
            cuda.compress_model(bad)


def test_c_argument_checks_without_context():
    lib = cuda.load()
    a = np.zeros((16, 16, 3), np.uint8)
    out = np.zeros(1 << 16, np.uint8)
    n, st, size = C.c_uint64(0), C.c_int32(0), C.c_size_t(0)

    def model(pin, jp, cap=out.size):
        return lib.jpegqs_cuda_compress_model(C.byref(pin), C.byref(jp), out.ctypes.data, cap, C.byref(n), C.byref(st))
    good_pin = cuda._PixelsIn(a.ctypes.data, 16, 16, 3, 48)
    good = cuda._JpegParams(75, 2, 0)
    assert model(good_pin, good) == 0 and st.value == 0
    bad_params = [cuda._JpegParams(0, 2, 0), cuda._JpegParams(101, 2, 0), cuda._JpegParams(75, 3, 0),
                  cuda._JpegParams(75, -1, 0), cuda._JpegParams(75, 2, 2)]
    bad_pins = [cuda._PixelsIn(a.ctypes.data, 16, 16, 2, 48), cuda._PixelsIn(a.ctypes.data, 16, 16, 4, 64),
                cuda._PixelsIn(a.ctypes.data, 0, 16, 3, 48), cuda._PixelsIn(a.ctypes.data, 65536, 16, 3, 3 * 65536),
                cuda._PixelsIn(a.ctypes.data, 16, 0, 3, 48), cuda._PixelsIn(a.ctypes.data, 16, 16, 3, 47),
                cuda._PixelsIn(None, 16, 16, 3, 48)]
    for jp in bad_params:
        assert model(good_pin, jp) == -2
        assert lib.jpegqs_cuda_compress_bound(C.byref(good_pin), C.byref(jp), C.byref(size)) == -2
        assert lib.jpegqs_cuda_compress_workspace_bytes(1, C.byref(good_pin), C.byref(jp), C.byref(size)) == -2
    for pin in bad_pins:
        assert model(pin, good) == -2, (pin.width, pin.height, pin.channels)
        if pin.pixels_dev:
            assert lib.jpegqs_cuda_compress_bound(C.byref(pin), C.byref(good), C.byref(size)) == -2
            assert lib.jpegqs_cuda_compress_workspace_bytes(1, C.byref(pin), C.byref(good), C.byref(size)) == -2
    assert model(good_pin, good, 19) == -2                     # smaller than the 20-byte prefix
    assert "cap" in lib.jpegqs_cuda_last_error(None).decode()
    assert model(good_pin, good, 200) == 0 and st.value == cuda.ENCODE_OVERFLOW and n.value > 200


def test_bound_and_workspace_formulas():
    lib = cuda.load()
    size = C.c_size_t(0)

    def a256(x):
        return (x + 255) // 256 * 256
    for w, h, ch, s in ((1, 1, 1, 0), (1920, 1080, 3, 2), (33, 17, 3, 1), (100, 7, 3, 0), (64, 64, 1, 2)):
        pin, jp = cuda._PixelsIn(None, w, h, ch, w * ch), cuda._JpegParams(75, s, 0)
        lh, lv = (1, 1) if ch == 1 or s == 0 else (2, 1) if s == 1 else (2, 2)
        if ch == 1:
            U = -(-w // 8) * -(-h // 8)
        else:
            U = -(-w // (8 * lh)) * -(-h // (8 * lv)) * (lh * lv + 2)
        assert lib.jpegqs_cuda_compress_bound(C.byref(pin), C.byref(jp), C.byref(size)) == 0
        assert size.value == 20 + 1680 + 2 * -(-U * 1665 // 8)
        coef = 0
        for k in range(ch):
            hs, vs = (lh, lv) if k == 0 else (1, 1)
            coef += a256(128 * -(-(-(-w * hs // lh)) // 8) * -(-(-(-h * vs // lv)) // 8))
        T, Wd = -(-U // 256), -(-U * 1665 // 32) + 2
        enc = 32768 + a256(2 * U) + a256(8 * T) + a256(4 * Wd) + a256(4 * -(-4 * Wd // 4096))
        assert lib.jpegqs_cuda_compress_workspace_bytes(1, C.byref(pin), C.byref(jp), C.byref(size)) == 0
        assert size.value == 256 + coef + enc, (w, h, ch, s)
