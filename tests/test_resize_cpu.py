"""The crop-and-resize stage of jpegqs_cuda_pixels_batch_resized, without a GPU: resize_model (the
device's weight tables and per-pixel arithmetic on one CPU thread) is Pillow's
Image.fromarray(P).crop(box).resize(size, filter) byte for byte, over a seeded sweep of L and RGB
pictures, both layouts, all five convolution filters, up- and downscales, one-axis and same-size
resizes, crops touching each edge, extreme ratios and saturated content whose negative lobes clamp.
A numpy restatement of Pillow's Resample.c equals the model, and four plausible mistakes in it each
give a picture Pillow does not.  Also the argument checks of the Python keywords, of resize_model and
of the C calls without a context."""
import ctypes as C
import math

import numpy as np
import pytest

PIL = pytest.importorskip("PIL.Image")
Image = PIL

import decode_files as df
from jpegqs_b200 import cuda

FILTERS = {"box": Image.Resampling.BOX, "bilinear": Image.Resampling.BILINEAR, "hamming": Image.Resampling.HAMMING,
           "bicubic": Image.Resampling.BICUBIC, "lanczos": Image.Resampling.LANCZOS}


def _pillow(a, size, crop, filt):
    im = Image.fromarray(a if a.ndim == 2 or a.shape[2] == 3 else a[..., 0])
    if crop is not None:
        im = im.crop(crop)
    return np.asarray(im.resize(size, FILTERS[filt]))


def _content(rng, h, w, c, kind):
    shape = (h, w) if c == 1 else (h, w, c)
    if kind == "random":
        return rng.randint(0, 256, shape).astype(np.uint8)
    if kind == "saturated":
        return (rng.randint(0, 2, shape) * 255).astype(np.uint8)
    if kind == "columns":                     # alternating 0 / 255 columns: the largest lobes
        a = np.zeros(shape, np.uint8)
        a[:, ::2] = 255
        return a
    if kind == "checker":
        yy, xx = np.indices((h, w))
        a = (((yy + xx) & 1) * 255).astype(np.uint8)
        return a if c == 1 else np.repeat(a[..., None], c, 2)
    # a sinusoid driven past both rails
    yy, xx = np.indices((h, w))
    f = rng.uniform(0.2, 2.5)
    a = np.clip(128 + 400 * np.sin(f * xx + 0.7 * f * yy), 0, 255).astype(np.uint8)
    return a if c == 1 else np.stack([a, 255 - a, a[::-1]], 2)


def _cases():
    """(picture, size, crop, filter): a seeded sweep, then the shapes a loader or thumbnailer asks for"""
    rng = np.random.RandomState(2026)
    kinds = ("random", "saturated", "columns", "checker", "sine")
    out = []
    for i in range(900):
        big = i % 10 == 0
        h, w = rng.randint(1, 300 if big else 90, 2)
        a = _content(rng, h, w, (1, 3)[i % 2], kinds[i % 5])
        crop = None
        mode = rng.randint(4)
        if mode == 1:                         # a crop touching one edge, or two
            l = 0 if rng.rand() < 0.5 else rng.randint(w)
            t = 0 if rng.rand() < 0.5 else rng.randint(h)
            r = w if rng.rand() < 0.5 else rng.randint(l + 1, w + 1)
            b = h if rng.rand() < 0.5 else rng.randint(t + 1, h + 1)
            crop = (l, t, r, b)
        elif mode == 2:
            l, t = rng.randint(w), rng.randint(h)
            crop = (l, t, rng.randint(l + 1, w + 1), rng.randint(t + 1, h + 1))
        cw, ch = (crop[2] - crop[0], crop[3] - crop[1]) if crop else (w, h)
        which = rng.randint(5)
        if which == 0:
            size = (cw, ch)                                        # same size
        elif which == 1:
            size = (cw, int(rng.randint(1, 130)))                  # one axis only
        elif which == 2:
            size = (int(rng.randint(1, 130)), ch)
        else:
            size = tuple(int(x) for x in rng.randint(1, 130, 2))   # up, down or both
        out.append((a, size, crop, list(FILTERS)[i % 5]))
    for filt in FILTERS:
        out.append((_content(rng, 1, 1, 3, "random"), (1, 1), None, filt))
        out.append((_content(rng, 1, 1, 1, "random"), (17, 5), None, filt))
        out.append((_content(rng, 37, 53, 3, "sine"), (224, 224), (0, 0, 53, 37), filt))
    return out


CASES = _cases()


def test_model_is_pillow_over_the_sweep():
    bad = []
    for k, (a, size, crop, filt) in enumerate(CASES):
        want = _pillow(a, size, crop, filt)
        got = cuda.resize_model(a, size, crop, filt)
        if not np.array_equal(got, want):
            bad.append((k, a.shape, size, crop, filt))
        if a.ndim == 3:
            chw = cuda.resize_model(a, size, crop, filt, layout="chw")
            if not np.array_equal(chw.transpose(1, 2, 0), want):
                bad.append((k, "chw", a.shape, size, crop, filt))
    assert not bad, bad[:10]


@pytest.mark.parametrize("shape,size,filt", [
    ((2, 3000), (5, 2), "lanczos"),               # horizontal kernel size 3 601
    ((1500, 2), (2, 3), "lanczos"),
    ((5, 7), (900, 400), "bicubic"),
    ((5, 7, 3), (900, 400), "lanczos"),
    ((1081, 1921, 3), (224, 224), "lanczos"),
    ((1081, 1921, 3), (224, 224), "bicubic"),
    ((1, 3000), (1, 1), "hamming"),
])
def test_extreme_ratios(shape, size, filt):
    rng = np.random.RandomState(7)
    a = rng.randint(0, 256, shape).astype(np.uint8)
    if shape[0] > 1000:
        a[:] = 0
        a[:, ::2] = 255
    assert np.array_equal(cuda.resize_model(a, size, None, filt), _pillow(a, size, None, filt))


def test_grey_keeps_one_channel():
    a = _content(np.random.RandomState(3), 40, 30, 1, "sine")
    assert cuda.resize_model(a, (12, 9)).shape == (9, 12)
    for layout in ("hwc", "chw"):
        three = cuda.resize_model(a[..., None], (12, 9), layout=layout)
        assert three.shape == ((9, 12, 1) if layout == "hwc" else (1, 9, 12))
        assert np.array_equal(three.reshape(9, 12), _pillow(a, (12, 9), None, "bicubic"))


# ---- a numpy restatement of Resample.c, and mistakes it must not make -----------------------------

_F054, _F046 = float(np.float32(0.54)), float(np.float32(0.46))


def _sinc(x):
    if x == 0.0:
        return 1.0
    x = x * math.pi
    return math.sin(x) / x


def _hamming(x):
    x = abs(x)
    if x == 0.0:
        return 1.0
    if x >= 1.0:
        return 0.0
    x = x * math.pi
    return math.sin(x) / x * (_F054 + _F046 * math.cos(x))


def _bicubic(x):
    a = -0.5
    x = abs(x)
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


KERNELS = {"box": (lambda x: 1.0 if -0.5 < x <= 0.5 else 0.0, 0.5),
           "bilinear": (lambda x: max(0.0, 1.0 - abs(x)), 1.0),
           "hamming": (_hamming, 1.0),
           "bicubic": (_bicubic, 2.0),
           "lanczos": (lambda x: _sinc(x) * _sinc(x / 3) if -3.0 <= x < 3.0 else 0.0, 3.0)}


def _axis(n_in, n_out, filt, mutant):
    fn, sup = KERNELS[filt]
    scale = n_in / n_out
    fs = scale if mutant == "no_filterscale_clamp" else max(scale, 1.0)
    support = sup * fs
    bounds, weights = [], []
    for xx in range(n_out):
        center = (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        count = min(int(center + support + 0.5), n_in) - xmin
        w = [fn((x + xmin - center + 0.5) * (1.0 / fs)) for x in range(count)]
        ww = 0.0
        for v in w:
            ww += v
        w = [v / ww if ww != 0.0 else v for v in w]
        if mutant == "truncated_weights":
            k = [int(v * (1 << 22)) for v in w]
        else:
            k = [int(-0.5 + v * (1 << 22)) if v < 0 else int(0.5 + v * (1 << 22)) for v in w]
        bounds.append((xmin, count))
        weights.append(np.array(k, np.int64))
    return bounds, weights


def _pass(a, axis, bounds, weights, clip):
    """one pass along axis (1: horizontal, 0: vertical) of an int64 [H, W, C] picture"""
    outs = []
    for (lo, count), k in zip(bounds, weights):
        win = a[:, lo:lo + count] if axis == 1 else a[lo:lo + count]
        ss = (1 << 21) + np.tensordot(win, k, axes=([axis], [0]))
        assert np.abs(ss).max(initial=0) < 2 ** 31          # Pillow's int accumulator fits an int32
        v = ss >> 22
        outs.append(np.clip(v, 0, 255) if clip else v)
    return np.stack(outs, axis)


def _restated(a, size, crop, filt, mutant=None):
    p = a if a.ndim == 3 else a[..., None]
    if crop is not None:
        p = p[crop[1]:crop[3], crop[0]:crop[2]]
    p = p.astype(np.int64)
    hb, hk = _axis(p.shape[1], size[0], filt, mutant)
    vb, vk = _axis(p.shape[0], size[1], filt, mutant)
    clip_mid = mutant != "unclipped_intermediate"
    if mutant == "vertical_first":
        out = _pass(_pass(p, 0, vb, vk, True), 1, hb, hk, True)
    else:
        out = np.clip(_pass(_pass(p, 1, hb, hk, clip_mid), 0, vb, vk, True), 0, 255)
    out = out.astype(np.uint8)
    return out if a.ndim == 3 else out[..., 0]


MUTANTS = ("unclipped_intermediate", "no_filterscale_clamp", "truncated_weights", "vertical_first")


def test_restatement_is_the_model_and_mutants_are_caught():
    caught = dict.fromkeys(MUTANTS, False)
    for a, size, crop, filt in CASES[::4]:
        want = cuda.resize_model(a, size, crop, filt)
        assert np.array_equal(_restated(a, size, crop, filt), want), (a.shape, size, crop, filt)
        for m in MUTANTS:
            if not caught[m] and not np.array_equal(_restated(a, size, crop, filt, m), _pillow(a, size, crop, filt)):
                caught[m] = True
    assert all(caught.values()), caught


# ---- argument checks ------------------------------------------------------------------------------

def test_resize_model_checks_its_arguments():
    a = np.zeros((10, 20, 3), np.uint8)
    for bad in (a.astype(np.int16), np.zeros((10, 20, 2), np.uint8), np.zeros((0, 5), np.uint8), np.zeros(5, np.uint8)):
        with pytest.raises(ValueError, match="pixels"):
            cuda.resize_model(bad, (4, 4))
    for size in ((0, 4), (4, 65536), (4,), "44", (4.0, 4), None):
        with pytest.raises(ValueError, match="size"):
            cuda.resize_model(a, size)
    for crop in ((0, 0, 21, 10), (0, 0, 20, 11), (5, 0, 5, 10), (0, 4, 20, 2), (-1, 0, 5, 5), (0, 0, 5)):
        with pytest.raises(ValueError, match="crop"):
            cuda.resize_model(a, (4, 4), crop)
    for filt in ("nearest", 0, Image.Resampling.NEAREST, 6, "cubic", None, True):
        with pytest.raises(ValueError, match="filter"):
            cuda.resize_model(a, (4, 4), filter=filt)
    with pytest.raises(ValueError, match="layout"):
        cuda.resize_model(a, (4, 4), layout="hcw")
    # Pillow's Image.Resampling values are taken as they are
    assert np.array_equal(cuda.resize_model(a, (4, 4), filter=Image.Resampling.LANCZOS), cuda.resize_model(a, (4, 4), filter="lanczos"))


def test_c_model_checks_its_arguments():
    lib = cuda.load()
    src = (C.c_uint8 * 600)()
    out = (C.c_uint8 * 48)(*([7] * 48))
    f = lib.jpegqs_cuda_resize_model

    def box(*v):
        return C.byref(cuda._ResizeBox(*v))
    assert f(src, 20, 10, 3, 0, 3, box(0, 0, 0, 0, 4, 4), out) == 0
    for args, why in [((None, 20, 10, 3, 0, 3, box(0, 0, 0, 0, 4, 4), out), "NULL"),
                      ((src, 20, 10, 3, 0, 3, None, out), "NULL"),
                      ((src, 0, 10, 3, 0, 3, box(0, 0, 0, 0, 4, 4), out), "size"),
                      ((src, 20, 10, 2, 0, 3, box(0, 0, 0, 0, 4, 4), out), "channels"),
                      ((src, 20, 10, 3, 2, 3, box(0, 0, 0, 0, 4, 4), out), "layout"),
                      ((src, 20, 10, 3, 0, 0, box(0, 0, 0, 0, 4, 4), out), "filter"),
                      ((src, 20, 10, 3, 0, 6, box(0, 0, 0, 0, 4, 4), out), "filter"),
                      ((src, 20, 10, 3, 0, 3, box(0, 0, 21, 10, 4, 4), out), "outside"),
                      ((src, 20, 10, 3, 0, 3, box(0, 5, 20, 5, 4, 4), out), "empty"),
                      ((src, 20, 10, 3, 0, 3, box(0, 0, 0, 0, 0, 4), out), "1..65535"),
                      ((src, 20, 10, 3, 0, 3, box(0, 0, 0, 0, 4, 65536), out), "1..65535")]:
        for k in range(48):
            out[k] = 7
        assert f(*args) == -2, why
        assert why in lib.jpegqs_cuda_last_error(None).decode(), why
        assert bytes(out) == bytes([7] * 48), why         # nothing written


def _unbound():
    """A QsContext without a device: the wrapper's checks run before it touches one."""
    c = object.__new__(cuda.QsContext)
    c.lib = cuda.load()                   # the picture sizes come from the host-only route walk
    return c


def test_python_keywords_check_their_arguments():
    good = df.pillow_jpeg(64, 48, quality=75)          # a 64 x 48 picture, 32 x 24 at d = 2
    ctx = _unbound()
    dp = cuda.QsContext.decode_pixels
    assert dp(ctx, [], 0, 3, size=(4, 4)) == []
    for size in ((0, 4), (4, 70000), (4,), "ab", (4.5, 4), [(4, 4)], [(4, 4), (4, 0)]):
        with pytest.raises(ValueError, match="size"):
            dp(ctx, [good, good], 0, 3, size=size)
    with pytest.raises(ValueError, match="file 1: size"):
        dp(ctx, [good, good], 0, 3, size=[(4, 4), (0, 4)])
    for crop in ((0, 0, 4, 4), [(0, 0, 4, 4)], [None, (4, 4, 2, 2)], [None, (0, 0, 4)], [None, (-1, 0, 4, 4)]):
        with pytest.raises(ValueError, match="crop"):
            dp(ctx, [good, good], 0, 3, crop=crop)
    with pytest.raises(ValueError, match="file 1: crop"):
        dp(ctx, [good, good], 0, 3, crop=[None, (4, 4, 2, 2)])
    for filt in ("nearest", 0, Image.Resampling.NEAREST, 9, "cubic"):
        with pytest.raises(ValueError, match="filter"):
            dp(ctx, [good], 0, 3, size=(4, 4), filter=filt)
    # against the file's picture: 64 x 48, or 32 x 24 at scale_denom 2
    with pytest.raises(ValueError, match="file 1: crop .* outside the 64 x 48 picture"):
        dp(ctx, [good, good], 0, 3, size=(4, 4), crop=[(0, 0, 64, 48), (0, 0, 65, 48)])
    with pytest.raises(ValueError, match="file 0: crop .* outside the 32 x 24 picture"):
        dp(ctx, [good], 0, 3, crop=[(0, 0, 33, 10)], scale_denom=2)


def test_c_call_without_a_context():
    lib = cuda.load()
    data = df.pillow_jpeg(64, 48, quality=75)
    ptrs = (C.c_char_p * 1)(data)
    lens = (C.c_size_t * 1)(len(data))
    buf = (C.c_uint8 * (8 * 8 * 3))()
    outs = (C.c_void_p * 1)(C.addressof(buf))
    rc = (C.c_int * 1)(7)
    res = (cuda._PixelsResult * 1)()
    res[0].channels = 9
    boxes = (cuda._ResizeBox * 1)(cuda._ResizeBox(0, 0, 0, 0, 8, 8))
    f = lib.jpegqs_cuda_pixels_batch_resized
    assert f(None, 1, ptrs, lens, 0, 3, 0, 1, 3, boxes, 0, outs, 0, rc, res) == -2
    assert f(None, 1, ptrs, lens, 0, 3, 0, 1, 3, None, 0, outs, 0, rc, res) == -2
    assert f(None, 0, None, None, 0, 3, 0, 1, 3, None, 0, None, 0, None, None) == -2
    assert rc[0] == 7 and res[0].channels == 9 and not res[0].reason      # nothing touched
    assert bytes(buf) == bytes(len(buf))
