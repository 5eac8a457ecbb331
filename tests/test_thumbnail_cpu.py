"""Thumbnails and reducing_gap without a GPU: reduce_model (the device reduce on one CPU thread) is
Pillow's Image.reduce, resize_model_box is Image.resize(box=float box, reducing_gap=), and
thumbnail_model - thumbnail_geometry's size and draft scale, then the batch's planning of the reduce
and the resize - is Image.open(f).thumbnail(...) byte for byte on JPEG files, after exif_transpose or
convert as well.  A numpy restatement of the chain equals the model, and four plausible mistakes in it
each give a picture Pillow does not.  Also the argument checks in C and Python."""
import ctypes as C
import io
import math

import numpy as np
import pytest

PIL = pytest.importorskip("PIL.Image")
Image = PIL
from PIL import ImageOps

from jpegqs_b200 import cuda

FILTERS = {"box": Image.Resampling.BOX, "bilinear": Image.Resampling.BILINEAR, "hamming": Image.Resampling.HAMMING,
           "bicubic": Image.Resampling.BICUBIC, "lanczos": Image.Resampling.LANCZOS}


def _content(rng, h, w, c, kind):
    shape = (h, w) if c == 1 else (h, w, c)
    if kind == "random":
        return rng.randint(0, 256, shape).astype(np.uint8)
    if kind == "saturated":
        return (rng.randint(0, 2, shape) * 255).astype(np.uint8)
    return np.full(shape, 255, np.uint8)                  # every sum at its largest


def _img(a):
    return Image.fromarray(a)


# ---- reduce --------------------------------------------------------------------------------------

def _reduce_cases():
    rng = np.random.RandomState(2026)
    out = []
    for fx in range(1, 17):
        for fy in range(1, 17):
            if (fx * 7 + fy * 3) % 4 and not (fx in (1, 2, 3, 8, 16) and fy in (1, 2, 3, 8, 16)):
                continue
            h, w = int(rng.randint(1, 4 * fy + 9)), int(rng.randint(1, 4 * fx + 9))
            kind = ("random", "saturated", "max")[(fx + fy) % 3]
            a = _content(rng, h, w, (1, 3)[(fx * fy) % 2], kind)
            box = None
            if (fx + 2 * fy) % 3 == 1:                    # a box touching one edge or none
                l, t = int(rng.randint(w)), int(rng.randint(h))
                box = (l, t, int(rng.randint(l + 1, w + 1)), int(rng.randint(t + 1, h + 1)))
            elif (fx + 2 * fy) % 3 == 2:
                box = (0, int(rng.randint(h)), w, h)
                box = (box[0], box[1], box[2], max(box[3], box[1] + 1))
            out.append((a, (fx, fy), box))
    for c in (1, 3):                                      # 1 x 1 and 1-pixel-wide pictures
        for shape in ((1, 1), (1, 37), (29, 1)):
            a = _content(rng, shape[0], shape[1], c, "random")
            for f in ((1, 1), (2, 2), (5, 1), (1, 7), (16, 16)):
                out.append((a, f, None))
    return out


REDUCE_CASES = _reduce_cases()


def test_reduce_model_is_pillow():
    bad = []
    for k, (a, f, box) in enumerate(REDUCE_CASES):
        want = np.asarray(_img(a).reduce(f, box))
        got = cuda.reduce_model(a, f, box)
        if not np.array_equal(got, want):
            bad.append((k, a.shape, f, box))
    assert not bad, bad[:10]


def _np_reduce(a, f, box=None, exact=False):
    """Reduce.c restated: ((sum + n / 2) * m) >> 24, m = (uint32)(float(2^32) / float(256 n))"""
    a = a.astype(np.int64)
    if a.ndim == 2:
        a = a[..., None]
    l, t, r, b = box if box is not None else (0, 0, a.shape[1], a.shape[0])
    fx, fy = f
    ow, oh = -(-(r - l) // fx), -(-(b - t) // fy)
    out = np.zeros((oh, ow, a.shape[2]), np.int64)
    for y in range(oh):
        for x in range(ow):
            cell = a[t + y * fy:min(t + y * fy + fy, b), l + x * fx:min(l + x * fx + fx, r)]
            n = cell.shape[0] * cell.shape[1]
            s = cell.sum(axis=(0, 1))
            if exact:
                out[y, x] = (s + n // 2) // n
            else:
                m = int(np.float32(2.0 ** 32) / np.float32(256 * n))
                out[y, x] = (((s + n // 2) * m) & 0xFFFFFFFF) >> 24
    return out.astype(np.uint8)


def test_numpy_reduce_is_the_model_and_the_exact_mean_is_not_pillow():
    exact_differs = 0
    for a, f, box in REDUCE_CASES[::3]:
        want = np.asarray(_img(a).reduce(f, box))
        got = _np_reduce(a, f, box).reshape(want.shape)
        assert np.array_equal(got, cuda.reduce_model(a, f, box))
        exact_differs += not np.array_equal(_np_reduce(a, f, box, exact=True).reshape(want.shape), want)
    assert exact_differs
    # even for power-of-two squares the exact mean is not Pillow's arithmetic on every sample
    a = _content(np.random.RandomState(5), 64, 64, 3, "random")
    for f in ((3, 3), (5, 7), (6, 6)):
        assert not np.array_equal(_np_reduce(a, f, exact=True), np.asarray(_img(a).reduce(f)))


# ---- resize from a float box ---------------------------------------------------------------------

def _box_cases(n=150):
    rng = np.random.RandomState(11)
    out = []
    for i in range(n):
        h, w = (int(v) for v in rng.randint(2, 120, 2))
        a = _content(rng, h, w, (1, 3)[i % 2], ("random", "saturated")[i % 2 // 1 % 2])
        x0, x1 = sorted(rng.uniform(0, w, 2))
        y0, y1 = sorted(rng.uniform(0, h, 2))
        if x1 - x0 < 0.25:
            x0, x1 = 0.0, float(w)
        if y1 - y0 < 0.25:
            y0, y1 = 0.0, float(h)
        size = (int(rng.randint(1, 90)), int(rng.randint(1, 90)))
        out.append((a, size, (x0, y0, x1, y1), list(FILTERS)[i % 5]))
    return out


BOX_CASES = _box_cases()


def test_resize_model_box_is_pillow():
    bad = []
    for k, (a, size, box, filt) in enumerate(BOX_CASES):
        want = np.asarray(_img(a).resize(size, FILTERS[filt], box=box))
        if not np.array_equal(cuda.resize_model_box(a, size, box, filt), want):
            bad.append((k, a.shape, size, box, filt))
    assert not bad, bad[:10]


def test_resize_model_box_reducing_gap_is_pillow():
    rng = np.random.RandomState(12)
    bad = []
    for k in range(60):
        h, w = (int(v) for v in rng.randint(20, 400, 2))
        a = _content(rng, h, w, (1, 3)[k % 2], "random")
        size = (int(rng.randint(1, 60)), int(rng.randint(1, 60)))
        gap = (1.0, 1.5, 2.0, 3.0)[k % 4]
        filt = list(FILTERS)[k % 5]
        box = None if k % 3 else (float(rng.uniform(0, w / 4)), float(rng.uniform(0, h / 4)), float(w), float(h))
        want = np.asarray(_img(a).resize(size, FILTERS[filt], box=box, reducing_gap=gap))
        if not np.array_equal(cuda.resize_model_box(a, size, box, filt, gap), want):
            bad.append((k, a.shape, size, box, filt, gap))
    assert not bad, bad[:10]


def test_integer_box_gives_the_crop_planner_tables():
    """the float-box planner and the integer-crop planner build the same tables for the whole picture:
    random content tells any weight or bound apart"""
    rng = np.random.RandomState(13)
    for k in range(200):
        h, w = (int(v) for v in rng.randint(1, 150, 2))
        a = _content(rng, h, w, (1, 3)[k % 2], "random")
        size = (int(rng.randint(1, 200)), int(rng.randint(1, 200)))
        filt = list(FILTERS)[k % 5]
        want = cuda.resize_model(a, size, None, filt)
        assert np.array_equal(cuda.resize_model_box(a, size, (0, 0, w, h), filt), want), (k, a.shape, size, filt)
        assert np.array_equal(cuda.resize_model_box(a, size, None, filt), want)


# ---- a numpy restatement of the chain, and its mutants --------------------------------------------

def _sinc(x):
    return 1.0 if x == 0.0 else math.sin(x * math.pi) / (x * math.pi)


def _hamming(x):
    x = abs(x)
    if x == 0.0:
        return 1.0
    if x >= 1.0:
        return 0.0
    x = x * math.pi
    return math.sin(x) / x * (float(np.float32(0.54)) + float(np.float32(0.46)) * math.cos(x))


def _bicubic(x):
    x = abs(x)
    if x < 1.0:
        return (1.5 * x - 2.5) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * -0.5
    return 0.0


KERNELS = {"box": (lambda x: 1.0 if -0.5 < x <= 0.5 else 0.0, 0.5), "bilinear": (lambda x: max(0.0, 1.0 - abs(x)), 1.0),
           "hamming": (_hamming, 1.0), "bicubic": (_bicubic, 2.0),
           "lanczos": (lambda x: _sinc(x) * _sinc(x / 3) if -3.0 <= x < 3.0 else 0.0, 3.0)}


def _axis(n_in, in0, in1, n_out, filt, double_box):
    fn, sup = KERNELS[filt]
    if not double_box:
        in0, in1 = float(np.float32(in0)), float(np.float32(in1))
        scale = float(np.float32(in1) - np.float32(in0)) / n_out
    else:
        scale = (in1 - in0) / n_out
    fs = max(scale, 1.0)
    support = sup * fs
    rows = []
    for xx in range(n_out):
        center = in0 + (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        count = min(int(center + support + 0.5), n_in) - xmin
        w = [fn((x + xmin - center + 0.5) * (1.0 / fs)) for x in range(count)]
        ww = sum(w)
        w = [v / ww if ww != 0.0 else v for v in w]
        rows.append((xmin, [int(-0.5 + v * (1 << 22)) if v < 0 else int(0.5 + v * (1 << 22)) for v in w]))
    return rows


def _np_resize(a, size, box, filt, double_box=False):
    a = a.astype(np.int64)
    if a.ndim == 2:
        a = a[..., None]
    h, w = a.shape[:2]
    hx = _axis(w, box[0], box[2], size[0], filt, double_box)
    vy = _axis(h, box[1], box[3], size[1], filt, double_box)
    first, last = vy[0][0], vy[-1][0] + len(vy[-1][1])
    mid = np.zeros((last - first, size[0], a.shape[2]), np.int64)
    for xx, (x0, k) in enumerate(hx):
        s = (1 << 21) + (a[first:last, x0:x0 + len(k)] * np.array(k, np.int64)[None, :, None]).sum(1)
        mid[:, xx] = np.clip(s >> 22, 0, 255)
    out = np.zeros((size[1], size[0], a.shape[2]), np.int64)
    for yy, (y0, k) in enumerate(vy):
        s = (1 << 21) + (mid[y0 - first:y0 - first + len(k)] * np.array(k, np.int64)[:, None, None]).sum(0)
        out[yy] = np.clip(s >> 22, 0, 255)
    return out.astype(np.uint8)


def _np_resize_gap(a, size, box, filt, gap, mutant=None):
    """Image.resize(size, filt, box, reducing_gap=gap) restated"""
    h, w = a.shape[:2]
    box = box if box is not None else (0, 0, w, h)
    fx = int((box[2] - box[0]) / size[0] / gap) or 1
    fy = int((box[3] - box[1]) / size[1] / gap) or 1
    if fx > 1 or fy > 1:
        sup = KERNELS[filt][1] - (0.0 if mutant == "safe_box_no_half" else 0.5)
        sx, sy = sup * (box[2] - box[0]) / size[0], sup * (box[3] - box[1]) / size[1]
        rb = (max(0, int(box[0] - sx)), max(0, int(box[1] - sy)), min(w, math.ceil(box[2] + sx)), min(h, math.ceil(box[3] + sy)))
        if mutant == "plain_box":
            rb = (int(box[0]), int(box[1]), math.ceil(box[2]), math.ceil(box[3]))
        a = _np_reduce(a, (fx, fy), rb)
        box = ((box[0] - rb[0]) / fx, (box[1] - rb[1]) / fy, (box[2] - rb[0]) / fx, (box[3] - rb[1]) / fy)
    return _np_resize(a, size, box, filt, double_box=mutant == "double_box")


def _chain_cases():
    rng = np.random.RandomState(17)
    out = []
    for k in range(24):
        h, w = (int(v) for v in rng.randint(40, 300, 2))
        a = _content(rng, h, w, (1, 3)[k % 2], "random")
        size = (int(rng.randint(3, 40)), int(rng.randint(3, 40)))
        box = (float(rng.uniform(0, 3)), float(rng.uniform(0, 3)), w - float(rng.uniform(0, 3)), h - float(rng.uniform(0, 3)))
        out.append((a, size, box, list(FILTERS)[k % 5], (1.0, 1.5, 2.0)[k % 3]))
    return out


CHAIN_CASES = _chain_cases()


def test_numpy_chain_is_the_model():
    for a, size, box, filt, gap in CHAIN_CASES[:10]:
        want = np.asarray(_img(a).resize(size, FILTERS[filt], box=box, reducing_gap=gap))
        got = _np_resize_gap(a, size, box, filt, gap).reshape(want.shape)
        assert np.array_equal(got, want)
        assert np.array_equal(cuda.resize_model_box(a, size, box, filt, gap), want)


@pytest.mark.parametrize("mutant", ["exact_mean", "double_box", "safe_box_no_half", "plain_box"])
def test_chain_mutants_are_not_pillow(mutant):
    differs = 0
    for a, size, box, filt, gap in CHAIN_CASES:
        want = np.asarray(_img(a).resize(size, FILTERS[filt], box=box, reducing_gap=gap))
        if mutant == "exact_mean":
            global _np_reduce
            keep = _np_reduce
            _np_reduce = lambda x, f, b=None, exact=False: keep(x, f, b, True)
            try:
                got = _np_resize_gap(a, size, box, filt, gap)
            finally:
                _np_reduce = keep
        else:
            got = _np_resize_gap(a, size, box, filt, gap, mutant)
        differs += not np.array_equal(got.reshape(want.shape), want)
    if mutant == "double_box":                 # the plain float-box resizes tell the box's precision apart
        for a, size, box, filt in BOX_CASES:
            want = np.asarray(_img(a).resize(size, FILTERS[filt], box=box))
            assert np.array_equal(_np_resize(a, size, box, filt).reshape(want.shape), want)
            differs += not np.array_equal(_np_resize(a, size, box, filt, double_box=True).reshape(want.shape), want)
    assert differs, mutant


# ---- thumbnail geometry and the chain on JPEG files -----------------------------------------------

def test_thumbnail_geometry_is_pillow():
    rng = np.random.RandomState(19)
    sizes = [(3000, 5), (5, 3000), (1, 1), (1920, 1080), (1080, 1920), (640, 480), (256, 256)]
    sizes += [tuple(int(v) for v in rng.randint(1, 3000, 2)) for _ in range(150)]
    for k, (W, H) in enumerate(sizes):
        for bound in ((256, 256), (int(rng.randint(1, 400)), int(rng.randint(1, 400))), (W, H), (W + 1, H - 1 or 1)):
            im = Image.new("L", (W, H))
            im.thumbnail(bound)
            s, got = cuda.thumbnail_geometry(W, H, bound)
            assert got == im.size, (W, H, bound)
            for gap in (None, 1.0, 1.5, 2.0, 3.0):
                s, _ = cuda.thumbnail_geometry(W, H, bound, gap)
                want = 1
                if gap is not None and not (bound[0] >= W and bound[1] >= H):
                    sc = min(W // int(bound[0] * gap), H // int(bound[1] * gap))
                    want = next(v for v in (8, 4, 2, 1) if sc >= v or v == 1)
                assert s == want, (W, H, bound, gap)
                assert cuda.thumbnail_geometry(W, H, bound, gap, loaded=True)[0] == 1


def _jpeg(a, subsampling, quality=90, exif=None):
    f = io.BytesIO()
    kw = {"quality": quality}
    if a.ndim == 3:
        kw["subsampling"] = subsampling
    if exif is not None:
        kw["exif"] = exif
    Image.fromarray(a).save(f, "JPEG", **kw)
    return f.getvalue()


def _photo(rng, h, w, c):
    yy, xx = np.indices((h, w))
    base = 128 + 60 * np.sin(xx / 9.0) * np.cos(yy / 13.0) + rng.normal(0, 20, (h, w))
    a = np.clip(base, 0, 255).astype(np.uint8)
    return a if c == 1 else np.stack([a, np.clip(255 - base, 0, 255).astype(np.uint8), a[::-1]], 2)


def _drafted(data, bound, gap):
    """the picture Pillow's thumbnail starts from: Image.open, and the draft it makes"""
    im = Image.open(io.BytesIO(data))
    if gap is not None and not (bound[0] >= im.width and bound[1] >= im.height):
        im.draft(None, (int(bound[0] * gap), int(bound[1] * gap)))
    return np.asarray(im)


def _thumb_files():
    rng = np.random.RandomState(23)
    out = []
    for (h, w), c, sub in [((480, 640), 3, 2), ((1080, 1920), 3, 2), ((333, 517), 3, 1), ((517, 333), 3, 0),
                           ((301, 299), 1, 0), ((5, 3000), 3, 2), ((3000, 5), 1, 0), ((128, 128), 3, 2),
                           ((2048, 1536), 3, 0)]:
        out.append(_jpeg(_photo(rng, h, w, c), sub))
    return out


THUMB_FILES = _thumb_files()


@pytest.mark.parametrize("gap", [None, 1.0, 1.5, 2.0, 3.0])
def test_thumbnail_model_is_pillow_on_jpeg_files(gap):
    bad = []
    for k, data in enumerate(THUMB_FILES):
        W, H = Image.open(io.BytesIO(data)).size
        bounds = [(256, 256), (100, 40), (40, 900), (W, H), (W * 2, H * 2)]
        s, _ = cuda.thumbnail_geometry(W, H, (64, 64), gap)
        bounds.append((-(-W // s), -(-H // s)))                        # the drafted size exactly
        for j, bound in enumerate(bounds):
            filt = list(FILTERS)[(k + j) % 5]
            im = Image.open(io.BytesIO(data))
            im.thumbnail(bound, FILTERS[filt], reducing_gap=gap)
            want = np.asarray(im)
            try:
                got = cuda.thumbnail_model(_drafted(data, bound, gap), (W, H), bound, filt, gap)
            except ValueError as e:                                    # Pillow's vertical-first resize
                assert "taller than wide" in str(e) and H > 100 * W, (k, bound, e)
                continue
            if got.shape != want.shape or not np.array_equal(got, want):
                bad.append((k, (W, H), bound, filt))
    assert not bad, bad


@pytest.mark.parametrize("seq", ["exif", "transpose", "RGB", "L"])
def test_loaded_sequences_are_pillow(seq):
    """exif_transpose, transpose and convert load the picture: thumbnail then shrinks by reduce alone"""
    rng = np.random.RandomState(29)
    exif = Image.Exif()
    exif[0x0112] = 6
    data = _jpeg(_photo(rng, 700, 1100, 3), 2, exif=exif.tobytes())
    for bound, filt, gap in [((256, 256), "bicubic", 2.0), ((64, 200), "lanczos", 1.0), ((150, 150), "box", 3.0),
                             ((300, 300), "hamming", None)]:
        im = Image.open(io.BytesIO(data))
        im = {"exif": lambda: ImageOps.exif_transpose(im), "transpose": lambda: im.transpose(Image.Transpose.ROTATE_90),
              "RGB": lambda: im.convert("RGB"), "L": lambda: im.convert("L")}[seq]()
        pic = np.asarray(im).copy()
        im.thumbnail(bound, FILTERS[filt], reducing_gap=gap)
        got = cuda.thumbnail_model(pic, (pic.shape[1], pic.shape[0]), bound, filt, gap, loaded=True)
        assert np.array_equal(got, np.asarray(im)), (bound, filt, gap)


# ---- argument errors ------------------------------------------------------------------------------

def test_python_argument_errors():
    a = np.zeros((10, 10, 3), np.uint8)
    with pytest.raises(ValueError):
        cuda.reduce_model(a, 0)
    with pytest.raises(ValueError):
        cuda.reduce_model(a, (2, 2), (0, 0, 11, 10))
    with pytest.raises(ValueError):
        cuda.reduce_model(a, (4096, 4096))                              # a cell of 2^24 samples
    with pytest.raises(ValueError):
        cuda.resize_model_box(a, (5, 5), (0, 0, 10.5, 10))
    with pytest.raises(ValueError):
        cuda.resize_model_box(a, (5, 5), None, "bicubic", 0.5)
    with pytest.raises(ValueError):
        cuda.resize_model_box(a, (5, 5), None, "nearest")
    with pytest.raises(ValueError):
        cuda.resize_model_box(np.zeros((2000, 3), np.uint8), (1, 10))  # Pillow resizes it vertically first
    for bad in ((0, 5), (5, 70000), "256", (2.5, 3)):
        with pytest.raises(ValueError):
            cuda.thumbnail_geometry(100, 100, bad)
    for gap in (0.5, float("nan"), float("inf"), True, "2"):
        with pytest.raises(ValueError):
            cuda.thumbnail_geometry(100, 100, (10, 10), gap)
    ctx = cuda.QsContext.__new__(cuda.QsContext)                       # the checks run before the device
    ctx.lib, ctx.h, ctx.device = cuda.load(), None, 0
    files = [THUMB_FILES[0], THUMB_FILES[1]]
    for kw, words in [(dict(thumbnail=(64, 64), size=(10, 10)), "thumbnail takes no size"),
                      (dict(thumbnail=(64, 64), crop=[None, None]), "thumbnail takes no size"),
                      (dict(thumbnail=(64, 64), scale_denom=2), "thumbnail takes no size"),
                      (dict(thumbnail=[(64, 64), (0, 64)]), "file 1"),
                      (dict(thumbnail=[(64, 64)]), "a list of 2"),
                      (dict(thumbnail=(64, 64), reducing_gap=0.9), "reducing_gap"),
                      (dict(size=(64, 64), reducing_gap=-1), "reducing_gap")]:
        for call in (ctx.decode_pixels, ctx.reencode):
            with pytest.raises(ValueError, match=words):
                call(files, 0, 0, **kw)


def test_c_argument_errors():
    lib = cuda.load()
    s, w, h = C.c_int(), C.c_int(), C.c_int()
    for args in [(0, 10, 5, 5, 2.0, 0), (10, 10, 0, 5, 2.0, 0), (10, 10, 5, 5, 0.5, 0), (10, 10, 5, 5, float("nan"), 0),
                 (10, 10, 5, 5, 2.0, 2)]:
        assert lib.jpegqs_cuda_thumbnail_geometry(*args, C.byref(s), C.byref(w), C.byref(h)) == -2, args
    assert lib.jpegqs_cuda_thumbnail_geometry(10, 10, 5, 5, 0.0, 0, C.byref(s), C.byref(w), C.byref(h)) == 0
    assert (s.value, w.value, h.value) == (1, 5, 5)
    src = np.zeros(300, np.uint8)
    out = np.zeros(300, np.uint8)
    assert lib.jpegqs_cuda_reduce_model(src.ctypes.data, 10, 10, 3, 0, 1, None, out.ctypes.data) == -2
    assert lib.jpegqs_cuda_reduce_model(src.ctypes.data, 10, 10, 2, 1, 1, None, out.ctypes.data) == -2
    assert lib.jpegqs_cuda_reduce_model(None, 10, 10, 3, 1, 1, None, out.ctypes.data) == -2
    assert lib.jpegqs_cuda_resize_model_box(src.ctypes.data, 10, 10, 3, 0, 0, None, 5, 5, 0.0, out.ctypes.data) == -2
    assert lib.jpegqs_cuda_resize_model_box(src.ctypes.data, 10, 10, 3, 0, 3, None, 5, 5, 0.99, out.ctypes.data) == -2
    assert lib.jpegqs_cuda_resize_model_box(src.ctypes.data, 10, 10, 3, 0, 3, (C.c_double * 4)(0, 0, 0, 10), 5, 5, 0.0,
                                            out.ctypes.data) == -2
    # the batch calls refuse bad thumbnail arguments without a context; with one, before anything runs
    n = 1
    data = (C.c_char_p * n)(THUMB_FILES[0])
    lens = (C.c_size_t * n)(len(THUMB_FILES[0]))
    rc = (C.c_int * n)()
    res = (cuda._PixelsResult * n)()
    outs = (C.c_void_p * n)(out.ctypes.data)
    box = (cuda._ResizeBox * n)(cuda._ResizeBox(0, 0, 0, 0, 64, 64))
    assert lib.jpegqs_cuda_pixels_batch_reduced(None, n, data, lens, 0, 0, 0, 1, 3, box, None, 0, 0, outs, 0, rc, res, 1,
                                                2.0) == -2
    jp = cuda._JpegParams(75, 2, 0)
    jo, jl = (C.c_void_p * n)(), (C.c_size_t * n)()
    assert lib.jpegqs_cuda_pixels_batch_jpeg_reduced(None, n, data, lens, 0, 0, 1, 3, box, C.byref(jp), 0, rc, res, jo, jl,
                                                     None, 0, 1, 2.0) == -2
