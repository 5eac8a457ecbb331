"""The blur and sharpen filters' host model (jpegqs_cuda_image_filter_model, the device's per-sample
functions and pass plan on one CPU thread) against Pillow's Image.filter with ImageFilter.BoxBlur,
GaussianBlur and UnsharpMask, byte for byte; a numpy restatement of the arithmetic that equals both; seven
mutants of it that Pillow's bytes reject; and the argument checks of the Python layer and the C model."""
import zlib

import numpy as np
import pytest

from jpegqs_b200 import cuda

Image = pytest.importorskip("PIL.Image")
ImageFilter = pytest.importorskip("PIL.ImageFilter")
F = ImageFilter


def pillow(a, filters):
    im = Image.fromarray(a)
    for f in filters if isinstance(filters, list) else [filters]:
        im = im.filter(f)
    return np.asarray(im)


def picture(rng, h, w, ch, binary=False):
    a = rng.randint(0, 256, (h, w, ch) if ch == 3 else (h, w)).astype(np.uint8)
    return (a > 127).astype(np.uint8) * 255 if binary else a


# ---- a numpy restatement, with the mutants as switches -------------------------------------------------
def box_line(p, R, double_ww=False, no_half=False, keep=False):
    """one box pass along the last axis; keep: the unrounded value (the no-uint8-rounding mutant)"""
    r = int(R)
    if double_ww:
        ww = int(16777216.0 / (R * 2.0 + 1.0))
    else:
        ww = int(np.float32(16777216.0) / (np.float32(R) * np.float32(2.0) + np.float32(1.0)))
    fw = (2 ** 24 - (2 * r + 1) * ww) // 2
    n = p.shape[-1]
    q = np.pad(p, [(0, 0)] * (p.ndim - 1) + [(r + 1, r + 1)], mode="edge")
    cs = np.concatenate([np.zeros(p.shape[:-1] + (1,), q.dtype), np.cumsum(q, axis=-1)], axis=-1)
    x = np.arange(n)
    acc = cs[..., x + 2 * r + 2] - cs[..., x + 1]
    far = q[..., x] + q[..., x + 2 * r + 2]
    v = acc * ww + far * fw
    if keep:
        return v / 2.0 ** 24
    return (v + (0 if no_half else 2 ** 23)) >> 24


def gauss_box(s):
    """BoxBlur.c's _gaussian_blur_radius(s, 3), in float32 where Pillow types float"""
    f = np.float32
    s = f(s)
    sigma2 = f(s * s / f(3))
    L = f(np.sqrt(12.0 * float(sigma2) + 1.0))
    l = f(np.floor((float(L) - 1.0) / 2.0))
    a = (f(2) * l + f(1)) * (l * (l + f(1)) - f(3) * sigma2)
    a = f(a / (f(6) * (sigma2 - (l + f(1)) * (l + f(1)))))
    return float(l + a)


def blur(a, rx, ry, passes, order="rows", **m):
    x = (a if a.ndim == 3 else a[..., None]).astype(np.int64)
    keep = m.get("keep", False)

    def rows(v):
        return np.moveaxis(box_line(np.moveaxis(v, 1, -1), rx, **m), -1, 1)

    def cols(v):
        return np.moveaxis(box_line(np.moveaxis(v, 0, -1), ry, **m), -1, 0)

    R, Cc = ([rows] * passes if rx else []), ([cols] * passes if ry else [])
    seq = R + Cc if order == "rows" else Cc + R if order == "cols" else [f for pair in zip(R, Cc) for f in pair]
    for f in seq:
        x = f(x)
    if keep:
        x = np.floor(x + 0.5).astype(np.int64)
    return x.reshape(a.shape)


def restated(a, f, ge=False, floor_div=False, **m):
    if isinstance(f, F.BoxBlur):
        rx, ry = f.radius if isinstance(f.radius, tuple) else (f.radius, f.radius)
        return blur(a, float(np.float32(rx)), float(np.float32(ry)), 1, **m).astype(np.uint8)
    if isinstance(f, F.GaussianBlur):
        sx, sy = f.radius if isinstance(f.radius, tuple) else (f.radius, f.radius)
        return blur(a, gauss_box(sx), gauss_box(sy), 3, **m).astype(np.uint8)
    g = gauss_box(f.radius)
    b = blur(a, g, g, 3, **m)
    d = a.astype(np.int64) - b
    q = d * f.percent
    div = q // 100 if floor_div else np.where(q < 0, -((-q) // 100), q // 100)
    sharp = np.clip(a + div, 0, 255)
    return np.where(np.abs(d) >= f.threshold if ge else np.abs(d) > f.threshold, sharp, a).astype(np.uint8)


def restated_chain(a, filters, **m):
    for f in filters:
        a = restated(a, f, **m)
    return a


# ---- the cases ------------------------------------------------------------------------------------------
SHAPES = [(1, 1), (1, 9), (9, 1), (1, 40), (40, 1), (7, 5), (16, 23), (24, 24)]
FILTERS = [F.BoxBlur(0), F.BoxBlur(0.05), F.BoxBlur(0.5), F.BoxBlur(0.99), F.BoxBlur(1), F.BoxBlur(2.5),
           F.BoxBlur((3, 0)), F.BoxBlur((0, 4.25)), F.BoxBlur(30), F.BoxBlur((1.5, 60)),
           F.GaussianBlur(0), F.GaussianBlur(0.05), F.GaussianBlur(0.6), F.GaussianBlur(), F.GaussianBlur(2.7),
           F.GaussianBlur((5, 0)), F.GaussianBlur((0, 1.1)), F.GaussianBlur(-3.3), F.GaussianBlur((-2, 7.5)),
           F.GaussianBlur(30),
           F.UnsharpMask(), F.UnsharpMask(0, 150, 3), F.UnsharpMask(0.4, 300, 0), F.UnsharpMask(2, 150, 3),
           F.UnsharpMask(3.5, -50, 0), F.UnsharpMask(1, 500, 255), F.UnsharpMask(1.7, 100, -1),
           F.UnsharpMask(-2, 250, 10), F.UnsharpMask(30, 120, 1)]


def _name(f):
    return f"{type(f).__name__}{vars(f)}"


@pytest.mark.parametrize("f", FILTERS, ids=_name)
@pytest.mark.parametrize("ch", [1, 3])
def test_model_is_pillow(f, ch):
    rng = np.random.RandomState(zlib.crc32(f"{_name(f)} {ch}".encode()))
    for h, w in SHAPES:
        for binary in (False, True):
            a = picture(rng, h, w, ch, binary)
            assert np.array_equal(cuda.image_filter_model(a, f), pillow(a, f)), (h, w, binary)


def test_model_is_pillow_radius_sweep():
    """fractional radii 0.05 .. 12 in steps of 0.05, every filter, L and RGB"""
    rng = np.random.RandomState(5)
    grey, rgb = picture(rng, 19, 31, 1), picture(rng, 13, 17, 3, binary=True)
    for r in np.arange(0.05, 12.0, 0.05):
        r = float(r)
        for f in (F.BoxBlur(r), F.BoxBlur((r, 12 - r)), F.GaussianBlur(r), F.UnsharpMask(r, 180, 2)):
            for a in (grey, rgb):
                assert np.array_equal(cuda.image_filter_model(a, f), pillow(a, f)), (_name(f), a.shape)


@pytest.mark.parametrize("ch", [1, 3])
def test_model_is_pillow_radius_past_the_picture(ch):
    rng = np.random.RandomState(6)
    a = picture(rng, 6, 11, ch)
    for f in (F.BoxBlur(11), F.BoxBlur((10.5, 6)), F.BoxBlur((200, 5.5)), F.GaussianBlur((6, 11)),
              F.GaussianBlur(400), F.UnsharpMask(9, 200, 0)):
        assert np.array_equal(cuda.image_filter_model(a, f), pillow(a, f)), _name(f)


def test_model_is_pillow_at_the_radius_cap():
    rng = np.random.RandomState(7)
    for a in (picture(rng, 5, 9, 1), picture(rng, 4, 3, 3)):
        for f in (F.BoxBlur(65535), F.BoxBlur((65535, 0.5)), F.GaussianBlur(65535), F.GaussianBlur(-65535),
                  F.UnsharpMask(65535, 8421504, 0), F.UnsharpMask(2, -8421504, 1)):
            assert np.array_equal(cuda.image_filter_model(a, f), pillow(a, f)), _name(f)


def test_model_is_pillow_wider_than_the_fused_rows():
    """rows of more than 16384 bytes take the per-pass line path on the device, and in the model"""
    rng = np.random.RandomState(8)
    for a in (picture(rng, 3, 5500, 3), picture(rng, 2, 16400, 1, binary=True)):
        for f in (F.GaussianBlur(20), F.BoxBlur((7.5, 1)), F.UnsharpMask(2, 150, 3)):
            assert np.array_equal(cuda.image_filter_model(a, f), pillow(a, f)), (_name(f), a.shape)


CHAINS = [[F.GaussianBlur(1.5), F.UnsharpMask(2, 150, 3)], [F.UnsharpMask(), F.UnsharpMask(1, 300, 0)],
          [F.BoxBlur((2, 0)), F.BoxBlur((0, 2)), F.GaussianBlur(0)], [F.BoxBlur(0), F.UnsharpMask(0.5, 90, 0)],
          [F.UnsharpMask(0, 100, 0), F.BoxBlur(1.25), F.GaussianBlur((0, 3)), F.UnsharpMask(4, 60, 5)]]


@pytest.mark.parametrize("chain", range(len(CHAINS)))
@pytest.mark.parametrize("ch", [1, 3])
def test_chain_is_pillow(chain, ch):
    rng = np.random.RandomState(chain * 2 + ch)
    for h, w in ((1, 1), (12, 1), (1, 12), (21, 14)):
        a = picture(rng, h, w, ch)
        assert np.array_equal(cuda.image_filter_model(a, CHAINS[chain]), pillow(a, CHAINS[chain])), (h, w)


def test_restatement_is_the_model():
    rng = np.random.RandomState(9)
    for h, w, ch in ((1, 1, 1), (9, 14, 3), (17, 5, 1), (1, 30, 3)):
        a = picture(rng, h, w, ch)
        for f in FILTERS:
            assert np.array_equal(restated(a, f), cuda.image_filter_model(a, f)), (_name(f), a.shape)
        for chain in CHAINS:
            assert np.array_equal(restated_chain(a, chain), cuda.image_filter_model(a, chain))


MUTANTS = {"threshold >=": dict(ge=True), "floor division": dict(floor_div=True), "double ww": dict(double_ww=True),
           "no + 2^23": dict(no_half=True), "columns before rows": dict(order="cols"),
           "interleaved passes": dict(order="interleave"), "no uint8 rounding between passes": dict(keep=True)}


@pytest.mark.parametrize("mutant", list(MUTANTS))
def test_mutants_are_not_pillow(mutant):
    rng = np.random.RandomState(10)
    pics = [picture(rng, 23, 29, 3), picture(rng, 31, 17, 1, binary=True), picture(rng, 40, 40, 3, binary=True)]
    filters = [F.UnsharpMask(r, p, t) for r in (0.8, 2, 3.3) for p in (-50, 150, 333) for t in (0, 3, 9)]
    filters += [F.BoxBlur(float(r)) for r in np.arange(0.05, 20, 0.05)]
    filters += [F.GaussianBlur(float(r)) for r in np.arange(0.1, 20, 0.1)]
    m = MUTANTS[mutant]
    for f in filters:
        for a in pics:
            if not np.array_equal(restated(a, f, **m), pillow(a, f)):
                return
    pytest.fail(f"the {mutant} mutant gives Pillow's bytes on every case")


# ---- argument checks ---------------------------------------------------------------------------------
def test_none_and_empty_are_a_copy():
    a = picture(np.random.RandomState(11), 5, 6, 3)
    assert np.array_equal(cuda.image_filter_model(a, None), a)
    assert np.array_equal(cuda.image_filter_model(a, []), a)


def test_classes_take_pillows_defaults():
    a = picture(np.random.RandomState(12), 14, 9, 3)
    assert np.array_equal(cuda.image_filter_model(a, F.GaussianBlur), pillow(a, F.GaussianBlur))
    assert np.array_equal(cuda.image_filter_model(a, [F.UnsharpMask, F.GaussianBlur(1)]),
                          pillow(a, [F.UnsharpMask, F.GaussianBlur(1)]))
    with pytest.raises(TypeError):                     # BoxBlur has no default radius, in Pillow as here
        cuda.image_filter_model(a, F.BoxBlur)


@pytest.mark.parametrize("f,name", [(F.SHARPEN, "SHARPEN"), (F.SMOOTH, "SMOOTH"), (F.DETAIL(), "DETAIL"),
                                    (F.Kernel((3, 3), [1] * 9), "Kernel"), (F.MedianFilter(3), "MedianFilter"),
                                    (F.RankFilter(3, 1), "RankFilter"), ("blur", "str")])
def test_other_filters_are_refused_by_name(f, name):
    a = np.zeros((4, 4), np.uint8)
    for filt in (f, [F.GaussianBlur(1), f]):
        with pytest.raises(ValueError, match=name):
            cuda.image_filter_model(a, filt)


def _refused(f, match):
    with pytest.raises(ValueError, match=match):
        cuda.image_filter_model(np.zeros((4, 4, 3), np.uint8), f)


def test_bad_values_are_refused():
    b = F.BoxBlur(1)
    b.radius = -1
    _refused(b, "radius must be >= 0")
    b.radius = (2, -0.5)
    _refused(b, "radius must be >= 0")
    for r in (65535.5, -65536, float("inf"), float("nan"), (1, 70000)):
        _refused(F.GaussianBlur(r), "radius")
    _refused(F.BoxBlur(1e7), "radius")
    _refused(F.GaussianBlur((1, 2, 3)), "radius")
    _refused(F.UnsharpMask(1e6, 150, 3), "radius")
    _refused(F.UnsharpMask(2, 150.0, 3), "percent")
    _refused(F.UnsharpMask(2, 8421505, 3), "percent")
    _refused(F.UnsharpMask(2, -8421505, 3), "percent")
    _refused(F.UnsharpMask(2, 150, 3.0), "threshold")
    _refused(F.UnsharpMask(2, 150, 2 ** 31), "threshold")
    _refused(F.UnsharpMask("2", 150, 3), "radius")


def test_c_model_refusals():
    lib = cuda.load()
    a = np.zeros((3, 4, 3), np.uint8)
    out = np.zeros_like(a)

    def run(kind, rx, ry, percent=0, threshold=0, n=1, ch=3):
        f = (cuda._ImageFilter * 1)(cuda._ImageFilter(kind, rx, ry, percent, threshold))
        return lib.jpegqs_cuda_image_filter_model(a.ctypes.data, 4, 3, ch, f, n, out.ctypes.data)

    assert run(1, 1.0, 2.0) == 0
    assert run(2, -1.0, 2.0) == 0
    assert run(3, 2.0, 2.0, 8421504, -5) == 0
    for args in ((0, 1.0, 1.0), (4, 1.0, 1.0), (1, -1.0, 1.0), (2, float("nan"), 1.0), (2, 1.0, 65536.0),
                 (3, 1.0, 2.0, 150, 3), (3, 1.0, 1.0, 8421505, 3)):
        assert run(*args) == -2, args
        assert "filter 0" in lib.jpegqs_cuda_last_error(None).decode()
    assert run(1, 1.0, 1.0, n=65) == -2
    assert run(1, 1.0, 1.0, ch=4) == -2
    assert "channels" in lib.jpegqs_cuda_last_error(None).decode()
