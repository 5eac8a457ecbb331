"""CPU side of the scaled render (include/jpegqs_cuda.h jpegqs_cuda_render_scaled_async): render_model,
the library's restatement of the render on one CPU thread, is libjpeg's scaled decode (scale_num 1,
scale_denom d, JDCT_ISLOW, fancy up-sampling) byte for byte, with the SIMD and the C code paths of the
library, on every sampling the render takes (render_images.SAMPLINGS and GEOMETRIES), on sizes where the up-samplers change branch, and on
quantized, oracle-smoothed and saturated coefficient sets.  A numpy restatement of the same rules
(_restated) is pinned to render_model, and mutants of it - a reduced-IDCT constant, the "no fancy
up-sampling at scaled size 1" rule, the downsampled-width rounding - each disagree with libjpeg on
these cases, so the cases would catch those mistakes in the library.  No GPU needed."""
import ctypes as C

import numpy as np
import pytest

import hard_content as hc
import libjpeg_pixels as lp
import libjpeg_scaled as ls
import oracle_lib as ol
from jpegqs_b200 import cuda as qc
from jpegqs_b200.image import JCS_YCbCr
from render_images import GEOMETRIES, SAMPLINGS, make

needs_libjpeg = pytest.mark.skipif(lp.JPEG_SO is None, reason="no libjpeg inside Pillow")

SCALES = (2, 4, 8)
# 1x1, odd sizes, and widths at which a 4:2:2 chroma's downsampled width at the scaled size is 1, 2
# or 3 (5 and 12 at 1/2, 8, 16 and 24 at 1/4), where h2v1 switches between replication and fancy
SIZES = ((1, 1), (7, 9), (33, 47), (203, 149), (5, 6), (12, 20), (8, 3), (16, 5), (24, 17))


def _as_rgb(px):
    return np.repeat(px, 3, axis=2) if px.shape[2] == 1 else px


def _coefficient_sets(ss, w, h):
    """(name, image): still quantized under coarse, fine and random tables, saturated content, and the
    oracle's smoothing at q3 and at q6 (which up-samples 4:2:0 chroma to 4:4:4)"""
    im = make(w, h, ss, "k50", "synth", seed=3)
    yield "k50", im
    yield "k10-saturated", make(w, h, ss, "k10", "saturated", seed=5)
    yield "rand", make(w, h, ss, "rand", "synth", seed=7)
    yield "q3", ol.run_oracle(im, 0, 2)[1]
    yield "q6", ol.run_oracle(make(w, h, ss, "k90", "saturated", seed=9), 7, 1)[1]


# ---- the numpy restatement and its mutants ----------------------------------------------------

def _geometry(image, d, mutant=None):
    """per component (DCT scaled size, downsampled width, height, h expansion, v expansion)"""
    cs = image.comps
    maxh, maxv = max(c.h_samp for c in cs), max(c.v_samp for c in cs)
    m = 8 // d
    out = []
    for c in cs:
        s = m
        while s < 8 and (maxh * m) % (c.h_samp * s * 2) == 0 and (maxv * m) % (c.v_samp * s * 2) == 0:
            s *= 2
        if mutant == "dsw_round":
            cw = image.width * c.h_samp * s // (maxh * 8)
        else:
            cw = -(-image.width * c.h_samp * s // (maxh * 8))
        ch = -(-image.height * c.v_samp * s // (maxv * 8))
        out.append((s, max(cw, 1), ch, maxh * m // (c.h_samp * s), maxv * m // (c.v_samp * s)))
    return out


def _red4(v, k4):
    t0 = v[0] << 14
    t2 = v[2] * 15137 - v[6] * 6270
    t10, t12 = t0 + t2, t0 - t2
    z1, z2, z3, z4 = v[7], v[5], v[3], v[1]
    o0 = -z1 * 1730 + z2 * 11893 - z3 * 17799 + z4 * k4
    o2 = -z1 * 4176 - z2 * 4926 + z3 * 7373 + z4 * 20995
    return np.stack([t10 + o2, t12 + o0, t12 - o0, t10 - o2])


def _red2(v):
    t10 = v[0] << 15
    t0 = -v[7] * 5906 + v[5] * 6967 - v[3] * 10426 + v[1] * 29692
    return np.stack([t10 + t0, t10 - t0])


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def _samples(comp, s, mutant=None):
    """the component's samples at DCT scaled size s: [hblk * s, wblk * s] int64"""
    if s == 8:
        return lp._plane(comp)
    c = comp.coef.astype(np.int64).reshape(comp.hblk, comp.wblk, 8, 8)
    if comp.quant is not None and int(np.bitwise_or.reduce(comp.quant.astype(np.int64))) > 1:
        c = c * comp.quant.astype(np.int64).reshape(8, 8)
    if s == 1:
        v = _descale(c[:, :, 0, 0], 3) & 1023
        return np.select([v < 128, v < 512, v < 896], [v + 128, 255, 0], v - 896)
    fn, p1, p2 = ((lambda v: _red4(v, 8698 if mutant == "idct_const" else 8697)), 12, 19) if s == 4 else (_red2, 13, 20)
    ws = _descale(fn(np.moveaxis(c, 2, 0)), p1)                  # columns: [row, by, bx, col]
    px = np.clip(_descale(fn(np.moveaxis(ws, 3, 0)), p2) + 128, 0, 255)   # rows: [col, row, by, bx]
    return np.transpose(px, (2, 1, 3, 0)).reshape(comp.hblk * s, comp.wblk * s)


def _restated(image, d, mutant=None):
    """render_model's pixels [ceil(H/d), ceil(W/d), 3], restated in numpy"""
    w, h = -(-image.width // d), -(-image.height // d)
    fancy = d != 8 if mutant != "fancy_at_1" else d == 8
    planes = []
    for comp, (s, cw, ch, hs, vs) in zip(image.comps, _geometry(image, d, mutant)):
        p = _samples(comp, s, mutant)
        if fancy or (hs, vs) == (1, 1):
            planes.append(lp._upsample(p, hs, vs, cw, ch, w, h))
        else:
            oy, ox = np.mgrid[0:h, 0:w]
            planes.append(p[np.minimum(oy // vs, ch - 1), np.minimum(ox // hs, cw - 1)])
    if len(planes) == 1:
        planes = planes * 3
    y, c1, c2 = planes
    if image.colorspace == JCS_YCbCr and len(image.comps) == 3:
        cb, cr = c1 - 128, c2 - 128
        r = y + ((91881 * cr + 32768) >> 16)
        g = y + ((-22554 * cb + 32768 - 46802 * cr) >> 16)
        b = y + ((116130 * cb + 32768) >> 16)
        y, c1, c2 = (np.clip(v, 0, 255) for v in (r, g, b))
    return np.stack([y, c1, c2], -1).astype(np.uint8)


# ---- render_model against libjpeg ---------------------------------------------------------------

@needs_libjpeg
@pytest.mark.parametrize("ss", SAMPLINGS + GEOMETRIES)
def test_model_full_size_is_libjpeg(ss):
    """d = 1 is the unscaled render: libjpeg_pixels' decode and render_async's arithmetic"""
    for name, im in _coefficient_sets(ss, 203, 149):
        got = qc.render_model(im)
        assert np.array_equal(got, lp.decode(im)), name
        assert np.array_equal(got, lp.device_model(im)), name
        assert np.array_equal(got.transpose(2, 0, 1), qc.render_model(im, layout="chw")), name


@needs_libjpeg
@pytest.mark.parametrize("d", SCALES)
@pytest.mark.parametrize("ss", SAMPLINGS + GEOMETRIES)
def test_model_is_libjpegs_scaled_decode(ss, d):
    for w, h in SIZES:
        for name, im in _coefficient_sets(ss, w, h):
            got = qc.render_model(im, scale_denom=d)
            assert got.shape == (-(-h // d), -(-w // d), 3)
            for simd in (True, False):
                want, _ = ls.decode(im, d, simd=simd)
                assert np.array_equal(got, _as_rgb(want)), (name, w, h, simd)
            assert np.array_equal(got.transpose(2, 0, 1), qc.render_model(im, layout="chw", scale_denom=d))


@needs_libjpeg
@pytest.mark.parametrize("ss", ["422", "420", "440", "411"] + list(GEOMETRIES))
def test_scaled_geometry_is_libjpegs(ss):
    """the DCT scaled sizes jpeg_start_decompress chose are the ones the restatement (and the library,
    through the test above) uses: 4:2:0 chroma at 1/2 takes the full 8x8 IDCT, for instance"""
    im = make(64, 48, ss, "k50", "synth", seed=1)
    for d in SCALES:
        _, sizes = ls.decode(im, d)
        assert sizes == [g[0] for g in _geometry(im, d)], d
    assert [g[0] for g in _geometry(make(64, 48, "420", "k50", "synth", 1), 2)] == [4, 8, 8]


@needs_libjpeg
@pytest.mark.parametrize("d", (1,) + SCALES)
def test_model_reads_upsampled_chroma(d):
    """upsampled=(cb, cr) renders components 1 and 2 from luma-sized arrays, as the 4:4:4 set the
    smoothing writes"""
    im = make(203, 149, "420", "k90", "saturated", seed=2)
    ret, out, up = ol.run_oracle(im, 7, 1, with_upsampled=True)
    assert up
    # the 4:2:0 geometry with the run's luma and tables (all ones after a run), chroma from the pair
    src = im.clone()
    for c, o in zip(src.comps, out.comps):
        c.quant = o.quant
    src.comps[0].coef = out.comps[0].coef
    got = qc.render_model(src, upsampled=(out.comps[1].coef, out.comps[2].coef), scale_denom=d)
    assert np.array_equal(got, qc.render_model(out, scale_denom=d))
    assert np.array_equal(got, _as_rgb(ls.decode(out, d)[0]))


@needs_libjpeg
def test_hard_files_decode_like_libjpeg(tmp_path):
    """files Pillow writes (progressive, restart markers, grey), read with the library's reader"""
    PIL = pytest.importorskip("PIL.Image")
    from test_cli import _picture
    for name, (w, h, gray, kw) in {"420": (161, 97, False, dict(quality=75)),
                                   "422": (130, 51, False, dict(quality=30, subsampling=1)),
                                   "gray": (97, 61, True, dict(quality=85)),
                                   "progressive": (200, 133, False, dict(quality=50, progressive=True))}.items():
        path = str(tmp_path / f"{name}.jpg")
        _picture(w, h, gray, 5).save(path, **kw)
        im = qc.read_jpeg(open(path, "rb").read())
        for d in SCALES:
            assert np.array_equal(qc.render_model(im, scale_denom=d), _as_rgb(ls.decode_file(path, d)[0])), (name, d)


# ---- the restatement, and its mutants -------------------------------------------------------------

MUTANTS = ("idct_const", "fancy_at_1", "dsw_round")


@needs_libjpeg
def test_mutants_are_caught():
    """_restated equals render_model on the cases above; each mutant of it differs from libjpeg on at
    least one of them, so the same mistake in the library would fail test_model_is_libjpegs_scaled_decode"""
    caught = {m: [] for m in MUTANTS}
    for ss in SAMPLINGS:
        for w, h in ((203, 149), (33, 47), (12, 20), (24, 17)):
            for name, im in _coefficient_sets(ss, w, h):
                for d in SCALES:
                    want = _as_rgb(ls.decode(im, d)[0])
                    assert np.array_equal(_restated(im, d), qc.render_model(im, scale_denom=d)), (ss, w, h, name, d)
                    for m in MUTANTS:
                        got = _restated(im, d, m)
                        if got.shape != want.shape or not np.array_equal(got, want):
                            caught[m].append((ss, w, h, name, d))
    for m in MUTANTS:
        assert caught[m], f"mutant {m} is not caught"


# ---- argument checks ---------------------------------------------------------------------------------

@pytest.mark.parametrize("d", [0, 3, 16, -2])
def test_c_rejects_bad_scale_without_a_context(d):
    lib = qc.load()
    im = make(16, 16, "420", "k50", "synth", seed=1)
    arrays = [np.ascontiguousarray(c.coef) for c in im.comps]
    arr = qc._image_array([im], [[a.ctypes.data for a in arrays]])
    out = np.zeros(16 * 16 * 3, np.uint8)
    assert lib.jpegqs_cuda_render_model(arr, 0, 0, d, out.ctypes.data) == -2
    assert "scale_denom" in lib.jpegqs_cuda_last_error(None).decode()
    assert not out.any()
    # no context: an argument error, nothing else touched
    assert lib.jpegqs_cuda_render_scaled_async(None, 1, arr, None, 0, d, (C.c_void_p * 1)(out.ctypes.data), None) == -2
    assert lib.jpegqs_cuda_pixels_batch_scaled(None, 0, None, None, 0, 0, 0, d, 0, None, 0, None, None) == -2


@pytest.mark.parametrize("d", [0, 3, 16, 2.0, True, "2"])
def test_python_rejects_bad_scale(d):
    im = make(16, 16, "420", "k50", "synth", seed=1)
    with pytest.raises(ValueError, match="scale_denom"):
        qc.render_model(im, scale_denom=d)
    from test_render_async_cpu import _ctx, _tensors
    with pytest.raises(ValueError, match="scale_denom"):
        _ctx().render_async([im], [_tensors(im, device="meta")], scale_denom=d)
    with pytest.raises(ValueError, match="scale_denom"):
        _ctx().decode_pixels([b"\xff\xd8"], 0, 1, scale_denom=d)


def test_python_checks_scaled_output_shapes():
    import torch
    from test_render_async_cpu import _ctx, _tensors
    im = make(203, 149, "420", "k50", "synth", seed=1)
    ts = _tensors(im, device="meta")
    with pytest.raises(ValueError, match=r"shape \(149, 203, 3\), expected \(38, 51, 3\)"):
        _ctx().render_async([im], [ts], scale_denom=4, out=[torch.empty((149, 203, 3), dtype=torch.uint8, device="meta")])
    with pytest.raises(ValueError, match=r"expected \(3, 19, 26\)"):
        _ctx().render_async([im], [ts], layout="chw", scale_denom=8,
                            out=[torch.empty((3, 38, 51), dtype=torch.uint8, device="meta")])
    assert qc.render_model(im, scale_denom=4).shape == (38, 51, 3)


def test_model_rejects_what_the_render_does_not_take():
    im = hc.make_image(16, 16, "420", hc.TABLES["k50"], "synth", seed=1)
    im.comps = im.comps[:2]
    with pytest.raises(qc.QsError, match="1 or 3 components"):
        qc.render_model(im, scale_denom=2)
