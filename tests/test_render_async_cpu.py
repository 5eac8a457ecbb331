"""CPU side of the stream-ordered render: the libjpeg pixel oracle (tests/libjpeg_pixels.py) is
pinned to Pillow's own decodes, fails loudly where libjpeg cannot code a coefficient set, and agrees
with the renderers' arithmetic (libjpeg_pixels.device_model) on synthetic and saturated content;
and QsContext.render_async checks its arguments before the library is called."""
import numpy as np
import pytest

import hard_content as hc
import libjpeg_pixels as lp
import oracle_lib as ol
import wave_geometry as wg
from jpegqs_b200 import cuda as qc
from render_images import GEOMETRIES, SAMPLINGS, make

PIL = pytest.importorskip("PIL.Image")
needs_libjpeg = pytest.mark.skipif(lp.JPEG_SO is None, reason="no libjpeg inside Pillow")

from test_cli import _picture  # noqa: E402

PILLOW_FILES = [("420", 64, 48, False, dict(quality=75)),
                ("422", 160, 120, False, dict(quality=30, subsampling=1, optimize=True)),
                ("444", 123, 77, False, dict(quality=90, subsampling=0)),
                ("gray", 97, 61, True, dict(quality=85)),
                ("progressive", 200, 133, False, dict(quality=50, subsampling=2, progressive=True)),
                ("restart", 250, 190, False, dict(quality=80, restart_marker_rows=1))]


@needs_libjpeg
@pytest.mark.parametrize("name,w,h,gray,kw", PILLOW_FILES, ids=[f[0] for f in PILLOW_FILES])
def test_round_trip_is_pillows_decode(tmp_path, name, w, h, gray, kw):
    path = str(tmp_path / "in.jpg")
    _picture(w, h, gray, 5).save(path, **kw)
    got = lp.decode(lp.read_coefficients(path))
    assert np.array_equal(got, np.asarray(PIL.open(path).convert("RGB")))


@needs_libjpeg
@pytest.mark.parametrize("ss", ["440", "411"] + list(GEOMETRIES))
def test_written_file_is_what_pillow_decodes(tmp_path, ss):
    """Samplings Pillow cannot write: the helper's own file, opened by Pillow."""
    path = str(tmp_path / "out.jpg")
    im = make(203, 149, ss, "k50", "saturated", seed=1)
    got = lp.decode(im, jpeg_path=path)
    assert np.array_equal(got, np.asarray(PIL.open(path).convert("RGB")))
    assert [(c.h_samp, c.v_samp) for c in lp.read_coefficients(path).comps] == [(c.h_samp, c.v_samp) for c in im.comps]


@needs_libjpeg
def test_uncodable_coefficients_fail_loudly():
    im = hc.make_image(64, 16, "gray", hc.TABLES["k50"], "synth", seed=1)
    im.comps[0].coef = im.comps[0].coef.copy()
    im.comps[0].coef[0, 0, 0], im.comps[0].coef[0, 1, 0] = -1500, 1500     # a DC difference of 12 bits
    with pytest.raises(lp.LibjpegError):
        lp.decode(im)


# Pillow's libjpeg-turbo decodes with its SIMD islow IDCT; the library renders with the reference's
# 32-bit islow and a clamp.  Measured here on every sampling, for still-quantized and smoothed
# coefficients of synthetic and saturated content (letterbox bars, full-contrast strokes, Nyquist
# checkers, wrapping ramps) under coarse, fine and random quant tables: no pixel differs.
@needs_libjpeg
@pytest.mark.parametrize("ss", SAMPLINGS + GEOMETRIES)
def test_renderer_arithmetic_is_libjpegs(ss):
    for content in ("synth", "saturated"):
        for table in ("k10", "k90", "rand"):
            im = make(203, 149, ss, table, content, seed=5)
            assert np.array_equal(lp.device_model(im), lp.decode(im)), (content, table)
            for flags in (0, 7, 8):
                out = ol.run_oracle(im, flags, 1)[1]
                assert np.array_equal(lp.device_model(out), lp.decode(out)), (content, table, flags)


# ---- the Python argument checks of render_async ----------------------------------------------

class _Untouchable:
    def __getattr__(self, name):
        raise AssertionError(f"the library was called ({name}) before the arguments were checked")


def _ctx():
    ctx = object.__new__(qc.QsContext)
    ctx.lib, ctx.h, ctx.device = _Untouchable(), None, 0
    return ctx


def _image():
    return wg.geometry(64, 48, "420")


def _tensors(im, dtype=None, device="cpu"):
    import torch
    return [torch.zeros((c.hblk, c.wblk, 64), dtype=dtype or torch.int16, device=device) for c in im.comps]


def test_render_async_rejects_wrong_coefficient_tensors():
    import torch
    im = _image()
    with pytest.raises(TypeError, match="dtype"):
        _ctx().render_async([im], [_tensors(im, dtype=torch.int32)])
    with pytest.raises(ValueError, match="coefficient tensors"):
        _ctx().render_async([im], [_tensors(im)[:2]])
    ts = _tensors(im)
    ts[0] = torch.zeros((im.comps[0].wblk, im.comps[0].hblk, 64), dtype=torch.int16).transpose(0, 1)
    with pytest.raises(ValueError, match="contiguous"):
        _ctx().render_async([im], [ts])
    with pytest.raises(ValueError, match="expected cuda:0"):
        _ctx().render_async([im], [_tensors(im)])
    with pytest.raises(ValueError, match="CUDA tensors"):
        qc.render_async([im], [_tensors(im)])


def test_render_async_rejects_wrong_outputs():
    import torch
    im = _image()
    ts = _tensors(im, device="meta")
    with pytest.raises(ValueError, match="shape"):
        _ctx().render_async([im], [ts], out=[torch.empty((3, 48, 64), dtype=torch.uint8, device="meta")])
    with pytest.raises(TypeError, match="uint8"):
        _ctx().render_async([im], [ts], out=[torch.empty((48, 64, 3), dtype=torch.int16, device="meta")])
    with pytest.raises(ValueError, match="contiguous"):
        _ctx().render_async([im], [ts], layout="chw",
                            out=[torch.empty((64, 48, 3), dtype=torch.uint8, device="meta").permute(2, 1, 0)])
    with pytest.raises(ValueError, match="one entry per image"):
        _ctx().render_async([im], [ts], out=[])
    with pytest.raises(ValueError, match="layout"):
        _ctx().render_async([im], [ts], layout="nhwc")


def test_render_async_rejects_wrong_status_and_up():
    import torch
    im = _image()
    ts = _tensors(im, device="meta")
    with pytest.raises(ValueError, match="status"):
        _ctx().render_async([im], [ts], status=torch.zeros((2, 2), dtype=torch.int32, device="meta"))
    with pytest.raises(ValueError, match="status"):
        _ctx().render_async([im], [ts], status=torch.zeros((1, 2), dtype=torch.int64, device="meta"))
    with pytest.raises(ValueError, match="up-sampled but up"):
        _ctx().render_async([im], [ts], status=[True])
    with pytest.raises(ValueError, match="two tensors"):
        _ctx().render_async([im], [ts], up=[(ts[1],)])
    with pytest.raises(ValueError, match="expected cuda:0"):
        _ctx().render_async([im], [ts], up=[tuple(_tensors(im, device="meta")[:1] * 2)])
