"""jpegqs_cuda_pixels_batch / QsContext.decode_pixels checks that need no GPU: the Python wrapper's
argument checks, the C call without a context, and the output size rule callers size out[i] with
(transcode_route's width, height and component count)."""
import ctypes as C

import pytest

PIL = pytest.importorskip("PIL.Image")

import decode_files as df
from jpegqs_b200 import cuda
from test_cli import FILES, write_jpegs


@pytest.fixture(scope="module")
def jpegs(tmp_path_factory):
    return write_jpegs(str(tmp_path_factory.mktemp("jpegs")))


def _unbound():
    """A QsContext without a device: the wrapper's checks run before it touches one."""
    return object.__new__(cuda.QsContext)


def test_python_wrapper_checks_its_arguments():
    good = df.pillow_jpeg(64, 48, quality=75)
    ctx = _unbound()
    assert cuda.QsContext.decode_pixels(ctx, [], 0, 3) == []
    assert cuda.QsContext.decode_pixels(ctx, (), 0, 3) == []
    for bad in (good, "text", None, 12, bytearray(good), memoryview(good)):
        with pytest.raises(TypeError):
            cuda.QsContext.decode_pixels(ctx, bad, 0, 3)
    for bad in ([good, None], [good, "text"], [12]):
        with pytest.raises(TypeError):
            cuda.QsContext.decode_pixels(ctx, bad, 0, 3)
    for layout in ("rgb", "HWC", 0, None):
        with pytest.raises(ValueError):
            cuda.QsContext.decode_pixels(ctx, [good], 0, 3, layout=layout)
    for device in ("gpu", "cuda:0", 0, None):
        with pytest.raises(ValueError):
            cuda.QsContext.decode_pixels(ctx, [good], 0, 3, device=device)
    with pytest.raises(ValueError):
        cuda.QsContext.decode_pixels(ctx, [good], 0, 3, max_device_bytes=-1)


def test_c_call_without_a_context():
    lib = cuda.load()
    data = df.pillow_jpeg(64, 48, quality=75)
    ptrs = (C.c_char_p * 1)(data)
    lens = (C.c_size_t * 1)(len(data))
    buf = (C.c_uint8 * (64 * 48 * 3))()
    outs = (C.c_void_p * 1)(C.addressof(buf))
    rc = (C.c_int * 1)(7)
    res = (cuda._PixelsResult * 1)()
    res[0].channels = 9
    f = lib.jpegqs_cuda_pixels_batch
    assert f(None, 1, ptrs, lens, 0, 3, 0, 0, outs, 0, rc, res) == -2
    assert f(None, 1, None, None, 0, 3, 0, 0, None, 0, None, None) == -2
    assert f(None, 0, None, None, 0, 3, 0, 0, None, 0, None, None) == -2
    assert f(None, 1, ptrs, lens, 0, 3, 5, 7, outs, 0, rc, res) == -2
    assert rc[0] == 7 and res[0].channels == 9 and not res[0].reason      # nothing touched
    assert bytes(buf) == bytes(len(buf))


def _route_shape(data):
    info = cuda._FileInfo()
    assert cuda.load().jpegqs_cuda_transcode_route(data, len(data), None, C.byref(info)) >= 0
    return info.image_width, info.image_height, info.ncomp


def test_output_size_rule(jpegs):
    """Width, height and channels from transcode_route's info, for every flavour the suite writes: grey
    files give one channel, colour files three; CMYK reports four components, which the call rejects."""
    for name, w, h, gray, _ in FILES:
        with open(jpegs[name], "rb") as f:
            assert _route_shape(f.read()) == (w, h, 1 if gray else 3), name
    assert _route_shape(df.pillow_jpeg(120, 80, "CMYK", quality=85)) == (120, 80, 4)
