"""Thumbnails on the GPU.  decode_pixels(thumbnail=) and reencode(thumbnail=) give, for file i, Pillow's
    im = Image.open(F); [im = exif_transpose(im) / im.transpose(...)]; [im = im.convert(mode)]
    im.thumbnail(bound, filter, reducing_gap); [im.save(...)]
with F the file the jpegqs tool writes for the same options (the input file at -q 3 -n 0): each file at
its own draft scale, 1 to 8 in one call, then Pillow's reduce and float-box resize.  Both layouts and
output kinds, host-decoded files, orientation and mode (CMYK included), the 8K file to 256 px and to 16 px
with gap 1.0, forced splits and shuffled order, a refused file failing alone, and reducing_gap on the
size / crop path against crop().resize(reducing_gap=)."""
import ctypes as C
import io

import numpy as np
import pytest
from PIL import ImageOps

from test_gpu_pixels_batch import corpus, ctx  # noqa: F401  (module fixtures)
from test_gpu_pixel_modes import METHODS, OPTS, files, tool_file  # noqa: F401  (module fixtures)

import jpegqs_b200 as qs
from jpegqs_b200 import cuda

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
Image = pytest.importorskip("PIL.Image")

FILTERS = {"lanczos": Image.Resampling.LANCZOS, "bilinear": Image.Resampling.BILINEAR,
           "bicubic": Image.Resampling.BICUBIC, "box": Image.Resampling.BOX, "hamming": Image.Resampling.HAMMING}
NAMES = ["base420", "base444", "prog420", "gray", "opt422", "prog444", "rst", "progrst", "tinyprog", "dense444", "coarse420"]
BOUNDS = [(256, 256), (64, 64), (24, 30), (4000, 4000), (100, 300), (33, 17), (128, 96)]


def _names(corpus):  # noqa: F811
    return [n for n in NAMES if n in corpus]


def pillow_thumb(data, bound, filt="bicubic", gap=2.0, o=None, mode=None):
    im = Image.open(io.BytesIO(data))
    if o == "exif":
        im = ImageOps.exif_transpose(im)
    elif o is not None:                           # an explicit orientation loads the picture, 1 included
        im = im.transpose(METHODS[o]) if o != 1 else im.copy()
    if mode is not None:
        im = im.convert(mode)
    im.thumbnail(bound, FILTERS[filt], reducing_gap=gap)
    return np.asarray(im)


def _host(t, layout="hwc"):
    a = t.cpu().numpy()
    a = a if layout == "hwc" else a.transpose(1, 2, 0)
    return a[..., 0] if a.shape[2] == 1 else a


@pytest.mark.parametrize("opt", ["q3", "q6", "q3n0"])
@pytest.mark.parametrize("layout,device", [("hwc", "cuda"), ("chw", "cpu"), ("chw", "cuda"), ("hwc", "cpu")])
def test_decode_thumbnail_is_pillow(ctx, corpus, tool_file, opt, layout, device):  # noqa: F811
    names = _names(corpus)
    datas = [corpus[n] for n in names]
    _, flags, niter = OPTS[opt]
    bounds = [BOUNDS[k % len(BOUNDS)] for k in range(len(names))]
    scales = set()
    for gap, filt in ((2.0, "bicubic"), (1.0, "lanczos"), (None, "bilinear"), (3.0, "box"), (1.5, "hamming")):
        got = ctx.decode_pixels(datas, flags | qs.JPEGQS_TRANSCODE, niter, layout, device, thumbnail=bounds, filter=filt,
                                reducing_gap=gap)
        for n, data, bound, rec in zip(names, datas, bounds, got):
            want = pillow_thumb(tool_file(data, opt), bound, filt, gap)
            assert np.array_equal(_host(rec[0], layout), want), (n, bound, gap, filt)
            w, h = Image.open(io.BytesIO(data)).size
            scales.add(cuda.thumbnail_geometry(w, h, bound, gap)[0])
    assert scales >= {1, 2, 4, 8}, scales


@pytest.mark.parametrize("opt", ["q3", "q3n0"])
def test_reencode_thumbnail_is_pillow_save(ctx, corpus, tool_file, opt):  # noqa: F811
    names = _names(corpus)
    datas = [corpus[n] for n in names]
    _, flags, niter = OPTS[opt]
    bounds = [BOUNDS[(k + 2) % len(BOUNDS)] for k in range(len(names))]
    for progressive, quality, sub in ((False, 85, "4:2:0"), (True, 75, "4:4:4")):
        got = ctx.reencode(datas, flags | qs.JPEGQS_TRANSCODE, niter, quality=quality, subsampling=sub,
                           thumbnail=bounds, progressive=progressive)
        for n, data, bound, rec in zip(names, datas, bounds, got):
            f = io.BytesIO()
            Image.fromarray(pillow_thumb(tool_file(data, opt), bound)).save(f, "JPEG", quality=quality, subsampling=sub,
                                                                             progressive=progressive)
            assert rec[0] == f.getvalue(), (n, bound, progressive)


@pytest.mark.parametrize("seq", [("exif", None), (6, None), (None, "RGB"), (None, "L"), ("exif", "RGB")])
def test_loaded_thumbnail_is_pillow(ctx, files, tool_file, seq):  # noqa: F811
    o, mode = seq
    names = sorted(n for n in files if n not in ("corpus_damaged", "corpus_stop")
                   and (mode is not None or Image.open(io.BytesIO(files[n])).mode in ("RGB", "L")))
    datas = [files[n] for n in names]
    _, flags, niter = OPTS["q6"]
    bounds = [BOUNDS[k % len(BOUNDS)] for k in range(len(names))]
    got = ctx.decode_pixels(datas, flags | qs.JPEGQS_TRANSCODE, niter, thumbnail=bounds, orientation=o, mode=mode)
    enc = ctx.reencode(datas, flags | qs.JPEGQS_TRANSCODE, niter, thumbnail=bounds, orientation=o, mode=mode)
    for n, data, bound, rec, erec in zip(names, datas, bounds, got, enc):
        want = pillow_thumb(tool_file(data, "q6"), bound, o=o, mode=mode)
        assert np.array_equal(_host(rec[0]), want), (n, bound, seq)
        f = io.BytesIO()
        Image.fromarray(want).save(f, "JPEG", quality=75, subsampling="4:2:0")    # reencode's defaults
        assert erec[0] == f.getvalue(), (n, bound, seq)


@pytest.mark.parametrize("bound,gap,o", [((256, 256), 2.0, None), ((16, 16), 1.0, None), ((16, 16), 1.0, 1),
                                         ((256, 256), 2.0, 6)])
def test_8k(ctx, corpus, tool_file, bound, gap, o):  # noqa: F811
    _, flags, niter = OPTS["q3"]
    (pix, *_), = ctx.decode_pixels([corpus["8k"]], flags | qs.JPEGQS_TRANSCODE, niter, thumbnail=bound,
                                   reducing_gap=gap, orientation=o)
    want = pillow_thumb(tool_file(corpus["8k"], "q3"), bound, gap=gap, o=o)
    assert np.array_equal(_host(pix), want)


def test_splits_and_order_change_nothing(ctx, corpus):  # noqa: F811
    names = _names(corpus) + ["8k"]
    datas = [corpus[n] for n in names]
    bounds = [BOUNDS[k % len(BOUNDS)] for k in range(len(names))]
    _, flags, niter = OPTS["q6"]
    full = [bytes(r[0].cpu().numpy()) for r in ctx.decode_pixels(datas, flags, niter, thumbnail=bounds)]
    perm = np.random.RandomState(3).permutation(len(names))
    for budget in (1, 24 << 20):
        got = ctx.decode_pixels([datas[k] for k in perm], flags, niter, thumbnail=[bounds[k] for k in perm],
                                max_device_bytes=budget, device="cpu")
        for k, rec in zip(perm, got):
            assert bytes(rec[0].numpy()) == full[k], (names[k], budget)
    enc_full = [r[0] for r in ctx.reencode(datas, flags, niter, thumbnail=bounds)]
    enc = ctx.reencode([datas[k] for k in perm], flags, niter, thumbnail=[bounds[k] for k in perm], max_device_bytes=1)
    assert [r[0] for r in enc] == [enc_full[k] for k in perm]


def test_a_refused_file_fails_alone(ctx, corpus):  # noqa: F811
    """the 8K picture loaded (orientation given) to 1 x 1 with gap 1.0 needs cells of 2^25 samples"""
    names = ["base420", "8k", "gray"]
    datas = [corpus[n] for n in names]
    _, flags, niter = OPTS["q6"]
    bounds = [(40, 40), (1, 1), (40, 40)]
    sizes = []
    for d, b in zip(datas, bounds):
        w, h = Image.open(io.BytesIO(d)).size
        c = 1 if Image.open(io.BytesIO(d)).mode == "L" else 3
        _, (tw, th) = cuda.thumbnail_geometry(w, h, b, 1.0, loaded=True)
        sizes.append(tw * th * c)
    n = len(datas)
    bufs = [(C.c_uint8 * (s + 1))(*([0xA5] * (s + 1))) for s in sizes]
    outs = (C.c_void_p * n)(*[C.addressof(b) for b in bufs])
    rc = (C.c_int * n)()
    res = (cuda._PixelsResult * n)()
    boxes = (cuda._ResizeBox * n)(*[cuda._ResizeBox(0, 0, 0, 0, *b) for b in bounds])
    ret = ctx.lib.jpegqs_cuda_pixels_batch_reduced(ctx.h, n, (C.c_char_p * n)(*datas), (C.c_size_t * n)(*map(len, datas)),
                                                   flags, niter, 0, 1, 3, boxes, (C.c_int32 * n)(1, 1, 1), 0, 0, outs, 0,
                                                   rc, res, 1, 1.0)
    assert ret == 0
    assert list(rc) == [0, -2, 0]
    assert "2^23" in ctx.lib.jpegqs_cuda_last_error(ctx.h).decode()
    assert bytes(bufs[1]) == b"\xa5" * (sizes[1] + 1)
    for k in (0, 2):
        (want, *_), = ctx.decode_pixels([datas[k]], flags, niter, thumbnail=bounds[k], reducing_gap=1.0, orientation=1,
                                        device="cpu")
        assert bytes(bufs[k])[:-1] == bytes(want.numpy()) and bufs[k][sizes[k]] == 0xA5


def test_reducing_gap_on_the_resize_path(ctx, corpus, tool_file):  # noqa: F811
    names = _names(corpus)
    datas = [corpus[n] for n in names]
    _, flags, niter = OPTS["q6"]
    rng = np.random.RandomState(8)
    crops, sizes = [], []
    for d in datas:
        w, h = Image.open(io.BytesIO(d)).size
        l, t = int(rng.randint(w // 3)), int(rng.randint(h // 3))
        crops.append((l, t, w - int(rng.randint(w // 4)), h - int(rng.randint(h // 4))))
        sizes.append((int(rng.randint(1, 50)), int(rng.randint(1, 50))))
    for gap, filt in ((2.0, "bicubic"), (1.0, "lanczos"), (3.0, "hamming")):
        got = ctx.decode_pixels(datas, flags | qs.JPEGQS_TRANSCODE, niter, size=sizes, crop=crops, filter=filt,
                                reducing_gap=gap)
        for n, data, crop, size, rec in zip(names, datas, crops, sizes, got):
            pic = Image.open(io.BytesIO(tool_file(data, "q6")))
            want = np.asarray(pic.crop(crop).resize(size, FILTERS[filt], reducing_gap=gap))
            assert np.array_equal(_host(rec[0]), want), (n, crop, size, gap)
    # reducing_gap None is the resize as before
    a = ctx.decode_pixels(datas, flags, niter, size=sizes, crop=crops, reducing_gap=None)
    b = ctx.decode_pixels(datas, flags, niter, size=sizes, crop=crops)
    assert all(torch.equal(x[0], y[0]) for x, y in zip(a, b))
