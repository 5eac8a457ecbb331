"""Blur and sharpen on the GPU.  decode_pixels(image_filter=) and reencode(image_filter=) give, for file i,
Pillow's
    im = Image.open(F); [exif_transpose / transpose] [convert(mode)] [crop().resize() | thumbnail()]
    im = im.filter(F1).filter(F2)...; [im.save(...)]
with F the file the jpegqs tool writes for the same options.  Both layouts and output kinds, sequential
and progressive saves, size / crop, scale_denom, thumbnail, orientation and mode (CMYK included), the 8K
file at full size with a large Gaussian radius, a file wider than the fused row kernel holds, forced splits
with shuffled order, a refused file failing alone, and image_filter None and [] against the call without
it."""
import ctypes as C
import io

import numpy as np
import pytest
from PIL import ImageFilter as F, ImageOps

from test_gpu_pixels_batch import corpus, ctx  # noqa: F401  (module fixtures)
from test_gpu_pixel_modes import METHODS, OPTS, files, tool_file  # noqa: F401  (module fixtures)

import jpegqs_b200 as qs
from jpegqs_b200 import cuda

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
Image = pytest.importorskip("PIL.Image")

NAMES = ["base420", "base444", "prog420", "gray", "opt422", "prog444", "rst", "progrst", "tinyprog", "dense444", "coarse420"]
CHAINS = [F.UnsharpMask(2, 150, 3), F.GaussianBlur(3.3), F.BoxBlur((4, 0.5)), [F.GaussianBlur((0, 2)), F.UnsharpMask],
          [F.BoxBlur(1), F.UnsharpMask(1.5, 300, 0), F.GaussianBlur(0)]]


def _names(corpus):  # noqa: F811
    return [n for n in NAMES if n in corpus]


def _chain(c):
    return c if isinstance(c, list) else [c]


def filtered(pixels, chain):
    im = Image.fromarray(pixels)
    for f in _chain(chain):
        im = im.filter(f)
    return np.asarray(im)


def pillow(data, chain, o=None, mode=None, size=None, crop=None, thumb=None):
    im = Image.open(io.BytesIO(data))
    if o == "exif":
        im = ImageOps.exif_transpose(im)
    elif o is not None:
        im = im.transpose(METHODS[o]) if o != 1 else im.copy()
    if mode is not None:
        im = im.convert(mode)
    if crop is not None:
        im = im.crop(crop)
    if size is not None:
        im = im.resize(size, Image.Resampling.BICUBIC)
    if thumb is not None:
        im.thumbnail(thumb)
    return filtered(np.asarray(im), chain)


def _host(t, layout="hwc"):
    a = t.cpu().numpy()
    a = a if layout == "hwc" else a.transpose(1, 2, 0)
    return a[..., 0] if a.shape[2] == 1 else a


@pytest.mark.parametrize("chain", range(len(CHAINS)))
@pytest.mark.parametrize("layout,device", [("hwc", "cuda"), ("chw", "cpu"), ("chw", "cuda"), ("hwc", "cpu")])
def test_decode_filter_is_pillow(ctx, corpus, tool_file, chain, layout, device):  # noqa: F811
    names = _names(corpus)
    datas = [corpus[n] for n in names]
    _, flags, niter = OPTS["q3"]
    got = ctx.decode_pixels(datas, flags | qs.JPEGQS_TRANSCODE, niter, layout, device, image_filter=CHAINS[chain])
    for n, data, rec in zip(names, datas, got):
        assert np.array_equal(_host(rec[0], layout), pillow(tool_file(data, "q3"), CHAINS[chain])), n


@pytest.mark.parametrize("opt", ["q3", "q3n0"])
def test_reencode_filter_is_pillow_save(ctx, corpus, tool_file, opt):  # noqa: F811
    names = _names(corpus)
    datas = [corpus[n] for n in names]
    _, flags, niter = OPTS[opt]
    for progressive, quality, sub, chain in ((False, 85, "4:2:0", CHAINS[0]), (True, 75, "4:4:4", CHAINS[3])):
        got = ctx.reencode(datas, flags | qs.JPEGQS_TRANSCODE, niter, quality=quality, subsampling=sub,
                           progressive=progressive, image_filter=chain)
        for n, data, rec in zip(names, datas, got):
            f = io.BytesIO()
            Image.fromarray(pillow(tool_file(data, opt), chain)).save(f, "JPEG", quality=quality, subsampling=sub,
                                                                      progressive=progressive)
            assert rec[0] == f.getvalue(), (n, progressive)


def test_after_resize_scale_and_thumbnail(ctx, corpus, tool_file):  # noqa: F811
    names = _names(corpus)
    datas = [corpus[n] for n in names]
    _, flags, niter = OPTS["q6"]
    fl = flags | qs.JPEGQS_TRANSCODE
    chain = [F.UnsharpMask(2, 150, 3)]
    rng = np.random.RandomState(4)
    crops, sizes = [], []
    for d in datas:
        w, h = Image.open(io.BytesIO(d)).size
        crops.append((int(rng.randint(w // 3)), int(rng.randint(h // 3)), w - int(rng.randint(w // 4)),
                      h - int(rng.randint(h // 4))))
        sizes.append((int(rng.randint(1, 90)), int(rng.randint(1, 90))))
    got = ctx.decode_pixels(datas, fl, niter, size=sizes, crop=crops, image_filter=chain)
    enc = ctx.reencode(datas, fl, niter, size=sizes, crop=crops, image_filter=chain)
    for n, data, crop, size, rec, erec in zip(names, datas, crops, sizes, got, enc):
        want = pillow(tool_file(data, "q6"), chain, crop=crop, size=size)
        assert np.array_equal(_host(rec[0]), want), (n, crop, size)
        f = io.BytesIO()
        Image.fromarray(want).save(f, "JPEG", quality=75, subsampling="4:2:0")
        assert erec[0] == f.getvalue(), n
    for scale in (2, 8):
        # the scaled decode itself is checked against libjpeg elsewhere; the filter applies to what it gives
        base = ctx.decode_pixels(datas, fl, niter, scale_denom=scale)
        got = ctx.decode_pixels(datas, fl, niter, "chw", scale_denom=scale, image_filter=F.GaussianBlur(1.5))
        for n, b, rec in zip(names, base, got):
            assert np.array_equal(_host(rec[0], "chw"), filtered(_host(b[0]), F.GaussianBlur(1.5))), (n, scale)
    got = ctx.decode_pixels(datas, fl, niter, thumbnail=(256, 256), image_filter=chain)
    enc = ctx.reencode(datas, fl, niter, thumbnail=(256, 256), image_filter=chain, progressive=True)
    for n, data, rec, erec in zip(names, datas, got, enc):
        want = pillow(tool_file(data, "q6"), chain, thumb=(256, 256))
        assert np.array_equal(_host(rec[0]), want), n
        f = io.BytesIO()
        Image.fromarray(want).save(f, "JPEG", quality=75, subsampling="4:2:0", progressive=True)
        assert erec[0] == f.getvalue(), n


@pytest.mark.parametrize("seq", [("exif", None), (6, None), (None, "RGB"), (None, "L"), ("exif", "RGB")])
def test_orientation_and_mode(ctx, files, tool_file, seq):  # noqa: F811
    o, mode = seq
    names = sorted(n for n in files if n not in ("corpus_damaged", "corpus_stop")
                   and (mode is not None or Image.open(io.BytesIO(files[n])).mode in ("RGB", "L")))
    datas = [files[n] for n in names]
    _, flags, niter = OPTS["q6"]
    chain = [F.BoxBlur(2), F.UnsharpMask(1, 200, 2)]
    got = ctx.decode_pixels(datas, flags | qs.JPEGQS_TRANSCODE, niter, "chw", orientation=o, mode=mode, image_filter=chain)
    enc = ctx.reencode(datas, flags | qs.JPEGQS_TRANSCODE, niter, orientation=o, mode=mode, image_filter=chain)
    for n, data, rec, erec in zip(names, datas, got, enc):
        want = pillow(tool_file(data, "q6"), chain, o=o, mode=mode)
        assert np.array_equal(_host(rec[0], "chw"), want), (n, seq)
        f = io.BytesIO()
        Image.fromarray(want).save(f, "JPEG", quality=75, subsampling="4:2:0")
        assert erec[0] == f.getvalue(), (n, seq)


@pytest.mark.parametrize("chain", [F.GaussianBlur(40), [F.BoxBlur((25, 3)), F.UnsharpMask(3, 120, 2)]])
def test_8k_full_size(ctx, corpus, tool_file, chain):  # noqa: F811
    """the 8K file's rows (23040 bytes) are wider than the fused row kernel holds"""
    _, flags, niter = OPTS["q3"]
    for layout in ("hwc", "chw"):
        (pix, *_), = ctx.decode_pixels([corpus["8k"]], flags | qs.JPEGQS_TRANSCODE, niter, layout, image_filter=chain)
        assert np.array_equal(_host(pix, layout), pillow(tool_file(corpus["8k"], "q3"), chain)), layout


def test_wide_file_with_narrow_ones(ctx, corpus, tool_file):  # noqa: F811
    """a synthesized 6000 x 40 RGB and a 16500 x 24 grey JPEG (rows past 16384 bytes) with two narrow files in
    one call: the fused and the per-pass row launches together"""
    rng = np.random.RandomState(12)
    wide = []
    for w, h, mode in ((6000, 40, "RGB"), (16500, 24, "L")):
        a = rng.randint(0, 256, (h, w // 50 + 1, 3)).astype(np.uint8)
        im = Image.fromarray(a).resize((w, h), Image.Resampling.BILINEAR).convert(mode)
        f = io.BytesIO()
        im.save(f, "JPEG", quality=90)
        wide.append(f.getvalue())
    datas = [wide[0], corpus["base420"], wide[1], corpus["gray"]]
    _, flags, niter = OPTS["q3"]
    for chain in (F.GaussianBlur(20), [F.BoxBlur((0, 3)), F.UnsharpMask(2, 150, 3)], F.BoxBlur((9.5, 0))):
        got = ctx.decode_pixels(datas, flags | qs.JPEGQS_TRANSCODE, niter, image_filter=chain)
        for k, (data, rec) in enumerate(zip(datas, got)):
            assert np.array_equal(_host(rec[0]), pillow(tool_file(data, "q3"), chain)), (k, chain)


def test_splits_and_order_change_nothing(ctx, corpus):  # noqa: F811
    names = _names(corpus) + ["8k"]
    datas = [corpus[n] for n in names]
    _, flags, niter = OPTS["q6"]
    chain = [F.GaussianBlur(2), F.UnsharpMask(2, 150, 3)]
    full = [bytes(r[0].cpu().numpy()) for r in ctx.decode_pixels(datas, flags, niter, image_filter=chain)]
    perm = np.random.RandomState(3).permutation(len(names))
    for budget in (1, 48 << 20):
        got = ctx.decode_pixels([datas[k] for k in perm], flags, niter, max_device_bytes=budget, device="cpu",
                                image_filter=chain)
        for k, rec in zip(perm, got):
            assert bytes(rec[0].numpy()) == full[k], (names[k], budget)
    enc_full = [r[0] for r in ctx.reencode(datas, flags, niter, thumbnail=(200, 200), image_filter=chain)]
    enc = ctx.reencode([datas[k] for k in perm], flags, niter, thumbnail=(200, 200), image_filter=chain, max_device_bytes=1)
    assert [r[0] for r in enc] == [enc_full[k] for k in perm]


def test_a_refused_file_fails_alone(ctx, corpus):  # noqa: F811
    """the 8K picture loaded (orientation given) to a 1 x 1 thumbnail with gap 1.0 needs cells of 2^25 samples"""
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
    filt = (cuda._ImageFilter * 1)(cuda._ImageFilter(3, 2.0, 2.0, 150, 3))
    ret = ctx.lib.jpegqs_cuda_pixels_batch_filtered(ctx.h, n, (C.c_char_p * n)(*datas), (C.c_size_t * n)(*map(len, datas)),
                                                    flags, niter, 0, 1, 3, boxes, (C.c_int32 * n)(1, 1, 1), 0, 0, outs, 0,
                                                    rc, res, 1, 1.0, filt, 1)
    assert ret == 0
    assert list(rc) == [0, -2, 0]
    assert bytes(bufs[1]) == b"\xa5" * (sizes[1] + 1)
    for k in (0, 2):
        (want, *_), = ctx.decode_pixels([datas[k]], flags, niter, thumbnail=bounds[k], reducing_gap=1.0, orientation=1,
                                        device="cpu", image_filter=F.UnsharpMask(2, 150, 3))
        assert bytes(bufs[k])[:-1] == bytes(want.numpy()) and bufs[k][sizes[k]] == 0xA5


def test_none_and_empty_are_the_call_without(ctx, corpus):  # noqa: F811
    names = _names(corpus)
    datas = [corpus[n] for n in names]
    _, flags, niter = OPTS["q6"]
    for kw in ({}, {"size": (64, 48)}, {"thumbnail": (100, 100)}, {"orientation": "exif", "mode": "RGB"}):
        base = ctx.decode_pixels(datas, flags, niter, "chw", **kw)
        for f in (None, [], ()):
            got = ctx.decode_pixels(datas, flags, niter, "chw", image_filter=f, **kw)
            assert all(torch.equal(x[0], y[0]) and x[1:] == y[1:] for x, y in zip(got, base)), (kw, f)
        enc = ctx.reencode(datas, flags, niter, **kw)
        assert [r[0] for r in ctx.reencode(datas, flags, niter, image_filter=[], **kw)] == [r[0] for r in enc]


def test_bad_filters_are_refused_before_anything_runs(ctx, corpus):  # noqa: F811
    datas = [corpus["base420"]]
    for f, match in ((F.SHARPEN, "SHARPEN"), (F.MedianFilter(3), "MedianFilter"), (F.UnsharpMask(2, 1.5, 3), "percent"),
                     (F.GaussianBlur(1e5), "radius")):
        with pytest.raises(ValueError, match=match):
            ctx.decode_pixels(datas, 0, 0, image_filter=f)
        with pytest.raises(ValueError, match=match):
            ctx.reencode(datas, 0, 0, image_filter=[F.BoxBlur(1), f])
