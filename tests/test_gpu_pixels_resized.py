"""Cropped and resized pixels on the GPU.  jpegqs_cuda_pixels_batch_resized (QsContext.decode_pixels with
size / crop / filter) gives, for every file, Pillow's Image.fromarray(P).crop(box).resize(size, filter)
of the picture P that libjpeg decodes from the coefficients the render reads: the file `jpegqs` writes
for the same flags and niter, or the input file where do_quantsmooth returns early; at d = 2, libjpeg's
scaled decode of it.  Every filter, both layouts, both output kinds, per-file crops and sizes in one
call, host-route, device-flagged and grey files at odd device offsets, an 8K file to 224 x 224 and a
small file upscaled 15x.  A bad crop changes no other file; forced splits and file order change no
byte; the results other than the pixels are pixels_batch_scaled's."""
import ctypes as C

import numpy as np
import pytest

import libjpeg_pixels as lp
from test_gpu_pixels_batch import _shape, corpus, ctx  # noqa: F401  (module fixtures)
from test_gpu_pixels_scaled import OPTS, _c_scaled, reference  # noqa: F401  (module fixture)

import jpegqs_b200 as qs
from jpegqs_b200 import cuda

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(lp.JPEG_SO is None, reason="no libjpeg inside Pillow")]

torch = pytest.importorskip("torch")
Image = pytest.importorskip("PIL.Image")

FILTERS = {"lanczos": 1, "bilinear": 2, "bicubic": 3, "box": 4, "hamming": 5}


def _picture(data, d):
    w, h, _ = _shape(data)
    return -(-w // d), -(-h // d)


def _boxes(names, datas, d, seed):
    """per file (left, top, right, bottom, width, height): the whole picture or a random crop, to a
    random size from 1 x 1 to about twice the crop; tinyprog is upscaled about 15x"""
    rng = np.random.RandomState(seed)
    out = []
    for n, data in zip(names, datas):
        pw, ph = _picture(data, d)
        if n == "tinyprog":
            out.append((0, 0, 0, 0, pw * 15, ph * 15 + 1))
            continue
        if rng.rand() < 0.3:
            l = t = r = b = 0
            cw, ch = pw, ph
        else:
            l, t = rng.randint(pw), rng.randint(ph)
            r, b = rng.randint(l + 1, pw + 1), rng.randint(t + 1, ph + 1)
            cw, ch = r - l, b - t
        out.append((l, t, r, b, int(rng.randint(1, 2 * cw + 2)), int(rng.randint(1, 2 * ch + 2))))
    return out


def _c_resized(ctx, datas, flags, niter, layout, d, filt, boxes, on_device, budget=0):  # noqa: F811
    """jpegqs_cuda_pixels_batch_resized with outputs of width * height * channels bytes at odd byte offsets
    of one device tensor (a guard byte after each) or in host buffers.  Returns
    [(rc, bytes or None, (channels, host_decoded, warnings, smoothed, stop, upsampled, reason))]."""
    n = len(datas)
    sizes = [b[4] * b[5] * (1 if _shape(x)[2] == 1 else 3) for x, b in zip(datas, boxes)]
    offs, o = [], 1
    for s in sizes:
        offs.append(o)
        o += s + 1 + (o & 2)
    if on_device:
        flat = torch.full((o + 1,), 0xA5, dtype=torch.uint8, device=f"cuda:{ctx.device}")
        outs = (C.c_void_p * n)(*[flat.data_ptr() + x for x in offs])
    else:
        bufs = [(C.c_uint8 * (s + 1))(*([0xA5] * (s + 1))) for s in sizes]
        outs = (C.c_void_p * n)(*[C.addressof(b) for b in bufs])
    torch.cuda.synchronize(ctx.device)
    rc = (C.c_int * n)()
    res = (cuda._PixelsResult * n)()
    cb = (cuda._ResizeBox * n)(*[cuda._ResizeBox(*b) for b in boxes])
    ret = ctx.lib.jpegqs_cuda_pixels_batch_resized(ctx.h, n, (C.c_char_p * n)(*datas),
                                                   (C.c_size_t * n)(*[len(x) for x in datas]), flags | qs.JPEGQS_TRANSCODE,
                                                   niter, layout, d, FILTERS[filt], cb, on_device, outs, budget, rc, res)
    assert ret == 0, ctx.lib.jpegqs_cuda_last_error(ctx.h).decode()
    if on_device:
        host = flat.cpu().numpy().tobytes()
        got = [host[x:x + s] for x, s in zip(offs, sizes)]
        assert all(host[x + s] == 0xA5 for x, s in zip(offs, sizes))
    else:
        got = [bytes(b)[:s] for b, s in zip(bufs, sizes)]
        assert all(b[s] == 0xA5 for b, s in zip(bufs, sizes))
    for i in range(n):
        if rc[i]:
            assert got[i] == b"\xa5" * sizes[i], i             # untouched
    return [(rc[i], got[i] if rc[i] == 0 else None,
             (res[i].channels, res[i].host_decoded, res[i].warnings, res[i].smoothed, res[i].stop, res[i].upsampled,
              (res[i].reason or b"").decode())) for i in range(n)]


def _hwc(body, box, channels, layout):
    a = np.frombuffer(body, dtype=np.uint8)
    w, h = box[4], box[5]
    return a.reshape(h, w, channels) if layout == 0 else a.reshape(channels, h, w).transpose(1, 2, 0)


def _pillow(pixels, box, filt):
    """Pillow's crop().resize() of a libjpeg picture [H, W, C] -> [h, w, C]"""
    im = Image.fromarray(pixels[..., 0] if pixels.shape[2] == 1 else pixels)
    if any(box[:4]):
        im = im.crop(box[:4])
    out = np.asarray(im.resize(box[4:6], getattr(Image.Resampling, filt.upper())))
    return out[..., None] if out.ndim == 2 else out


def _names(corpus):  # noqa: F811
    return sorted(n for n in corpus if n not in ("cmyk", "8k"))


@pytest.mark.parametrize("on_device", [1, 0])
@pytest.mark.parametrize("layout", [0, 1])
@pytest.mark.parametrize("opt", sorted(OPTS))
def test_pixels_are_pillows_resize_of_libjpegs_decode(ctx, corpus, reference, opt, layout, on_device):  # noqa: F811
    names = _names(corpus)
    datas = [corpus[n] for n in names]
    _, flags, niter = OPTS[opt]
    for d in (1, 2):
        for k, filt in enumerate(FILTERS):
            boxes = _boxes(names, datas, d, seed=100 * d + 10 * k + layout + 2 * on_device)
            got = _c_resized(ctx, datas, flags, niter, layout, d, filt, boxes, on_device)
            for n, b, (rc, pix, res) in zip(names, boxes, got):
                assert rc == 0, n
                want = _pillow(reference(n, opt, d), b, filt)
                assert np.array_equal(_hwc(pix, b, want.shape[2], layout), want), (n, opt, layout, on_device, d, filt, b)
            # everything but the pixels is the scaled call's
            if k == 0:
                scaled = _c_scaled(ctx, datas, flags, niter, layout, d, on_device)
                assert [(g[0], g[2]) for g in got] == [(s[0], s[2]) for s in scaled]


@pytest.mark.parametrize("layout", [0, 1])
def test_8k_to_224_lanczos(ctx, corpus, reference, layout):  # noqa: F811
    data = corpus["8k"]
    _, flags, niter = OPTS["q3"]
    for d, box in ((1, (1680, 0, 6000, 4320, 224, 224)), (2, (0, 0, 0, 0, 224, 224))):
        (rc, pix, _), = _c_resized(ctx, [data], flags, niter, layout, d, "lanczos", [box], 1)
        assert rc == 0
        assert np.array_equal(_hwc(pix, box, 3, layout), _pillow(reference("8k", "q3", d), box, "lanczos")), d


@pytest.mark.parametrize("on_device", [1, 0])
def test_bad_crop_changes_no_other_file(ctx, corpus, on_device):  # noqa: F811
    names = ["base420", "gray", "prog420", "garbled", "base444"]
    datas = [corpus[n] for n in names]
    _, flags, niter = OPTS["q6"]
    boxes = _boxes(names, datas, 1, seed=5)
    good = _c_resized(ctx, datas, flags, niter, 0, 1, "bicubic", boxes, on_device)
    pw, ph = _picture(datas[2], 1)
    for bad in ((0, 0, pw + 1, ph, 8, 8), (3, 3, 3, 9, 8, 8), (0, ph, pw, ph + 1, 8, 8)):
        got = _c_resized(ctx, datas, flags, niter, 0, 1, "bicubic", boxes[:2] + [bad] + boxes[3:], on_device)
        assert got[2][0] == -2 and got[2][2] == (0, 0, 0, 0, 0, 0, "")
        assert "file 2" in ctx.lib.jpegqs_cuda_last_error(ctx.h).decode()
        assert got[:2] + got[3:] == good[:2] + good[3:]


@pytest.mark.parametrize("d", [1, 2])
def test_splits_order_and_output_kinds_change_nothing(ctx, corpus, d):  # noqa: F811
    names = _names(corpus)
    datas = [corpus[n] for n in names]
    _, flags, niter = OPTS["q6"]
    boxes = _boxes(names, datas, d, seed=77 + d)
    whole = _c_resized(ctx, datas, flags, niter, 1, d, "hamming", boxes, 1)
    for budget, on_device in ((1, 1), (3 << 20, 0), (0, 0)):
        assert _c_resized(ctx, datas, flags, niter, 1, d, "hamming", boxes, on_device, budget) == whole, (budget, on_device)
    perm = list(np.random.RandomState(d).permutation(len(names)))
    got = _c_resized(ctx, [datas[i] for i in perm], flags, niter, 1, d, "hamming", [boxes[i] for i in perm], 1)
    for i, g in zip(perm, got):
        assert g == whole[i], names[i]


@pytest.mark.parametrize("layout", [0, 1])
def test_grey_files_at_odd_offsets(ctx, corpus, reference, layout):  # noqa: F811
    names = ["tinyprog", "base444", "gray", "tinyprog", "base420", "gray"]
    datas = [corpus[n] for n in names]
    _, flags, niter = OPTS["q6"]
    boxes = _boxes(names, datas, 1, seed=3)
    got = _c_resized(ctx, datas, flags, niter, layout, 1, "bilinear", boxes, 1)
    for n, b, (rc, pix, res) in zip(names, boxes, got):
        want = _pillow(reference(n, "q6", 1), b, "bilinear")
        assert rc == 0 and np.array_equal(_hwc(pix, b, want.shape[2], layout), want), n


def test_python_call(ctx, corpus, reference):  # noqa: F811
    _, flags, niter = OPTS["q6"]
    names = ["base420", "gray", "prog420", "garbled"]
    datas = [corpus[n] for n in names]
    flags |= qs.JPEGQS_TRANSCODE
    for d in (1, 2):
        full = ctx.decode_pixels(datas, flags, niter, scale_denom=d)
        crops = [None, (1, 2, 30, 20), (10, 0, 50, 40), None]
        for layout in ("hwc", "chw"):
            dev = ctx.decode_pixels(datas, flags, niter, layout=layout, scale_denom=d, size=(40, 30), crop=crops,
                                    filter="lanczos")
            cpu = qs.decode_pixels(datas, flags, niter, layout=layout, device="cpu", gpu=0, scale_denom=d, size=(40, 30),
                                   crop=crops, filter=Image.Resampling.LANCZOS)
            for n, a, b, f, c in zip(names, dev, cpu, full, crops):
                box = (c or (0, 0, 0, 0)) + (40, 30)
                want = _pillow(reference(n, "q6", d), box, "lanczos")
                got = a[0].cpu().numpy()
                assert np.array_equal(got if layout == "hwc" else got.transpose(1, 2, 0), want), (n, d, layout)
                assert torch.equal(a[0].cpu(), b[0]) and a[1:] == b[1:] == f[1:], n
        # per-file sizes, the default filter (bicubic), and a crop without size: the crop as it is
        sized = ctx.decode_pixels(datas, flags, niter, scale_denom=d, size=[(7, 9), (64, 3), (1, 1), (90, 70)])
        for n, a, s in zip(names, sized, [(7, 9), (64, 3), (1, 1), (90, 70)]):
            assert np.array_equal(a[0].cpu().numpy(), _pillow(reference(n, "q6", d), (0, 0, 0, 0) + s, "bicubic")), n
        cropped = ctx.decode_pixels(datas, flags, niter, scale_denom=d, crop=crops)
        for a, f, c in zip(cropped, full, crops):
            want = f[0] if c is None else f[0][c[1]:c[3], c[0]:c[2]]
            assert torch.equal(a[0], want)
    with pytest.raises(ValueError, match="file 3: crop"):
        ctx.decode_pixels(datas, flags, niter, crop=[None, None, None, (0, 0, 10000, 5)])
