"""EXIF orientation on the GPU.  jpegqs_cuda_pixels_batch_oriented (QsContext.decode_pixels with
orientation) gives, for every file and orientation o, Pillow's Image.transpose of the picture the
unoriented call gives (which the earlier tests pin to libjpeg), then Pillow's crop and resize of that;
reencode(orientation="exif") is Pillow's save of it.  Orientations 1..8 in both layouts and output kinds at
d = 1, 2 and 8 over the pixels-batch corpus, sizes around the 128 x 64 tile, orientation 0 on files with
a spliced EXIF APP1, NULL and all-ones against the existing calls, and render_oriented_async eagerly and
replayed from a CUDA graph."""
import ctypes as C
import io
import struct

import numpy as np
import pytest

from test_gpu_pixels_batch import _shape, corpus, ctx  # noqa: F401  (module fixtures)
from test_gpu_pixels_scaled import OPTS, _c_scaled, _images, _run_result

import jpegqs_b200 as qs
from jpegqs_b200 import cuda

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
Image = pytest.importorskip("PIL.Image")

T = Image.Transpose
METHODS = {2: T.FLIP_LEFT_RIGHT, 3: T.ROTATE_180, 4: T.FLIP_TOP_BOTTOM, 5: T.TRANSPOSE, 6: T.ROTATE_270,
           7: T.TRANSVERSE, 8: T.ROTATE_90}
FILTERS = {"lanczos": 1, "bilinear": 2, "bicubic": 3, "box": 4, "hamming": 5}


def turn(a, o):
    """Pillow's Image.transpose for orientation o of a picture [H, W, C]"""
    if o == 1:
        return a
    t = np.asarray(Image.fromarray(a[..., 0] if a.shape[2] == 1 else a).transpose(METHODS[o]))
    return t[..., None] if t.ndim == 2 else t


def exif_app1(o: int) -> bytes:
    """an APP1 segment whose IFD0 holds Orientation (SHORT) o"""
    tiff = b"II*\0" + struct.pack("<LH", 8, 1) + struct.pack("<HHLHH", 0x0112, 3, 1, o, 0) + b"\0\0\0\0"
    payload = b"Exif\0\0" + tiff
    return b"\xff\xe1" + struct.pack(">H", len(payload) + 2) + payload


def tagged(data: bytes, o: int) -> bytes:
    return data[:2] + exif_app1(o) + data[2:]


def _dims(data, d, o):
    w, h, c = _shape(data)
    w, h = -(-w // d), -(-h // d)
    return (h, w, 1 if c == 1 else 3) if o >= 5 else (w, h, 1 if c == 1 else 3)


def _c_oriented(ctx, datas, flags, niter, layout, d, orient, on_device, boxes=None, filt="bicubic", budget=0):  # noqa: F811
    """jpegqs_cuda_pixels_batch_oriented with outputs at odd byte offsets of one device tensor (a guard byte
    after each) or in host buffers.  Returns [(rc, pixels [H', W', C] or None, results)]; a failing file's
    output is untouched."""
    n = len(datas)
    os_ = orient if orient is not None else [1] * n
    if boxes is None:
        dims = [_dims(x, d, max(o, 1) if o else qs.exif_orientation(x)) for x, o in zip(datas, os_)]
    else:
        dims = [(b[4], b[5], 1 if _shape(x)[2] == 1 else 3) for x, b in zip(datas, boxes)]
    sizes = [w * h * c for w, h, c in dims]
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
    cb = (cuda._ResizeBox * n)(*[cuda._ResizeBox(*b) for b in boxes]) if boxes is not None else None
    co = (C.c_int32 * n)(*orient) if orient is not None else None
    ret = ctx.lib.jpegqs_cuda_pixels_batch_oriented(ctx.h, n, (C.c_char_p * n)(*datas),
                                                    (C.c_size_t * n)(*[len(x) for x in datas]), flags | qs.JPEGQS_TRANSCODE,
                                                    niter, layout, d, FILTERS[filt], cb, co, on_device, outs, budget, rc,
                                                    res)
    assert ret == 0, ctx.lib.jpegqs_cuda_last_error(ctx.h).decode()
    if on_device:
        host = flat.cpu().numpy().tobytes()
        got = [host[x:x + s] for x, s in zip(offs, sizes)]
        assert all(host[x + s] == 0xA5 for x, s in zip(offs, sizes))
    else:
        got = [bytes(b)[:s] for b, s in zip(bufs, sizes)]
        assert all(b[s] == 0xA5 for b, s in zip(bufs, sizes))
    out = []
    for i in range(n):
        if rc[i]:
            assert got[i] == b"\xa5" * sizes[i], i             # untouched
        w, h, c = dims[i]
        a = np.frombuffer(got[i], dtype=np.uint8)
        a = a.reshape(h, w, c) if layout == 0 else a.reshape(c, h, w).transpose(1, 2, 0)
        out.append((rc[i], a if rc[i] == 0 else None,
                    (res[i].channels, res[i].host_decoded, res[i].warnings, res[i].smoothed, res[i].stop,
                     res[i].upsampled, (res[i].reason or b"").decode())))
    return out


def _unoriented(ctx, datas, flags, niter, d):  # noqa: F811
    """the existing call's pictures [H, W, C] (device outputs, HWC) and results"""
    got = _c_scaled(ctx, datas, flags, niter, 0, d, 1)
    out = []
    for x, (rc, body, res) in zip(datas, got):
        w, h, c = _dims(x, d, 1)
        out.append((rc, np.frombuffer(body, dtype=np.uint8).reshape(h, w, c) if rc == 0 else None, res))
    return out


def _names(corpus):  # noqa: F811
    return sorted(n for n in corpus if n != "8k")


@pytest.mark.parametrize("on_device", [1, 0])
@pytest.mark.parametrize("layout", [0, 1])
@pytest.mark.parametrize("opt", sorted(OPTS))
def test_every_orientation_is_pillows_transpose(ctx, corpus, opt, layout, on_device):  # noqa: F811
    names = _names(corpus)
    datas = [corpus[n] for n in names]
    _, flags, niter = OPTS[opt]
    for d in (1, 2, 8):
        ref = _unoriented(ctx, datas, flags, niter, d)
        for shift in range(8):
            orient = [(k + shift) % 8 + 1 for k in range(len(names))]
            got = _c_oriented(ctx, datas, flags, niter, layout, d, orient, on_device)
            for n, o, (rc, pix, res), (rrc, rpix, rres) in zip(names, orient, got, ref):
                if n == "cmyk":
                    assert rc == -3 and rrc == -3
                    continue
                assert rc == 0 and res == rres, (n, o)
                assert np.array_equal(pix, turn(rpix, o)), (n, opt, layout, on_device, d, o)


@pytest.mark.parametrize("d", [1, 2])
def test_null_and_all_ones_are_the_existing_call(ctx, corpus, d):  # noqa: F811
    names = _names(corpus)
    datas = [corpus[n] for n in names]
    _, flags, niter = OPTS["q6"]
    for layout, on_device in ((0, 1), (1, 0)):
        want = _c_scaled(ctx, datas, flags, niter, layout, d, on_device)
        for orient in (None, [1] * len(datas)):
            got = _c_oriented(ctx, datas, flags, niter, layout, d, orient, on_device)
            for (rc, pix, res), (wrc, wbody, wres) in zip(got, want):
                assert rc == wrc and res == wres
                if rc == 0:
                    body = pix.tobytes() if layout == 0 else pix.transpose(2, 0, 1).tobytes()
                    assert body == wbody


def test_8k_file(ctx, corpus):  # noqa: F811
    _, flags, niter = OPTS["q3"]
    data = [corpus["8k"]]
    for d, layout, on_device, orients in ((1, 0, 1, range(1, 9)), (2, 1, 0, (3, 6, 7))):
        ref = _unoriented(ctx, data, flags, niter, d)[0][1]
        for o in orients:
            (rc, pix, _), = _c_oriented(ctx, data, flags, niter, layout, d, [o], on_device)
            assert rc == 0 and np.array_equal(pix, turn(ref, o)), (d, o)


EDGES = (1, 7, 64, 65, 127, 128, 129, 200)


@pytest.fixture(scope="module")
def edge_files():
    """pictures of every width and height in EDGES, colour 4:2:0 / 4:2:2 / 4:4:4 and grey"""
    out = []
    rng = np.random.RandomState(3)
    for i, w in enumerate(EDGES):
        for j, h in enumerate(EDGES):
            k = i * len(EDGES) + j
            grey = k % 5 == 4
            ramp = (np.arange(w)[None, :] * 3 + np.arange(h)[:, None] * 2) % 170
            a = ramp[..., None] + rng.randint(0, 86, (h, w, 1 if grey else 3))
            a = a[..., 0] if grey else a
            a = a.astype(np.uint8)
            b = io.BytesIO()
            Image.fromarray(a).save(b, "JPEG", quality=60 + k % 30, subsampling=k % 3)
            out.append(b.getvalue())
    return out


@pytest.mark.parametrize("layout,on_device", [(0, 1), (1, 0), (0, 0), (1, 1)])
def test_sizes_around_the_tile(ctx, edge_files, layout, on_device):  # noqa: F811
    _, flags, niter = OPTS["q6"]
    for d in (1, 2):
        ref = _unoriented(ctx, edge_files, flags, niter, d)
        for shift in range(4):
            orient = [5 + (k + shift) % 4 for k in range(len(edge_files))]
            got = _c_oriented(ctx, edge_files, flags, niter, layout, d, orient, on_device)
            for k, (o, (rc, pix, _), (_, rpix, _)) in enumerate(zip(orient, got, ref)):
                assert rc == 0 and np.array_equal(pix, turn(rpix, o)), (k, d, o, rpix.shape)


def test_mixed_orientations_and_the_files_own(ctx, corpus):  # noqa: F811
    names = _names(corpus)
    _, flags, niter = OPTS["q6"]
    tags = [k % 8 + 1 for k in range(len(names))]
    plain = [corpus[n] for n in names]
    spliced = [tagged(x, o) for x, o in zip(plain, tags)]
    assert [qs.exif_orientation(x) for x in spliced] == tags
    ref = _unoriented(ctx, plain, flags, niter, 1)
    # 0 everywhere, then 0 for every other file and explicit values (unrelated to the tag) for the rest
    for orient in ([0] * len(names), [0 if k % 2 else (k * 3) % 8 + 1 for k in range(len(names))]):
        want = [t if o == 0 else o for o, t in zip(orient, tags)]
        for layout, on_device in ((0, 1), (1, 0)):
            got = _c_oriented(ctx, spliced, flags, niter, layout, 1, orient, on_device)
            for n, o, (rc, pix, res), (rrc, rpix, rres) in zip(names, want, got, ref):
                assert rc == rrc and res == rres, n              # same route, same coefficients
                if rc == 0:
                    assert np.array_equal(pix, turn(rpix, o)), (n, o, layout)


def _oriented_boxes(datas, orient, d, seed):
    """per file a random crop of the ORIENTED picture (or none) and a size up to about twice the crop"""
    rng = np.random.RandomState(seed)
    out = []
    for x, o in zip(datas, orient):
        pw, ph, _ = _dims(x, d, o)
        if rng.rand() < 0.3:
            l = t = r = b = 0
            cw, ch = pw, ph
        else:
            l, t = rng.randint(pw), rng.randint(ph)
            r, b = rng.randint(l + 1, pw + 1), rng.randint(t + 1, ph + 1)
            cw, ch = r - l, b - t
        out.append((l, t, r, b, int(rng.randint(1, 2 * cw + 2)), int(rng.randint(1, 2 * ch + 2))))
    return out


def _pillow_resize(pixels, box, filt):
    im = Image.fromarray(pixels[..., 0] if pixels.shape[2] == 1 else pixels)
    if any(box[:4]):
        im = im.crop(box[:4])
    out = np.asarray(im.resize(box[4:6], getattr(Image.Resampling, filt.upper())))
    return out[..., None] if out.ndim == 2 else out


@pytest.mark.parametrize("filt", sorted(FILTERS))
def test_transpose_then_crop_then_resize(ctx, corpus, filt):  # noqa: F811
    names = [n for n in _names(corpus) if n != "cmyk"]
    datas = [corpus[n] for n in names]
    _, flags, niter = OPTS["q3"]
    for d, layout, on_device in ((1, 0, 1), (2, 1, 0)):
        ref = _unoriented(ctx, datas, flags, niter, d)
        orient = [(k + len(filt)) % 8 + 1 for k in range(len(names))]
        boxes = _oriented_boxes(datas, orient, d, seed=len(filt) + d)
        got = _c_oriented(ctx, datas, flags, niter, layout, d, orient, on_device, boxes, filt)
        for n, o, b, (rc, pix, _), (_, rpix, _) in zip(names, orient, boxes, got, ref):
            assert rc == 0, n
            assert np.array_equal(pix, _pillow_resize(turn(rpix, o), b, filt)), (n, o, b, d)


@pytest.mark.parametrize("on_device", [1, 0])
def test_a_crop_valid_only_unoriented_fails_alone(ctx, corpus, on_device):  # noqa: F811
    names = ["rst", "base420", "gray"]                    # rst: 250 x 190, landscape
    datas = [corpus[n] for n in names]
    _, flags, niter = OPTS["q3"]
    ref = _unoriented(ctx, datas, flags, niter, 1)
    orient = [6, 8, 5]
    boxes = [(0, 0, 250, 190, 50, 40)] + _oriented_boxes(datas[1:], orient[1:], 1, seed=5)
    got = _c_oriented(ctx, datas, flags, niter, 0, 1, orient, on_device, boxes, "bilinear")
    assert got[0][0] == -2
    assert "crop" in ctx.lib.jpegqs_cuda_last_error(ctx.h).decode()
    for o, b, (rc, pix, _), (_, rpix, _) in list(zip(orient, boxes, got, ref))[1:]:
        assert rc == 0 and np.array_equal(pix, _pillow_resize(turn(rpix, o), b, "bilinear"))
    # the same crop in the oriented picture (190 x 250) is fine
    (rc, pix, _), = _c_oriented(ctx, datas[:1], flags, niter, 0, 1, [6], on_device, [(0, 0, 190, 250, 50, 40)], "bilinear")
    assert rc == 0 and np.array_equal(pix, _pillow_resize(turn(ref[0][1], 6), (0, 0, 190, 250, 50, 40), "bilinear"))


def test_bad_values_do_nothing(ctx, corpus):  # noqa: F811
    datas = [corpus["base420"], corpus["gray"]]
    _, flags, niter = OPTS["q3"]
    for bad in ([1, 9], [-1, 1]):
        with pytest.raises(AssertionError, match="orientation"):
            _c_oriented(ctx, datas, flags, niter, 0, 1, bad, 1)


def _pillow_save(a, quality, subsampling, optimize):
    b = io.BytesIO()
    Image.fromarray(a if a.shape[2] == 3 else a[:, :, 0]).save(b, "JPEG", quality=quality, subsampling=subsampling,
                                                               optimize=optimize)
    return b.getvalue()


PY_NAMES = ["base420", "base444", "prog420", "gray", "opt422", "rst", "tinyprog", "damaged", "garbled", "stop"]


def test_reencode_exif_is_pillows_save_of_the_transposed_picture(ctx, corpus):  # noqa: F811
    _, flags, niter = OPTS["q3"]
    tags = [k % 8 + 1 for k in range(len(PY_NAMES))]
    plain = [corpus[n] for n in PY_NAMES]
    spliced = [tagged(x, o) for x, o in zip(plain, tags)]
    for d, (q, s, opt) in ((1, (85, "4:2:0", False)), (2, (95, "4:4:4", True))):
        got = ctx.reencode(spliced, flags | qs.JPEGQS_TRANSCODE, niter, q, s, opt, scale_denom=d, orientation="exif")
        pix = ctx.decode_pixels(plain, flags | qs.JPEGQS_TRANSCODE, niter, device="cpu", scale_denom=d)
        for n, o, g, p in zip(PY_NAMES, tags, got, pix):
            assert g[0] == _pillow_save(turn(p[0].numpy(), o), q, s, opt), (n, o, d)
            assert g[1:] == p[1:], n
            assert g[0][:4] == b"\xff\xd8\xff\xe0" and b"Exif" not in g[0]       # JFIF, no tag
    # crop and size in the oriented picture
    sizes = [(64, 48)] * len(PY_NAMES)
    got = ctx.reencode(spliced, flags | qs.JPEGQS_TRANSCODE, niter, 80, "4:2:0", False, size=sizes, orientation="exif")
    pix = ctx.decode_pixels(spliced, flags | qs.JPEGQS_TRANSCODE, niter, device="cpu", size=sizes, orientation="exif")
    for n, g, p in zip(PY_NAMES, got, pix):
        assert g[0] == _pillow_save(p[0].numpy(), 80, "4:2:0", False), n


def test_python_decode_pixels(ctx, corpus):  # noqa: F811
    _, flags, niter = OPTS["q6"]
    plain = [corpus[n] for n in PY_NAMES]
    tags = [(k * 5) % 8 + 1 for k in range(len(PY_NAMES))]
    spliced = [tagged(x, o) for x, o in zip(plain, tags)]
    ref = ctx.decode_pixels(plain, flags | qs.JPEGQS_TRANSCODE, niter, device="cpu")
    for layout in ("hwc", "chw"):
        for orientation, want in (("exif", tags), (6, [6] * len(tags)), ([0, 2] * 5, [t if k % 2 == 0 else 2 for k, t in enumerate(tags)])):
            got = ctx.decode_pixels(spliced, flags | qs.JPEGQS_TRANSCODE, niter, layout=layout, orientation=orientation)
            for n, o, g, r in zip(PY_NAMES, want, got, ref):
                a = g[0].cpu().numpy()
                a = a if layout == "hwc" else a.transpose(1, 2, 0)
                assert g[0].is_cuda and np.array_equal(a, turn(r[0].numpy(), o)), (n, o, layout)
                assert g[1:] == r[1:]
    # None is today's call
    got = ctx.decode_pixels(spliced, flags | qs.JPEGQS_TRANSCODE, niter, device="cpu")
    assert all(np.array_equal(g[0].numpy(), r[0].numpy()) for g, r in zip(got, ref))


@pytest.mark.parametrize("layout", ["hwc", "chw"])
def test_render_every_orientation_is_the_transposed_model(ctx, layout):  # noqa: F811
    ims = _images()
    work = [im.clone() for im in ims]
    coefs = [[torch.from_numpy(np.ascontiguousarray(c.coef)).cuda() for c in im.comps] for im in work]
    status, ups = ctx.run_async(work, coefs, 7, 2)
    torch.cuda.synchronize()
    models = {}
    for d in (1, 2, 8):
        for n in range(len(ims)):
            im, up = _run_result(work, coefs, status, ups, n)
            m = cuda.render_model(im, up, "hwc", d)
            models[(n, d)] = m
        for shift in range(8):
            orient = [(n + shift) % 8 + 1 for n in range(len(ims))]
            out = ctx.render_async(work, coefs, status, ups, layout=layout, scale_denom=d, orientation=orient)
            torch.cuda.synchronize()
            for n, o in enumerate(orient):
                a = out[n].cpu().numpy()
                a = a if layout == "hwc" else a.transpose(1, 2, 0)
                assert np.array_equal(a, turn(models[(n, d)], o)), (n, d, o)


def test_render_oriented_in_a_graph(ctx):  # noqa: F811
    ims = _images()[:2]
    work = [im.clone() for im in ims]
    static = [[torch.from_numpy(np.ascontiguousarray(c.coef)).cuda() for c in im.comps] for im in work]
    plan = {1: [6, 3], 2: [8, 5]}
    outs = {d: [torch.empty(_dims_of(im, d, o), dtype=torch.uint8, device="cuda") for im, o in zip(ims, plan[d])]
            for d in plan}
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        status, ups = ctx.run_async(work, static, 7, 2)
        for d in plan:
            ctx.render_async(work, static, status, ups, out=outs[d], scale_denom=d, orientation=plan[d])
    import hard_content as hc
    for seed in (0, 1):
        inputs = ims if seed == 0 else [hc.make_image(im.width, im.height, ss, hc.TABLES[t], "synth", seed=31)
                                        for im, ss, t in zip(ims, ("420", "422"), ("k50", "k90"))]
        for ts, im in zip(static, inputs):
            for t, c in zip(ts, im.comps):
                t.copy_(torch.from_numpy(c.coef))
        g.replay()
        torch.cuda.synchronize()
        ref = [im.clone() for im in inputs]
        rc = [[torch.from_numpy(np.ascontiguousarray(c.coef)).cuda() for c in im.comps] for im in ref]
        rst, rups = ctx.run_async(ref, rc, 7, 2)
        torch.cuda.synchronize()
        for n in range(len(ims)):
            im, up = _run_result(ref, rc, rst, rups, n)
            for d in plan:
                want = turn(cuda.render_model(im, up, "hwc", d), plan[d][n])
                assert np.array_equal(outs[d][n].cpu().numpy(), want), (seed, n, d)


def _dims_of(im, d, o):
    w, h = -(-im.width // d), -(-im.height // d)
    return (w, h, 3) if o >= 5 else (h, w, 3)


def test_render_rejects_bad_orientation_with_nothing_enqueued(ctx):  # noqa: F811
    im = _images()[1]
    coefs = [[torch.from_numpy(np.ascontiguousarray(c.coef)).cuda() for c in im.comps]]
    out = torch.zeros(im.height * im.width * 3, dtype=torch.uint8, device="cuda")
    arr = cuda._image_array([im], [[t.data_ptr() for t in coefs[0]]])
    torch.cuda.synchronize()
    for o in (0, 9, -3):
        assert ctx.lib.jpegqs_cuda_render_oriented_async(ctx.h, 1, arr, None, 0, 1, (C.c_int32 * 1)(o),
                                                         (C.c_void_p * 1)(out.data_ptr()), None) == -2
        assert "orientation" in ctx.lib.jpegqs_cuda_last_error(ctx.h).decode()
    torch.cuda.synchronize()
    assert not out.any()
