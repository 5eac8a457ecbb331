"""Colour modes on the GPU.  decode_pixels(mode="RGB" / "L") gives, for file i, Pillow's
    im = Image.open(F); im.draft(None, (W // d, H // d)) at d > 1; im = im.transpose(...) for an orientation;
    im = im.convert(mode); im.crop(box).resize(size, filter) when given
with F the file the jpegqs tool writes for the same options (the input file at -q 3 -n 0).  CMYK, YCCK
(Adobe transform 2, and 1 read as YCCK), grey, YCbCr and untransformed RGB files, both layouts, device and
host outputs, every scale, the eight orientations on a CMYK and a YCCK file, crop and resize with every
filter, an 8K CMYK file, mixed batches under forced splits and shuffled, reencode against Pillow's save,
render_async(mode=) eagerly and replayed from a CUDA graph, and mode None / 0 against the existing calls."""
import io
import os
import subprocess

import numpy as np
import pytest

from test_gpu_pixels_batch import corpus, ctx  # noqa: F401  (module fixtures)
from test_pixel_modes_cpu import FILES, YCCK_FACTORS, cmyk_file, ycck_file

import jpegqs_b200 as qs
from jpegqs_b200 import cuda

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
Image = pytest.importorskip("PIL.Image")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "jpeg-quantsmooth_b200", "csrc", "jpegqs")
OPTS = {"q3": (["-q", "3", "-n", "3"], qs.quality_to_flags(3), 3),
        "q6": (["-q", "6", "-n", "3"], qs.quality_to_flags(6), 3),
        "q3n0": (["-q", "3", "-n", "0"], qs.quality_to_flags(3), 0)}
T = Image.Transpose
METHODS = {2: T.FLIP_LEFT_RIGHT, 3: T.ROTATE_180, 4: T.FLIP_TOP_BOTTOM, 5: T.TRANSPOSE, 6: T.ROTATE_270,
           7: T.TRANSVERSE, 8: T.ROTATE_90}
FILTERS = {"lanczos": Image.Resampling.LANCZOS, "bilinear": Image.Resampling.BILINEAR,
           "bicubic": Image.Resampling.BICUBIC, "box": Image.Resampling.BOX, "hamming": Image.Resampling.HAMMING}


@pytest.fixture(scope="module")
def files(corpus):  # noqa: F811
    """name -> bytes: the CPU test's colour spaces, the pixel corpus' files, a large CMYK and YCCK file"""
    out = dict(FILES)
    for k in ("base420", "gray", "cmyk", "prog420", "damaged", "stop"):
        if k in corpus:
            out["corpus_" + k] = corpus[k]
    out["big_cmyk"] = cmyk_file(700, 300, 21, quality=85)
    out["big_ycck"] = ycck_file(530, 270, YCCK_FACTORS["y2k2"], seed=22)
    return out


@pytest.fixture(scope="module")
def tool_file(tmp_path_factory):
    """(data, opt) -> the file the render's coefficients come from: the tool's output, or the input at q3n0"""
    tmp = tmp_path_factory.mktemp("modes")
    cache = {}

    def get(data, opt):
        key = (data, opt)
        if key not in cache:
            if opt == "q3n0":
                cache[key] = data
            else:
                src, dst = tmp / "src.jpg", tmp / "dst.jpg"
                src.write_bytes(data)
                r = subprocess.run([EXE] + OPTS[opt][0] + [str(src), str(dst)], capture_output=True, text=True)
                assert r.returncode in (0, 2) and dst.exists(), r.stderr
                cache[key] = dst.read_bytes()
                dst.unlink()
        return cache[key]
    return get


def pillow(data, d=1, mode="RGB", o=1, box=None, size=None, filt="bicubic"):
    im = Image.open(io.BytesIO(data))
    w, h = im.size
    if d > 1:
        im.draft(None, (w // d, h // d))
        assert im.size == (-(-w // d), -(-h // d))
    if o > 1:
        im = im.transpose(METHODS[o])
    im = im.convert(mode)
    if size is not None:
        im = im.resize(size, FILTERS[filt], box=box)
    out = np.asarray(im)
    return out if out.ndim == 3 else out[..., None]


def hwc(t, layout):
    a = t.cpu().numpy()
    return a if layout == "hwc" else np.moveaxis(a, 0, -1)


DECODABLE = ["q90", "q50", "q20_progressive", "restart", "ycck_444", "ycck_y2k2", "ycck_k_alone", "adobe1", "adobe7",
             "no_app14", "grey", "ycbcr420", "ycbcr444", "keep_rgb", "corpus_base420", "corpus_gray", "corpus_cmyk",
             "corpus_prog420"]


@pytest.mark.parametrize("opt", sorted(OPTS))
@pytest.mark.parametrize("layout,device", [("hwc", "cuda"), ("chw", "cpu")])
@pytest.mark.parametrize("mode", ["RGB", "L"])
def test_decode_pixels_mode_is_pillows_convert(ctx, files, tool_file, opt, layout, device, mode):  # noqa: F811
    names = [n for n in DECODABLE if n in files]
    _, flags, niter = OPTS[opt]
    recs = ctx.decode_pixels([files[n] for n in names], flags, niter, layout=layout, device=device, mode=mode)
    for n, r in zip(names, recs):
        want = pillow(tool_file(files[n], opt), 1, mode)
        got = hwc(r[0], layout)
        assert got.shape == want.shape and np.array_equal(got, want), (n, opt)


@pytest.mark.parametrize("d", [2, 4, 8])
@pytest.mark.parametrize("mode", ["RGB", "L"])
def test_every_scale(ctx, files, tool_file, d, mode):  # noqa: F811
    names = ["q90", "q20_progressive", "ycck_y2k2", "ycck_k_alone", "adobe1", "grey", "ycbcr420", "big_cmyk", "big_ycck"]
    recs = ctx.decode_pixels([files[n] for n in names], OPTS["q6"][1], 3, scale_denom=d, mode=mode)
    for n, r in zip(names, recs):
        assert np.array_equal(hwc(r[0], "hwc"), pillow(tool_file(files[n], "q6"), d, mode)), (n, d)


@pytest.mark.parametrize("name", ["big_cmyk", "big_ycck"])
@pytest.mark.parametrize("layout", ["hwc", "chw"])
def test_every_orientation(ctx, files, tool_file, name, layout):  # noqa: F811
    data = files[name]
    for mode in ("RGB", "L"):
        for d in (1, 2):
            recs = ctx.decode_pixels([data] * 8, 0, 3, layout=layout, scale_denom=d, orientation=list(range(1, 9)),
                                     mode=mode)
            for o, r in zip(range(1, 9), recs):
                assert np.array_equal(hwc(r[0], layout), pillow(tool_file(data, "q3"), d, mode, o)), (name, mode, d, o)


@pytest.mark.parametrize("filt", sorted(FILTERS))
def test_crop_and_resize(ctx, files, tool_file, filt):  # noqa: F811
    names = ["big_cmyk", "big_ycck", "corpus_base420", "corpus_gray"]
    datas = [files[n] for n in names]
    for mode in ("RGB", "L"):
        crops, sizes = [], []
        for k, (data, o) in enumerate(zip(datas, [6, 1, 3, 8])):
            w, h = Image.open(io.BytesIO(data)).size
            w, h = (h, w) if o >= 5 else (w, h)                     # the crop is in the oriented picture
            crops.append((k + 3, 2 * k + 1, w - 5, h - k - 2))
            sizes.append((w // 3 + k, h // 2 + 7))
        recs = ctx.decode_pixels(datas, 0, 3, size=sizes, crop=crops, filter=filt, mode=mode, orientation=[6, 1, 3, 8])
        for data, c, s, o, r in zip(datas, crops, sizes, [6, 1, 3, 8], recs):
            im = Image.open(io.BytesIO(tool_file(data, "q3"))).transpose(METHODS[o]) if o > 1 else \
                Image.open(io.BytesIO(tool_file(data, "q3")))
            want = np.asarray(im.convert(mode).crop(c).resize(s, FILTERS[filt]))
            want = want if want.ndim == 3 else want[..., None]
            assert np.array_equal(hwc(r[0], "hwc"), want), (mode, filt)


def test_8k_cmyk_file(ctx, tool_file):  # noqa: F811
    data = cmyk_file(7680, 4320, 31, quality=90)
    for mode in ("RGB", "L"):
        r = ctx.decode_pixels([data], OPTS["q6"][1], 3, mode=mode)[0]
        assert np.array_equal(hwc(r[0], "hwc"), pillow(tool_file(data, "q6"), 1, mode))


@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("budget", [0, 3 << 20])
def test_mixed_batch_splits_and_order(ctx, files, seed, budget):  # noqa: F811
    names = sorted(files)
    rng = np.random.default_rng(seed)
    order = list(rng.permutation(len(names)))
    for mode in ("RGB", "L"):
        single = {}
        for n in names:
            try:
                single[n] = hwc(ctx.decode_pixels([files[n]], 0, 3, mode=mode)[0][0], "hwc")
            except cuda.QsError:
                single[n] = None
        good = [names[i] for i in order if single[names[i]] is not None]
        recs = ctx.decode_pixels([files[n] for n in good], 0, 3, mode=mode, max_device_bytes=budget)
        for n, r in zip(good, recs):
            assert np.array_equal(hwc(r[0], "hwc"), single[n]), n
        assert "corpus_damaged" not in good or single["corpus_damaged"] is not None


def test_mode_zero_is_the_existing_call(ctx, files, corpus):  # noqa: F811
    names = [n for n in corpus if n not in ("cmyk", "8k", "garbled")]
    datas = [corpus[n] for n in names]
    for d in (1, 4):
        a = ctx.decode_pixels(datas, 0, 3, scale_denom=d)
        b = ctx.decode_pixels(datas, 0, 3, scale_denom=d, mode=None, orientation=[1] * len(datas))
        for x, y in zip(a, b):
            assert np.array_equal(x[0].cpu().numpy(), y[0].cpu().numpy())
    with pytest.raises(cuda.QsError):
        ctx.decode_pixels([corpus["cmyk"]], 0, 3)                  # 4 components without a mode: still -3
    with pytest.raises(cuda.QsError):
        ctx.decode_pixels([corpus["cmyk"]], 0, 3, mode=None)
    for bad in ("CMYK", "rgb", 1):
        with pytest.raises(ValueError):
            ctx.decode_pixels([corpus["cmyk"]], 0, 3, mode=bad)
        with pytest.raises(ValueError):
            ctx.reencode([corpus["cmyk"]], 0, 3, mode=bad)


def _c_mode(ctx, datas, mode):
    import ctypes as C
    lib = cuda.load()
    n = len(datas)
    outs = [np.zeros(1 << 20, np.uint8) for _ in datas]
    rc = (C.c_int * n)()
    res = (cuda._PixelsResult * n)()
    ret = lib.jpegqs_cuda_pixels_batch_mode(ctx.h, n, (C.c_char_p * n)(*datas), (C.c_size_t * n)(*map(len, datas)),
                                            0, 3, 0, 1, 0, None, None, mode, 0,
                                            (C.c_void_p * n)(*[o.ctypes.data for o in outs]), 0, rc, res)
    return ret, list(rc), [bytes(o) for o in outs], [r.channels for r in res]


def test_c_mode_zero_and_bad_modes(ctx, files, corpus):  # noqa: F811
    datas = [corpus["base420"], corpus["gray"], corpus["cmyk"]]
    ret, rc, outs, ch = _c_mode(ctx, datas, 0)
    assert ret == 0 and rc == [0, 0, -3] and ch[:2] == [3, 1]
    ref = ctx.decode_pixels(datas[:2], 0, 3, device="cpu")
    for o, r in zip(outs, ref):
        t = r[0].numpy().tobytes()
        assert o[:len(t)] == t
    ret, rc, _, ch = _c_mode(ctx, datas, 1)
    assert ret == 0 and rc == [0, 0, 0] and ch == [3, 3, 3]
    for bad in (-1, 3):
        ret, rc, outs, _ = _c_mode(ctx, datas, bad)
        assert ret == -2 and not any(any(o) for o in outs)


@pytest.mark.parametrize("mode", ["RGB", "L"])
def test_reencode_mode_is_pillows_save(ctx, files, tool_file, mode):  # noqa: F811
    names = ["q90", "ycck_y2k2", "adobe1", "grey", "ycbcr420", "big_cmyk"]
    recs = ctx.reencode([files[n] for n in names], 0, 3, quality=85, subsampling="4:2:0", mode=mode)
    for n, r in zip(names, recs):
        b = io.BytesIO()
        Image.open(io.BytesIO(tool_file(files[n], "q3"))).convert(mode).save(b, "JPEG", quality=85, subsampling=2)
        assert r[0] == b.getvalue(), n


def _device_image(data):
    im = cuda.read_jpeg(data)
    return im, [torch.from_numpy(np.ascontiguousarray(c.coef)).cuda() for c in im.comps]


@pytest.mark.parametrize("mode", ["RGB", "L"])
def test_render_async_in_a_graph(ctx, files, mode):  # noqa: F811
    names = ["q90", "ycck_y2k2", "adobe7", "grey", "ycbcr420", "keep_rgb", "big_ycck"]
    ims, coefs = zip(*[_device_image(files[n]) for n in names if n in files])
    want = [cuda.render_model(im, scale_denom=2, mode=mode) for im in ims]
    eager = ctx.render_async(list(ims), list(coefs), scale_denom=2, mode=mode, orientation=[1, 6, 3, 5, 1, 8, 2][:len(ims)])
    torch.cuda.synchronize()
    for o, e, w in zip([1, 6, 3, 5, 1, 8, 2], eager, want):
        t = np.asarray(Image.fromarray(w[..., 0] if w.shape[2] == 1 else w).transpose(METHODS[o])) if o > 1 else w
        t = t if t.ndim == 3 else t[..., None]
        assert np.array_equal(e.cpu().numpy(), t)
    out = [torch.empty_like(e) for e in eager]
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        ctx.render_async(list(ims), list(coefs), scale_denom=2, mode=mode, out=out, stream=s,
                         orientation=[1, 6, 3, 5, 1, 8, 2][:len(ims)])
    for _ in range(2):
        for t in out:
            t.zero_()
        g.replay()
        torch.cuda.synchronize()
        for a, b in zip(out, eager):
            assert torch.equal(a, b)


def test_render_async_checks_the_colour_space(ctx, files):  # noqa: F811
    im, coef = _device_image(files["q90"])
    bad = im.clone()
    bad.colorspace = qs.JCS_YCbCr
    with pytest.raises(cuda.QsError):
        ctx.render_async([bad], [coef], mode="RGB")
    with pytest.raises(cuda.QsError):
        ctx.render_async([im], [coef])                           # 4 components, the file's own colour: -3
