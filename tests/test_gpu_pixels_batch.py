"""jpegqs_cuda_pixels_batch (QsContext.decode_pixels) on the GPU: every file's pixels are the body of
what `jpegqs --ppm` writes for it with the same -q / -n, in both layouts and both output kinds, and
they do not depend on the files beside them, their order, the sub-batch budget or the context's
earlier calls.  Also libjpeg-turbo's decode at -n 0, the run statuses against transcode_batch, the
one-channel store of grey images at odd byte offsets, and the Python call."""
import ctypes as C
import io
import os
import subprocess

import numpy as np
import pytest

PIL = pytest.importorskip("PIL.Image")

import decode_files as df
import scan_files as sf
from test_cli import EXE, FILES, _big_picture, _picture
from test_gpu_transcode_batch import _c_batch as _tc_batch, _damaged, _stop_file

import jpegqs_b200 as qs
from jpegqs_b200 import cuda

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")


def _garbled(good):
    """Stuffed 0xFF bytes in the middle of the entropy-coded data: all-ones bit patterns, which no
    Huffman code has.  The device decoder flags the file; the reader recovers with warnings."""
    d = bytearray(good)
    d[len(d) * 3 // 5:len(d) * 3 // 5 + 32] = b"\xff\x00" * 16
    return bytes(d)


@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    """name -> bytes: every tool flavour (prog420 is progressive without restart markers: host route),
    CMYK, a scan script with restart markers, the 8K file, two damaged files and a stopping image."""
    d = tmp_path_factory.mktemp("corpus")
    out = {}
    for k, (name, w, h, gray, kw) in enumerate(FILES):
        p = d / f"{name}.jpg"
        _picture(w, h, gray, k).save(str(p), comment=b"made by the test suite", **kw)
        out[name] = p.read_bytes()
    out["cmyk"] = df.pillow_jpeg(120, 80, "CMYK", quality=85)
    scripted = [(n, b) for n, b in sf.scripted() if "rst" in n]
    if scripted:
        out["script_" + scripted[0][0]] = scripted[0][1]
    p = d / "8k.jpg"
    _big_picture(7680, 4320, 5).save(str(p), quality=90)
    out["8k"] = p.read_bytes()
    out["damaged"] = _damaged(out["base420"])
    out["garbled"] = _garbled(out["base420"])
    out["stop"] = _stop_file()
    return out


@pytest.fixture(scope="module")
def ctx():
    c = cuda.QsContext(0)
    yield c
    c.close()


OPTS = {"q3": (["-q", "3", "-n", "3"], qs.quality_to_flags(3), 3),
        "q6": (["-q", "6", "-n", "3"], qs.quality_to_flags(6), 3),
        "n0": (["-q", "6", "-n", "0"], qs.quality_to_flags(6), 0)}


def _ppm(path, args, out):
    """(exit status, body of the PPM / PGM the tool writes or None)"""
    r = subprocess.run([EXE] + args + ["--ppm", str(path), str(out)], capture_output=True, text=True)
    body = None
    if os.path.exists(out):
        with open(out, "rb") as f:
            magic, dims, maxval, body = f.read().split(b"\n", 3)
        assert magic in (b"P5", b"P6") and maxval == b"255"
        os.unlink(out)
    return r.returncode, body


@pytest.fixture(scope="module")
def tool(corpus, tmp_path_factory):
    """(name, opt) -> the tool's (exit status, body), computed once."""
    d = tmp_path_factory.mktemp("tool")
    for n, b in corpus.items():
        (d / f"{n}.jpg").write_bytes(b)
    cache = {}

    def get(name, opt):
        if (name, opt) not in cache:
            cache[(name, opt)] = _ppm(d / f"{name}.jpg", OPTS[opt][0], d / f"{name}.ppm")
        return cache[(name, opt)]
    return get


def _shape(data):
    info = cuda._FileInfo()
    assert cuda.load().jpegqs_cuda_transcode_route(data, len(data), None, C.byref(info)) >= 0
    return info.image_width, info.image_height, info.ncomp


def _c_batch(ctx, datas, flags, niter, layout, on_device, budget=0):
    """The C call; outputs of image_width * image_height * channels bytes (CMYK: 3 channels' worth, not
    written) - on the device at odd byte offsets of one flat tensor with a guard byte after each, or
    host buffers.  Returns [(rc, bytes or None, (channels, host_decoded, warnings, smoothed, stop,
    upsampled, reason))]."""
    n = len(datas)
    sizes = [w * h * (1 if c == 1 else 3) for w, h, c in (_shape(d) for d in datas)]
    offs, o = [], 1
    for s in sizes:
        offs.append(o)
        o += s + 1 + (o & 2)
    if on_device:
        flat = torch.full((o + 1,), 0xA5, dtype=torch.uint8, device=f"cuda:{ctx.device}")
        outs = (C.c_void_p * n)(*[flat.data_ptr() + x for x in offs])
    else:
        bufs = [(C.c_uint8 * (s + 1))(*([0] * s + [0xA5])) for s in sizes]
        outs = (C.c_void_p * n)(*[C.addressof(b) for b in bufs])
    torch.cuda.synchronize(ctx.device)
    ptrs = (C.c_char_p * n)(*datas)
    lens = (C.c_size_t * n)(*[len(d) for d in datas])
    rc = (C.c_int * n)()
    res = (cuda._PixelsResult * n)()
    ret = ctx.lib.jpegqs_cuda_pixels_batch(ctx.h, n, ptrs, lens, flags | qs.JPEGQS_TRANSCODE, niter, layout, on_device,
                                           outs, budget, rc, res)
    assert ret == 0, ctx.lib.jpegqs_cuda_last_error(ctx.h).decode()
    if on_device:
        host = flat.cpu().numpy().tobytes()
        got = [host[x:x + s] for x, s in zip(offs, sizes)]
        for x, s in zip(offs, sizes):
            assert host[x + s] == 0xA5                 # nothing written past a file's output
    else:
        got = [bytes(b)[:s] for b, s in zip(bufs, sizes)]
        assert all(b[s] == 0xA5 for b, s in zip(bufs, sizes))
    return [(rc[i], got[i] if rc[i] == 0 else None,
             (res[i].channels, res[i].host_decoded, res[i].warnings, res[i].smoothed, res[i].stop, res[i].upsampled,
              (res[i].reason or b"").decode())) for i in range(n)]


def _as_hwc(body, data, layout):
    """pixels in the tool's interleaved order"""
    w, h, c = _shape(data)
    c = 1 if c == 1 else 3
    a = np.frombuffer(body, dtype=np.uint8)
    return (a.reshape(h, w, c) if layout == 0 else a.reshape(c, h, w).transpose(1, 2, 0)).tobytes()


@pytest.mark.parametrize("on_device", [1, 0])
@pytest.mark.parametrize("layout", [0, 1])
@pytest.mark.parametrize("opt", sorted(OPTS))
def test_pixels_equal_the_tool(ctx, corpus, tool, opt, layout, on_device):
    names = sorted(corpus)
    _, flags, niter = OPTS[opt]
    got = _c_batch(ctx, [corpus[n] for n in names], flags, niter, layout, on_device)
    for n, (rc, pix, res) in zip(names, got):
        status, body = tool(n, opt)
        if n == "cmyk":
            assert rc == -3                            # JPEGQS_ERR_UNSUPPORTED
            assert status != 0 and body is None
            continue
        assert rc == 0, n
        assert _as_hwc(pix, corpus[n], layout) == body, (n, opt, layout, on_device)
        assert res[0] == (1 if _shape(corpus[n])[2] == 1 else 3)
        assert status == (2 if res[2] > 0 else 0), (n, status, res)
    by = dict(zip(names, got))
    for n in ("damaged", "garbled"):
        assert by[n][2][1] == 1 and "flagged" in by[n][2][6], n
    assert by["garbled"][2][2] > 0 and tool("garbled", opt)[0] == 2
    assert by["prog420"][2][1] == 1 and "restart markers" in by["prog420"][2][6]
    assert by["base420"][2][1] == 0 and by["base420"][2][6] == ""
    if opt != "n0":
        assert by["stop"][2][3] == 1 and by["stop"][2][4] != 0


def test_pixels_equal_libjpeg_turbo_at_n0(ctx, corpus):
    """Nothing smoothed (-q 3 -n 0): the pixels are libjpeg-turbo's (Pillow's) decode of the file."""
    names = [n for n in sorted(corpus) if n not in ("cmyk", "damaged", "garbled", "stop")]
    got = _c_batch(ctx, [corpus[n] for n in names], qs.quality_to_flags(3), 0, 0, 1)
    for n, (rc, pix, res) in zip(names, got):
        assert rc == 0 and res[3] == 0, n
        want = np.asarray(PIL.open(io.BytesIO(corpus[n])))
        assert pix == want.tobytes(), n


@pytest.mark.parametrize("opt", ["q3", "q6"])
def test_run_status_equals_transcode(ctx, corpus, opt):
    names = [n for n in sorted(corpus) if n != "cmyk"]
    _, flags, niter = OPTS[opt]
    tc = _tc_batch(ctx, [corpus[n] for n in names], flags | qs.JPEGQS_TRANSCODE, niter, False, 2)
    px = _c_batch(ctx, [corpus[n] for n in names], flags, niter, 0, 1)
    n_dev = 0
    for n, t, (rc, _, res) in zip(names, tc, px):
        if t[0] != cuda.TRANSCODE_OK:
            continue
        n_dev += 1
        assert (res[3], res[4], res[5]) == (t[2], t[3], t[4]), n
        assert res[1] == 0, n
    assert n_dev >= 10


@pytest.fixture(scope="module")
def singles(ctx, corpus):
    cache = {}

    def get(name, opt):
        if (name, opt) not in cache:
            _, flags, niter = OPTS[opt]
            cache[(name, opt)] = _c_batch(ctx, [corpus[name]], flags, niter, 0, 1)[0]
        return cache[(name, opt)]
    return get


@pytest.mark.parametrize("seed", [1, 2])
def test_order_does_not_matter(ctx, corpus, singles, seed):
    names = sorted(corpus)
    perm = list(np.random.RandomState(seed).permutation(len(names)))
    _, flags, niter = OPTS["q6"]
    got = _c_batch(ctx, [corpus[names[i]] for i in perm], flags, niter, 0, 1)
    for i, g in zip(perm, got):
        assert g == singles(names[i], "q6"), names[i]


@pytest.mark.parametrize("budget", [1, 3 << 20])
@pytest.mark.parametrize("on_device", [1, 0])
def test_splitting_is_invisible(ctx, corpus, singles, budget, on_device):
    names = sorted(corpus)
    _, flags, niter = OPTS["q3"]
    got = _c_batch(ctx, [corpus[n] for n in names], flags, niter, 0, on_device, budget)
    for n, g in zip(names, got):
        assert g == singles(n, "q3"), (n, budget)


def test_buffer_reuse_across_calls(corpus, singles):
    """Calls of growing and shrinking sizes on one context give the single-file results."""
    c = cuda.QsContext(0)
    _, flags, niter = OPTS["q3"]
    small = ["base420", "gray", "prog420", "damaged", "tinyprog", "rst"]
    for names in (small[:2], small, ["8k"] + small, small[:3], small):
        got = _c_batch(c, [corpus[n] for n in names], flags, niter, 0, 1)
        for n, g in zip(names, got):
            assert g == singles(n, "q3"), (n, names)
    assert c.last_device_ms > 0
    c.close()


@pytest.mark.parametrize("layout", [0, 1])
def test_grey_store_at_odd_offsets(ctx, corpus, tool, layout):
    """Grey files of widths that are not multiples of 4 (17x9, 97x61) written one byte per pixel at odd
    byte offsets of one flat tensor, between colour files, in both layouts."""
    names = ["tinyprog", "base444", "gray", "tinyprog", "base420", "gray"]
    _, flags, niter = OPTS["q6"]
    got = _c_batch(ctx, [corpus[n] for n in names], flags, niter, layout, 1)
    for n, (rc, pix, res) in zip(names, got):
        assert rc == 0
        assert _as_hwc(pix, corpus[n], layout) == tool(n, "q6")[1], (n, layout)
    assert got[0][2][0] == got[2][2][0] == 1 and got[1][2][0] == 3


def test_python_call(corpus):
    c = cuda.QsContext(0)
    _, flags, niter = OPTS["q6"]
    names = ["base420", "gray", "prog420", "garbled", "stop"]
    datas = [corpus[n] for n in names]
    for layout in ("hwc", "chw"):
        dev = c.decode_pixels(datas, flags | qs.JPEGQS_TRANSCODE, niter, layout=layout)
        cpu = c.decode_pixels(datas, flags | qs.JPEGQS_TRANSCODE, niter, layout=layout, device="cpu")
        for n, d, h in zip(names, dev, cpu):
            w_, h_, nc = _shape(corpus[n])
            shape = (h_, w_, nc) if layout == "hwc" else (nc, h_, w_)
            assert d[0].is_cuda and d[0].device.index == 0 and tuple(d[0].shape) == shape and d[0].dtype == torch.uint8
            assert not h[0].is_cuda and tuple(h[0].shape) == shape
            assert torch.equal(d[0].cpu(), h[0]) and d[1:] == h[1:], n
        by = dict(zip(names, dev))
        assert by["garbled"][1] > 0 and by["garbled"][2] == 1 and "flagged" in by["garbled"][6]
        assert by["prog420"][2] == 1 and by["base420"][2] == 0 and by["base420"][6] == ""
    single = qs.decode_pixels([corpus["gray"]], flags | qs.JPEGQS_TRANSCODE, niter, layout="chw", gpu=0)
    assert torch.equal(single[0][0], dev[1][0]) and single[0][1:] == dev[1][1:]
    for bad, idx in (([corpus["base420"], b"this is not a jpeg"], 1), ([corpus["gray"], corpus["base420"], corpus["cmyk"]], 2)):
        with pytest.raises(cuda.QsError, match=f"file {idx}"):
            c.decode_pixels(bad, flags, niter)
    c.close()


def test_c_call_checks_its_arguments(ctx, corpus):
    data = corpus["base420"]
    ptrs = (C.c_char_p * 2)(data, data)
    lens = (C.c_size_t * 2)(len(data), len(data))
    buf = (C.c_uint8 * (64 * 48 * 3 * 2))()
    outs = (C.c_void_p * 2)(C.addressof(buf), C.addressof(buf) + 64 * 48 * 3)
    rc = (C.c_int * 2)(7, 7)
    res = (cuda._PixelsResult * 2)()
    res[0].channels = res[1].channels = 9
    f = ctx.lib.jpegqs_cuda_pixels_batch
    assert f(ctx.h, 0, None, None, 0, 3, 0, 0, None, 0, None, None) == 0
    assert f(ctx.h, -1, ptrs, lens, 0, 3, 0, 0, outs, 0, rc, res) == -2
    for a in ((None, lens, outs, rc, res), (ptrs, None, outs, rc, res), (ptrs, lens, None, rc, res),
              (ptrs, lens, outs, None, res), (ptrs, lens, outs, rc, None)):
        assert f(ctx.h, 2, a[0], a[1], 0, 3, 0, 0, a[2], 0, a[3], a[4]) == -2
    for layout, on_device in ((2, 0), (-1, 0), (0, 2)):
        assert f(ctx.h, 2, ptrs, lens, 0, 3, layout, on_device, outs, 0, rc, res) == -2
    holes = (C.c_void_p * 2)(C.addressof(buf), None)
    assert f(ctx.h, 2, ptrs, lens, 0, 3, 0, 0, holes, 0, rc, res) == -2
    assert "file 1" in ctx.lib.jpegqs_cuda_last_error(ctx.h).decode()
    assert list(rc) == [7, 7] and res[0].channels == res[1].channels == 9
    assert bytes(buf) == bytes(len(buf))
