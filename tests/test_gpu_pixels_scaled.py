"""The scaled decode on the GPU.  jpegqs_cuda_pixels_batch_scaled (QsContext.decode_pixels with
scale_denom) gives, at 1/2, 1/4 and 1/8 size, libjpeg's scaled decode of the coefficients the unscaled
call renders: those of the file `jpegqs` writes for the same flags and niter, or of the input file where
do_quantsmooth returns early.  Both layouts, both output kinds, host-route, device-flagged and grey
files at odd device offsets; forced splits and file order change nothing; d = 1 is pixels_batch byte for
byte.  render_async with scale_denom after run_async equals render_model on the run's coefficients,
eagerly and replayed from a CUDA graph."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import hard_content as hc
import libjpeg_pixels as lp
import libjpeg_scaled as ls
from test_cli import EXE
from test_gpu_pixels_batch import _shape, corpus, ctx  # noqa: F401  (module fixtures)

import jpegqs_b200 as qs
from jpegqs_b200 import cuda

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(lp.JPEG_SO is None, reason="no libjpeg inside Pillow")]

torch = pytest.importorskip("torch")

SCALES = (2, 4, 8)
# name -> (tool arguments, flags, niter); q3n0 returns early, so its reference is the input file
OPTS = {"q3": (["-q", "3", "-n", "3"], qs.quality_to_flags(3), 3),
        "q6": (["-q", "6", "-n", "3"], qs.quality_to_flags(6), 3),
        "q6n0": (["-q", "6", "-n", "0"], qs.quality_to_flags(6), 0),
        "q3n0": (["-q", "3", "-n", "0"], qs.quality_to_flags(3), 0)}


@pytest.fixture(scope="module")
def reference(corpus, tmp_path_factory):  # noqa: F811
    """(name, opt, d) -> libjpeg's scaled decode [H', W', C] of the file the render's coefficients come
    from: what the tool writes, or the input file at q3n0 (files whose data libjpeg must recover from
    excepted: their coefficients are the library reader's, so the tool's file stands in)."""
    tmp = tmp_path_factory.mktemp("scaled")
    files, cache = {}, {}

    def source(name, opt):
        if (name, opt) not in files:
            src = tmp / f"{name}.jpg"
            src.write_bytes(corpus[name])
            if opt == "q3n0" and name not in ("damaged", "garbled"):
                files[(name, opt)] = str(src)
            else:
                dst = tmp / f"{name}.{opt}.out.jpg"
                r = subprocess.run([EXE] + OPTS[opt][0] + [str(src), str(dst)], capture_output=True, text=True)
                assert r.returncode in (0, 2) and os.path.exists(dst), (name, opt, r.stderr)
                files[(name, opt)] = str(dst)
        return files[(name, opt)]

    def get(name, opt, d):
        if (name, opt, d) not in cache:
            cache[(name, opt, d)] = ls.decode_file(source(name, opt), d)[0]
        return cache[(name, opt, d)]
    return get


def _c_scaled(ctx, datas, flags, niter, layout, d, on_device, budget=0):  # noqa: F811
    """jpegqs_cuda_pixels_batch_scaled with outputs of ceil(w/d) * ceil(h/d) * channels bytes at odd
    byte offsets of one device tensor (a guard byte after each) or in host buffers.  Returns
    [(rc, bytes or None, (channels, host_decoded, warnings, smoothed, stop, upsampled, reason))]."""
    n = len(datas)
    sizes = [-(-w // d) * -(-h // d) * (1 if c == 1 else 3) for w, h, c in (_shape(x) for x in datas)]
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
    rc = (C.c_int * n)()
    res = (cuda._PixelsResult * n)()
    ret = ctx.lib.jpegqs_cuda_pixels_batch_scaled(ctx.h, n, (C.c_char_p * n)(*datas),
                                                  (C.c_size_t * n)(*[len(x) for x in datas]), flags | qs.JPEGQS_TRANSCODE,
                                                  niter, layout, d, on_device, outs, budget, rc, res)
    assert ret == 0, ctx.lib.jpegqs_cuda_last_error(ctx.h).decode()
    if on_device:
        host = flat.cpu().numpy().tobytes()
        got = [host[x:x + s] for x, s in zip(offs, sizes)]
        assert all(host[x + s] == 0xA5 for x, s in zip(offs, sizes))
    else:
        got = [bytes(b)[:s] for b, s in zip(bufs, sizes)]
        assert all(b[s] == 0xA5 for b, s in zip(bufs, sizes))
    return [(rc[i], got[i] if rc[i] == 0 else None,
             (res[i].channels, res[i].host_decoded, res[i].warnings, res[i].smoothed, res[i].stop, res[i].upsampled,
              (res[i].reason or b"").decode())) for i in range(n)]


def _hwc(body, data, layout, d):
    w, h, c = _shape(data)
    c = 1 if c == 1 else 3
    a = np.frombuffer(body, dtype=np.uint8)
    w, h = -(-w // d), -(-h // d)
    return a.reshape(h, w, c) if layout == 0 else a.reshape(c, h, w).transpose(1, 2, 0)


@pytest.mark.parametrize("on_device", [1, 0])
@pytest.mark.parametrize("layout", [0, 1])
@pytest.mark.parametrize("opt", sorted(OPTS))
def test_pixels_are_libjpegs_scaled_decode(ctx, corpus, reference, opt, layout, on_device):  # noqa: F811
    names = sorted(corpus)
    _, flags, niter = OPTS[opt]
    for d in SCALES:
        got = _c_scaled(ctx, [corpus[n] for n in names], flags, niter, layout, d, on_device)
        for n, (rc, pix, res) in zip(names, got):
            if n == "cmyk":
                assert rc == -3
                continue
            assert rc == 0, n
            assert np.array_equal(_hwc(pix, corpus[n], layout, d), reference(n, opt, d)), (n, opt, layout, on_device, d)
        by = dict(zip(names, got))
        assert by["prog420"][2][1] == 1 and by["damaged"][2][1] == 1 and by["garbled"][2][2] > 0
        assert by["gray"][2][0] == 1 and by["base420"][2][1] == 0


def test_scale_one_is_pixels_batch(ctx, corpus):  # noqa: F811
    from test_gpu_pixels_batch import _c_batch
    names = sorted(corpus)
    datas = [corpus[n] for n in names]
    for opt in ("q3", "q6"):
        _, flags, niter = OPTS[opt]
        for layout, on_device in ((0, 1), (1, 0)):
            assert _c_scaled(ctx, datas, flags, niter, layout, 1, on_device) == \
                _c_batch(ctx, datas, flags, niter, layout, on_device), (opt, layout)


@pytest.mark.parametrize("d", SCALES)
def test_splits_and_order_change_nothing(ctx, corpus, d):  # noqa: F811
    names = sorted(corpus)
    _, flags, niter = OPTS["q6"]
    singles = {n: _c_scaled(ctx, [corpus[n]], flags, niter, 0, d, 1)[0] for n in names}
    for budget, on_device in ((1, 1), (3 << 20, 0)):
        got = _c_scaled(ctx, [corpus[n] for n in names], flags, niter, 0, d, on_device, budget)
        for n, g in zip(names, got):
            assert g == singles[n], (n, budget, on_device)
    perm = list(np.random.RandomState(d).permutation(len(names)))
    got = _c_scaled(ctx, [corpus[names[i]] for i in perm], flags, niter, 0, d, 1)
    for i, g in zip(perm, got):
        assert g == singles[names[i]], names[i]


@pytest.mark.parametrize("layout", [0, 1])
def test_grey_files_at_odd_offsets(ctx, corpus, reference, layout):  # noqa: F811
    names = ["tinyprog", "base444", "gray", "tinyprog", "base420", "gray"]
    _, flags, niter = OPTS["q6"]
    for d in SCALES:
        got = _c_scaled(ctx, [corpus[n] for n in names], flags, niter, layout, d, 1)
        for n, (rc, pix, res) in zip(names, got):
            assert rc == 0 and np.array_equal(_hwc(pix, corpus[n], layout, d), reference(n, "q6", d)), (n, d)


def test_python_call(ctx, corpus, reference):  # noqa: F811
    _, flags, niter = OPTS["q6"]
    names = ["base420", "gray", "prog420", "garbled"]
    datas = [corpus[n] for n in names]
    full = ctx.decode_pixels(datas, flags | qs.JPEGQS_TRANSCODE, niter)
    for d in SCALES:
        for layout in ("hwc", "chw"):
            dev = ctx.decode_pixels(datas, flags | qs.JPEGQS_TRANSCODE, niter, layout=layout, scale_denom=d)
            cpu = qs.decode_pixels(datas, flags | qs.JPEGQS_TRANSCODE, niter, layout=layout, device="cpu", gpu=0,
                                   scale_denom=d)
            for n, a, b, f in zip(names, dev, cpu, full):
                want = reference(n, "q6", d)
                got = a[0].cpu().numpy()
                assert np.array_equal(got if layout == "hwc" else got.transpose(1, 2, 0), want), (n, d, layout)
                assert torch.equal(a[0].cpu(), b[0]) and a[1:] == b[1:] == f[1:], n
    with pytest.raises(ValueError, match="scale_denom"):
        ctx.decode_pixels(datas, flags, niter, scale_denom=3)


# ---- render_scaled_async after run_async ---------------------------------------------------------

def _images():
    return [hc.make_image(208, 144, "420", hc.TABLES["k50"], "saturated", seed=9),   # up-samples at q6
            hc.make_image(203, 149, "422", hc.TABLES["k90"], "synth", seed=2),
            hc.make_image(97, 61, "gray", hc.TABLES["rand"], "saturated", seed=4),
            hc.make_image(1000, 700, "420", hc.TABLES["k10"], "synth", seed=5)]


def _run_result(work, coefs, status, ups, n):
    """(image, upsampled pair or None) as the device holds image n after the run"""
    o = work[n].clone()
    for c, t in zip(o.comps, coefs[n]):
        c.coef = t.cpu().numpy()
    up = None
    if int(status[n, 1].item()):
        up = tuple(u.cpu().numpy() for u in ups[n])
    return o, up


@pytest.mark.parametrize("layout", ["hwc", "chw"])
def test_render_after_run_is_render_model(ctx, layout):  # noqa: F811
    ims = _images()
    work = [im.clone() for im in ims]
    coefs = [[torch.from_numpy(np.ascontiguousarray(c.coef)).cuda() for c in im.comps] for im in work]
    status, ups = ctx.run_async(work, coefs, 7, 2)
    for d in (1,) + SCALES:
        out = ctx.render_async(work, coefs, status, ups, layout=layout, scale_denom=d)
        torch.cuda.synchronize()
        assert int(status[0, 1].item()) == 1 and int(status[2, 1].item()) == 0
        for n in range(len(ims)):
            im, up = _run_result(work, coefs, status, ups, n)
            assert np.array_equal(out[n].cpu().numpy(), cuda.render_model(im, up, layout, d)), (n, d)


def test_render_scaled_in_a_graph(ctx):  # noqa: F811
    ims = _images()[:2]
    work = [im.clone() for im in ims]
    static = [[torch.from_numpy(np.ascontiguousarray(c.coef)).cuda() for c in im.comps] for im in work]
    outs = {d: [torch.empty((-(-im.height // d), -(-im.width // d), 3), dtype=torch.uint8, device="cuda") for im in ims]
            for d in SCALES}
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        status, ups = ctx.run_async(work, static, 7, 2)
        for d in SCALES:
            ctx.render_async(work, static, status, ups, out=outs[d], scale_denom=d)
    for seed in (0, 1):
        # new coefficients under the tables fixed at capture
        inputs = ims if seed == 0 else [hc.make_image(im.width, im.height, ss, hc.TABLES[t], "synth", seed=31)
                                        for im, ss, t in zip(ims, ("420", "422"), ("k50", "k90"))]
        for ts, im in zip(static, inputs):
            for t, c in zip(ts, im.comps):
                t.copy_(torch.from_numpy(c.coef))
        g.replay()
        torch.cuda.synchronize()
        # the coefficients the replay smoothed, rendered on the host from the original inputs' run
        ref = [im.clone() for im in inputs]
        rc = [[torch.from_numpy(np.ascontiguousarray(c.coef)).cuda() for c in im.comps] for im in ref]
        rst, rups = ctx.run_async(ref, rc, 7, 2)
        torch.cuda.synchronize()
        for n in range(len(ims)):
            im, up = _run_result(ref, rc, rst, rups, n)
            for d in SCALES:
                assert np.array_equal(outs[d][n].cpu().numpy(), cuda.render_model(im, up, "hwc", d)), (seed, n, d)


def test_render_rejects_bad_scale_with_nothing_enqueued(ctx):  # noqa: F811
    im = _images()[1]
    coefs = [[torch.from_numpy(np.ascontiguousarray(c.coef)).cuda() for c in im.comps]]
    out = torch.zeros(im.height * im.width * 3, dtype=torch.uint8, device="cuda")
    arr = cuda._image_array([im], [[t.data_ptr() for t in coefs[0]]])
    torch.cuda.synchronize()
    for d in (0, 3, 16):
        assert ctx.lib.jpegqs_cuda_render_scaled_async(ctx.h, 1, arr, None, 0, d,
                                                       (C.c_void_p * 1)(out.data_ptr()), None) == -2
        assert "scale_denom" in ctx.lib.jpegqs_cuda_last_error(ctx.h).decode()
    torch.cuda.synchronize()
    assert not out.any()
