"""The stream-ordered render (jpegqs_cuda_render_async / QsContext.render_async) against libjpeg.

The reference pixels are always computed without the GPU: the oracle's coefficients
(ol.run_oracle with the up-sampling flag), or the untouched coefficients for a plain decode,
decoded by libjpeg-turbo through tests/libjpeg_pixels.py.  The cases cover every sampling (4:1:1
from render_images.py: box replication) with synthetic and saturated content at ragged sizes, plain decodes
and results of run_async, both layouts, render_rgb on the same coefficients, untouched inputs, a
batch in which the device decides per image where the chroma comes from, one CUDA graph holding
run_async and the render, the stream rules, scale, and argument errors that change nothing.
"""
import gc

import numpy as np
import pytest

import hard_content as hc
import libjpeg_pixels as lp
import oracle_lib as ol
from jpegqs_b200.cuda import QsContext, _image_array
from render_images import SAMPLINGS, make

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(lp.JPEG_SO is None, reason="no libjpeg inside Pillow")]

FLAG_SETS = [None, 0, 3, 7, 8, 33]          # None: the still-quantized input (a plain decode)
# (203, 149): several tiles, no dimension a multiple of the MCU; (4, 21): chroma 1-2 samples wide,
# so the fancy up-sampler falls back to replication
SIZES = [(203, 149), (4, 21)]
NITER = 1


@pytest.fixture(scope="module")
def torch():
    import torch as t
    return t


@pytest.fixture(scope="module")
def ctx():
    c = QsContext(0)
    yield c
    c.close()


def _to_device(torch, images):
    return [[torch.from_numpy(np.ascontiguousarray(c.coef)).cuda() for c in im.comps] for im in images]


def want_pixels(im, flags, niter=NITER):
    """libjpeg's pixels for what the oracle makes of im (flags None: im as it is)."""
    if flags is None:
        return lp.decode(im)
    return lp.decode(ol.run_oracle(im, flags, niter, threads=0, with_upsampled=True)[1])


def smooth(torch, ctx, images, flags, niter=NITER, stream=None):
    """Device copies of the images, smoothed by run_async unless flags is None.  Returns the
    work images (quant tables as run_async left them), coefficient tensors, status and up."""
    work = [im.clone() for im in images]
    coefs = _to_device(torch, work)
    status, ups = None, None
    if flags is not None:
        status, ups = ctx.run_async(work, coefs, flags, niter, stream=stream)
    return work, coefs, status, ups


def _host_result(work, coefs, status, ups, n):
    """Image n as the coefficients on the device say (for render_rgb)."""
    o = work[n].clone()
    for c, t in zip(o.comps, coefs[n]):
        c.coef = t.cpu().numpy()
    if status is not None and int(status[n, 1].item()):
        for j in (1, 2):
            o.comps[j].coef = ups[n][j - 1].cpu().numpy()
        for c in o.comps:
            c.h_samp = c.v_samp = 1
    return o


# ---- 1-3. samplings x inputs, both layouts, render_rgb, untouched inputs ----------------------

@pytest.mark.parametrize("flags", FLAG_SETS)
@pytest.mark.parametrize("ss", SAMPLINGS)
def test_pixels_are_libjpegs(torch, ctx, ss, flags):
    for content in ("synth", "saturated"):
        for k, (w, h) in enumerate(SIZES):
            table = ("k50", "k10", "rand", "k90")[(k + len(ss) + (flags or 0)) % 4]
            im = make(w, h, ss, table, content, seed=3 * k + (flags or 0))
            work, coefs, status, ups = smooth(torch, ctx, [im], flags)
            torch.cuda.synchronize()
            before = [t.clone() for t in coefs[0] + (list(ups[0]) if ups and ups[0] else [])]
            hwc = ctx.render_async(work, coefs, status, ups)[0]
            chw = ctx.render_async(work, coefs, status, ups, layout="chw")[0]
            torch.cuda.synchronize()
            what = (ss, flags, content, w, h)
            assert np.array_equal(hwc.cpu().numpy(), want_pixels(im, flags)), what
            assert torch.equal(chw, hwc.permute(2, 0, 1)), what
            after = coefs[0] + (list(ups[0]) if ups and ups[0] else [])
            assert all(torch.equal(a, b) for a, b in zip(before, after)), f"{what}: inputs changed"
            assert np.array_equal(ctx.render_rgb(_host_result(work, coefs, status, ups, 0)), hwc.cpu().numpy()), what


# ---- 4. the chroma source decided per image on the device ------------------------------------

def _mixed_batch():
    base = hc.make_image(208, 144, "420", hc.TABLES["k50"], "saturated", seed=9)
    big_quant = base.clone()
    big_quant.comps[1].quant = big_quant.comps[1].quant.copy()
    big_quant.comps[1].quant[5] = 0x800
    return [base,                                                         # up-samples
            hc.make_image(200, 120, "444", hc.TABLES["k90"], "synth", seed=2),   # cannot up-sample
            big_quant,                                                    # stopped by the host
            hc.with_dequant_edge(base, True, comp=0),                     # stopped on the device
            hc.make_image(96, 80, "gray", hc.TABLES["rand"], "saturated", seed=4),
            hc.make_image(203, 149, "420", hc.TABLES["k10"], "synth", seed=5)]    # given no coef_up


def test_device_chooses_the_chroma_source_per_image(torch, ctx):
    ims = _mixed_batch()
    work, coefs, status, ups = smooth(torch, ctx, ims, 7, niter=2)
    ups = list(ups)
    ups[5] = None
    st = status.cpu().numpy()
    assert [int(v) for v in st[:, 0]] == [0, 0, 1, 1, 0, 0]
    assert [int(v) for v in st[:, 1]] == [1, 0, 0, 0, 0, 1]
    got = ctx.render_async(work, coefs, status, ups)
    for n, im in enumerate(ims):
        if n == 2:
            # the quant value 0x800 leaves component 1 de-quantized with it (values up to 10240): AC
            # values beyond the 10 bits libjpeg can code, so libjpeg has no pixels for this set.
            # render_rgb, the defined arithmetic, on the same coefficients stands in; they are the
            # oracle's coefficients
            oracle = ol.run_oracle(im, 7, 2, threads=0)[1]
            with pytest.raises(lp.LibjpegError, match="out of range"):
                lp.decode(oracle)
            host = _host_result(work, coefs, status, ups, n)
            assert ol.images_equal(host, oracle)
            want = ctx.render_rgb(host)
        elif n == 5:        # without coef_up the render reads coef: the chroma as run_async left it there
            want = lp.decode(_host_result(work, coefs, None, None, n))
        else:
            want = want_pixels(im, 7, 2)
        assert np.array_equal(got[n].cpu().numpy(), want), n
    # status_dev NULL: the host flags (what run_device / run_batch report) decide instead
    host = [bool(v) for v in st[:, 1]]
    host[5] = False
    got2 = ctx.render_async(work, coefs, host, ups)
    for a, b in zip(got, got2):
        assert torch.equal(a, b)


def test_eager_pipeline_on_the_default_stream(torch, ctx):
    """run_async then render_async on torch's default stream, with no synchronisation between
    them and the stream held busy first: the render must see the smoothed coefficients and the
    status."""
    ims = [hc.make_image(208, 144, "420", hc.TABLES["k50"], "saturated", seed=21),
           hc.with_dequant_edge(hc.make_image(176, 136, "420", hc.TABLES["k50"], "synth", seed=22), True, comp=0)]
    work = [im.clone() for im in ims]
    pristine = _to_device(torch, work)
    coefs = [[torch.zeros_like(t) for t in ts] for ts in pristine]
    torch.cuda.synchronize()
    assert torch.cuda.current_stream().cuda_stream == 0
    torch.cuda._sleep(100_000_000)
    for ts, ps in zip(coefs, pristine):                  # the input arrives behind the spin
        for t, p in zip(ts, ps):
            t.copy_(p)
    status, ups = ctx.run_async(work, coefs, 7, 2)
    out = ctx.render_async(work, coefs, status, ups)
    assert [int(v) for v in status[:, 1].cpu()] == [1, 0]
    for o, im in zip(out, ims):
        assert np.array_equal(o.cpu().numpy(), want_pixels(im, 7, 2))


# ---- 5. one CUDA graph: run_async + render_async ---------------------------------------------

def test_graph_replays_follow_the_device_status(torch, ctx):
    tables = hc.TABLES["k50"]
    first = [hc.make_image(208, 160, "420", tables, "synth", seed=11),
             hc.make_image(176, 136, "420", tables, "saturated", seed=12)]
    second = [im.clone() for im in first]
    y = second[1].comps[0]
    y.coef = y.coef.copy()
    y.coef[3, 4, 1] = int(2048 // int(y.quant[1])) + 1          # de-quantizes past 2047: stop
    work = [im.clone() for im in first]
    static = _to_device(torch, work)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        status, ups = ctx.run_async(work, static, 7, 2)
        out = ctx.render_async(work, static, status, ups)
    flags_seen = []
    for inputs in (first, second, first):
        for ts, im in zip(static, inputs):
            for t, c in zip(ts, im.comps):
                t.copy_(torch.from_numpy(c.coef))
        g.replay()
        torch.cuda.synchronize()
        flags_seen.append([int(v) for v in status[:, 1].cpu()])
        for o, im in zip(out, inputs):
            assert np.array_equal(o.cpu().numpy(), want_pixels(im, 7, 2))
    assert flags_seen == [[1, 1], [1, 0], [1, 1]]


# ---- 6. stream behaviour ---------------------------------------------------------------------

def test_call_does_not_wait_for_the_stream(torch, ctx):
    im = hc.make_image(416, 288, "420", hc.TABLES["k50"], "synth", seed=4)
    coefs = _to_device(torch, [im])
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(200_000_000)                     # ~100 ms of spinning that ends by itself
        out = ctx.render_async([im], coefs)
    busy = not s.query()
    s.synchronize()
    assert busy, "render_async returned only after the stream had drained"
    assert np.array_equal(out[0].cpu().numpy(), lp.decode(im))


def test_host_structs_released_at_return(torch, ctx):
    ims = [hc.make_image(240, 160, "444", hc.TABLES["rand"], "synth", seed=2),
           hc.make_image(200, 120, "422", hc.TABLES["k10"], "saturated", seed=3)]
    work = [im.clone() for im in ims]
    coefs = _to_device(torch, work)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(50_000_000)                      # the kernel starts after the host has moved on
        out = ctx.render_async(work, coefs)
    for im in work:
        for c in im.comps:
            c.quant[...] = 3                               # the caller's quant tables, overwritten
    del work
    gc.collect()
    junk = [np.full(1 << 16, 0x7f7f, np.uint16) for _ in range(64)]
    s.synchronize()
    del junk
    for o, im in zip(out, ims):
        assert np.array_equal(o.cpu().numpy(), lp.decode(im))


def test_calls_in_flight_on_two_streams(torch, ctx):
    a = [hc.make_image(416, 288, "420", hc.TABLES["k50"], "saturated", seed=1)]
    b = [hc.make_image(304, 240, "422", hc.TABLES["k90"], "synth", seed=2)]
    c = [hc.make_image(256, 200, "gray", hc.TABLES["k10"], "saturated", seed=3)]
    ca, cb, cc = _to_device(torch, a), _to_device(torch, b), _to_device(torch, c)
    wc = [im.clone() for im in c]
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    with torch.cuda.stream(s1):
        torch.cuda._sleep(20_000_000)
    # two renders on two streams, then a run_async on one stream with a render on the other
    oa = ctx.render_async(a, ca, stream=s1)
    ob = ctx.render_async(b, cb, stream=s2)
    status, ups = ctx.run_async(wc, cc, 3, 2, stream=s1)
    ob2 = ctx.render_async(b, cb, layout="chw", stream=s2)
    torch.cuda.synchronize()
    assert np.array_equal(oa[0].cpu().numpy(), lp.decode(a[0]))
    assert np.array_equal(ob[0].cpu().numpy(), lp.decode(b[0]))
    assert torch.equal(ob2[0], ob[0].permute(2, 0, 1))
    assert np.array_equal(ctx.render_async(wc, cc, status, ups)[0].cpu().numpy(), want_pixels(c[0], 3, 2))


# ---- 7. scale --------------------------------------------------------------------------------

def test_8k_420(torch, ctx):
    im = hc.make_image(7680, 4320, "420", hc.TABLES["k50"], "saturated", seed=8)
    coefs = _to_device(torch, [im])
    out = ctx.render_async([im], coefs)
    assert np.array_equal(out[0].cpu().numpy(), lp.decode(im))


def test_batch_of_several_launches(torch, ctx):
    ims = [make(24 + 8 * (k % 5), 16 + 4 * (k % 3), SAMPLINGS[k % len(SAMPLINGS)], "k50",
                ("synth", "saturated")[k % 2], seed=k) for k in range(150)]
    coefs = _to_device(torch, ims)
    out = ctx.render_async(ims, coefs)
    assert ctx.last_launches == 3                          # 60 images per launch
    for o, im in zip(out, ims):
        assert np.array_equal(o.cpu().numpy(), lp.decode(im))


@pytest.mark.parametrize("layout", ["hwc", "chw"])
def test_outputs_at_odd_byte_offsets(torch, ctx, layout):
    ims = [make(w, h, ss, "k90", "saturated", seed=w) for w, h, ss in
           [(203, 149, "420"), (37, 13, "444"), (130, 70, "gray"), (64, 33, "411")]]
    coefs = _to_device(torch, ims)
    sizes = [im.width * im.height * 3 for im in ims]
    offs, o = [], 1
    for n in sizes:
        offs.append(o)
        o += n + 3
    flat = torch.full((o + 5,), 0xA5, dtype=torch.uint8, device="cuda")
    views = [flat[a:a + n].view(*((im.height, im.width, 3) if layout == "hwc" else (3, im.height, im.width)))
             for a, n, im in zip(offs, sizes, ims)]
    assert all(v.data_ptr() % 4 for v in views[:1])
    ctx.render_async(ims, coefs, layout=layout, out=views)
    torch.cuda.synchronize()
    for v, im in zip(views, ims):
        got = v.cpu().numpy()
        assert np.array_equal(got if layout == "hwc" else got.transpose(1, 2, 0), lp.decode(im))
    mask = torch.ones_like(flat, dtype=torch.bool)
    for a, n in zip(offs, sizes):
        mask[a:a + n] = False
    assert bool((flat[mask] == 0xA5).all()), "bytes outside the outputs were written"


def test_batched_tensor_unbind(torch, ctx):
    ims = [hc.make_image(120, 88, "420", hc.TABLES["k50"], "synth", seed=k) for k in range(4)]
    coefs = _to_device(torch, ims)
    batch = torch.empty((4, 88, 120, 3), dtype=torch.uint8, device="cuda")
    ctx.render_async(ims, coefs, out=batch.unbind(0))
    for k, im in enumerate(ims):
        assert np.array_equal(batch[k].cpu().numpy(), lp.decode(im))


# ---- 8. argument errors ----------------------------------------------------------------------

def test_argument_errors_change_nothing(torch, ctx):
    im = hc.make_image(208, 144, "420", hc.TABLES["k50"], "saturated", seed=8)
    coefs = _to_device(torch, [im])[0]
    out = torch.full((im.height, im.width, 3), 0x5A, dtype=torch.uint8, device="cuda")
    status = torch.zeros((1, 2), dtype=torch.int32, device="cuda")
    before = [t.clone() for t in coefs + [out]]
    lib = ctx.lib
    import ctypes as C

    def image():
        return _image_array([im], [[t.data_ptr() for t in coefs]], [])

    def call(arr, outs=None, layout=0):
        outs = (C.c_void_p * 1)(out.data_ptr()) if outs is None else outs
        return lib.jpegqs_cuda_render_async(ctx.h, 1, arr, status.data_ptr(), layout, outs, None)

    assert call(image(), outs=None, layout=0) == 0                             # the arguments as they are run
    torch.cuda.synchronize()
    ref = out.clone()
    out.fill_(0x5A)
    before[-1] = out.clone()
    assert lib.jpegqs_cuda_render_async(ctx.h, 1, image(), None, 0, None, None) == -2      # out_dev NULL
    assert call(image(), outs=(C.c_void_p * 1)(None)) == -2                                 # an entry NULL
    arr = image(); arr[0].comp[1].coef = None
    assert call(arr) == -2                                                                  # coef NULL
    arr = image(); arr[0].comp[0].coef = coefs[0].data_ptr() + 2
    assert call(arr) == -2                                                                  # coef misaligned
    arr = image(); arr[0].comp[1].coef_up = coefs[0].data_ptr() + 8; arr[0].comp[2].coef_up = coefs[0].data_ptr()
    assert call(arr) == -2                                                                  # coef_up misaligned
    arr = image(); arr[0].comp[2].h_samp = 5
    assert call(arr) == -2                                                                  # sampling 5
    arr = image(); arr[0].comp[2].v_samp = 0
    assert call(arr) == -2                                                                  # sampling 0
    arr = image(); arr[0].comp[1].wblk -= 1
    assert call(arr) == -2                                                                  # blocks short of cw
    arr = image(); arr[0].comp[0].hblk -= 1
    assert call(arr) == -2                                                                  # blocks short of ch
    assert call(image(), layout=2) == -2                                                    # unknown layout
    arr = image(); arr[0].ncomp = 2
    assert call(arr) == -3                                                                  # two components
    torch.cuda.synchronize()
    for a, b in zip(before, coefs + [out]):
        assert torch.equal(a, b)
    assert np.array_equal(ref.cpu().numpy(), lp.decode(im))
