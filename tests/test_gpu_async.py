"""The stream-ordered entry point (jpegqs_cuda_run_async / QsContext.run_async) against the oracle.

Every case compares coefficients, the device-side status (stop, upsampled), the up-sampled
chroma where the status says so, and the quant tables with ol.run_oracle on each image alone.
The cases cover flag sets x samplings on small images, wave-scale launches (the smoothing
launches are run_batch's on device buffers), the reference's `stop` decided on the device per
image, that the call neither waits nor reads host memory after it returns, two calls in flight
on one context, CUDA-graph replays, and argument errors that must leave everything untouched.
"""
import ctypes as C
import gc

import numpy as np
import pytest

import jpegqs_b200 as qs
import oracle_lib as ol
import hard_content as hc
import wave_geometry as wg
from jpegqs_b200.cuda import QsContext, _image_array

pytestmark = pytest.mark.gpu

FLAG_SETS = [0, 1, 3, 7, 16, 33, 8]


@pytest.fixture(scope="module")
def torch():
    import torch as t
    return t


@pytest.fixture(scope="module")
def sms(torch):
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def ctx():
    c = QsContext(0)
    yield c
    c.close()


def _to_device(torch, images):
    return [[torch.from_numpy(np.ascontiguousarray(c.coef)).cuda() for c in im.comps] for im in images]


def _results(images, coefs, status, ups):
    """(stop, image as the oracle reports it, upsampled) per image, after the stream is done."""
    st = status.cpu().numpy()
    out = []
    for n, im in enumerate(images):
        o = im.clone()
        for c, t in zip(o.comps, coefs[n]):
            c.coef = t.cpu().numpy()
        if st[n, 1]:
            for j in (1, 2):
                o.comps[j].coef = ups[n][j - 1].cpu().numpy()
            for c in o.comps:
                c.h_samp = c.v_samp = 1
        out.append((int(st[n, 0]), o, bool(st[n, 1])))
    return out


def run_async(torch, ctx, images, flags, niter, stream=None):
    """run_async on device copies of the images; images are cloned (run_async sets their
    quant tables to ones).  Returns what _results returns."""
    work = [im.clone() for im in images]
    coefs = _to_device(torch, work)
    torch.cuda.synchronize()
    status, ups = ctx.run_async(work, coefs, flags, niter, stream=stream)
    torch.cuda.synchronize()
    return _results(work, coefs, status, ups)


def _oracle(im, flags, niter):
    return ol.run_oracle(im, flags, niter, threads=0, with_upsampled=True)


def _check(got, want):
    (ret, out, ups), (oret, oout, oups) = got, want
    assert ret == oret
    assert ups == oups
    nd = ol.diff_count(out, oout)
    assert nd == 0, f"{nd} coefficients differ from the oracle"
    assert ol.images_equal(out, oout)


# ---- 1. flag sets x samplings, small images ---------------------------------------------------

@pytest.mark.parametrize("niter", [0, 1, 3])
@pytest.mark.parametrize("flags", FLAG_SETS)
def test_small_images(torch, ctx, flags, niter):
    for content in ("synth", "saturated"):
        for k, ss in enumerate(hc.SAMPLINGS):
            table = list(hc.TABLES)[(k + flags + niter) % len(hc.TABLES)]
            w, h = (208 + 16 * k, 144 + 8 * k) if not (flags & 4) else (208, 144 + 8 * k)
            im = hc.make_image(w, h, ss, hc.TABLES[table], content, seed=k + 100 * flags + niter)
            (got,) = run_async(torch, ctx, [im], flags, niter)
            _check(got, _oracle(im, flags, niter))


# ---- 2. wave scale ----------------------------------------------------------------------------
# The smoothing launches of run_async are those of run_batch on device buffers: the same job
# lists per pass; only the out-of-range flags they point at differ.
ROUTE = "batch_device"


def _wave_tiles(sms):
    return sms * wg.CTA_WARPS


def _size_420(flags, niter, tables, sms):
    """The first 4:2:0 size whose launches reach dynamic rounds plus a tail at 1.2-2.5 waves."""
    for w in (2048, 2560, 3072):
        h = 16
        while True:
            h += 16
            ls = wg.smooth_launches(wg.geometry(w, h, "420", tables), flags, niter, ROUTE, sms)
            big = max(l.tiles for l in ls)
            if big > 2.5 * _wave_tiles(sms):
                break
            if "dynamic+tail" in wg.regimes(ls) and big >= 1.2 * _wave_tiles(sms):
                return w, h
    raise AssertionError("no 4:2:0 size at wave scale")


@pytest.mark.parametrize("flags,table", [(0, "k50"), (7, "diag"), (1, "rand")])
def test_420_image_at_wave_scale(torch, ctx, sms, flags, table):
    tables = hc.TABLES[table]
    w, h = _size_420(flags, 2, tables, sms)
    im = hc.make_image(w, h, "420", tables, "saturated", seed=w + h)
    ls = wg.smooth_launches(im, flags, 2, ROUTE, sms)
    assert "dynamic+tail" in wg.regimes(ls) and 1.2 * _wave_tiles(sms) <= max(l.tiles for l in ls) <= 2.5 * _wave_tiles(sms)
    (got,) = run_async(torch, ctx, [im], flags, 2)
    _check(got, _oracle(im, flags, 2))


BATCH = [("420", "k50", "saturated", 1.0), ("444", "rand", "synth", 0.5), ("gray", "diag", "saturated", 0.75),
         ("422", "k90", "saturated", 0.6), ("440", "flat", "synth", 0.45), ("420", "k10", "synth", 0.35)]


def _batch_sizes(flags, niter, sms):
    for step in range(1, 400):
        geo = [(1024 + 8 * k, int(step * 16 * rel) + 16) for k, (_, _, _, rel) in enumerate(BATCH)]
        ims = [wg.geometry(w, h, ss, hc.TABLES[t]) for (w, h), (ss, t, _, _) in zip(geo, BATCH)]
        ls = wg.smooth_launches(ims, flags, niter, ROUTE, sms)
        big = max(l.tiles for l in ls)
        if big > 2.5 * _wave_tiles(sms):
            break
        if {"mixed", "dynamic+tail"} <= wg.regimes(ls) and big >= 1.2 * _wave_tiles(sms):
            return geo
    raise AssertionError("no batch size reaches mixed dynamic group tiles")


@pytest.mark.parametrize("flags", [0, 3])
def test_heterogeneous_batch_at_wave_scale(torch, ctx, sms, flags):
    geo = _batch_sizes(flags, 2, sms)
    ims = [hc.make_image(w, h, ss, hc.TABLES[t], content, seed=17 * k)
           for k, ((w, h), (ss, t, content, _)) in enumerate(zip(geo, BATCH))]
    ls = wg.smooth_launches(ims, flags, 2, ROUTE, sms)
    assert {"mixed", "dynamic+tail"} <= wg.regimes(ls)
    for im, got in zip(ims, run_async(torch, ctx, ims, flags, 2)):
        _check(got, _oracle(im, flags, 2))


def test_batch_larger_than_one_launch(torch, ctx):
    """More than 1024 components: sub-batches one after another on the stream."""
    ims = [hc.make_image(32 + 16 * (k % 3), 32, "420", hc.TABLES["k50"], "saturated", seed=k) for k in range(350)]
    ims[200] = hc.with_dequant_edge(ims[200], True, comp=0)
    got = run_async(torch, ctx, ims, 3, 2)
    assert got[200][0] == 1
    for im, g in zip(ims, got):
        _check(g, _oracle(im, 3, 2))


# ---- 3. stop decided on the device, per image -------------------------------------------------

def _stop_batch():
    base = hc.make_image(208, 144, "420", hc.TABLES["k50"], "saturated", seed=9)
    big_quant = base.clone()
    big_quant.comps[1].quant = big_quant.comps[1].quant.copy()
    big_quant.comps[1].quant[5] = 0x800
    return [hc.with_dequant_edge(base, False, comp=0),       # 2047 and -2048: goes on
            hc.with_dequant_edge(base, True, comp=0),        # 2048 in luma
            hc.with_dequant_edge(base, True, comp=2),        # 2048 in Cr
            big_quant]                                       # a quant value >= 0x800


@pytest.mark.parametrize("flags", [3, 7])
def test_stop_per_image(torch, ctx, flags):
    ims = _stop_batch()
    got = run_async(torch, ctx, ims, flags, 3)
    assert [g[0] for g in got] == [0, 1, 1, 1]
    if flags & 4:
        assert [g[2] for g in got] == [True, False, False, False]
    for im, g in zip(ims, got):
        _check(g, _oracle(im, flags, 3))


# ---- 4. no host wait --------------------------------------------------------------------------

def test_call_does_not_wait_for_the_stream(torch, ctx):
    im = hc.make_image(416, 288, "420", hc.TABLES["k50"], "synth", seed=4)
    work = im.clone()
    coefs = _to_device(torch, [work])
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(200_000_000)                     # ~100 ms of spinning (at ~2 GHz) that ends by itself
        status, ups = ctx.run_async([work], coefs, 7, 3)
    busy = not s.query()
    s.synchronize()
    assert busy, "run_async returned only after the stream had drained"
    _check(_results([work], coefs, status, ups)[0], _oracle(im, 7, 3))


# ---- 5. host inputs released at return --------------------------------------------------------

def test_host_inputs_released_at_return(torch, ctx):
    ims = _stop_batch()[:2] + [hc.make_image(240, 160, "444", hc.TABLES["rand"], "synth", seed=2)]
    work = [im.clone() for im in ims]
    coefs = _to_device(torch, work)
    tables = [c.quant for im in work for c in im.comps]
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(50_000_000)                      # the kernels start after the host has moved on
        status, ups = ctx.run_async(work, coefs, 3, 2)
    for q in tables:
        q[...] = 3                                         # the caller's quant tables, overwritten
    del tables
    gc.collect()
    junk = [np.full(1 << 16, 0x7f7f, np.uint16) for _ in range(64)]   # reuse of freed host memory
    s.synchronize()
    del junk
    for n, im in enumerate(ims):
        got = _results(work, coefs, status, ups)[n]
        want = _oracle(im, 3, 2)
        assert got[0] == want[0] and ol.diff_count(got[1], want[1]) == 0


# ---- 6. two calls in flight on one context ----------------------------------------------------

def test_two_calls_in_flight(torch, ctx):
    a = [hc.make_image(416, 288, "420", hc.TABLES["k50"], "saturated", seed=1), _stop_batch()[2]]
    b = [hc.make_image(304, 240, "422", hc.TABLES["diag"], "synth", seed=2),
         hc.make_image(256, 200, "gray", hc.TABLES["k90"], "saturated", seed=3)]
    wa, wb = [im.clone() for im in a], [im.clone() for im in b]
    ca, cb = _to_device(torch, wa), _to_device(torch, wb)
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    with torch.cuda.stream(s1):
        torch.cuda._sleep(20_000_000)
    sa, ua = ctx.run_async(wa, ca, 7, 3, stream=s1)
    sb, ub = ctx.run_async(wb, cb, 1 | 16, 2, stream=s2)
    torch.cuda.synchronize()
    for im, g in zip(a, _results(wa, ca, sa, ua)):
        _check(g, _oracle(im, 7, 3))
    for im, g in zip(b, _results(wb, cb, sb, ub)):
        _check(g, _oracle(im, 1 | 16, 2))


# ---- 7. CUDA graph ----------------------------------------------------------------------------

def _contents():
    """Three contents of one geometry and one pair of quant tables; the third stops the run."""
    tables = hc.TABLES["k50"]
    a = hc.make_image(208, 160, "420", tables, "synth", seed=11)
    b = hc.make_image(208, 160, "420", tables, "saturated", seed=12)
    c = a.clone()
    y = c.comps[0]
    y.coef = y.coef.copy()
    y.coef[3, 4, 1] = int(2048 // int(y.quant[1])) + 1      # de-quantizes past 2047: stop
    return [a, b, c]


@pytest.mark.parametrize("flags", [3, 7])
def test_graph_replays(torch, ctx, flags):
    contents = _contents()
    work = contents[0].clone()
    static = _to_device(torch, [work])
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        status, ups = ctx.run_async([work], static, flags, 3)
    stops = []
    for im in [contents[1], contents[2], contents[0]]:
        for t, c in zip(static[0], im.comps):
            t.copy_(torch.from_numpy(c.coef))
        g.replay()
        torch.cuda.synchronize()
        got = _results([work], static, status, ups)[0]
        want = _oracle(im, flags, 3)
        stops.append(got[0])
        _check(got, want)
    assert stops == [0, 1, 0]


# ---- 8. argument errors -----------------------------------------------------------------------

def test_argument_errors_change_nothing(torch, ctx):
    im = hc.make_image(208, 144, "420", hc.TABLES["k50"], "saturated", seed=8)
    coefs = _to_device(torch, [im])[0]
    y = im.comps[0]
    ups = [torch.zeros((y.hblk, y.wblk, 64), dtype=torch.int16, device="cuda") for _ in range(2)]
    need = qs.async_workspace_bytes([im], 7)
    ws = torch.zeros(need + 512, dtype=torch.uint8, device="cuda")
    status = torch.full((1, 2), -7, dtype=torch.int32, device="cuda")
    before = [t.clone() for t in coefs + ups + [ws, status]]
    lib = ctx.lib

    def call(arr, ws_ptr, ws_bytes, st_ptr):
        return lib.jpegqs_cuda_run_async(ctx.h, 1, arr, 7, 3, ws_ptr, ws_bytes, st_ptr, None)

    def image():
        return _image_array([im], [[t.data_ptr() for t in coefs]], [[None] + [u.data_ptr() for u in ups]])

    base = ws.data_ptr()
    assert base % 256 == 0
    assert call(image(), base, need - 1, status.data_ptr()) == -2              # one byte short
    assert call(image(), base + 1, need, status.data_ptr()) == -2              # misaligned
    assert call(image(), base, need, None) == -2                               # NULL status
    arr = image()
    arr[0].ncomp = 11
    assert call(arr, base, need, status.data_ptr()) == -2                      # ncomp 11
    arr = image()
    arr[0].comp[2].coef_up = None
    assert call(arr, base, need, status.data_ptr()) == -2                      # UPSAMPLE_UV without coef_up
    torch.cuda.synchronize()
    for a, b in zip(before, coefs + ups + [ws, status]):
        assert torch.equal(a, b)
    # the same arguments, put right, run
    assert call(image(), base, need, status.data_ptr()) == 0
    torch.cuda.synchronize()
    assert status[0, 0].item() == _oracle(im, 7, 3)[0]
