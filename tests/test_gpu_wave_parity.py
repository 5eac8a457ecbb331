"""Parity with the oracle at wave scale, on content that needs clamping.

The smoothing kernel's tile schedule has a dynamic phase (group tiles taken by atomics, with
the switch to the table-independent schedule when a group's warps sit in jobs with different
chunk schedules) and a static tail.  A launch reaches the dynamic phase only from about one
wave of tiles (16 warps x 32 blocks per SM) up, so small images run the tail only.  Every case
here is sized from the device's SM count, first asserts the regime it was built for
(tests/wave_geometry.py):

  (i)   dynamic rounds plus a ragged tail      - "dynamic+tail"
  (ii)  whole dynamic rounds, no tail          - "rounds"
  (iii) just below one wave: the tail only     - "tail"
  (iv)  a dynamic group tile spanning jobs whose chunk schedules differ - "mixed"

and then compares every coefficient, the return value, the up-sampling flag and the quant
tables with the oracle.  Content is the synthetic generator's or tests/hard_content.py's
saturated content (letterbox bars, full-contrast strokes, Nyquist checker, wrapping ramps),
which drives the +-1023 clamps, the saturating byte pack of the IDCT and the FDCT clamps.
"""
import ctypes as C

import numpy as np
import pytest

import jpegqs_b200 as qs
import oracle_lib as ol
import hard_content as hc
import wave_geometry as wg
from jpegqs_b200.cuda import _Image, _Slab, _fill_image, QsContext

pytestmark = pytest.mark.gpu

WIDTHS = (2048, 2560, 3072, 4096, 1536)


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def ctx():
    c = QsContext(0)
    yield c
    c.close()


def _wave_tiles(sms):
    return sms * wg.CTA_WARPS


def _in_regime(launches, regime, sms):
    if not launches:
        return False
    wt, big = _wave_tiles(sms), max(l.tiles for l in launches)
    rs = wg.regimes(launches)
    if regime == "i":
        return "dynamic+tail" in rs and 1.2 * wt <= big <= 2.5 * wt
    if regime == "ii":
        return any(l.regime == "rounds" and l.tiles >= wt for l in launches) and big <= 2.5 * wt
    if regime == "iii":
        return rs == {"tail"} and 0.85 * wt <= big < wt
    if regime == "iv":
        return "mixed" in rs and big <= 2.5 * wt
    raise ValueError(regime)


def _size(route, ss, flags, niter, tables, regime, sms, slabs=True):
    """The first (width, height) at which the run's launches are in `regime`."""
    mv = 2 if ss in ("420", "440") else 1
    for w in WIDTHS:
        h = 8 * mv
        while True:
            h += 8 * mv
            ls = wg.smooth_launches(wg.geometry(w, h, ss, tables), flags, niter, route, sms, slabs)
            if ls and max(l.tiles for l in ls) > 2.5 * _wave_tiles(sms):
                break
            if _in_regime(ls, regime, sms):
                return w, h
    raise AssertionError(f"no size puts {route} {ss} flags {flags} in regime {regime}")


def _size_lowq(ss, sms):
    """LOW_QUALITY runs another kernel: about 1.5 waves of blocks."""
    w = 2048
    h = 16
    while wg.geometry(w, h, ss).num_blocks < 1.5 * _wave_tiles(sms) * wg.TILE:
        h += 16
    return w, h


def _check(got, want):
    (ret, out, ups), (oret, oout, oups) = got, want
    assert ret == oret
    assert ups == oups
    nd = ol.diff_count(out, oout)
    assert nd == 0, f"{nd} coefficients differ from the oracle"
    assert ol.images_equal(out, oout)


# ---- the entry points --------------------------------------------------------------------

def _collect(image, ci, coefs, ups):
    out = image.clone()
    for c, t in zip(out.comps, coefs):
        c.coef = t.cpu().numpy()
    QsContext._collect(out, ci, [u.cpu().numpy() for u in ups])
    return out


def _device_buffers(image, stream):
    """Device copies of the coefficients, refreshed on `stream` from a pristine copy just before
    the call (what bench.py does), and zeroed up-sampled chroma planes for 3-component images."""
    import torch
    pristine = [torch.from_numpy(np.ascontiguousarray(c.coef)).cuda() for c in image.comps]
    torch.cuda.synchronize()
    with torch.cuda.stream(stream):
        bufs = [torch.empty_like(p) for p in pristine]
        y = image.comps[0]
        ups = [torch.zeros((y.hblk, y.wblk, 64), dtype=torch.int16, device="cuda")
               for _ in range(2 if len(image.comps) >= 3 else 0)]
        for t, p in zip(bufs, pristine):
            t.copy_(p)
    return bufs, ups


def run_device(ctx, image, flags, niter):
    """jpegqs_cuda_run_device on torch tensors, on a non-default stream."""
    import torch
    s = torch.cuda.Stream()
    bufs, ups = _device_buffers(image, s)
    ci = _Image()
    _fill_image(ci, image, [t.data_ptr() for t in bufs], [None] + [u.data_ptr() for u in ups])
    with torch.cuda.stream(s):
        ret = ctx._check(ctx.lib.jpegqs_cuda_run_device(ctx.h, C.byref(ci), flags & 0x7f, niter, 0, None, None,
                                                        C.c_void_p(s.cuda_stream)))
    s.synchronize()
    return ret, _collect(image, ci, bufs, ups), bool(ci.upsampled)


def run_slab_device(ctx, image, flags, niter):
    """jpegqs_cuda_run_slab, world 1, device buffers: the stop decision is taken on the device."""
    import torch
    s = torch.cuda.Stream()
    bufs, ups = _device_buffers(image, s)
    ci = _Image()
    _fill_image(ci, image, [t.data_ptr() for t in bufs], [None] + [u.data_ptr() for u in ups])
    g = _Slab()
    g.rank, g.world = 0, 1
    for k, c in enumerate(image.comps):
        g.row0[k], g.hblk_total[k] = 0, c.hblk
    with torch.cuda.stream(s):
        ret = ctx._check(ctx.lib.jpegqs_cuda_run_slab(ctx.h, None, C.byref(ci), C.byref(g), flags & 0x7f, niter, 1,
                                                      C.c_void_p(s.cuda_stream)))
    s.synchronize()
    return ret, _collect(image, ci, bufs, ups), bool(ci.upsampled)


def run_batch_device(ctx, images, flags, niter):
    import torch
    s = torch.cuda.Stream()
    arr = (_Image * len(images))()
    keep = []
    for n, im in enumerate(images):
        bufs, ups = _device_buffers(im, s)
        keep.append((bufs, ups))
        _fill_image(arr[n], im, [t.data_ptr() for t in bufs], [None] + [u.data_ptr() for u in ups])
    rets = (C.c_int * len(images))()
    with torch.cuda.stream(s):
        ctx._check(ctx.lib.jpegqs_cuda_run_batch(ctx.h, len(images), arr, flags & 0x7f, niter, 1, rets,
                                                 C.c_void_p(s.cuda_stream)))
    s.synchronize()
    return [(rets[n], _collect(im, arr[n], *keep[n]), bool(arr[n].upsampled)) for n, im in enumerate(images)]


def run_host(ctx, image, flags, niter, slabs):
    ctx.set_tuning(6, int(slabs))
    try:
        ret, out = ctx.do_quantsmooth(image, flags, niter)
    finally:
        ctx.set_tuning(6, 1)
    return ret, out, _up_flag(image, out)


def _up_flag(image, out):
    """The host wrappers report the flag by rewriting every component's sampling to 1x1."""
    return len(out.comps) >= 3 and (image.comps[0].h_samp, image.comps[0].v_samp) != (1, 1) and \
        (out.comps[0].h_samp, out.comps[0].v_samp) == (1, 1)


def _oracle(image, flags, niter):
    return ol.run_oracle(image, flags, niter, threads=0, with_upsampled=True)


# ---- single images through run_device / run_slab ------------------------------------------

SINGLE = [
    # (route, sampling, flags, niter, table, content, regime)
    ("device", "420", 0, 2, "k50", "saturated", "i"),
    ("device", "420", 1, 2, "k10", "saturated", "i"),
    ("device", "420", 3, 2, "rand", "synth", "i"),
    ("device", "420", 7, 2, "diag", "saturated", "i"),
    ("device", "444", 16, 2, "k90", "saturated", "i"),
    ("device", "422", 32 | 1, 2, "k97", "saturated", "i"),
    ("device", "440", 7, 2, "flat", "saturated", "i"),
    ("device", "422", 0, 2, "rand", "saturated", "i"),
    ("device", "gray", 1, 2, "rand", "saturated", "ii"),
    ("device", "gray", 16, 2, "k97", "synth", "ii"),
    ("device", "gray", 0, 2, "k50", "saturated", "iii"),
    ("device", "444", 3, 2, "diag", "synth", "iii"),
    ("slab_device", "420", 7, 2, "k50", "saturated", "i"),
    ("slab_device", "444", 1, 2, "rand", "saturated", "i"),
    ("slab_device", "440", 3, 2, "k90", "synth", "i"),
    ("slab_device", "gray", 32, 2, "flat", "saturated", "ii"),
]


@pytest.mark.parametrize("route,ss,flags,niter,table,content,regime", SINGLE)
def test_single_image_at_wave_scale(ctx, sms, route, ss, flags, niter, table, content, regime):
    tables = hc.TABLES[table]
    w, h = _size(route, ss, flags, niter, tables, regime, sms)
    im = hc.make_image(w, h, ss, tables, content, seed=w + h)
    assert _in_regime(wg.smooth_launches(im, flags, niter, route, sms), regime, sms)
    run = run_device if route == "device" else run_slab_device
    _check(run(ctx, im, flags, niter), _oracle(im, flags, niter))


@pytest.mark.parametrize("ss,flags", [("420", 8), ("444", 8 | 1), ("gray", 8)])
def test_low_quality_clamps_at_wave_scale(ctx, sms, ss, flags):
    """LOW_QUALITY (its own kernel) on saturated content: the FDCT clamp and the final clamp."""
    w, h = _size_lowq(ss, sms)
    im = hc.make_image(w, h, ss, hc.TABLES["k10"], "saturated", seed=3)
    assert wg.smooth_launches(im, flags, 2, "device", sms) == []
    _check(run_device(ctx, im, flags, 2), _oracle(im, flags, 2))


# ---- the host entry point, with the slab pipeline on and off -------------------------------

HOST = [
    ("gray", 0, 3, "k90", "saturated"),
    ("420", 7, 3, "k50", "saturated"),
    ("444", 1, 2, "rand", "synth"),
    ("422", 16, 3, "diag", "saturated"),
]


@pytest.mark.parametrize("slabs", [1, 0])
@pytest.mark.parametrize("ss,flags,niter,table,content", HOST)
def test_host_entry_point_at_wave_scale(ctx, sms, ss, flags, niter, table, content, slabs):
    tables = hc.TABLES[table]
    w, h = _size("host", ss, flags, niter, tables, "i", sms, slabs=bool(slabs))
    im = hc.make_image(w, h, ss, tables, content, seed=w + 3 * h)
    launches = wg.smooth_launches(im, flags, niter, "host", sms, slabs=bool(slabs))
    assert _in_regime(launches, "i", sms)
    if slabs:
        assert "tail" in wg.regimes(launches)                    # the one-wave slabs
    _check(run_host(ctx, im, flags, niter, slabs), _oracle(im, flags, niter))


# ---- heterogeneous batches: group tiles straddle jobs with different schedules --------------

BATCH = [("420", "k50", "saturated", 1.0), ("444", "rand", "synth", 0.5), ("gray", "diag", "saturated", 0.75),
         ("422", "k90", "saturated", 0.6), ("440", "flat", "synth", 0.45), ("420", "k10", "synth", 0.35)]


def _batch_sizes(route, flags, niter, sms):
    """Heights scaled together until the batch's launches are at wave scale with mixed groups."""
    for step in range(1, 400):
        geo = [(1024 + 8 * k, int(step * 16 * rel) + 16) for k, (_, _, _, rel) in enumerate(BATCH)]
        ims = [wg.geometry(w, h, ss, hc.TABLES[t]) for (w, h), (ss, t, _, _) in zip(geo, BATCH)]
        ls = wg.smooth_launches(ims, flags, niter, route, sms)
        if max(l.tiles for l in ls) > 2.5 * _wave_tiles(sms):
            break
        if _in_regime(ls, "iv", sms) and "dynamic+tail" in wg.regimes(ls) and \
                max(l.tiles for l in ls) >= 1.2 * _wave_tiles(sms):
            return geo
    raise AssertionError("no batch size reaches mixed dynamic group tiles")


@pytest.mark.parametrize("on_device,flags", [(1, 0), (1, 3), (0, 0), (0, 16 | 1)])
def test_heterogeneous_batch_at_wave_scale(ctx, sms, on_device, flags):
    route = "batch_device" if on_device else "batch_host"
    niter = 2
    geo = _batch_sizes(route, flags, niter, sms)
    ims = [hc.make_image(w, h, ss, hc.TABLES[t], content, seed=17 * k)
           for k, ((w, h), (ss, t, content, _)) in enumerate(zip(geo, BATCH))]
    ls = wg.smooth_launches(ims, flags, niter, route, sms)
    assert _in_regime(ls, "iv", sms) and "dynamic+tail" in wg.regimes(ls)
    if on_device:
        got = run_batch_device(ctx, ims, flags, niter)
    else:
        rets, outs = ctx.run_batch_host(ims, flags, niter)
        got = [(r, o, _up_flag(im, o)) for r, o, im in zip(rets, outs, ims)]
    for im, g in zip(ims, got):
        _check(g, _oracle(im, flags, niter))


# ---- the legal-range boundary: 2047 goes on, 2048 stops --------------------------------------

@pytest.mark.parametrize("route", ["device", "slab_device"])
@pytest.mark.parametrize("stop", [False, True])
@pytest.mark.parametrize("flags", [0, 7])
def test_dequant_range_boundary_at_wave_scale(ctx, sms, route, stop, flags):
    """run_device decides the reference's `stop` on the host, run_slab on the device."""
    tables = hc.TABLES["k50"]
    w, h = _size(route, "420", flags, 2, tables, "i", sms)
    im = hc.with_dequant_edge(hc.make_image(w, h, "420", tables, "saturated", seed=5), stop)
    if not stop:
        assert _in_regime(wg.smooth_launches(im, flags, 2, route, sms), "i", sms)
    run = run_device if route == "device" else run_slab_device
    got, want = run(ctx, im, flags, 2), _oracle(im, flags, 2)
    assert want[0] == int(stop)
    _check(got, want)


# ---- saturated content through the small-image route (tail branch) --------------------------

SMALL_FLAGS = [0, 1, 3, 7, 16, 32 | 1, 8, 8 | 3, 9 | 4, 24]


@pytest.mark.parametrize("flags", SMALL_FLAGS)
def test_saturated_small_images(ctx, flags):
    for k, ss in enumerate(hc.SAMPLINGS):
        table = list(hc.TABLES)[(k + flags) % len(hc.TABLES)]
        w, h = (208 + 16 * k, 144 + 8 * k) if not (flags & 4) else (208, 144 + 8 * k)
        im = hc.make_image(w, h, ss, hc.TABLES[table], "saturated", seed=k + 100 * flags)
        _check(run_host(ctx, im, flags, 2, 1), _oracle(im, flags, 2))
