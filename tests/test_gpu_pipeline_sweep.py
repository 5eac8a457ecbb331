"""The pixel pipeline on the GPU over a seeded corpus and mixed per-file options (tests/pipeline_files.py).

For every call of the plan, decode_pixels gives each file exactly Pillow's array, and reencode exactly
Pillow's file: Image.open(F), libjpeg's scaled decode at scale_denom > 1, the orientation, convert(mode),
crop().resize() or thumbnail(), the filters and save, with F the file the jpegqs tool writes for the same
options (the input file at -q 3 -n 0).  One call runs through jpegqs_cuda_pixels_batch_filtered into odd
offsets of one device buffer with a guard byte after each picture, and one through
jpegqs_cuda_pixels_batch_jpeg_filtered, whose files the library allocates.  Each file's result does not
depend on the files beside it, their order, the sub-batch budget, the output kind or the layout."""
import ctypes as C

import numpy as np
import pytest

import libjpeg_pixels as lp
import pipeline_files as pf
from test_gpu_pixels_batch import ctx  # noqa: F401  (module fixture)
from test_gpu_pixel_modes import OPTS, tool_file  # noqa: F401  (module fixture)

import jpegqs_b200 as qs
from jpegqs_b200 import cuda

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(lp.JPEG_SO is None, reason="no libjpeg inside Pillow")]

torch = pytest.importorskip("torch")

MODES = {None: 0, "RGB": 1, "L": 2}


@pytest.fixture(scope="module")
def corpus():
    return pf.files()


@pytest.fixture(scope="module")
def plan(corpus):  # noqa: F811
    return pf.plan(corpus)


def _hwc(t, layout):
    a = t.cpu().numpy()
    return np.ascontiguousarray(a if layout == "hwc" else a.transpose(1, 2, 0))


def run(ctx, call, datas, cases, layout=None, device=None, budget=0):  # noqa: F811
    """the call on these files: [H, W, C] arrays, or the JPEG files' bytes"""
    _, flags, niter = OPTS[call["opt"]]
    kw = dict(scale_denom=call["scale"], orientation=pf.orientation_arg(call, cases), mode=call["mode"],
              image_filter=pf.pil_filters(call["chain"]), max_device_bytes=budget, **pf.geometry_args(call, cases))
    if call["kind"] == "reencode":
        return [r[0] for r in ctx.reencode(datas, flags | qs.JPEGQS_TRANSCODE, niter, **pf.save_args(call), **kw)]
    layout = layout or call["layout"]
    recs = ctx.decode_pixels(datas, flags | qs.JPEGQS_TRANSCODE, niter, layout, device or call["device"], **kw)
    return [_hwc(r[0], layout) for r in recs]


@pytest.fixture(scope="module")
def sweep(ctx, corpus, plan, tool_file):  # noqa: F811
    """call index -> (files, Pillow's results, the call's results)"""
    cache = {}

    def get(c):
        if c not in cache:
            call = plan[c]
            datas = [corpus[k]["data"] for k in call["files"]]
            refs = [pf.reference(tool_file(d, call["opt"]), call, cs) for d, cs in zip(datas, call["cases"])]
            cache[c] = (datas, refs, run(ctx, call, datas, call["cases"]))
        return cache[c]
    return get


def _equal(got, want):
    return got == want if isinstance(want, bytes) else got.shape == want.shape and np.array_equal(got, want)


def _mismatches(corpus, call, idx, got, want, what=""):  # noqa: F811
    bad = []
    for j, g, w in zip(idx, got, want):
        if not _equal(g, w):
            k = call["files"][j]
            bad.append(f"{what}{pf.describe(corpus[k], call, call['cases'][j])}: {pf.first_difference(g, w)}")
    return bad


@pytest.mark.parametrize("c", range(len(pf.CALLS)))
def test_call_is_pillow(corpus, plan, sweep, c):  # noqa: F811
    _, refs, got = sweep(c)
    bad = _mismatches(corpus, plan[c], range(len(refs)), got, refs)
    assert not bad, f"{len(bad)} of {len(refs)} files differ from Pillow:\n" + "\n".join(bad)


@pytest.mark.parametrize("c", range(len(pf.CALLS)))
def test_result_is_the_files_own(ctx, corpus, plan, sweep, c):  # noqa: F811
    """alone (every fourth file), split into one-file sub-batches, reversed, the other output kind, the
    other layout: each file's result is the same"""
    call = plan[c]
    datas, _, full = sweep(c)
    cases = call["cases"]
    n = len(datas)
    bad = []
    for j in range(0, n, 4):
        bad += _mismatches(corpus, call, [j], run(ctx, call, [datas[j]], [cases[j]]), [full[j]], "alone: ")
    bad += _mismatches(corpus, call, range(n), run(ctx, call, datas, cases, budget=1), full, "max_device_bytes=1: ")
    rev = list(range(n))[::-1]
    got = run(ctx, call, [datas[j] for j in rev], [cases[j] for j in rev])
    bad += _mismatches(corpus, call, rev, got, [full[j] for j in rev], "reversed: ")
    if call["kind"] == "decode":
        other = {"cuda": "cpu", "cpu": "cuda"}[call["device"]]
        bad += _mismatches(corpus, call, range(n), run(ctx, call, datas, cases, device=other), full, f"device {other}: ")
        other = {"hwc": "chw", "chw": "hwc"}[call["layout"]]
        bad += _mismatches(corpus, call, range(n), run(ctx, call, datas, cases, layout=other), full, f"layout {other}: ")
    assert not bad, "\n".join(bad)


def _c_args(call, datas):
    """the C arguments both filtered entry points share: boxes, orientations, filters"""
    n, g, cases = len(datas), call["geometry"], call["cases"]
    boxes = None
    if g == "thumbnail":
        boxes = (cuda._ResizeBox * n)(*[cuda._ResizeBox(0, 0, 0, 0, *cs["bound"]) for cs in cases])
    elif g is not None:
        boxes = (cuda._ResizeBox * n)(*[cuda._ResizeBox(*(cs["crop"] or (0, 0, 0, 0)), *cs["size"]) for cs in cases])
    o = pf.orientation_arg(call, cases)
    orient = None if o is None else (C.c_int32 * n)(*([0] * n if o == "exif" else [o] * n if isinstance(o, int) else o))
    filt = cuda._image_filters(pf.pil_filters(call["chain"]), "test")
    return boxes, orient, filt


def test_filtered_entry_point_at_odd_offsets(ctx, corpus, plan, sweep):  # noqa: F811
    """call 1 (CHW, per-file orientations 0..8, crops and sizes, a chain) through
    jpegqs_cuda_pixels_batch_filtered: every picture at an odd offset of one device buffer, a guard byte
    after each"""
    call = plan[1]
    datas, refs, _ = sweep(1)
    n = len(datas)
    want = [np.ascontiguousarray(r.transpose(2, 0, 1)).tobytes() for r in refs]          # CHW
    offs, o = [], 1
    for w in want:
        offs.append(o)
        o = (o + len(w) + 1 + (o & 2)) | 1                 # odd, 1 or 3 mod 4
    flat = torch.full((o + 1,), 0xA5, dtype=torch.uint8, device=f"cuda:{ctx.device}")
    outs = (C.c_void_p * n)(*[flat.data_ptr() + x for x in offs])
    torch.cuda.synchronize(ctx.device)
    boxes, orient, filt = _c_args(call, datas)
    rc = (C.c_int * n)()
    res = (cuda._PixelsResult * n)()
    _, flags, niter = OPTS[call["opt"]]
    ret = ctx.lib.jpegqs_cuda_pixels_batch_filtered(ctx.h, n, (C.c_char_p * n)(*datas), (C.c_size_t * n)(*map(len, datas)),
                                                    flags | qs.JPEGQS_TRANSCODE, niter, 1, call["scale"],
                                                    cuda.RESIZE_FILTERS[call["filter"]], boxes, orient, MODES[call["mode"]],
                                                    1, outs, 0, rc, res, 0, 0.0, filt, len(filt))
    assert ret == 0, ctx.lib.jpegqs_cuda_last_error(ctx.h).decode()
    assert list(rc) == [0] * n
    host = flat.cpu().numpy().tobytes()
    bad = [f"{pf.describe(corpus[call['files'][j]], call, call['cases'][j])}" for j in range(n)
           if host[offs[j]:offs[j] + len(want[j])] != want[j]]
    bad += [f"guard byte after file {j} overwritten" for j in range(n) if host[offs[j] + len(want[j])] != 0xA5]
    bad += ["byte 0 overwritten"] * (host[0] != 0xA5)
    assert not bad, "\n".join(bad)


def test_jpeg_filtered_entry_point(ctx, corpus, plan, sweep):  # noqa: F811
    """call 10 (L, per-file orientations, thumbnails with gap 1.0, a chain of four, progressive) through
    jpegqs_cuda_pixels_batch_jpeg_filtered: each file in a buffer the library allocates, released with
    jpegqs_cuda_transcode_free"""
    call = plan[10]
    datas, refs, _ = sweep(10)
    n = len(datas)
    boxes, orient, filt = _c_args(call, datas)
    jp = cuda._jpeg_params(call["quality"], call["subsampling"], call["optimize"], "test", call["progressive"])
    rc = (C.c_int * n)()
    res = (cuda._PixelsResult * n)()
    outs = (C.c_void_p * n)()
    olen = (C.c_size_t * n)()
    _, flags, niter = OPTS[call["opt"]]
    ret = ctx.lib.jpegqs_cuda_pixels_batch_jpeg_filtered(ctx.h, n, (C.c_char_p * n)(*datas),
                                                         (C.c_size_t * n)(*map(len, datas)), flags | qs.JPEGQS_TRANSCODE,
                                                         niter, call["scale"], cuda.RESIZE_FILTERS[call["filter"]], boxes,
                                                         C.byref(jp), 0, rc, res, outs, olen, orient, MODES[call["mode"]], 1,
                                                         call["gap"], filt, len(filt))
    try:
        assert ret == 0, ctx.lib.jpegqs_cuda_last_error(ctx.h).decode()
        assert list(rc) == [0] * n and all(outs[j] for j in range(n))
        got = [C.string_at(outs[j], olen[j]) for j in range(n)]
    finally:
        for j in range(n):
            if outs[j]:
                ctx.lib.jpegqs_cuda_transcode_free(outs[j])
    bad = _mismatches(corpus, call, range(n), got, refs)
    assert not bad, "\n".join(bad)
