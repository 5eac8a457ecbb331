"""The pixel pipeline sweep's plan and reference, without a GPU (tests/pipeline_files.py).

The plan is deterministic and reaches every edge it was written for.  For every case whose reference file
is the input file (q3 -n 0), the Pillow reference equals the CPU models composed in the same order:
render_model(read_jpeg(file), mode=, scale_denom=), a numpy transpose, resize_model_box / thumbnail_model,
image_filter_model, compress_model.  That checks the sweep's own reference, and the models' composition,
before any GPU runs."""
import numpy as np
import pytest

import libjpeg_pixels as lp
import pipeline_files as pf

from jpegqs_b200 import cuda

pytestmark = pytest.mark.skipif(lp.JPEG_SO is None, reason="no libjpeg inside Pillow")

# every edge the plan is written to reach; coverage(plan) must name each one
EDGES = [
    # files
    "file 1 x 1", "file 1 x N", "file N x 1",
    "rows one byte below a multiple of 256", "rows a multiple of 256", "rows just above a multiple of 256",
    "sampling 444", "sampling 422", "sampling 420", "sampling grey", "sampling 411", "sampling 440",
    "colour ycbcr", "colour grey", "colour cmyk", "colour ycck",
    "coding baseline", "coding optimize", "coding progressive", "coding progressive_rst", "coding restart",
    "content random", "content gradient", "content hard",
    *[f"exif orientation {o}" for o in range(2, 9)],
    # flags, output, scale, orientation and mode
    "opt q3n0", "opt q6", "opt q3",
    "output hwc cuda", "output hwc cpu", "output chw cuda", "output chw cpu",
    "scale 1", "scale 2", "scale 4", "scale 8",
    "orientation None", "orientation exif", "orientation one value", "orientation list", "every orientation in one call",
    "mode None", "mode RGB", "mode L",
    # geometry
    "geometry None", "geometry crop",
    "geometry gap gap 1.0", "geometry gap gap 2.0", "geometry gap gap 3.0",
    "geometry thumbnail gap None", "geometry thumbnail gap 1.0", "geometry thumbnail gap 2.0",
    "geometry thumbnail gap 3.0",
    *[f"crop kind {k}" for k in pf.CROP_KINDS],
    *[f"crop and size with {f}" for f in ("lanczos", "bilinear", "bicubic", "hamming", "box")],
    "crop with a reduce", "thumbnail bound larger than the picture",
    # filters
    "chain of 0", "chain of 1", "chain of 2", "chain of 3", "chain of 4",
    "gaussian radius 0", "gaussian radius 0.3", "gaussian fractional radius", "gaussian radius larger than the picture",
    "box blur with one axis 0", "box radius at least the picture", "one-axis box blur in the middle of a chain",
    "unsharp percent 0", "unsharp large percent", "unsharp threshold 0", "unsharp threshold 255",
    # reencode
    "quality 1", "quality 50", "quality 95", "quality 100",
    "subsampling 4:4:4", "subsampling 4:2:2", "subsampling 4:2:0", "optimize", "progressive",
    # the combinations
    "filter rows past 16384 beside narrow rows after a resize",
    "orientation 5-8 with chw, crop, resize and filter", "chw colour resize without a filter, rows past 256 bytes",
    "cmyk and ycck with grey and rgb in a thumbnail call", "cmyk and ycck with grey and rgb in a filter call",
    "scale 4 then resize and filter", "scale 8 then resize and filter",
    "mode L, filter, progressive reencode",
    "render scales 1, 2, 4 and 8 in one call", "render layouts hwc and chw in one call",
    "thumbnail drafted from a fractional box",
]
N0_CALLS = [c for c, s in enumerate(pf.CALLS) if s["opt"] == "q3n0"]


@pytest.fixture(scope="module")
def corpus():
    return pf.files()


@pytest.fixture(scope="module")
def plan(corpus):
    return pf.plan(corpus)


def test_plan_is_deterministic(corpus, plan):
    again = pf.files()
    assert [f["data"] for f in again] == [f["data"] for f in corpus]
    assert pf.plan(again) == plan


def test_plan_mixes_the_corpus(corpus, plan):
    assert 110 <= len(corpus) <= 130 and len({f["name"] for f in corpus}) == len(corpus)
    assert len(plan) == 13 and all(len(call["files"]) >= 24 for call in plan)
    assert {k for call in plan for k in call["files"]} == set(range(len(corpus)))
    assert sum(f["exif"] > 1 for f in corpus) * 3 >= len(corpus) - 3
    assert sum(call["opt"] == "q3n0" for call in plan) >= 9


def test_coverage_names_every_edge(corpus, plan):
    missing = [e for e in EDGES if e not in pf.coverage(plan, corpus)]
    assert not missing, missing


def test_draft_scale_is_the_thumbnail_geometry(corpus, plan):
    """coverage's restatement of Pillow's draft, which names the render scales of a call, is the library's"""
    for call in plan:
        if call["geometry"] != "thumbnail":
            continue
        for k, cs in zip(call["files"], call["cases"]):
            w, h = pf.oriented(corpus[k], cs["orient"])
            loaded = call["orientation"] is not None or call["mode"] is not None
            want = cuda.thumbnail_geometry(w, h, cs["bound"], call["gap"], loaded)[0]
            assert (1 if loaded else pf.draft_scale(w, h, cs["bound"], call["gap"])) == want, (call["index"], k)


def _orient(a, o):
    """Pillow's transposes of an [H, W, C] array"""
    return {1: a, 2: a[:, ::-1], 3: a[::-1, ::-1], 4: a[::-1], 5: a.transpose(1, 0, 2), 6: np.rot90(a, -1),
            7: a.transpose(1, 0, 2)[::-1, ::-1], 8: np.rot90(a, 1)}[o]


def model(f, call, case):
    """the CPU models composed in Pillow's order, on the input file"""
    g = call["geometry"]
    loaded = call["orientation"] is not None or case["mode"] is not None
    full = pf.oriented(f, case["orient"])
    scale = case["scale"]
    if g == "thumbnail":
        scale, _ = cuda.thumbnail_geometry(*full, case["bound"], call["gap"], loaded)
    a = cuda.render_model(cuda.read_jpeg(f["data"]), scale_denom=scale, mode=case["mode"])
    if case["mode"] is None and f["colour"] == "grey":
        a = a[..., :1]                                      # the render model writes grey as three equal channels
    a = np.ascontiguousarray(_orient(a, case["orient"]))
    if g == "thumbnail":
        a = cuda.thumbnail_model(a, full, case["bound"], call["filter"], call["gap"], loaded)
    elif g is not None:
        if case["crop"] is not None:
            left, top, right, bottom = case["crop"]
            a = np.ascontiguousarray(a[top:bottom, left:right])
        a = cuda.resize_model_box(a, case["size"], None, call["filter"], call["gap"] if g == "gap" else None)
    if call["chain"]:
        a = cuda.image_filter_model(a, pf.pil_filters(call["chain"]))
    if call["kind"] == "reencode":
        return cuda.compress_model(a, **pf.save_args(call))
    return a


@pytest.mark.parametrize("c", N0_CALLS)
def test_reference_is_the_composed_models(corpus, plan, c):
    call = plan[c]
    bad = []
    for k, case in zip(call["files"], call["cases"]):
        f = corpus[k]
        want, got = pf.reference(f["data"], call, case), model(f, call, case)
        if isinstance(want, bytes):
            if got != want:
                bad.append(f"{pf.describe(f, call, case)}: {len(got)} bytes against Pillow's {len(want)}")
        elif got.shape != want.shape or not np.array_equal(got, want):
            bad.append(f"{pf.describe(f, call, case)}: {pf.first_difference(got, want)}")
    assert not bad, "\n".join(bad)
