"""A seeded corpus of JPEG files and a plan of mixed calls for the GPU pixel pipeline.

The pipeline is every stage of decode_pixels / reencode after the smoothing: the render (scale, orientation
and mode), the reduce, the crop and resize, the thumbnail, the filters and the compressor.  The CPU model
sweeps pin each stage's arithmetic, and the GPU tests of each stage use one fixed corpus with one or two
options at a time.  What neither reaches is the device-only code between the stages: the block-to-picture
searches of the resize, reduce and filter kernels, the render order and its mapping back to the files,
the buffer plan, the crop offsets after a reduce, thumbnail's draft after an orientation or a mode, and
the sub-batch split.  This module gives the inputs that reach them:

  * `files()`: about 120 JPEG files, 1 x 1 to 16500 x 8, every sampling (4:4:4, 4:2:2, 4:2:0, grey,
    4:1:1, 4:4:0), CMYK and YCCK, baseline, optimized, progressive with and without restart markers and
    sequential with them, random, gradient and saturated content, a third with an EXIF orientation.
  * `plan(files)`: thirteen calls, each mixing 24 or more of them, with per-file orientations, crops,
    sizes, thumbnail bounds and a filter chain drawn from a fixed seed.
  * `reference(...)`: what Pillow gives for one file of one call, in Pillow's order.
  * `coverage(plan, files)`: the edges the plan reaches, so that an edit cannot drop one unnoticed.

Nothing here touches a GPU."""
from __future__ import annotations

import io

import numpy as np
from PIL import Image, ImageFilter

import decode_files as df
import hard_content as hc
import libjpeg_scaled as ls
from render_images import make
from test_orientation_cpu import exif, splice, tag
from test_pixel_modes_cpu import YCCK_FACTORS, cmyk_file, libjpeg_reference, ycck_file

T = Image.Transpose
METHODS = {2: T.FLIP_LEFT_RIGHT, 3: T.ROTATE_180, 4: T.FLIP_TOP_BOTTOM, 5: T.TRANSPOSE, 6: T.ROTATE_270,
           7: T.TRANSVERSE, 8: T.ROTATE_90}
RESAMPLE = {"lanczos": Image.Resampling.LANCZOS, "bilinear": Image.Resampling.BILINEAR,
            "bicubic": Image.Resampling.BICUBIC, "box": Image.Resampling.BOX, "hamming": Image.Resampling.HAMMING}
SAMPLINGS = ("444", "422", "420", "411", "440")
CODINGS = ("baseline", "optimize", "progressive", "progressive_rst", "restart")
CONTENTS = ("random", "gradient", "hard")
ROW_MAX = 16384                                      # csrc/qs_filter.h QS_FILTER_ROW_MAX


# ---- files ------------------------------------------------------------------------------------------
def _content(w, h, channels, content, seed):
    rng = np.random.RandomState(seed)
    if content == "random":
        return rng.randint(0, 256, (h, w, channels)).astype(np.uint8)
    if content == "gradient":
        yy, xx = np.mgrid[0:h, 0:w].astype(np.int64)
        a, b = rng.randint(1, 9, 2)
        return np.stack([(xx * a * 255 // max(w, 1) + yy * b) % 256, (yy * 255 // max(h, 1) + xx) % 256,
                         (xx + yy) * 255 // max(w + h, 1)][:channels], -1).astype(np.uint8)
    return np.stack([hc.saturated_pixels(c, 0, h, w, 1, 1, seed, h, w) for c in range(channels)], -1).astype(np.uint8)


def _save(pixels, grey, sampling, coding, quality):
    im = Image.fromarray(pixels[..., 0] if grey else pixels)
    kw = {"quality": quality}
    if not grey:
        kw["subsampling"] = {"444": 0, "422": 1, "420": 2}[sampling]
    if coding == "optimize":
        kw["optimize"] = True
    elif coding == "progressive":
        kw["progressive"] = True
    elif coding == "progressive_rst":
        kw.update(progressive=True, restart_marker_blocks=3)
    elif coding == "restart":
        kw["restart_marker_rows" if quality % 2 else "restart_marker_blocks"] = 1 + quality % 5
    b = io.BytesIO()
    im.save(b, "JPEG", **kw)
    return b.getvalue()


def _sizes():
    """(w, h, kind): the fixed edges, then seeded sizes"""
    out = [(1, 1, None), (1, 37, None), (53, 1, None), (2, 2, None), (7, 9, None), (8, 8, None), (9, 17, None),
           (15, 16, None), (16, 16, None), (17, 17, None)]
    # w * channels on each side of a multiple of 256 (85 * 3 = 255, 86 * 3 = 258, 256 * 3 = 768)
    for k, w in enumerate((85, 86, 255, 256, 257)):
        out += [(w, 5 + 3 * k, "grey"), (w, 11 + 2 * k, "rgb")]
    out += [(1000, 37, None), (1537, 90, "grey"), (2000, 23, None)]
    out += [(6000, 24, "rgb"), (16500, 8, "grey")]            # rows past ROW_MAX
    rng = np.random.RandomState(2024)
    while len(out) < 120:
        w, h = (int(v) for v in rng.randint(1, 401, 2))
        if max(w, h) <= 100 * min(w, h):
            out.append((w, h, None))
    return out


def files():
    """[dict(name, data, w, h, colour, sampling, coding, content, exif)]: colour 'ycbcr', 'grey', 'cmyk' or
    'ycck'; sampling one of SAMPLINGS or 'grey' (4 components: the writer's); exif the orientation tag (1:
    none)"""
    out = []
    for k, (w, h, kind) in enumerate(_sizes()):
        r = np.random.RandomState(k)
        content = CONTENTS[k % 3]
        coding = CODINGS[(k // 3) % 5]
        quality = int(r.randint(30, 96))
        colour = kind if kind in ("grey",) else "ycbcr"
        if kind is None:
            colour = ("ycbcr", "ycbcr", "grey", "ycbcr", "cmyk", "ycbcr", "ycck", "ycbcr")[k % 8] if k >= 25 else \
                ("ycbcr", "grey")[k % 2]
        sampling = "grey" if colour == "grey" else SAMPLINGS[k % 5] if colour == "ycbcr" else "444"
        if colour == "cmyk":
            data = cmyk_file(w, h, k, quality=quality, **({"progressive": True} if coding.startswith("prog") else {}))
            coding = "progressive" if coding.startswith("prog") else "baseline"
        elif colour == "ycck":
            sampling = ("444", "y2k2", "k_alone")[k % 3]
            data = ycck_file(w, h, YCCK_FACTORS[sampling], seed=k)
            coding = "baseline"
        elif sampling in ("411", "440"):
            data = df.coef_writer_jpeg(make(w, h, sampling, ("k50", "k90", "rand")[k % 3],
                                            "saturated" if content == "hard" else "synth", k))
            coding, content = "baseline", "hard" if content == "hard" else "synth"
        else:
            grey = colour == "grey"
            data = _save(_content(w, h, 3, content, k), grey, sampling, coding, quality)
        o = 2 + k % 7 if k % 3 == 1 else 1
        if o > 1:
            data = splice(data, exif([tag("SHORT", [o])]))
        out.append(dict(name=f"f{k:03d}_{w}x{h}_{colour}_{sampling}_{coding}_{content}" + (f"_exif{o}" if o > 1 else ""),
                        data=data, w=w, h=h, colour=colour, sampling=sampling, coding=coding, content=content, exif=o))
    return out


# ---- the plan ---------------------------------------------------------------------------------------
# a filter is ("gauss", radius), ("box", radius) or ("unsharp", radius, percent, threshold); radius a number
# or (x, y)
CALLS = [
    # plain render then a filter: the 1-pixel pictures, rows around 256 bytes, rows past ROW_MAX
    dict(kind="decode", opt="q3n0", layout="hwc", device="cuda", scale=1, orientation=None, mode=None,
         geometry=None, chain=[("unsharp", 2.0, 150, 3)]),
    # orientations 5..8 among a per-file list, CHW, crop and resize, a filter
    dict(kind="decode", opt="q3n0", layout="chw", device="cuda", scale=1, orientation="list", mode=None,
         geometry="crop", filter="lanczos", chain=[("box", (3, 0)), ("gauss", 0.3)]),
    # a one-axis BoxBlur in the middle of a chain, after a resize; wide rows beside narrow ones
    dict(kind="decode", opt="q3n0", layout="hwc", device="cpu", scale=1, orientation=None, mode=None,
         geometry="crop", filter="bicubic", chain=[("gauss", 1.7), ("box", (0, 1)), ("unsharp", 1.0, 300, 0)]),
    # 1/4 scale, then crop, resize and a blur wider than most pictures
    dict(kind="decode", opt="q3n0", layout="chw", device="cpu", scale=4, orientation="exif", mode=None,
         geometry="crop", filter="hamming", chain=[("gauss", 50.0)]),
    # 1/8 scale with one orientation and RGB (CMYK and YCCK included), a box blur past the picture
    dict(kind="decode", opt="q3n0", layout="hwc", device="cuda", scale=8, orientation=6, mode="RGB",
         geometry="crop", filter="box", chain=[("box", 400), ("unsharp", 0.5, 0, 0)]),
    # RGB, size with a reducing gap, CHW without a filter: the resize writes the caller's layout
    dict(kind="decode", opt="q3n0", layout="chw", device="cuda", scale=1, orientation=None, mode="RGB",
         geometry="gap", gap=2.0, filter="bicubic", chain=None),
    # thumbnails without a gap, RGB: every colour space in one thumbnail and filter call
    dict(kind="decode", opt="q3n0", layout="hwc", device="cuda", scale=1, orientation=None, mode="RGB",
         geometry="thumbnail", gap=None, filter="bicubic", chain=[("unsharp", 2.0, 80, 255)]),
    # the tool's file at q6: thumbnails after EXIF orientation (loaded: no draft)
    dict(kind="decode", opt="q6", layout="chw", device="cpu", scale=1, orientation="exif", mode=None,
         geometry="thumbnail", gap=2.0, filter="lanczos", chain=[("gauss", 2.5), ("box", (1.5, 0.5))]),
    # the tool's file at q3: reencode after size with gap 1.0
    dict(kind="reencode", opt="q3", scale=1, orientation=None, mode=None, geometry="gap", gap=1.0, filter="hamming",
         chain=[("box", 1), ("unsharp", 1.5, 200, 2)], quality=95, subsampling="4:4:4", optimize=True,
         progressive=False),
    # reencode at 1/2 scale after size with gap 3.0 and crops, lowest quality
    dict(kind="reencode", opt="q3n0", scale=2, orientation="exif", mode=None, geometry="gap", gap=3.0,
         filter="bilinear", chain=None, quality=1, subsampling="4:2:2", optimize=False, progressive=False),
    # L, a chain of four, a per-file orientation list, thumbnails with gap 1.0, progressive
    dict(kind="reencode", opt="q3n0", scale=1, orientation="list", mode="L", geometry="thumbnail", gap=1.0,
         filter="box", chain=[("gauss", 0.0), ("box", (2, 0)), ("gauss", 0.6), ("unsharp", 0.5, 5000, 255)],
         quality=50, subsampling="4:2:0", optimize=False, progressive=True),
    # RGB thumbnails with gap 3.0 after one orientation, quality 100, optimized progressive
    dict(kind="reencode", opt="q3n0", scale=1, orientation=8, mode="RGB", geometry="thumbnail", gap=3.0,
         filter="bicubic", chain=[("unsharp", 3.0, 0, 255), ("gauss", (0.0, 3.5))], quality=100,
         subsampling="4:2:0", optimize=True, progressive=True),
    # thumbnails with neither orientation nor mode, gap 2.0: each file drafts at its own scale (1, 2, 4 or 8)
    # from the box (0, 0, W / s, H / s), so one call renders under several keys; CHW without a filter, so a
    # file the bound covers is rendered straight into the caller's layout beside HWC renders
    dict(kind="decode", opt="q3n0", layout="chw", device="cpu", scale=1, orientation=None, mode=None,
         geometry="thumbnail", gap=2.0, filter="hamming", chain=None, draft=True),
]
CROP_KINDS = ("1x1", "up15", "same", "one_axis_w", "one_axis_h", "edge_left", "edge_top", "edge_right", "edge_bottom",
              "whole", "random")


def oriented(f, o):
    return (f["h"], f["w"]) if o >= 5 else (f["w"], f["h"])


def picture(f, case):
    """(width, height, channels) of the rendered picture of file f in a case: scaled, then oriented"""
    d = case["scale"]
    w, h = oriented(f, case["orient"])
    ch = 1 if case["mode"] == "L" or (case["mode"] is None and f["colour"] == "grey") else 3
    return -(-w // d), -(-h // d), ch


def _crop_size(rng, pw, ph, kind):
    """(crop or None, (width, height)) of one crop kind in a pw x ph picture"""
    def span(n):
        a = int(rng.randint(n))
        return a, int(rng.randint(a + 1, n + 1))
    (l, r), (t, b) = span(pw), span(ph)
    if kind == "1x1":
        return (l, t, r, b), (1, 1)
    if kind == "up15":
        cw, ch = min(pw, int(rng.randint(1, 7))), min(ph, int(rng.randint(1, 7)))
        l, t = int(rng.randint(pw - cw + 1)), int(rng.randint(ph - ch + 1))
        return (l, t, l + cw, t + ch), (15 * cw, 15 * ch + int(rng.randint(2)))
    if kind == "same":
        return (l, t, r, b), (r - l, b - t)
    if kind == "one_axis_w":
        return None, (int(rng.randint(1, min(2 * pw + 2, 900))), ph)
    if kind == "one_axis_h":
        return None, (pw, int(rng.randint(1, min(2 * ph + 2, 600))))
    if kind == "edge_left":
        l = 0
    elif kind == "edge_top":
        t = 0
    elif kind == "edge_right":
        r = pw
    elif kind == "edge_bottom":
        b = ph
    elif kind == "whole":
        return None, (int(rng.randint(1, min(2 * pw + 2, 700))), int(rng.randint(1, min(2 * ph + 2, 500))))
    return (l, t, r, b), (int(rng.randint(1, min(2 * (r - l) + 2, 700))), int(rng.randint(1, min(2 * (b - t) + 2, 500))))


def _gap_crop_size(rng, pw, ph):
    """a crop (or None) and a size below it, often by more than the gap, so that a reduce runs"""
    crop = None
    l, t, r, b = 0, 0, pw, ph
    if rng.rand() < 0.7:
        l, t = int(rng.randint((pw + 1) // 2)), int(rng.randint((ph + 1) // 2))
        r, b = int(rng.randint(l + 1, pw + 1)), int(rng.randint(t + 1, ph + 1))
        crop = (l, t, r, b)
    f = int(rng.randint(1, 13))
    return crop, (max(1, (r - l) // f), max(1, (b - t) // max(1, f + int(rng.randint(-1, 2)))))


def draft_scale(w, h, bound, gap):
    """the libjpeg scale Pillow's thumbnail drafts a w x h JPEG file at (1 when the bound covers the picture
    or gap is None): JpegImageFile.draft(None, (int(bw * gap), int(bh * gap)))"""
    if gap is None or (bound[0] >= w and bound[1] >= h):
        return 1
    s = min(w // int(bound[0] * gap), h // int(bound[1] * gap))
    return next(d for d in (8, 4, 2, 1) if s >= d or d == 1)


def _draft_bound(rng, pw, ph, gap, pos):
    """a bound under which a pw x ph file drafts at 1 / (1, 2, 4, 8)[pos % 4] where its size allows"""
    want = (1, 2, 4, 8)[pos % 4]
    for s in (want, 4, 2):
        if pw >= 2 * s * gap and ph >= 2 * s * gap:
            return (int(pw // (s * gap)) - int(rng.randint(2)), int(ph // (s * gap)) - int(rng.randint(2)))
    return tuple(int(v) for v in rng.randint(1, 300, 2))


def _members(fl, c, call):
    """the files of call c: every fourth file from a shifted start, with the edge files added to the
    calls that need them, and none the call cannot take"""
    big = {k for k, f in enumerate(fl) if f["w"] >= 1500}
    ks = [k for k in range(len(fl)) if k % 4 == c % 4 and k not in big]
    if c in (0, 2, 12):                              # the wide rows, with narrow ones
        ks += [k for k in big if k not in ks]
    if c in (0, 1, 2, 6, 8, 10, 12):                 # the 1-pixel and the 256-byte rows
        ks += [k for k in range(20) if k not in ks]
    ks = sorted(set(ks))
    if call["mode"] is None:
        ks = [k for k in ks if fl[k]["colour"] not in ("cmyk", "ycck")]
    elif c in (4, 6):                                # every 4-component file where a mode takes them
        ks = sorted(set(ks) | {k for k, f in enumerate(fl) if f["colour"] in ("cmyk", "ycck") and k not in big})
    return ks


def plan(fl):
    """[call]: each call is CALLS[c] with "files" (indices into fl) and "cases", one per file:
    dict(orientation (the call's argument for this file), orient (the orientation it resolves to),
    crop, size, bound, scale, mode)"""
    out = []
    for c, spec in enumerate(CALLS):
        rng = np.random.RandomState(100 + c)
        call = dict(spec, index=c)
        ks, cases = [], []
        for pos, k in enumerate(_members(fl, c, spec)):
            f = fl[k]
            o_arg = spec["orientation"]
            if o_arg == "list":
                o_arg = (pos + c) % 9
            o = f["exif"] if o_arg in ("exif", 0) else 1 if o_arg is None else o_arg
            case = dict(orientation=o_arg, orient=o, scale=spec["scale"], mode=spec["mode"], crop=None, size=None,
                        bound=None)
            pw, ph, ch = picture(f, case)
            g = spec["geometry"]
            if g is not None and ph > 100 * pw:
                continue                             # Pillow resizes such a picture vertically first: refused
            if g == "crop":
                kind = "one_axis_h" if pw * ch > ROW_MAX else CROP_KINDS[(pos + c) % len(CROP_KINDS)]
                case["crop"], case["size"] = _crop_size(rng, pw, ph, kind)
                case["crop_kind"] = kind
            elif g == "gap":
                case["crop"], case["size"] = _gap_crop_size(rng, pw, ph)
            elif g == "thumbnail" and spec.get("draft"):
                case["bound"] = _draft_bound(rng, pw, ph, spec["gap"], pos)
            elif g == "thumbnail":
                case["bound"] = ((pw + int(rng.randint(1, 50)), ph + int(rng.randint(1, 50))) if pos % 6 == 0 else
                                 tuple(int(v) for v in rng.randint(1, 300, 2)))
            ks.append(k)
            cases.append(case)
        call["files"], call["cases"] = ks, cases
        out.append(call)
    return out


def orientation_arg(call, cases):
    """the orientation argument of decode_pixels / reencode for these cases of a call"""
    o = call["orientation"]
    return [cs["orientation"] for cs in cases] if o == "list" else o


def geometry_args(call, cases):
    """the keyword arguments of the call's geometry for these of its cases"""
    g = call["geometry"]
    if g is None:
        return {}
    kw = {"filter": call["filter"]}
    if g == "thumbnail":
        kw.update(thumbnail=[cs["bound"] for cs in cases], reducing_gap=call["gap"])
    else:
        kw.update(size=[cs["size"] for cs in cases], crop=[cs["crop"] for cs in cases])
        if g == "gap":
            kw["reducing_gap"] = call["gap"]
    return kw


def pil_filters(chain):
    """the chain as Pillow's ImageFilter instances, or None"""
    if chain is None:
        return None
    out = []
    for f in chain:
        if f[0] == "gauss":
            out.append(ImageFilter.GaussianBlur(f[1]))
        elif f[0] == "box":
            out.append(ImageFilter.BoxBlur(f[1]))
        else:
            out.append(ImageFilter.UnsharpMask(f[1], f[2], f[3]))
    return out


def save_args(call):
    return dict(quality=call["quality"], subsampling=call["subsampling"], optimize=call["optimize"],
                progressive=call["progressive"])


# ---- the reference ----------------------------------------------------------------------------------
def _as_hwc(a):
    a = np.asarray(a)
    return a[..., None] if a.ndim == 2 else a


def reference(src, call, case):
    """Pillow's result for one file of a call: src is the file the render's coefficients come from (the
    input file at q3n0, else the file the jpegqs tool writes).  Image.open; at scale d > 1 libjpeg's
    scaled decode (with Pillow's conversions for a mode); the orientation; convert(mode); crop().resize()
    or thumbnail(); the filters; for reencode, save.  Returns [H, W, C] uint8, or the JPEG file's bytes."""
    d = case["scale"]
    if d > 1:
        px = libjpeg_reference(src, d, case["mode"]) if case["mode"] else ls.decode_bytes(src, d)[0]
        im = Image.fromarray(px[..., 0] if px.shape[2] == 1 else px)
    else:
        im = Image.open(io.BytesIO(src))
    if call["orientation"] is not None:
        o = case["orient"]
        im = im.transpose(METHODS[o]) if o != 1 else im.copy()
    if case["mode"] is not None and d == 1:
        im = im.convert(case["mode"])
    g = call["geometry"]
    if g == "thumbnail":
        im.thumbnail(case["bound"], RESAMPLE[call["filter"]], reducing_gap=call["gap"])
    elif g is not None:
        if case["crop"] is not None:
            im = im.crop(case["crop"])
        im = im.resize(case["size"], RESAMPLE[call["filter"]], reducing_gap=call.get("gap") if g == "gap" else None)
    for f in pil_filters(call["chain"]) or []:
        im = im.filter(f)
    if call["kind"] == "reencode":
        b = io.BytesIO()
        im.save(b, "JPEG", **save_args(call))
        return b.getvalue()
    return _as_hwc(im)


def describe(f, call, case):
    """one line naming a file and its call's options, for a failure message"""
    opts = {k: call[k] for k in ("kind", "opt", "layout", "device", "scale", "mode", "geometry", "filter", "gap",
                                 "chain", "quality", "subsampling", "optimize", "progressive") if k in call}
    geo = {k: case[k] for k in ("orient", "crop", "size", "bound") if case.get(k) is not None}
    return f"call {call['index']} {f['name']} ({f['w']} x {f['h']}, {f['sampling']}, {f['colour']}) {geo} {opts}"


def first_difference(got, want):
    """where two results first differ: the shapes, the first differing pixel (y, x, c) of two arrays, or
    the first differing byte of two files"""
    if isinstance(want, bytes):
        k = next((i for i, (a, b) in enumerate(zip(got, want)) if a != b), min(len(got), len(want)))
        return f"{len(got)} bytes against {len(want)}, first difference at byte {k}"
    if got.shape != want.shape:
        return f"shape {got.shape} against {want.shape}"
    y, x, c = (int(v) for v in np.argwhere(got != want)[0])
    return f"pixel (y {y}, x {x}, c {c}): {got[y, x, c]} against {want[y, x, c]}, {int((got != want).sum())} samples differ"


# ---- coverage ---------------------------------------------------------------------------------------
def _reduces(crop, size, pw, ph, gap):
    cw, chh = (crop[2] - crop[0], crop[3] - crop[1]) if crop else (pw, ph)
    return int(cw / size[0] / gap) > 1 or int(chh / size[1] / gap) > 1


def coverage(pl, fl):
    """the set of edges (strings) the plan reaches"""
    e = set()
    for call in pl:
        c, g, chain = call["index"], call["geometry"], call["chain"] or []
        e.add("opt " + call["opt"])
        e.add(f"scale {call['scale']}")
        e.add(f"mode {call['mode']}")
        o = call["orientation"]
        e.add("orientation " + ("None" if o is None else o if isinstance(o, str) else "one value"))
        if call["kind"] == "decode":
            e.add(f"output {call['layout']} {call['device']}")
        else:
            e.add(f"quality {call['quality']}")
            e.add(f"subsampling {call['subsampling']}")
            if call["optimize"]:
                e.add("optimize")
            if call["progressive"]:
                e.add("progressive")
        e.add(f"geometry {g}" + (f" gap {call['gap']}" if g in ("gap", "thumbnail") else ""))
        e.add(f"chain of {len(chain)}")
        for k, f in enumerate(chain):
            if f[0] == "box" and isinstance(f[1], tuple) and 0 in f[1]:
                e.add("box blur with one axis 0")
                if 0 < k < len(chain) - 1:
                    e.add("one-axis box blur in the middle of a chain")
            if f[0] == "gauss":
                r = f[1] if isinstance(f[1], tuple) else (f[1], f[1])
                if 0.0 in r:
                    e.add("gaussian radius 0")
                if 0.3 in r:
                    e.add("gaussian radius 0.3")
                if any(v % 1 and v != 0.3 for v in r):
                    e.add("gaussian fractional radius")
            if f[0] == "unsharp":
                e.add({0: "unsharp percent 0"}.get(f[2], "unsharp large percent" if f[2] >= 300 else "unsharp percent"))
                e.add({0: "unsharp threshold 0", 255: "unsharp threshold 255"}.get(f[3], "unsharp threshold"))
        colours, rows, keys = set(), [], set()
        for k, cs in zip(call["files"], call["cases"]):
            f = fl[k]
            pw, ph, ch = picture(f, cs)
            colours.add(f["colour"])
            e.update({f"sampling {f['sampling']}", f"colour {f['colour']}", f"coding {f['coding']}",
                      f"content {f['content']}"})
            if o in ("exif", "list") and cs["orientation"] in ("exif", 0) and f["exif"] > 1:
                e.add(f"exif orientation {f['exif']}")
            if cs["orient"] >= 5 and call.get("layout") == "chw" and cs["crop"] and cs["size"] and chain:
                e.add("orientation 5-8 with chw, crop, resize and filter")
            if (f["w"], f["h"]) == (1, 1):
                e.add("file 1 x 1")
            elif f["w"] == 1:
                e.add("file 1 x N")
            elif f["h"] == 1:
                e.add("file N x 1")
            if g or chain:
                for r in {pw * ch}:
                    if r >= 255 and r % 256 == 255:
                        e.add("rows one byte below a multiple of 256")
                    elif r >= 256 and r % 256 == 0:
                        e.add("rows a multiple of 256")
                    elif r > 256 and r % 256 <= 3:
                        e.add("rows just above a multiple of 256")
            if g in ("crop", "gap") and cs["crop"] is not None:
                e.add(f"crop and size with {call['filter']}")
            if g == "crop":
                e.add("crop kind " + cs["crop_kind"])
            if g == "gap" and cs["crop"] and _reduces(cs["crop"], cs["size"], pw, ph, call["gap"]):
                e.add("crop with a reduce")
            if g == "thumbnail" and cs["bound"][0] >= pw and cs["bound"][1] >= ph:
                e.add("thumbnail bound larger than the picture")
            # the render key of csrc/qs_transcode.cu pixels_batch: the draft scale, and the layout the render
            # writes (HWC when a later stage follows)
            s = cs["scale"]
            if g == "thumbnail" and o is None and call["mode"] is None:
                s = draft_scale(pw, ph, cs["bound"], call["gap"])
                if s > 1 and (pw % s or ph % s):
                    e.add("thumbnail drafted from a fractional box")
            covered = g == "thumbnail" and cs["bound"][0] >= pw and cs["bound"][1] >= ph
            keys.add((s, "hwc" if chain or (g is not None and not covered) else call.get("layout", "hwc")))
            if chain:
                out_w, out_h = (cs["size"] if cs["size"] else (pw, ph))
                if g == "thumbnail":
                    out_w, out_h = min(pw, cs["bound"][0]), min(ph, cs["bound"][1])
                rows.append(out_w * ch)
                for fl_ in chain:
                    r = fl_[1] if isinstance(fl_[1], tuple) else (fl_[1], fl_[1])
                    if fl_[0] == "gauss" and max(r) > max(out_w, out_h):
                        e.add("gaussian radius larger than the picture")
                    if fl_[0] == "box" and max(r) >= max(out_w, out_h):
                        e.add("box radius at least the picture")
                if call["scale"] in (4, 8) and cs["size"]:
                    e.add(f"scale {call['scale']} then resize and filter")
        if {"cmyk", "ycck"} <= colours and {"grey", "ycbcr"} <= colours:
            if g == "thumbnail":
                e.add("cmyk and ycck with grey and rgb in a thumbnail call")
            if chain:
                e.add("cmyk and ycck with grey and rgb in a filter call")
        if g in ("crop", "gap") and not chain and call.get("layout") == "chw" and any(
                cs["size"][0] > 85 and picture(fl[k], cs)[2] == 3 for k, cs in zip(call["files"], call["cases"])):
            e.add("chw colour resize without a filter, rows past 256 bytes")
        if g in ("crop", "gap") and chain and rows and max(rows) > ROW_MAX and min(rows) <= ROW_MAX:
            e.add("filter rows past 16384 beside narrow rows after a resize")
        if call["mode"] == "L" and chain and call.get("progressive"):
            e.add("mode L, filter, progressive reencode")
        if {s for s, _ in keys} >= {1, 2, 4, 8}:
            e.add("render scales 1, 2, 4 and 8 in one call")
        if len({lay for _, lay in keys}) == 2:
            e.add("render layouts hwc and chw in one call")
        if o == "list":
            if len({cs["orient"] for cs in call["cases"]}) == 8:
                e.add("every orientation in one call")
    return e
