"""Device time of the render kernel per EXIF orientation, and files per second of decode_pixels with
orientation="exif" against today's byte-identical alternative: decode_pixels to host memory followed by
Pillow's transpose on the calling thread.

    python tools/pixels_oriented_timing.py [--reps 5] [--warmup 2] [--iters 20] [--quick] [--parent-lib PATH]

Render: CUDA events around `iters` back-to-back calls of jpegqs_cuda_render_oriented_async on device
coefficients (the host reader's, de-quantized by the render) for orientations 1, 3 and 6, and of the
existing jpegqs_cuda_render_async, on the 8K file of the test suite and on 64 x 1080p 4:2:0 q85 files.
--parent-lib names a build of the library from before orientation existed; its render_async is timed in
the same process, alternating with this build's, as the no-regression check.  Each row is the median over
the reps after the warm-up reps, in ms per call.
decode_pixels: the 64 x 1080p files with an EXIF APP1 tagged 6, at -q 3, three iterations, device outputs,
for orientation=None, orientation="exif", and host outputs + Pillow's Image.transpose(ROTATE_270) (what
ImageOps.exif_transpose applies).  The arms alternate within every rep; medians of the wall time.  Before
timing, the "exif" pixels are checked equal to the Pillow arm's for every file.  Prints the card and its
power limit."""
import argparse
import collections
import ctypes
import os
import statistics
import struct
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")]

from pixels_batch_timing import card, jpeg  # noqa: E402


def tagged(data: bytes, o: int) -> bytes:
    """data with an EXIF APP1 (IFD0: Orientation o) after its SOI"""
    tiff = b"II*\0" + struct.pack("<LH", 8, 1) + struct.pack("<HHLHH", 0x0112, 3, 1, o, 0) + b"\0\0\0\0"
    payload = b"Exif\0\0" + tiff
    return data[:2] + b"\xff\xe1" + struct.pack(">H", len(payload) + 2) + payload + data[2:]


def render_lib(path):
    """the render entry points of a library build, loaded on their own (an older build lacks the rest)"""
    lib = ctypes.CDLL(path)
    lib.jpegqs_cuda_create.argtypes = [ctypes.c_int, ctypes.POINTER(ctypes.c_void_p)]
    lib.jpegqs_cuda_destroy.argtypes = [ctypes.c_void_p]
    lib.jpegqs_cuda_render_async.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                                             ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
    if hasattr(lib, "jpegqs_cuda_render_oriented_async"):
        lib.jpegqs_cuda_render_oriented_async.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p,
                                                          ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                                          ctypes.c_void_p, ctypes.c_void_p]
    h = ctypes.c_void_p()
    assert lib.jpegqs_cuda_create(0, ctypes.byref(h)) == 0
    return lib, h


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--parent-lib", default=None)
    a = ap.parse_args()
    import torch
    from PIL import Image
    import jpegqs_b200 as qs
    from jpegqs_b200 import cuda
    from test_cli import _big_picture
    import io
    flags, niter = qs.quality_to_flags(3) | qs.JPEGQS_TRANSCODE, 3
    ctx = cuda.QsContext(0)
    print(f"card: {card()}  ({ctx.device_name})")
    k = 4 if a.quick else 1
    b = io.BytesIO()
    _big_picture(7680, 4320, 5).save(b, "JPEG", quality=90)
    sets = collections.OrderedDict([("8K 4:2:0 q90", [b.getvalue()]),
                                    (f"{64 // k} x 1080p q85", [jpeg(1920, 1080, i % 8) for i in range(64 // k)])])

    libs = collections.OrderedDict([("this build", (ctx.lib, ctx.h))])
    if a.parent_lib:
        libs["parent"] = render_lib(a.parent_lib)

    def render_setup(files):
        ims = [cuda.read_jpeg(f) for f in files]
        coefs = [[torch.from_numpy(np.ascontiguousarray(c.coef)).cuda() for c in im.comps] for im in ims]
        arr = cuda._image_array(ims, [[t.data_ptr() for t in cs] for cs in coefs])
        outs = {}
        for o in (1, 3, 6):
            ts = [torch.empty(im.height * im.width * 3, dtype=torch.uint8, device="cuda") for im in ims]
            outs[o] = (ts, (ctypes.c_void_p * len(ims))(*[t.data_ptr() for t in ts]))
        return ims, coefs, arr, outs

    # every call on one explicit stream, with the events: a NULL stream would be each context's own
    st = torch.cuda.Stream()
    handle = ctypes.c_void_p(st.cuda_stream)

    def time_calls(call, iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        rcs = [call(handle) for _ in range(iters)]
        e1.record(st)
        e1.synchronize()
        assert not any(rcs), rcs
        return e0.elapsed_time(e1) / iters

    print("\n| workload | " + " | ".join(["orientation 1, ms", "orientation 3, ms", "orientation 6, ms"] +
                                          [f"render_async ({k}), ms" for k in libs]) + " |")
    print("|---|" + "---|" * (3 + len(libs)))
    for name, files in sets.items():
        ims, coefs, arr, outs = render_setup(files)
        n = len(ims)
        calls = collections.OrderedDict()
        for o in (1, 3, 6):
            ors = (ctypes.c_int32 * n)(*([o] * n))
            calls[f"o{o}"] = (lambda ors, ptrs: lambda s: ctx.lib.jpegqs_cuda_render_oriented_async(
                ctx.h, n, arr, None, 0, 1, ors, ptrs, s))(ors, outs[o][1])
        for key, (lib, h) in libs.items():
            calls[key] = (lambda lib, h: lambda s: lib.jpegqs_cuda_render_async(h, n, arr, None, 0, outs[1][1], s))(lib, h)
        # the orientations' pixels: Pillow's transpose of orientation 1's
        for c in calls.values():
            assert c(handle) == 0
        st.synchronize()
        base = [t.cpu().numpy().reshape(im.height, im.width, 3) for t, im in zip(outs[1][0], ims)]
        for o, m in ((3, Image.Transpose.ROTATE_180), (6, Image.Transpose.ROTATE_270)):
            for t, p in zip(outs[o][0], base):
                want = np.asarray(Image.fromarray(p).transpose(m))
                assert np.array_equal(t.cpu().numpy().reshape(want.shape), want), (name, o)
        keys = list(calls)
        times = {x: [] for x in keys}
        for rep in range(a.warmup + a.reps):
            for x in (keys if rep % 2 == 0 else keys[::-1]):
                dt = time_calls(calls[x], a.iters)
                if rep >= a.warmup:
                    times[x].append(dt)
        med = {x: statistics.median(v) for x, v in times.items()}
        print(f"| {name} | " + " | ".join(f"{med[x]:.3f}" for x in keys) + " |", flush=True)
        del coefs, outs
    for key, (lib, h) in libs.items():
        if key != "this build":
            lib.jpegqs_cuda_destroy(h)

    files = [tagged(f, 6) for f in sets[f"{64 // k} x 1080p q85"]]

    def pillow():
        return [np.asarray(Image.fromarray(r[0].numpy()).transpose(Image.Transpose.ROTATE_270))
                for r in ctx.decode_pixels(files, flags, niter, device="cpu")]

    arms = collections.OrderedDict([
        ("orientation=None", lambda: (ctx.decode_pixels(files, flags, niter), torch.cuda.synchronize())),
        ('orientation="exif"', lambda: (ctx.decode_pixels(files, flags, niter, orientation="exif"),
                                        torch.cuda.synchronize())),
        ("host decode + Pillow transpose", pillow)])
    got = ctx.decode_pixels(files, flags, niter, orientation="exif")
    for g, p in zip(got, pillow()):
        assert np.array_equal(g[0].cpu().numpy(), p)
    print("\npixels checked: decode_pixels(orientation=\"exif\") = Pillow's transpose of the host decode, every file")
    keys = list(arms)
    times = {x: [] for x in keys}
    for rep in range(a.warmup + a.reps):
        for x in (keys if rep % 2 == 0 else keys[::-1]):
            t0 = time.perf_counter()
            arms[x]()
            dt = time.perf_counter() - t0
            if rep >= a.warmup:
                times[x].append(dt)
    print(f"\n| {len(files)} x 1080p tagged 6 | " + " | ".join(f"{x}, files/s" for x in keys) + " |")
    print("|---|" + "---|" * len(keys))
    print("| decode_pixels | " + " | ".join(f"{len(files) / statistics.median(times[x]):.0f}" for x in keys) + " |")
    ctx.close()


if __name__ == "__main__":
    main()
