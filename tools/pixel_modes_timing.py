"""Device time of the render kernel with a colour mode, and files per second of decode_pixels(mode="RGB") on a
mix holding about 1 % CMYK files against today's workaround: transcode_batch, then Pillow's
Image.open().convert("RGB") of every file on the calling thread.

    python tools/pixel_modes_timing.py [--reps 5] [--warmup 2] [--iters 20] [--quick]

Render: CUDA events around `iters` back-to-back calls of jpegqs_cuda_render_mode_async on device coefficients
(the host reader's, de-quantized by the render), for 64 x 1080p CMYK 4:4:4, YCCK with Y and K 2x2 over 1x1
Cb and Cr, and YCbCr 4:2:0 files; the YCbCr row also times the existing jpegqs_cuda_render_async.  The
calls alternate within every rep; each figure is the median over the reps after the warm-up reps, in ms per
call.  decode_pixels: 99 1080p YCbCr files and one CMYK file, at -q 3, three iterations, device outputs;
before timing, its pixels are checked equal to the workaround's for every file.  Prints the card and its
power limit."""
import argparse
import collections
import ctypes
import io
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")]

from pixels_batch_timing import card, jpeg  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--quick", action="store_true")
    a = ap.parse_args()
    import torch
    from PIL import Image
    import jpegqs_b200 as qs
    from jpegqs_b200 import cuda
    from decode_files import pillow_jpeg
    from test_pixel_modes_cpu import YCCK_FACTORS, ycck_file
    flags, niter = qs.quality_to_flags(3) | qs.JPEGQS_TRANSCODE, 3
    ctx = cuda.QsContext(0)
    print(f"card: {card()}  ({ctx.device_name})")
    k = 8 if a.quick else 1
    n = 64 // k
    sets = collections.OrderedDict([
        (f"{n} x 1080p CMYK 4:4:4", [pillow_jpeg(1920, 1080, "CMYK", i, quality=85) for i in range(n)]),
        (f"{n} x 1080p YCCK, Y and K 2x2", [ycck_file(1920, 1080, YCCK_FACTORS["y2k2"], seed=i) for i in range(n)]),
        (f"{n} x 1080p YCbCr 4:2:0", [jpeg(1920, 1080, i % 8) for i in range(n)])])

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

    print("\n| workload | mode RGB, ms | mode L, ms | render_async, ms |")
    print("|---|---|---|---|")
    for name, files in sets.items():
        ims = [cuda.read_jpeg(f) for f in files]
        coefs = [[torch.from_numpy(np.ascontiguousarray(c.coef)).cuda() for c in im.comps] for im in ims]
        arr = cuda._image_array(ims, [[t.data_ptr() for t in cs] for cs in coefs])
        cs = (ctypes.c_int32 * len(ims))(*[im.colorspace for im in ims])
        outs = [torch.empty(im.height * im.width * 3, dtype=torch.uint8, device="cuda") for im in ims]
        ptrs = (ctypes.c_void_p * len(ims))(*[t.data_ptr() for t in outs])
        calls = collections.OrderedDict()
        for m in (1, 2):
            calls[m] = (lambda m: lambda s: ctx.lib.jpegqs_cuda_render_mode_async(ctx.h, len(ims), arr, None, 0, 1, None,
                                                                                 cs, m, ptrs, s))(m)
        if len(ims[0].comps) == 3:
            calls["async"] = lambda s: ctx.lib.jpegqs_cuda_render_async(ctx.h, len(ims), arr, None, 0, ptrs, s)
        keys = list(calls)
        times = {x: [] for x in keys}
        for rep in range(a.warmup + a.reps):
            for x in (keys if rep % 2 == 0 else keys[::-1]):
                dt = time_calls(calls[x], a.iters)
                if rep >= a.warmup:
                    times[x].append(dt)
        med = {x: statistics.median(v) for x, v in times.items()}
        print(f"| {name} | {med[1]:.3f} | {med[2]:.3f} | " + (f"{med['async']:.3f}" if "async" in med else "-") + " |",
              flush=True)
        del coefs, outs

    nf = 100 // k
    files = [jpeg(1920, 1080, i % 8) for i in range(nf - 1)]
    files.insert(nf // 2, pillow_jpeg(1920, 1080, "CMYK", 3, quality=85))

    def workaround():
        return [np.asarray(Image.open(io.BytesIO(d)).convert("RGB")) for d, _ in ctx.transcode_batch(files, flags, niter)]

    arms = collections.OrderedDict([
        ('decode_pixels(mode="RGB")', lambda: (ctx.decode_pixels(files, flags, niter, mode="RGB"), torch.cuda.synchronize())),
        ("transcode_batch + Pillow convert", workaround)])
    got = ctx.decode_pixels(files, flags, niter, mode="RGB")
    for g, p in zip(got, workaround()):
        assert np.array_equal(g[0].cpu().numpy(), p)
    print(f"\npixels checked: decode_pixels(mode=\"RGB\") = Pillow's convert of the transcoded file, all {nf} files")
    keys = list(arms)
    times = {x: [] for x in keys}
    for rep in range(a.warmup + a.reps):
        for x in (keys if rep % 2 == 0 else keys[::-1]):
            t0 = time.perf_counter()
            arms[x]()
            dt = time.perf_counter() - t0
            if rep >= a.warmup:
                times[x].append(dt)
    print(f"\n| {nf} x 1080p, 1 CMYK | " + " | ".join(f"{x}, files/s" for x in keys) + " |")
    print("|---|" + "---|" * len(keys))
    print("| -q 3 -n 3 | " + " | ".join(f"{nf / statistics.median(times[x]):.0f}" for x in keys) + " |")
    ctx.close()


if __name__ == "__main__":
    main()
