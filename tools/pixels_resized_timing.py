"""Files per second of QsContext.decode_pixels with size / crop / filter (the resize on the GPU, byte for
byte Pillow's crop().resize()), against today's byte-identical alternative: decode_pixels to host memory
followed by Pillow's crop().resize() on the calling thread.  Also the two resize kernels' device time.

    python tools/pixels_resized_timing.py [--reps 5] [--warmup 2] [--quick]

Workloads: 64 files of 1080p 4:2:0 q85 and the 192-file web mix of tools/pixels_batch_timing.py, at -q 3,
three iterations, scale_denom 1.  Targets: a 224 x 224 centre crop (the largest centred square) with
BILINEAR, as a training loader asks, and a thumbnail whose longest side is 256 with BICUBIC.  Arms:
  device   decode_pixels(size=..., crop=...) with device outputs
  host     the same with host outputs
  pillow   decode_pixels(device="cpu") then Image.fromarray(p).crop().resize() per file
  unresized device   decode_pixels with device outputs and no resize, for scale
Before timing, every arm's bytes are checked equal for every file.  The arms alternate within every rep
(forward, then backward); the table gives medians after the warm-up reps of the wall time around each
arm.  A separate torch.profiler run of one batch per workload and target sums the resize kernels' device
time.  Prints the card and its power limit."""
import argparse
import collections
import ctypes
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")]

from pixels_batch_timing import card, workloads  # noqa: E402


def centre_square(w, h):
    s = min(w, h)
    left, top = (w - s) // 2, (h - s) // 2
    return (left, top, left + s, top + s), (224, 224)


def longest_256(w, h):
    m = max(w, h)
    return None, (max(1, round(w * 256 / m)), max(1, round(h * 256 / m)))


TARGETS = collections.OrderedDict([("224x224 centre crop, bilinear", (centre_square, "bilinear")),
                                   ("256 longest side, bicubic", (longest_256, "bicubic"))])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--quick", action="store_true")
    a = ap.parse_args()
    import torch
    from PIL import Image
    import jpegqs_b200 as qs
    from jpegqs_b200 import cuda
    flags, niter = qs.quality_to_flags(3) | qs.JPEGQS_TRANSCODE, 3
    ctx = cuda.QsContext(0)
    print(f"card: {card()}  ({ctx.device_name})")
    sets = workloads(a.quick)
    for k in [k for k in sets if k.startswith("256 x") or "progressive" in k]:
        sets.pop(k)

    def plan(files, target):
        how, filt = TARGETS[target]
        shapes = []
        for f in files:
            info = cuda._FileInfo()
            assert ctx.lib.jpegqs_cuda_transcode_route(f, len(f), None, ctypes.byref(info)) >= 0
            shapes.append(how(info.image_width, info.image_height))
        return [c for c, _ in shapes], [s for _, s in shapes], filt

    def gpu(files, crops, sizes, filt, device):
        out = ctx.decode_pixels(files, flags, niter, device=device, size=sizes, crop=crops, filter=filt)
        torch.cuda.synchronize()
        return out

    def pillow(files, crops, sizes, filt):
        out = []
        resample = getattr(Image.Resampling, filt.upper())
        for r, c, s in zip(ctx.decode_pixels(files, flags, niter, device="cpu"), crops, sizes):
            p = r[0].numpy()
            im = Image.fromarray(p[..., 0] if p.shape[2] == 1 else p)
            if c is not None:
                im = im.crop(c)
            out.append(np.asarray(im.resize(s, resample)))
        return out

    arms = collections.OrderedDict([("device", lambda f, c, s, x: gpu(f, c, s, x, "cuda")),
                                    ("host", lambda f, c, s, x: gpu(f, c, s, x, "cpu")),
                                    ("pillow", pillow),
                                    ("unresized device", lambda f, c, s, x: gpu(f, None, None, x, "cuda"))])

    # correctness first: every arm's bytes, every file
    for name, files in sets.items():
        for target in TARGETS:
            crops, sizes, filt = plan(files, target)
            dev, host, pil = (arms[k](files, crops, sizes, filt) for k in ("device", "host", "pillow"))
            for d, h, p in zip(dev, host, pil):
                assert torch.equal(d[0].cpu(), h[0]), (name, target)
                assert np.array_equal(h[0].numpy().reshape(p.shape), p), (name, target)
    print("pixels checked: device outputs = host outputs = Pillow's crop().resize() of the host decode, every file")

    keys = list(arms)
    print("\n| workload | target | " + " | ".join(f"{k}, files/s" for k in keys) + " |")
    print("|---|---|" + "---|" * len(keys))
    for name, files in sets.items():
        for target in TARGETS:
            crops, sizes, filt = plan(files, target)
            times = {k: [] for k in keys}
            for rep in range(a.warmup + a.reps):
                for k in (keys if rep % 2 == 0 else keys[::-1]):
                    t0 = time.perf_counter()
                    arms[k](files, crops, sizes, filt)
                    dt = time.perf_counter() - t0
                    if rep >= a.warmup:
                        times[k].append(dt)
            med = {k: statistics.median(v) for k, v in times.items()}
            print(f"| {name} | {target} | " + " | ".join(f"{len(files) / med[k]:.0f}" for k in keys) + " |", flush=True)

    from torch.profiler import ProfilerActivity, profile
    print("\n| workload | target | horizontal pass, ms | vertical pass, ms | render, ms |")
    print("|---|---|---|---|---|")
    for name, files in sets.items():
        for target in TARGETS:
            crops, sizes, filt = plan(files, target)
            gpu(files, crops, sizes, filt, "cuda")
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                gpu(files, crops, sizes, filt, "cuda")
            t = collections.Counter()
            for ev in prof.events():
                if ev.device_type != torch.autograd.DeviceType.CUDA:
                    continue
                us = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
                for key in ("qs_resize_h_kernel", "qs_resize_v_kernel", "qs_render_async_kernel"):
                    if key in ev.name:
                        t[key] += us
            print(f"| {name} | {target} | {t['qs_resize_h_kernel'] / 1000:.3f} | {t['qs_resize_v_kernel'] / 1000:.3f} | "
                  f"{t['qs_render_async_kernel'] / 1000:.3f} |", flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
