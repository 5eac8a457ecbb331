"""Files per second of QsContext.reencode (JPEG files to smoothed JPEG files, Pillow's save on the GPU) against
today's byte-identical alternative: decode_pixels to host memory followed by Pillow's Image.save on the
calling thread.  Also the mean output size, the size of the jpegqs tool's files (transcode_batch, every
quantization value 1) for comparison, and the compressor and encoder kernels' device time.

    python tools/reencode_timing.py [--reps 5] [--warmup 2] [--quick]

Workloads: 64 files of 1080p 4:2:0 q85 and the 192-file web mix of tools/pixels_batch_timing.py, at -q 3,
three iterations, whole pictures and thumbnails whose longest side is 256 (BICUBIC); output quality 85,
4:2:0, with optimize off and on.  Arms:
  reencode          reencode(...), host outputs
  pillow            decode_pixels(device="cpu") then Image.fromarray(p).save(...) per file
  pixels device     decode_pixels with device outputs and the same size, for scale
Before timing, the reencode and pillow arms' bytes are checked equal for every file.  The arms alternate
within every rep (forward, then backward); the table gives medians after the warm-up reps of the wall
time around each arm.  A separate torch.profiler run of one batch per case sums the kernels' device
time.  Prints the card and its power limit, read in the same run."""
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

from pixels_batch_timing import card, workloads  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--quick", action="store_true")
    a = ap.parse_args()
    import torch
    from PIL import Image, ImageFile
    ImageFile.MAXBLOCK = 1 << 28      # Pillow's optimize needs the whole file in one buffer
    import jpegqs_b200 as qs
    from jpegqs_b200 import cuda
    flags, niter = qs.quality_to_flags(3) | qs.JPEGQS_TRANSCODE, 3
    ctx = cuda.QsContext(0)
    print(f"card: {card()}  ({ctx.device_name})")
    sets = workloads(a.quick)
    for k in [k for k in sets if k.startswith("256 x") or "progressive" in k]:
        sets.pop(k)

    def thumbs(files):
        out = []
        for f in files:
            info = cuda._FileInfo()
            assert ctx.lib.jpegqs_cuda_transcode_route(f, len(f), None, ctypes.byref(info)) >= 0
            w, h = info.image_width, info.image_height
            m = max(w, h)
            out.append((max(1, round(w * 256 / m)), max(1, round(h * 256 / m))))
        return out

    def reencode(files, size, opt):
        return [r[0] for r in ctx.reencode(files, flags, niter, 85, "4:2:0", opt, size=size)]

    def pillow(files, size, opt):
        out = []
        for r in ctx.decode_pixels(files, flags, niter, device="cpu", size=size):
            p = r[0].numpy()
            b = io.BytesIO()
            Image.fromarray(p[..., 0] if p.shape[2] == 1 else p).save(b, "JPEG", quality=85, subsampling="4:2:0", optimize=opt)
            out.append(b.getvalue())
        return out

    def pixels(files, size, opt):
        out = ctx.decode_pixels(files, flags, niter, size=size)
        torch.cuda.synchronize()
        return out

    arms = collections.OrderedDict([("reencode", reencode), ("pillow", pillow), ("pixels device", pixels)])
    cases = []
    for name, files in sets.items():
        for target, size in (("whole", None), ("256 longest side", thumbs(files))):
            for opt in (False, True):
                cases.append((name, files, target, size, opt))

    for name, files, target, size, opt in cases:
        assert reencode(files, size, opt) == pillow(files, size, opt), (name, target, opt)
    print("files checked: reencode = Pillow's save of decode_pixels(device='cpu'), every file, every case")

    keys = list(arms)
    print("\n| workload | target | optimize | " + " | ".join(f"{k}, files/s" for k in keys) +
          " | reencode, mean bytes | jpegqs tool's file, mean bytes |")
    print("|---|---|---|" + "---|" * (len(keys) + 2))
    tool_bytes = {}
    for name, files, target, size, opt in cases:
        if name not in tool_bytes:
            tool_bytes[name] = np.mean([len(b) for b, _ in ctx.transcode_batch(files, flags, niter)])
        times = {k: [] for k in keys}
        for rep in range(a.warmup + a.reps):
            for k in (keys if rep % 2 == 0 else keys[::-1]):
                t0 = time.perf_counter()
                arms[k](files, size, opt)
                dt = time.perf_counter() - t0
                if rep >= a.warmup:
                    times[k].append(dt)
        med = {k: statistics.median(v) for k, v in times.items()}
        mean = np.mean([len(b) for b in reencode(files, size, opt)])
        tb = f"{tool_bytes[name]:.0f}" if target == "whole" else "-"
        print(f"| {name} | {target} | {int(opt)} | " + " | ".join(f"{len(files) / med[k]:.0f}" for k in keys) +
              f" | {mean:.0f} | {tb} |", flush=True)

    from torch.profiler import ProfilerActivity, profile
    print("\n| workload | target | optimize | compressor, ms | encoder (all qe_ kernels), ms | render, ms | files |")
    print("|---|---|---|---|---|---|---|")
    for name, files, target, size, opt in cases:
        reencode(files, size, opt)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            reencode(files, size, opt)
        t = collections.Counter()
        for ev in prof.events():
            if ev.device_type != torch.autograd.DeviceType.CUDA:
                continue
            us = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
            if "qc_compress_kernel" in ev.name:
                t["c"] += us
            elif "qe_" in ev.name and "kernel" in ev.name:
                t["e"] += us
            elif "qs_render_async_kernel" in ev.name:
                t["r"] += us
        print(f"| {name} | {target} | {int(opt)} | {t['c'] / 1000:.3f} | {t['e'] / 1000:.3f} | {t['r'] / 1000:.3f} | "
              f"{len(files)} |", flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
