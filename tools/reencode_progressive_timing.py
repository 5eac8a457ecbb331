"""Files per second of QsContext.reencode(progressive=True) (JPEG files to smoothed progressive JPEG files,
Pillow's save(progressive=True) on the GPU) against the sequential reencode(optimize=True) and today's
byte-identical alternative: decode_pixels to host memory followed by Pillow's save(progressive=True) on
the calling thread.  Also the progressive coder's share of the batch's device time and the run-resolution
kernel's time.

    python tools/reencode_progressive_timing.py [--reps 5] [--warmup 2] [--quick]

Workloads: 64 files of 1080p 4:2:0 q85, the 192-file web mix of tools/pixels_batch_timing.py and one
8K (7680 x 4320) 4:2:0 file, at -q 3, three iterations, whole pictures and thumbnails whose longest side
is 256 (BICUBIC); output quality 85, 4:2:0.  Arms:
  progressive       reencode(..., progressive=True)
  sequential opt    reencode(..., optimize=True)
  pillow            decode_pixels(device="cpu") then Image.fromarray(p).save(..., progressive=True) per file
Before timing, the progressive and pillow arms' bytes are checked equal for every file.  The arms
alternate within every rep (forward, then backward); the table gives medians after the warm-up reps of
the wall time around each arm.  A separate torch.profiler run of one batch per case sums the kernels'
device time.  Prints the card and its power limit, read in the same run."""
import argparse
import collections
import ctypes
import io
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")]

from pixels_batch_timing import card, jpeg, workloads  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--quick", action="store_true")
    a = ap.parse_args()
    import torch
    from PIL import Image, ImageFile
    ImageFile.MAXBLOCK = 1 << 28
    import jpegqs_b200 as qs
    from jpegqs_b200 import cuda
    flags, niter = qs.quality_to_flags(3) | qs.JPEGQS_TRANSCODE, 3
    ctx = cuda.QsContext(0)
    print(f"card: {card()}  ({ctx.device_name})")
    sets = workloads(a.quick)
    for k in [k for k in sets if k.startswith("256 x") or "progressive" in k]:
        sets.pop(k)
    sets["1 x 8K 4:2:0"] = [jpeg(7680, 4320, 0)]

    def thumbs(files):
        out = []
        for f in files:
            info = cuda._FileInfo()
            assert ctx.lib.jpegqs_cuda_transcode_route(f, len(f), None, ctypes.byref(info)) >= 0
            w, h = info.image_width, info.image_height
            m = max(w, h)
            out.append((max(1, round(w * 256 / m)), max(1, round(h * 256 / m))))
        return out

    def progressive(files, size):
        return [r[0] for r in ctx.reencode(files, flags, niter, 85, "4:2:0", size=size, progressive=True)]

    def sequential(files, size):
        return [r[0] for r in ctx.reencode(files, flags, niter, 85, "4:2:0", True, size=size)]

    def pillow(files, size):
        out = []
        for r in ctx.decode_pixels(files, flags, niter, device="cpu", size=size):
            p = r[0].numpy()
            b = io.BytesIO()
            Image.fromarray(p[..., 0] if p.shape[2] == 1 else p).save(b, "JPEG", quality=85, subsampling="4:2:0",
                                                                       progressive=True)
            out.append(b.getvalue())
        return out

    arms = collections.OrderedDict([("progressive", progressive), ("sequential opt", sequential), ("pillow", pillow)])
    cases = []
    for name, files in sets.items():
        for target, size in (("whole", None), ("256 longest side", thumbs(files))):
            cases.append((name, files, target, size))
    for name, files, target, size in cases:
        assert progressive(files, size) == pillow(files, size), (name, target)
    print("files checked: reencode(progressive=True) = Pillow's progressive save of decode_pixels(device='cpu')")

    keys = list(arms)
    print("\n| workload | target | " + " | ".join(f"{k}, files/s" for k in keys) + " |")
    print("|---|---|" + "---|" * len(keys))
    for name, files, target, size in cases:
        times = {k: [] for k in keys}
        for rep in range(a.warmup + a.reps):
            for k in (keys if rep % 2 == 0 else keys[::-1]):
                t0 = time.perf_counter()
                arms[k](files, size)
                if rep >= a.warmup:
                    times[k].append(time.perf_counter() - t0)
        print(f"| {name} | {target} | " + " | ".join(f"{len(files) / statistics.median(times[k]):.1f}" for k in keys) +
              " |", flush=True)

    from torch.profiler import ProfilerActivity, profile
    print("\n| workload | target | all kernels, ms | progressive coder (qp_), ms | share | qp_runs_kernel, ms | "
          "compressor, ms | sequential coder (qe_, optimize), ms |")
    print("|---|---|---|---|---|---|---|---|")
    per_kernel = collections.Counter()
    for name, files, target, size in cases:
        t = collections.Counter()
        for arm, tag in ((progressive, "p"), (sequential, "s")):
            arm(files, size)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                arm(files, size)
            for ev in prof.events():
                if ev.device_type != torch.autograd.DeviceType.CUDA:
                    continue
                us = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
                if tag == "p":
                    t["all"] += us
                    if ev.name.startswith("qp_"):
                        t["qp"] += us
                        if name.startswith("1 x 8K") and target == "whole":
                            per_kernel[ev.name.split("(")[0]] += us
                    if "qp_runs_kernel" in ev.name:
                        t["runs"] += us
                    if "qc_compress_kernel" in ev.name:
                        t["c"] += us
                elif ev.name.startswith("qe_"):
                    t["qe"] += us
        print(f"| {name} | {target} | {t['all'] / 1000:.3f} | {t['qp'] / 1000:.3f} | {t['qp'] / max(t['all'], 1):.1%} | "
              f"{t['runs'] / 1000:.3f} | {t['c'] / 1000:.3f} | {t['qe'] / 1000:.3f} |", flush=True)
    print("\n8K whole picture, progressive coder per kernel:\n\n| kernel | ms |\n|---|---|")
    for k, us in per_kernel.most_common():
        print(f"| {k} | {us / 1000:.3f} |")
    ctx.close()


if __name__ == "__main__":
    main()
