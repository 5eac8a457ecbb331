"""Files per second of QsContext.reencode(thumbnail=(256, 256)) (Pillow's Image.thumbnail, then save, on the
GPU) against the byte-identical host route - decode_pixels(device="cpu"), then Pillow's thumbnail and save
on the calling thread - and against reencode(size=...) with the same output sizes (one scale, no reduce,
not Pillow's thumbnail bytes).  Also the reduce kernel's device time.

    python tools/thumbnail_timing.py [--reps 5] [--warmup 2] [--quick]

Workloads: 64 files of 1080p 4:2:0 q85 and the 192-file web mix of tools/pixels_batch_timing.py, at -q 3,
three iterations; output quality 85, 4:2:0.  Arms:
  thumbnail     reencode(..., thumbnail=(256, 256))  (reducing_gap 2.0: draft scale, then reduce and resize)
  host          decode_pixels(device="cpu") then Image.fromarray(p).thumbnail(...) and save per file
  size          reencode(..., size=thumbnail sizes)  (today's call: full-size render, one resize)
Before timing, the thumbnail arm's bytes are checked against the host arm's.  The arms alternate within
every rep (forward, then backward); the table gives medians after the warm-up reps of the wall time around
each arm.  A separate torch.profiler run sums the reduce kernel's device time for the thumbnail arm, and for
thumbnail with orientation=1 (a loaded picture: no draft, the whole shrink is the reduce).  Prints the card
and its power limit, read in the same run."""
import argparse
import collections
import io
import os
import statistics
import sys
import time

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
    from PIL import Image
    import jpegqs_b200 as qs
    from jpegqs_b200 import cuda
    flags, niter = qs.quality_to_flags(3) | qs.JPEGQS_TRANSCODE, 3
    ctx = cuda.QsContext(0)
    print(f"card: {card()}  ({ctx.device_name})")
    sets = workloads(a.quick)
    sets = {k: v for k, v in sets.items() if k.startswith("64 x") or "web" in k}
    bound = (256, 256)

    def thumbnail(files, orientation=None):
        return [r[0] for r in ctx.reencode(files, flags, niter, 85, "4:2:0", thumbnail=bound, orientation=orientation)]

    def host(files):
        # Pillow's thumbnail of the decoded picture: a loaded picture, so no draft
        out = []
        for r in ctx.decode_pixels(files, flags, niter, device="cpu"):
            p = r[0].numpy()
            im = Image.fromarray(p[..., 0] if p.shape[2] == 1 else p)
            im.thumbnail(bound)
            b = io.BytesIO()
            im.save(b, "JPEG", quality=85, subsampling="4:2:0")
            out.append(b.getvalue())
        return out

    def sizes_of(files):
        out = []
        for f in files:
            w, h = Image.open(io.BytesIO(f)).size
            out.append(cuda.thumbnail_geometry(w, h, bound)[1])
        return out

    size_cache = {}

    def size(files):
        key = id(files)
        if key not in size_cache:
            size_cache[key] = sizes_of(files)
        return [r[0] for r in ctx.reencode(files, flags, niter, 85, "4:2:0", size=size_cache[key])]

    # the thumbnail arm with orientation 1 loads the picture, as host's fromarray does: equal bytes
    for name, files in sets.items():
        assert thumbnail(files, orientation=1) == host(files), name
    print("files checked: reencode(thumbnail=, orientation=1) = Pillow's thumbnail and save of decode_pixels(device='cpu')")

    arms = collections.OrderedDict([("thumbnail", thumbnail), ("thumbnail, orientation=1", lambda f: thumbnail(f, 1)),
                                    ("host", host), ("size", size)])
    keys = list(arms)
    print("\n| workload | " + " | ".join(f"{k}, files/s" for k in keys) + " |")
    print("|---|" + "---|" * len(keys))
    for name, files in sets.items():
        times = {k: [] for k in keys}
        for rep in range(a.warmup + a.reps):
            for k in (keys if rep % 2 == 0 else keys[::-1]):
                t0 = time.perf_counter()
                arms[k](files)
                if rep >= a.warmup:
                    times[k].append(time.perf_counter() - t0)
        print(f"| {name} | " + " | ".join(f"{len(files) / statistics.median(times[k]):.1f}" for k in keys) + " |",
              flush=True)

    from torch.profiler import ProfilerActivity, profile
    print("\n| workload | arm | all kernels, ms | qs_reduce_kernel, ms | resize kernels, ms |\n|---|---|---|---|---|")
    for name, files in sets.items():
        for arm in ("thumbnail", "thumbnail, orientation=1"):
            arms[arm](files)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                arms[arm](files)
            t = collections.Counter()
            for ev in prof.events():
                if ev.device_type != torch.autograd.DeviceType.CUDA:
                    continue
                us = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
                t["all"] += us
                if "qs_reduce_kernel" in ev.name:
                    t["reduce"] += us
                if "qs_resize_" in ev.name:
                    t["resize"] += us
            print(f"| {name} | {arm} | {t['all'] / 1000:.3f} | {t['reduce'] / 1000:.3f} | {t['resize'] / 1000:.3f} |",
                  flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
