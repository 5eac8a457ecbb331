"""Files per second of the blur and sharpen filters on the GPU (decode_pixels / reencode with image_filter=,
Pillow's ImageFilter on the device) against the same calls without a filter and against the byte-identical
host route, and each filter kernel's device time against the HBM bound.

    python tools/image_filter_timing.py [--reps 5] [--warmup 2] [--quick]

Workloads: the 64 x 1080p 4:2:0 q85 batch and the 192-file web mix of tools/pixels_batch_timing.py, and one
8K (7680 x 4320) file, at -q 3, three iterations.  Arms, alternating within every rep (forward, then
backward), medians after the warm-up reps of the wall time around each arm:
  thumbnail + unsharp   reencode(thumbnail=(256, 256), image_filter=UnsharpMask(2, 150, 3)), quality 85
  thumbnail             the same call without a filter
  host                  decode_pixels(device="cpu", thumbnail=(256, 256)), then Pillow's filter and save
  full + gaussian       decode_pixels(image_filter=GaussianBlur(20)) at full size, on the device
  full                  the same call without a filter
Before timing, the first arm's bytes are checked against the host arm's.  A separate torch.profiler run
gives each filter kernel's device time; a pass reads and writes the picture once, so its HBM bound is
2 W H C bytes over 3.35 TB/s (H100 SXM data sheet), and the share is that bound over the kernel's time.
Prints the card and its power limit, read in the same run."""
import argparse
import collections
import io
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")]

from pixels_batch_timing import card, jpeg, workloads  # noqa: E402

HBM = 3.35e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--quick", action="store_true")
    a = ap.parse_args()
    import torch
    from PIL import Image, ImageFilter
    import jpegqs_b200 as qs
    from jpegqs_b200 import cuda
    flags, niter = qs.quality_to_flags(3) | qs.JPEGQS_TRANSCODE, 3
    ctx = cuda.QsContext(0)
    print(f"card: {card()}  ({ctx.device_name})")
    sets = workloads(a.quick)
    sets = {k: v for k, v in sets.items() if k.startswith("64 x") or "web" in k}
    big = {"1 x 8K": [jpeg(7680, 4320, 0)]}
    bound, unsharp, gauss = (256, 256), ImageFilter.UnsharpMask(2, 150, 3), ImageFilter.GaussianBlur(20)

    def thumb(files, f=None):
        return [r[0] for r in ctx.reencode(files, flags, niter, 85, "4:2:0", thumbnail=bound, image_filter=f)]

    def host(files):
        out = []
        for r in ctx.decode_pixels(files, flags, niter, device="cpu", thumbnail=bound):
            p = r[0].numpy()
            im = Image.fromarray(p[..., 0] if p.shape[2] == 1 else p).filter(unsharp)
            b = io.BytesIO()
            im.save(b, "JPEG", quality=85, subsampling="4:2:0")
            out.append(b.getvalue())
        return out

    def full(files, f=None):
        out = ctx.decode_pixels(files, flags, niter, image_filter=f)
        torch.cuda.synchronize()
        return out

    for name, files in sets.items():
        assert thumb(files, unsharp) == host(files), name
    print("files checked: reencode(thumbnail=, image_filter=UnsharpMask(2, 150, 3)) = decode_pixels(device='cpu', "
          "thumbnail=) + Pillow's filter and save")

    def table(arms, groups):
        keys = list(arms)
        print("\n| workload | " + " | ".join(f"{k}, files/s" for k in keys) + " |")
        print("|---|" + "---|" * len(keys))
        for name, files in groups.items():
            times = {k: [] for k in keys}
            for rep in range(a.warmup + a.reps):
                for k in (keys if rep % 2 == 0 else keys[::-1]):
                    t0 = time.perf_counter()
                    arms[k](files)
                    if rep >= a.warmup:
                        times[k].append(time.perf_counter() - t0)
            print(f"| {name} | " + " | ".join(f"{len(files) / statistics.median(times[k]):.1f}" for k in keys) + " |",
                  flush=True)

    table(collections.OrderedDict([("thumbnail + unsharp", lambda f: thumb(f, unsharp)), ("thumbnail", thumb),
                                   ("host", host)]), sets)
    table(collections.OrderedDict([("full + gaussian(20)", lambda f: full(f, gauss)), ("full", full)]),
          {**{k: v for k, v in sets.items() if k.startswith("64 x")}, **big})

    from torch.profiler import ProfilerActivity, profile
    print("\n| workload | arm | kernel | launches | device ms | HBM bound ms | share of HBM bound |\n|---|---|---|---|---|---|---|")
    runs = [(n, "thumbnail + unsharp", f, lambda f: thumb(f, unsharp)) for n, f in sets.items()]
    runs += [(n, "full + gaussian(20)", f, lambda f: full(f, gauss)) for n, f in {**sets, **big}.items()
             if not n.startswith("192")]
    for name, arm, files, fn in runs:
        if arm.startswith("thumb"):
            pics = []
            for f in files:
                w, h = Image.open(io.BytesIO(f)).size
                pics.append(cuda.thumbnail_geometry(w, h, bound)[1])
        else:
            pics = [Image.open(io.BytesIO(f)).size for f in files]
        pic_bytes = sum(w * h * 3 for w, h in pics)
        fn(files)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn(files)
        t, cnt = collections.Counter(), collections.Counter()
        for ev in prof.events():
            if ev.device_type != torch.autograd.DeviceType.CUDA or "qs_filter_" not in ev.name:
                continue
            k = ev.name.split("(")[0].replace("void ", "")
            t[k] += ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
            cnt[k] += 1
        for k in sorted(t):
            ms = t[k] / 1000
            b = 2 * pic_bytes * cnt[k] / HBM * 1000
            print(f"| {name} | {arm} | {k} | {cnt[k]} | {ms:.3f} | {b:.3f} | {b / ms:.0%} |", flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
