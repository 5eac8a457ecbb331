"""Files per second of QsContext.decode_pixels (JPEG files to smoothed pixels, many files per launch)
against the same call one file at a time, and against the host path the jpegqs tool's --ppm takes
(read_jpeg + do_quantsmooth + render_rgb per file).

    python tools/pixels_batch_timing.py [--reps 5] [--warmup 2] [--quick] [--profile-dir DIR]

Workloads (seeded pictures, 8 distinct per set, repeated): 256 files of 256x256, 64 of 1080p 4:2:0 q85,
192 "web" files of mixed sizes, and 16 of 1080p progressive without restart markers (all of which the
host reader decodes).  -q 3, three iterations.  The three arms alternate within every rep, and the
table gives medians after the warm-up reps of the wall time around each arm: decode_pixels returns when
every tensor is complete on the device; the host path when every array is in host memory.  Before
timing, every file's pixels are checked to be equal across the arms.  A torch.profiler run of one batch
per workload gives the per-kernel split (--profile-dir also writes its Chrome traces).  Prints the card
and its power limit."""
import argparse
import collections
import io
import os
import statistics
import subprocess
import sys
import time

import numpy as np
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def picture(w, h, seed):
    rng = np.random.RandomState(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float32)
    a = np.stack([128 + 70 * np.sin(x / 31.0) + 40 * np.cos(y / 19.0), 128 + 60 * np.cos((x + y) / 47.0),
                  128 + 80 * np.sin((x - y) / 23.0)], -1) + rng.normal(0, 9, (h, w, 3)).astype(np.float32)
    return Image.fromarray(a.clip(0, 255).astype(np.uint8), "RGB")


def jpeg(w, h, seed, quality=85, **kw):
    b = io.BytesIO()
    picture(w, h, seed).save(b, "JPEG", quality=quality, **kw)
    return b.getvalue()


def workloads(quick):
    k = 4 if quick else 1
    sets = collections.OrderedDict()
    sets["256 x 256x256"] = [jpeg(256, 256, i % 8) for i in range(256 // k)]
    sets["64 x 1080p q85"] = [jpeg(1920, 1080, i % 8) for i in range(64 // k)]
    rng = np.random.RandomState(1)
    sizes = [(320, 240), (480, 320), (640, 480), (800, 600), (1024, 768), (1280, 720), (1280, 960), (1920, 1080)]
    pool = {s: [jpeg(s[0], s[1], i, quality=int(rng.randint(70, 95))) for i in range(2)] for s in sizes}
    sets["192 x web mix"] = [pool[sizes[rng.randint(len(sizes))]][rng.randint(2)] for _ in range(192 // k)]
    sets["16 x 1080p progressive, no restarts"] = [jpeg(1920, 1080, i % 8, progressive=True) for i in range(16 // k)]
    return sets


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except Exception as e:            # noqa: BLE001 - the card line is informative only
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--profile-dir", default=None)
    a = ap.parse_args()
    import torch
    import jpegqs_b200 as qs
    from jpegqs_b200 import cuda
    flags, niter = qs.quality_to_flags(3) | qs.JPEGQS_TRANSCODE, 3
    ctx = cuda.QsContext(0)
    print(f"card: {card()}  ({ctx.device_name})")
    sets = workloads(a.quick)

    def host_path(f):
        _, out = ctx.do_quantsmooth(cuda.read_jpeg(f), flags, niter)
        rgb = ctx.render_rgb(out)
        return rgb[..., :1] if len(out.comps) == 1 else rgb

    arms = collections.OrderedDict()
    arms["decode_pixels, batch"] = lambda files: (ctx.decode_pixels(files, flags, niter), torch.cuda.synchronize())
    arms["decode_pixels, one file per call"] = lambda files: ([ctx.decode_pixels([f], flags, niter) for f in files],
                                                              torch.cuda.synchronize())
    arms["read_jpeg + do_quantsmooth + render_rgb"] = lambda files: [host_path(f) for f in files]

    print("\n| workload | " + " | ".join(f"{k}, files/s" for k in arms) + " | batch vs host path |")
    print("|---|" + "---|" * (len(arms) + 1))
    for name, files in sets.items():
        batch = ctx.decode_pixels(files, flags, niter)
        for f, rec in zip(files, batch):
            one = ctx.decode_pixels([f], flags, niter)[0]
            assert torch.equal(one[0], rec[0]) and one[1:] == rec[1:], name
            assert np.array_equal(host_path(f), rec[0].cpu().numpy()), name
        times = {k: [] for k in arms}
        keys = list(arms)
        for rep in range(a.warmup + a.reps):
            for k in (keys if rep % 2 == 0 else keys[::-1]):
                t0 = time.perf_counter()
                arms[k](files)
                dt = time.perf_counter() - t0
                if rep >= a.warmup:
                    times[k].append(dt)
        med = {k: statistics.median(v) for k, v in times.items()}
        print(f"| {name} | " + " | ".join(f"{len(files) / med[k]:.0f}" for k in arms) +
              f" | {med[keys[2]] / med[keys[0]]:.2f}x |", flush=True)

    from torch.profiler import ProfilerActivity, profile
    for j, (name, files) in enumerate(sets.items()):
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            ctx.decode_pixels(files, flags, niter)
            torch.cuda.synchronize()
        if a.profile_dir:
            os.makedirs(a.profile_dir, exist_ok=True)
            prof.export_chrome_trace(os.path.join(a.profile_dir, f"pixels_batch_{j}.json"))
        tot = collections.Counter()
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA:
                key = ev.name if len(ev.name) < 60 else ev.name[:57] + "..."
                tot[key] += ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
        s = sum(tot.values())
        print(f"\nprofile of one decode_pixels batch, {name}: {s / 1000:.2f} ms of device activity")
        for k, v in tot.most_common(10):
            print(f"  {v / 1000:8.3f} ms  {100 * v / max(s, 1):5.1f} %  {k}")
    ctx.close()


if __name__ == "__main__":
    main()
