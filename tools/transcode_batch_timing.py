"""Files per second of QsContext.transcode_batch (many files per launch) against a loop of
QsContext.transcode (one file per call), and of the `jpegqs --batch` process.

    python tools/transcode_batch_timing.py [--reps 5] [--warmup 2] [--before-exe PATH] [--quick]

Workloads (seeded pictures, 8 distinct per set, repeated): 256 files of 256x256, 256 of 640x480, 64 of
1080p 4:2:0 q85, and 192 "web" files of mixed sizes.  The two arms alternate within every rep; the table
gives medians after the warm-up reps:
  - wall: time around the call (both arms return only when every file is back in host memory);
  - run_async: device time of the smoothing kernels by CUDA events (jpegqs_cuda_last_device_ms), summed
    over the loop's calls for the loop arm, and the batch call's own (one sub-batch) for the batch arm.
A torch.profiler run of one batch per workload gives the per-kernel split.  The tool part times whole
`jpegqs -q 3 --batch` processes on the 64 x 1080p and 256 x 256x256 sets with this tree's tool, and with
--before-exe (a tool built from the previous commit, which transcodes one pair per call) when given.
Prints the card and its power limit."""
import argparse
import collections
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
EXE = os.path.join(ROOT, "jpeg-quantsmooth_b200", "csrc", "jpegqs")


def picture(w, h, seed):
    rng = np.random.RandomState(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float32)
    a = np.stack([128 + 70 * np.sin(x / 31.0) + 40 * np.cos(y / 19.0), 128 + 60 * np.cos((x + y) / 47.0),
                  128 + 80 * np.sin((x - y) / 23.0)], -1) + rng.normal(0, 9, (h, w, 3)).astype(np.float32)
    return Image.fromarray(a.clip(0, 255).astype(np.uint8), "RGB")


def jpeg(w, h, seed, quality=85):
    import io
    b = io.BytesIO()
    picture(w, h, seed).save(b, "JPEG", quality=quality)
    return b.getvalue()


def workloads(quick):
    k = 4 if quick else 1
    sets = collections.OrderedDict()
    sets["256 x 256x256"] = [jpeg(256, 256, i % 8) for i in range(256 // k)]
    sets["256 x 640x480"] = [jpeg(640, 480, i % 8) for i in range(256 // k)]
    sets["64 x 1080p q85"] = [jpeg(1920, 1080, i % 8) for i in range(64 // k)]
    rng = np.random.RandomState(1)
    sizes = [(320, 240), (480, 320), (640, 480), (800, 600), (1024, 768), (1280, 720), (1280, 960), (1920, 1080)]
    pool = {s: [jpeg(s[0], s[1], i, quality=int(rng.randint(70, 95))) for i in range(2)] for s in sizes}
    sets["192 x web mix"] = [pool[sizes[rng.randint(len(sizes))]][rng.randint(2)] for _ in range(192 // k)]
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
    ap.add_argument("--before-exe", default=None)
    ap.add_argument("--quick", action="store_true")
    a = ap.parse_args()
    import jpegqs_b200 as qs
    from jpegqs_b200 import cuda
    flags = qs.quality_to_flags(3) | qs.JPEGQS_TRANSCODE
    ctx = cuda.QsContext(0)
    print(f"card: {card()}  ({ctx.device_name})")
    sets = workloads(a.quick)

    print("\n| workload | loop of transcode, files/s | transcode_batch, files/s | speed-up | run_async ms, loop / batch |")
    print("|---|---|---|---|---|")
    for name, files in sets.items():
        want = ctx.transcode_batch(files, flags, 3)
        assert all(w == ctx.transcode(f, flags, 3) for w, f in zip(want, files)), name
        t_loop, t_batch, d_loop, d_batch = [], [], [], []
        for rep in range(a.warmup + a.reps):
            order = ("loop", "batch") if rep % 2 == 0 else ("batch", "loop")
            for arm in order:
                if arm == "loop":
                    dev = 0.0
                    t0 = time.perf_counter()
                    for f in files:
                        ctx.transcode(f, flags, 3)
                        dev += ctx.last_device_ms
                    dt = time.perf_counter() - t0
                    if rep >= a.warmup:
                        t_loop.append(dt); d_loop.append(dev)
                else:
                    t0 = time.perf_counter()
                    ctx.transcode_batch(files, flags, 3)
                    dt = time.perf_counter() - t0
                    if rep >= a.warmup:
                        t_batch.append(dt); d_batch.append(ctx.last_device_ms)
        tl, tb = statistics.median(t_loop), statistics.median(t_batch)
        print(f"| {name} | {len(files) / tl:.0f} | {len(files) / tb:.0f} | {tl / tb:.2f}x | "
              f"{statistics.median(d_loop):.2f} / {statistics.median(d_batch):.2f} |", flush=True)

    # per-kernel split of one batch
    import torch
    from torch.profiler import ProfilerActivity, profile
    for name, files in sets.items():
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            ctx.transcode_batch(files, flags, 3)
            torch.cuda.synchronize()
        tot = collections.Counter()
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA:
                key = ev.name if len(ev.name) < 60 else ev.name[:57] + "..."
                tot[key] += ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
        s = sum(tot.values())
        print(f"\nprofile of one batch, {name}: {s / 1000:.2f} ms of device activity")
        for k, v in tot.most_common(10):
            print(f"  {v / 1000:8.3f} ms  {100 * v / max(s, 1):5.1f} %  {k}")

    # the tool: whole processes
    exes = [("this tree", EXE)] + ([("before", a.before_exe)] if a.before_exe else [])
    with tempfile.TemporaryDirectory() as d:
        for name in ("64 x 1080p q85", "256 x 256x256"):
            paths = []
            for i, f in enumerate(sets[name]):
                p = os.path.join(d, f"in{i:04d}.jpg")
                open(p, "wb").write(f)
                paths.append(p)
            times = {t: [] for t, _ in exes}
            outs = {}
            for rep in range(1 + a.reps):
                for tag, exe in (exes if rep % 2 == 0 else exes[::-1]):
                    od = os.path.join(d, tag.replace(" ", "_"))
                    os.makedirs(od, exist_ok=True)
                    pairs = [x for i, p in enumerate(paths) for x in (p, os.path.join(od, f"{i:04d}.jpg"))]
                    t0 = time.perf_counter()
                    r = subprocess.run([exe, "-q", "3", "-i", "0", "--batch"] + pairs, capture_output=True, text=True)
                    dt = time.perf_counter() - t0
                    assert r.returncode == 0, r.stderr[-2000:]
                    if rep:
                        times[tag].append(dt)
                    outs[tag] = [open(os.path.join(od, f"{i:04d}.jpg"), "rb").read() for i in range(len(paths))]
            if len(outs) > 1:
                assert outs["this tree"] == outs["before"], name
            line = ", ".join(f"{t}: median {statistics.median(v):.3f} s (min {min(v):.3f}, max {max(v):.3f})"
                             for t, v in times.items())
            print(f"\njpegqs --batch, {name}: {line}")
    ctx.close()


if __name__ == "__main__":
    main()
