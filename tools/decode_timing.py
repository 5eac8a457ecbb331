"""Times the JPEG decode paths on one GPU (run on an H100; prints the card and its power limit).

  * device time of decode_async (CUDA events around the call, enqueued behind a spin so the
    host's set-up is not inside the window), in MB/s of entropy-coded data and Mpix/s;
  * host wall time of read_jpeg at the default thread count;
  * on the 8K file, the split of the decoder's device time over its kernels (torch.profiler);
  * end to end per image: decode_async -> run_async (q3 n3) -> render_async (the render only for
    1 or 3 components), CUDA events;

on one 8K 4:2:0 q90 file without restart markers, a batch of 64 1080p 4:2:0 q85 files, and one
CMYK file.  Medians of --reps runs after --warmup, arms alternating.  Writes nothing.

    python tools/decode_timing.py [--reps 10] [--warmup 3]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import torch  # noqa: E402

import decode_files as df  # noqa: E402
import jpegqs_b200 as qs  # noqa: E402


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def workload(name, files, ctx, reps, warmup):
    parsed = [qs.parse_jpeg(f) for f in files]
    images, scans = [p[0] for p in parsed], [p[1] for p in parsed]
    data = [torch.frombuffer(bytearray(f), dtype=torch.uint8).cuda() for f in files]
    ent = sum(len(f) - s.entropy_offset for f, s in zip(files, scans))
    mpix = sum(im.width * im.height for im in images) / 1e6
    out, _ = ctx.decode_async(images, scans, data)
    t_dec, t_e2e, t_host = [], [], []
    for it in range(warmup + reps):
        for arm in ("dec", "e2e", "host") if it % 2 == 0 else ("host", "e2e", "dec"):
            if arm == "host":
                t0 = time.perf_counter()
                for f in files:
                    qs.read_jpeg(f)
                dt = (time.perf_counter() - t0) * 1e3
                if it >= warmup:
                    t_host.append(dt)
                continue
            torch.cuda.synchronize()
            torch.cuda._sleep(20_000_000)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            coefs, status = ctx.decode_async(images, scans, data, out=out)
            if arm == "e2e":
                work = [im.clone() for im in images]
                st, ups = ctx.run_async(work, coefs, 3, 3)
                if all(len(im.comps) in (1, 3) for im in images):      # render takes 1 or 3 components
                    ctx.render_async(work, coefs, st, ups)
            e1.record()
            torch.cuda.synchronize()
            assert int(status.abs().sum()) == 0
            if it >= warmup:
                (t_dec if arm == "dec" else t_e2e).append(e0.elapsed_time(e1))
    d, e, h = float(np.median(t_dec)), float(np.median(t_e2e)), float(np.median(t_host))
    n = len(files)
    print(f"{name}: {n} file(s), {ent / 1e6:.2f} MB entropy data, {mpix:.1f} Mpix")
    print(f"  decode_async device time {d:.3f} ms ({ent / 1e3 / d:.0f} MB/s, {mpix / d * 1e3:.0f} Mpix/s)")
    print(f"  read_jpeg host wall time {h:.3f} ms")
    tail = "render_async" if all(len(im.comps) in (1, 3) for im in images) else "(no render: 4 components)"
    print(f"  decode -> run_async q3 n3 -> {tail}: {e:.3f} ms, {e / n:.3f} ms per image")


def kernel_shares(name, files, ctx, reps):
    """Device time per decoder kernel (torch.profiler's CUDA kernel records), summed over reps calls."""
    from torch.profiler import ProfilerActivity, profile
    parsed = [qs.parse_jpeg(f) for f in files]
    data = [torch.frombuffer(bytearray(f), dtype=torch.uint8).cuda() for f in files]
    out, _ = ctx.decode_async([p[0] for p in parsed], [p[1] for p in parsed], data)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            ctx.decode_async([p[0] for p in parsed], [p[1] for p in parsed], data, out=out)
        torch.cuda.synchronize()
    tot = {}
    for e in prof.events():
        if e.device_type.name == "CUDA" and "qd_" in e.name:
            k = e.name.split("(")[0].split(" ")[-1]
            tot[k] = tot.get(k, 0.0) + e.device_time_total / 1e3 / reps
    whole = sum(tot.values())
    print(f"{name}: decoder kernels per call (torch.profiler), {whole:.3f} ms in all")
    for k, v in sorted(tot.items(), key=lambda kv: -kv[1]):
        print(f"  {k:<20s} {v:8.3f} ms  {100 * v / whole:5.1f} %")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    ctx = qs.QsContext(0)
    print(card())
    workload("8K 4:2:0 q90, no restart markers", [df.pillow_jpeg(7680, 4320, quality=90, subsampling=2)], ctx, a.reps, a.warmup)
    workload("64 x 1080p 4:2:0 q85", [df.pillow_jpeg(1920, 1080, quality=85, subsampling=2, seed=s) for s in range(64)],
             ctx, a.reps, a.warmup)
    kernel_shares("8K 4:2:0 q90", [df.pillow_jpeg(7680, 4320, quality=90, subsampling=2)], ctx, a.reps)
    workload("CMYK 2048x1536 q90", [df.pillow_jpeg(2048, 1536, "CMYK", quality=90)], ctx, a.reps, a.warmup)


if __name__ == "__main__":
    main()
