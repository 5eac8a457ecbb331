"""Times the scan decoder (decode_scans_async) against the host reader on one GPU (run on an H100;
prints the card and its power limit).

  * device time of decode_scans_async (CUDA events around the call, enqueued behind a spin so the
    host's set-up is not inside the window);
  * host wall time of read_jpeg at the default thread count;
  * a separate torch.profiler run: the device time per kernel and per scan kind (byte pass, first
    scans, DC refinement, AC refinement), so the share of the serial AC refinement is visible;

on one 8K 4:2:0 q90 progressive file without restart markers, the same picture with a restart
marker every MCU row, and a batch of 64 1080p 4:2:0 q85 progressive files.  Medians of --reps runs
after --warmup, arms alternating.  Writes nothing.

    python tools/decode_scans_timing.py [--reps 10] [--warmup 3]
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

KIND = {"qs_zero_kernel": "set-up", "qs_store_kernel": "set-up", "qs_scan_kernel": "bytes", "qs_seg_kernel": "bytes",
        "qs_compact_kernel": "bytes", "qs_iv_kernel": "first scans", "qs_sync_kernel": "first scans",
        "qs_chain_kernel": "first scans", "qs_place_kernel": "first scans", "qs_final_kernel": "first scans",
        "qs_dcr_kernel": "DC refinement", "qs_acr_kernel": "AC refinement (serial per interval)"}


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def _prepare(files):
    parsed = [qs.parse_jpeg_scans(f) for f in files]
    assert all(p[1] is not None for p in parsed)
    data = [torch.frombuffer(bytearray(f), dtype=torch.uint8).cuda() for f in files]
    return [p[0] for p in parsed], [p[1] for p in parsed], data


def workload(name, files, ctx, reps, warmup):
    images, scans, data = _prepare(files)
    ent = sum(sum(r.end - r.offset for r in s) for s in scans)
    mpix = sum(im.width * im.height for im in images) / 1e6
    out, _ = ctx.decode_scans_async(images, scans, data)
    t_dev, t_host = [], []
    for it in range(warmup + reps):
        for arm in ("dev", "host") if it % 2 == 0 else ("host", "dev"):
            if arm == "host":
                t0 = time.perf_counter()
                for f in files:
                    qs.read_jpeg(f)
                if it >= warmup:
                    t_host.append((time.perf_counter() - t0) * 1e3)
                continue
            torch.cuda.synchronize()
            torch.cuda._sleep(20_000_000)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            _, status = ctx.decode_scans_async(images, scans, data, out=out)
            e1.record()
            torch.cuda.synchronize()
            assert int(status.abs().sum()) == 0
            if it >= warmup:
                t_dev.append(e0.elapsed_time(e1))
    d, h = float(np.median(t_dev)), float(np.median(t_host))
    nsc = sum(len(s) for s in scans)
    print(f"{name}: {len(files)} file(s), {nsc} scans, {ent / 1e6:.2f} MB entropy data, {mpix:.1f} Mpix, "
          f"{ctx.last_launches} launches")
    print(f"  decode_scans_async device time {d:.3f} ms ({mpix / d * 1e3:.0f} Mpix/s)")
    print(f"  read_jpeg host wall time       {h:.3f} ms  (device / host = {d / h:.2f})")


def kernel_shares(name, files, ctx, reps):
    from torch.profiler import ProfilerActivity, profile
    images, scans, data = _prepare(files)
    out, _ = ctx.decode_scans_async(images, scans, data)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            ctx.decode_scans_async(images, scans, data, out=out)
        torch.cuda.synchronize()
    tot = {}
    for e in prof.events():
        if e.device_type.name == "CUDA" and "qs_" in e.name:
            k = e.name.split("(")[0].split(" ")[-1]
            tot[k] = tot.get(k, 0.0) + e.device_time_total / 1e3 / reps
    whole = sum(tot.values())
    print(f"{name}: kernels per call (torch.profiler), {whole:.3f} ms in all")
    for k, v in sorted(tot.items(), key=lambda kv: -kv[1]):
        print(f"  {k:<20s} {v:8.3f} ms  {100 * v / whole:5.1f} %")
    kinds = {}
    for k, v in tot.items():
        kinds[KIND.get(k, k)] = kinds.get(KIND.get(k, k), 0.0) + v
    print("  by scan kind:")
    for k, v in sorted(kinds.items(), key=lambda kv: -kv[1]):
        print(f"    {k:<36s} {v:8.3f} ms  {100 * v / whole:5.1f} %")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    ctx = qs.QsContext(0)
    print(card())
    big = df.pillow_jpeg(7680, 4320, quality=90, subsampling=2, progressive=True)
    big_rst = df.pillow_jpeg(7680, 4320, quality=90, subsampling=2, progressive=True, restart_marker_rows=1)
    hd = [df.pillow_jpeg(1920, 1080, quality=85, subsampling=2, progressive=True, seed=s) for s in range(64)]
    workload("8K 4:2:0 q90 progressive, no restart markers", [big], ctx, a.reps, a.warmup)
    workload("8K 4:2:0 q90 progressive, a restart marker every MCU row", [big_rst], ctx, a.reps, a.warmup)
    workload("64 x 1080p 4:2:0 q85 progressive", hd, ctx, a.reps, a.warmup)
    kernel_shares("8K progressive, no restarts", [big], ctx, a.reps)
    kernel_shares("8K progressive, restarts", [big_rst], ctx, a.reps)
    kernel_shares("64 x 1080p progressive", hd, ctx, a.reps)


if __name__ == "__main__":
    main()
