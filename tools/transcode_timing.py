"""Wall time of `jpegqs --batch` on its device route (decode, smoothing and encode on the GPU) against
its host codec (JPEGQS_HOST_CODEC=1, the reader and writer on host threads around do_quantsmooth).

    python tools/transcode_timing.py [--reps 3] [--warmup 1] [--quick]

The two routes alternate, each rep runs both.  Workloads: 64 x 1080p 4:2:0 q85 sequential, 64 x 1080p
progressive with restart markers, 64 x 1080p progressive without (the device route sends those to the
host codec: a control that must not move), 8 x 8K 4:2:0 q90, 256 files of 256 x 256; and one 8K file
per process.  Times are whole processes (CUDA start-up included); the table gives the median and the
files' output bytes are checked equal between the routes.  Prints the card and its power limit."""
import argparse
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "jpeg-quantsmooth_b200", "csrc", "jpegqs")


def picture(w, h, seed):
    rng = np.random.RandomState(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float32)
    a = np.stack([128 + 70 * np.sin(x / 31.0) + 40 * np.cos(y / 19.0), 128 + 60 * np.cos((x + y) / 47.0),
                  128 + 80 * np.sin((x - y) / 23.0)], -1) + rng.normal(0, 9, (h, w, 3)).astype(np.float32)
    return Image.fromarray(a.clip(0, 255).astype(np.uint8), "RGB")


def make_set(d, name, count, w, h, distinct=8, **save):
    os.makedirs(os.path.join(d, name), exist_ok=True)
    files = []
    for i in range(count):
        p = os.path.join(d, name, f"{i:04d}.jpg")
        if i < distinct:
            picture(w, h, i).save(p, **save)
        else:
            os.link(files[i % distinct], p)
        files.append(p)
    return files


def run(files, out_dir, env, args):
    os.makedirs(out_dir, exist_ok=True)
    pairs = []
    for i, f in enumerate(files):
        pairs += [f, os.path.join(out_dir, f"{i:04d}.jpg")]
    cmd = [EXE, "-i", "0"] + args + (["--batch"] if len(files) > 1 else []) + pairs
    t0 = time.perf_counter()
    r = subprocess.run(cmd, env=env, capture_output=True, text=True)
    dt = time.perf_counter() - t0
    if r.returncode:
        sys.exit(f"jpegqs failed ({r.returncode}): {r.stderr[-2000:]}")
    return dt, r.stderr


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:                                   # noqa: BLE001
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--quick", action="store_true", help="small workloads only (a check that the script runs)")
    ap.add_argument("--args", default="-q 3", help="jpegqs options (default: -q 3, three iterations)")
    a = ap.parse_args()
    args = a.args.split()
    print(f"card: {card()}", flush=True)
    with tempfile.TemporaryDirectory(prefix="transcode_timing_") as d:
        n1080, n8k = (8, 1) if a.quick else (64, 8)
        sets = [
            (f"{n1080} x 1080p 4:2:0 q85 sequential", make_set(d, "seq", n1080, 1920, 1080, quality=85)),
            (f"{n1080} x 1080p progressive, restart markers", make_set(d, "progrst", n1080, 1920, 1080, quality=85,
                                                                        progressive=True, restart_marker_rows=1)),
            (f"{n1080} x 1080p progressive, no restart markers (host on both)",
             make_set(d, "prog", n1080, 1920, 1080, quality=85, progressive=True)),
            (f"{n8k} x 8K 4:2:0 q90", make_set(d, "8k", n8k, 7680, 4320, distinct=min(n8k, 4), quality=90)),
            (f"{32 if a.quick else 256} x 256x256 q85", make_set(d, "small", 32 if a.quick else 256, 256, 256, distinct=16,
                                                               quality=85)),
            ("one 8K 4:2:0 q90 file per process", None),
        ]
        sets[-1] = (sets[-1][0], sets[3][1][:1])
        envs = {"device": dict(os.environ), "host": dict(os.environ, JPEGQS_HOST_CODEC="1")}
        rows = []
        for label, files in sets:
            times = {"device": [], "host": []}
            for rep in range(a.warmup + a.reps):
                for route in ("device", "host") if rep % 2 == 0 else ("host", "device"):
                    dt, _ = run(files, os.path.join(d, "out_" + route), envs[route], args)
                    if rep >= a.warmup:
                        times[route].append(dt)
            for i in range(len(files)):
                p = lambda r: open(os.path.join(d, "out_" + r, f"{i:04d}.jpg"), "rb").read()
                if p("device") != p("host"):
                    sys.exit(f"{label}: file {i} differs between the routes")
            dev, host = statistics.median(times["device"]), statistics.median(times["host"])
            rows.append((label, len(files), dev, host))
            print(f"{label}: device {dev:.3f} s, host {host:.3f} s, host/device {host / dev:.2f}x "
                  f"(device {['%.3f' % t for t in times['device']]}, host {['%.3f' % t for t in times['host']]})",
                  flush=True)
        print()
        print(f"jpegqs {' '.join(args)} --batch wall time, median of {a.reps} (after {a.warmup} warm-up), on {card()}")
        print("| workload | device route | host codec | host / device |")
        print("|---|---|---|---|")
        for label, n, dev, host in rows:
            print(f"| {label} | {dev:.3f} s | {host:.3f} s | {host / dev:.2f}x |")


if __name__ == "__main__":
    main()
