"""Device time of the stream-ordered render (render_async) next to jpegqs_cuda_render_rgb on device
buffers, and the bytes/s the render reaches against the algorithmic minimum.

    python tools/render_timing.py [--calls 20] [--warmup 3] [--out FILE]

Workloads (synthetic content, Annex-K quality 50 tables), smoothed once by run_async with flags 0
(the CLI's -q 3) and 3 iterations; the timed calls decode the smoothed coefficients:
  8K    one 7680x4320 4:2:0 image
  1080p 16 x 1920x1080 4:2:0 images
Arms, alternating call by call, each bracketed by CUDA events on one stream, median of --calls
after --warmup rounds:
  render_async               one call for the whole batch, its Python set-up included
  render_async_behind_spin   the same call enqueued behind a spinning kernel: device work only
  render_rgb                 jpegqs_cuda_render_rgb(on_device = 1) through ctypes, once per image
                             (it synchronises inside; its window holds its own set-up)
The minimum traffic is the coefficients read once (128 bytes per block of every component) plus
the pixels written once (3 bytes per pixel); bytes/s = that over the device-only time, beside the
H100 SXM data-sheet 3.35 TB/s.  Prints the card's name and power limit (read-only nvidia-smi query).
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys


sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import jpegqs_b200 as qs                                    # noqa: E402
from jpegqs_b200 import synth                               # noqa: E402
from jpegqs_b200.cuda import _image_array                   # noqa: E402

FLAGS, NITER = 0, 3
HBM_BYTES_PER_S = 3.35e12


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:
        return f"unknown ({e})"


def run(args):
    import torch
    torch.cuda.init()
    ctx = qs.QsContext(0)
    stream = torch.cuda.Stream()
    out = {"card": card(), "device": ctx.device_name, "calls": args.calls, "warmup": args.warmup,
           "smoothing": {"flags": FLAGS, "niter": NITER}}
    print("card:", out["card"], flush=True)

    def workload(name, w, h, n):
        ims = [synth.make_image(w, h, "420", quality=50, seed=k + 1) for k in range(n)]
        coefs = [[torch.from_numpy(c.coef).cuda() for c in im.comps] for im in ims]
        with torch.cuda.stream(stream):
            status, ups = ctx.run_async(ims, coefs, FLAGS, NITER)
        stream.synchronize()
        outs = [torch.empty((h, w, 3), dtype=torch.uint8, device="cuda") for _ in ims]
        ref = [torch.empty_like(o) for o in outs]
        arr = _image_array(ims, [[t.data_ptr() for t in ts] for ts in coefs], [])

        def render_async():
            ctx.render_async(ims, coefs, status, ups, out=outs, stream=stream)

        def render_rgb():
            for i in range(n):
                rc = ctx.lib.jpegqs_cuda_render_rgb(ctx.h, C.byref(arr[i]), 1, C.c_void_p(ref[i].data_ptr()),
                                                    C.c_void_p(stream.cuda_stream))
                assert rc == 0, rc

        arms = {"render_async": render_async, "render_async_behind_spin": render_async, "render_rgb": render_rgb}
        res = {k: [] for k in arms}
        for i in range(args.warmup + args.calls):
            for label, fn in arms.items():
                if label.endswith("behind_spin"):
                    with torch.cuda.stream(stream):
                        torch.cuda._sleep(40_000_000)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(stream)                             # behind a spin: fires when the spin ends,
                fn()                                         # after the host has enqueued the call
                b.record(stream)
                b.synchronize()
                if i >= args.warmup:
                    res[label].append(a.elapsed_time(b))
        blocks = sum(c.wblk * c.hblk for im in ims for c in im.comps)
        min_bytes = blocks * 128 + n * w * h * 3
        row = {k: {"ms_median": statistics.median(v), "ms_min": min(v), "ms_max": max(v)} for k, v in res.items()}
        dev = row["render_async_behind_spin"]["ms_median"]
        row["min_bytes"] = min_bytes
        row["bytes_per_s"] = min_bytes / (dev * 1e-3)
        row["share_of_hbm_peak"] = row["bytes_per_s"] / HBM_BYTES_PER_S
        row["outputs_identical"] = all(torch.equal(o, r) for o, r in zip(outs, ref))
        out[name] = row
        print(name, json.dumps(row), flush=True)

    workload("8k_420", 7680, 4320, 1)
    workload("1080p_420_x16", 1920, 1080, 16)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out")
    run(ap.parse_args())
