"""Device time per image of the stream-ordered entry point (run_async) next to the blocking
device-buffer entry points, plus run_async's host enqueue time and a CUDA-graph replay.

    python tools/async_timing.py [--calls 20] [--warmup 3] [--out FILE]

Workloads (synthetic content, Annex-K quality 50 tables, flags 0 = the CLI's -q 3, 3 iterations):
  8K    one 7680x4320 4:2:0 image: run_device vs run_async
  1080p 16 x 1920x1080 4:2:0 images in one call: run_batch(on_device) vs run_async, and a
        replay of a CUDA graph captured around run_async
Every timed call starts from the same quantized coefficients (restored by a device copy before
the start event) and is bracketed by CUDA events on its stream; the arms alternate call by call.
Such a window also holds whatever host set-up comes before the call's first kernel; the arm
"run_async_behind_spin" enqueues the call behind a spinning kernel, so its window is device work
only (the blocking entry points cannot be timed that way: they wait inside the call).
The enqueue time is host time from the call until it returns, without any synchronisation: it is
not device time.  Prints the card's name and power limit (read-only nvidia-smi query) first.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import jpegqs_b200 as qs                                    # noqa: E402
from jpegqs_b200 import synth                               # noqa: E402
from jpegqs_b200.image import CoefImage, Component          # noqa: E402

FLAGS, NITER = 0, 3


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                                  # the numbers still stand, unlabelled
        return f"unknown ({e})"


def describe(im):
    """Geometry and quant tables only (what the entry points read from a CoefImage), fresh per call:
    run_async sets the quant tables it was given to ones."""
    z = np.zeros((1, 1, 64), dtype=np.int16)
    return CoefImage(im.width, im.height, im.colorspace,
                     [Component(np.broadcast_to(z, tuple(c.coef.shape)), c.quant.copy(), c.h_samp, c.v_samp,
                                c.quant_tbl_no) for c in im.comps])


class Images:
    """Device-resident working buffers, their pristine copies and luma-sized chroma outputs."""

    def __init__(self, torch, images):
        self.torch, self.images = torch, images
        self.pristine = [[c.coef for c in im.comps] for im in images]
        self.work = [[t.clone() for t in ts] for ts in self.pristine]
        self.ups = [[torch.empty_like(im.comps[0].coef) for _ in range(2)] for im in images]

    def restore(self):
        for ws, ps in zip(self.work, self.pristine):
            for w, p in zip(ws, ps):
                w.copy_(p)

    def ptrs(self):
        return [[t.data_ptr() for t in ts] for ts in self.work], [[None] + [u.data_ptr() for u in us] for us in self.ups]

    def digest(self):
        """a cheap fingerprint of the smoothed coefficients, to tell that the arms agree"""
        w = self.torch.arange(1, 65, device=self.work[0][0].device, dtype=self.torch.int64)
        return [int((t.to(self.torch.int64) * w).sum().item()) for ts in self.work for t in ts]


def timed(torch, stream, fn, per):
    """device time of what fn enqueues on stream (fn may also block), per image"""
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record(stream)
    with torch.cuda.stream(stream):
        fn()
    end.record(stream)
    end.synchronize()
    return start.elapsed_time(end) / per


def run(args):
    import torch
    torch.cuda.init()
    ctx = qs.QsContext(0)
    stream = torch.cuda.Stream()
    out = {"card": card(), "device": ctx.device_name, "calls": args.calls, "warmup": args.warmup,
           "flags": FLAGS, "niter": NITER}
    print("card:", out["card"], flush=True)

    def measure(name, ims, arms):
        """arms: {label: fn(images) -> None}, each enqueueing one call on `stream`.  An arm whose
        label ends in "behind_spin" is enqueued while the stream still spins (torch.cuda._sleep,
        ~20 ms) and its start event is recorded after the spin: its window holds device work only,
        no host set-up."""
        res = {k: [] for k in arms}
        digests = {}
        for i in range(args.warmup + args.calls):
            for label, fn in arms.items():
                with torch.cuda.stream(stream):
                    ims.restore()
                    if label.endswith("behind_spin"):
                        torch.cuda._sleep(40_000_000)
                ms = timed(torch, stream, lambda: fn(ims), len(ims.images))
                if i >= args.warmup:
                    res[label].append(ms)
                if i == args.warmup + args.calls - 1:
                    digests[label] = ims.digest()
        same = len({tuple(d) for d in digests.values()}) == 1
        row = {label: {"ms_per_image_median": statistics.median(v), "ms_per_image_min": min(v),
                       "ms_per_image_max": max(v)} for label, v in res.items()}
        row["outputs_identical"] = same
        out[name] = row
        print(name, json.dumps(row), flush=True)

    def via_device(ims):
        cp, up = ims.ptrs()
        ctx.run_device(ims.images[0], cp[0], up[0], FLAGS, NITER, stream.cuda_stream)

    def via_batch(ims):
        cp, up = ims.ptrs()
        ctx.run_batch_device(ims.images, cp, up, FLAGS, NITER, stream.cuda_stream)

    def via_async(ims):
        ctx.run_async([describe(im) for im in ims.images], ims.work, FLAGS, NITER,
                      up=[tuple(u) for u in ims.ups], stream=stream)

    big = Images(torch, [synth.make_image_torch(7680, 4320, "420", 50, seed=1)])
    measure("8k_420", big, {"run_device": via_device, "run_async": via_async, "run_async_behind_spin": via_async})
    del big
    hd = Images(torch, [synth.make_image_torch(1920, 1080, "420", 50, seed=100 + k) for k in range(16)])
    measure("16x1080p_420", hd, {"run_batch_device": via_batch, "run_async": via_async,
                                 "run_async_behind_spin": via_async})

    # enqueue time of run_async (host clock, no synchronisation inside the window)
    enq = []
    for i in range(args.warmup + args.calls):
        with torch.cuda.stream(stream):
            hd.restore()
        stream.synchronize()
        descs = [describe(im) for im in hd.images]
        t0 = time.perf_counter()
        ctx.run_async(descs, hd.work, FLAGS, NITER, up=[tuple(u) for u in hd.ups], stream=stream)
        t1 = time.perf_counter()
        stream.synchronize()
        if i >= args.warmup:
            enq.append((t1 - t0) * 1e3)
    out["16x1080p_420"]["run_async_enqueue_ms_per_call"] = {"median": statistics.median(enq), "min": min(enq),
                                                            "max": max(enq)}
    print("run_async enqueue (host) ms per 16-image call:", json.dumps(out["16x1080p_420"]["run_async_enqueue_ms_per_call"]),
          flush=True)

    # a CUDA graph captured around run_async, replayed on restored inputs
    ref = None
    with torch.cuda.stream(stream):
        hd.restore()
    stream.synchronize()
    via_async(hd)
    stream.synchronize()
    ref = hd.digest()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(stream):
        hd.restore()
    stream.synchronize()
    with torch.cuda.graph(g, stream=stream):
        ctx.run_async([describe(im) for im in hd.images], hd.work, FLAGS, NITER, up=[tuple(u) for u in hd.ups])
    reps = []
    for i in range(args.warmup + args.calls):
        with torch.cuda.stream(stream):
            hd.restore()
        ms = timed(torch, stream, lambda: g.replay(), 16)
        if i >= args.warmup:
            reps.append(ms)
    out["16x1080p_420"]["graph_replay"] = {"ms_per_image_median": statistics.median(reps), "ms_per_image_min": min(reps),
                                           "ms_per_image_max": max(reps), "outputs_identical": hd.digest() == ref}
    print("graph replay", json.dumps(out["16x1080p_420"]["graph_replay"]), flush=True)
    ctx.close()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the result as JSON here")
    args = ap.parse_args()
    res = run(args)
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
