"""Files per second of QsContext.decode_pixels at scale_denom 1, 2, 4 and 8 (libjpeg's scaled decode of
the smoothed coefficients), with device outputs and with host outputs, and the render kernel's device
time at each scale.

    python tools/pixels_scaled_timing.py [--reps 5] [--warmup 2] [--quick]

Workloads: those of tools/pixels_batch_timing.py - 256 files of 256x256, 64 of 1080p 4:2:0 q85 and 192
"web" files of mixed sizes - at -q 3, three iterations.  Before timing, every distinct file's pixels at
every scale are checked to be libjpeg-turbo's scaled decode (tests/libjpeg_scaled.py) of the file
`transcode` writes for it, and the host outputs to equal the device outputs.  The eight arms alternate
within every rep (forward, then backward); the table gives medians after the warm-up reps of the wall
time around each arm (decode_pixels returns when every output is complete).  A separate torch.profiler
run of one batch per workload and scale sums the render kernel's device time.  Prints the card and its
power limit."""
import argparse
import collections
import os
import statistics
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")]

from pixels_batch_timing import card, workloads  # noqa: E402

SCALES = (1, 2, 4, 8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--quick", action="store_true")
    a = ap.parse_args()
    import torch
    import jpegqs_b200 as qs
    import libjpeg_scaled as ls
    from jpegqs_b200 import cuda
    flags, niter = qs.quality_to_flags(3) | qs.JPEGQS_TRANSCODE, 3
    ctx = cuda.QsContext(0)
    print(f"card: {card()}  ({ctx.device_name})")
    sets = workloads(a.quick)
    sets.pop("16 x 1080p progressive, no restarts")

    arms = collections.OrderedDict()
    for d in SCALES:
        arms[f"d={d} device"] = (d, "cuda")
        arms[f"d={d} host"] = (d, "cpu")

    def run(files, d, device):
        out = ctx.decode_pixels(files, flags, niter, device=device, scale_denom=d)
        torch.cuda.synchronize()
        return out

    # correctness first: every distinct file, every scale, against libjpeg's scaled decode
    with tempfile.TemporaryDirectory() as tmp:
        for name, files in sets.items():
            distinct = list(dict.fromkeys(files))
            written = []
            for i, f in enumerate(distinct):
                data, why = ctx.transcode(f, flags, niter)
                assert data is not None, (name, why)
                p = os.path.join(tmp, f"{i}.jpg")
                with open(p, "wb") as fh:
                    fh.write(data)
                written.append(p)
            for d in SCALES:
                dev, host = run(distinct, d, "cuda"), run(distinct, d, "cpu")
                for p, r, h in zip(written, dev, host):
                    want = ls.decode_file(p, d)[0]
                    assert np.array_equal(r[0].cpu().numpy(), want), (name, d, p)
                    assert torch.equal(r[0].cpu(), h[0]), (name, d)
    print("pixels checked: libjpeg-turbo's scaled decode of the smoothed file, every scale, both output kinds")

    keys = list(arms)
    print("\n| workload | " + " | ".join(f"{k}, files/s" for k in keys) + " |")
    print("|---|" + "---|" * len(keys))
    for name, files in sets.items():
        times = {k: [] for k in keys}
        for rep in range(a.warmup + a.reps):
            for k in (keys if rep % 2 == 0 else keys[::-1]):
                t0 = time.perf_counter()
                run(files, *arms[k])
                dt = time.perf_counter() - t0
                if rep >= a.warmup:
                    times[k].append(dt)
        med = {k: statistics.median(v) for k, v in times.items()}
        print(f"| {name} | " + " | ".join(f"{len(files) / med[k]:.0f}" for k in keys) + " |", flush=True)

    from torch.profiler import ProfilerActivity, profile
    print("\n| workload | " + " | ".join(f"render kernel at d={d}, ms" for d in SCALES) + " |")
    print("|---|" + "---|" * len(SCALES))
    for name, files in sets.items():
        row = []
        for d in SCALES:
            run(files, d, "cuda")
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                run(files, d, "cuda")
            t = 0.0
            for ev in prof.events():
                if ev.device_type == torch.autograd.DeviceType.CUDA and "qs_render_async_kernel" in ev.name:
                    t += ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
            row.append(t / 1000)
        print(f"| {name} | " + " | ".join(f"{v:.3f}" for v in row) + " |", flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
