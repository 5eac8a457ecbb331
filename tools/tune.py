"""Kernel-variant sweep on the 8K q3 workload (device-resident).  Usage on a GPU machine:
    python tools/tune.py [--flags 0] [--variants sync:maxn[:wpg[:gs[:uni[:merge]]]],...]
Prints per-variant average smoothing-pass launch time and checks that every variant
produces byte-identical output."""
import argparse
import hashlib
import os
import pickle
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import jpegqs_b200 as qs

ap = argparse.ArgumentParser()
ap.add_argument("--flags", type=int, default=0)
ap.add_argument("--niter", type=int, default=3)
ap.add_argument("--width", type=int, default=7680)
ap.add_argument("--height", type=int, default=4320)
ap.add_argument("--variants", default="0:4,1:4,1:3,1:2")
ap.add_argument("--steps", type=int, default=3)
args = ap.parse_args()

ctx = qs.cuda.QsContext(0)
ctx.set_profiling(True)
cache = f"/tmp/qs_tune_{args.width}x{args.height}.pkl"     # the generator takes ~10 s at 8K: keep it between runs of one session
if os.path.exists(cache):
    with open(cache, "rb") as fh:
        im = pickle.load(fh)
else:
    im = qs.synth.make_image(args.width, args.height, "420")
    with open(cache, "wb") as fh:
        pickle.dump(im, fh, protocol=4)
dev = torch.device("cuda", 0)
host = [torch.from_numpy(np.ascontiguousarray(c.coef)) for c in im.comps]
stream = torch.cuda.current_stream().cuda_stream or 1   # 1 = cudaStreamLegacy
ref_hash = None
for v in args.variants.split(","):
    f = [int(x) for x in v.split(":")]
    sync, maxn, wpg, gs = f[0], f[1], (f[2] if len(f) > 2 else 4), (f[3] if len(f) > 3 else 1)
    uni = f[4] if len(f) > 4 else 1
    merge = f[5] if len(f) > 5 else None
    ctx.set_tuning(5, uni)
    if merge is not None:
        ctx.set_tuning(8, merge)
    if sync != 2:
        ctx.set_tuning(0, sync)
    ctx.set_tuning(1, maxn)
    if wpg != 4:
        ctx.set_tuning(2, wpg)
    sm, n, tot, idm, idn = 0.0, 0, 0.0, 0.0, 0
    for i in range(args.steps + 1):
        bufs = [h.to(dev) for h in host]
        ups = []
        if args.flags & 4:
            y = im.comps[0]
            ups = [None] + [torch.empty((y.hblk, y.wblk, 64), dtype=torch.int16, device=dev).data_ptr() for _ in range(2)]
        torch.cuda.synchronize()
        ctx.run_device(im, [t.data_ptr() for t in bufs], ups, args.flags, args.niter, stream)
        if i:
            a, b, c, d = ctx.kernel_stats()
            sm += c; n += d; tot += ctx.last_device_ms; idm += a; idn += b
    h = hashlib.sha1(b"".join(t.cpu().numpy().tobytes() for t in bufs)).hexdigest()
    if ref_hash is None:
        ref_hash = h
    print(f"sync={sync} maxn={maxn} wpg={wpg} gs={gs} uni={uni} merge={merge}: smooth {sm / n:.3f} ms/launch, idct pass {1e3 * idm / max(idn, 1):.1f} us/launch, whole run {tot / args.steps:.3f} ms, "
          f"{args.width * args.height / 1e6 / (tot / args.steps / 1e3):.0f} Mpix/s, same_output={h == ref_hash}, sha1={h[:12]}", flush=True)
