"""Times the JPEG encode paths on one GPU (run on an H100; prints the card and its power limit).

  * device time of encode_async with standard (optimize 0) and optimal (optimize 1) tables, CUDA
    events around the call, enqueued behind a spin so the host's set-up is not inside the window;
  * the whole device pipeline per image: decode_async -> run_async (q3 n3) -> encode_async;
  * the current route to a file: synchronise + copy the coefficients to pinned host memory (CUDA
    events), and the jpegqs tool's host writer (`jpegqs -v 1` reports "encode + write" per file);

on one 8K (7680x4320) 4:2:0 file and a batch of 64 1080p 4:2:0 files, both smoothed at q3 n3 first.
Medians of --reps runs after --warmup, arms alternating.  Temporary files only.

    python tools/encode_timing.py [--reps 10] [--warmup 3]
"""
import argparse
import os
import re
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import torch  # noqa: E402

import decode_files as df  # noqa: E402
import jpegqs_b200 as qs  # noqa: E402

EXE = os.path.join(ROOT, "jpeg-quantsmooth_b200", "csrc", "jpegqs")


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def timed(fn):
    torch.cuda.synchronize()
    torch.cuda._sleep(20_000_000)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    r = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), r


def host_writer_ms(files):
    """The tool's "encode + write" wall time, summed over the files (-q 3 -n 3, the same smoothing)."""
    total = 0.0
    with tempfile.TemporaryDirectory() as d:
        for k, f in enumerate(files):
            src, dst = os.path.join(d, f"{k}.jpg"), os.path.join(d, f"{k}o.jpg")
            with open(src, "wb") as fh:
                fh.write(f)
            r = subprocess.run([EXE, "-q", "3", "-n", "3", "-v", "1", "-i", "0", src, dst], capture_output=True, text=True)
            m = re.search(r"encode \+ write ([0-9.]+) ms", r.stderr)
            if r.returncode or not m:
                return None
            total += float(m.group(1))
    return total


def workload(name, files, ctx, reps, warmup):
    parsed = [qs.parse_jpeg(f) for f in files]
    images, scans = [p[0] for p in parsed], [p[1] for p in parsed]
    data = [torch.frombuffer(bytearray(f), dtype=torch.uint8).cuda() for f in files]
    heads = []
    for f in files:
        pre, ids, tbls = qs.jpeg_prefix(f)
        heads.append((torch.frombuffer(bytearray(pre), dtype=torch.uint8).cuda(), ids, tbls))
    coefs, dst = ctx.decode_async(images, scans, data)
    work = [im.clone() for im in images]
    rst, ups = ctx.run_async(work, coefs, 0, 3)
    torch.cuda.synchronize()
    assert int(dst.abs().sum()) == 0
    host = [[torch.empty(t.shape, dtype=t.dtype, pin_memory=True) for t in c] for c in coefs]
    hup = [[torch.empty(t.shape, dtype=t.dtype, pin_memory=True) for t in u] if u is not None else None for u in ups]
    mpix = sum(im.width * im.height for im in images) / 1e6
    t = {"enc0": [], "enc1": [], "pipe": [], "d2h": []}
    nbytes = 0
    for it in range(warmup + reps):
        arms = list(t) if it % 2 == 0 else list(reversed(list(t)))
        for arm in arms:
            if arm in ("enc0", "enc1"):
                ms, (out, ln, st) = timed(lambda: ctx.encode_async(work, coefs, heads, arm == "enc1", rst, ups))
                assert int(st.abs().sum()) == 0
                nbytes = int(ln.sum())
            elif arm == "pipe":
                def pipe():
                    w = [im.clone() for im in images]
                    c, _ = ctx.decode_async(images, scans, data)
                    s, u = ctx.run_async(w, c, 0, 3)
                    return ctx.encode_async(w, c, heads, False, s, u)
                ms, _ = timed(pipe)
            else:
                def d2h():
                    for hs, cs in zip(host, coefs):
                        for h, c in zip(hs, cs):
                            h.copy_(c, non_blocking=True)
                    for hs, us in zip(hup, ups):
                        if hs is not None:
                            for h, u in zip(hs, us):
                                h.copy_(u, non_blocking=True)
                ms, _ = timed(d2h)
            if it >= warmup:
                t[arm].append(ms)
    med = {k: float(np.median(v)) for k, v in t.items()}
    n = len(files)
    hw = host_writer_ms(files)
    cbytes = sum(x.numel() * 2 for c in coefs for x in c)
    print(f"{name}: {n} image(s), {mpix:.1f} Mpix, {cbytes / 1e6:.1f} MB of coefficients, {nbytes / 1e6:.2f} MB of output")
    print(f"  encode_async optimize 0: {med['enc0']:.3f} ms ({med['enc0'] / n:.3f} ms per image, {mpix / med['enc0'] * 1e3:.0f} Mpix/s)")
    print(f"  encode_async optimize 1: {med['enc1']:.3f} ms ({med['enc1'] / n:.3f} ms per image)")
    print(f"  decode -> run_async q3 n3 -> encode (optimize 0): {med['pipe']:.3f} ms, {med['pipe'] / n:.3f} ms per image")
    print(f"  current route: synchronise + D2H of the coefficients {med['d2h']:.3f} ms; jpegqs host writer "
          + (f"{hw:.1f} ms ({hw / n:.2f} ms per image)" if hw is not None else "not measured (tool failed)"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    ctx = qs.QsContext(0)
    print(card())
    workload("8K 4:2:0 q90, smoothed q3 n3", [df.pillow_jpeg(7680, 4320, quality=90, subsampling=2)], ctx, a.reps, a.warmup)
    workload("64 x 1080p 4:2:0 q85, smoothed q3 n3",
             [df.pillow_jpeg(1920, 1080, quality=85, subsampling=2, seed=s) for s in range(64)], ctx, a.reps, a.warmup)


if __name__ == "__main__":
    main()
