"""The device JPEG decoders on the stream corpus (stream_files.py): every legal and warned file and the
large boundary files, in one batched call per decoder and knob, with guard regions around the
outputs, the workspace and the status array.  The device must give exactly its CPU model's status and,
where that is 0, the model's coefficients.  Then end to end: transcode_batch at -n 0 and decode_pixels
at niter 0 give libjpeg's coefficients and pixels for every legal file, whichever route it takes.
Every file is decoded a fixed number of times."""
import ctypes as C
import io
import os
import subprocess

import numpy as np
import pytest

import decode_files as df
import libjpeg_pixels as lp
import stream_files as sf
import jpegqs_b200 as qs
from jpegqs_b200 import cuda
from jpegqs_b200.cuda import QsContext

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(lp.JPEG_SO is None, reason="no libjpeg inside Pillow")]

EXE = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "jpeg-quantsmooth_b200", "csrc", "jpegqs")
LEGAL = sf.corpus() + sf.boundary_files()
# FF FF 00 (libjpeg: one data byte FF) is no T.81 stream, but the device must still match its model
ALL = LEGAL + sf.warned() + [sf.StreamFile(f"stuffed_fill_{n}", sf.stuffed_fill(d), "warned", "stuffed_fill")
                             for n, d, _ in sf.bases()[:3]]
G = 1 << 16                                                 # guard bytes around the workspace
CG = 4096                                                   # guard elements around each output array


@pytest.fixture(scope="module")
def torch():
    import torch as t
    return t


@pytest.fixture(scope="module")
def ctx():
    c = QsContext(0)
    yield c
    c.close()


def _guarded_outputs(torch, images):
    """per image, per component: (whole buffer, the [hblk, wblk, 64] view between two guards)"""
    out = []
    for im in images:
        row = []
        for c in im.comps:
            n = c.hblk * c.wblk * 64
            buf = torch.full((n + 2 * CG,), 0x5A5A, dtype=torch.int16, device="cuda")
            row.append((buf, buf[CG:CG + n].view(c.hblk, c.wblk, 64)))
        out.append(row)
    return out


def _check(torch, files, images, outs, ws, st, models):
    assert bool((ws[:G] == 0x6D).all()) and bool((ws[-G:] == 0x6D).all())
    n = len(files)
    assert bool((st[:64] == 0x1234567).all()) and bool((st[64 + n:] == 0x1234567).all())
    status = st[64:64 + n].cpu().tolist()
    for f, row, s, (marr, mst) in zip(files, outs, status, models):
        assert s == mst, (f.name, hex(s), hex(mst))
        for buf, _ in row:
            assert bool((buf[:CG] == 0x5A5A).all()) and bool((buf[-CG:] == 0x5A5A).all()), f.name
        if s == 0:
            assert all(np.array_equal(v.cpu().numpy(), m) for (_, v), m in zip(row, marr)), f.name


@pytest.mark.parametrize("sub_bytes", [cuda.DECODE_SUB_MIN, cuda.DECODE_SUB_DEFAULT])
def test_decode_async_equals_the_model(torch, ctx, sub_bytes):
    files = [f for f in ALL if qs.parse_jpeg(f.data)[1] is not None]
    parsed = [qs.parse_jpeg(f.data) for f in files]
    images, scans = [p[0] for p in parsed], [p[1] for p in parsed]
    models = [qs.decode_model(im, sc, f.data, sub_bytes)[:2] for f, im, sc in zip(files, images, scans)]
    data = [torch.frombuffer(bytearray(f.data), dtype=torch.uint8).cuda() for f in files]
    outs = _guarded_outputs(torch, images)
    n = len(files)
    need = qs.decode_workspace_bytes(images, scans, [len(f.data) for f in files])
    ws = torch.full((need + 2 * G,), 0x6D, dtype=torch.uint8, device="cuda")
    st = torch.full((n + 2 * 64,), 0x1234567, dtype=torch.int32, device="cuda")
    arr = cuda._image_array(images, [[v.data_ptr() for _, v in row] for row in outs])
    ctx.set_tuning(9, sub_bytes)
    try:
        rc = ctx.lib.jpegqs_cuda_decode_async(ctx.h, n, arr, (cuda._Scan * n)(*scans),
                                              (C.c_void_p * n)(*[t.data_ptr() for t in data]),
                                              (C.c_size_t * n)(*[len(f.data) for f in files]), ws.data_ptr() + G, need,
                                              st.data_ptr() + 256, None)
        torch.cuda.synchronize()
    finally:
        ctx.set_tuning(9, cuda.DECODE_SUB_DEFAULT)
    assert rc == 0
    _check(torch, files, images, outs, ws, st, models)


@pytest.mark.parametrize("sub_bytes", [cuda.DECODE_SUB_MIN, cuda.DECODE_SUB_DEFAULT])
def test_decode_scans_async_equals_the_model(torch, ctx, sub_bytes):
    files = ALL
    parsed = [qs.parse_jpeg_scans(f.data) for f in files]
    images, scans = [p[0] for p in parsed], [p[1] for p in parsed]
    assert all(s is not None for s in scans)
    models = [qs.decode_scans_model(im, sc, f.data, sub_bytes) for f, im, sc in zip(files, images, scans)]
    data = [torch.frombuffer(bytearray(f.data), dtype=torch.uint8).cuda() for f in files]
    outs = _guarded_outputs(torch, images)
    n = len(files)
    need = qs.decode_scans_workspace_bytes(images, scans, [len(f.data) for f in files])
    ws = torch.full((need + 2 * G,), 0x6D, dtype=torch.uint8, device="cuda")
    st = torch.full((n + 2 * 64,), 0x1234567, dtype=torch.int32, device="cuda")
    arr = cuda._image_array(images, [[v.data_ptr() for _, v in row] for row in outs])
    keep, ptrs, counts = cuda._scan_arrays(scans)
    ctx.set_tuning(9, sub_bytes)
    try:
        rc = ctx.lib.jpegqs_cuda_decode_scans_async(ctx.h, n, arr, ptrs, counts,
                                                    (C.c_void_p * n)(*[t.data_ptr() for t in data]),
                                                    (C.c_size_t * n)(*[len(f.data) for f in files]), ws.data_ptr() + G,
                                                    need, st.data_ptr() + 256, None)
        torch.cuda.synchronize()
    finally:
        ctx.set_tuning(9, cuda.DECODE_SUB_DEFAULT)
    assert rc == 0
    _check(torch, files, images, outs, ws, st, models)


def test_transcode_batch_copies_the_coefficients(ctx, tmp_path):
    """transcode_batch at -n 0; the files it hands back to the caller ((None, reason): fill bytes before
    RSTn, 0-bit padding, AC refinement without restarts) go through the jpegqs tool, which transcodes
    them on the host as a caller of the batch call does"""
    res = ctx.transcode_batch([f.data for f in LEGAL], 0, 0)
    routes = {"device": 0, "fallback": 0}
    for f, (out, reason) in zip(LEGAL, res):
        if out is None:
            assert reason, f.name
            routes["fallback"] += 1
            src, dst = tmp_path / "in.jpg", tmp_path / "out.jpg"
            src.write_bytes(f.data)
            r = subprocess.run([EXE, "-n", "0", "-i", "0", str(src), str(dst)], capture_output=True, text=True)
            assert r.returncode == 0, (f.name, r.stderr)
            out = dst.read_bytes()
        else:
            routes["device"] += 1
        got = df.libjpeg_coefficients(out)
        want = df.libjpeg_coefficients(f.data)
        assert all(np.array_equal(a.coef, b.coef) for a, b in zip(got.comps, want.comps)), f.name
    assert routes["device"] > len(LEGAL) // 2 and routes["fallback"] > 0, routes


def test_decode_pixels_equal_libjpeg(ctx):
    from PIL import Image
    res = ctx.decode_pixels([f.data for f in LEGAL], qs.JPEGQS_TRANSCODE, 0)
    for f, rec in zip(LEGAL, res):
        px = rec[0].cpu().numpy()
        want = np.asarray(Image.open(io.BytesIO(f.data)))
        assert np.array_equal(px.reshape(want.shape), want), (f.name, rec[-1])
