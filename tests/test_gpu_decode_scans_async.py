"""jpegqs_cuda_decode_scans_async / QsContext.decode_scans_async on the GPU against libjpeg-turbo's
jpeg_read_coefficients and the host reader: every flavour of the CPU tests, an 8K progressive file
without restarts, a batch of several launch groups, progressive input through decode -> run_async ->
encode against the jpegqs tool's file, the stream rules, argument errors, a graph replay and damaged
files beside good ones with guard regions."""
import ctypes as C
import subprocess

import numpy as np
import pytest

import decode_files as df
import libjpeg_pixels as lp
import scan_files as sf
from test_decode_scans_cpu import HARD, PILLOW, SCRIPTED, _cut_at_sos, _damaged
from test_encode_cpu import EXE, _tool_flags
import jpegqs_b200 as qs
from jpegqs_b200 import cuda
from jpegqs_b200.cuda import QsContext

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(lp.JPEG_SO is None, reason="no libjpeg inside Pillow")]

ALL = PILLOW + SCRIPTED + HARD


@pytest.fixture(scope="module")
def torch():
    import torch as t
    return t


@pytest.fixture(scope="module")
def ctx():
    c = QsContext(0)
    yield c
    c.close()


def _dev(torch, data):
    return torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()


def _same(coefs, ref):
    return len(coefs) == len(ref.comps) and all(np.array_equal(t.cpu().numpy(), c.coef) for t, c in zip(coefs, ref.comps))


@pytest.mark.parametrize("sub_bytes", [cuda.DECODE_SUB_MIN, cuda.DECODE_SUB_DEFAULT])
def test_flavours_equal_libjpeg(torch, ctx, sub_bytes):
    ctx.set_tuning(9, sub_bytes)
    try:
        parsed = [qs.parse_jpeg_scans(d) for _, d in ALL]
        coefs, status = ctx.decode_scans_async([p[0] for p in parsed], [p[1] for p in parsed],
                                               [_dev(torch, d) for _, d in ALL])
        torch.cuda.synchronize()
        st = status.cpu().tolist()
        for (name, data), c, s in zip(ALL, coefs, st):
            assert s == 0, name
            assert _same(c, df.libjpeg_coefficients(data)), name
    finally:
        ctx.set_tuning(9, cuda.DECODE_SUB_DEFAULT)


def test_8k_progressive_without_restarts(torch, ctx):
    data = df.pillow_jpeg(7680, 4320, quality=90, subsampling=2, progressive=True)
    im, scans = qs.parse_jpeg_scans(data)
    assert all(r.restart_interval == 0 for r in scans)
    coefs, status = ctx.decode_scans_async([im], [scans], [_dev(torch, data)])
    torch.cuda.synchronize()
    assert int(status[0]) == 0
    ref = qs.read_jpeg(data)
    assert all(np.array_equal(t.cpu().numpy(), c.coef) for t, c in zip(coefs[0], ref.comps))


def test_mixed_batch_over_several_groups(torch, ctx):
    kinds = [d for _, d in PILLOW[:4]] + [dict(SCRIPTED)["seq_per_comp_420"], dict(SCRIPTED)["succ_al3_420_rst3"],
                                          df.pillow_jpeg(120, 80, quality=80), df.pillow_jpeg(120, 80, "CMYK", quality=85)]
    files = [kinds[i % len(kinds)] for i in range(37)]            # 3 groups of up to 16 images
    parsed = [qs.parse_jpeg_scans(d) for d in files]
    data = [_dev(torch, d) for d in files]
    coefs, status = ctx.decode_scans_async([p[0] for p in parsed], [p[1] for p in parsed], data)
    torch.cuda.synchronize()
    assert status.cpu().tolist() == [0] * len(files)
    for i, d in enumerate(files):
        one, s1 = ctx.decode_scans_async([parsed[i][0]], [parsed[i][1]], [data[i]])
        torch.cuda.synchronize()
        assert int(s1[0]) == 0
        assert all(torch.equal(a, b) for a, b in zip(coefs[i], one[0])), i


@pytest.mark.parametrize("args", [["-q", "3", "-o"], ["-q", "6", "-o"]])
def test_progressive_pipeline_gives_the_tools_file(torch, ctx, tmp_path, args):
    for name in ("prog_420", "prog_444", "prog_gray"):
        data = dict(PILLOW)[name]
        src, dst = tmp_path / "in.jpg", tmp_path / "out.jpg"
        src.write_bytes(data)
        r = subprocess.run([EXE, *args, str(src), str(dst)], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        want = dst.read_bytes()
        flags, niter = _tool_flags(args)
        im, scans = qs.parse_jpeg_scans(data)
        coefs, dst_st = ctx.decode_scans_async([im], [scans], [_dev(torch, data)])
        work = [im.clone()]
        rst, ups = ctx.run_async(work, coefs, flags, niter)
        pre, ids, tbls = qs.jpeg_prefix(data, 2)
        out, lengths, status = ctx.encode_async(work, coefs, [(_dev(torch, pre), ids, tbls)], True, rst, ups)
        torch.cuda.synchronize()
        assert int(dst_st[0]) == 0 and int(status[0]) == 0
        assert bytes(out[0][:int(lengths[0])].cpu().numpy()) == want, name


def test_stream_rules(torch, ctx):
    data = dict(PILLOW)["prog_420"]
    im, scans = qs.parse_jpeg_scans(data)
    ref = df.libjpeg_coefficients(data)
    d = _dev(torch, data)
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(200_000_000)
        coefs, st = ctx.decode_scans_async([im], [scans], [d], stream=s)
        busy = not s.query()
    assert busy
    s.synchronize()
    assert int(st[0]) == 0 and _same(coefs[0], ref)


def test_argument_errors_leave_outputs_untouched(torch, ctx):
    data = dict(PILLOW)["prog_420"]
    im, scans = qs.parse_jpeg_scans(data)
    d = _dev(torch, data)
    out = [[torch.full((c.hblk, c.wblk, 64), 77, dtype=torch.int16, device="cuda") for c in im.comps]]
    bad = cuda.ScanList(cuda._ScanRec.from_buffer_copy(r) for r in scans)
    bad[-1].Al = 14
    for args in (([im], [bad], [d]), ([im], [scans], [d[:100]])):
        with pytest.raises((cuda.QsError, ValueError)):
            ctx.decode_scans_async(*args, out=out)
    with pytest.raises(ValueError):
        ctx.decode_scans_async([im], [None], [d], out=out)
    torch.cuda.synchronize()
    assert all(bool((t == 77).all()) for t in out[0])


def test_c_argument_errors_enqueue_nothing(torch, ctx):
    """The C entry point itself: a workspace too small or not 256-byte aligned, a NULL data pointer and
    a bad scan record are refused before anything is enqueued - outputs and status stay as they were."""
    data = dict(PILLOW)["prog_420"]
    im, scans = qs.parse_jpeg_scans(data)
    d = _dev(torch, data)
    out = [torch.full((c.hblk, c.wblk, 64), 77, dtype=torch.int16, device="cuda") for c in im.comps]
    status = torch.full((1,), 1234, dtype=torch.int32, device="cuda")
    need = qs.decode_scans_workspace_bytes([im], [scans], [len(data)])
    ws = torch.empty(need + 512, dtype=torch.uint8, device="cuda")
    arr = cuda._image_array([im], [[t.data_ptr() for t in out]])
    keep, ptrs, counts = cuda._scan_arrays([scans])
    bad = cuda.ScanList(cuda._ScanRec.from_buffer_copy(r) for r in scans)
    bad[3].Se = 64
    kb, bptrs, bcounts = cuda._scan_arrays([bad])
    lens = (C.c_size_t * 1)(len(data))
    dptr, nullptr = (C.c_void_p * 1)(d.data_ptr()), (C.c_void_p * 1)(None)
    base = ws.data_ptr()
    cases = [(ptrs, counts, dptr, base, need - 1), (ptrs, counts, dptr, base + 16, need),
             (ptrs, counts, nullptr, base, need), (bptrs, bcounts, dptr, base, need)]
    torch.cuda.synchronize()
    for sp, cn, dp, w, size in cases:
        rc = ctx.lib.jpegqs_cuda_decode_scans_async(ctx.h, 1, arr, sp, cn, dp, lens, w, size, status.data_ptr(), None)
        assert rc == -2
        assert ctx.last_launches == 0
    torch.cuda.synchronize()
    assert int(status[0]) == 1234 and all(bool((t == 77).all()) for t in out)
    rc = ctx.lib.jpegqs_cuda_decode_scans_async(ctx.h, 1, arr, ptrs, counts, dptr, lens, base, need, status.data_ptr(), None)
    torch.cuda.synchronize()
    assert rc == 0 and int(status[0]) == 0 and _same(out, df.libjpeg_coefficients(data))


def test_graph_replay_rewrites_garbage(torch, ctx):
    data = dict(SCRIPTED)["split_bands_420_rst3"]
    im, scans = qs.parse_jpeg_scans(data)
    ref = df.libjpeg_coefficients(data)
    d = _dev(torch, data)
    out = [[torch.empty((c.hblk, c.wblk, 64), dtype=torch.int16, device="cuda") for c in im.comps]]
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):                                   # warm up: allocations outside the graph
        ctx.decode_scans_async([im], [scans], [d], out=out, stream=s)
    s.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        _, status = ctx.decode_scans_async([im], [scans], [d], out=out, stream=s)
    for t in out[0]:
        t.random_(-30000, 30000)
    g.replay()
    torch.cuda.synchronize()
    assert int(status[0]) == 0 and _same(out[0], ref)


def test_damaged_files_beside_good_ones(torch, ctx):
    rng = np.random.default_rng(11)
    good = dict(PILLOW)["prog_420"]
    files = []
    for it in range(24):
        src = [good, dict(SCRIPTED)["succ_al3_420_rst3"], dict(PILLOW)["prog_rst_blocks5"]][it % 3]
        dmg = _damaged(rng, src, it % 3)
        try:
            im, scans = qs.parse_jpeg_scans(dmg)
        except cuda.QsError:
            continue
        if scans is not None:
            files.append((dmg, im, scans))
        files.append((good, *qs.parse_jpeg_scans(good)))
    for extra in (1, 2):                                         # cut just after an SOS header
        dmg = _cut_at_sos(good, extra)
        files.append((dmg, *qs.parse_jpeg_scans(dmg)))
    guard = 4096
    bufs, views = [], []
    for _, im, _ in files:
        b = [torch.full((c.hblk * c.wblk * 64 + 2 * guard,), 0x5A5A, dtype=torch.int16, device="cuda") for c in im.comps]
        bufs.append(b)
        views.append([x[guard:-guard].view(c.hblk, c.wblk, 64) for x, c in zip(b, im.comps)])
    _, status = ctx.decode_scans_async([f[1] for f in files], [f[2] for f in files],
                                       [_dev(torch, f[0]) for f in files], out=views)
    torch.cuda.synchronize()
    st = status.cpu().tolist()
    for (data, _, _), b, v, s in zip(files, bufs, views, st):
        assert all(bool((x[:guard] == 0x5A5A).all()) and bool((x[-guard:] == 0x5A5A).all()) for x in b)
        if s == 0:
            ref = qs.read_jpeg(data)
            assert all(np.array_equal(t.cpu().numpy(), c.coef) for t, c in zip(v, ref.comps))
    assert any(st) and st.count(0) >= 12
