"""jpegqs_cuda_decode_async / QsContext.decode_async on the GPU against libjpeg-turbo's
jpeg_read_coefficients: every flavour at the default and the smallest subsequence size, an 8K file
whose subsequences span many thread blocks, a mixed batch of several launch groups, the pipeline
decode -> run_async -> render_async on torch's default stream, the stream rules, one CUDA graph
replayed on a second file, argument errors, and malformed files next to good ones."""
import numpy as np
import pytest

import decode_files as df
import libjpeg_pixels as lp
import oracle_lib as ol
import jpegqs_b200 as qs
from jpegqs_b200 import cuda
from jpegqs_b200.cuda import QsContext

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(lp.JPEG_SO is None, reason="no libjpeg inside Pillow")]

FLAVOURS = df.flavours()


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


def _same(tensors, ref):
    return len(tensors) == len(ref.comps) and all(np.array_equal(t.cpu().numpy(), c.coef) for t, c in zip(tensors, ref.comps))


@pytest.mark.parametrize("sub_bytes", [cuda.DECODE_SUB_DEFAULT, cuda.DECODE_SUB_MIN])
def test_flavours_equal_libjpeg(torch, ctx, sub_bytes):
    ctx.set_tuning(9, sub_bytes)
    try:
        for name, data in FLAVOURS + [(n, d) for n, _, d in df.hard_sets()]:
            im, scan = qs.parse_jpeg(data)
            coefs, status = ctx.decode_async([im], [scan], [_dev(torch, data)])
            torch.cuda.synchronize()
            assert int(status[0]) == 0, name
            assert _same(coefs[0], df.libjpeg_coefficients(data)), name
    finally:
        ctx.set_tuning(9, cuda.DECODE_SUB_DEFAULT)


def test_8k_without_restarts(torch, ctx):
    data = df.pillow_jpeg(7680, 4320, quality=90, subsampling=2)
    im, scan = qs.parse_jpeg(data)
    assert scan.restart_interval == 0
    assert (len(data) - scan.entropy_offset) // cuda.DECODE_SUB_DEFAULT > 8 * 128     # many thread blocks
    ref = df.libjpeg_coefficients(data)
    for sub_bytes in (cuda.DECODE_SUB_DEFAULT, 4096):
        ctx.set_tuning(9, sub_bytes)
        coefs, status = ctx.decode_async([im], [scan], [_dev(torch, data)])
        torch.cuda.synchronize()
        assert int(status[0]) == 0 and _same(coefs[0], ref), sub_bytes
    ctx.set_tuning(9, cuda.DECODE_SUB_DEFAULT)


def test_mixed_batch_equals_single_decodes(torch, ctx):
    # every other flavour: restart and non-restart files, 1, 3 and 4 components, writer 4:1:1 / 4:4:0,
    # more than two launch groups of 8
    files = [d for _, d in FLAVOURS][::2] + [dict(FLAVOURS)[n] for n in ("rst_blocks7", "cmyk", "keep_rgb", "writer_440")]
    assert len(files) > 16
    parsed = [qs.parse_jpeg(d) for d in files]
    coefs, status = ctx.decode_async([p[0] for p in parsed], [p[1] for p in parsed], [_dev(torch, d) for d in files])
    torch.cuda.synchronize()
    assert ctx.last_launches == 10 * -(-len(files) // 8)
    assert status.cpu().tolist() == [0] * len(files)
    for i, d in enumerate(files):
        one, st = ctx.decode_async([parsed[i][0]], [parsed[i][1]], [_dev(torch, d)])
        torch.cuda.synchronize()
        assert all(torch.equal(a, b) for a, b in zip(coefs[i], one[0])), i


@pytest.mark.parametrize("flags", [0, 3, 7])
def test_pipeline_on_the_default_stream(torch, ctx, flags):
    data = dict(FLAVOURS)["420_q75"]
    ref = df.libjpeg_coefficients(data)
    im, scan = qs.parse_jpeg(data)
    dev = _dev(torch, data)
    torch.cuda.synchronize()
    torch.cuda._sleep(50_000_000)
    coefs, status = ctx.decode_async([im], [scan], [dev])
    work = [im.clone()]
    st2, ups = ctx.run_async(work, coefs, flags, 1)
    rgb = ctx.render_async(work, coefs, st2, ups)[0]
    torch.cuda.synchronize()
    assert int(status[0]) == 0
    oret, oout = ol.run_oracle(ref, flags, 1, with_upsampled=True)[:2]
    up = int(st2[0, 1])
    got = [t.cpu().numpy() for t in coefs[0]]
    if up:
        got[1:3] = [u.cpu().numpy() for u in ups[0]]
    assert all(np.array_equal(a, b.coef) for a, b in zip(got, oout.comps))
    assert np.array_equal(rgb.cpu().numpy(), lp.decode(oout))


def test_plain_render_is_libjpegs(torch, ctx):
    data = dict(FLAVOURS)["422_q75"]
    im, scan = qs.parse_jpeg(data)
    coefs, status = ctx.decode_async([im], [scan], [_dev(torch, data)])
    rgb = ctx.render_async([im], coefs)[0]
    torch.cuda.synchronize()
    assert int(status[0]) == 0
    assert np.array_equal(rgb.cpu().numpy(), lp.decode(df.libjpeg_coefficients(data)))


def test_stream_rules(torch, ctx):
    data = dict(FLAVOURS)["444_q75"]
    ref = df.libjpeg_coefficients(data)
    im, scan = qs.parse_jpeg(data)
    s = torch.cuda.Stream()
    dev = _dev(torch, data)
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(200_000_000)
        im2, scan2 = qs.parse_jpeg(data)
        coefs, status = ctx.decode_async([im2], [scan2], [dev], stream=s)
        busy = not s.query()
        del im2, scan2                                           # host inputs may go at return
    assert busy
    s.synchronize()
    assert int(status[0]) == 0 and _same(coefs[0], ref)
    # two calls on two streams, separate workspaces
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    other = dict(FLAVOURS)["gray_q75"]
    imo, scano = qs.parse_jpeg(other)
    devo = _dev(torch, other)
    torch.cuda.synchronize()
    with torch.cuda.stream(s1):
        torch.cuda._sleep(20_000_000)
        c1, t1 = ctx.decode_async([im], [scan], [dev], stream=s1)
    with torch.cuda.stream(s2):
        torch.cuda._sleep(20_000_000)
        c2, t2 = ctx.decode_async([imo], [scano], [devo], stream=s2)
    torch.cuda.synchronize()
    assert int(t1[0]) == 0 and int(t2[0]) == 0
    assert _same(c1[0], ref) and _same(c2[0], df.libjpeg_coefficients(other))


def test_argument_errors_change_nothing(torch, ctx):
    data = dict(FLAVOURS)["420_q75"]
    im, scan = qs.parse_jpeg(data)
    dev = _dev(torch, data)
    out = [torch.full((c.hblk, c.wblk, 64), 7, dtype=torch.int16, device="cuda") for c in im.comps]
    before = [t.clone() for t in out]
    lib = ctx.lib
    import ctypes as C
    arr = cuda._image_array([im], [[t.data_ptr() for t in out]])
    lens = (C.c_size_t * 1)(len(data))
    ptrs = (C.c_void_p * 1)(dev.data_ptr())
    need = qs.decode_workspace_bytes([im], [scan], [len(data)])
    ws = torch.empty(need + 256, dtype=torch.uint8, device="cuda")
    st = torch.full((1,), 99, dtype=torch.int32, device="cuda")
    sc = (cuda._Scan * 1)(scan)
    assert lib.jpegqs_cuda_decode_async(ctx.h, 1, arr, sc, ptrs, lens, ws.data_ptr(), need - 1, st.data_ptr(), None) == -2
    assert lib.jpegqs_cuda_decode_async(ctx.h, 1, arr, sc, ptrs, lens, ws.data_ptr() + 16, need, st.data_ptr(), None) == -2
    bad = cuda._Scan.from_buffer_copy(scan); bad.dc_tbl[0] = 3
    assert lib.jpegqs_cuda_decode_async(ctx.h, 1, arr, (cuda._Scan * 1)(bad), ptrs, lens, ws.data_ptr(), need, st.data_ptr(), None) == -2
    arr2 = cuda._image_array([im], [[out[0].data_ptr() + 2] + [t.data_ptr() for t in out[1:]]])
    assert lib.jpegqs_cuda_decode_async(ctx.h, 1, arr2, sc, ptrs, lens, ws.data_ptr(), need, st.data_ptr(), None) == -2
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(out, before)) and int(st[0]) == 99
    with pytest.raises(ValueError):
        ctx.decode_async([im], [scan], [dev[:scan.entropy_offset]])


def test_graph_replays_on_the_next_file(torch, ctx):
    a = df.pillow_jpeg(160, 96, quality=80, seed=1)
    b = df.pillow_jpeg(160, 96, quality=80, seed=2)
    ia, sa = qs.parse_jpeg(a)
    ib, sb = qs.parse_jpeg(b)
    assert len(b) <= len(a) + 4096
    buf = torch.zeros(len(a) + 4096, dtype=torch.uint8, device="cuda")
    buf[:len(a)] = _dev(torch, a)
    work = [ia.clone()]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                                   # warm-up outside the capture
        ctx.decode_async([ia], [sa], [buf])
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        coefs, status = ctx.decode_async([ia], [sa], [buf])
        st2, ups = ctx.run_async(work, coefs, 3, 1)
        rgb = ctx.render_async(work, coefs, st2, ups)[0]
    buf.zero_()
    buf[:len(b)] = _dev(torch, b)
    g.replay()
    torch.cuda.synchronize()
    assert int(status[0]) == 0
    oret, oout = ol.run_oracle(df.libjpeg_coefficients(b), 3, 1, with_upsampled=True)[:2]
    assert all(np.array_equal(t.cpu().numpy(), c.coef) for t, c in zip(coefs[0], oout.comps))
    assert np.array_equal(rgb.cpu().numpy(), lp.decode(oout))


def test_malformed_files_beside_good_ones(torch, ctx):
    good = dict(FLAVOURS)["420_q75"]
    rst = dict(FLAVOURS)["rst_blocks7"]
    im, scan = qs.parse_jpeg(good)
    imr, scanr = qs.parse_jpeg(rst)
    off, offr = scan.entropy_offset, scanr.entropy_offset
    trunc = good[:off + (len(good) - off) // 2]
    flip = bytearray(good); flip[off + 40] ^= 0xFF; flip[off + 41] = 0x00
    p = rst.index(b"\xff\xd3", offr)
    no_rst = rst[:p] + rst[p + 2:]
    files = [(im, scan, good), (im, scan, trunc), (imr, scanr, rst), (imr, scanr, no_rst), (im, scan, bytes(flip))]
    G = 4096
    outs, guards = [], []
    for i, s_, d in files:
        per = []
        for c in i.comps:
            n = c.hblk * c.wblk * 64
            big = torch.full((n + 2 * G,), 0x2B2B, dtype=torch.int16, device="cuda")
            guards.append(big)
            per.append(big[G:G + n].view(c.hblk, c.wblk, 64))
        outs.append(per)
    coefs, status = ctx.decode_async([f[0] for f in files], [f[1] for f in files], [_dev(torch, f[2]) for f in files], out=outs)
    torch.cuda.synchronize()
    st = status.cpu().tolist()
    assert st[0] == 0 and st[2] == 0
    assert st[1] & (cuda.DECODE_TRUNCATED | cuda.DECODE_UNITS)
    assert st[3] & cuda.DECODE_RESTART
    assert st[4] != 0 or _same(coefs[4], qs.read_jpeg(bytes(flip)))
    assert _same(coefs[0], df.libjpeg_coefficients(good)) and _same(coefs[2], df.libjpeg_coefficients(rst))
    for big in guards:
        assert bool((big[:G] == 0x2B2B).all()) and bool((big[-G:] == 0x2B2B).all())


def _damaged():
    good = dict(FLAVOURS)["420_q75"]
    rst = dict(FLAVOURS)["rst_blocks7"]
    off = qs.parse_jpeg(good)[1].entropy_offset
    offr = qs.parse_jpeg(rst)[1].entropy_offset
    flip = bytearray(good)
    for p in range(off + 5, len(good) - 2, 53):
        flip[p] ^= 0xA5
    p = rst.index(b"\xff\xd2", offr)
    return [good, good[:off + 1], good[:off + (len(good) - off) // 3], bytes(flip), rst[:p] + rst[p + 2:],
            dict(FLAVOURS)["cmyk"][:-300], rst, dict(FLAVOURS)["gray_q100"], dict(FLAVOURS)["writer_411"]]


@pytest.mark.parametrize("sub_bytes", [cuda.DECODE_SUB_MIN, cuda.DECODE_SUB_DEFAULT])
def test_workspace_and_status_stay_in_bounds(torch, ctx, sub_bytes):
    """Damaged and good files in one call through the C ABI, with guard regions around the
    workspace and the status array: the decoder writes only inside the sizes it documents."""
    import ctypes as C
    files = _damaged()
    parsed = [qs.parse_jpeg(f) for f in files]
    images, scans = [p[0] for p in parsed], [p[1] for p in parsed]
    data = [_dev(torch, f) for f in files]
    out = [[torch.empty((c.hblk, c.wblk, 64), dtype=torch.int16, device="cuda") for c in im.comps] for im in images]
    n, G = len(files), 1 << 16
    need = qs.decode_workspace_bytes(images, scans, [len(f) for f in files])
    ws = torch.full((need + 2 * G,), 0x6D, dtype=torch.uint8, device="cuda")
    st = torch.full((n + 2 * 64,), 0x1234567, dtype=torch.int32, device="cuda")
    arr = cuda._image_array(images, [[t.data_ptr() for t in o] for o in out])
    ctx.set_tuning(9, sub_bytes)
    try:
        rc = ctx.lib.jpegqs_cuda_decode_async(ctx.h, n, arr, (cuda._Scan * n)(*scans),
                                              (C.c_void_p * n)(*[t.data_ptr() for t in data]),
                                              (C.c_size_t * n)(*[len(f) for f in files]), ws.data_ptr() + G, need,
                                              st.data_ptr() + 256, None)
        torch.cuda.synchronize()
    finally:
        ctx.set_tuning(9, cuda.DECODE_SUB_DEFAULT)
    assert rc == 0
    assert bool((ws[:G] == 0x6D).all()) and bool((ws[-G:] == 0x6D).all())
    assert bool((st[:64] == 0x1234567).all()) and bool((st[-64:] == 0x1234567).all())
    status = st[64:64 + n].cpu().tolist()
    assert [status[i] for i in (0, 6, 7, 8)] == [0, 0, 0, 0]
    assert all(status[i] != 0 for i in (1, 2, 4, 5)), status
    assert status[4] & cuda.DECODE_RESTART
    for i in (0, 6, 7, 8):
        assert _same(out[i], df.libjpeg_coefficients(files[i])), i


def test_two_threads_on_two_contexts(torch):
    """One host thread per context, both decoding at once: every call's descriptors are its own."""
    import threading
    names = ["420_q75", "cmyk", "rst_blocks7", "gray_q100", "writer_440", "444_q100", "422_q30", "keep_rgb", "size_33x47"]
    files = [dict(FLAVOURS)[n] for n in names]
    refs = [df.libjpeg_coefficients(f) for f in files]
    errors = []

    def worker(order):
        c = QsContext(0)
        try:
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                for rep in range(6):
                    picks = order[rep % len(order):] + order[:rep % len(order)]
                    parsed = [qs.parse_jpeg(files[k]) for k in picks]
                    coefs, status = c.decode_async([p[0] for p in parsed], [p[1] for p in parsed],
                                                   [_dev(torch, files[k]) for k in picks], stream=s)
                    s.synchronize()
                    for j, k in enumerate(picks):
                        if int(status[j]) != 0 or not _same(coefs[j], refs[k]):
                            errors.append((names[k], rep))
        except Exception as e:                                   # noqa: BLE001
            errors.append(repr(e))
        finally:
            c.close()

    ts = [threading.Thread(target=worker, args=(list(range(len(files))),)),
          threading.Thread(target=worker, args=(list(reversed(range(len(files)))),))]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors
