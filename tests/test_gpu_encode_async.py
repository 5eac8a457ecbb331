"""jpegqs_cuda_encode_async / QsContext.encode_async on the GPU against the CPU model and the jpegqs
tool's writer: every flavour with standard and optimal tables, the unmodified reference tool's bytes
through decode -> run_async -> encode, an 8K image, a batch of several launch groups, one CUDA graph
holding the whole pipeline with an image that stops and one that up-samples, OVERFLOW and RANGE
beside good images with guard regions, the stream rules and argument errors."""
import ctypes as C
import hashlib
import io

import numpy as np
import pytest

import decode_files as df
import hard_content as hc
import libjpeg_pixels as lp
from golden_io import reference_files
from render_images import make
from test_cli import REF_TOOL_CASES, file_key, write_jpegs
from test_encode_cpu import ALL, NAT, _gray, _tool_flags, model_bytes, tool_bytes
import jpegqs_b200 as qs
from jpegqs_b200 import cuda
from jpegqs_b200.cuda import QsContext

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(lp.JPEG_SO is None, reason="no libjpeg inside Pillow")]


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


def _head(torch, data, copy=2):
    pre, ids, tbls = qs.jpeg_prefix(data, copy)
    return (_dev(torch, pre), ids, tbls), (pre, ids, tbls)


def _files(out, lengths, status):
    ln, st = lengths.cpu().tolist(), status.cpu().tolist()
    return [bytes(o[:n].cpu().numpy()) if s == 0 else None for o, n, s in zip(out, ln, st)], st


def _upload(torch, im):
    return [torch.from_numpy(np.ascontiguousarray(c.coef)).cuda() for c in im.comps]


@pytest.mark.parametrize("optimize", [False, True])
def test_flavours_equal_the_model_and_the_tool(torch, ctx, tmp_path, optimize):
    from PIL import Image
    for name, data in ALL:
        im = qs.read_jpeg(data)
        head, _ = _head(torch, data)
        out, lengths, status = ctx.encode_async([im], [_upload(torch, im)], [head], optimize)
        torch.cuda.synchronize()
        (got,), st = _files(out, lengths, status)
        assert st == [0], name
        assert got == model_bytes(data, optimize) == tool_bytes(tmp_path, data, optimize), name
        Image.open(io.BytesIO(got)).load()
        back = df.libjpeg_coefficients(got)
        assert all(np.array_equal(a.coef, b.coef) for a, b in zip(back.comps, im.comps)), name


@pytest.fixture(scope="module")
def jpegs(tmp_path_factory):
    return write_jpegs(str(tmp_path_factory.mktemp("jpegs")))


@pytest.mark.parametrize("name,args", REF_TOOL_CASES)
def test_reference_tools_bytes(torch, ctx, jpegs, name, args):
    data = open(jpegs[name], "rb").read()
    flags, niter = _tool_flags(args)
    im, scan = qs.parse_jpeg(data)
    if scan is not None:
        coefs, dst = ctx.decode_async([im], [scan], [_dev(torch, data)])
    else:
        im = qs.read_jpeg(data)
        coefs, dst = [_upload(torch, im)], torch.zeros(1, dtype=torch.int32, device="cuda")
    work = [im.clone()]
    rst, ups = ctx.run_async(work, coefs, flags, niter)
    head, _ = _head(torch, data)
    out, lengths, status = ctx.encode_async(work, coefs, [head], "-o" in args, rst, ups)
    torch.cuda.synchronize()
    (got,), st = _files(out, lengths, status)
    assert int(dst[0]) == 0 and st == [0]
    assert hashlib.sha256(got).hexdigest() == reference_files()["jpegqs_ref"][file_key(name, args)]


def test_8k_and_a_mixed_batch(torch, ctx):
    big = df.pillow_jpeg(7680, 4320, quality=90, subsampling=2)
    files = [big] + [d for _, d in ALL]                # 1, 3 and 4 components, every sampling
    assert len(files) > 2 * 16
    ims = [qs.read_jpeg(d) for d in files]
    heads = [_head(torch, d) for d in files]
    for optimize in (False, True):
        out, lengths, status = ctx.encode_async(ims, [_upload(torch, im) for im in ims], [h[0] for h in heads], optimize)
        torch.cuda.synchronize()
        assert ctx.last_launches == (10 if optimize else 9) * -(-len(files) // 16)
        got, st = _files(out, lengths, status)
        assert st == [0] * len(files)
        for i, (d, im) in enumerate(zip(files, ims)):
            want, s = qs.encode_model(im, [c.coef for c in im.comps], *heads[i][1], optimize)
            assert s == 0 and got[i] == want, i
            if i in (0, 5, len(files) - 1):
                one, ln, s1 = ctx.encode_async([im], [_upload(torch, im)], [heads[i][0]], optimize)
                torch.cuda.synchronize()
                assert _files(one, ln, s1)[0][0] == want


def _stop_file():
    im = hc.with_dequant_edge(make(64, 48, "420", "k50", "synth", 3), True)
    return df.coef_writer_jpeg(im)


def test_graph_pipeline_with_a_stop_and_an_up_sample(torch, ctx):
    """decode -> run_async (q6: UPSAMPLE_UV) -> encode in one graph: one image stops (written at its
    own sampling), one up-samples (written 1x1 from coef_up); each file equals the model run on what
    the run left on the device.  A replay on second files of the same headers gives their bytes."""
    a = [_stop_file(), df.pillow_jpeg(160, 96, quality=80, seed=1), df.pillow_jpeg(97, 61, "L", quality=75, seed=1)]
    b = [_stop_file(), df.pillow_jpeg(160, 96, quality=80, seed=2), df.pillow_jpeg(97, 61, "L", quality=75, seed=2)]
    parsed = [qs.parse_jpeg(d) for d in a]
    assert all(len(y) <= len(x) + 4096 for x, y in zip(a, b)) and all(p[1] is not None for p in parsed)
    bufs = [torch.zeros(len(d) + 4096, dtype=torch.uint8, device="cuda") for d in a]
    for buf, d in zip(bufs, a):
        buf[:len(d)] = _dev(torch, d)
    heads = [_head(torch, d)[0] for d in a]
    ims = [p[0] for p in parsed]
    flags = qs.quality_to_flags(6)

    def pipeline():
        work = [im.clone() for im in ims]
        coefs, dst = ctx.decode_async(ims, [p[1] for p in parsed], bufs)
        rst, ups = ctx.run_async(work, coefs, flags, 1)
        out, lengths, status = ctx.encode_async(work, coefs, heads, True, rst, ups)
        return work, coefs, dst, rst, ups, out, lengths, status

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        pipeline()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        work, coefs, dst, rst, ups, out, lengths, status = pipeline()

    def check(files):
        got, st = _files(out, lengths, status)
        r = rst.cpu().tolist()
        assert dst.cpu().tolist() == [0, 0, 0] and st == [0, 0, 0]
        assert r[0][0] != 0 and r[0][1] == 0 and r[1][1] == 1 and r[2][1] == 0
        for i in range(3):
            arrays = [t.cpu().numpy() for t in coefs[i]]
            up = [u.cpu().numpy() for u in ups[i]] if r[i][1] else None
            pre, ids, tbls = qs.jpeg_prefix(files[i])
            want, s_ = qs.encode_model(work[i], arrays, pre, ids, tbls, True, up=up)
            assert s_ == 0 and got[i] == want, i
        assert b"\xff\xc0\x00\x11\x08" in got[1] and got[1][got[1].index(b"\xff\xc0") + 11] == 0x11   # luma 1x1

    g.replay()
    torch.cuda.synchronize()
    check(a)
    for buf, d in zip(bufs, b):
        buf.zero_()
        buf[:len(d)] = _dev(torch, d)
    g.replay()
    torch.cuda.synchronize()
    check(b)


def test_overflow_range_and_guards(torch, ctx):
    data = dict(df.flavours())["420_q75"]
    im = qs.read_jpeg(data)
    head, host = _head(torch, data)
    want = model_bytes(data)
    rb = np.zeros((2, 3, 64), np.int16)
    rb[1, 1, NAT[5]] = 1024
    rim = _gray(rb)
    rdata = df.pillow_jpeg(24, 16, "L", quality=75)
    rhead, _ = _head(torch, rdata)
    ims = [im, im, im, rim, im]
    caps = [len(want) - 1, len(want), len(want) + 1000, 4096, len(want)]
    G = 4096
    bigs = [torch.full((c + 2 * G,), 0x5A, dtype=torch.uint8, device="cuda") for c in caps]
    outs = [b[G:G + c] for b, c in zip(bigs, caps)]
    n = len(ims)
    need = qs.encode_workspace_bytes(ims)
    ws = torch.full((need + 2 * G,), 0x6D, dtype=torch.uint8, device="cuda")
    ln = torch.full((n + 16,), 0x1234, dtype=torch.int64, device="cuda")
    st = torch.full((n + 16,), 0x1234, dtype=torch.int32, device="cuda")
    coefs = [_upload(torch, x) for x in ims]
    arr = cuda._image_array(ims, [[t.data_ptr() for t in c] for c in coefs])
    hs = (cuda._Head * n)(*[cuda._head(h[0].data_ptr(), h[0].numel(), h[1], h[2], len(x.comps))
                            for h, x in zip([head, head, head, rhead, head], ims)])
    rc = ctx.lib.jpegqs_cuda_encode_async(ctx.h, n, arr, hs, 0, None, (C.c_void_p * n)(*[o.data_ptr() for o in outs]),
                                          (C.c_size_t * n)(*caps), ln.data_ptr() + 64, st.data_ptr() + 32,
                                          ws.data_ptr() + G, need, None)
    torch.cuda.synchronize()
    assert rc == 0
    lens, stat = ln[8:8 + n].cpu().tolist(), st[8:8 + n].cpu().tolist()
    assert stat == [cuda.ENCODE_OVERFLOW, 0, 0, cuda.ENCODE_RANGE, 0]
    assert lens[0] == lens[1] == lens[2] == lens[4] == len(want)
    for i in (1, 2, 4):
        assert bytes(outs[i][:len(want)].cpu().numpy()) == want
    for b in bigs:
        assert bool((b[:G] == 0x5A).all()) and bool((b[-G:] == 0x5A).all())
    assert bool((ws[:G] == 0x6D).all()) and bool((ws[-G:] == 0x6D).all())
    assert bool((ln[:8] == 0x1234).all()) and bool((ln[8 + n:] == 0x1234).all())
    assert bool((st[:8] == 0x1234).all()) and bool((st[8 + n:] == 0x1234).all())


def test_stream_rules(torch, ctx):
    data = dict(df.flavours())["444_q75"]
    im = qs.read_jpeg(data)
    want = model_bytes(data)
    coefs = _upload(torch, im)
    head, _ = _head(torch, data)
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(200_000_000)
        out, ln, st = ctx.encode_async([im.clone()], [coefs], [head], stream=s)
        busy = not s.query()
    assert busy
    s.synchronize()
    assert _files(out, ln, st)[0] == [want]
    other = dict(df.flavours())["gray_q75"]
    imo = qs.read_jpeg(other)
    co, ho = _upload(torch, imo), _head(torch, other)[0]
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s1):
        torch.cuda._sleep(20_000_000)
        r1 = ctx.encode_async([im], [coefs], [head], True, stream=s1)
    with torch.cuda.stream(s2):
        torch.cuda._sleep(20_000_000)
        r2 = ctx.encode_async([imo], [co], [ho], True, stream=s2)
    torch.cuda.synchronize()
    assert _files(*r1)[0] == [model_bytes(data, True)] and _files(*r2)[0] == [model_bytes(other, True)]


def test_argument_errors_change_nothing(torch, ctx):
    data = dict(df.flavours())["420_q75"]
    im = qs.read_jpeg(data)
    coefs = _upload(torch, im)
    head, _ = _head(torch, data)
    cap = qs.encode_bound(im, head[0].numel())
    out = torch.full((cap,), 7, dtype=torch.uint8, device="cuda")
    ln = torch.full((1,), 99, dtype=torch.int64, device="cuda")
    st = torch.full((1,), 99, dtype=torch.int32, device="cuda")
    need = qs.encode_workspace_bytes([im])
    ws = torch.full((need + 256,), 3, dtype=torch.uint8, device="cuda")

    def call(arr, h=None, c=cap, w=ws.data_ptr(), size=need):
        h = h or cuda._head(head[0].data_ptr(), head[0].numel(), head[1], head[2], 3)
        return ctx.lib.jpegqs_cuda_encode_async(ctx.h, 1, arr, (cuda._Head * 1)(h), 0, None, (C.c_void_p * 1)(out.data_ptr()),
                                                (C.c_size_t * 1)(c), ln.data_ptr(), st.data_ptr(), w, size, None)
    good = cuda._image_array([im], [[t.data_ptr() for t in coefs]])
    assert call(good, size=need - 1) == -2
    assert call(good, w=ws.data_ptr() + 16) == -2
    assert call(good, c=head[0].numel() - 1) == -2
    assert call(cuda._image_array([im], [[coefs[0].data_ptr() + 2] + [t.data_ptr() for t in coefs[1:]]])) == -2
    assert call(good, h=cuda._head(head[0].data_ptr(), head[0].numel(), head[1], (0, 1, 7), 3)) == -2
    up = cuda._image_array([im], [[t.data_ptr() for t in coefs]])
    up[0].upsampled = 1                                          # no coef_up
    assert call(up) == -2
    bad = im.clone()
    bad.comps[1].h_samp = 2
    assert call(cuda._image_array([bad], [[t.data_ptr() for t in coefs]])) == -2
    torch.cuda.synchronize()
    assert bool((out == 7).all()) and int(ln[0]) == 99 and int(st[0]) == 99 and bool((ws == 3).all())
    with pytest.raises(ValueError):
        ctx.encode_async([im], [coefs], [(head[0].to(torch.int16), head[1], head[2])])
    with pytest.raises(ValueError):
        ctx.encode_async([im], [coefs], [head], out=[out], capacity=[cap + 1])


def test_run_status_up_sampled_without_coef_up_is_flagged(torch, ctx):
    """An image run_async up-sampled on the device, encoded with its status but without up: written
    at its own sampling (the model on the arrays as they are) and flagged NO_UP, not silently."""
    data = df.pillow_jpeg(160, 96, quality=80, seed=3)
    im, scan = qs.parse_jpeg(data)
    coefs, dst = ctx.decode_async([im], [scan], [_dev(torch, data)])
    work = [im.clone()]
    rst, ups = ctx.run_async(work, coefs, qs.quality_to_flags(6), 1)
    head, host = _head(torch, data)
    out, lengths, status = ctx.encode_async(work, coefs, [head], False, rst)
    torch.cuda.synchronize()
    assert rst.cpu().tolist()[0][1] == 1 and status.cpu().tolist() == [cuda.ENCODE_NO_UP]
    want, s = qs.encode_model(work[0], [t.cpu().numpy() for t in coefs[0]], *host)
    assert s == 0 and bytes(out[0][:int(lengths[0])].cpu().numpy()) == want
