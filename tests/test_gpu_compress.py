"""JPEG files written on the GPU.  jpegqs_cuda_compress_async (QsContext.compress_async) gives, for every
device picture, compress_model's bytes, which are Pillow's Image.save(quality, subsampling, optimize):
for a mixed batch of sizes, grey and RGB pictures, crops of bigger tensors at odd byte offsets and an
8K picture at quality 95, eagerly and replayed from a CUDA graph after the inputs are overwritten.  An
undersized capacity gives OVERFLOW with the needed length and no byte written past it; bad arguments
enqueue nothing.  jpegqs_cuda_pixels_batch_jpeg (QsContext.reencode) gives, for every file, Pillow's
save of the picture decode_pixels gives with the same arguments, at -q 3, -q 6 and -n 0, at d = 1 and
2, with and without a 224 x 224 crop or a 256-pixel bound, for grey, host-route and device-flagged
files; a file the render cannot take, a file the reader rejects and a bad crop fail alone; forced
splits and file order change no byte."""
import ctypes as C
import io

import numpy as np
import pytest

from test_gpu_pixels_batch import OPTS, _shape, corpus, ctx  # noqa: F401  (module fixtures)

import jpegqs_b200 as qs
from jpegqs_b200 import cuda

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
Image = pytest.importorskip("PIL.Image")
ImageFile = pytest.importorskip("PIL.ImageFile")
# with optimize, Pillow gives libjpeg one output buffer of max(MAXBLOCK, about W * H) bytes and
# fails on files larger than that (noise at high quality); a larger buffer changes no byte
ImageFile.MAXBLOCK = 1 << 28

SUBS = ("4:4:4", "4:2:2", "4:2:0")


def pillow(a, quality, subsampling, optimize):
    b = io.BytesIO()
    a = np.asarray(a)
    Image.fromarray(a if a.shape[2] == 3 else a[:, :, 0]).save(b, "JPEG", quality=quality, subsampling=subsampling,
                                                               optimize=optimize)
    return b.getvalue()


def _pictures(seed, dev):
    """host arrays and device views of them: crops of wider tensors (row stride > W * C) at odd byte
    offsets, grey and RGB, sizes around the block and MCU boundaries"""
    rng = np.random.RandomState(seed)
    sizes = [(1, 1, 3), (9, 17, 1), (16, 16, 3), (22, 18, 3), (33, 31, 1), (121, 77, 3), (240, 320, 3), (57, 300, 1)]
    hosts, views, keep = [], [], []
    for k, (h, w, c) in enumerate(sizes):
        a = rng.randint(0, 256, (h, w, c)).astype(np.uint8)
        if k % 3 == 1:
            yy, xx = np.indices((h, w))
            a = np.repeat(((xx * 7 + yy * 3) % 256).astype(np.uint8)[:, :, None], c, 2)
        stride = w * c + 5 * (k % 2)
        flat = torch.full((1 + k + stride * h + 7,), 0x5A, dtype=torch.uint8, device=dev)
        v = torch.as_strided(flat, (h, w, c), (stride, c, 1), 1 + k)
        v.copy_(torch.from_numpy(a))
        hosts.append(a); views.append(v); keep.append(flat)
    return hosts, views, keep


@pytest.mark.parametrize("sub", SUBS)
@pytest.mark.parametrize("quality,optimize", [(75, False), (95, True), (10, False)])
def test_batch_equals_model_and_pillow(ctx, sub, quality, optimize):  # noqa: F811
    dev = f"cuda:{ctx.device}"
    hosts, views, _keep = _pictures(quality, dev)
    out, lens, st = ctx.compress_async(views, quality, sub, optimize)
    torch.cuda.synchronize()
    assert ctx.last_launches > 0
    st, lens = st.cpu().numpy(), lens.cpu().numpy()
    assert not (st & cuda.ENCODE_RANGE).any() and (st == 0).all()
    for a, o, n in zip(hosts, out, lens):
        got = o[:int(n)].cpu().numpy().tobytes()
        assert got == cuda.compress_model(a, quality, sub, optimize) == pillow(a, quality, sub, optimize), a.shape


def test_8k_at_q95(ctx):  # noqa: F811
    rng = np.random.RandomState(8)
    yy, xx = np.indices((4320, 7680))
    a = np.stack([(xx // 3 + yy // 5) % 256, (xx * yy // 97) % 256, rng.randint(0, 256, (4320, 7680))], 2).astype(np.uint8)
    small = rng.randint(0, 256, (61, 97, 1)).astype(np.uint8)
    t = [torch.from_numpy(a).to(f"cuda:{ctx.device}"), torch.from_numpy(small).to(f"cuda:{ctx.device}")]
    out, lens, st = ctx.compress_async(t, 95, "4:2:0", False)
    torch.cuda.synchronize()
    assert st.cpu().tolist() == [0, 0]
    for x, o, n in zip((a, small), out, lens.cpu().tolist()):
        assert o[:n].cpu().numpy().tobytes() == pillow(x, 95, "4:2:0", False)


def test_graph_replay_reads_current_inputs(ctx):  # noqa: F811
    dev = f"cuda:{ctx.device}"
    hosts, views, _keep = _pictures(3, dev)
    s = torch.cuda.Stream(dev)
    with torch.cuda.stream(s):
        ctx.compress_async(views, 85, "4:2:0", True, stream=s)        # warm-up: allocator pools
    s.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        out, lens, st = ctx.compress_async(views, 85, "4:2:0", True, stream=s)
    rng = np.random.RandomState(4)
    for rep in range(2):
        fresh = [rng.randint(0, 256, a.shape).astype(np.uint8) for a in hosts]
        for v, a in zip(views, fresh):
            v.copy_(torch.from_numpy(a))
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
        assert (st.cpu().numpy() == 0).all()
        for a, o, n in zip(fresh, out, lens.cpu().tolist()):
            assert o[:n].cpu().numpy().tobytes() == pillow(a, 85, "4:2:0", True), (rep, a.shape)


def test_overflow_reports_the_length_and_writes_nothing_past_the_cap(ctx):  # noqa: F811
    dev = f"cuda:{ctx.device}"
    rng = np.random.RandomState(5)
    pics = [rng.randint(0, 256, (40, 56, 3)).astype(np.uint8), rng.randint(0, 256, (30, 20, 1)).astype(np.uint8)]
    want = [pillow(a, 90, "4:2:2", False) for a in pics]
    for cap in (20, 101, 400):
        bufs = [torch.full((cap + 64,), 0xA5, dtype=torch.uint8, device=dev) for _ in pics]
        out, lens, st = ctx.compress_async([torch.from_numpy(a).to(dev) for a in pics], 90, "4:2:2", False,
                                           out=[b[:cap] for b in bufs])
        torch.cuda.synchronize()
        assert st.cpu().tolist() == [cuda.ENCODE_OVERFLOW] * 2
        assert lens.cpu().tolist() == [len(w) for w in want]
        for b, w in zip(bufs, want):
            h = b.cpu().numpy().tobytes()
            assert h[:cap] == w[:cap] and h[cap:] == b"\xa5" * 64, cap


def test_bad_arguments_enqueue_nothing(ctx):  # noqa: F811
    dev = f"cuda:{ctx.device}"
    lib = ctx.lib
    pic = torch.zeros((16, 16, 3), dtype=torch.uint8, device=dev)
    ws = torch.empty(1 << 20, dtype=torch.uint8, device=dev)
    out = torch.empty(1 << 16, dtype=torch.uint8, device=dev)
    ls = torch.empty(1, dtype=torch.int64, device=dev)
    sts = torch.empty(1, dtype=torch.int32, device=dev)

    def call(pin, jp, cap=out.numel(), wsb=ws.numel(), wsp=ws.data_ptr()):
        return lib.jpegqs_cuda_compress_async(ctx.h, 1, C.byref(pin), C.byref(jp), (C.c_void_p * 1)(out.data_ptr()),
                                              (C.c_size_t * 1)(cap), C.c_void_p(ls.data_ptr()), C.c_void_p(sts.data_ptr()),
                                              C.c_void_p(wsp), wsb, None)
    good_pin, good = cuda._PixelsIn(pic.data_ptr(), 16, 16, 3, 48), cuda._JpegParams(75, 2, 0)
    assert call(good_pin, good) == 0 and ctx.last_launches > 0
    torch.cuda.synchronize()
    bad = [(good_pin, cuda._JpegParams(0, 2, 0)), (good_pin, cuda._JpegParams(101, 2, 0)),
           (good_pin, cuda._JpegParams(75, 3, 0)), (cuda._PixelsIn(pic.data_ptr(), 16, 16, 2, 48), good),
           (cuda._PixelsIn(pic.data_ptr(), 16, 16, 4, 64), good), (cuda._PixelsIn(pic.data_ptr(), 0, 16, 3, 48), good),
           (cuda._PixelsIn(pic.data_ptr(), 65536, 16, 3, 3 * 65536), good), (cuda._PixelsIn(None, 16, 16, 3, 48), good)]
    for pin, jp in bad:
        assert call(pin, jp) == -2 and ctx.last_launches == 0
    assert call(good_pin, good, cap=19) == -2 and ctx.last_launches == 0
    assert call(good_pin, good, wsb=1000) == -2 and ctx.last_launches == 0
    assert call(good_pin, good, wsp=ws.data_ptr() + 16) == -2 and ctx.last_launches == 0
    with pytest.raises(ValueError, match="quality"):
        ctx.compress_async([pic], 0)
    with pytest.raises(ValueError, match="subsampling"):
        ctx.compress_async([pic], 75, "4:1:1")


# ---- JPEG files in, JPEG files out ----
PY_NAMES = ["base420", "base444", "prog420", "gray", "opt422", "rst", "tinyprog", "damaged", "garbled", "stop",
            "coarse420"]
SETTINGS = [(85, "4:2:0", False), (95, "4:4:4", True), (50, "4:2:2", False)]


def _geometry(datas, d, kind):
    """per file (size, crop) for kind None, 'crop' (a centred 224 x 224 crop, smaller pictures whole, to
    224 x 224) or 'thumb' (longest side 256)"""
    sizes, crops = [], []
    for data in datas:
        w, h, _ = _shape(data)
        pw, ph = -(-w // d), -(-h // d)
        if kind == "crop":
            cw, ch = min(224, pw), min(224, ph)
            l, t = (pw - cw) // 2, (ph - ch) // 2
            crops.append((l, t, l + cw, t + ch)); sizes.append((224, 224))
        else:
            m = max(pw, ph)
            crops.append(None); sizes.append((max(1, pw * 256 // m), max(1, ph * 256 // m)))
    return sizes, crops


@pytest.mark.parametrize("opt", ["q3", "q6", "n0"])
@pytest.mark.parametrize("d", [1, 2])
@pytest.mark.parametrize("kind", [None, "crop", "thumb"])
def test_reencode_equals_pillow_save_of_decode_pixels(ctx, corpus, opt, d, kind):  # noqa: F811
    _, flags, niter = OPTS[opt]
    datas = [corpus[n] for n in PY_NAMES]
    kw = {}
    if kind:
        sizes, crops = _geometry(datas, d, kind)
        kw = dict(size=sizes, crop=crops, filter="bilinear" if kind == "crop" else "bicubic")
    q, s, o = SETTINGS[(d + len(opt) + (len(kind) if kind else 0)) % 3]
    got = ctx.reencode(datas, flags | qs.JPEGQS_TRANSCODE, niter, q, s, o, scale_denom=d, **kw)
    pix = ctx.decode_pixels(datas, flags | qs.JPEGQS_TRANSCODE, niter, device="cpu", scale_denom=d, **kw)
    for n, g, p in zip(PY_NAMES, got, pix):
        assert g[0] == pillow(p[0].numpy(), q, s, o), (n, opt, d, kind)
        assert g[1:] == p[1:], n
    by = dict(zip(PY_NAMES, got))
    assert by["prog420"][2] == 1 and by["damaged"][2] == 1 and by["garbled"][2] == 1 and by["base420"][2] == 0
    assert Image.open(io.BytesIO(by["gray"][0])).mode == "L"


def test_reencode_8k(ctx, corpus):  # noqa: F811
    _, flags, niter = OPTS["q3"]
    datas = [corpus["8k"], corpus["base420"]]
    got = ctx.reencode(datas, flags | qs.JPEGQS_TRANSCODE, niter, 95, "4:2:0")
    pix = ctx.decode_pixels(datas, flags | qs.JPEGQS_TRANSCODE, niter, device="cpu")
    for g, p in zip(got, pix):
        assert g[0] == pillow(p[0].numpy(), 95, "4:2:0", False)


@pytest.mark.parametrize("budget", [1, 300000])
def test_splits_and_order_change_nothing(ctx, corpus, budget):  # noqa: F811
    _, flags, niter = OPTS["q6"]
    names = PY_NAMES
    datas = [corpus[n] for n in names]
    sizes, crops = _geometry(datas, 2, "thumb")
    whole = ctx.reencode(datas, flags, niter, 80, "4:2:0", True, scale_denom=2, size=sizes, crop=crops)
    split = ctx.reencode(datas, flags, niter, 80, "4:2:0", True, scale_denom=2, size=sizes, crop=crops, max_device_bytes=budget)
    assert split == whole
    perm = np.random.RandomState(budget).permutation(len(names))
    shuffled = ctx.reencode([datas[i] for i in perm], flags, niter, 80, "4:2:0", True, scale_denom=2,
                            size=[sizes[i] for i in perm], crop=[crops[i] for i in perm])
    assert [whole[i] for i in perm] == shuffled


def test_failures_stay_alone(ctx, corpus):  # noqa: F811
    """the C call: a CMYK file (the render takes 1 or 3 components), a file the reader rejects and a crop
    outside its picture fail; the files beside them are what reencode gives for them alone"""
    _, flags, niter = OPTS["q3"]
    names = ["base420", "cmyk", "junk", "gray", "badcrop", "base444"]
    datas = [corpus.get(n, b"\xff\xd8\xff\xd9" if n == "junk" else corpus["opt422"]) for n in names]
    boxes = []
    for n, data in zip(names, datas):
        w, h, _ = _shape(data) if n != "junk" else (8, 8, 3)
        boxes.append(cuda._ResizeBox(0, 0, w + 1, h, 50, 40) if n == "badcrop" else cuda._ResizeBox(0, 0, w, h, 50, 40))
    n = len(datas)
    rc, res = (C.c_int * n)(), (cuda._PixelsResult * n)()
    outs, olen = (C.c_void_p * n)(), (C.c_size_t * n)()
    jp = cuda._JpegParams(70, 1, 0)
    ret = ctx.lib.jpegqs_cuda_pixels_batch_jpeg(ctx.h, n, (C.c_char_p * n)(*datas), (C.c_size_t * n)(*[len(x) for x in datas]),
                                                flags, niter, 1, 2, (cuda._ResizeBox * n)(*boxes), C.byref(jp), 0, rc, res,
                                                outs, olen)
    assert ret == 0
    assert [rc[i] for i in range(n)] == [0, -3, -2, 0, -2, 0]
    for i, name in enumerate(names):
        if rc[i]:
            assert not outs[i]
            continue
        alone = ctx.reencode([datas[i]], flags, niter, 70, "4:2:2", size=(50, 40), filter="bilinear")[0][0]
        assert C.string_at(outs[i], olen[i]) == alone, name
        ctx.lib.jpegqs_cuda_transcode_free(outs[i])


def test_python_checks_before_running(ctx, corpus):  # noqa: F811
    datas = [corpus["base420"], corpus["gray"]]
    for kw, what in ((dict(quality=0), "quality"), (dict(quality=101), "quality"), (dict(subsampling=3), "subsampling"),
                     (dict(size=(0, 5)), "file 0"), (dict(crop=[(0, 0, 9999, 10), None]), "file 0"),
                     (dict(filter="nearest"), "filter")):
        with pytest.raises(ValueError, match=what):
            ctx.reencode(datas, 0, 1, **kw)
    got = qs.reencode(datas, 0, 1)
    assert [g[0][:2] for g in got] == [b"\xff\xd8"] * 2
