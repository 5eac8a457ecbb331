"""Progressive JPEG files written on the GPU.  compress_async(progressive=True) gives, for every device
picture, compress_model's progressive bytes, which are Pillow's Image.save(..., progressive=True): for
mixed batches of strided crops, every sampling, grey pictures and more than one launch group, for an
8K picture at quality 95 and a flat 8K picture whose AC scans are one long EOB-run segment, and when
replayed from a CUDA graph after the inputs are overwritten; also the CPU tests' targeted content and a
4K tiling of a block whose refinement scans carry correction bits only.  A capacity at the bound holds worst-case
content; below the file's length the call reports OVERFLOW and writes nothing past the capacity.
Sequential files from the same pictures are unchanged.  reencode(progressive=True) gives Pillow's
progressive save of the picture decode_pixels gives, at -q 3, -q 6 and -n 0, at d = 1 and 2, whole, as
224 crops and as 256-pixel thumbnails, with orientation, mode "L" and forced sub-batch splits."""
import io

import numpy as np
import pytest

from test_gpu_pixels_batch import OPTS, corpus, ctx  # noqa: F401  (module fixtures)
from test_gpu_compress import PY_NAMES, _geometry, _pictures

import jpegqs_b200 as qs
from jpegqs_b200 import cuda

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
Image = pytest.importorskip("PIL.Image")
ImageFile = pytest.importorskip("PIL.ImageFile")
ImageFile.MAXBLOCK = 1 << 28

SUBS = ("4:4:4", "4:2:2", "4:2:0")


def pillow(a, quality, subsampling, optimize=False, progressive=True):
    b = io.BytesIO()
    a = np.asarray(a)
    Image.fromarray(a if a.shape[2] == 3 else a[:, :, 0]).save(b, "JPEG", quality=quality, subsampling=subsampling,
                                                               optimize=optimize, progressive=progressive)
    return b.getvalue()


@pytest.mark.parametrize("sub", SUBS)
@pytest.mark.parametrize("quality,optimize", [(75, False), (95, True), (10, False)])
def test_batch_equals_model_and_pillow(ctx, sub, quality, optimize):  # noqa: F811
    dev = f"cuda:{ctx.device}"
    hosts, views, keep = [], [], []
    for seed in range(3):                            # 24 pictures: two launch groups
        h, v, k = _pictures(quality + seed, dev)
        hosts += h; views += v; keep += k
    out, lens, st = ctx.compress_async(views, quality, sub, optimize, progressive=True)
    torch.cuda.synchronize()
    st, lens = st.cpu().numpy(), lens.cpu().numpy()
    assert (st == 0).all()
    for a, o, n in zip(hosts, out, lens):
        got = o[:int(n)].cpu().numpy().tobytes()
        assert got == cuda.compress_model(a, quality, sub, optimize, progressive=True) == pillow(a, quality, sub), a.shape


def test_8k_at_q95_and_flat(ctx):  # noqa: F811
    rng = np.random.RandomState(8)
    yy, xx = np.indices((4320, 7680))
    a = np.stack([(xx // 3 + yy // 5) % 256, (xx * yy // 97) % 256, rng.randint(0, 256, (4320, 7680))], 2).astype(np.uint8)
    flat = np.full((4320, 7680, 3), (90, 140, 200), np.uint8)
    small = rng.randint(0, 256, (61, 97, 1)).astype(np.uint8)
    pics = (a, flat, small)
    t = [torch.from_numpy(x).to(f"cuda:{ctx.device}") for x in pics]
    out, lens, st = ctx.compress_async(t, 95, "4:2:0", False, progressive=True)
    torch.cuda.synchronize()
    assert st.cpu().tolist() == [0, 0, 0]
    for x, o, n in zip(pics, out, lens.cpu().tolist()):
        assert o[:n].cpu().numpy().tobytes() == pillow(x, 95, "4:2:0")


def test_graph_replay_reads_current_inputs(ctx):  # noqa: F811
    dev = f"cuda:{ctx.device}"
    hosts, views, _keep = _pictures(3, dev)
    s = torch.cuda.Stream(dev)
    with torch.cuda.stream(s):
        ctx.compress_async(views, 85, "4:2:0", True, stream=s, progressive=True)
    s.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        out, lens, st = ctx.compress_async(views, 85, "4:2:0", True, stream=s, progressive=True)
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
            assert o[:n].cpu().numpy().tobytes() == pillow(a, 85, "4:2:0"), (rep, a.shape)


def test_bound_holds_worst_case_and_overflow_writes_nothing_past_the_cap(ctx):  # noqa: F811
    dev = f"cuda:{ctx.device}"
    rng = np.random.RandomState(5)
    pics = [rng.randint(0, 256, (200, 264, 3)).astype(np.uint8), rng.randint(0, 256, (130, 90, 1)).astype(np.uint8)]
    want = [pillow(a, 100, "4:4:4") for a in pics]
    bound = [cuda.compress_bound(a.shape, 100, "4:4:4", progressive=True) for a in pics]
    assert all(b > len(w) for b, w in zip(bound, want))
    for caps in (bound, [20, 20], [101, 400], [len(w) - 1 for w in want], [len(w) - 3 for w in want]):
        bufs = [torch.full((cap + 64,), 0xA5, dtype=torch.uint8, device=dev) for cap in caps]
        out, lens, st = ctx.compress_async([torch.from_numpy(a).to(dev) for a in pics], 100, "4:4:4", False,
                                           out=[b[:cap] for b, cap in zip(bufs, caps)], progressive=True)
        torch.cuda.synchronize()
        assert lens.cpu().tolist() == [len(w) for w in want]
        fits = caps is bound
        assert st.cpu().tolist() == [0 if fits else cuda.ENCODE_OVERFLOW] * 2
        for b, w, cap in zip(bufs, want, caps):
            h = b.cpu().numpy().tobytes()
            if fits:
                assert h[:len(w)] == w
            else:                                    # all but the EOI, which is written only when it fits
                k = min(cap, len(w) - 2)
                assert h[:k] == w[:k] and h[k:cap] == b"\xa5" * (cap - k), cap
            assert h[cap:] == b"\xa5" * 64, cap


def test_sequential_files_unchanged(ctx):  # noqa: F811
    dev = f"cuda:{ctx.device}"
    hosts, views, _keep = _pictures(11, dev)
    for prog in (False, True, False):
        out, lens, st = ctx.compress_async(views, 80, "4:2:2", True, progressive=prog)
        torch.cuda.synchronize()
        assert (st.cpu().numpy() == 0).all()
        for a, o, n in zip(hosts, out, lens.cpu().tolist()):
            assert o[:n].cpu().numpy().tobytes() == pillow(a, 80, "4:2:2", True, prog), (prog, a.shape)
    with pytest.raises(ValueError, match="progressive"):
        ctx.compress_async(views, 80, progressive=1)


@pytest.mark.parametrize("opt", ["q3", "q6", "n0"])
@pytest.mark.parametrize("d", [1, 2])
@pytest.mark.parametrize("kind", [None, "crop", "thumb"])
def test_reencode_equals_pillow_progressive_save(ctx, corpus, opt, d, kind):  # noqa: F811
    _, flags, niter = OPTS[opt]
    datas = [corpus[n] for n in PY_NAMES]
    kw = {}
    if kind:
        sizes, crops = _geometry(datas, d, kind)
        kw = dict(size=sizes, crop=crops, filter="bilinear" if kind == "crop" else "bicubic")
    q, s = ((85, "4:2:0"), (95, "4:4:4"), (50, "4:2:2"))[(d + len(opt) + (len(kind) if kind else 0)) % 3]
    got = ctx.reencode(datas, flags | qs.JPEGQS_TRANSCODE, niter, q, s, scale_denom=d, progressive=True, **kw)
    pix = ctx.decode_pixels(datas, flags | qs.JPEGQS_TRANSCODE, niter, device="cpu", scale_denom=d, **kw)
    for n, g, p in zip(PY_NAMES, got, pix):
        assert g[0] == pillow(p[0].numpy(), q, s), (n, opt, d, kind)
        assert g[1:] == p[1:], n
    by = dict(zip(PY_NAMES, got))
    assert by["prog420"][2] == 1 and by["base420"][2] == 0
    assert Image.open(io.BytesIO(by["gray"][0])).mode == "L"


@pytest.mark.parametrize("orientation,mode", [("exif", None), (None, "L"), ("exif", "L")])
def test_reencode_orientation_and_mode(ctx, corpus, orientation, mode):  # noqa: F811
    _, flags, niter = OPTS["q3"]
    datas = [corpus[n] for n in PY_NAMES]
    sizes, crops = _geometry(datas, 1, "thumb")
    kw = dict(size=sizes, crop=crops, orientation=orientation, mode=mode)
    got = ctx.reencode(datas, flags, niter, 90, "4:2:0", True, progressive=True, **kw)
    pix = ctx.decode_pixels(datas, flags, niter, device="cpu", **kw)
    for n, g, p in zip(PY_NAMES, got, pix):
        assert g[0] == pillow(p[0].numpy(), 90, "4:2:0"), (n, orientation, mode)


@pytest.mark.parametrize("budget", [1, 300000])
def test_splits_change_nothing(ctx, corpus, budget):  # noqa: F811
    _, flags, niter = OPTS["q6"]
    datas = [corpus[n] for n in PY_NAMES]
    sizes, crops = _geometry(datas, 2, "thumb")
    whole = ctx.reencode(datas, flags, niter, 80, "4:2:0", scale_denom=2, size=sizes, crop=crops, progressive=True)
    split = ctx.reencode(datas, flags, niter, 80, "4:2:0", scale_denom=2, size=sizes, crop=crops, progressive=True,
                         max_device_bytes=budget)
    assert split == whole
    pix = ctx.decode_pixels(datas, flags, niter, device="cpu", scale_denom=2, size=sizes, crop=crops)
    assert [w[0] for w in whole] == [pillow(p[0].numpy(), 80, "4:2:0") for p in pix]


def test_targeted_content_equals_model(ctx):  # noqa: F811
    """test_compress_progressive_cpu's targeted pictures (runs past 0x7FFF blocks, correction-bit runs cut
    at 937 bits, zero gaps, negative DCs, odd block counts), and the correction-only tile over 4K, where
    one refinement segment spans thousands of tiles"""
    from test_compress_progressive_cpu import TARGETED, _only_corrections_block
    pics = [(a, q, s) for a, q, s, _ in TARGETED]
    pics.append((np.tile(_only_corrections_block(), (270, 480, 3)), 100, "4:4:4"))
    for a, q, s in pics:
        out, lens, st = ctx.compress_async([torch.from_numpy(a).to(f"cuda:{ctx.device}")], q, s, progressive=True)
        torch.cuda.synchronize()
        assert st.cpu().tolist() == [0]
        got = out[0][:int(lens[0])].cpu().numpy().tobytes()
        assert got == cuda.compress_model(a, q, s, progressive=True) == pillow(a, q, s), (a.shape, q, s)
