"""Every sampling geometry of hard_content.FACTORS through the GPU entry points, byte for byte.

The geometries are the ones libjpeg codes beyond grey / 4:4:4 / 4:2:2 / 4:2:0 / 4:4:0 / 4:1:1:
factors of 3 (box up-sampling by 3, the clipped last cell of the generic JOINT_YUV down-sample),
4 on either axis (MCU rows of 4 block rows, 10 blocks per MCU), 3x3 and 4x4 luma (more than 10
blocks per MCU), a 16x8 MCU whose ratios are all 1, chroma sampled above luma, Cb / Cr of
different factors, and grey files whose SOF gives factors other than 1x1.  Against what each is
checked:

  * smoothing (do_quantsmooth, run_async, the wave-scale tile scheduler): ol.run_oracle, with the
    return value and whether the chroma was up-sampled;
  * sharded smoothing (run_host_multi, the pass-level slabs) on one device: the one-rank result and
    the oracle;
  * render_async at d = 1, 2, 4, 8, plain and after run_async, both layouts: libjpeg's decode /
    scaled decode of the same coefficients and render_model;
  * decode_async / decode_scans_async: jpeg_read_coefficients;
  * pixels_batch / _scaled: the tool's --ppm body, and libjpeg's decode at every scale of the file
    the tool writes; transcode_batch: the bytes the tool writes with the host codec;
  * non-integral ratios: render_async refuses them before anything is enqueued."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import decode_files as df
import hard_content as hc
import libjpeg_pixels as lp
import libjpeg_scaled as ls
import oracle_lib as ol
import scan_files as sf
import jpegqs_b200 as qs
from jpegqs_b200 import cuda
from jpegqs_b200 import multigpu as mg
from jpegqs_b200.cuda import QsContext, _image_array
from render_images import GEOMETRIES as RENDER_GEOMETRIES, make
from test_cli import EXE
from test_gpu_async import _check, _oracle, run_async
from test_gpu_edge import _run_slabs_one_gpu
from test_gpu_pixels_batch import _as_hwc, _c_batch, _ppm
from test_gpu_pixels_scaled import _c_scaled, _hwc
from test_gpu_render_async import smooth
from test_gpu_slab_engine import _devices
from test_gpu_transcode_batch import _c_batch as _tc_batch

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(lp.JPEG_SO is None, reason="no libjpeg inside Pillow")]

torch = pytest.importorskip("torch")

GEOMETRIES = hc.GEOMETRIES
FLAG_SETS = (0, 1, 3, 7, 15, 16, 33)
# ragged (24k +- 1, 32k +- 1), a multiple of every MCU but 3x3's, below 8, and 40 x 37: a factor of 3
# leaves the generic down-sample a last cell of one luma column / row there
SIZES = ((23, 65), (97, 31), (48, 48), (5, 3), (40, 37))
# grey, and geometries whose chroma is not 1x1: JOINT_YUV and UPSAMPLE_UV never apply
NO_UPSAMPLE = tuple(g for g in GEOMETRIES if len(hc.factors(g)) == 1 or any(f != (1, 1) for f in hc.factors(g)[1:]))


@pytest.fixture(scope="module")
def ctx():
    c = QsContext(0)
    yield c
    c.close()


def _images(ss):
    return [make(w, h, ss, ("k50", "k90", "rand", "k10", "diag")[k], content, seed=7 * k + len(ss))
            for content in ("synth", "saturated") for k, (w, h) in enumerate(SIZES)]


# ---- 1. smoothing ---------------------------------------------------------------------------------

@pytest.mark.parametrize("ss", GEOMETRIES)
def test_smoothing_is_the_oracles(ctx, ss):
    ims = _images(ss)
    for flags in FLAG_SETS:
        niter = 1 + flags % 3
        wants = [_oracle(im, flags, niter) for im in ims]
        for im, (oret, oout, oups) in zip(ims, wants):
            ret, out = ctx.do_quantsmooth(im, flags, niter)
            assert ret == oret, (ss, flags, im.width, im.height)
            assert ol.images_equal(out, oout), (ss, flags, im.width, im.height, ol.diff_count(out, oout))
            if ss in NO_UPSAMPLE or not flags & 4:
                assert not oups and [(c.h_samp, c.v_samp) for c in out.comps] == list(hc.factors(ss))
        for got, want in zip(run_async(torch, ctx, ims, flags, niter), wants):
            _check(got, want)
        if flags & 4 and ss not in NO_UPSAMPLE:
            assert any(w[2] for w in wants), (ss, flags)                          # UPSAMPLE_UV ran


@pytest.mark.parametrize("ss,flags,niter", [("31", 3, 2), ("410", 7, 1), ("13", 15, 2)])
def test_wave_scale(ctx, ss, flags, niter):
    """About 2400 x 1600: the persistent tile scheduler runs many tiles of these component shapes."""
    im = make(2401, 1599, ss, "k50", "saturated", seed=11)
    want = _oracle(im, flags, niter)
    _check(run_async(torch, ctx, [im], flags, niter)[0], want)
    ret, out = ctx.do_quantsmooth(im, flags, niter)
    assert ret == want[0] and ol.images_equal(out, want[1])


# ---- 2. sharded on one device ---------------------------------------------------------------------

SHARDED = ("13", "14", "24", "11_22_22")


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("ss", SHARDED)
def test_run_host_multi_is_shard_invariant(ctx, ss, world):
    os.environ["JPEGQS_MIN_BLOCKS_PER_GPU"] = "1"
    try:
        m = cuda.QsMulti(_devices(world))
    finally:
        del os.environ["JPEGQS_MIN_BLOCKS_PER_GPU"]
    try:
        for k, (w, h) in enumerate(((121, 223), (64, 193))):
            im = make(w, h, ss, ("k50", "k90")[k], ("synth", "saturated")[k], seed=k + 1)
            assert m.plan(im) == world, (ss, w, h)
            for flags in (3, 7):
                ret, out = m.do_quantsmooth(im, flags, 2)
                oret, want = ol.run_oracle(im, flags, 2)
                one = ctx.do_quantsmooth(im, flags, 2)
                assert ret == oret == one[0]
                assert ol.images_equal(out, want), (ss, w, h, flags, ol.diff_count(out, want))
                assert ol.images_equal(one[1], want)
    finally:
        m.close()


@pytest.mark.parametrize("nshards", [2, 3])
@pytest.mark.parametrize("ss", SHARDED)
def test_pass_level_slabs_are_shard_invariant(ctx, ss, nshards):
    im = make(121, 223, ss, "k50", "synth", seed=3)
    for flags in (0, 1):
        got = _run_slabs_one_gpu(ctx, im, flags, 2, nshards)
        one = _run_slabs_one_gpu(ctx, im, flags, 2, 1)
        _, want = ol.run_oracle(im, flags, 2)
        for g, o, c in zip(got, one, want.comps):
            assert np.array_equal(g, c.coef) and np.array_equal(o, c.coef), (flags, nshards)


@pytest.mark.parametrize("ss", SHARDED + ("31", "410"))
def test_pass_level_luma_chroma_handover(ctx, ss):
    """jpegqs_cuda_pass_downsample / _upsample at these factors (one slab, the whole image)."""
    dev = torch.device("cuda", 0)
    for flags, (w, h) in ((3, (121, 83)), (7, (96, 95))):
        im = make(w, h, ss, "k50", "saturated", seed=w)
        comps = [mg.SlabComp(torch.from_numpy(np.ascontiguousarray(c.coef)).to(dev),
                             torch.zeros((c.hblk * 8 + 2, mg.plane_stride(c.wblk)), dtype=torch.uint8, device=dev),
                             c.wblk, c.hblk, c.quant, k == 0, c.h_samp, c.v_samp, 0, c.hblk)
                 for k, c in enumerate(im.comps)]
        passes = mg.CudaPasses(ctx, torch.cuda.current_stream().cuda_stream)
        stop, ups = mg.run_slab(passes, comps, flags, 2, 0, 1, None, None, mg.SlabGeom(True, w, h))
        torch.cuda.synchronize()
        oret, want, oups = _oracle(im, flags, 2)
        assert stop == oret and bool(ups) == oups, (ss, flags)
        for k, (c, o) in enumerate(zip(comps, want.comps)):
            got = (c.coef_up if ups and k in (1, 2) else c.coef).cpu().numpy()
            assert got.shape == o.coef.shape and np.array_equal(got, o.coef), (ss, flags, k)


# ---- 3. render ------------------------------------------------------------------------------------

def _libjpeg(im, d):
    """libjpeg's RGB pixels of a coefficient set at scale 1/d (a grey set's grey channel repeated)"""
    px = lp.decode(im) if d == 1 else ls.decode(im, d)[0]
    return np.repeat(px, 3, axis=2) if px.shape[2] == 1 else px


@pytest.mark.parametrize("d", [1, 2, 4, 8])
@pytest.mark.parametrize("ss", RENDER_GEOMETRIES + ("440", "411"))
def test_render_is_libjpegs(ctx, ss, d):
    # scaled widths of 127, 128 and 129 (about the 128 x 64 tile), ragged sizes, chroma 1-3 samples wide
    ims = [make(w, 64 * d + 1, ss, "k90", "synth", seed=d + w) for w in (127 * d, 128 * d, 128 * d + 1)]
    assert [-(-im.width // d) for im in ims] == [127, 128, 129]
    ims += [make(203, 149, ss, "rand", "saturated", seed=2),
            make(13, 7, ss, "k50", "synth", seed=3), make(3, 5, ss, "k10", "saturated", seed=4)]
    for flags in (None, 3, 7):
        work, coefs, status, ups = smooth(torch, ctx, ims, flags)
        if flags is None:
            srcs = ims
        else:
            res = [_oracle(im, flags, 1) for im in ims]
            st = status.cpu().numpy()
            assert [int(v) for v in st[:, 0]] == [r[0] for r in res]
            assert [bool(v) for v in st[:, 1]] == [r[2] for r in res]
            srcs = [r[1] for r in res]
        hwc = ctx.render_async(work, coefs, status, ups, scale_denom=d)
        chw = ctx.render_async(work, coefs, status, ups, layout="chw", scale_denom=d)
        torch.cuda.synchronize()
        for n, src in enumerate(srcs):
            what = (ss, d, flags, src.width, src.height)
            got = hwc[n].cpu().numpy()
            assert np.array_equal(got, _libjpeg(src, d)), what
            assert np.array_equal(got, cuda.render_model(src, scale_denom=d)), what
            assert torch.equal(chw[n], hwc[n].permute(2, 0, 1)), what


def test_render_refuses_non_integral_ratios(ctx):
    """Y 3x1 over Cb 2x1: no libjpeg up-sampler takes a ratio of 3/2.  JPEGQS_ERR_UNSUPPORTED, and
    nothing is written."""
    lib = ctx.lib
    for f in (((3, 1), (2, 1), (1, 1)), ((1, 3), (1, 1), (1, 2)), ((2, 2), (3, 1), (1, 1))):
        im = hc.make_image(40, 37, f, hc.TABLES["k50"], "synth", seed=1)
        coefs = [torch.from_numpy(np.ascontiguousarray(c.coef)).cuda() for c in im.comps]
        out = torch.full((im.height * im.width * 3,), 0x5A, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        arr = _image_array([im], [[t.data_ptr() for t in coefs]], [])
        outs = (C.c_void_p * 1)(out.data_ptr())
        assert lib.jpegqs_cuda_render_async(ctx.h, 1, arr, None, 0, outs, None) == -3, f      # UNSUPPORTED
        for d in (2, 8):
            assert lib.jpegqs_cuda_render_scaled_async(ctx.h, 1, arr, None, 0, d, outs, None) == -3, (f, d)
        torch.cuda.synchronize()
        assert bool((out == 0x5A).all()), f
        with pytest.raises(cuda.QsError):
            cuda.render_model(im)


# ---- 4. entropy decoders --------------------------------------------------------------------------

def _dev(data):
    return torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()


def _same(coefs, ref):
    return len(coefs) == len(ref.comps) and all(np.array_equal(t.cpu().numpy(), c.coef) for t, c in zip(coefs, ref.comps))


def test_decode_async_mixed_batch(ctx):
    files = df.geometry_files() + df.flavours()[:24:3]
    parsed = [qs.parse_jpeg(d) for _, d in files]
    coefs, status = ctx.decode_async([p[0] for p in parsed], [p[1] for p in parsed], [_dev(d) for _, d in files])
    torch.cuda.synchronize()
    assert status.cpu().tolist() == [0] * len(files)
    for (name, data), c in zip(files, coefs):
        assert _same(c, df.libjpeg_coefficients(data)), name


def test_decode_scans_async_mixed_batch(ctx):
    files = sf.geometry_progressive() + [(n, d) for n, d in sf.scripted()][:6]
    parsed = [qs.parse_jpeg_scans(d) for _, d in files]
    coefs, status = ctx.decode_scans_async([p[0] for p in parsed], [p[1] for p in parsed], [_dev(d) for _, d in files])
    torch.cuda.synchronize()
    assert status.cpu().tolist() == [0] * len(files)
    for (name, data), c in zip(files, coefs):
        assert _same(c, df.libjpeg_coefficients(data)), name


# ---- 5. end to end --------------------------------------------------------------------------------

OPTS = {"q3": (["-q", "3", "-n", "3"], qs.quality_to_flags(3), 3),
        "q6": (["-q", "6", "-n", "3"], qs.quality_to_flags(6), 3)}
HOST = dict(os.environ, JPEGQS_HOST_CODEC="1")


@pytest.fixture(scope="module")
def files():
    """name -> bytes: every render geometry with and without restart markers, and the two files of one
    scan per component (host route)."""
    return dict(df.geometry_files() + df.per_component_files())


@pytest.fixture(scope="module")
def tool(files, tmp_path_factory):
    """(name, opt) -> (the tool's --ppm body, the path of the file it writes, or None where it writes
    none: a 3x3 / 4x4 luma that stays sub-sampled has more than 10 blocks per MCU, which the encoder
    does not write in one interleaved scan)"""
    d = tmp_path_factory.mktemp("samplings")
    cache = {}

    def get(name, opt):
        if (name, opt) not in cache:
            src = d / f"{name}.jpg"
            src.write_bytes(files[name])
            status, body = _ppm(src, OPTS[opt][0], d / f"{name}.{opt}.ppm")
            assert status == 0, (name, opt)
            dst = d / f"{name}.{opt}.jpg"
            r = subprocess.run([EXE, "-i", "0"] + OPTS[opt][0] + [str(src), str(dst)], capture_output=True, text=True,
                               env=HOST)
            if r.returncode and "more than 10 blocks per MCU" in r.stderr and name in ("writer_33", "writer_44"):
                dst = None
            else:
                assert r.returncode == 0, r.stderr
            cache[(name, opt)] = body, dst and str(dst)
        return cache[(name, opt)]
    return get


@pytest.fixture(scope="module")
def scaled(files, tool):
    """(name, opt, d) -> libjpeg's decode at 1/d of the file the tool writes; where it writes none,
    of the oracle's smoothing of the file's coefficients (written one scan per component)"""
    cache = {}

    def get(name, opt, d):
        if (name, opt, d) not in cache:
            path = tool(name, opt)[1]
            if path is None:
                _, flags, niter = OPTS[opt]
                cache[(name, opt, d)] = ls.decode(ol.run_oracle(qs.read_jpeg(files[name]), flags, niter)[1], d)[0]
            else:
                cache[(name, opt, d)] = ls.decode_file(path, d)[0]
        return cache[(name, opt, d)]
    return get


@pytest.mark.parametrize("opt", sorted(OPTS))
def test_pixels_equal_the_tool(ctx, files, tool, scaled, opt):
    names = sorted(files)
    datas = [files[n] for n in names]
    _, flags, niter = OPTS[opt]
    for layout, on_device in ((0, 1), (1, 0), (0, 0), (1, 1)):
        for n, (rc, pix, res) in zip(names, _c_batch(ctx, datas, flags, niter, layout, on_device)):
            assert rc == 0, n
            assert _as_hwc(pix, files[n], layout) == tool(n, opt)[0], (n, opt, layout, on_device)
            assert _as_hwc(pix, files[n], layout) == scaled(n, opt, 1).tobytes(), (n, opt, layout, on_device)
            assert res[1] == (n in ("writer_33", "writer_44")), (n, res)
        for d in (2, 4, 8):
            for n, (rc, pix, res) in zip(names, _c_scaled(ctx, datas, flags, niter, layout, d, on_device)):
                assert rc == 0, n
                assert np.array_equal(_hwc(pix, files[n], layout, d), scaled(n, opt, d)), (n, opt, layout, on_device, d)
    assert [n for n in names if tool(n, opt)[1] is None] == (["writer_33", "writer_44"] if opt == "q3" else [])


@pytest.mark.parametrize("opt", sorted(OPTS))
def test_transcode_batch_equals_the_tool(ctx, files, tool, opt):
    names = sorted(files)
    _, flags, niter = OPTS[opt]
    got = _tc_batch(ctx, [files[n] for n in names], flags | qs.JPEGQS_TRANSCODE, niter, False, 2)
    for n, (rc, data, *_rest) in zip(names, got):
        if n in ("writer_33", "writer_44"):
            assert rc == cuda.TRANSCODE_FALLBACK and "10 blocks" in _rest[-1], (n, rc)
            continue
        assert rc == cuda.TRANSCODE_OK, (n, _rest)
        assert data == open(tool(n, opt)[1], "rb").read(), (n, opt)
        # and libjpeg reads back the oracle's smoothing of the file's coefficients
        ret, want = ol.run_oracle(qs.read_jpeg(files[n]), flags, niter)
        back = df.libjpeg_coefficients(data)
        assert [(c.h_samp, c.v_samp) for c in back.comps] == [(c.h_samp, c.v_samp) for c in want.comps], n
        assert all(np.array_equal(a.coef, b.coef) for a, b in zip(back.comps, want.comps)), (n, opt)


def test_orientation_6_on_31(ctx, files):
    """The transposing store takes a 3x1 luma like any other: orientation 6 is Pillow's ROTATE_270
    (np.rot90 clockwise) of the unoriented pixels."""
    data = files["writer_31"]
    flags = qs.quality_to_flags(6)
    for d in (1, 2):
        plain = ctx.decode_pixels([data], flags, 3, scale_denom=d)[0][0].cpu().numpy()
        turned = ctx.decode_pixels([data], flags, 3, scale_denom=d, orientation=6)[0][0].cpu().numpy()
        assert np.array_equal(turned, np.rot90(plain, -1)), d
