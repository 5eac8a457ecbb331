"""The JPEG reading entry points on the host: parse_jpeg, read_jpeg, the decode workspace formula and
argument checks, and decode_model - decode_async's algorithm run on the CPU - against
libjpeg-turbo's jpeg_read_coefficients.  No GPU is used."""
import ctypes as C

import numpy as np
import pytest

import decode_files as df
import libjpeg_pixels as lp
import jpegqs_b200 as qs
from jpegqs_b200 import cuda

pytestmark = pytest.mark.skipif(lp.JPEG_SO is None, reason="no libjpeg inside Pillow")

KNOBS = [cuda.DECODE_SUB_MIN, cuda.DECODE_SUB_MIN + 1, 1000, cuda.DECODE_SUB_DEFAULT]
FLAVOURS = df.flavours()
HARD = df.hard_sets()
PROG = df.progressive()
# units the synchronisation may decode past a subsequence's end on CMYK / untransformed-RGB files at
# the default knob.  The files below hold about 30 blocks per subsequence: a decoder that
# synchronised on MCU starts would never meet the speculative decode and re-decode all of them.
OVERRUN_BOUND = 8


def _same(a, b):
    return len(a) == len(b.comps) and all(np.array_equal(np.asarray(x), y.coef) for x, y in zip(a, b.comps))


@pytest.mark.parametrize("name,data", FLAVOURS + PROG, ids=[n for n, _ in FLAVOURS + PROG])
def test_parse_and_read_match_libjpeg(name, data):
    ref = df.libjpeg_coefficients(data)
    im, scan = qs.parse_jpeg(data)
    assert (im.width, im.height, im.colorspace) == (ref.width, ref.height, ref.colorspace)
    for a, b in zip(im.comps, ref.comps):
        assert (a.h_samp, a.v_samp, a.wblk, a.hblk) == (b.h_samp, b.v_samp, b.wblk, b.hblk)
        assert np.array_equal(a.quant, b.quant)
        assert a.coef.strides == (0, 0, 0)                      # placeholders cost no memory
    assert (scan is None) == name.startswith("prog")
    got = qs.read_jpeg(data)
    assert _same([c.coef for c in got.comps], ref)


@pytest.mark.parametrize("name,data", df.per_component_files(), ids=[n for n, _ in df.per_component_files()])
def test_per_component_scans_take_the_host_route(name, data):
    """3x3 and 4x4 luma: more blocks per MCU than one interleaved scan holds, so libjpeg writes one scan
    per component; the transcode takes the host route and read_jpeg still reads libjpeg's coefficients"""
    ref = df.libjpeg_coefficients(data)
    assert [(c.h_samp, c.v_samp) for c in ref.comps][1:] == [(1, 1), (1, 1)] and ref.comps[0].h_samp >= 3
    assert qs.transcode_route(data) == ("host", "more than 10 blocks per MCU")
    im, scan = qs.parse_jpeg(data)
    assert scan is None
    assert [(a.h_samp, a.v_samp, a.wblk, a.hblk) for a in im.comps] == [(b.h_samp, b.v_samp, b.wblk, b.hblk) for b in ref.comps]
    assert _same([c.coef for c in qs.read_jpeg(data).comps], ref)


def test_parse_rejects():
    data = df.pillow_jpeg(64, 48, quality=75)
    sos = data.index(b"\xff\xda")
    with pytest.raises(cuda.QsError):
        qs.parse_jpeg(data[:sos - 20])                          # truncated inside a marker segment
    sof = data.index(b"\xff\xc0")
    for code in (b"\xc3", b"\xc9"):                             # lossless, arithmetic
        with pytest.raises(cuda.QsError):
            qs.parse_jpeg(data[:sof + 1] + code + data[sof + 2:])
    with pytest.raises(cuda.QsError):
        qs.parse_jpeg(b"not a jpeg")


@pytest.mark.parametrize("sub_bytes", KNOBS)
@pytest.mark.parametrize("name,data", FLAVOURS, ids=[n for n, _ in FLAVOURS])
def test_model_equals_libjpeg(name, data, sub_bytes):
    ref = df.libjpeg_coefficients(data)
    im, scan = qs.parse_jpeg(data)
    out, status, over = qs.decode_model(im, scan, data, sub_bytes)
    assert status == 0
    assert _same(out, ref)


@pytest.mark.parametrize("name,image,data", HARD, ids=[n for n, _, _ in HARD])
def test_model_decodes_hard_content_back(name, image, data):
    ref = df.libjpeg_coefficients(data)
    assert _same([c.coef for c in image.comps], ref)          # the writer kept the set
    im, scan = qs.parse_jpeg(data)
    for sub_bytes in (cuda.DECODE_SUB_MIN, cuda.DECODE_SUB_DEFAULT):
        out, status, _ = qs.decode_model(im, scan, data, sub_bytes)
        assert status == 0 and _same(out, ref), sub_bytes


def test_hard_content_reaches_the_extremes():
    vals = np.concatenate([np.asarray(c.coef).reshape(-1, 64) for _, im, _ in HARD for c in im.comps])
    assert np.abs(vals[:, 1:]).max() >= 256                     # 9-bit AC values (long value fields)
    assert (vals[:, 63] != 0).any()                             # EOB never sent after coefficient 63


ONE_PAIR = {"cmyk": dict(mode="CMYK", quality=30),
            "cmyk_rst": dict(mode="CMYK", quality=30, restart_marker_rows=4),
            "keep_rgb": dict(quality=30, keep_rgb=True, subsampling=0)}


@pytest.mark.parametrize("name", sorted(ONE_PAIR))
def test_one_table_pair_synchronises_on_blocks(name):
    data = df.pillow_jpeg(320, 240, **ONE_PAIR[name])
    im, scan = qs.parse_jpeg(data)
    out, status, over = qs.decode_model(im, scan, data, cuda.DECODE_SUB_DEFAULT)
    assert status == 0 and _same(out, df.libjpeg_coefficients(data))
    units_per_sub = sum(c.wblk * c.hblk for c in im.comps) / len(over)
    assert units_per_sub >= 3 * OVERRUN_BOUND
    assert int(over.max()) <= OVERRUN_BOUND


def _expected_ws(im, scan, n):
    a = lambda x: (x + 255) // 256 * 256
    L = n - scan.entropy_offset
    if len(im.comps) == 1:
        nmcu = im.comps[0].wblk * im.comps[0].hblk
    else:
        mh = max(c.h_samp for c in im.comps); mv = max(c.v_samp for c in im.comps)
        nmcu = -(-im.width // (8 * mh)) * -(-im.height // (8 * mv))
    I = -(-nmcu // scan.restart_interval) if scan.restart_interval else 1
    return 16384 + a(L + 8) + a(24 * -(-L // 4096)) + 2 * a(4 * I) + a(96 * (L // 32 + I))


def test_workspace_formula():
    items = [(qs.parse_jpeg(d), len(d)) for _, d in FLAVOURS]
    total = 0
    for (im, scan), n in items:
        got = qs.decode_workspace_bytes([im], [scan], [n])
        assert got == _expected_ws(im, scan, n)
        total += got
    assert qs.decode_workspace_bytes([i for (i, _), _ in items], [s for (_, s), _ in items], [n for _, n in items]) == total


def test_argument_checks():
    data = dict(FLAVOURS)["420_q75"]
    im, scan = qs.parse_jpeg(data)
    def rejected(im2, sc2, n=len(data)):
        with pytest.raises(cuda.QsError):
            qs.decode_workspace_bytes([im2], [sc2], [n])
    rejected(im, scan, scan.entropy_offset)                    # no entropy-coded data
    sc = cuda._Scan.from_buffer_copy(scan); sc.ac_tbl[1] = 3   # absent table
    rejected(im, sc)
    sc = cuda._Scan.from_buffer_copy(scan); sc.comp[1] = 0     # not a permutation
    rejected(im, sc)
    sc = cuda._Scan.from_buffer_copy(scan); sc.ncomp = 2
    rejected(im, sc)
    bad = im.clone(); bad.comps[1].coef = cuda._placeholder((bad.comps[1].hblk + 1, bad.comps[1].wblk, 64))
    rejected(bad, scan)                                         # geometry that disagrees
    # the model takes the same checks, and a misaligned / NULL array
    lib = cuda.load()
    ci = cuda._Image()
    arrs = [np.zeros((c.hblk, c.wblk, 64), np.int16) for c in im.comps]
    cuda._fill_image(ci, im, [a.ctypes.data + 2 for a in arrs], [])
    st = C.c_int32(0)
    assert lib.jpegqs_cuda_decode_model(C.byref(ci), C.byref(scan), data, len(data), 512, C.byref(st), None, 0, None) == -2
    cuda._fill_image(ci, im, [a.ctypes.data for a in arrs], [])
    ci.comp[0].rows = 16
    assert lib.jpegqs_cuda_decode_model(C.byref(ci), C.byref(scan), data, len(data), 512, C.byref(st), None, 0, None) == -2
    with pytest.raises(cuda.QsError):
        qs.decode_model(im, scan, data, cuda.DECODE_SUB_MIN - 1)


GUARD = 4096


def _mutants():
    rng = np.random.default_rng(2024)
    bases = [dict(FLAVOURS)[n] for n in ("420_q75", "rst_blocks7", "cmyk", "gray_q100", "writer_411")]
    out = []
    for k in range(300):
        data = bytearray(bases[k % len(bases)])
        im, scan = qs.parse_jpeg(bytes(data))
        off = scan.entropy_offset
        kind = k % 3
        if kind == 0:                                           # truncated
            data = data[:int(rng.integers(off + 1, len(data)))]
        elif kind == 1:                                         # bytes flipped in the segment
            for _ in range(int(rng.integers(1, 4))):
                p = int(rng.integers(off, len(data) - 2))
                data[p] ^= int(rng.integers(1, 256))
        else:                                                   # an RST removed (or a byte, without restarts)
            seg = bytes(data[off:])
            rs = [i for i in range(len(seg) - 1) if seg[i] == 0xFF and 0xD0 <= seg[i + 1] <= 0xD7]
            if rs:
                p = off + rs[int(rng.integers(0, len(rs)))]
                del data[p:p + 2]
            else:
                del data[int(rng.integers(off, len(data) - 2))]
        out.append((im, scan, bytes(data)))
    return out


def test_mutated_files_flag_or_match_the_reader():
    flagged = 0
    for im, scan, data in _mutants():
        bufs = [np.full(c.hblk * c.wblk * 64 + 2 * GUARD, 0x5A5A, dtype=np.int16) for c in im.comps]
        views = [b[GUARD:GUARD + c.hblk * c.wblk * 64].reshape(c.hblk, c.wblk, 64) for b, c in zip(bufs, im.comps)]
        if len(data) <= scan.entropy_offset:
            continue
        _, status, _ = qs.decode_model(im, scan, data, 48, out=views)
        for b in bufs:
            assert (b[:GUARD] == 0x5A5A).all() and (b[-GUARD:] == 0x5A5A).all()
        if status == 0:
            assert _same(views, qs.read_jpeg(data))
        else:
            flagged += 1
    assert flagged > 100
