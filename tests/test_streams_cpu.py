"""The JPEG readers on legal streams libjpeg-turbo's writer never emits (stream_files.py): fill bytes
before markers, 0-bit padding, marker segments between scans, merged and moved DHT segments, restart
intervals that change or exceed the image, unusual component identifiers and table slots, and
Huffman codes up to 16 bits.  The reference is libjpeg-turbo's jpeg_read_coefficients: read_jpeg
(one thread and threaded), decode_model / decode_scans_model and the jpegqs tool must give its
coefficients.  No GPU is used."""
import os
import re
import subprocess

import numpy as np
import pytest

import decode_files as df
import libjpeg_pixels as lp
import stream_files as sf
import jpegqs_b200 as qs
from jpegqs_b200 import cuda

pytestmark = pytest.mark.skipif(lp.JPEG_SO is None, reason="no libjpeg inside Pillow")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "jpeg-quantsmooth_b200", "csrc", "jpegqs")
REFCLI = os.path.join(ROOT, "oracle", "_ref", "refcli_cpu")
KNOBS = [cuda.DECODE_SUB_MIN, cuda.DECODE_SUB_MIN + 1, cuda.DECODE_SUB_DEFAULT]
CORPUS = sf.corpus()
WARNED = sf.warned()
# the features the device decoders may flag (a nonzero status sends the file to the host reader):
# 0-bit padding (the device checks that padding is 1-bits), and fill bytes before RSTn (the byte
# passes end the segment at an FF that is followed by neither 00 nor RSTn).  Fill bytes before the
# marker that ends a scan must decode with status 0.
DEVICE_MAY_FLAG = ("fill_rst", "zero_pad")
REF_BUILT = os.path.exists(REFCLI)


class TableSlotsDiffer(AssertionError):
    """jq_write's output differs from libjpeg's only in the Huffman table slots of an RGB file
    (DESIGN.md section 3.7, known deviation)"""


def _rgb(f):
    return qs.parse_jpeg(f.data)[0].colorspace == 2


def _tool_params():
    """the corpus, the RGB files a strict expected failure where the reference CLI is built"""
    mark = pytest.mark.xfail(strict=True, raises=TableSlotsDiffer,
                             reason="RGB: jq_write gives later components Huffman tables 1, libjpeg tables 0")
    return [pytest.param(f, id=f.name, marks=[mark] if REF_BUILT and _rgb(f) else []) for f in CORPUS]


def _only_table_slots_differ(ours: bytes, ref: bytes) -> bool:
    """the same bytes up to the first DHT, the same slot-0 tables, libjpeg's SOS selectors all 0 and
    ours 0 then 0x11 (the coefficients are compared separately)"""
    po, pr = sf.pieces(ours), sf.pieces(ref)
    first = lambda ps: next(i for i, (c, _) in enumerate(ps) if c == 0xC4)
    if sf.join(po[:first(po)]) != sf.join(pr[:first(pr)]):
        return False
    dho, dhr = [b for c, b in po if c == 0xC4], [b for c, b in pr if c == 0xC4]
    if any(b[4] & 15 for b in dhr) or [b for b in dho if not b[4] & 15] != dhr:
        return False
    so, sr = next(b for c, b in po if c == 0xDA), next(b for c, b in pr if c == 0xDA)
    n = so[4]
    return (so[:6] == sr[:6] and so[5:5 + 2 * n:2] == sr[5:5 + 2 * n:2] and set(sr[6:6 + 2 * n:2]) == {0}
            and list(so[6:6 + 2 * n:2]) == [0] + [0x11] * (n - 1) and so[5 + 2 * n:] == sr[5 + 2 * n:])


def _same(arrays, ref):
    return len(arrays) == len(ref.comps) and all(np.array_equal(np.asarray(a), c.coef) for a, c in zip(arrays, ref.comps))


def _ids(files):
    return [f.name for f in files]


def test_corpus_reaches_what_it_claims():
    names = {f.name for f in CORPUS}
    assert len(names) == len(CORPUS)
    for f in CORPUS:
        assert f.cls == "legal" and not sf.libjpeg_warns(f.data), f.name
    assert WARNED and all(sf.libjpeg_warns(f.data) for f in WARNED)
    assert any(n.startswith("zero_pad_rst_") for n in names) and any(n.startswith("zero_pad_eoi_") for n in names)
    for f in CORPUS:                                        # the fill bytes are where the name says
        if f.feature in ("fill", "fill_rst"):
            where = f.name.split("_")[1]
            code = {"rst": rb"[\xd0-\xd7]", "every": rb"[\xd0-\xd7]", "eoi": rb"\xd9", "sos": rb"\xda", "dht": rb"\xc4"}[where]
            assert re.search(rb"[^\xff]\xff{%d}" % (int(f.name[4]) + 1) + code, f.data), f.name
    # the long-code tables use every length 2..16, and the DC table's 16-bit codes carry category 11
    for f in CORPUS:
        if f.feature == "long_codes":
            dht = [b for c, b in sf.pieces(f.data) if c == 0xC4]
            assert any(list(b[5:21]) == sf.AC_BITS[1:] for b in dht) and any(list(b[5:21]) == sf.DC_BITS[1:] for b in dht)
    assert [sf.dc_categories(sf._dc11_file(ss)) for ss in ("gray", "444")] == [11, 11]
    dc = sf.long_tables(1)[0]
    assert dc[1][-1] == 11 and dc[0][16] == 2                # category 11 has a 16-bit code


@pytest.mark.parametrize("threaded", [False, True], ids=["one_thread", "threaded"])
@pytest.mark.parametrize("f", CORPUS, ids=_ids(CORPUS))
def test_read_jpeg_equals_libjpeg(f, threaded, monkeypatch, capfd):
    """read_jpeg on one thread, and on the threaded paths forced onto these small files (restart
    intervals side by side, speculative chunks, progressive scans side by side).  Fill bytes before a
    restart marker or before the marker that ends a sequential scan must not make the threaded
    reader give up: it decodes them itself."""
    ref = df.libjpeg_coefficients(f.data)
    if threaded:
        monkeypatch.setenv("JPEGQS_PAR_MIN_BYTES", "200")
        monkeypatch.setenv("JPEGQS_CODEC_THREADS", "6")
        monkeypatch.setenv("JPEGQS_CODEC_TRACE", "1")
    else:
        monkeypatch.setenv("JPEGQS_SERIAL_DECODE", "1")
    got = qs.read_jpeg(f.data)
    assert _same([c.coef for c in got.comps], ref)
    trace = capfd.readouterr().err
    if threaded and f.feature in ("fill", "fill_rst") and "prog" not in f.name and "succ" not in f.name:
        assert "abandoned" not in trace and "reading the file again" not in trace, trace
        assert ("chunks" if f.name.endswith("_plain") else "restart intervals") in trace, trace


@pytest.mark.parametrize("f", CORPUS + WARNED, ids=_ids(CORPUS + WARNED))
def test_device_models_agree_or_flag(f):
    """decode_model / decode_scans_model: status 0 with libjpeg's coefficients, or a nonzero status -
    only for the features in DEVICE_MAY_FLAG (and for files libjpeg warns about)"""
    ref = df.libjpeg_coefficients(f.data)
    im, scan = qs.parse_jpeg(f.data)
    im2, scans = qs.parse_jpeg_scans(f.data)
    assert scans is not None, f.name
    for sub in KNOBS:
        results = [("scans", *qs.decode_scans_model(im2, scans, f.data, sub))]
        if scan is not None:
            out, st, _ = qs.decode_model(im, scan, f.data, sub)
            results.append(("seq", out, st))
        for who, out, st in results:
            if st == 0:
                assert _same(out, ref), (who, sub)
            else:
                assert f.cls == "warned" or f.feature in DEVICE_MAY_FLAG, (who, sub, hex(st))


@pytest.mark.parametrize("f", _tool_params())
def test_tool_copies_the_coefficients(f, tmp_path):
    """transcode_route gives a route, `jpegqs -n 0` exits 0 and writes libjpeg's coefficients of the
    input - the reference CLI's file byte for byte where it is built"""
    route, why = qs.transcode_route(f.data)
    assert route in ("device", "host") and why
    src, out = tmp_path / "in.jpg", tmp_path / "out.jpg"
    src.write_bytes(f.data)
    r = subprocess.run([EXE, "-n", "0", "-i", "0", str(src), str(out)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert _same([c.coef for c in df.libjpeg_coefficients(out.read_bytes()).comps], df.libjpeg_coefficients(f.data))
    if REF_BUILT:
        ref = tmp_path / "ref.jpg"
        r = subprocess.run([REFCLI, "-n", "0", "-i", "0", str(src), str(ref)], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        if out.read_bytes() != ref.read_bytes() and _rgb(f) and _only_table_slots_differ(out.read_bytes(), ref.read_bytes()):
            assert _same([c.coef for c in df.libjpeg_coefficients(ref.read_bytes()).comps], df.libjpeg_coefficients(f.data))
            raise TableSlotsDiffer(f.name)
        assert out.read_bytes() == ref.read_bytes()


@pytest.mark.parametrize("f", WARNED, ids=_ids(WARNED))
def test_warned_files_flag_or_agree(f, monkeypatch):
    ref = df.libjpeg_coefficients(f.data)
    for serial in (True, False):
        monkeypatch.setenv("JPEGQS_PAR_MIN_BYTES", "200")
        if serial:
            monkeypatch.setenv("JPEGQS_SERIAL_DECODE", "1")
        else:
            monkeypatch.delenv("JPEGQS_SERIAL_DECODE")
        try:
            got = qs.read_jpeg(f.data)
        except cuda.QsError:
            continue
        assert _same([c.coef for c in got.comps], ref), serial


@pytest.mark.parametrize("base", ["rst_blocks7", "plain"])
def test_fill_before_a_stuffed_zero(base, monkeypatch, capfd):
    """FF FF 00 is no marker, so T.81 does not call the first FF fill; libjpeg reads the three bytes as
    one data byte FF, without a warning.  read_jpeg does the same on one thread; the threaded
    restart-interval and chunk paths give up on it and leave the file to the one-thread decoder.
    The device models flag it or agree."""
    src = dict((n, d) for n, d, _ in sf.bases())["rst_blocks7"] if base != "plain" else df.pillow_jpeg(250, 190, quality=75)
    data = sf.stuffed_fill(src)
    assert not sf.libjpeg_warns(data)
    ref = df.libjpeg_coefficients(data)
    assert _same([c.coef for c in ref.comps], df.libjpeg_coefficients(src))
    monkeypatch.setenv("JPEGQS_SERIAL_DECODE", "1")
    assert _same([c.coef for c in qs.read_jpeg(data).comps], ref)
    monkeypatch.delenv("JPEGQS_SERIAL_DECODE")
    monkeypatch.setenv("JPEGQS_PAR_MIN_BYTES", "200")
    monkeypatch.setenv("JPEGQS_CODEC_THREADS", "6")
    monkeypatch.setenv("JPEGQS_CODEC_TRACE", "1")
    assert _same([c.coef for c in qs.read_jpeg(data).comps], ref)
    assert "decoded on" not in capfd.readouterr().err
    im, scan = qs.parse_jpeg(data)
    for sub in KNOBS:
        out, st, _ = qs.decode_model(im, scan, data, sub)
        assert st != 0 or _same(out, ref), sub


def test_boundary_files_reach_the_byte_pass_edges():
    """Together the boundary files put an RSTn's FF on the last byte of a 4096-byte chunk, an FF00 pair
    across a chunk edge and across a 16-byte thread span, and hold one-byte restart intervals (the
    smallest an interval can be: at least one code bit, the rest 1-bit padding).  Offsets count from
    each scan's entropy offset, as qd_scan_body's do."""
    total = {}
    for f in sf.boundary_files():
        _, scan = qs.parse_jpeg(f.data)
        assert scan.restart_interval == 1
        for k, v in sf.boundary_hits(f.data, scan.entropy_offset).items():
            total[k] = total.get(k, 0) + v
    assert all(v > 0 for v in total.values()), total


@pytest.mark.parametrize("f", sf.boundary_files(), ids=lambda f: f.name)
def test_boundary_files_decode(f):
    ref = df.libjpeg_coefficients(f.data)
    im, scan = qs.parse_jpeg(f.data)
    for sub in (cuda.DECODE_SUB_MIN, cuda.DECODE_SUB_DEFAULT):
        out, st, _ = qs.decode_model(im, scan, f.data, sub)
        assert st == 0 and _same(out, ref), sub
    assert _same([c.coef for c in qs.read_jpeg(f.data).comps], ref)
