"""The scan decoder on the host: parse_jpeg_scans, the workspace formula, argument checks and
decode_scans_model - decode_scans_async's algorithm on one CPU thread - against libjpeg-turbo's
jpeg_read_coefficients on progressive and multi-scan files.  No GPU is used."""
import ctypes as C

import numpy as np
import pytest

import decode_files as df
import libjpeg_pixels as lp
import scan_files as sf
import jpegqs_b200 as qs
from jpegqs_b200 import cuda

pytestmark = pytest.mark.skipif(lp.JPEG_SO is None, reason="no libjpeg inside Pillow")

PILLOW = sf.pillow_progressive()
SCRIPTED = sf.scripted()
HARD = sf.hard_progressive()
GEOMETRY = sf.geometry_progressive()
KNOBS = [cuda.DECODE_SUB_MIN, cuda.DECODE_SUB_DEFAULT]


def _same(a, ref):
    return len(a) == len(ref.comps) and all(np.array_equal(np.asarray(x), y.coef) for x, y in zip(a, ref.comps))


@pytest.mark.parametrize("sub_bytes", KNOBS)
@pytest.mark.parametrize("name,data", PILLOW + SCRIPTED + HARD + GEOMETRY, ids=[n for n, _ in PILLOW + SCRIPTED + HARD + GEOMETRY])
def test_model_equals_libjpeg(name, data, sub_bytes):
    ref = df.libjpeg_coefficients(data)
    im, scans = qs.parse_jpeg_scans(data)
    assert scans is not None
    out, status = qs.decode_scans_model(im, scans, data, sub_bytes)
    assert status == 0
    assert _same(out, ref)


def test_scan_kinds_are_covered():
    kinds = set()
    for _, data in PILLOW + SCRIPTED:
        _, scans = qs.parse_jpeg_scans(data)
        for r in scans:
            prog = r.sof == 0xC2
            kinds.add("seq" if not prog else ("dc" if r.Ss == 0 else "ac") + ("_refine" if r.Ah else "_first"))
            if prog and r.Ss == 0:
                assert r.Se == 0
    assert kinds == {"seq", "dc_first", "ac_first", "dc_refine", "ac_refine"}


def test_parse_records_every_scan():
    data = dict(SCRIPTED)["succ_al3_420_rst3"]
    im, scans = qs.parse_jpeg_scans(data)
    assert len(scans) == 1 + 3 + 3 * 4
    assert all(r.restart_interval == 3 for r in scans)
    for r in scans:                                             # each segment ends at a marker that is not RSTn
        assert data[r.end] == 0xFF and data[r.end + 1] in (0xC4, 0xDA, 0xD9, 0xDD)
    assert [(r.Ss, r.Se, r.Ah, r.Al) for r in scans[:2]] == [(0, 0, 0, 3), (1, 63, 0, 3)]
    # a sequential file: one record, the scan parse_jpeg gives
    seq = df.pillow_jpeg(64, 48, quality=75)
    _, one = qs.parse_jpeg_scans(seq)
    _, sc = qs.parse_jpeg(seq)
    assert len(one) == 1 and one[0].offset == sc.entropy_offset and (one[0].Ss, one[0].Se) == (0, 63)


def test_parse_rejects_what_the_reader_rejects():
    data = df.pillow_jpeg(64, 48, quality=75, progressive=True)
    sof = data.index(b"\xff\xc2")
    with pytest.raises(cuda.QsError):
        qs.parse_jpeg_scans(data[:sof + 1] + b"\xc9" + data[sof + 2:])
    with pytest.raises(cuda.QsError):
        qs.parse_jpeg_scans(b"not a jpeg")
    # more scans than the device decoder takes: the host reader's file
    many = sf.rescan(df.pillow_jpeg(32, 32, "L", quality=90), [((0,), 0, 0, 0, 0)] + [((0,), k, k, 0, 0) for k in range(1, 64)])
    im, scans = qs.parse_jpeg_scans(many)
    assert scans is not None and len(scans) == 64
    lib = cuda.load()
    ci, recs, n = cuda._Image(), (cuda._ScanRec * 4)(), C.c_int(0)
    assert lib.jpegqs_cuda_jpeg_parse_scans(many, len(many), C.byref(ci), recs, 4, C.byref(n)) == -3 and n.value == 64


def _a(x):
    return (x + 255) // 256 * 256


def test_workspace_formula_and_existing_decoder_unchanged():
    for name, data in SCRIPTED[:6] + PILLOW[:3]:
        im, scans = qs.parse_jpeg_scans(data)
        want = 0
        for r in scans:
            L = r.end - r.offset
            comps = [im.comps[c] for c in r.comp[:r.ncomp]]
            if r.ncomp == 1:
                mcus = comps[0].wblk * comps[0].hblk
            else:
                mh, mv = max(c.h_samp for c in im.comps), max(c.v_samp for c in im.comps)
                mcus = -(-im.width // (8 * mh)) * -(-im.height // (8 * mv))
            I = -(-mcus // r.restart_interval) if r.restart_interval else 1
            first = r.Ah == 0
            want += 16384 + _a(L + 8) + _a(24 * -(-L // 4096)) + 2 * _a(4 * I) + (_a(96 * (L // 32 + I)) if first else 0)
        assert qs.decode_scans_workspace_bytes([im], [scans], [len(data)]) == want, name
    # decode_async's workspace for sequential files: its formula, untouched
    for name, data in df.flavours()[:4]:
        im, sc = qs.parse_jpeg(data)
        L = len(data) - sc.entropy_offset
        mh, mv = max(c.h_samp for c in im.comps), max(c.v_samp for c in im.comps)
        mcus = -(-im.width // (8 * mh)) * -(-im.height // (8 * mv))
        I = -(-mcus // sc.restart_interval) if sc.restart_interval else 1
        want = 16384 + _a(L + 8) + _a(24 * -(-L // 4096)) + 2 * _a(4 * I) + _a(96 * (L // 32 + I))
        assert qs.decode_workspace_bytes([im], [sc], [len(data)]) == want


def test_argument_errors():
    data = dict(PILLOW)["prog_420"]
    im, scans = qs.parse_jpeg_scans(data)
    with pytest.raises(cuda.QsError):
        qs.decode_scans_model(im, scans, data, 31)                 # knob below 32
    bad = cuda.ScanList(cuda._ScanRec.from_buffer_copy(r) for r in scans)
    bad[1].end = len(data) + 1                                  # past the data
    with pytest.raises(cuda.QsError):
        qs.decode_scans_workspace_bytes([im], [bad], [len(data)])
    for field, value in (("Se", 64), ("Al", 14), ("sof", 0xC3), ("ncomp", 0)):
        bad = cuda.ScanList(cuda._ScanRec.from_buffer_copy(r) for r in scans)
        setattr(bad[2], field, value)
        with pytest.raises(cuda.QsError):
            qs.decode_scans_model(im, bad, data)
    bad = cuda.ScanList(cuda._ScanRec.from_buffer_copy(r) for r in scans)
    ac = next(r for r in bad if r.Ss > 0)
    ac.ncomp, ac.comp[1] = 2, 1                                 # an AC scan of two components
    with pytest.raises(cuda.QsError):
        qs.decode_scans_model(im, bad, data)
    bad = cuda.ScanList(cuda._ScanRec.from_buffer_copy(r) for r in scans)
    ac = next(r for r in bad if r.Ss > 0)
    ac.ac_present[ac.ac_tbl[0]] = 0                             # an absent table
    with pytest.raises(cuda.QsError):
        qs.decode_scans_model(im, bad, data)
    with pytest.raises(cuda.QsError):
        qs.decode_scans_workspace_bytes([im], [cuda.ScanList()], [len(data)])   # no scans


def _damaged(rng, data, kind):
    b = bytearray(data)
    if kind == 0:
        return bytes(b[:rng.integers(len(b) // 3, len(b))])
    if kind == 1:
        for _ in range(rng.integers(1, 4)):
            p = int(rng.integers(len(b) // 4, len(b) - 2))
            b[p] ^= 1 << int(rng.integers(0, 8))
        return bytes(b)
    i = bytes(b).find(b"\xff\xd1")
    return bytes(b[:i] + b[i + 2:]) if i > 0 else bytes(b)


def _cut_at_sos(data, extra):
    """data cut `extra` bytes after the header of its second SOS: a partial download."""
    sos = data.index(b"\xff\xda", data.index(b"\xff\xda") + 2)
    return data[:sos + 2 + int.from_bytes(data[sos + 2:sos + 4], "big") + extra]


def test_cut_at_an_sos():
    """A file cut at the end of an SOS header has a scan without entropy-coded bytes: only the host
    reader takes it.  One byte later the device decoder takes it and flags it; the file's last byte
    belongs to the segment."""
    data = dict(PILLOW)["prog_420"]
    cut = _cut_at_sos(data, 0)
    im, scans = qs.parse_jpeg_scans(cut)
    assert scans is None
    qs.read_jpeg(cut)
    for extra in (1, 2, 9):
        cut = _cut_at_sos(data, extra)
        im, scans = qs.parse_jpeg_scans(cut)
        assert scans is not None and scans[-1].end == len(cut) and scans[-1].end - scans[-1].offset == extra
        qs.decode_scans_workspace_bytes([im], [scans], [len(cut)])
        _, status = qs.decode_scans_model(im, scans, cut)
        assert status != 0


def test_damaged_files_status_zero_implies_equality():
    rng = np.random.default_rng(7)
    sources = [dict(PILLOW)["prog_420"], dict(SCRIPTED)["succ_al3_420_rst3"], dict(SCRIPTED)["split_bands_gray"],
               dict(PILLOW)["prog_rst_blocks5"]]
    flagged = 0
    for it in range(80):
        src = sources[it % len(sources)]
        data = _damaged(rng, src, it % 3)
        try:
            im, scans = qs.parse_jpeg_scans(data)
        except cuda.QsError:
            continue
        if scans is None:
            continue
        guard = 4096
        bufs = [np.full(c.hblk * c.wblk * 64 + 2 * guard, 0x5A5A, np.int16) for c in im.comps]
        views = [b[guard:-guard].reshape(c.hblk, c.wblk, 64) for b, c in zip(bufs, im.comps)]
        _, status = qs.decode_scans_model(im, scans, data, cuda.DECODE_SUB_MIN, out=views)
        for b in bufs:
            assert (b[:guard] == 0x5A5A).all() and (b[-guard:] == 0x5A5A).all()
        if status == 0:
            ref = qs.read_jpeg(data)
            assert all(np.array_equal(v, c.coef) for v, c in zip(views, ref.comps))
        else:
            flagged += 1
    assert flagged > 10
    # cut at and just after an SOS header, guards included
    for extra in (0, 1, 2):
        data = _cut_at_sos(sources[it % len(sources)], extra)
        im, scans = qs.parse_jpeg_scans(data)
        if scans is None:
            continue
        bufs = [np.full(c.hblk * c.wblk * 64 + 2 * 4096, 0x5A5A, np.int16) for c in im.comps]
        views = [b[4096:-4096].reshape(c.hblk, c.wblk, 64) for b, c in zip(bufs, im.comps)]
        _, status = qs.decode_scans_model(im, scans, data, cuda.DECODE_SUB_MIN, out=views)
        assert status != 0 and all((b[:4096] == 0x5A5A).all() and (b[-4096:] == 0x5A5A).all() for b in bufs)
