"""JPEG files whose byte streams are legal (T.81) but unlike anything libjpeg-turbo's writer emits, for
the reader tests (test_streams_cpu.py, test_gpu_streams.py).

Every file starts as a libjpeg-turbo file (Pillow, or scan_files.rescan) and is then changed by byte
surgery - fill bytes before markers, 0-bit padding, marker segments moved, merged or inserted, scans
of two files spliced, component identifiers and table selectors relabelled - or written again by a
small libjpeg program (built at first use, as scan_files.py builds its own) with custom Huffman
tables whose codes reach 16 bits.  Each entry is a StreamFile: a name, the bytes, its class and the
feature it exercises.  class "legal": libjpeg-turbo reads the coefficients the file was made from,
without a warning; "warned": libjpeg-turbo reads them but warns.

boundary_files() are large files with a restart marker every MCU (every block for grey) whose
markers and stuffed FF00 pairs fall on the edges of the device byte passes' chunks and thread spans
(boundary_hits measures that)."""
from __future__ import annotations

import os
import subprocess
import tempfile
from dataclasses import dataclass

import numpy as np

import decode_files as df
import hard_content as hc
import libjpeg_pixels as lp
import scan_files as sf

QD_CHUNK, QD_SPAN = 4096, 16            # qs_decode.h QD_CHUNK, and 16 bytes per byte-pass thread
FILLS = (1, 2, 7)


@dataclass
class StreamFile:
    name: str
    data: bytes
    cls: str                              # "legal" or "warned"
    feature: str                          # fill (before a marker that ends a scan), fill_rst, zero_pad,
                                          # layout, dri, ids, long_codes, boundary, garbage


# ---------------------------------------------------------------- the byte stream
def pieces(data: bytes):
    """The file as [code, bytes] pairs in order: every marker with its segment (code 0xD8 / 0xD9 alone),
    and after each SOS its entropy-coded data with the RSTn markers inside as code None."""
    out, p = [[0xD8, data[:2]]], 2
    while p < len(data):
        assert data[p] == 0xFF, p
        code = data[p + 1]
        if code == 0xD9:
            out.append([0xD9, data[p:p + 2]])
            assert p + 2 == len(data)
            break
        n = int.from_bytes(data[p + 2:p + 4], "big")
        out.append([code, data[p:p + 2 + n]])
        p += 2 + n
        if code == 0xDA:
            q = p
            while not (data[q] == 0xFF and data[q + 1] != 0 and not 0xD0 <= data[q + 1] <= 0xD7):
                q += 1
            out.append([None, data[p:q]])
            p = q
    return out


def join(ps) -> bytes:
    return b"".join(b for _, b in ps)


def rst_offsets(seg: bytes):
    """offsets of the RSTn markers in entropy-coded data"""
    return [i for i in range(len(seg) - 1) if seg[i] == 0xFF and 0xD0 <= seg[i + 1] <= 0xD7]


def _segment(code: int, payload: bytes) -> bytes:
    return bytes([0xFF, code]) + (len(payload) + 2).to_bytes(2, "big") + payload


def _index(ps, code, k=0):
    """position in ps of the k-th piece with this code"""
    return [i for i, (c, _) in enumerate(ps) if c == code][k]


# ---------------------------------------------------------------- 1. fill bytes
def fill_rst(data: bytes, n: int, which=None) -> bytes:
    """n FF fill bytes before RST marker `which` (an index over the whole file), or before every one"""
    ps, k = pieces(data), 0
    for piece in ps:
        if piece[0] is not None:
            continue
        seg, out, last = piece[1], b"", 0
        for r in rst_offsets(seg):
            if which is None or k == which:
                out += seg[last:r] + b"\xff" * n
                last = r
            k += 1
        piece[1] = out + seg[last:]
    return join(ps)


def fill_before(data: bytes, n: int, code: int, k: int) -> bytes:
    """n FF fill bytes before the k-th marker with this code"""
    ps = pieces(data)
    i = _index(ps, code, k)
    ps[i][1] = b"\xff" * n + ps[i][1]
    return join(ps)


def _dht_between_scans(data: bytes) -> int:
    """k of the first DHT that follows a scan"""
    ps = pieces(data)
    return sum(1 for c, _ in ps[:_index(ps, 0xDA)] if c == 0xC4)


# ---------------------------------------------------------------- 2. 0-bit padding
def zero_pad(data: bytes, before: str) -> bytes | None:
    """The first interval end before an RST (before="rst") or the scan end before EOI (before="eoi")
    whose padding bits can be cleared: the trailing 1-bits of the last byte, as many as libjpeg still
    reads the same coefficients with (the rest are data).  None when no such byte is found."""
    want = df.libjpeg_coefficients(data)
    ps = pieces(data)
    spots = []
    for i, (c, seg) in enumerate(ps):
        if c is None:
            ends = rst_offsets(seg) if before == "rst" else ([len(seg)] if ps[i + 1][0] == 0xD9 else [])
            spots += [(i, e) for e in ends]
    for i, e in spots:
        seg = ps[i][1]
        b = seg[e - 1]
        if e < 2 or seg[e - 2] == 0xFF or b == 0xFF:        # a stuffed byte or an FF: not plain padding
            continue
        ones = 0
        while ones < 8 and b >> ones & 1:
            ones += 1
        for j in range(min(ones, 7), 0, -1):
            trial = [list(x) for x in ps]
            trial[i][1] = seg[:e - 1] + bytes([b & ~((1 << j) - 1) & 0xFF]) + seg[e:]
            out = join(trial)
            got = df.libjpeg_coefficients(out)
            if all(np.array_equal(a.coef, g.coef) for a, g in zip(want.comps, got.comps)) and not libjpeg_warns(out):
                return out
    return None


# ---------------------------------------------------------------- 3. marker segments and table layouts
def insert_before(data: bytes, code: int, k: int, segs: bytes) -> bytes:
    ps = pieces(data)
    i = _index(ps, code, k)
    ps.insert(i, [0xFE, segs])
    return join(ps)


def dht_merged(data: bytes) -> bytes:
    """every run of DHT segments merged into one segment holding all their tables"""
    ps, out = pieces(data), []
    for c, b in ps:
        if c == 0xC4 and out and out[-1][0] == 0xC4:
            out[-1][1] = _segment(0xC4, out[-1][1][4:] + b[4:])
        else:
            out.append([c, b])
    return join(out)


def dht_first(data: bytes) -> bytes:
    """the DHT segments before the first scan moved, one table each, right after SOI (before DQT and SOF)"""
    ps = pieces(data)
    first_sos = _index(ps, 0xDA)
    dht = [p for p in ps[:first_sos] if p[0] == 0xC4]
    rest = [p for i, p in enumerate(ps) if not (i < first_sos and p[0] == 0xC4)]
    return join(rest[:1] + dht + rest[1:])


def dri_changed(a: bytes, b: bytes, k: int, ri: int) -> bytes:
    """a's scans before scan k, then DRI(ri) and b's scans from k on: a and b hold the same
    coefficients under the same scan script, with restart intervals ri_a and ri"""
    pa, pb = pieces(a), pieces(b)
    def cut(ps):                                            # start of the markers that lead to scan k
        i = _index(ps, 0xDA, k)
        while ps[i - 1][0] is not None:
            i -= 1
        return i
    return join(pa[:cut(pa)]) + _segment(0xDD, ri.to_bytes(2, "big")) + join(pb[cut(pb):])


# ---------------------------------------------------------------- 4. component identity
def relabel(data: bytes, ids=None, swap_tables=False, adobe=None) -> bytes:
    """component identifiers replaced (SOF and every SOS), Huffman table slots 0 and 1 swapped (DHT and
    SOS), and / or the JFIF APP0 replaced by an Adobe APP14 with this transform"""
    ps, out = pieces(data), []
    sw = (lambda t: {0: 1, 1: 0}.get(t, t)) if swap_tables else (lambda t: t)
    old = None
    for c, b in ps:
        b = bytearray(b)
        if c in (0xC0, 0xC1, 0xC2):
            nf = b[9]
            old = [b[10 + 3 * i] for i in range(nf)]
            if ids:
                for i in range(nf):
                    b[10 + 3 * i] = ids[i]
        elif c == 0xDA:
            ns = b[4]
            for i in range(ns):
                if ids:
                    b[5 + 2 * i] = ids[old.index(b[5 + 2 * i])]
                t = b[6 + 2 * i]
                b[6 + 2 * i] = sw(t >> 4) << 4 | sw(t & 15)
        elif c == 0xC4:
            p = 4
            while p < len(b):
                b[p] = (b[p] & 0xF0) | sw(b[p] & 15)
                p += 17 + sum(b[p + 1:p + 17])
        elif c == 0xE0 and adobe is not None and bytes(b[4:9]) == b"JFIF\x00":
            b = bytearray(_segment(0xEE, b"Adobe" + bytes([0, 100, 0, 0, 0, 0, adobe])))
        out.append([c, bytes(b)])
    return join(out)


# ---------------------------------------------------------------- 5. long Huffman codes
PROGRAM = r'''
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <jpeglib.h>
/* retable in.jpg out.jpg spec.bin: spec = int32 nscans, restart_interval, then per scan int32 ncomp, comp[4],
 * then 4 tables (DC 0, DC 1, AC 0, AC 1) of 17 + 256 bytes (bits, huffval).  The coefficients of in.jpg are
 * written again with these tables: optimize_coding = FALSE, the table pointers set. */
int main(int argc, char **argv) {
	struct jpeg_decompress_struct di; struct jpeg_compress_struct co; struct jpeg_error_mgr e1, e2;
	FILE *f, *o, *s; int hdr[2], i, k; jpeg_scan_info *sc = NULL; unsigned char t[4][17 + 256];
	if (argc != 4 || !(f = fopen(argv[1], "rb")) || !(s = fopen(argv[3], "rb"))) return 2;
	if (fread(hdr, 4, 2, s) != 2) return 2;
	if (hdr[0]) {
		sc = calloc((size_t)hdr[0], sizeof(*sc));
		for (i = 0; i < hdr[0]; i++) {
			int r[5];
			if (fread(r, 4, 5, s) != 5) return 2;
			sc[i].comps_in_scan = r[0];
			for (k = 0; k < 4; k++) sc[i].component_index[k] = r[1 + k];
			sc[i].Ss = 0; sc[i].Se = 63; sc[i].Ah = 0; sc[i].Al = 0;
		}
	}
	if (fread(t, sizeof(t), 1, s) != 1) return 2;
	di.err = jpeg_std_error(&e1);
	jpeg_create_decompress(&di);
	jpeg_stdio_src(&di, f);
	jpeg_read_header(&di, TRUE);
	jvirt_barray_ptr *arr = jpeg_read_coefficients(&di);
	co.err = jpeg_std_error(&e2);
	jpeg_create_compress(&co);
	if (!(o = fopen(argv[2], "wb"))) return 2;
	jpeg_stdio_dest(&co, o);
	jpeg_copy_critical_parameters(&di, &co);
	co.restart_interval = (unsigned)hdr[1]; co.optimize_coding = FALSE;
	if (sc) { co.scan_info = sc; co.num_scans = hdr[0]; }
	for (i = 0; i < 4; i++) {
		JHUFF_TBL *h = jpeg_alloc_huff_table((j_common_ptr)&co);
		memcpy(h->bits, t[i], 17); memcpy(h->huffval, t[i] + 17, 256); h->sent_table = FALSE;
		if (i < 2) co.dc_huff_tbl_ptrs[i] = h; else co.ac_huff_tbl_ptrs[i - 2] = h;
	}
	for (i = 0; i < co.num_components; i++) { co.comp_info[i].dc_tbl_no = i ? 1 : 0; co.comp_info[i].ac_tbl_no = i ? 1 : 0; }
	jpeg_write_coefficients(&co, arr);
	jpeg_finish_compress(&co); jpeg_destroy_compress(&co);
	jpeg_finish_decompress(&di); jpeg_destroy_decompress(&di);
	fclose(o); fclose(f); fclose(s);
	return 0;
}
'''

_exe = None
_tmp = None


def _program() -> str:
    global _exe, _tmp
    if _exe is None:
        if lp.JPEG_SO is None:
            raise lp.LibjpegError("no libjpeg shared library inside Pillow")
        _tmp = tempfile.TemporaryDirectory(prefix="stream_files_")
        src, exe = os.path.join(_tmp.name, "retable.c"), os.path.join(_tmp.name, "retable")
        with open(src, "w") as f:
            f.write(PROGRAM)
        subprocess.run(["/usr/bin/gcc", "-O1", "-I", os.path.join(lp.ROOT, "include", "libjpeg62"), src, "-o", exe,
                        lp.JPEG_SO, f"-Wl,-rpath,{os.path.dirname(lp.JPEG_SO)}"], check=True)
        _exe = exe
    return _exe


# DC: 12 symbols, one code of each length 1..10 and two of 16 bits; the categories in an order that
# gives the long codes to the large differences and some of the small ones
DC_BITS = [0] + [1] * 10 + [0] * 5 + [2]
DC_VALS = [5, 4, 6, 3, 7, 2, 8, 1, 9, 0, 10, 11]
# AC: all 162 symbols, codes of every length 2..16 (a code of length 1 would leave room for only
# one code per length below it), most of them 12 to 15 bits: longer than the decoders' 9- and
# 10-bit look-ups
AC_BITS = [0, 0] + [1] * 8 + [4, 5, 21, 41, 41, 41, 1]
AC_SYMBOLS = [0x00, 0xF0] + [r << 4 | s for r in range(16) for s in range(1, 11)]


def long_tables(seed: int):
    """(DC bits, DC vals), (AC bits, AC vals): the symbols of the AC table in a seeded order, so the
    common ones (EOB, short runs of small values) get long codes as often as short ones"""
    assert sum(DC_BITS) == 12 and sum(AC_BITS) == 162 == len(AC_SYMBOLS)
    assert sum(n << (16 - l) for l, n in enumerate(AC_BITS)) < 1 << 16 > sum(n << (16 - l) for l, n in enumerate(DC_BITS))
    ac = list(np.random.RandomState(seed).permutation(AC_SYMBOLS))
    return (DC_BITS, DC_VALS), (AC_BITS, ac)


def retable(data: bytes, per_component_scans: bool = False, restart_interval: int = 0) -> bytes:
    """data's coefficients written by libjpeg with long_tables (slot 0: luma, slot 1: chroma), as one
    interleaved scan or one scan per component.  libjpeg's progressive writer always computes its own
    tables, so the scripts here are sequential."""
    nc = len(df.libjpeg_coefficients(data).comps)
    words = [nc if per_component_scans else 0, restart_interval]
    if per_component_scans:
        for c in range(nc):
            words += [1, c, 0, 0, 0]
    tabs = b""
    (db0, dv0), (ab0, av0) = long_tables(1)
    (db1, dv1), (ab1, av1) = long_tables(2)
    for bits, vals in ((db0, dv0), (db1, dv1[::-1]), (ab0, av0), (ab1, av1)):
        tabs += bytes(bits) + bytes(vals) + bytes(256 - len(vals))
    with tempfile.TemporaryDirectory() as d:
        i, o, s = (os.path.join(d, n) for n in ("i.jpg", "o.jpg", "s.bin"))
        open(i, "wb").write(data)
        open(s, "wb").write(np.array(words, np.int32).tobytes() + tabs)
        r = subprocess.run([_program(), i, o, s], capture_output=True, text=True)
        if r.returncode:
            raise lp.LibjpegError(f"libjpeg: {(r.stderr or r.stdout).strip()} (exit {r.returncode})")
        return open(o, "rb").read()


def dc_categories(data: bytes) -> int:
    """the largest DC difference category (SSSS) of an interleaved or one-component scan of a 4:4:4 or
    grey file without restarts: there the coding order of each component's blocks is raster order"""
    ref = df.libjpeg_coefficients(data)
    top = 0
    for c in ref.comps:
        assert (c.h_samp, c.v_samp) == (1, 1)
        dc = c.coef[..., 0].astype(np.int64).reshape(-1)
        diff = np.abs(np.diff(np.concatenate([[0], dc])))
        top = max(top, int(diff.max()).bit_length())
    return top


def _dc11_file(ss: str) -> bytes:
    """hard_content's saturated set under a flat quant table of ones: DC values near +-1024 whose
    differences reach category 11"""
    im = hc.make_image(64, 48, ss, hc.flat(1), "saturated", seed=9)
    return df.coef_writer_jpeg(im)


# ---------------------------------------------------------------- the corpus
def libjpeg_warns(data: bytes) -> bool:
    """libjpeg-turbo's jpeg_read_coefficients of the file printed a warning"""
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "f.jpg")
        open(p, "wb").write(data)
        r = subprocess.run([lp._program(), "dump", p, os.path.join(d, "c.bin")], capture_output=True, text=True)
        if r.returncode:
            raise lp.LibjpegError(r.stderr.strip())
        return bool(r.stderr.strip())


def bases():
    """(name, bytes, progressive) of the files the surgery starts from: sequential and progressive,
    colour and grey, with restart markers"""
    c420 = df.pillow_jpeg(131, 77, quality=88, subsampling=2, seed=11)
    grey = df.pillow_jpeg(90, 70, "L", quality=92, seed=5)
    return [("rst_blocks7", df.pillow_jpeg(250, 190, quality=75, restart_marker_blocks=7), False),
            ("rst_gray", df.pillow_jpeg(97, 61, "L", quality=90, restart_marker_blocks=3), False),
            ("prog_rst_blocks5", df.pillow_jpeg(250, 190, quality=75, progressive=True, restart_marker_blocks=5), True),
            ("succ_al3_420_rst3", sf.rescan(c420, sf.successive(3), restart_interval=3), True),
            ("succ_al3_gray_rst3", sf.rescan(grey, sf.successive(1), restart_interval=3), True)]


def corpus():
    """every StreamFile but the boundary ones"""
    out = []
    add = lambda name, data, feature: out.append(StreamFile(name, data, "legal", feature))
    for name, data, prog in bases():
        nrst = sum(len(rst_offsets(b)) for c, b in pieces(data) if c is None)
        nsos = sum(1 for c, _ in pieces(data) if c == 0xDA)
        for n in FILLS:
            add(f"fill{n}_rst_{name}", fill_rst(data, n, nrst // 2), "fill_rst")
            add(f"fill{n}_every_rst_{name}", fill_rst(data, n), "fill_rst")
            add(f"fill{n}_eoi_{name}", fill_before(data, n, 0xD9, 0), "fill")
            if prog:
                add(f"fill{n}_sos_{name}", fill_before(data, n, 0xDA, nsos // 2), "fill")
                add(f"fill{n}_dht_{name}", fill_before(data, n, 0xC4, _dht_between_scans(data)), "fill")
        for before in ("rst", "eoi"):
            z = zero_pad(data, before)
            if z is not None:                               # (the last byte may be all data, or stuffed)
                add(f"zero_pad_{before}_{name}", z, "zero_pad")
    plain = df.pillow_jpeg(250, 190, quality=75)
    for n in FILLS:
        add(f"fill{n}_eoi_plain", fill_before(plain, n, 0xD9, 0), "fill")

    prog = df.pillow_jpeg(250, 190, quality=75, progressive=True, seed=4)
    nsos = sum(1 for c, _ in pieces(prog) if c == 0xDA)
    add("com_app_between_scans", insert_before(insert_before(prog, 0xDA, 2, _segment(0xFE, b"a comment between scans")),
                                               0xDA, nsos - 1, _segment(0xE5, b"APP5 between scans\0" + bytes(40))), "layout")
    for name, data in (("seq", plain), ("prog", prog)):
        add(f"dht_merged_{name}", dht_merged(data), "layout")
        add(f"dht_first_{name}", dht_first(data), "layout")

    c420 = df.pillow_jpeg(131, 77, quality=88, subsampling=2, seed=11)
    add("dri_change_prog", dri_changed(sf.rescan(c420, sf.successive(3), restart_interval=3),
                                       sf.rescan(c420, sf.successive(3), restart_interval=5), 4, 5), "dri")
    add("dri_change_seq", dri_changed(sf.rescan(c420, sf.per_component_sequential(3), restart_interval=4),
                                      sf.rescan(c420, sf.per_component_sequential(3), restart_interval=9), 1, 9), "dri")
    nmcu = 17 * 10                                          # 131 x 77 at 4:2:0
    for ri in (nmcu, 65535):
        add(f"ri{ri}_seq", sf.rescan(c420, restart_interval=ri), "dri")
        add(f"ri{ri}_prog", sf.rescan(c420, sf.successive(3), restart_interval=ri), "dri")

    for name, data in (("seq", plain), ("prog", prog)):
        add(f"ids_012_{name}", relabel(data, ids=[0, 1, 2]), "ids")
        add(f"ids_rgb_adobe0_{name}", relabel(data, ids=list(b"RGB"), adobe=0), "ids")
        add(f"tables_swapped_{name}", relabel(data, swap_tables=True), "ids")

    c444 = df.pillow_jpeg(120, 88, quality=95, subsampling=0, seed=6)
    for name, data in (("420", plain), ("444", c444), ("gray", df.pillow_jpeg(97, 61, "L", quality=90))):
        add(f"long_codes_{name}", retable(data), "long_codes")
        add(f"long_codes_{name}_rst3", retable(data, restart_interval=3), "long_codes")
        if name != "gray":
            add(f"long_codes_{name}_per_comp", retable(data, per_component_scans=True, restart_interval=5), "long_codes")
    for ss in ("gray", "444"):
        add(f"long_codes_dc11_{ss}", retable(_dc11_file(ss)), "long_codes")
    return out


def warned():
    """files libjpeg reads with a warning: garbage bytes before EOI, or before the first RSTn
    (JWRN_EXTRANEOUS_DATA), each file with one of the two"""
    out = []
    for name, data, _ in bases()[:3]:
        ps = pieces(data)
        i = _index(ps, 0xD9)
        ps[i][1] = b"\x12\x34" + ps[i][1]
        out.append(StreamFile(f"garbage_eoi_{name}", join(ps), "warned", "garbage"))
        ps = pieces(data)
        piece = next(p for p in ps if p[0] is None and rst_offsets(p[1]))
        r = rst_offsets(piece[1])[0]
        piece[1] = piece[1][:r] + b"\xff\x00\x77" + piece[1][r:]
        out.append(StreamFile(f"garbage_rst_{name}", join(ps), "warned", "garbage"))
    return [f for f in out if libjpeg_warns(f.data)]     # (bytes the entropy decoder read ahead go unreported)


def stuffed_fill(data: bytes) -> bytes:
    """one FF added before the FF of the first stuffed FF00 pair: FF FF 00, which is no marker, so not
    T.81's fill; libjpeg's jpeg_fill_bit_buffer reads it as one data byte FF, without a warning"""
    ps = pieces(data)
    piece = next(p for p in ps if p[0] is None and b"\xff\x00" in p[1])
    i = piece[1].index(b"\xff\x00")
    piece[1] = piece[1][:i] + b"\xff" + piece[1][i:]
    return join(ps)


# ---------------------------------------------------------------- 6. device byte-pass boundaries
BOUNDARY_SIZE = (2048, 1536)


def _flat_pixels(w, h, channels):
    yy, xx = np.mgrid[0:h, 0:w]
    base = (100 + (xx // 96) * 3 + (yy // 80) * 2).astype(np.uint8)
    return np.stack([base, base // 2 + 40, 200 - base], -1) if channels == 3 else base


def boundary_files():
    """busy and flat content, colour (a restart every MCU) and grey (every block)"""
    import io
    from PIL import Image
    w, h = BOUNDARY_SIZE
    out = []
    for kind in ("busy", "flat"):
        for mode in ("RGB", "L"):
            if kind == "busy":
                px = df.pixels(w, h, 3, seed=21)
                px = px if mode == "RGB" else np.ascontiguousarray(px[..., 0])
            else:
                px = _flat_pixels(w, h, 3 if mode == "RGB" else 1)
            b = io.BytesIO()
            Image.fromarray(px).save(b, "JPEG", quality=95 if kind == "busy" else 50, restart_marker_blocks=1)
            out.append(StreamFile(f"boundary_{kind}_{'color' if mode == 'RGB' else 'gray'}", b.getvalue(), "legal", "boundary"))
    return out


def boundary_hits(data: bytes, off: int):
    """which byte-pass edges the entropy-coded data from offset off (the scan's entropy offset, where
    qd_scan_body measures its chunks from) reaches: counts of RSTn markers whose FF ends a chunk, of
    FF00 pairs split by a chunk edge and by a 16-byte thread span, and of one-byte restart intervals"""
    seg = np.frombuffer(data, np.uint8)[off:].astype(np.int64)
    ff = np.flatnonzero(seg[:-1] == 0xFF)
    nxt = seg[ff + 1]
    rst = ff[(nxt & 0xF8) == 0xD0]
    stuffed = ff[nxt == 0]
    # an interval of one byte: an RST (or the scan start) followed by one data byte and an RST
    starts = np.concatenate([[-2], rst])
    one_byte = int(np.sum(np.diff(starts) == 3))
    return {"rst_ff_ends_chunk": int(np.sum(rst % QD_CHUNK == QD_CHUNK - 1)),
            "ff00_across_chunk": int(np.sum(stuffed % QD_CHUNK == QD_CHUNK - 1)),
            "ff00_across_span": int(np.sum(stuffed % QD_SPAN == QD_SPAN - 1)),
            "one_byte_interval": one_byte}
