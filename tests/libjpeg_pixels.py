"""Pixel oracle: what libjpeg itself decodes a coefficient set to.

A small C program, built at first use against the libjpeg-turbo inside Pillow's wheel (declared by
include/libjpeg62, as tests/test_real_libjpeg.py does), either

  * reads a JPEG file's coefficients with jpeg_read_coefficients (`read_coefficients`), or
  * writes a coefficient set with jpeg_write_coefficients - its own quant table per component,
    16-bit DQT entries where a value needs them, optimised Huffman tables - and decodes that file
    with jpeg_read_scanlines to JCS_RGB with JDCT_ISLOW and fancy up-sampling (`decode`).

A coefficient set libjpeg cannot code (an AC value or DC difference beyond the 10 / 11 bits of 8-bit
JPEG) makes libjpeg's error_exit end the program, and `decode` raises LibjpegError: callers never
get pixels for such a set.

`device_model` restates on the CPU the arithmetic the library's renderers use (the reference's
32-bit islow IDCT with a clamp, libjpeg's up-sampling rules, jdcolor.c's fixed-point YCbCr -> RGB),
so the CPU tests can tell where that arithmetic and libjpeg-turbo's SIMD decoder part ways.
Nothing here touches a GPU.
"""
from __future__ import annotations

import glob
import os
import subprocess
import tempfile

import numpy as np

from jpegqs_b200.image import CoefImage, Component, JCS_YCbCr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _pillow_libjpeg():
    try:
        import PIL
    except ImportError:
        return None
    so = sorted(glob.glob(os.path.join(os.path.dirname(os.path.realpath(PIL.__file__)), "..", "pillow.libs", "libjpeg*.so*")))
    return os.path.realpath(so[0]) if so else None


JPEG_SO = _pillow_libjpeg()


class LibjpegError(RuntimeError):
    pass


PROGRAM = r'''
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <jpeglib.h>
/* file format: int32 ncomp, color_space, width, height; per component int32 h_samp, v_samp, wblk, hblk,
 * quant[64]; then per component int16 [hblk][wblk][64] */
static void die(const char *m) { fprintf(stderr, "%s\n", m); exit(2); }
static void rd(void *p, size_t n, FILE *f) { if (fread(p, 1, n, f) != n) die("short read"); }

static int dump(const char *in, const char *out) {
	struct jpeg_decompress_struct di; struct jpeg_error_mgr err; FILE *f = fopen(in, "rb"), *o = fopen(out, "wb");
	int c; JDIMENSION y;
	if (!f || !o) die("open");
	di.err = jpeg_std_error(&err);
	jpeg_create_decompress(&di);
	jpeg_stdio_src(&di, f);
	jpeg_read_header(&di, TRUE);
	jvirt_barray_ptr *arr = jpeg_read_coefficients(&di);
	int hdr[4] = {di.num_components, (int)di.jpeg_color_space, (int)di.image_width, (int)di.image_height};
	fwrite(hdr, sizeof(int), 4, o);
	for (c = 0; c < di.num_components; c++) {
		jpeg_component_info *k = &di.comp_info[c]; int h[4 + 64], i;
		h[0] = k->h_samp_factor; h[1] = k->v_samp_factor; h[2] = (int)k->width_in_blocks; h[3] = (int)k->height_in_blocks;
		for (i = 0; i < 64; i++) h[4 + i] = k->quant_table->quantval[i];
		fwrite(h, sizeof(int), 68, o);
	}
	for (c = 0; c < di.num_components; c++) {
		jpeg_component_info *k = &di.comp_info[c];
		for (y = 0; y < k->height_in_blocks; y++) {
			JBLOCKARRAY r = di.mem->access_virt_barray((j_common_ptr)&di, arr[c], y, 1, FALSE);
			fwrite(r[0], sizeof(JBLOCK), k->width_in_blocks, o);
		}
	}
	jpeg_finish_decompress(&di); jpeg_destroy_decompress(&di);
	fclose(f); fclose(o);
	return 0;
}

static int decode(const char *in, const char *out, const char *jpg) {
	FILE *f = fopen(in, "rb"), *o; int hdr[4], h[3][68], c; JDIMENSION y;
	struct jpeg_compress_struct co; struct jpeg_decompress_struct di; struct jpeg_error_mgr e1, e2;
	unsigned char *buf = NULL; unsigned long size = 0; jvirt_barray_ptr arr[3];
	if (!f) die("open");
	rd(hdr, sizeof(hdr), f);
	if (hdr[0] != 1 && hdr[0] != 3) die("1 or 3 components");
	for (c = 0; c < hdr[0]; c++) rd(h[c], sizeof(h[c]), f);
	co.err = jpeg_std_error(&e1);
	jpeg_create_compress(&co);
	jpeg_mem_dest(&co, &buf, &size);
	co.image_width = (JDIMENSION)hdr[2]; co.image_height = (JDIMENSION)hdr[3];
	co.input_components = hdr[0]; co.in_color_space = (J_COLOR_SPACE)hdr[1];
	jpeg_set_defaults(&co);
	jpeg_set_colorspace(&co, (J_COLOR_SPACE)hdr[1]);
	co.optimize_coding = TRUE;
	for (c = 0; c < hdr[0]; c++) {
		int i; JQUANT_TBL *t = jpeg_alloc_quant_table((j_common_ptr)&co);
		for (i = 0; i < 64; i++) t->quantval[i] = (UINT16)h[c][4 + i];
		t->sent_table = FALSE;
		co.quant_tbl_ptrs[c] = t;
		co.comp_info[c].quant_tbl_no = c;
		co.comp_info[c].h_samp_factor = h[c][0]; co.comp_info[c].v_samp_factor = h[c][1];
		/* rounded up to whole MCUs, as jdcoefct.c requests them: the encoder reads v_samp rows at a time */
		arr[c] = co.mem->request_virt_barray((j_common_ptr)&co, JPOOL_IMAGE, TRUE,
				(JDIMENSION)((h[c][2] + h[c][0] - 1) / h[c][0] * h[c][0]), (JDIMENSION)((h[c][3] + h[c][1] - 1) / h[c][1] * h[c][1]), h[c][1]);
	}
	{	/* an interleaved scan holds at most 10 blocks per MCU: more (3x3, 4x4 luma) go one scan per component */
		static jpeg_scan_info one[MAX_COMPS_IN_SCAN]; int n = 0;
		for (c = 0; c < hdr[0]; c++) n += h[c][0] * h[c][1];
		if (n > 10 && hdr[0] > 1 && hdr[0] <= MAX_COMPS_IN_SCAN) {
			for (c = 0; c < hdr[0]; c++) {
				one[c].comps_in_scan = 1; one[c].component_index[0] = c;
				one[c].Ss = 0; one[c].Se = 63; one[c].Ah = 0; one[c].Al = 0;
			}
			co.scan_info = one; co.num_scans = hdr[0];
		}
	}
	jpeg_write_coefficients(&co, arr);
	for (c = 0; c < hdr[0]; c++) {
		if ((int)co.comp_info[c].width_in_blocks != h[c][2] || (int)co.comp_info[c].height_in_blocks != h[c][3])
			die("block geometry differs from libjpeg's");
		for (y = 0; y < (JDIMENSION)h[c][3]; y++) {
			JBLOCKARRAY r = co.mem->access_virt_barray((j_common_ptr)&co, arr[c], y, 1, TRUE);
			rd(r[0], sizeof(JBLOCK) * (size_t)h[c][2], f);
		}
	}
	fclose(f);
	jpeg_finish_compress(&co); jpeg_destroy_compress(&co);
	if (jpg[0]) { FILE *j = fopen(jpg, "wb"); if (!j) die("open"); fwrite(buf, 1, size, j); fclose(j); }

	di.err = jpeg_std_error(&e2);
	jpeg_create_decompress(&di);
	jpeg_mem_src(&di, buf, size);
	jpeg_read_header(&di, TRUE);
	di.out_color_space = JCS_RGB; di.dct_method = JDCT_ISLOW; di.do_fancy_upsampling = TRUE;
	jpeg_start_decompress(&di);
	if (di.output_components != 3) die("not RGB");
	unsigned char *px = malloc((size_t)di.output_width * di.output_height * 3);
	while (di.output_scanline < di.output_height) {
		JSAMPROW r = px + (size_t)di.output_scanline * di.output_width * 3;
		jpeg_read_scanlines(&di, &r, 1);
	}
	jpeg_finish_decompress(&di); jpeg_destroy_decompress(&di);
	o = fopen(out, "wb");
	if (!o) die("open");
	fwrite(px, 3, (size_t)di.output_width * di.output_height, o);
	fclose(o); free(px); free(buf);
	return 0;
}

int main(int argc, char **argv) {
	if (argc >= 4 && !strcmp(argv[1], "dump")) return dump(argv[2], argv[3]);
	if (argc >= 4 && !strcmp(argv[1], "decode")) return decode(argv[2], argv[3], argc > 4 ? argv[4] : "");
	die("usage: pixels dump in.jpg out.bin | decode in.bin out.rgb [out.jpg]");
	return 2;
}
'''

_exe = None
_tmp = None


def _program() -> str:
    global _exe, _tmp
    if _exe is None:
        if JPEG_SO is None:
            raise LibjpegError("no libjpeg shared library inside Pillow")
        _tmp = tempfile.TemporaryDirectory(prefix="libjpeg_pixels_")
        src, exe = os.path.join(_tmp.name, "pixels.c"), os.path.join(_tmp.name, "pixels")
        with open(src, "w") as f:
            f.write(PROGRAM)
        subprocess.run(["/usr/bin/gcc", "-O1", "-I", os.path.join(ROOT, "include", "libjpeg62"), src, "-o", exe,
                        JPEG_SO, f"-Wl,-rpath,{os.path.dirname(JPEG_SO)}"], check=True)
        _exe = exe
    return _exe


def _run(*args):
    r = subprocess.run([_program(), *args], capture_output=True, text=True)
    if r.returncode:
        raise LibjpegError(f"libjpeg: {(r.stderr or r.stdout).strip()} (exit {r.returncode})")


def read_coefficients(path: str) -> CoefImage:
    """The coefficient set of a JPEG file, as jpeg_read_coefficients gives it."""
    with tempfile.TemporaryDirectory() as d:
        out = os.path.join(d, "c.bin")
        _run("dump", path, out)
        raw = open(out, "rb").read()
    hdr = np.frombuffer(raw, np.int32, 4)
    nc, cs, w, h = (int(v) for v in hdr)
    info = np.frombuffer(raw, np.int32, 68 * nc, 16).reshape(nc, 68)
    off = 16 + 68 * 4 * nc
    comps = []
    for c in range(nc):
        hs, vs, wb, hb = (int(v) for v in info[c, :4])
        coef = np.frombuffer(raw, np.int16, hb * wb * 64, off).reshape(hb, wb, 64).copy()
        off += coef.nbytes
        comps.append(Component(coef=coef, quant=info[c, 4:].astype(np.uint16), h_samp=hs, v_samp=vs,
                               quant_tbl_no=min(c, 1)))
    return CoefImage(width=w, height=h, colorspace=cs, comps=comps)


def decode(image: CoefImage, jpeg_path: str | None = None) -> np.ndarray:
    """libjpeg's JCS_RGB pixels [H, W, 3] uint8 for this coefficient set (components without a
    quant table are written with an all-ones table).  jpeg_path: also keep the file written."""
    nc = len(image.comps)
    parts = [np.array([nc, image.colorspace, image.width, image.height], np.int32).tobytes()]
    for c in image.comps:
        q = np.ones(64, np.int32) if c.quant is None else np.asarray(c.quant, np.int32)
        parts.append(np.concatenate([np.array([c.h_samp, c.v_samp, c.wblk, c.hblk], np.int32), q]).tobytes())
    for c in image.comps:
        parts.append(np.ascontiguousarray(c.coef, np.int16).tobytes())
    with tempfile.TemporaryDirectory() as d:
        src, out = os.path.join(d, "c.bin"), os.path.join(d, "px.rgb")
        with open(src, "wb") as f:
            f.write(b"".join(parts))
        _run("decode", src, out, jpeg_path or "")
        px = np.fromfile(out, np.uint8)
    return px.reshape(image.height, image.width, 3)


# ---- the renderers' arithmetic, restated -----------------------------------------------------

def _islow_1d(v, rnd):
    """reference idct.h islow butterfly along axis 0 of v (int64), RND folded into the even part"""
    z2, z3 = v[2], v[6]
    z1 = (z2 + z3) * 4433
    a, b = z1 - z3 * 15137, z1 + z2 * 6270
    t0, t1 = (v[0] + v[4]) * 8192 + rnd, (v[0] - v[4]) * 8192 + rnd
    e0, e3, e1, e2 = t0 + b, t0 - b, t1 + a, t1 - a
    t0, t1, t2, t3 = v[7], v[5], v[3], v[1]
    z1, z2, z3, z4 = t0 + t3, t1 + t2, t0 + t2, t1 + t3
    z5 = (z3 + z4) * 9633
    t0, t1, t2, t3 = t0 * 2446, t1 * 16819, t2 * 25172, t3 * 12299
    z1, z2, z3, z4 = z1 * 7373, z2 * 20995, z5 - z3 * 16069, z5 - z4 * 3196
    t0, t1, t2, t3 = t0 + z3 - z1, t1 + z4 - z2, t2 + z3 - z2, t3 + z4 - z1
    return np.stack([e0 + t3, e1 + t2, e2 + t1, e3 + t0, e3 - t0, e2 - t1, e1 - t2, e0 - t3])


def _plane(comp) -> np.ndarray:
    """islow IDCT of a component: [hblk * 8, wblk * 8] samples (int64)."""
    c = comp.coef.astype(np.int64).reshape(comp.hblk, comp.wblk, 8, 8)        # [by, bx, row, col]
    if comp.quant is not None and int(np.bitwise_or.reduce(comp.quant.astype(np.int64))) > 1:
        c = c * comp.quant.astype(np.int64).reshape(8, 8)
    ws = _islow_1d(np.moveaxis(c, 2, 0), 1024) >> 11                          # columns: [row, by, bx, col]
    px = _islow_1d(np.moveaxis(ws, 3, 0), 257 << 17) >> 18                   # rows: [col, row, by, bx]
    px = np.clip(px, 0, 255)
    return np.transpose(px, (2, 1, 3, 0)).reshape(comp.hblk * 8, comp.wblk * 8)


def _upsample(p, hs, vs, cw, ch, w, h):
    oy, ox = np.mgrid[0:h, 0:w]

    def at(x, y):
        return p[y, x]
    if hs == 1 and vs == 1:
        return at(ox, oy)
    if hs == 2 and vs == 1 and cw > 2:
        x = ox >> 1
        v = at(x, oy)
        odd = np.where(x == cw - 1, v, (v * 3 + at(np.minimum(x + 1, cw - 1), oy) + 2) >> 2)
        even = np.where(x == 0, v, (v * 3 + at(np.maximum(x - 1, 0), oy) + 1) >> 2)
        return np.where(ox & 1, odd, even)
    if hs == 2 and vs == 2 and cw > 2:
        x, y = ox >> 1, oy >> 1
        y1 = np.where(oy & 1, np.minimum(y + 1, ch - 1), np.maximum(y - 1, 0))
        cur = at(x, y) * 3 + at(x, y1)
        xr, xl = np.minimum(x + 1, cw - 1), np.maximum(x - 1, 0)
        odd = np.where(x == cw - 1, (cur * 4 + 7) >> 4, (cur * 3 + at(xr, y) * 3 + at(xr, y1) + 7) >> 4)
        even = np.where(x == 0, (cur * 4 + 8) >> 4, (cur * 3 + at(xl, y) * 3 + at(xl, y1) + 8) >> 4)
        return np.where(ox & 1, odd, even)
    if hs == 1 and vs == 2:
        y = oy >> 1
        y1 = np.where(oy & 1, np.minimum(y + 1, ch - 1), np.maximum(y - 1, 0))
        return (at(ox, y) * 3 + at(ox, y1) + np.where(oy & 1, 2, 1)) >> 2
    return at(np.minimum(ox // hs, cw - 1), np.minimum(oy // vs, ch - 1))


def device_model(image: CoefImage) -> np.ndarray:
    """The pixels the library's renderers compute for this coefficient set, [H, W, 3] uint8."""
    w, h, cs = image.width, image.height, image.comps
    maxh, maxv = max(c.h_samp for c in cs), max(c.v_samp for c in cs)
    s = []
    for c in cs:
        cw, ch = -(-w * c.h_samp // maxh), -(-h * c.v_samp // maxv)
        s.append(_upsample(_plane(c), maxh // c.h_samp, maxv // c.v_samp, cw, ch, w, h))
    if len(cs) == 1:
        s = [s[0]] * 3
    y, c1, c2 = s
    if image.colorspace == JCS_YCbCr and len(cs) == 3:
        cb, cr = c1 - 128, c2 - 128
        r = y + ((91881 * cr + 32768) >> 16)
        g = y + ((-22554 * cb + 32768 - 46802 * cr) >> 16)
        b = y + ((116130 * cb + 32768) >> 16)
        y, c1, c2 = (np.clip(v, 0, 255) for v in (r, g, b))
    return np.stack([y, c1, c2], -1).astype(np.uint8)
