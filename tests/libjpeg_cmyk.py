"""libjpeg itself for 4-component files: writing a coefficient set in its colour space, and decoding a file at
scale 1/d with JCS_CMYK output (libjpeg-turbo has no CMYK -> RGB conversion).

A small C program, built at first use against the libjpeg-turbo inside Pillow's wheel (declared by
include/libjpeg62, as tests/libjpeg_pixels.py does):
  - `write` is jpeg_write_coefficients of a coefficient set with 1, 3 or 4 components, its own quant table
    per component, jpeg_set_colorspace(colorspace) - so a JCS_YCCK set gets libjpeg's Adobe marker with
    transform 2 and a JCS_CMYK one transform 0 - and optimized Huffman tables;
  - `decode` is jpeg_read_scanlines at scale_num 1, scale_denom d, JDCT_ISLOW and fancy up-sampling, to
    JCS_CMYK for a 4-component file (a YCCK file's samples through ycck_cmyk_convert), JCS_GRAYSCALE for a
    grey one and JCS_RGB otherwise.
Nothing here touches a GPU."""
from __future__ import annotations

import os
import subprocess
import tempfile

import numpy as np

import libjpeg_pixels as lp
from jpegqs_b200.image import CoefImage

LibjpegError = lp.LibjpegError

PROGRAM = r'''
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <jpeglib.h>
/* coefficient file: int32 ncomp, color_space, width, height; per component int32 h_samp, v_samp, wblk, hblk,
 * quant[64]; then per component int16 [hblk][wblk][64] */
static void die(const char *m) { fprintf(stderr, "%s\n", m); exit(2); }
static void rd(void *p, size_t n, FILE *f) { if (fread(p, 1, n, f) != n) die("short read"); }

static int write_coefs(const char *in, const char *out) {
	FILE *f = fopen(in, "rb"), *o = fopen(out, "wb"); int hdr[4], h[4][68], c; JDIMENSION y;
	struct jpeg_compress_struct co; struct jpeg_error_mgr e; jvirt_barray_ptr arr[4];
	if (!f || !o) die("open");
	rd(hdr, sizeof(hdr), f);
	if (hdr[0] != 1 && hdr[0] != 3 && hdr[0] != 4) die("1, 3 or 4 components");
	for (c = 0; c < hdr[0]; c++) rd(h[c], sizeof(h[c]), f);
	co.err = jpeg_std_error(&e);
	jpeg_create_compress(&co);
	jpeg_stdio_dest(&co, o);
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
		arr[c] = co.mem->request_virt_barray((j_common_ptr)&co, JPOOL_IMAGE, TRUE,
				(JDIMENSION)((h[c][2] + h[c][0] - 1) / h[c][0] * h[c][0]), (JDIMENSION)((h[c][3] + h[c][1] - 1) / h[c][1] * h[c][1]), h[c][1]);
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
	fclose(o);
	return 0;
}

/* output: int32 width, height, channels; then the scanlines */
static int decode(const char *in, int d, const char *out) {
	struct jpeg_decompress_struct di; struct jpeg_error_mgr err;
	FILE *f = fopen(in, "rb"), *o = fopen(out, "wb"); int hdr[3]; unsigned char *px;
	if (!f || !o) die("open");
	di.err = jpeg_std_error(&err);
	jpeg_create_decompress(&di);
	jpeg_stdio_src(&di, f);
	jpeg_read_header(&di, TRUE);
	di.scale_num = 1; di.scale_denom = (unsigned)d;
	di.dct_method = JDCT_ISLOW; di.do_fancy_upsampling = TRUE;
	di.out_color_space = di.num_components == 4 ? JCS_CMYK : di.num_components == 1 ? JCS_GRAYSCALE : JCS_RGB;
	jpeg_start_decompress(&di);
	hdr[0] = (int)di.output_width; hdr[1] = (int)di.output_height; hdr[2] = di.output_components;
	fwrite(hdr, sizeof(int), 3, o);
	px = malloc((size_t)di.output_width * di.output_height * di.output_components);
	while (di.output_scanline < di.output_height) {
		JSAMPROW r = px + (size_t)di.output_scanline * di.output_width * di.output_components;
		jpeg_read_scanlines(&di, &r, 1);
	}
	fwrite(px, 1, (size_t)di.output_width * di.output_height * di.output_components, o);
	jpeg_finish_decompress(&di); jpeg_destroy_decompress(&di);
	fclose(f); fclose(o); free(px);
	return 0;
}

int main(int argc, char **argv) {
	if (argc == 4 && !strcmp(argv[1], "write")) return write_coefs(argv[2], argv[3]);
	if (argc == 5 && !strcmp(argv[1], "decode")) return decode(argv[2], atoi(argv[3]), argv[4]);
	die("usage: cmyk write in.bin out.jpg | decode in.jpg d out.bin");
	return 2;
}
'''

_exe = None
_tmp = None


def _program() -> str:
    global _exe, _tmp
    if _exe is None:
        if lp.JPEG_SO is None:
            raise LibjpegError("no libjpeg shared library inside Pillow")
        _tmp = tempfile.TemporaryDirectory(prefix="libjpeg_cmyk_")
        src, exe = os.path.join(_tmp.name, "cmyk.c"), os.path.join(_tmp.name, "cmyk")
        with open(src, "w") as f:
            f.write(PROGRAM)
        subprocess.run(["/usr/bin/gcc", "-O1", "-I", os.path.join(lp.ROOT, "include", "libjpeg62"), src, "-o", exe,
                        lp.JPEG_SO, f"-Wl,-rpath,{os.path.dirname(lp.JPEG_SO)}"], check=True)
        _exe = exe
    return _exe


def _run(*args):
    r = subprocess.run([_program(), *args], capture_output=True, text=True)
    if r.returncode:
        raise LibjpegError(f"libjpeg: {(r.stderr or r.stdout).strip()} (exit {r.returncode})")


def write_coefficients(image: CoefImage) -> bytes:
    """the file jpeg_write_coefficients makes of a coefficient set, in image.colorspace"""
    parts = [np.array([len(image.comps), image.colorspace, image.width, image.height], np.int32).tobytes()]
    for c in image.comps:
        q = np.ones(64, np.int32) if c.quant is None else np.asarray(c.quant, np.int32)
        parts.append(np.concatenate([np.array([c.h_samp, c.v_samp, c.wblk, c.hblk], np.int32), q]).tobytes())
    for c in image.comps:
        parts.append(np.ascontiguousarray(c.coef, np.int16).tobytes())
    with tempfile.TemporaryDirectory() as d:
        src, out = os.path.join(d, "c.bin"), os.path.join(d, "c.jpg")
        with open(src, "wb") as f:
            f.write(b"".join(parts))
        _run("write", src, out)
        with open(out, "rb") as f:
            return f.read()


def decode_bytes(data: bytes, d: int) -> np.ndarray:
    """libjpeg's decode of a file at scale 1/d: [H', W', C], C = 4 (libjpeg's CMYK, not inverted) for a
    4-component file, 1 for a grey one, 3 otherwise"""
    with tempfile.TemporaryDirectory() as tmp:
        path, out = os.path.join(tmp, "in.jpg"), os.path.join(tmp, "px.bin")
        with open(path, "wb") as f:
            f.write(data)
        _run("decode", path, str(int(d)), out)
        raw = open(out, "rb").read()
    w, h, ch = (int(v) for v in np.frombuffer(raw, np.int32, 3))
    return np.frombuffer(raw, np.uint8, w * h * ch, 12).reshape(h, w, ch)
