"""Scaled-decode oracle: what libjpeg itself gives at scale_num 1, scale_denom d.

A small C program, built at first use against the libjpeg-turbo inside Pillow's wheel (declared by
include/libjpeg62, as tests/libjpeg_pixels.py does), decodes a JPEG file with jpeg_read_scanlines at
scale_num = 1, scale_denom = d, JDCT_ISLOW and fancy up-sampling, to JCS_RGB (JCS_GRAYSCALE for a grey
file), and reports each component's DCT_scaled_size as jpeg_start_decompress set it.

`decode_file` takes a file; `decode` takes a coefficient set, which libjpeg_pixels first writes with
jpeg_write_coefficients.  simd=False runs the library with JSIMD_FORCENONE=1, its C code paths only.
Nothing here touches a GPU.
"""
from __future__ import annotations

import os
import subprocess
import tempfile

import numpy as np

import libjpeg_pixels as lp
from jpegqs_b200.image import CoefImage

ROOT = lp.ROOT
JPEG_SO = lp.JPEG_SO
LibjpegError = lp.LibjpegError

PROGRAM = r'''
#include <stdio.h>
#include <stdlib.h>
#include <jpeglib.h>
/* output: int32 width, height, channels, ncomp, DCT_scaled_size[ncomp]; then the scanlines */
int main(int argc, char **argv) {
	struct jpeg_decompress_struct di; struct jpeg_error_mgr err;
	FILE *f, *o; int c, hdr[4]; unsigned char *px;
	if (argc != 4) { fprintf(stderr, "usage: scaled in.jpg d out.bin\n"); return 2; }
	f = fopen(argv[1], "rb"); o = fopen(argv[3], "wb");
	if (!f || !o) { fprintf(stderr, "open\n"); return 2; }
	di.err = jpeg_std_error(&err);
	jpeg_create_decompress(&di);
	jpeg_stdio_src(&di, f);
	jpeg_read_header(&di, TRUE);
	di.scale_num = 1; di.scale_denom = (unsigned)atoi(argv[2]);
	di.dct_method = JDCT_ISLOW; di.do_fancy_upsampling = TRUE;
	di.out_color_space = di.num_components == 1 ? JCS_GRAYSCALE : JCS_RGB;
	jpeg_start_decompress(&di);
	hdr[0] = (int)di.output_width; hdr[1] = (int)di.output_height; hdr[2] = di.output_components; hdr[3] = di.num_components;
	fwrite(hdr, sizeof(int), 4, o);
	for (c = 0; c < di.num_components; c++) fwrite(&di.comp_info[c].DCT_scaled_size, sizeof(int), 1, o);
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
'''

_exe = None
_tmp = None


def _program() -> str:
    global _exe, _tmp
    if _exe is None:
        if JPEG_SO is None:
            raise LibjpegError("no libjpeg shared library inside Pillow")
        _tmp = tempfile.TemporaryDirectory(prefix="libjpeg_scaled_")
        src, exe = os.path.join(_tmp.name, "scaled.c"), os.path.join(_tmp.name, "scaled")
        with open(src, "w") as f:
            f.write(PROGRAM)
        subprocess.run(["/usr/bin/gcc", "-O1", "-I", os.path.join(ROOT, "include", "libjpeg62"), src, "-o", exe,
                        JPEG_SO, f"-Wl,-rpath,{os.path.dirname(JPEG_SO)}"], check=True)
        _exe = exe
    return _exe


def decode_file(path: str, d: int, simd: bool = True):
    """(pixels [H', W', C] uint8, [DCT_scaled_size per component]) of libjpeg's decode of a JPEG file at
    scale 1/d; C = 1 for a grey file, 3 otherwise."""
    env = dict(os.environ)
    env.pop("JSIMD_FORCENONE", None)
    if not simd:
        env["JSIMD_FORCENONE"] = "1"
    with tempfile.TemporaryDirectory() as tmp:
        out = os.path.join(tmp, "px.bin")
        r = subprocess.run([_program(), path, str(int(d)), out], capture_output=True, text=True, env=env)
        if r.returncode:
            raise LibjpegError(f"libjpeg: {(r.stderr or r.stdout).strip()} (exit {r.returncode})")
        raw = open(out, "rb").read()
    w, h, ch, nc = (int(v) for v in np.frombuffer(raw, np.int32, 4))
    sizes = [int(v) for v in np.frombuffer(raw, np.int32, nc, 16)]
    px = np.frombuffer(raw, np.uint8, w * h * ch, 16 + 4 * nc).reshape(h, w, ch)
    return px, sizes


def decode_bytes(data: bytes, d: int, simd: bool = True):
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "in.jpg")
        with open(path, "wb") as f:
            f.write(data)
        return decode_file(path, d, simd)


def decode(image: CoefImage, d: int, simd: bool = True):
    """decode_file of the file jpeg_write_coefficients writes for this coefficient set (libjpeg_pixels'
    writer: its own quant table per component, all ones for a component without one)."""
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "c.jpg")
        lp.decode(image, jpeg_path=path)
        return decode_file(path, d, simd)
