"""JPEG files of many scan scripts for the scan decoder tests (parse_jpeg_scans / decode_scans_model /
decode_scans_async).

Pillow writes libjpeg-turbo's default progressive script; custom scripts are written by a small C
program, built at first use against the libjpeg-turbo inside Pillow's wheel (as libjpeg_pixels.py
does), that reads a file's coefficients with jpeg_read_coefficients and writes them again with
jpeg_write_coefficients under a jpeg_scan_info script and restart interval of our choosing."""
from __future__ import annotations

import os
import subprocess
import tempfile

import numpy as np

import decode_files as df
import libjpeg_pixels as lp

PROGRAM = r'''
#include <stdio.h>
#include <stdlib.h>
#include <jpeglib.h>
/* rescan in.jpg out.jpg script.bin: script = int32 nscans, restart_interval, restart_rows, optimize,
 * then per scan int32 ncomp, comp[4], Ss, Se, Ah, Al (nscans 0: sequential, one scan) */
int main(int argc, char **argv) {
	struct jpeg_decompress_struct di; struct jpeg_compress_struct co; struct jpeg_error_mgr e1, e2;
	FILE *f, *o, *s; int hdr[4], i, k; jpeg_scan_info *sc = NULL;
	if (argc != 4 || !(f = fopen(argv[1], "rb")) || !(s = fopen(argv[3], "rb"))) return 2;
	if (fread(hdr, 4, 4, s) != 4) return 2;
	if (hdr[0]) {
		sc = calloc((size_t)hdr[0], sizeof(*sc));
		for (i = 0; i < hdr[0]; i++) {
			int r[9];
			if (fread(r, 4, 9, s) != 9) return 2;
			sc[i].comps_in_scan = r[0];
			for (k = 0; k < 4; k++) sc[i].component_index[k] = r[1 + k];
			sc[i].Ss = r[5]; sc[i].Se = r[6]; sc[i].Ah = r[7]; sc[i].Al = r[8];
		}
	}
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
	co.restart_interval = (unsigned)hdr[1]; co.restart_in_rows = hdr[2]; co.optimize_coding = hdr[3] != 0;
	if (sc) { co.scan_info = sc; co.num_scans = hdr[0]; }
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
        _tmp = tempfile.TemporaryDirectory(prefix="scan_files_")
        src, exe = os.path.join(_tmp.name, "rescan.c"), os.path.join(_tmp.name, "rescan")
        with open(src, "w") as f:
            f.write(PROGRAM)
        subprocess.run(["/usr/bin/gcc", "-O1", "-I", os.path.join(lp.ROOT, "include", "libjpeg62"), src, "-o", exe,
                        lp.JPEG_SO, f"-Wl,-rpath,{os.path.dirname(lp.JPEG_SO)}"], check=True)
        _exe = exe
    return _exe


def rescan(data: bytes, script=None, restart_interval: int = 0, restart_rows: int = 0, optimize: bool = True) -> bytes:
    """data's coefficients written again by libjpeg under a scan script: a list of (components, Ss,
    Se, Ah, Al) with components a tuple of frame component indices; None: one sequential scan."""
    script = script or []
    words = [len(script), restart_interval, restart_rows, int(optimize)]
    for comps, ss, se, ah, al in script:
        words += [len(comps), *(list(comps) + [0] * (4 - len(comps))), ss, se, ah, al]
    with tempfile.TemporaryDirectory() as d:
        i, o, s = (os.path.join(d, n) for n in ("i.jpg", "o.jpg", "s.bin"))
        open(i, "wb").write(data)
        open(s, "wb").write(np.array(words, np.int32).tobytes())
        r = subprocess.run([_program(), i, o, s], capture_output=True, text=True)
        if r.returncode:
            raise lp.LibjpegError(f"libjpeg: {(r.stderr or r.stdout).strip()} (exit {r.returncode})")
        return open(o, "rb").read()


def per_component_sequential(nc):
    return [((c,), 0, 63, 0, 0) for c in range(nc)]


def spectral_only(nc):
    s = [(tuple(range(nc)), 0, 0, 0, 0)]
    for c in range(nc):
        s += [((c,), 1, 5, 0, 0), ((c,), 6, 63, 0, 0)]
    return s


def successive(nc):
    """DC and AC successive approximation down from Al = 3."""
    s = [(tuple(range(nc)), 0, 0, 0, 3)]
    for c in range(nc):
        s.append(((c,), 1, 63, 0, 3))
    for al in (2, 1, 0):
        s.append((tuple(range(nc)), 0, 0, al + 1, al))
        for c in range(nc):
            s.append(((c,), 1, 63, al + 1, al))
    return s


def dc_per_component(nc):
    s = [((c,), 0, 0, 0, 1) for c in range(nc)]
    s += [((c,), 1, 63, 0, 1) for c in range(nc)]
    s += [((c,), 0, 0, 1, 0) for c in range(nc)]
    s += [((c,), 1, 63, 1, 0) for c in range(nc)]
    return s


def split_bands(nc):
    """bands 1-2 / 3-9 / 10-63 first at Al = 1 and refined, the refinements in a different split."""
    s = [(tuple(range(nc)), 0, 0, 0, 1)]
    for c in range(nc):
        s += [((c,), 1, 2, 0, 1), ((c,), 3, 9, 0, 1), ((c,), 10, 63, 0, 1)]
    s.append((tuple(range(nc)), 0, 0, 1, 0))
    for c in range(nc):
        s += [((c,), 1, 9, 1, 0), ((c,), 10, 63, 1, 0)]
    return s


SCRIPTS = {"seq_per_comp": per_component_sequential, "spectral": spectral_only, "succ_al3": successive,
           "dc_per_comp": dc_per_component, "split_bands": split_bands}


def flat(w: int, h: int, mode: str = "RGB") -> bytes:
    """Nearly flat content: long end-of-band runs in every AC scan."""
    from PIL import Image
    import io
    yy, xx = np.mgrid[0:h, 0:w]
    base = (100 + (xx // 64) * 3 + (yy // 64) * 2).astype(np.uint8)
    im = Image.fromarray(np.stack([base, base // 2 + 40, 200 - base], -1)) if mode == "RGB" else Image.fromarray(base)
    b = io.BytesIO()
    im.save(b, "JPEG", quality=50, progressive=True)
    return b.getvalue()


def pillow_progressive():
    """(name, bytes) of Pillow progressive files: samplings, grey, CMYK, keep_rgb, sizes, restarts."""
    out = []
    for ss, sub in (("420", 2), ("422", 1), ("444", 0)):
        out.append((f"prog_{ss}", df.pillow_jpeg(250, 190, subsampling=sub, quality=80, progressive=True, seed=3)))
    out.append(("prog_gray", df.pillow_jpeg(97, 61, "L", quality=75, progressive=True)))
    out.append(("prog_cmyk", df.pillow_jpeg(120, 80, "CMYK", quality=85, progressive=True)))
    out.append(("prog_keep_rgb", df.pillow_jpeg(120, 80, quality=90, keep_rgb=True, subsampling=0, progressive=True)))
    for w, h in ((1, 1), (17, 9), (250, 190)):
        out.append((f"prog_size_{w}x{h}", df.pillow_jpeg(w, h, quality=85, progressive=True, seed=w)))
    out.append(("prog_rst_blocks5", df.pillow_jpeg(250, 190, quality=75, progressive=True, restart_marker_blocks=5)))
    out.append(("prog_rst_rows1", df.pillow_jpeg(250, 190, quality=75, progressive=True, restart_marker_rows=1)))
    out.append(("prog_opt", df.pillow_jpeg(203, 149, quality=85, progressive=True, optimize=True)))
    return out


def scripted():
    """(name, bytes) of libjpeg files under the custom scripts, 4:2:0 colour and grey, with and
    without restart markers."""
    base = {"420": df.pillow_jpeg(131, 77, quality=88, subsampling=2, seed=11),
            "gray": df.pillow_jpeg(90, 70, "L", quality=92, seed=5)}
    out = []
    for name, fn in SCRIPTS.items():
        for kind, data in base.items():
            nc = 1 if kind == "gray" else 3
            out.append((f"{name}_{kind}", rescan(data, fn(nc))))
            out.append((f"{name}_{kind}_rst3", rescan(data, fn(nc), restart_interval=3)))
    out.append(("flat_prog", flat(256, 160)))
    out.append(("flat_rst2", rescan(flat(256, 160), successive(3), restart_interval=2)))
    out.append(("flat_gray_rst7", rescan(flat(200, 120, "L"), successive(1), restart_interval=7)))
    out.append(("seq_multi_rst", rescan(base["420"], per_component_sequential(3), restart_interval=4)))
    return out


def hard_progressive():
    """The hard_content sets re-encoded progressive, with successive approximation and split bands."""
    out = []
    for name, im, data in df.hard_sets():
        nc = len(im.comps)
        try:
            out.append((f"hard_{name}", rescan(data, successive(nc) if nc == 1 else split_bands(nc))))
        except lp.LibjpegError:
            continue
    return out


def geometry_progressive():
    """decode_files.geometry_files re-encoded progressive: successive approximation and split bands,
    with and without restart markers."""
    out = []
    for name, data in df.geometry_files():
        if name.endswith(("_rst7", "_rows1")):
            continue
        g = name[len("writer_"):]
        nc = 1 if g.startswith("g") else 3
        out.append((f"succ_{g}", rescan(data, successive(nc))))
        out.append((f"succ_{g}_rst3", rescan(data, successive(nc), restart_interval=3)))
        out.append((f"split_{g}", rescan(data, split_bands(nc))))
        out.append((f"split_{g}_rst5", rescan(data, split_bands(nc), restart_interval=5)))
    return out
