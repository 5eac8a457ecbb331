"""The libjpeg-facing half meets a REAL libjpeg: Pillow's wheel carries libjpeg-turbo 3.1
(libjpeg API/ABI 6.2, no headers); include/libjpeg62/jpeglib.h declares that API by hand and the
shipped library is compiled against it.

CPU leg: the hand-declared structs are accepted by the real library (its own struct-size /
version check) and a real decode through them gives the coefficients csrc/jpegcoef.c reads;
the lossless transcodes of random files are libjpeg-turbo's bytes.
GPU leg: the reference's CLI on real libjpeg wrote (SHA-256 stored in tests/golden/reference/ref_files.json)
the very bytes this repository's tool writes; and the reference's OWN callers run on the CUDA back end with real libjpeg -
oracle/_ref/refcli_b200 is the unmodified reference quantsmooth.c whose SIMD dispatcher links
the tier workers exported by libjpegqs_b200.so; example_b200 is the reference's example.c
(jpegqs_start_decompress -> jpeg_read_scanlines) - and must reproduce the all-CPU builds of the
same sources (refcli_cpu / example_cpu) byte for byte.  Those two need the reference's sources
(oracle/Makefile builds them into oracle/_ref when they are at hand) and skip without them."""
import glob
import os
import subprocess

import numpy as np
import pytest

PIL = pytest.importorskip("PIL.Image")
import PIL as _PIL  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "jpeg-quantsmooth_b200", "csrc")
REFDIR = os.path.join(ROOT, "oracle", "_ref")
_so = sorted(glob.glob(os.path.join(os.path.dirname(os.path.realpath(_PIL.__file__)), "..", "pillow.libs", "libjpeg*.so*")))
JPEG_SO = os.path.realpath(_so[0]) if _so else None
pytestmark = pytest.mark.skipif(JPEG_SO is None, reason="no libjpeg shared library inside Pillow")

from test_cli import EXE, _picture, file_key, sha256, write_jpegs  # noqa: E402


def write_mcu_jpegs(d):
    # sizes that are multiples of the MCU: the reference's UPSAMPLE_UV reads uninitialised memory
    # otherwise (DESIGN.md "reference quirks"), so q6 is compared on these only
    out = {}
    for name, w, h, kw in (("mcu420", 192, 144, dict(quality=60)), ("mcuprog", 256, 160, dict(quality=85, progressive=True)),
                           ("mcu422", 160, 96, dict(quality=40, subsampling=1))):
        p = os.path.join(d, name + ".jpg")
        _picture(w, h, False, 11).save(p, **kw)
        out[name] = p
    return out


@pytest.fixture(scope="module")
def jpegs(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("real"))
    out = write_jpegs(d)
    out.update(write_mcu_jpegs(d))
    return out


DUMP = r'''
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <jpeglib.h>
#ifdef USE_JQ
#include "jpegcoef.h"
#endif
static void dump(struct jpeg_decompress_struct *ci, jvirt_barray_ptr *arr) {
	int c;
	printf("%ux%u %d cs%d\n", ci->image_width, ci->image_height, ci->num_components, (int)ci->jpeg_color_space);
	for (c = 0; c < ci->num_components; c++) {
		jpeg_component_info *k = &ci->comp_info[c]; unsigned long h = 1469598103934665603ul; JDIMENSION y, x; int i;
		for (y = 0; y < k->height_in_blocks; y++) {
			JBLOCKARRAY r = ci->mem->access_virt_barray((j_common_ptr)ci, arr[c], y, 1, FALSE);
			for (x = 0; x < k->width_in_blocks; x++) for (i = 0; i < 64; i++) h = (h ^ (unsigned short)r[0][x][i]) * 1099511628211ul;
		}
		for (i = 0; i < 64; i++) h = (h ^ k->quant_table->quantval[i]) * 1099511628211ul;
		printf("%d: %dx%d t%d %ux%u %lx\n", c, k->h_samp_factor, k->v_samp_factor, k->quant_tbl_no, k->width_in_blocks, k->height_in_blocks, h);
	}
}
int main(int argc, char **argv) {
	(void)argc;
#ifdef USE_JQ
	FILE *f = fopen(argv[1], "rb"); static unsigned char buf[1 << 22]; size_t n = fread(buf, 1, sizeof(buf), f);
	jq_image im; char err[256];
	if (jq_read(buf, n, 2, &im, err)) { puts(err); return 1; }
	dump(&im.cinfo, im.coef_arrays);
#else
	struct jpeg_decompress_struct ci; struct jpeg_error_mgr err; FILE *f = fopen(argv[1], "rb");
	ci.err = jpeg_std_error(&err);
	jpeg_create_decompress(&ci);          /* the real library checks sizeof(ci) and the version here */
	jpeg_stdio_src(&ci, f);
	jpeg_read_header(&ci, TRUE);
	dump(&ci, jpeg_read_coefficients(&ci));
	{ struct jpeg_compress_struct co; co.err = jpeg_std_error(&err); jpeg_create_compress(&co); jpeg_destroy_compress(&co); }
#endif
	return 0;
}
'''


def test_declared_abi_is_the_real_librarys_and_both_codecs_agree(jpegs, tmp_path):
    src = tmp_path / "dump.c"
    src.write_text(DUMP)
    inc = ["-I", os.path.join(ROOT, "include", "libjpeg62"), "-I", os.path.join(ROOT, "include"), "-I", CSRC]
    real, ours = str(tmp_path / "dump_real"), str(tmp_path / "dump_jq")
    subprocess.run(["/usr/bin/gcc", "-O1"] + inc + [str(src), "-o", real, JPEG_SO, f"-Wl,-rpath,{os.path.dirname(JPEG_SO)}"], check=True)
    subprocess.run(["/usr/bin/gcc", "-O1", "-DUSE_JQ"] + inc + [str(src), os.path.join(CSRC, "jpegcoef.c"), "-o", ours, "-lpthread"], check=True)
    for name, path in jpegs.items():
        a = subprocess.run([real, path], capture_output=True, text=True)
        b = subprocess.run([ours, path], capture_output=True, text=True)
        assert a.returncode == 0 and b.returncode == 0, (name, a.stderr, b.stdout)
        assert a.stdout == b.stdout, name


def _have(*names):
    return all(os.path.exists(os.path.join(REFDIR, n)) for n in names)


# -q 2 is LOW_QUALITY with UPSAMPLE_UV: on 4:2:0 files whose width is not a multiple of the MCU
# (prog420, rst) the reference pads the up-sampled plane from uninitialised memory (DESIGN.md
# "reference quirks"), so those two pairs have no defined answer to compare with
REF_CLI_CASES = [(name, args) for name in ("base420", "gray", "prog420", "opt422", "rst")
                 for args in (["-q", "3", "-n", "2"], ["-q", "4", "-n", "1", "-o"], ["-q", "2"])
                 if not (args == ["-q", "2"] and name in ("prog420", "rst"))]
CODEC_DIFFTEST_RUNS = [(77, 30)]


@pytest.mark.gpu
def test_reference_cli_on_real_libjpeg_writes_this_codecs_bytes(jpegs, tmp_path):
    """quantsmooth.c + libjpeg-turbo vs the same smoothing behind csrc/jpegcoef.c + jpegqs.c:
    the files are byte-identical, i.e. the codec reproduces jpeg_copy_critical_parameters +
    jpeg_write_coefficients + jcopy_markers (JFIF / Adobe handling included)."""
    from golden_io import reference_files
    want = reference_files()["refcli_cpu"]
    for name, args in REF_CLI_CASES:
        b = str(tmp_path / "jq.jpg")
        r = subprocess.run([EXE, "-i", "0"] + args + [jpegs[name], b], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        assert sha256(b) == want[file_key(name, args)], (name, args)


def test_random_files_one_thread_threaded_and_libjpeg_turbo_agree(tmp_path):
    """A short run of tools/codec_difftest.py: random size / quality / sub-sampling / optimised tables /
    restart intervals / progressive files; the lossless transcode must give libjpeg-turbo's bytes with the
    one-thread reader and with the threaded reader (random thread count and chunk size)."""
    seed, n = CODEC_DIFFTEST_RUNS[0]
    r = subprocess.run([os.sys.executable, os.path.join(ROOT, "tools", "codec_difftest.py"), str(seed), str(n)], cwd=str(tmp_path),
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert f"done {n} bad 0" in r.stdout, r.stdout[-2000:]


@pytest.mark.gpu
@pytest.mark.skipif(not _have("refcli_cpu", "refcli_b200"), reason="oracle/_ref not built")
@pytest.mark.parametrize("args", [["-q", "3"], ["-q", "4", "-n", "2"], ["-q", "5", "-n", "2"], ["-q", "6"], ["-q", "1"], ["-q", "3", "-o"]])
def test_unmodified_reference_cli_runs_on_the_cuda_back_end(jpegs, tmp_path, args):
    # each file costs a fresh process with its CUDA start-up: the flavours are spread over the argument sets
    # (q6 on MCU-multiple sizes only, see the fixture)
    names = {"-q 3": ("base420", "prog420", "gray", "rst"), "-q 4 -n 2": ("prog420", "opt422", "base444"),
             "-q 5 -n 2": ("base420", "mcu420", "base444"), "-q 6": ("mcu420", "mcuprog", "mcu422"),
             "-q 1": ("gray", "opt422", "rst"), "-q 3 -o": ("base420", "prog420", "opt422")}[" ".join(args)]
    for name in names:
        a, b = str(tmp_path / "cpu.jpg"), str(tmp_path / "b200.jpg")
        r1 = subprocess.run([os.path.join(REFDIR, "refcli_cpu"), "-i", "0"] + args + [jpegs[name], a], capture_output=True, text=True)
        r2 = subprocess.run([os.path.join(REFDIR, "refcli_b200"), "-i", "16"] + args + [jpegs[name], b], capture_output=True, text=True)
        assert r1.returncode == 0 and r2.returncode == 0, (r1.stderr, r2.stderr)
        assert "CUDA sm_90a" in r2.stderr, r2.stderr            # it really went through the tier slot into the GPU
        assert open(a, "rb").read() == open(b, "rb").read(), (name, args)


@pytest.mark.gpu
@pytest.mark.skipif(not _have("example_cpu", "example_b200"), reason="oracle/_ref not built")
def test_reference_example_decodes_through_the_helpers_on_the_cuda_back_end(jpegs, tmp_path):
    """example.c: jpeg_read_header -> jpegqs_start_decompress (q6, n3, progress callback) ->
    jpeg_read_scanlines -> jpegqs_finish_decompress -> BMP, with real libjpeg doing the IDCT /
    colour conversion after the re-armed decoder (quantsmooth.h:2861-2876).  Same pixels, same
    progress lines as the all-CPU build; and the device renderer (jpegqs --ppm) gives them too."""
    exe = os.path.join(CSRC, "jpegqs")
    for name in ("mcu420", "mcuprog", "mcu422", "gray", "base444"):
        a, b = str(tmp_path / "cpu.bmp"), str(tmp_path / "b200.bmp")
        r1 = subprocess.run([os.path.join(REFDIR, "example_cpu"), jpegs[name], a], capture_output=True, text=True)
        r2 = subprocess.run([os.path.join(REFDIR, "example_b200"), jpegs[name], b], capture_output=True, text=True)
        assert r1.returncode == 0 and r2.returncode == 0, (r1.stderr, r2.stderr)
        assert r1.stdout == r2.stdout, name                       # the progress callback sequence
        assert open(a, "rb").read() == open(b, "rb").read(), name
        ppm = str(tmp_path / "dev.ppm")
        assert subprocess.run([exe, "-q", "6", "-i", "0", "--ppm", jpegs[name], ppm]).returncode == 0
        assert np.array_equal(np.asarray(PIL.open(ppm).convert("RGB")), np.asarray(PIL.open(a).convert("RGB"))), name
