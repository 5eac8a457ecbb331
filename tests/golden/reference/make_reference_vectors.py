"""Generates the reference's answers that the tests compare against, from the UNMODIFIED
reference built into oracle/_ref by oracle/Makefile:

    python tests/golden/reference/make_reference_vectors.py

  ref_kernels.npz     islow IDCT, float FDCT / IDCT and weight tables of the reference on the
                      seeded inputs of tests/test_oracle_vs_reference.py
  ref_driver.npz      the reference's do_quantsmooth results (return value, coefficients,
  ref_sweep.npz       sampling factors, quant tables, progress sequences) for every case of
                      tests/test_oracle_vs_reference.py and tests/test_gpu_edge.py (two files
                      to keep each under 1 MB)
  ref_files.json      SHA-256 of the files the reference tools write for the JPEG files the
                      CLI tests generate (tests/test_cli.py, tests/test_real_libjpeg.py) and of
                      the lossless transcodes of tools/codec_difftest.py
  ref_saturated.npz   the reference's results on small saturated-content images
                      (the sampling geometries of tests/hard_content.py FACTORS: synthetic
                      content in ref_driver.npz, grey ones in ref_sweep.npz, saturated
                      content here)
  ref_saturated.json  golden_io.result_digest of its results on wave-scale saturated-content
                      images (tests/hard_content.py; tests/test_oracle_vs_reference.py)

An archive is only rewritten when its arrays change (numpy stamps each member with the time it
was written), so regenerating leaves unchanged files byte-identical.  Name parts to regenerate
only those: kernels, driver, files, saturated.

Inputs are not stored: every test regenerates them from its seed (numpy RandomState, Pillow).
"""
import hashlib
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import jpegqs_b200 as qs          # noqa: E402
import oracle_lib as ol           # noqa: E402
import golden_io as gio           # noqa: E402
REFDIR = os.path.join(ROOT, "oracle", "_ref")


def _save_npz(path, d):
    if os.path.exists(path):
        with np.load(path) as z:
            if sorted(z.files) == sorted(d) and all(np.array_equal(z[k], np.asarray(d[k])) and
                                                    z[k].dtype == np.asarray(d[k]).dtype for k in d):
                return
    np.savez_compressed(path, **d)


def kernels():
    ref = ol.reflib()
    d = {}
    rng = np.random.RandomState(1)
    idct = []
    for scale in (8, 200, 2047):
        for _ in range(200):
            c = rng.randint(-scale, scale + 1, size=64).astype(np.int16)
            if rng.rand() < 0.3:
                c[rng.rand(64) < 0.8] = 0
            a = np.zeros((8, 24), dtype=np.uint8)
            ref.qsref_idct_islow(c.ctypes.data, a.ctypes.data, 24)
            idct.append(a)
    d["idct_islow"] = np.stack(idct)
    rng = np.random.RandomState(2)
    fd, fi = [], []
    for _ in range(300):
        x = (rng.rand(64).astype(np.float32) - 0.5) * np.float32(rng.choice([1, 255, 4096]))
        for fn, acc in ((ref.qsref_fdct_float, fd), (ref.qsref_idct_float, fi)):
            a = np.zeros(64, dtype=np.float32)
            xa = x.copy()
            fn(xa.ctypes.data, a.ctypes.data)
            acc.append(a)
    d["fdct_float"], d["idct_float"] = np.stack(fd), np.stack(fi)
    for flags, size in ((0, 160), (1, 272)):
        a = np.zeros((64, size), dtype=np.float32)
        assert ref.qsref_tables(flags, a.ctypes.data) == size
        d[f"tables{flags}"] = a
    _save_npz(os.path.join(HERE, "ref_kernels.npz"), d)


def driver():
    import test_oracle_vs_reference as tv
    import test_gpu_edge as te
    d, e = {}, {}
    for case in tv.CASES:
        w, h, ss, flags, niter, quality = case
        gio.put_result(d, tv.case_key("driver", case), *ol.run_reference(qs.synth.make_image(w, h, ss, quality=quality), flags, niter))
    for case in tv.ADVERSARIAL:
        kind, flags, niter = case
        gio.put_result(e, tv.case_key("adv", case), *ol.run_reference(gio.adversarial_image(kind), flags, niter))
    im = qs.synth.make_image(96, 80, "420")
    r1, a = ol.run_reference(im, 7, 2, scatter_rows=True, threads=3)
    r2, b = ol.run_reference(im, 7, 2, threads=1)
    assert r1 == r2 and ol.images_equal(a, b)
    gio.put_result(e, "scattered", r1, a)
    seq = []
    gio.put_result(e, "progress", *ol.run_reference(im, 0, 3, progprec=7, progress=lambda _, cur, mx: seq.append((cur, mx)) or 0))
    e["progress.seq"] = np.array(seq, dtype=np.int32)
    seq = []
    gio.put_result(e, "cancel", *ol.run_reference(im, 0, 3, progprec=7, progress=lambda _, cur, mx: (seq.append(cur), 5 if len(seq) >= 2 else 0)[1]))
    e["cancel.seq"] = np.array(seq, dtype=np.int32)
    for case, (im, flags, niter) in enumerate(tv.sweep_cases()):
        gio.put_result(e, f"sweep{case}", *ol.run_reference(im, flags, niter))
    for case in te.ENTRY_CASES:
        flags, niter, ss = case
        gio.put_result(e, tv.case_key("entry", case), *ol.run_reference(qs.synth.make_image(120, 72, ss), flags, niter, scatter_rows=True))
    for case in tv.GEOMETRY_CASES:               # grey ones in ref_sweep.npz, to keep each under 1 MB
        if case[4] == "synth":
            gio.put_result(e if case[2].startswith("g") else d, tv.case_key("geo", case),
                           *ol.run_reference(*tv.geometry_case(case)))
    _save_npz(os.path.join(HERE, "ref_driver.npz"), d)
    _save_npz(os.path.join(HERE, "ref_sweep.npz"), e)


def saturated():
    import test_oracle_vs_reference as tv
    d = {}
    for case in tv.SATURATED_SMALL:
        gio.put_result(d, tv.case_key("sat", case), *ol.run_reference(*tv.saturated_case(case)))
    for case in tv.GEOMETRY_CASES:
        if case[4] == "saturated":
            gio.put_result(d, tv.case_key("geo", case), *ol.run_reference(*tv.geometry_case(case)))
    _save_npz(os.path.join(HERE, "ref_saturated.npz"), d)
    digests = {tv.case_key("satw", case): gio.result_digest(*ol.run_reference(*tv.saturated_case(case)))
               for case in tv.SATURATED_WAVE}
    with open(os.path.join(HERE, "ref_saturated.json"), "w") as f:
        json.dump(digests, f, indent=1, sort_keys=True)
        f.write("\n")


def _sha(path):
    return hashlib.sha256(open(path, "rb").read()).hexdigest()


def files():
    import test_cli as tc
    import test_real_libjpeg as tr
    out = {"jpegqs_ref": {}, "refcli_cpu": {}, "codec_difftest": {}}
    with tempfile.TemporaryDirectory() as t:
        jpegs = tc.write_jpegs(t)
        jpegs.update(tr.write_mcu_jpegs(t))
        o = os.path.join(t, "out.jpg")
        for name, args in tc.REF_TOOL_CASES:
            subprocess.run([os.path.join(REFDIR, "jpegqs_ref"), "-i", "0"] + args + [jpegs[name], o], check=True, capture_output=True)
            out["jpegqs_ref"][tc.file_key(name, args)] = _sha(o)
        for name, args in tr.REF_CLI_CASES:
            subprocess.run([os.path.join(REFDIR, "refcli_cpu"), "-i", "0"] + args + [jpegs[name], o], check=True, capture_output=True)
            out["refcli_cpu"][tc.file_key(name, args)] = _sha(o)
        for seed, n in tr.CODEC_DIFFTEST_RUNS:
            r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "codec_difftest.py"), str(seed), str(n), "--record"],
                               cwd=t, capture_output=True, text=True, check=True)
            out["codec_difftest"][str(seed)] = json.loads(r.stdout.splitlines()[-1])
    with open(os.path.join(HERE, "ref_files.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    ol.ensure_built()
    assert ol.have_ref("scalar"), "needs oracle/_ref (make -C oracle ref with the reference sources)"
    parts = sys.argv[1:] or ["kernels", "driver", "files", "saturated"]
    for part in parts:
        {"kernels": kernels, "driver": driver, "files": files, "saturated": saturated}[part]()
