"""jpegqs_cuda_transcode_batch (QsContext.transcode_batch) on the GPU: every file of a batch comes back
exactly as jpegqs_cuda_transcode gives it alone - bytes, return code, smoothed / stop / upsampled and
reason - whatever the order of the files, the sub-batch budget, and the files that fall back or stop
beside it.  Also the jpegqs tool's --batch, whose device pairs now go through the batch call."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

PIL = pytest.importorskip("PIL.Image")

import decode_files as df
import hard_content as hc
import scan_files as sf
from render_images import make
from test_cli import EXE, FILES, _big_picture, _picture
import jpegqs_b200 as qs
from jpegqs_b200 import cuda

pytestmark = pytest.mark.gpu


def _damaged(good):
    """An EOI marker in the middle of the entropy-coded data: the device decoder flags it."""
    d = bytearray(good)
    d[len(d) * 3 // 5:len(d) * 3 // 5 + 2] = b"\xff\xd9"
    return bytes(d)


def _stop_file():
    """A coefficient that de-quantizes past 2047: the run stops for this image."""
    return df.coef_writer_jpeg(hc.with_dequant_edge(make(64, 48, "420", "k50", "synth", 3), True))


@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    """name -> bytes: every tool flavour, CMYK, a scan script with restart markers, the 8K file, a
    damaged file and a stopping image."""
    d = tmp_path_factory.mktemp("corpus")
    out = {}
    for k, (name, w, h, gray, kw) in enumerate(FILES):
        p = d / f"{name}.jpg"
        _picture(w, h, gray, k).save(str(p), comment=b"made by the test suite", **kw)
        out[name] = p.read_bytes()
    out["cmyk"] = df.pillow_jpeg(120, 80, "CMYK", quality=85)
    scripted = [(n, b) for n, b in sf.scripted() if "rst" in n]
    if scripted:
        out["script_" + scripted[0][0]] = scripted[0][1]
    p = d / "8k.jpg"
    _big_picture(7680, 4320, 5).save(str(p), quality=90)
    out["8k"] = p.read_bytes()
    out["damaged"] = _damaged(out["base420"])
    out["stop"] = _stop_file()
    return out


@pytest.fixture(scope="module")
def ctx():
    c = cuda.QsContext(0)
    yield c
    c.close()


def _c_single(ctx, data, flags, niter, optimize, copy):
    res = cuda._TranscodeResult()
    rc = ctx.lib.jpegqs_cuda_transcode(ctx.h, data, len(data), flags, niter, int(optimize), copy, C.byref(res))
    return _take(ctx, rc, res)


def _take(ctx, rc, res):
    data = None
    if rc == cuda.TRANSCODE_OK:
        data = C.string_at(res.data, res.len)
        ctx.lib.jpegqs_cuda_transcode_free(res.data)
    else:
        assert not res.data
    return (rc, data, res.smoothed, res.stop, res.upsampled, (res.reason or b"").decode())


def _c_batch(ctx, datas, flags, niter, optimize, copy, budget=0):
    n = len(datas)
    ptrs = (C.c_char_p * n)(*datas)
    lens = (C.c_size_t * n)(*[len(d) for d in datas])
    rc = (C.c_int * n)()
    res = (cuda._TranscodeResult * n)()
    ret = ctx.lib.jpegqs_cuda_transcode_batch(ctx.h, n, ptrs, lens, flags, niter, int(optimize), copy, budget, rc, res)
    assert ret == 0, ctx.lib.jpegqs_cuda_last_error(ctx.h).decode()
    return [_take(ctx, rc[i], res[i]) for i in range(n)]


OPTS = {"q3": (qs.quality_to_flags(3), 3), "q6": (qs.quality_to_flags(6), 3), "n0": (qs.quality_to_flags(6), 0)}


@pytest.fixture(scope="module")
def singles(ctx, corpus):
    """(name, opt, optimize, copy) -> the single call's result, computed once."""
    cache = {}

    def get(name, opt, optimize, copy):
        key = (name, opt, optimize, copy)
        if key not in cache:
            flags, niter = OPTS[opt]
            cache[key] = _c_single(ctx, corpus[name], flags | qs.JPEGQS_TRANSCODE, niter, optimize, copy)
        return cache[key]
    return get


@pytest.mark.parametrize("copy", [0, 2])
@pytest.mark.parametrize("optimize", [False, True])
@pytest.mark.parametrize("opt", sorted(OPTS))
def test_batch_equals_single(ctx, corpus, singles, opt, optimize, copy):
    names = sorted(corpus)
    flags, niter = OPTS[opt]
    got = _c_batch(ctx, [corpus[n] for n in names], flags | qs.JPEGQS_TRANSCODE, niter, optimize, copy)
    for n, g in zip(names, got):
        assert g == singles(n, opt, optimize, copy), (n, opt, optimize, copy)
    by = dict(zip(names, got))
    assert by["damaged"][0] == cuda.TRANSCODE_FALLBACK and "flagged" in by["damaged"][5]
    assert by["prog420"][0] == cuda.TRANSCODE_FALLBACK and "restart markers" in by["prog420"][5]
    assert by["base420"][0] == cuda.TRANSCODE_OK
    if opt != "n0":
        assert by["stop"][2] == 1 and by["stop"][3] != 0
    else:
        assert by["gray"][2] == 0                  # gray at -n 0 -q 6: nothing to up-sample, not smoothed
        assert by["base420"][2] == 1 and by["base420"][4] == 1


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_order_does_not_matter(ctx, corpus, singles, seed):
    names = sorted(corpus)
    perm = list(np.random.RandomState(seed).permutation(len(names)))
    flags, niter = OPTS["q6"]
    got = _c_batch(ctx, [corpus[names[i]] for i in perm], flags | qs.JPEGQS_TRANSCODE, niter, False, 2)
    for i, g in zip(perm, got):
        assert g == singles(names[i], "q6", False, 2), names[i]


@pytest.mark.parametrize("budget", [1, 3 << 20, 40 << 20])
def test_splitting_is_invisible(ctx, corpus, singles, budget):
    """1 byte: every file alone; 3 MB: pairs and small groups of the small files; 40 MB: most small
    files together, the 8K file (about 1.5 GB of needs) bigger than the budget and alone."""
    names = sorted(corpus)
    flags, niter = OPTS["q3"]
    got = _c_batch(ctx, [corpus[n] for n in names], flags | qs.JPEGQS_TRANSCODE, niter, False, 2, budget)
    for n, g in zip(names, got):
        assert g == singles(n, "q3", False, 2), (n, budget)


def test_fallbacks_are_isolated(ctx, corpus, singles):
    names = ["base420", "damaged", "rst", "prog420", "cmyk", "stop", "opt422", "damaged", "gray"]
    flags, niter = OPTS["q3"]
    got = _c_batch(ctx, [corpus[n] for n in names], flags | qs.JPEGQS_TRANSCODE, niter, False, 2)
    for n, g in zip(names, got):
        assert g == singles(n, "q3", False, 2), n
    assert got[1][0] == got[7][0] == cuda.TRANSCODE_FALLBACK and "flagged" in got[1][5]
    assert got[3][0] == cuda.TRANSCODE_FALLBACK and "restart markers" in got[3][5]
    assert got[5][3] != 0 and got[5][0] == cuda.TRANSCODE_OK


def test_a_rejected_file(ctx, corpus, singles):
    names = ["base420", None, "gray"]
    datas = [corpus[n] if n else b"this is not a jpeg" for n in names]
    flags, niter = OPTS["q3"]
    n = len(datas)
    ptrs = (C.c_char_p * n)(*datas)
    lens = (C.c_size_t * n)(*[len(d) for d in datas])
    rc = (C.c_int * n)()
    res = (cuda._TranscodeResult * n)()
    assert ctx.lib.jpegqs_cuda_transcode_batch(ctx.h, n, ptrs, lens, flags | qs.JPEGQS_TRANSCODE, niter, 0, 2, 0, rc, res) == 0
    assert rc[1] == -2 and not res[1].data
    assert "file 1" in ctx.lib.jpegqs_cuda_last_error(ctx.h).decode()
    for i in (0, 2):
        assert _take(ctx, rc[i], res[i]) == singles(names[i], "q3", False, 2)
    with pytest.raises(cuda.QsError, match="file 1"):
        ctx.transcode_batch(datas, flags | qs.JPEGQS_TRANSCODE, niter)


def test_python_call_and_buffer_reuse(corpus, singles):
    """A second call on the same context after one with bigger files gives the same bytes; the module
    call and QsContext.transcode_batch agree with transcode."""
    c = cuda.QsContext(0)
    flags, niter = OPTS["q3"]
    small = ["base420", "progrst", "cmyk", "damaged", "gray"]
    first = c.transcode_batch([corpus[n] for n in ["8k"] + small], flags | qs.JPEGQS_TRANSCODE, niter)
    second = c.transcode_batch([corpus[n] for n in small], flags | qs.JPEGQS_TRANSCODE, niter)
    assert first[1:] == second
    for n, (data, why) in zip(small, second):
        want = singles(n, "q3", False, 2)
        assert data == want[1] and (why is None) == (want[0] == cuda.TRANSCODE_OK)
        assert c.transcode(corpus[n], flags | qs.JPEGQS_TRANSCODE, niter) == (data, why)
    assert first[0][0] == singles("8k", "q3", False, 2)[1]
    assert c.last_device_ms > 0
    c.close()
    assert qs.transcode_batch([corpus["base420"]], flags | qs.JPEGQS_TRANSCODE, niter, device=0) == [second[0]]


MASK = re.compile(r"[0-9]+\.[0-9]+ms")


def _tool(args, env):
    return subprocess.run([EXE] + args, capture_output=True, text=True, env=env)


def test_tool_batch_is_unchanged(corpus, tmp_path):
    """About 40 mixed pairs - small files first so that batches form, then the 8K file, an in-place pair
    and a missing input - give the same bytes, exit status and -i lines (timings masked) as one pair
    after the other and as the host codec.  The missing input's message comes from a reader thread, so
    its place among the -i lines is not fixed: it is compared as a line, the -i lines in order."""
    src = tmp_path / "src"
    src.mkdir()
    small = [n for n in sorted(corpus) if n != "8k"]
    paths = {}
    for n in corpus:
        paths[n] = src / f"{n}.jpg"
        paths[n].write_bytes(corpus[n])

    def run(tag, extra_env):
        d = tmp_path / tag
        d.mkdir()
        inplace = d / "inplace.jpg"
        shutil.copy(paths["base444"], inplace)
        pairs, outs = [], []
        for k in range(3):
            for n in small:
                o = d / f"{k}_{n}.jpg"
                pairs += [str(paths[n]), str(o)]
                outs.append(o)
        pairs += [str(paths["8k"]), str(d / "8k.jpg"), str(inplace), str(inplace), str(tmp_path / "missing.jpg"),
                  str(d / "missing.jpg"), str(paths["gray"]), str(d / "last.jpg")]
        outs += [d / "8k.jpg", inplace, d / "last.jpg"]
        r = _tool(["-q", "3", "-i", "15", "--batch"] + pairs, dict(os.environ, **extra_env))
        assert not (d / "missing.jpg").exists()
        return r, [o.read_bytes() if o.exists() else None for o in outs], len(pairs) // 2

    serial = run("serial", {"JPEGQS_NO_PIPELINE": "1"})
    assert serial[2] >= 40
    # the messages that are not -i lines (the missing input, the reader's warnings on the damaged file):
    # on the host codec a reader thread prints them, possibly in the middle of an -i line of the
    # calling thread, so they are taken out of the text by value and counted
    info = re.compile(r"^(component\[|quant\[|SIMD type|quantsmooth|([0-9a-f]{4} )+$)")
    messages = {l + "\n" for l in serial[0].stderr.splitlines() if not info.match(l)}
    assert any("missing.jpg" in m for m in messages)

    def split(stderr):
        counts = {m: stderr.count(m) for m in messages}
        for m in messages:
            stderr = stderr.replace(m, "")
        return MASK.sub("<t>ms", stderr), counts
    want = split(serial[0].stderr)
    for tag, env in (("pipe", {}), ("host", {"JPEGQS_HOST_CODEC": "1"})):
        other = run(tag, env)
        assert other[0].returncode == serial[0].returncode != 0, (serial[0].stderr, other[0].stderr)
        assert other[1] == serial[1], tag
        assert split(other[0].stderr) == want, tag


def test_c_call_checks_its_arguments(ctx, corpus):
    data = corpus["base420"]
    ptrs = (C.c_char_p * 2)(data, data)
    lens = (C.c_size_t * 2)(len(data), len(data))
    rc = (C.c_int * 2)(7, 7)
    res = (cuda._TranscodeResult * 2)()
    f = ctx.lib.jpegqs_cuda_transcode_batch
    assert f(ctx.h, 0, None, None, 0, 3, 0, 2, 0, None, None) == 0
    assert f(ctx.h, -1, ptrs, lens, 0, 3, 0, 2, 0, rc, res) == -2
    for args in ((None, lens, rc, res), (ptrs, None, rc, res), (ptrs, lens, None, res), (ptrs, lens, rc, None)):
        assert f(ctx.h, 2, args[0], args[1], 0, 3, 0, 2, 0, args[2], args[3]) == -2
    assert list(rc) == [7, 7]
    for copy in (-1, 3):
        assert f(ctx.h, 2, ptrs, lens, 0, 3, 0, copy, 0, rc, res) == -2
        assert "copy" in ctx.lib.jpegqs_cuda_last_error(ctx.h).decode()
    holes = (C.c_char_p * 2)(data, None)
    assert f(ctx.h, 2, holes, lens, 0, 3, 0, 2, 0, rc, res) == -2
    assert "file 1" in ctx.lib.jpegqs_cuda_last_error(ctx.h).decode()
    assert not res[0].data and not res[1].data
