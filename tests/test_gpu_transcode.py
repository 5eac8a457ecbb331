"""The jpegqs tool's device route (decode, smoothing and encode on the GPU) against its host codec
(JPEGQS_HOST_CODEC=1), each in its own process: the same bytes, exit statuses and messages.  Also
QsContext.transcode, the Python form of the same call."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

PIL = pytest.importorskip("PIL.Image")

import decode_files as df
from golden_io import reference_files
from test_cli import EXE, FILES, REF_TOOL_CASES, file_key, write_jpegs
from test_transcode_cpu import FLAVOUR_ROUTE

pytestmark = pytest.mark.gpu

HOST = dict(os.environ, JPEGQS_HOST_CODEC="1")
DEVICE = dict(os.environ, JPEGQS_CODEC_TRACE="1")


@pytest.fixture(scope="module")
def jpegs(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("jpegs"))
    out = write_jpegs(d)
    p = os.path.join(d, "cmyk.jpg")
    open(p, "wb").write(df.pillow_jpeg(120, 80, "CMYK", quality=85))
    out["cmyk"] = p
    return out


@pytest.fixture(scope="module")
def big(tmp_path_factory):
    """An 8K 4:2:0 q90 file."""
    from test_cli import _big_picture
    p = str(tmp_path_factory.mktemp("big") / "8k.jpg")
    _big_picture(7680, 4320, 5).save(p, quality=90)
    return p


def _run(args, env, **kw):
    return subprocess.run([EXE] + args, capture_output=True, text=True, env=env, **kw)


def _pair(tmp_path, args, src, tag=""):
    """(device route result, its bytes, host route result, its bytes) of one pair."""
    a, b = str(tmp_path / f"dev{tag}.jpg"), str(tmp_path / f"host{tag}.jpg")
    r1, r2 = _run(args + [src, a], DEVICE), _run(args + [src, b], HOST)
    read = lambda p: open(p, "rb").read() if os.path.exists(p) else None
    return r1, read(a), r2, read(b)


ARG_SETS = sorted({tuple(a) for _, a in REF_TOOL_CASES}) + [("-q", "3", "-c", "0"), ("-q", "3", "-c", "1"),
                                                           ("-q", "3", "-c", "2"), ("-q", "4", "-o")]


@pytest.mark.parametrize("args", ARG_SETS, ids=[" ".join(a) for a in ARG_SETS])
def test_every_flavour_and_option(jpegs, tmp_path, args):
    """Every flavour in one --batch process per route; the reference tool's SHA-256 where it has one."""
    args = list(args)
    names = [f[0] for f in FILES]
    out = {}
    for tag, env in (("dev", DEVICE), ("host", HOST)):
        pairs = []
        for n in names:
            pairs += [jpegs[n], str(tmp_path / f"{tag}_{n}.jpg")]
        r = _run(["-i", "0"] + args + ["--batch"] + pairs, env)
        assert r.returncode == 0, r.stderr
        out[tag] = r
    ref = reference_files()["jpegqs_ref"]
    for n in names:
        dev, host = (open(tmp_path / f"{t}_{n}.jpg", "rb").read() for t in ("dev", "host"))
        assert dev == host, (n, args)
        assert f"jpegqs: {jpegs[n]}: {FLAVOUR_ROUTE[n]} route" in out["dev"].stderr
        key = file_key(n, args)
        if key in ref:
            import hashlib
            assert hashlib.sha256(dev).hexdigest() == ref[key], key


@pytest.mark.parametrize("name", ["base420", "base444", "gray", "opt422"])
def test_early_return_corners(jpegs, tmp_path, name):
    """-n 0 -q 6: 4:2:0 and 4:2:2 are up-sampled without smoothing, 4:4:4 is run with zero iterations
    (its quant tables become ones), gray returns at once (its tables stay)."""
    r1, a, r2, b = _pair(tmp_path, ["-n", "0", "-q", "6", "-i", "0"], jpegs[name])
    assert r1.returncode == r2.returncode == 0, r1.stderr
    assert a == b
    assert "device route" in r1.stderr


@pytest.mark.parametrize("q", ["3", "6"])
def test_8k_file(big, tmp_path, q):
    r1, a, r2, b = _pair(tmp_path, ["-q", q, "-i", "0"], big)
    assert r1.returncode == r2.returncode == 0, r1.stderr
    assert a == b
    assert "device route (sequential, one scan)" in r1.stderr


def test_mixed_batch(jpegs, big, tmp_path):
    """Small files of every kind, then an 8K file (the device buffers grow), an in-place pair, the same
    output twice and a missing input: the files equal the host route's and those of single pairs."""
    def run(tag, env):
        d = tmp_path / tag
        d.mkdir()
        inplace = str(d / "inplace.jpg")
        shutil.copy(jpegs["dense444"], inplace)
        o = lambda n: str(d / f"{n}.jpg")
        args = ["-q", "3", "-i", "0", "--batch"]
        for n in ("base420", "rst", "progrst", "prog420", "gray", "opt422", "cmyk"):
            args += [jpegs[n], o(n)]
        args += [big, o("big"), inplace, inplace, str(tmp_path / "missing.jpg"), o("missing"),
                 jpegs["base444"], o("twice"), jpegs["coarse420"], o("twice"), jpegs["tinyprog"], o("tinyprog")]
        r = _run(args, env)
        assert r.returncode == 1 and "missing.jpg" in r.stderr, r.stderr
        assert not os.path.exists(o("missing"))
        names = ("base420", "rst", "progrst", "prog420", "gray", "opt422", "cmyk", "big", "inplace", "twice", "tinyprog")
        return {n: open(o(n), "rb").read() for n in names}
    dev, host = run("dev", DEVICE), run("host", HOST)
    assert dev == host
    for n in ("base420", "progrst", "cmyk", "coarse420"):
        single = str(tmp_path / f"single_{n}.jpg")
        assert _run(["-q", "3", "-i", "0", jpegs[n], single], DEVICE).returncode == 0
        assert open(single, "rb").read() == dev["twice" if n == "coarse420" else n], n


def _mutations(jpegs, count=60):
    """Seeded damage of the small flavours, made as test_cli.test_codec_survives_corrupt_input makes it,
    plus an EOI marker in the middle of the entropy-coded data (the device decoder runs out of data,
    the host reader decodes zeros)."""
    rng = np.random.RandomState(11)
    seeds = [open(jpegs[n], "rb").read() for n in ("base420", "progrst", "gray", "rst", "base444", "opt422", "cmyk")]
    out = []
    for it in range(count):
        d = bytearray(seeds[it % len(seeds)])
        mode = rng.randint(4)
        if mode == 0:
            for _ in range(rng.randint(1, 6)):
                d[rng.randint(len(d))] = rng.randint(256)
        elif mode == 1:
            d = d[:rng.randint(2, len(d))]
        elif mode == 2:
            i = rng.randint(2, len(d) - 4)
            d[i:i + 4] = bytes(rng.randint(0, 256, 4).tolist())
        else:
            i = rng.randint(len(d))
            d = d[:i] + bytes(rng.randint(0, 256, rng.randint(1, 40)).tolist()) + d[i:]
        out.append(bytes(d))
    d = bytearray(seeds[0])
    d[len(d) * 3 // 5:len(d) * 3 // 5 + 2] = b"\xff\xd9"
    out.append(bytes(d))
    return out


def test_damaged_files(jpegs, tmp_path):
    """Exit status and output (or its absence) are the host route's; the trace says when the device
    decoder handed a file back."""
    fell_back = 0
    for it, data in enumerate(_mutations(jpegs)):
        src = tmp_path / f"m{it}.jpg"
        src.write_bytes(data)
        r1, a, r2, b = _pair(tmp_path, ["-q", "3", "-n", "1", "-i", "0"], str(src), tag=str(it))
        assert r1.returncode == r2.returncode, (it, r1.stderr, r2.stderr)
        assert a == b, it
        fell_back += "host route after all" in r1.stderr
    assert fell_back >= 1


@pytest.mark.parametrize("info", ["15", "31"])
@pytest.mark.parametrize("name", ["base420", "progrst", "gray", "opt422"])
def test_info_lines(jpegs, tmp_path, name, info):
    """-i lines: the same lines in the same order; only the timings differ."""
    mask = lambda s: re.sub(r"[0-9]+\.[0-9]+ms", "<t>ms", s)
    r1, a, r2, b = _pair(tmp_path, ["-q", "6", "-i", info], jpegs[name])
    assert r1.returncode == r2.returncode == 0
    dev = "".join(l for l in r1.stderr.splitlines(True) if not l.startswith("jpegqs: ") or "route" not in l)
    assert mask(dev) == mask(r2.stderr)
    assert a == b


def test_stdin_and_stdout(jpegs):
    data = open(jpegs["base420"], "rb").read()
    outs = []
    for env in (DEVICE, HOST):
        r = subprocess.run([EXE, "-q", "3", "-i", "0", "-", "-"], input=data, capture_output=True, env=env)
        assert r.returncode == 0, r.stderr
        outs.append(r.stdout)
    assert outs[0] == outs[1] and outs[0][:2] == b"\xff\xd8"
    assert b"device route" in subprocess.run([EXE, "-q", "3", "-i", "0", "-", "-"], input=data, capture_output=True,
                                             env=DEVICE).stderr


def test_python_transcode(jpegs, big, tmp_path):
    """QsContext.transcode gives the tool's bytes; files of different geometries in a row reuse the
    context (its buffers grow); a file for the host route comes back as None with its reason."""
    import jpegqs_b200 as qs
    ctx = qs.QsContext(0)
    cases = [("base420", "3", []), ("dense444", "6", ["-o"]), ("progrst", "4", []), ("base420", "6", []),
             ("cmyk", "3", ["-c", "0"]), ("gray", "5", [])]
    for name, q, extra in cases * 2:
        want = str(tmp_path / "want.jpg")
        assert _run(["-q", q, "-i", "0"] + extra + [jpegs[name], want], HOST).returncode == 0
        flags = qs.quality_to_flags(int(q)) | qs.JPEGQS_TRANSCODE
        copy = 0 if "-c" in extra else 2
        out, why = ctx.transcode(open(jpegs[name], "rb").read(), flags, 3, optimize="-o" in extra, copy=copy)
        assert why is None and out == open(want, "rb").read(), (name, q, extra)
    out, why = qs.transcode(open(big, "rb").read(), qs.quality_to_flags(3), 3, device=0)
    assert why is None and out[:2] == b"\xff\xd8"
    out, why = ctx.transcode(open(jpegs["prog420"], "rb").read(), qs.quality_to_flags(3), 3)
    assert out is None and "restart markers" in why
    d = bytearray(open(jpegs["base420"], "rb").read())
    d[len(d) * 3 // 5:len(d) * 3 // 5 + 2] = b"\xff\xd9"
    out, why = ctx.transcode(bytes(d), qs.quality_to_flags(3), 3)
    assert out is None and "flagged" in why
    with pytest.raises(qs.cuda.QsError):
        ctx.transcode(b"not a jpeg", 0, 3)
    with pytest.raises(TypeError):
        ctx.transcode("text", 0, 3)
