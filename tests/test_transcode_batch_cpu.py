"""jpegqs_cuda_transcode_batch / QsContext.transcode_batch argument checks that need no GPU, and the
jpegqs tool's --batch on a machine without one: it reports the missing back end for every pair, as
one pair after the other does, exits 2 and writes nothing."""
import ctypes as C
import os
import subprocess

import pytest

PIL = pytest.importorskip("PIL.Image")

import decode_files as df
from jpegqs_b200 import cuda
from test_cli import EXE, write_jpegs


@pytest.fixture(scope="module")
def jpegs(tmp_path_factory):
    return write_jpegs(str(tmp_path_factory.mktemp("jpegs")))


def _unbound():
    """A QsContext without a device: the wrapper's checks run before it touches one."""
    return object.__new__(cuda.QsContext)


def test_python_wrapper_checks_its_arguments():
    good = df.pillow_jpeg(64, 48, quality=75)
    ctx = _unbound()
    assert cuda.QsContext.transcode_batch(ctx, [], 0, 3) == []
    assert cuda.QsContext.transcode_batch(ctx, (), 0, 3) == []
    for bad in (good, "text", None, 12, bytearray(good)):
        with pytest.raises(TypeError):
            cuda.QsContext.transcode_batch(ctx, bad, 0, 3)
    for bad in ([good, None], [good, "text"], [12]):
        with pytest.raises(TypeError):
            cuda.QsContext.transcode_batch(ctx, bad, 0, 3)
    for copy in (-1, 3):
        with pytest.raises(ValueError):
            cuda.QsContext.transcode_batch(ctx, [good], 0, 3, copy=copy)
    with pytest.raises(ValueError):
        cuda.QsContext.transcode_batch(ctx, [good], 0, 3, max_device_bytes=-1)


def test_c_call_without_a_context():
    lib = cuda.load()
    data = df.pillow_jpeg(64, 48, quality=75)
    ptrs = (C.c_char_p * 1)(data)
    lens = (C.c_size_t * 1)(len(data))
    rc = (C.c_int * 1)(7)
    res = (cuda._TranscodeResult * 1)()
    assert lib.jpegqs_cuda_transcode_batch(None, 1, ptrs, lens, 0, 3, 0, 2, 0, rc, res) == -2
    assert lib.jpegqs_cuda_transcode_batch(None, 0, None, None, 0, 3, 0, 2, 0, None, None) == -2
    assert rc[0] == 7 and not res[0].data                     # nothing touched


def _no_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")


def test_tool_batch_without_a_gpu(jpegs, tmp_path):
    _no_gpu()
    names = ["base420", "gray", "progrst", "rst", "base444"]
    outs = [tmp_path / f"{n}.jpg" for n in names]
    pairs = [a for n, o in zip(names, outs) for a in (jpegs[n], str(o))]
    runs = {}
    for tag, env in (("pipe", {}), ("serial", {"JPEGQS_NO_PIPELINE": "1"}), ("host", {"JPEGQS_HOST_CODEC": "1"})):
        r = subprocess.run([EXE, "-q", "3", "--batch"] + pairs, capture_output=True, text=True,
                           env=dict(os.environ, **env))
        assert r.returncode == 2, r.stderr
        assert r.stderr.count("CUDA back end unavailable") == len(names), r.stderr
        assert not any(o.exists() for o in outs)
        runs[tag] = r.stderr
    assert runs["pipe"] == runs["serial"] == runs["host"]
