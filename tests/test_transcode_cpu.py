"""The transcode route (jpegqs_cuda_transcode_route, Python transcode_route) and the jpegqs tool's
choice of route, on a machine without a GPU.  The route is host-only: a file goes to the device only
when its whole marker walk is clean, a device decoder takes it, it is not a progressive file with an
AC refinement scan without restart markers, and the encoder takes its geometry."""
import os
import subprocess

import pytest

PIL = pytest.importorskip("PIL.Image")

import decode_files as df
import scan_files as sf
import jpegqs_b200 as qs
from test_cli import EXE, FILES, write_jpegs

# the FILES flavours of test_cli.py: Pillow's progressive files without restart markers carry AC
# refinement scans, so only progrst goes to the device among the progressive ones
FLAVOUR_ROUTE = {"base420": "device", "base444": "device", "prog420": "host", "gray": "device", "opt422": "device",
                 "prog444": "host", "rst": "device", "progrst": "device", "tinyprog": "host", "dense444": "device",
                 "coarse420": "device"}


@pytest.fixture(scope="module")
def jpegs(tmp_path_factory):
    return write_jpegs(str(tmp_path_factory.mktemp("jpegs")))


def _route(data):
    return qs.transcode_route(data)[0]


def test_every_flavour_has_a_route():
    assert sorted(FLAVOUR_ROUTE) == sorted(f[0] for f in FILES)


@pytest.mark.parametrize("name", [f[0] for f in FILES])
def test_route_of_the_tool_flavours(jpegs, name):
    route, reason = qs.transcode_route(open(jpegs[name], "rb").read())
    assert route == FLAVOUR_ROUTE[name], reason
    if route == "host":
        assert "restart" in reason


def _scripted_route(name):
    # AC refinement scans (Ah > 0, Ss > 0) without restart markers stay on the host
    refines = name.startswith(("succ_al3", "dc_per_comp", "split_bands", "flat_prog"))
    return "host" if refines and "rst" not in name else "device"


@pytest.mark.parametrize("name,data", sf.scripted(), ids=[n for n, _ in sf.scripted()])
def test_route_of_the_scan_scripts(name, data):
    route, reason = qs.transcode_route(data)
    assert route == _scripted_route(name), reason


def test_route_of_progressive_files_with_and_without_restart_markers():
    pic = dict(quality=80, progressive=True, seed=3)
    assert _route(df.pillow_jpeg(250, 190, **pic)) == "host"
    assert _route(df.pillow_jpeg(250, 190, restart_marker_rows=1, **pic)) == "device"
    assert _route(df.pillow_jpeg(250, 190, restart_marker_blocks=5, **pic)) == "device"


def test_more_than_64_scans_stay_on_the_host():
    gray = df.pillow_jpeg(90, 70, "L", quality=92, seed=5)
    script = [((0,), 0, 0, 0, 1), ((0,), 0, 0, 1, 0)] + [((0,), k, k, 0, 0) for k in range(1, 64)]
    data = sf.rescan(gray, script)
    assert data.count(b"\xff\xda") >= 65
    route, reason = qs.transcode_route(data)
    assert route == "host" and "64" in reason
    assert _route(sf.rescan(gray, script[:64])) == "device"             # 64 scans: the device takes them


def _sos_end(data):
    i = data.index(b"\xff\xda")
    return i + 2 + int.from_bytes(data[i + 2:i + 4], "big")


def test_damaged_marker_walks_stay_on_the_host(jpegs):
    data = open(jpegs["base420"], "rb").read()
    assert _route(data) == "device"
    assert _route(data[:_sos_end(data)]) == "host"                     # cut at the SOS: no data, no EOI
    assert _route(data[:-2]) == "host"                                # no EOI
    i = data.index(b"\xff\xdb")
    assert _route(data[:i] + b"\x12\x34\x56" + data[i:]) == "host"     # extraneous bytes before a marker
    prog = df.pillow_jpeg(250, 190, quality=80, progressive=True, restart_marker_rows=1, seed=3)
    assert _route(prog[:_sos_end(prog)]) == "host"


def test_cmyk_and_gray_files_go_to_the_device():
    assert _route(df.pillow_jpeg(120, 80, "CMYK", quality=85)) == "device"
    assert _route(df.pillow_jpeg(97, 61, "L", quality=75)) == "device"


def test_a_file_the_reader_rejects_is_an_error():
    for bad in (b"this is not a jpeg", b"", b"\xff\xd8\xff\xdb\x00"):
        with pytest.raises(qs.cuda.QsError):
            qs.transcode_route(bad)


def test_route_arguments_are_checked():
    for bad in (None, "text", 12, [0xFF, 0xD8]):
        with pytest.raises(TypeError):
            qs.transcode_route(bad)
    assert _route(bytearray(df.pillow_jpeg(64, 48, quality=75))) == "device"
    assert _route(memoryview(df.pillow_jpeg(64, 48, quality=75))) == "device"


def _no_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")


def test_tool_without_a_gpu_on_a_device_route_file(jpegs, tmp_path):
    """As before the device route existed: the tool reports the missing back end, exits 2 and writes
    nothing."""
    _no_gpu()
    out = tmp_path / "o.jpg"
    env = dict(os.environ, JPEGQS_CODEC_TRACE="1")
    r = subprocess.run([EXE, "-q", "3", jpegs["base420"], str(out)], capture_output=True, text=True, env=env)
    assert r.returncode == 2 and "CUDA back end unavailable" in r.stderr, r.stderr
    assert "device route" in r.stderr
    assert not out.exists()
    host = subprocess.run([EXE, "-q", "3", jpegs["base420"], str(out)], capture_output=True, text=True,
                          env=dict(os.environ, JPEGQS_HOST_CODEC="1"))
    assert host.returncode == 2 and host.stderr == r.stderr.replace(
        f"jpegqs: {jpegs['base420']}: device route (sequential, one scan)\n", "")
    assert not out.exists()


def test_tool_without_a_gpu_when_nothing_is_smoothed(jpegs, tmp_path):
    """Nothing to smooth and nothing to up-sample (a gray file at -q 6 -n 0): the host route needs no
    device, so the device route hands the file back to it."""
    _no_gpu()
    a, b = tmp_path / "a.jpg", tmp_path / "b.jpg"
    env = dict(os.environ, JPEGQS_CODEC_TRACE="1")
    r = subprocess.run([EXE, "-q", "6", "-n", "0", "-i", "0", jpegs["gray"], str(a)], capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr
    assert "host route after all" in r.stderr
    r = subprocess.run([EXE, "-q", "6", "-n", "0", "-i", "0", jpegs["gray"], str(b)], env=dict(os.environ, JPEGQS_HOST_CODEC="1"))
    assert r.returncode == 0 and a.read_bytes() == b.read_bytes()


def test_tool_with_n0_takes_the_host_route(jpegs, tmp_path):
    out = tmp_path / "o.jpg"
    env = dict(os.environ, JPEGQS_CODEC_TRACE="1")
    r = subprocess.run([EXE, "-n", "0", "-i", "0", jpegs["base420"], str(out)], capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr
    assert f"jpegqs: {jpegs['base420']}: host route (nothing to smooth)" in r.stderr
    assert out.exists()


def test_tool_host_codec_knob_and_ppm_keep_the_host_route(jpegs, tmp_path):
    env = dict(os.environ, JPEGQS_CODEC_TRACE="1", JPEGQS_HOST_CODEC="1")
    r = subprocess.run([EXE, "-q", "3", "-i", "0", jpegs["base420"], str(tmp_path / "o.jpg")], capture_output=True,
                       text=True, env=env)
    assert "host route (JPEGQS_HOST_CODEC)" in r.stderr
    env = dict(os.environ, JPEGQS_CODEC_TRACE="1")
    r = subprocess.run([EXE, "-q", "3", "-i", "0", "--ppm", jpegs["base420"], str(tmp_path / "o.ppm")], capture_output=True,
                       text=True, env=env)
    assert "host route (--ppm)" in r.stderr
    r = subprocess.run([EXE, "-q", "3", "-i", "0", jpegs["prog420"], str(tmp_path / "o.jpg")], capture_output=True,
                       text=True, env=env)
    assert "host route (progressive AC refinement scan without restart markers)" in r.stderr
