"""jpeg_prefix and the encoder's CPU model (jpegqs_cuda_encode_model: the device encoder's steps on
one thread) against the jpegqs tool's own writer.  The tool run with `-n 0` never reaches the CUDA
back end, so its output is jq_write's bytes for the file's coefficients: the model must give them
byte for byte - every decoder flavour, the hard_content sets, progressive inputs, standard and
optimal tables, the optimal-table corner cases - and, after smoothing with the oracle, the bytes the
unmodified reference tool wrote (tests/golden/reference/ref_files.json)."""
import heapq
import os
import subprocess

import numpy as np
import pytest

import decode_files as df
import libjpeg_pixels as lp
import oracle_lib as ol
from golden_io import reference_files
from test_cli import EXE, FILES, REF_TOOL_CASES, file_key, write_jpegs
import jpegqs_b200 as qs
from jpegqs_b200 import cuda
from jpegqs_b200.image import CoefImage, Component, JCS_GRAYSCALE

pytestmark = pytest.mark.skipif(lp.JPEG_SO is None, reason="no libjpeg inside Pillow")


def tool_bytes(tmp_path, data, optimize=False, copy=2):
    src, out = tmp_path / "in.jpg", tmp_path / "out.jpg"
    src.write_bytes(data)
    r = subprocess.run([EXE, "-n", "0", "-i", "0", "-c", str(copy)] + (["-o"] if optimize else []) + [str(src), str(out)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return out.read_bytes()


def model_bytes(data, optimize=False, copy=2):
    pre, ids, tbls = qs.jpeg_prefix(data, copy)
    im = qs.read_jpeg(data)
    got, st = qs.encode_model(im, [c.coef for c in im.comps], pre, ids, tbls, optimize)
    assert st == 0
    return got


@pytest.fixture(scope="module")
def jpegs(tmp_path_factory):
    return write_jpegs(str(tmp_path_factory.mktemp("jpegs")))


@pytest.mark.parametrize("name", [f[0] for f in FILES])
def test_prefix_is_the_tools(jpegs, tmp_path, name):
    data = open(jpegs[name], "rb").read()
    for copy in (0, 1, 2):
        want = tool_bytes(tmp_path, data, copy=copy)
        pre, ids, tbls = qs.jpeg_prefix(data, copy)
        assert want.startswith(pre) and want[len(pre):len(pre) + 2] == b"\xff\xdb", (name, copy)
        assert len(ids) == len(tbls) == len(qs.parse_jpeg(data)[0].comps)


def test_prefix_keeps_markers_between_progressive_scans(tmp_path):
    """A COM and an APP9 after the first scan of a progressive file are copied like any other."""
    data = df.progressive()[0][1]
    sos = data.index(b"\xff\xda")
    nxt = data.index(b"\xff\xc4", sos)                 # the DHT before the second scan
    extra = b"\xff\xfe\x00\x07late!" + b"\xff\xe9\x00\x06app9"
    data = data[:nxt] + extra + data[nxt:]
    for copy in (1, 2):
        pre, _, _ = qs.jpeg_prefix(data, copy)
        assert tool_bytes(tmp_path, data, copy=copy).startswith(pre)
        assert b"late!" in pre and (b"app9" in pre) == (copy == 2)


@pytest.mark.parametrize("name", ["cmyk", "keep_rgb"])
def test_prefix_adobe(tmp_path, name):
    data = dict(df.flavours())[name]
    for copy in (0, 2):
        pre, ids, tbls = qs.jpeg_prefix(data, copy)
        assert b"Adobe" in pre and tool_bytes(tmp_path, data, copy=copy).startswith(pre)
    if name == "cmyk":
        assert tbls == (0, 0, 0, 0)                     # libjpeg's CMYK: one table for all four


ALL = df.flavours() + df.progressive() + [(n, d) for n, _, d in df.hard_sets()]


@pytest.mark.parametrize("optimize", [False, True])
@pytest.mark.parametrize("name", [n for n, _ in ALL])
def test_model_equals_the_tool(tmp_path, name, optimize):
    data = dict(ALL)[name]
    assert model_bytes(data, optimize) == tool_bytes(tmp_path, data, optimize)


@pytest.mark.parametrize("name", [n for n, _ in ALL if n.startswith("writer_")])
def test_written_file_reads_back(name):
    """jpeg_read_coefficients of the file the encoder writes gives back the coefficients it was given, on
    every sampling geometry: grey files whose SOF says 2x2, 3x1, 1x4 or 4x4 among them, whose one scan
    is not interleaved (one block per MCU, in raster order) whatever the factors"""
    data = dict(ALL)[name]
    want = df.libjpeg_coefficients(data)
    for optimize in (False, True):
        got = df.libjpeg_coefficients(model_bytes(data, optimize))
        assert [(c.h_samp, c.v_samp) for c in got.comps] == [(c.h_samp, c.v_samp) for c in want.comps]
        assert all(np.array_equal(a.coef, b.coef) for a, b in zip(got.comps, want.comps)), optimize


def test_sixteen_bit_tables_write_sof1(tmp_path):
    names = [n for n, im, _ in df.hard_sets() if any(c.quant is not None and c.quant.max() > 255 for c in im.comps)]
    assert names
    for n in names:
        data = dict(ALL)[n]
        got = model_bytes(data)
        assert b"\xff\xc1" in got[:got.index(b"\xff\xda")] and got == tool_bytes(tmp_path, data)


def _gray(blocks):
    """A grayscale CoefImage (quant ones) of [hblk, wblk, 64] natural-order blocks."""
    h, w = blocks.shape[:2]
    return CoefImage(width=8 * w, height=8 * h, colorspace=JCS_GRAYSCALE,
                     comps=[Component(coef=blocks.astype(np.int16), quant=np.ones(64, np.uint16))])


def _nat():
    zz = np.zeros(64, int)
    k = 0
    for s in range(15):
        rng = range(s + 1) if s % 2 else range(s, -1, -1)
        for i in rng:
            r, c = i, s - i
            if r < 8 and c < 8:
                zz[k] = r * 8 + c
                k += 1
    return zz


NAT = _nat()


def _written_by_libjpeg(im, tmp_path, optimize):
    """The model on a coefficient set libjpeg can write, against the tool on that file."""
    data = df.coef_writer_jpeg(im)
    assert model_bytes(data, optimize) == tool_bytes(tmp_path, data, optimize)
    return data


def test_flat_image_tables(tmp_path):
    b = np.zeros((6, 9, 64), np.int16)
    b[..., 0] = 5
    _written_by_libjpeg(_gray(b), tmp_path, True)


def test_equal_frequencies(tmp_path):
    b = np.zeros((8, 8, 64), np.int16)
    for s in range(1, 8):
        b[..., NAT[s]] = 1 << (s - 1)                   # symbols (0, 1) .. (0, 7) once per block
    _written_by_libjpeg(_gray(b), tmp_path, True)


def _unlimited_depth(freq):
    heap = [(f, i, 0) for i, f in enumerate(freq) if f] + [(1, 10 ** 6, 0)]
    heapq.heapify(heap)
    depth = {}
    nodes = {}
    k = 10 ** 7
    while len(heap) > 1:
        a, b = heapq.heappop(heap), heapq.heappop(heap)
        k += 1
        nodes[k] = (a[1], b[1])
        heapq.heappush(heap, (a[0] + b[0], k, 0))
    stack = [(heap[0][1], 0)]
    while stack:
        n, d = stack.pop()
        if n in nodes:
            stack += [(nodes[n][0], d + 1), (nodes[n][1], d + 1)]
        else:
            depth[n] = d
    return max(depth.values())


def test_length_limiting_runs(tmp_path):
    """Symbol counts 1, 1, 2, 4, .. 2^16: the unlimited Huffman tree is a chain deeper than 16, so K.3's
    adjustment runs."""
    counts = [1] + [1 << k for k in range(17)]
    syms = [(r, s) for r in (0, 1) for s in range(1, 11)]
    seq = [sym for sym, n in zip(syms, counts) for _ in range(n)]
    blocks, cur, pos = [], np.zeros(64, np.int16), 1
    for r, s in seq:
        if pos + r > 63:
            blocks.append(cur)
            cur, pos = np.zeros(64, np.int16), 1
        pos += r
        cur[NAT[pos]] = 1 << (s - 1)
        pos += 1
    blocks.append(cur)
    while len(blocks) % 16:
        blocks.append(np.zeros(64, np.int16))
    arr = np.array(blocks).reshape(-1, 16, 64)
    freq = [0] * 256
    for blk in arr.reshape(-1, 64):
        z = blk[NAT]
        nz = np.nonzero(z[1:])[0] + 1
        prev = 0
        for k in nz:
            run = k - prev - 1
            freq[0xF0] += run // 16
            freq[(run % 16) << 4 | int(abs(int(z[k]))).bit_length()] += 1
            prev = k
        if prev != 63:
            freq[0] += 1
    assert _unlimited_depth(freq) > 16
    _written_by_libjpeg(_gray(arr), tmp_path, True)


def test_range_limits(tmp_path):
    def status(b, opt):
        im = _gray(b)
        return qs.encode_model(im, [im.comps[0].coef], b"\xff\xd8", (1,), (0,), opt)[1]
    for opt in (False, True):
        b = np.zeros((2, 3, 64), np.int16)
        b[1, 1, NAT[5]] = 1024
        assert status(b, opt) == cuda.ENCODE_RANGE
        b[1, 1, NAT[5]] = -1024
        assert status(b, opt) == cuda.ENCODE_RANGE
        b = np.zeros((2, 3, 64), np.int16)
        b[0, 1, 0] = 2048                               # DC difference of category 12
        assert status(b, opt) == cuda.ENCODE_RANGE
    b = np.zeros((2, 4, 64), np.int16)
    b[..., NAT[9]] = 1023
    b[0, 1, NAT[20]] = -1023
    b[0, 0, 0], b[0, 1, 0], b[0, 2, 0] = -1024, 1016, -1024      # DC differences of category 11
    assert status(b, False) == 0 and status(b, True) == 0
    _written_by_libjpeg(_gray(b), tmp_path, False)
    _written_by_libjpeg(_gray(b), tmp_path, True)


def test_overflow_and_exact_capacity(jpegs):
    data = open(jpegs["base420"], "rb").read()
    pre, ids, tbls = qs.jpeg_prefix(data)
    im = qs.read_jpeg(data)
    arrays = [c.coef for c in im.comps]
    want, st = qs.encode_model(im, arrays, pre, ids, tbls)
    got, st2 = qs.encode_model(im, arrays, pre, ids, tbls, capacity=len(want))
    assert st == st2 == 0 and got == want
    got, st3 = qs.encode_model(im, arrays, pre, ids, tbls, capacity=len(want) - 1)
    assert st3 == cuda.ENCODE_OVERFLOW and len(got) == len(want) - 1


def _tool_flags(args):
    """The jpegqs tool's -q / -n / -f mapping (csrc/jpegqs.c main: quantsmooth.c:380-393's -q table,
    niter 3 unless -n, -f replaces the flags -q chose)."""
    q, n, f = 3, 3, None
    for k in range(0, len(args), 2):
        if args[k] == "-q":
            q = int(args[k + 1])
        elif args[k] == "-n":
            n = int(args[k + 1])
        elif args[k] == "-f":
            f = int(args[k + 1])
    return (qs.quality_to_flags(q) if f is None else f), n


def smoothed_file(data, args):
    """The tool's pipeline restated: read, smooth with the oracle, encode with the model."""
    flags, niter = _tool_flags(args)
    im = qs.read_jpeg(data)
    _, out, up = ol.run_oracle(im, flags, niter, with_upsampled=True)
    pre, ids, tbls = qs.jpeg_prefix(data, 2)
    geo = im.clone()
    for g, o in zip(geo.comps, out.comps):
        g.quant = o.quant
    arrays = [o.coef for o in out.comps]
    if up:
        got, st = qs.encode_model(geo, [arrays[0], im.comps[1].coef, im.comps[2].coef], pre, ids, tbls, "-o" in args,
                                  up=arrays[1:3])
    else:
        got, st = qs.encode_model(geo, arrays, pre, ids, tbls, "-o" in args)
    assert st == 0
    return got, up


@pytest.mark.parametrize("name,args", REF_TOOL_CASES)
def test_reference_tools_bytes(jpegs, name, args):
    import hashlib
    got, _ = smoothed_file(open(jpegs[name], "rb").read(), args)
    assert hashlib.sha256(got).hexdigest() == reference_files()["jpegqs_ref"][file_key(name, args)]


def _a(x):
    return (x + 255) // 256 * 256


def _units(im, up):
    cs = im.comps
    mh, mv = max(c.h_samp for c in cs), max(c.v_samp for c in cs)
    u = -(-im.width // (8 * mh)) * -(-im.height // (8 * mv)) * sum(c.h_samp * c.v_samp for c in cs)
    if up:
        u = max(u, -(-im.width // 8) * -(-im.height // 8) * 3)
    return u


@pytest.mark.parametrize("name", ["420_q75", "422_q30", "444_q100", "gray_q75", "cmyk", "keep_rgb", "writer_411", "size_1x1"])
def test_workspace_and_bound_formulas(name):
    im, _ = qs.parse_jpeg(dict(df.flavours())[name])
    up = cuda.upsample_can_trigger(im, 4)
    U = _units(im, up)
    T, W = -(-U // 256), -(-U * 1665 // 32) + 2
    ws = 32768 + _a(2 * U) + _a(8 * T) + _a(4 * W) + _a(4 * -(-4 * W // 4096))
    assert qs.encode_workspace_bytes([im]) == qs.encode_workspace_bytes([im], True) == ws
    assert qs.encode_workspace_bytes([im, im]) == 2 * ws
    assert qs.encode_bound(im, 321) == 321 + 1680 + 2 * -(-U * 1665 // 8)


def test_argument_checks():
    data = dict(df.flavours())["420_q75"]
    pre, ids, tbls = qs.jpeg_prefix(data)
    im = qs.read_jpeg(data)
    arrays = [c.coef for c in im.comps]
    with pytest.raises(cuda.QsError):
        qs.jpeg_prefix(b"not a jpeg")
    with pytest.raises(ValueError):
        qs.encode_model(im, arrays[:2], pre, ids, tbls)
    with pytest.raises(ValueError):
        qs.encode_model(im, arrays, pre, ids[:2], tbls)
    with pytest.raises(cuda.QsError):
        qs.encode_model(im, arrays, pre, ids, (0, 1, 4))
    with pytest.raises(cuda.QsError):
        qs.encode_model(im, arrays, pre, ids, tbls, capacity=len(pre) - 1)
    bad = im.clone()
    bad.comps[0].h_samp = 5
    with pytest.raises(cuda.QsError):
        qs.encode_workspace_bytes([bad])
    torch = pytest.importorskip("torch")
    with pytest.raises(ValueError):
        qs.encode_async([im], [[torch.from_numpy(a) for a in arrays]], [(torch.from_numpy(np.frombuffer(pre, np.uint8).copy()), ids, tbls)])
