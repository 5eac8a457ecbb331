"""Progressive files from the compressor, without a GPU: compress_model(progressive=True) writes exactly
the bytes of Pillow's Image.fromarray(P).save(f, "JPEG", quality=q, subsampling=s, optimize=o,
progressive=True), over test_compress_cpu's seeded sweep (grey and RGB, every sampling, sizes on both
sides of 8 and 16, qualities 1..100, five content kinds, both optimize values), with libjpeg-turbo's
SIMD code switched off, and on targeted content: EOB runs longer than 0x7FFF blocks, runs cut by the
937 correction-bit limit, folded and emitted ZRLs, negative odd DCs and MCU padding with odd block
counts.  A Python restatement of libjpeg's progressive coder (jcphuff.c, the state machine as written
there) over test_compress_cpu's numpy coefficients equals Pillow, and six plausible mistakes in it each
give a file Pillow does not write.  Also the C ABI's progressive bit, bound and workspace, and the
Python keyword."""
import ctypes as C
import io
import os
import subprocess
import sys

import numpy as np
import pytest

Image = pytest.importorskip("PIL.Image")
ImageFile = pytest.importorskip("PIL.ImageFile")
ImageFile.MAXBLOCK = 1 << 28

from jpegqs_b200 import cuda
from test_compress_cpu import CASES, SUBS, content, restated


def pillow(a, quality, subsampling, optimize=False):
    b = io.BytesIO()
    Image.fromarray(a if a.shape[2] == 3 else a[:, :, 0]).save(b, "JPEG", quality=quality, subsampling=subsampling,
                                                               optimize=optimize, progressive=True)
    return b.getvalue()


def model(a, q, s, o=False):
    return cuda.compress_model(a, q, s, o, progressive=True)


@pytest.mark.parametrize("i", range(0, len(CASES), 30))
def test_model_equals_pillow(i):
    for a, q, s, o in CASES[i:i + 30]:
        assert model(a, q, s, o) == pillow(a, q, s, o), (a.shape, q, s, o)


def test_optimize_changes_no_byte():
    for a, q, s, _ in CASES[::37]:
        assert model(a, q, s, False) == model(a, q, s, True) == pillow(a, q, s, False)


_SIMD_OFF = r'''
import io, sys
import numpy as np
from PIL import Image, ImageFile
ImageFile.MAXBLOCK = 1 << 28
d = np.load(sys.argv[1])
out = []
for k in range(int(d["n"])):
    a = d[f"a{k}"]
    b = io.BytesIO()
    Image.fromarray(a if a.shape[2] == 3 else a[:, :, 0]).save(b, "JPEG", quality=int(d[f"q{k}"]),
        subsampling=str(d[f"s{k}"]), optimize=bool(d[f"o{k}"]), progressive=True)
    out.append(b.getvalue())
open(sys.argv[2], "wb").write(b"".join(len(x).to_bytes(8, "little") + x for x in out))
'''


def test_model_equals_pillow_without_simd(tmp_path):
    """libjpeg-turbo's C code is the contract: jcphuff.c's SIMD prepare routines off give the same files"""
    sub = CASES[::9] + [(t[0], t[1], t[2], False) for t in TARGETED[:3]]
    arrays = {"n": len(sub)}
    for k, (a, q, s, o) in enumerate(sub):
        arrays.update({f"a{k}": a, f"q{k}": q, f"s{k}": s, f"o{k}": int(o)})
    np.savez(tmp_path / "in.npz", **arrays)
    script = tmp_path / "save.py"
    script.write_text(_SIMD_OFF)
    env = dict(os.environ, JSIMD_FORCENONE="1")
    subprocess.run([sys.executable, str(script), str(tmp_path / "in.npz"), str(tmp_path / "out.bin")], check=True, env=env)
    raw, pos = (tmp_path / "out.bin").read_bytes(), 0
    for a, q, s, o in sub:
        n = int.from_bytes(raw[pos:pos + 8], "little")
        assert model(a, q, s, o) == raw[pos + 8:pos + 8 + n], (a.shape, q, s, o)
        pos += 8 + n


# ---- targeted content ----
def _only_corrections_block():
    """an 8 x 8 grey block whose q100 coefficients are 0 or at least 4 in magnitude, at least 48 of them:
    tiled, every block of the two refinement scans has correction bits only"""
    for seed in range(1000):
        b = np.random.RandomState(seed).randint(0, 256, (8, 8, 1)).astype(np.uint8)
        coef = restated(b, 100, "4:4:4", False)[1][0][0, 0]
        ac = np.abs(coef[1:].astype(int))
        if ((ac == 0) | (ac >= 4)).all() and (ac >= 4).sum() >= 48:
            return b
    raise AssertionError("no block found")


def _targeted():
    rng = np.random.RandomState(31)
    out = [(np.full((1400, 1600, 1), 77, np.uint8), 75, "4:2:0", "EOB runs past 0x7FFF blocks"),
           (np.tile(_only_corrections_block(), (12, 10, 1)), 100, "4:4:4", "runs cut by the 937-bit limit"),
           (np.tile(_only_corrections_block(), (6, 7, 3)), 100, "4:2:0", "correction-bit runs in colour"),
           ((rng.randint(0, 40, (33, 17, 3))).astype(np.uint8), 90, "4:4:4", "negative odd DCs"),
           (np.clip(rng.normal(128, 30, (64, 64, 1)), 0, 255).astype(np.uint8), 30, "4:4:4", "sparse: long zero gaps")]
    for h, w in ((24, 40), (40, 24), (24, 24), (23, 39), (56, 72)):        # odd luma block counts
        for s in ("4:2:0", "4:2:2"):
            out.append((rng.randint(0, 256, (h, w, 3)).astype(np.uint8), 90, s, f"padding {h}x{w} {s}"))
    return out


TARGETED = _targeted()


@pytest.mark.parametrize("k", range(len(TARGETED)))
def test_targeted_content(k):
    a, q, s, what = TARGETED[k]
    assert model(a, q, s) == pillow(a, q, s), what


# ---- a Python restatement of libjpeg's progressive coder, and mistakes it could make ----
NAT = [0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21,
       28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61,
       54, 47, 55, 62, 63]
COLOUR = [((0, 1, 2), 0, 0, 0, 1), ((0,), 1, 5, 0, 2), ((2,), 1, 63, 0, 1), ((1,), 1, 63, 0, 1), ((0,), 6, 63, 0, 2),
          ((0,), 1, 63, 2, 1), ((0, 1, 2), 0, 0, 1, 0), ((2,), 1, 63, 1, 0), ((1,), 1, 63, 1, 0), ((0,), 1, 63, 1, 0)]
GREY = [((0,), 0, 0, 0, 1), ((0,), 1, 5, 0, 2), ((0,), 6, 63, 0, 2), ((0,), 1, 63, 2, 1), ((0,), 0, 0, 1, 0),
        ((0,), 1, 63, 1, 0)]
MUTANTS = ["pad_refine_zero", "pad_clamp", "no_be_limit", "zrl_unfolded", "one_table_pair", "truncating_shift"]


def gen_optimal(freq):
    """jchuff.c jpeg_gen_optimal_table: (BITS[1..16], HUFFVAL)"""
    freq = list(freq) + [1]
    size, others = [0] * 257, [-1] * 257
    while True:
        c1 = c2 = -1
        v = 10 ** 9
        for i in range(257):
            if freq[i] and freq[i] <= v:
                v, c1 = freq[i], i
        v = 10 ** 9
        for i in range(257):
            if freq[i] and freq[i] <= v and i != c1:
                v, c2 = freq[i], i
        if c2 < 0:
            break
        freq[c1] += freq[c2]
        freq[c2] = 0
        size[c1] += 1
        while others[c1] >= 0:
            c1 = others[c1]
            size[c1] += 1
        others[c1] = c2
        size[c2] += 1
        while others[c2] >= 0:
            c2 = others[c2]
            size[c2] += 1
    bits = [0] * 33
    for s in size:
        if s:
            bits[s] += 1
    for i in range(32, 16, -1):
        while bits[i] > 0:
            j = i - 2
            while bits[j] == 0:
                j -= 1
            bits[i] -= 2
            bits[i - 1] += 1
            bits[j + 1] += 2
            bits[j] -= 1
    i = 16
    while bits[i] == 0:
        i -= 1
    bits[i] -= 1
    return bits[1:17], [j for l in range(1, 33) for j in range(256) if size[j] == l]


def codes(bits, vals):
    out, code, k = {}, 0, 0
    for l in range(1, 17):
        for _ in range(bits[l - 1]):
            out[vals[k]] = (code, l)
            code, k = code + 1, k + 1
        code <<= 1
    return out


def _dc_units(arrays, factors, mutant):
    """(component, DC) per unit of an interleaved DC scan, MCU padding included (jccoefct.c
    compress_first_pass's dummy blocks)"""
    mx = -(-arrays[0].shape[1] // factors[0][0])
    my = -(-arrays[0].shape[0] // factors[0][1])
    for y in range(my):
        for x in range(mx):
            for c, (arr, (hs, vs)) in enumerate(zip(arrays, factors)):
                hb, wb = arr.shape[:2]
                for v in range(vs):
                    for h in range(hs):
                        bx, by = x * hs + h, y * vs + v
                        if mutant == "pad_clamp":
                            sx, sy = min(bx, wb - 1), min(by, hb - 1)
                        elif by < hb:
                            sx, sy = min(bx, wb - 1), by
                        else:
                            sx, sy = min(x * hs + hs - 1, wb - 1), hb - 1
                        yield c, int(arr[sy, sx, 0]), bx >= wb or by >= hb


def _scan_ops(a_units, blocks, comps, ss, se, ah, al, mutant):
    """the scan's ('sym', table, symbol, value bits, size) and ('bits', [bit, ...]) in jcphuff.c's order"""
    ops = []
    shift = (lambda v: int(v / (1 << al))) if mutant == "truncating_shift" else (lambda v: v >> al)
    if ss == 0:
        last = [0, 0, 0]
        for c, dc, pad in a_units:
            if ah == 0:
                v = shift(dc)
                d, last[c] = v - last[c], v
                n = abs(d).bit_length()
                ops.append(("sym", 1 if c else 0, n, d if d >= 0 else d + (1 << n) - 1, n))
            else:
                ops.append(("bits", [0 if pad and mutant == "pad_refine_zero" else (dc >> al) & 1]))
        return ops
    state = {"run": 0, "be": []}

    def flush():
        if state["run"]:
            n = state["run"].bit_length() - 1
            ops.append(("sym", 0, n << 4, state["run"] & ((1 << n) - 1), n))
            ops.append(("bits", state["be"]))
            state["run"], state["be"] = 0, []
    for b in blocks:
        z = [int(b[NAT[k]]) for k in range(64)]
        av = [abs(z[k]) >> al for k in range(64)]
        r, br = 0, []
        if ah == 0:
            for k in range(ss, se + 1):
                if not av[k]:
                    r += 1
                    continue
                flush()
                while r > 15:
                    ops.append(("sym", 0, 0xF0, 0, 0))
                    r -= 16
                n = av[k].bit_length()
                ops.append(("sym", 0, r << 4 | n, av[k] if z[k] > 0 else ~av[k] & ((1 << n) - 1), n))
                r = 0
            if r:
                state["run"] += 1
                if state["run"] == 0x7FFF:
                    flush()
            continue
        eob = max([k for k in range(ss, se + 1) if av[k] == 1], default=-1)
        for k in range(ss, se + 1):
            if not av[k]:
                r += 1
                continue
            while r > 15 and (k <= eob or mutant == "zrl_unfolded"):
                flush()
                ops.append(("sym", 0, 0xF0, 0, 0))
                r -= 16
                ops.append(("bits", br))
                br = []
            if av[k] > 1:
                br.append(av[k] & 1)
                continue
            flush()
            ops.append(("sym", 0, (r << 4) | 1, 1 if z[k] > 0 else 0, 1))
            ops.append(("bits", br))
            br, r = [], 0
        if r or br:
            state["run"] += 1
            state["be"] += br
            if state["run"] == 0x7FFF or (len(state["be"]) > 937 and mutant != "no_be_limit"):
                flush()
    flush()
    return ops


def restated_progressive(a, q, s, mutant=None):
    seq, arrays, _ = restated(a, q, s, False)
    c = len(arrays)
    si = SUBS.index(s) if isinstance(s, str) else s
    lh, lv = (1, 1) if c == 1 or si == 0 else (2, 1) if si == 1 else (2, 2)
    factors = [(lh, lv), (1, 1), (1, 1)] if c == 3 else [(1, 1)]
    i = 2                                            # the sequential file's prefix, DQT and SOF -> SOF2
    while seq[i + 1] not in (0xC0, 0xC1):
        i += 2 + int.from_bytes(seq[i + 2:i + 4], "big")
    sof_len = 2 + int.from_bytes(seq[i + 2:i + 4], "big")
    out = bytearray(seq[:i] + b"\xff\xc2" + seq[i + 2:i + sof_len])
    script = COLOUR if c == 3 else GREY
    scans = []
    for comps, ss, se, ah, al in script:
        if ss == 0:
            units = list(_dc_units(arrays, factors, mutant)) if c == 3 else \
                [(0, int(v), False) for v in arrays[0][:, :, 0].ravel()]
            ops = _scan_ops(units, None, comps, ss, se, ah, al, mutant)
        else:
            ops = _scan_ops(None, arrays[comps[0]].reshape(-1, 64), comps, ss, se, ah, al, mutant)
        scans.append(ops)
    if mutant == "one_table_pair":                   # one table per (class, id) over all scans
        total = {}
        for (comps, ss, se, ah, al), ops in zip(script, scans):
            for op in ops:
                if op[0] == "sym":
                    key = (ss > 0, op[1] if ss == 0 else min(comps[0], 1))
                    total.setdefault(key, [0] * 256)[op[2]] += 1
    for (comps, ss, se, ah, al), ops in zip(script, scans):
        tables = {}
        used = sorted({op[1] for op in ops if op[0] == "sym"}) if not (ss == 0 and ah) else []
        for t in used:
            freq = [0] * 256
            for op in ops:
                if op[0] == "sym" and op[1] == t:
                    freq[op[2]] += 1
            tid = t if ss == 0 else min(comps[0], 1)
            if mutant == "one_table_pair":
                freq = total[(ss > 0, tid)]
            bits, vals = gen_optimal(freq)
            out += b"\xff\xc4" + (19 + len(vals)).to_bytes(2, "big") + bytes([(0x10 if ss else 0) | tid] + bits + vals)
            tables[t] = codes(bits, vals)
        out += b"\xff\xda" + (6 + 2 * len(comps)).to_bytes(2, "big") + bytes([len(comps)])
        for k in comps:
            out += bytes([k + 1, (1 if ss == 0 and ah == 0 and k else 0) << 4 | (1 if se and k else 0)])
        out += bytes([ss, se, ah << 4 | al])
        bitstr = []
        for op in ops:
            if op[0] == "sym":
                code, n = tables[op[1]][op[2]]
                bitstr.append(format(code, f"0{n}b"))
                if op[4]:
                    bitstr.append(format(op[3], f"0{op[4]}b"))
            else:
                bitstr.append("".join(str(x) for x in op[1]))
        bitstr = "".join(bitstr)
        bitstr += "1" * (-len(bitstr) % 8)
        for j in range(0, len(bitstr), 8):
            v = int(bitstr[j:j + 8], 2)
            out += bytes([v, 0]) if v == 0xFF else bytes([v])
    return bytes(out + b"\xff\xd9")


MUTANT_CASES = [(content(np.random.RandomState(18), 24, 40, 3, "random"), 90, "4:2:0"),
                (content(np.random.RandomState(5), 40, 24, 3, "normal"), 85, "4:2:2"),
                ((np.random.RandomState(6).randint(0, 40, (17, 33, 3))).astype(np.uint8), 90, "4:4:4"),
                (TARGETED[1][0], 100, "4:4:4"),
                (TARGETED[4][0], 30, "4:4:4"),
                (content(np.random.RandomState(7), 40, 40, 1, "hard"), 75, "4:2:0")]


def test_restatement_equals_pillow_and_model():
    for a, q, s in MUTANT_CASES:
        want = pillow(a, q, s)
        assert restated_progressive(a, q, s) == want == model(a, q, s), (a.shape, q, s)


@pytest.mark.parametrize("mutant", MUTANTS)
def test_each_mutant_differs_from_pillow(mutant):
    assert any(restated_progressive(a, q, s, mutant) != pillow(a, q, s) for a, q, s in MUTANT_CASES), mutant


# ---- the C ABI and the Python keyword ----
def test_progressive_bit_and_rejected_values():
    lib = cuda.load()
    a = content(np.random.RandomState(9), 37, 29, 3, "normal")
    out = np.zeros(1 << 16, np.uint8)
    n, st, size = C.c_uint64(0), C.c_int32(0), C.c_size_t(0)
    pin = cuda._PixelsIn(a.ctypes.data, 29, 37, 3, 87)
    files = []
    for opt in (0x100, 0x101):
        jp = cuda._JpegParams(80, 1, opt)
        assert lib.jpegqs_cuda_compress_model(C.byref(pin), C.byref(jp), out.ctypes.data, out.size, C.byref(n),
                                              C.byref(st)) == 0 and st.value == 0
        files.append(out[:n.value].tobytes())
    assert files[0] == files[1] == pillow(a, 80, "4:2:2")
    for opt in (2, 4, 0x200, 0x102, -1):
        jp = cuda._JpegParams(80, 1, opt)
        assert lib.jpegqs_cuda_compress_model(C.byref(pin), C.byref(jp), out.ctypes.data, out.size, C.byref(n),
                                              C.byref(st)) == -2, opt
        assert lib.jpegqs_cuda_compress_bound(C.byref(pin), C.byref(jp), C.byref(size)) == -2
        assert lib.jpegqs_cuda_compress_workspace_bytes(1, C.byref(pin), C.byref(jp), C.byref(size)) == -2
    cap = len(files[0]) - 1
    jp = cuda._JpegParams(80, 1, 0x100)
    assert lib.jpegqs_cuda_compress_model(C.byref(pin), C.byref(jp), out.ctypes.data, cap, C.byref(n), C.byref(st)) == 0
    assert st.value == cuda.ENCODE_OVERFLOW and n.value == len(files[0])


def test_bound_and_workspace_formulas():
    lib = cuda.load()
    size = C.c_size_t(0)

    def a256(x):
        return (x + 255) // 256 * 256
    for w, h, ch, s in ((1, 1, 1, 0), (1920, 1080, 3, 2), (33, 17, 3, 1), (100, 7, 3, 0), (64, 64, 1, 2),
                        (7680, 4320, 3, 2), (65535, 65535, 3, 0)):
        pin, jp = cuda._PixelsIn(None, w, h, ch, w * ch), cuda._JpegParams(75, s, 0x101)
        lh, lv = (1, 1) if ch == 1 or s == 0 else (2, 1) if s == 1 else (2, 2)
        blocks = [(-(-(-(-w * (lh if k == 0 else 1) // lh)) // 8), -(-(-(-h * (lv if k == 0 else 1) // lv)) // 8))
                  for k in range(ch)]
        if ch == 1:
            U = blocks[0][0] * blocks[0][1]
        else:
            U = -(-w // (8 * lh)) * -(-h // (8 * lv)) * (lh * lv + 2)
        assert lib.jpegqs_cuda_compress_bound(C.byref(pin), C.byref(jp), C.byref(size)) == 0
        assert size.value == 20 + 6000 + 2 * (-(-U * 3928 // 8) + 10)
        coef = sum(a256(128 * bw * bh) for bw, bh in blocks)

        def r(x):
            return -(-x // 256) * 256
        if ch == 1:
            V = 6 * r(U)
        else:
            Y, Cb, Cr = (bw * bh for bw, bh in blocks)
            V = 2 * r(U) + 4 * r(Y) + 2 * r(Cb) + 2 * r(Cr)
        Wd = -(-U * 3928 // 32) + 10242
        enc = 73728 + a256(V) + a256(2 * V) + a256(8 * V) + a256(2 * V) + a256(8 * (V // 256)) + a256(4 * Wd) + \
            a256(4 * -(-4 * Wd // 4096))
        assert lib.jpegqs_cuda_compress_workspace_bytes(1, C.byref(pin), C.byref(jp), C.byref(size)) == 0
        assert size.value == 256 + coef + enc, (w, h, ch, s)


def test_python_keywords():
    a = content(np.random.RandomState(2), 20, 30, 3, "random")
    assert cuda.compress_model(a, 70, "4:2:0", progressive=True) == pillow(a, 70, "4:2:0")
    assert cuda.compress_model(a, 70, "4:2:0", progressive=False) == cuda.compress_model(a, 70, "4:2:0")
    assert cuda.compress_bound(a.shape, 70, "4:2:0", progressive=True) > cuda.compress_bound(a.shape, 70, "4:2:0")
    for bad in (1, 0, "yes", None, 1.0):
        with pytest.raises(ValueError, match="progressive"):
            cuda.compress_model(a, 70, "4:2:0", progressive=bad)
        with pytest.raises(ValueError, match="progressive"):
            cuda.compress_bound(a.shape, 70, "4:2:0", progressive=bad)
