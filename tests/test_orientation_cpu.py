"""jpegqs_cuda_jpeg_orientation against Pillow (no GPU): the orientation ImageOps.exif_transpose applies
to a file, for the quirks of Pillow's EXIF and XMP readers, a seeded fuzz of mutated payloads, and the
Python wrappers' argument checks."""
import ctypes as C
import io
import random
import struct
import warnings

import pytest
from PIL import Image

import decode_files as df
from test_resize_cpu import _unbound
from jpegqs_b200 import cuda

TRANSPOSES = {2, 3, 4, 5, 6, 7, 8}          # the keys of exif_transpose's method dict
XMP_ID = b"http://ns.adobe.com/xap/1.0/\0"
TYPES = {"BYTE": (1, "B"), "ASCII": (2, "s"), "SHORT": (3, "H"), "LONG": (4, "L"), "RATIONAL": (5, "LL"),
         "SBYTE": (6, "b"), "UNDEFINED": (7, "B"), "SSHORT": (8, "h"), "SLONG": (9, "l"), "SRATIONAL": (10, "ll"),
         "FLOAT": (11, "f"), "DOUBLE": (12, "d")}


def pillow_orientation(data: bytes) -> int:
    """what ImageOps.exif_transpose(Image.open(f)) applies: getexif's 0x0112, looked up in its dict"""
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        try:
            with Image.open(io.BytesIO(data)) as im:
                o = im.getexif().get(0x0112, 1)
        except Exception:
            o = 1
    try:
        return o if o in TRANSPOSES else 1
    except TypeError:                         # unhashable
        return 1


def orientation(data: bytes) -> int:
    lib = cuda.load()
    o = C.c_int32(-5)
    assert lib.jpegqs_cuda_jpeg_orientation(data, len(data), C.byref(o)) == 0, lib.jpegqs_cuda_last_error(None)
    return o.value


def segment(marker: int, payload: bytes) -> bytes:
    return bytes([0xFF, marker]) + struct.pack(">H", len(payload) + 2) + payload


def splice(base: bytes, *payloads: bytes) -> bytes:
    """APP1 segments with these payloads right after the SOI"""
    return base[:2] + b"".join(segment(0xE1, p) for p in payloads) + base[2:]


def entry(tag, typ, count, value: bytes, e: str) -> bytes:
    return struct.pack(e + "HHL", tag, typ, count) + value.ljust(4, b"\0")[:4]


def exif(entries, e: str = "<", ifd: int = 8, tail: bytes = b"", prefix: bytes = b"Exif\0\0") -> bytes:
    """an EXIF payload: TIFF header, IFD0 at `ifd` holding `entries` (bytes each), then `tail`"""
    head = (b"II*\0" if e == "<" else b"MM\0*") + struct.pack(e + "L", ifd)
    body = head.ljust(ifd, b"\0") + struct.pack(e + "H", len(entries)) + b"".join(entries) + struct.pack(e + "L", 0)
    return prefix + body + tail


def tag(name: str, values, e: str = "<", at: int = None) -> bytes:
    """an 0x0112 entry of type `name` with these values, inline or (at) at an offset"""
    typ, f = TYPES[name]
    if name == "ASCII":
        data, count = values, len(values)
    else:
        data = b"".join(struct.pack(e + f, *(v if isinstance(v, tuple) else (v,))) for v in values)
        count = len(values)
    return entry(0x0112, typ, count, struct.pack(e + "L", at) if at is not None else data, e)


def xmp(value: str, form: str = 'attr') -> bytes:
    body = f'<x:xmpmeta><rdf:Description tiff:Orientation="{value}"/></x:xmpmeta>' if form == "attr" else \
        f"<x:xmpmeta><tiff:Orientation>{value}</tiff:Orientation></x:xmpmeta>"
    return XMP_ID + body.encode()


@pytest.fixture(scope="module")
def base():
    return df.pillow_jpeg(24, 16, quality=80)


# the quirks table: (payloads, Pillow's orientation)
QUIRKS = {
    "short 6 LE": ([exif([tag("SHORT", [6])])], 6),
    "short 6 BE": ([exif([tag("SHORT", [6], ">")], ">")], 6),
    "long 6": ([exif([tag("LONG", [6])])], 6),
    "float 6.0": ([exif([tag("FLOAT", [6.0])])], 6),
    "rational 12/2": ([exif([tag("RATIONAL", [(12, 2)], at=26)], tail=struct.pack("<LL", 12, 2))], 6),
    "short count 2 {6, 3}": ([exif([tag("SHORT", [6, 3])])], 6),
    "byte 6": ([exif([tag("BYTE", [6])])], 1),
    "undefined 6": ([exif([tag("UNDEFINED", [6])])], 1),
    "ascii 6": ([exif([tag("ASCII", b"6")])], 1),
    "short 9": ([exif([tag("SHORT", [9])])], 1),
    "short 9 with xmp 8": ([exif([tag("SHORT", [9])]), xmp("8")], 1),
    "xmp-only 8": ([xmp("8")], 8),
    "xmp-only 8, element form": ([xmp("8", "elem")], 8),
    "bad tiff header": ([b"Exif\0\0XX*\0\x08\0\0\0" + b"\0" * 8], 1),
    "bad tiff header with xmp 8": ([b"Exif\0\0XX*\0\x08\0\0\0" + b"\0" * 8, xmp("8")], 1),
    # beyond the table
    "several exif app1s": ([exif([tag("SHORT", [1])], tail=b"\0" * 4), b"Exif\0\0" + b"\xff" * 8], 1),
    "exif after xmp": ([xmp("3"), exif([tag("SHORT", [5])])], 5),
    "exif without the tag, xmp 7": ([exif([entry(0x010F, 2, 4, b"abc\0", "<")]), xmp("7")], 7),
    "last xmp wins": ([xmp("3"), xmp("4")], 4),
    "xmp 9": ([xmp("9")], 1),
    "ifd offset past the end": ([exif([tag("SHORT", [6])], ifd=8)[:6] + b"II*\0\xff\0\0\0"], 1),
    "ifd offset past the end, xmp 2": ([b"Exif\0\0II*\0\xff\0\0\0", xmp("2")], 2),
    "value offset past the end": ([exif([tag("SHORT", [6, 6, 6], at=4000)])], 1),
    "value offset past the end after a tag": ([exif([tag("SHORT", [3]), tag("SHORT", [6, 6, 6], at=4000)])], 3),
    "count 0": ([exif([entry(0x0112, 3, 0, b"\x06\0", "<")])], 1),
    "count 0, xmp 6": ([exif([entry(0x0112, 3, 0, b"\x06\0", "<")]), xmp("6")], 6),
    "ifd cut mid-entry": ([exif([tag("SHORT", [4]), tag("SHORT", [6])])[:6 + 8 + 2 + 12 + 5]], 4),
    "last duplicate wins": ([exif([tag("SHORT", [6]), tag("SHORT", [3])])], 3),
    "unknown type skipped": ([exif([tag("SHORT", [6]), entry(0x0112, 14, 1, b"\x03", "<")])], 6),
    "sshort 8": ([exif([tag("SSHORT", [8])])], 8),
    "slong 2": ([exif([tag("SLONG", [2])])], 2),
    "sbyte 7": ([exif([tag("SBYTE", [7])])], 7),
    "double 5.0": ([exif([tag("DOUBLE", [5.0], at=26)], tail=struct.pack("<d", 5.0))], 5),
    "float 6.5": ([exif([tag("FLOAT", [6.5])])], 1),
    "srational -12/-2": ([exif([tag("SRATIONAL", [(-12, -2)], at=26)], tail=struct.pack("<ll", -12, -2))], 6),
    "rational 6/0": ([exif([tag("RATIONAL", [(6, 0)], at=26)], tail=struct.pack("<LL", 6, 0))], 1),
    "swapped tiff magic": ([b"Exif\0\0II\0*\x08\0\0\0" + struct.pack("<H", 1) + tag("SHORT", [8]) + b"\0" * 4], 8),
    "bigtiff header": ([b"Exif\0\0II+\0\x08\0\0\0" + struct.pack("<H", 1) + tag("SHORT", [8]) + b"\0" * 4], 1),
    "short header": ([b"Exif\0\0II*\0\x08\0"], 1),
    "empty exif": ([b"Exif\0\0", xmp("5")], 5),
    "doubled exif prefix": ([b"Exif\0\0" + exif([tag("SHORT", [6])])], 6),
    "two exif blocks joined": ([exif([tag("SHORT", [2])])[:-4], b"Exif\0\0" + b"\0" * 4], 2),
}


@pytest.mark.parametrize("name", sorted(QUIRKS))
def test_quirks_equal_pillow(base, name):
    payloads, want = QUIRKS[name]
    data = splice(base, *payloads)
    assert pillow_orientation(data) == want, "the table no longer describes the installed Pillow"
    assert orientation(data) == want


def test_no_metadata_and_plain_files(base):
    assert orientation(base) == 1
    for name, f in df.flavours() + df.progressive():
        assert orientation(f) == pillow_orientation(f) == 1, name


def test_markers_after_the_first_sos_are_ignored():
    prog = df.pillow_jpeg(48, 32, quality=80, progressive=True)
    second = prog.index(b"\xff\xda", prog.index(b"\xff\xda") + 2)
    data = prog[:second] + segment(0xE1, exif([tag("SHORT", [6])])) + prog[second:]
    assert pillow_orientation(data) == 1
    assert orientation(data) == 1
    # the same segment before the first scan counts
    assert orientation(splice(prog, exif([tag("SHORT", [6])]))) == 6


def mutate(rng: random.Random, p: bytearray) -> bytes:
    for _ in range(rng.randint(1, 4)):
        k = rng.randrange(5)
        if k == 0 and p:                                    # byte flips
            for _ in range(rng.randint(1, 3)):
                p[rng.randrange(len(p))] ^= 1 << rng.randrange(8)
        elif k == 1 and p:                                  # truncation
            del p[rng.randrange(len(p)):]
        elif k == 2 and len(p) >= 16:                       # a count, offset or length field
            at = rng.randrange(6, len(p) - 3)
            v = rng.choice([0, 1, 2, 3, 4, 5, 6, 8, 9, 12, 13, 16, 255, 0x112, 0xFFFF, rng.randrange(1 << 16)])
            p[at:at + 2] = struct.pack(rng.choice("<>") + "H", v)
        elif k == 3 and len(p) >= 16:                       # a 32-bit offset
            at = rng.randrange(6, len(p) - 5)
            p[at:at + 4] = struct.pack(rng.choice("<>") + "L", rng.choice([0, 8, 26, len(p), len(p) - 6, 1 << 31,
                                                                         rng.randrange(len(p) + 64)]))
        else:                                               # a digit of an XMP value
            i = p.find(b"Orientation")
            if i >= 0 and i + 13 < len(p):
                p[i + rng.choice([12, 13])] = rng.choice(b"0123456789=\">x")
    return bytes(p)


def seeds():
    e = "<"
    return [
        exif([tag("SHORT", [6])]), exif([tag("SHORT", [8], ">")], ">"),
        exif([entry(0x010F, 2, 8, struct.pack("<L", 38), e), tag("SHORT", [3])], tail=b"Canon\0\0\0"),
        exif([tag("RATIONAL", [(12, 2)], at=26)], tail=struct.pack("<LL", 12, 2)),
        exif([tag("FLOAT", [5.0]), tag("LONG", [7])]),
        exif([tag("SHORT", [2, 6, 6])], tail=b"\0" * 8),
        xmp("6"), xmp("8", "elem"),
        exif([tag("DOUBLE", [4.0], at=26)], tail=struct.pack("<d", 4.0)),
    ]


def test_fuzz_equals_pillow(base):
    rng = random.Random(20261017)
    bad = []
    sd = seeds()
    for it in range(3000):
        payloads = [mutate(rng, bytearray(rng.choice(sd))) for _ in range(rng.choice([1, 1, 1, 2, 3]))]
        payloads = [p for p in payloads if len(p) <= 60000]
        data = splice(base, *payloads)
        got, want = orientation(data), pillow_orientation(data)
        if got != want:
            bad.append((it, got, want, payloads))
    assert not bad, f"{len(bad)} mismatches, first {bad[:3]}"


def test_reader_rejects_and_null_arguments():
    lib = cuda.load()
    o = C.c_int32(-5)
    assert lib.jpegqs_cuda_jpeg_orientation(b"not a jpeg", 10, C.byref(o)) == -2
    assert lib.jpegqs_cuda_last_error(None)
    assert o.value == -5
    assert lib.jpegqs_cuda_jpeg_orientation(None, 0, C.byref(o)) == -2
    assert cuda.exif_orientation(splice(df.pillow_jpeg(8, 8), exif([tag("SHORT", [7])]))) == 7
    with pytest.raises(cuda.QsError):
        cuda.exif_orientation(b"\xff\xd8\xff")
    with pytest.raises(TypeError):
        cuda.exif_orientation("x")


def test_python_orientation_arguments():
    good = df.pillow_jpeg(64, 48, quality=75)
    ctx = _unbound()
    for f in (cuda.QsContext.decode_pixels, cuda.QsContext.reencode):
        assert f(ctx, [], 0, 3, orientation="exif") == []
        for bad in (9, 0, -1, "EXIF", "none", True, 6.0, [1], [1, 2, 3], [1, 9], [1, -1], [1, "6"], [1, None], b"\x01\x02"):
            with pytest.raises(ValueError, match="orientation"):
                f(ctx, [good, good], 0, 3, orientation=bad)
    # the crop is in the oriented picture: 48 x 64 at 5..8
    with pytest.raises(ValueError, match="file 0: crop .* outside the 48 x 64 picture"):
        cuda.QsContext.decode_pixels(ctx, [good], 0, 3, crop=[(0, 0, 64, 48)], orientation=6)
    with pytest.raises(ValueError, match="file 0: crop .* outside the 24 x 32 picture"):
        cuda.QsContext.reencode(ctx, [good], 0, 3, crop=[(0, 0, 32, 24)], orientation=[8], scale_denom=2)
    ra = cuda.QsContext.render_async
    for bad in (6, "exif", [0], [9], [1, 2]):
        with pytest.raises(ValueError, match="orientation"):
            ra(ctx, [cuda.parse_jpeg(good)[0]], [[]], orientation=bad)


def test_c_orientation_checks_without_a_context():
    lib = cuda.load()
    data = df.pillow_jpeg(16, 8)
    ptrs = (C.c_char_p * 1)(data)
    lens = (C.c_size_t * 1)(len(data))
    buf = (C.c_uint8 * (16 * 8 * 3))()
    outs = (C.c_void_p * 1)(C.addressof(buf))
    rc = (C.c_int * 1)(7)
    res = (cuda._PixelsResult * 1)()
    o = (C.c_int32 * 1)(9)
    assert lib.jpegqs_cuda_pixels_batch_oriented(None, 1, ptrs, lens, 0, 3, 0, 1, 3, None, o, 0, outs, 0, rc, res) == -2
    assert lib.jpegqs_cuda_render_oriented_async(None, 0, None, None, 0, 1, o, None, None) == -2
    assert rc[0] == 7 and bytes(buf) == bytes(len(buf))
