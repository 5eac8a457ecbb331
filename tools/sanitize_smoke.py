"""Small invocations of every kernel for compute-sanitizer (memcheck / racecheck / synccheck):
    compute-sanitizer --tool memcheck python tools/sanitize_smoke.py"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import jpegqs_b200 as qs

ctx = qs.cuda.QsContext(0)
for (w, h, ss, flags, niter) in [(96, 64, "420", 0, 2), (90, 50, "420", 7, 1), (64, 48, "444", 3, 1),
                                 (64, 48, "gray", 1, 1), (80, 48, "420", 8 | 7, 1), (72, 40, "422", 16, 1)]:
    im = qs.synth.make_image(w, h, ss)
    ret, out = ctx.do_quantsmooth(im, flags, niter)
    rgb = ctx.render_rgb(out)
    print(w, h, ss, flags, niter, "ret", ret, rgb.shape, flush=True)
ret, out = ctx.do_quantsmooth(qs.synth.make_image(96, 64, "420"), 1, 1)


# the JPEG decoder: good files of every kind, damaged ones beside them, a batch of more than one
# launch group (8 images), at the smallest subsequence size (key 9) and the default
import io  # noqa: E402

import numpy as np  # noqa: E402
import torch  # noqa: E402
from PIL import Image  # noqa: E402


def jpeg(w, h, mode="RGB", **save):
    yy, xx = np.mgrid[0:h, 0:w]
    px = np.stack([(xx * 3 + yy * 5) % 256, (xx * yy) % 251, (xx ^ yy) * 7 % 256, (xx + 2 * yy) % 256], -1).astype(np.uint8)
    im = Image.frombytes("CMYK", (w, h), px.tobytes()) if mode == "CMYK" else \
        Image.fromarray(np.ascontiguousarray(px[..., :3])).convert(mode)
    b = io.BytesIO()
    im.save(b, "JPEG", **save)
    return b.getvalue()


good = [jpeg(90, 50, quality=75), jpeg(61, 43, quality=90, restart_marker_blocks=3), jpeg(40, 24, "CMYK", quality=80),
        jpeg(33, 17, "L", quality=100), jpeg(48, 32, quality=85, keep_rgb=True, subsampling=0),
        jpeg(70, 30, quality=50, subsampling=1, optimize=True)]
base, rst = good[0], good[1]
off = qs.parse_jpeg(base)[1].entropy_offset
flip = bytearray(base)
for p in range(off + 5, len(base) - 2, 37):
    flip[p] ^= 0x5A
p = rst.index(b"\xff\xd1", qs.parse_jpeg(rst)[1].entropy_offset)
bad = [base[:off + (len(base) - off) // 3], bytes(flip), rst[:p] + rst[p + 2:], base[:off + 1]]
files = good + bad                                     # 10 images: two launch groups
for sub_bytes in (32, 512):
    ctx.set_tuning(9, sub_bytes)
    parsed = [qs.parse_jpeg(f) for f in files]
    data = [torch.frombuffer(bytearray(f), dtype=torch.uint8).cuda() for f in files]
    coefs, status = ctx.decode_async([p[0] for p in parsed], [p[1] for p in parsed], data)
    torch.cuda.synchronize()
    print("decode_async key 9 =", sub_bytes, "status", status.cpu().tolist(), flush=True)
ctx.set_tuning(9, 512)


# the JPEG encoder: good images of every kind, a RANGE image (AC 1024) and an OVERFLOW capacity (the
# exact length minus 1) in one batch of more than one launch group (16 images), standard and optimal
# tables; then decode -> run_async (q6) -> encode with the chroma source read from the run status
from jpegqs_b200.image import CoefImage, Component, JCS_GRAYSCALE  # noqa: E402

imgs, heads, hosts = [], [], []
for f in good * 3:                                     # 18 good images
    im = qs.read_jpeg(f)
    pre, ids, tbls = qs.jpeg_prefix(f)
    imgs.append(im); hosts.append((pre, ids, tbls))
    heads.append((torch.frombuffer(bytearray(pre), dtype=torch.uint8).cuda(), ids, tbls))
rb = np.zeros((2, 3, 64), np.int16)
rb[1, 1, 5] = 1024
imgs.append(CoefImage(width=24, height=16, colorspace=JCS_GRAYSCALE,
                      comps=[Component(coef=rb, quant=np.ones(64, np.uint16))]))
heads.append((torch.tensor([0xFF, 0xD8], dtype=torch.uint8, device="cuda"), (1,), (0,)))
coefs = [[torch.from_numpy(np.ascontiguousarray(c.coef)).cuda() for c in im.comps] for im in imgs]
for optimize in (False, True):
    exact = len(qs.encode_model(imgs[0], [c.coef for c in imgs[0].comps], *hosts[0], optimize)[0])
    caps = [exact - 1] + [qs.encode_bound(im, h[0].numel()) for im, h in zip(imgs[1:], heads[1:])]
    outs = [torch.empty(c, dtype=torch.uint8, device="cuda") for c in caps]
    out, lengths, status = ctx.encode_async(imgs, coefs, heads, optimize, out=outs, capacity=caps)
    torch.cuda.synchronize()
    print("encode_async optimize", int(optimize), "status", status.cpu().tolist(), flush=True)
im, scan = qs.parse_jpeg(base)
coefs, st = ctx.decode_async([im], [scan], [torch.frombuffer(bytearray(base), dtype=torch.uint8).cuda()])
work = [im.clone()]
rst, ups = ctx.run_async(work, coefs, 7, 1)
pre, ids, tbls = qs.jpeg_prefix(base)
out, lengths, status = ctx.encode_async(work, coefs, [(torch.frombuffer(bytearray(pre), dtype=torch.uint8).cuda(), ids, tbls)],
                                        True, rst, ups)
torch.cuda.synchronize()
print("decode -> run_async -> encode_async: run", rst.cpu().tolist(), "encode status", status.cpu().tolist(), flush=True)


# the scan decoder: progressive files of every kind (restart markers or not, grey, CMYK, untransformed
# RGB), damaged ones beside them (truncated, bytes flipped, an RST removed, cut one byte after an SOS),
# in a batch of more than one launch group (16 images), at the smallest subsequence size and the default
pgood = [jpeg(90, 50, quality=75, progressive=True), jpeg(61, 43, quality=90, progressive=True, restart_marker_blocks=3),
         jpeg(40, 24, "CMYK", quality=80, progressive=True), jpeg(33, 17, "L", quality=100, progressive=True),
         jpeg(48, 32, quality=85, keep_rgb=True, subsampling=0, progressive=True),
         jpeg(70, 30, quality=50, subsampling=1, optimize=True, progressive=True)]
pbase, prst = pgood[0], pgood[1]
pflip = bytearray(pbase)
for p in range(qs.parse_jpeg_scans(pbase)[1][0].offset + 5, len(pbase) - 2, 41):
    pflip[p] ^= 0x5A
p = prst.index(b"\xff\xd1")
last_sos = pbase.rindex(b"\xff\xda")
pbad = [pbase[:len(pbase) * 2 // 3], bytes(pflip), prst[:p] + prst[p + 2:],
        pbase[:last_sos + 2 + int.from_bytes(pbase[last_sos + 2:last_sos + 4], "big") + 1]]


def device_scans(f):
    """parse_jpeg_scans' records, or None for a file only the host reader takes or no reader takes"""
    try:
        return qs.parse_jpeg_scans(f)[1]
    except qs.cuda.QsError:
        return None


pfiles = [f for f in pgood * 3 + pbad if device_scans(f) is not None]
for sub_bytes in (32, 512):
    ctx.set_tuning(9, sub_bytes)
    parsed = [qs.parse_jpeg_scans(f) for f in pfiles]
    data = [torch.frombuffer(bytearray(f), dtype=torch.uint8).cuda() for f in pfiles]
    coefs, status = ctx.decode_scans_async([p[0] for p in parsed], [p[1] for p in parsed], data)
    torch.cuda.synchronize()
    print("decode_scans_async key 9 =", sub_bytes, len(pfiles), "images, status", status.cpu().tolist(), flush=True)
ctx.set_tuning(9, 512)


# EXIF orientation: files with spliced EXIF / XMP payloads (a tag of each transposing kind, a truncated IFD,
# a value offset past the block, an XMP packet) through the host reader, then the oriented render of
# every orientation in one launch (the flips and the staged transposes side by side), at d = 1 and 2
import struct  # noqa: E402


def app1(payload):
    return b"\xff\xe1" + struct.pack(">H", len(payload) + 2) + payload


def exif_tag(o, cut=None, off=None):
    e = struct.pack("<HHLHH", 0x0112, 3, 1 if off is None else 3, o, 0) if off is None else \
        struct.pack("<HHLL", 0x0112, 3, 3, off)
    p = b"Exif\0\0II*\0" + struct.pack("<LH", 8, 1) + e + b"\0\0\0\0"
    return p[:cut] if cut else p


payloads = [exif_tag(6), exif_tag(8), exif_tag(5, cut=20), exif_tag(7, off=4000),
            b"http://ns.adobe.com/xap/1.0/\0<x tiff:Orientation=\"7\"/>"]
ofiles = [f[:2] + app1(p) + f[2:] for f in (good[0], good[3], good[5]) for p in payloads]
print("exif orientations", [qs.exif_orientation(f) for f in ofiles], flush=True)
for d in (1, 2):
    px = ctx.decode_pixels(ofiles, 3, 1, scale_denom=d, orientation=[0, 1, 2, 3, 4] * 2 + [5, 6, 7, 8, 0])
    torch.cuda.synchronize()
    print("decode_pixels oriented d", d, [tuple(p[0].shape) for p in px], flush=True)

# colour modes: a CMYK and a YCCK file (Adobe transform 0 spliced to 1) beside grey and YCbCr ones, in both
# modes, with every orientation (the 4-component staging of 5..8 included), at d = 1 and 2
cm = jpeg(75, 41, "CMYK", quality=80)
yk = cm[:2] + cm[2:].replace(b"Adobe\x00\x64\x00\x00\x00\x00\x00", b"Adobe\x00\x64\x00\x00\x00\x00\x01", 1)
mfiles = [cm, yk, jpeg(40, 24, "L"), jpeg(70, 30, "RGB")] * 2
for d in (1, 2):
    for mode in ("RGB", "L"):
        px = ctx.decode_pixels(mfiles, 3, 1, scale_denom=d, mode=mode, orientation=[1, 2, 3, 4, 5, 6, 7, 8])
        print("decode_pixels mode", mode, "d", d, [tuple(p[0].shape) for p in px], flush=True)

# progressive files: grey and RGB pictures of every sampling, sizes with odd block counts, one flat
# picture whose AC scans are one long run segment
rng = np.random.RandomState(12)
pics = [torch.from_numpy(rng.randint(0, 256, (h, w, c)).astype(np.uint8)).cuda()
        for h, w, c in ((23, 39, 3), (40, 24, 1), (9, 130, 3))] + [torch.full((200, 296, 3), 90, dtype=torch.uint8).cuda()]
for sub in ("4:4:4", "4:2:2", "4:2:0"):
    out, lens, st = ctx.compress_async(pics, 90, sub, progressive=True)
    torch.cuda.synchronize()
    print("compress_async progressive", sub, lens.tolist(), st.tolist(), flush=True)

# thumbnails: files drafted to 1, 2 and 4 in one call, reduce cells with partial right and bottom edges
# (a loaded picture: orientation given, no draft), and reducing_gap on the crop path
tfiles = [jpeg(90, 50, quality=75), jpeg(333, 211, quality=85), jpeg(33, 17, "L", quality=100), jpeg(161, 97, quality=90)]
for o in (None, 6):
    px = ctx.decode_pixels(tfiles, 3, 1, thumbnail=[(40, 40), (30, 30), (8, 8), (13, 7)], orientation=o)
    print("decode_pixels thumbnail orientation", o, [tuple(p[0].shape) for p in px], flush=True)
px = ctx.decode_pixels(tfiles, 3, 1, size=(9, 5), crop=[None, (3, 5, 300, 200), None, (1, 1, 160, 96)], reducing_gap=1.0)
print("decode_pixels reducing_gap", [tuple(p[0].shape) for p in px], flush=True)

# blur and sharpen: fused rows and a row wider than the fused kernel holds (7000 x 3 bytes), a chain ending
# in UnsharpMask, CHW output, and a filtered reencode
from PIL import ImageFilter  # noqa: E402
ffiles = [jpeg(90, 50, quality=75), jpeg(7000, 9, quality=85), jpeg(33, 17, "L", quality=100)]
px = ctx.decode_pixels(ffiles, 3, 1, "chw", image_filter=[ImageFilter.GaussianBlur(5), ImageFilter.UnsharpMask(2, 150, 3)])
print("decode_pixels image_filter", [tuple(p[0].shape) for p in px], flush=True)
enc = ctx.reencode(ffiles, 3, 1, thumbnail=(40, 40), image_filter=ImageFilter.BoxBlur((3, 0)))
print("reencode image_filter", [len(r[0]) for r in enc], flush=True)
