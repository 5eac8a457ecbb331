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
