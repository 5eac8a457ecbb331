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

