"""Coefficient images for the render tests: hard_content's samplings plus 4:1:1 (luma sampled
4x1), whose chroma libjpeg up-samples by box replication (int_upsample)."""
import numpy as np

import hard_content as hc
from jpegqs_b200 import synth
from jpegqs_b200.image import CoefImage, Component, JCS_YCbCr, blocks_for

SAMPLINGS = hc.SAMPLINGS + ("411",)


def make_411(width, height, tables, content="synth", seed=1) -> CoefImage:
    comps = []
    for c, (hs, vs) in enumerate([(4, 1), (1, 1), (1, 1)]):
        wb, hb = blocks_for(width, hs, 4), blocks_for(height, vs, 1)
        q = np.asarray(tables[min(c, 1)], dtype=np.uint16).copy()
        if content == "saturated":
            px = hc.saturated_pixels(c, 0, hb * 8, wb * 8, 4 // hs, 1, seed, height, width)
        else:
            px = synth.pixels(c, 0, hb * 8, wb * 8, 4 // hs, 1, seed)
        comps.append(Component(coef=synth.quantize_blocks(px, q), quant=q, h_samp=hs, v_samp=vs,
                               quant_tbl_no=min(c, 1)))
    return CoefImage(width=width, height=height, colorspace=JCS_YCbCr, comps=comps)


def make(w, h, ss, table, content, seed):
    """An image of sampling ss (one of SAMPLINGS), hard_content table `table` and content."""
    if ss == "411":
        return make_411(w, h, hc.TABLES[table], content, seed)
    return hc.make_image(w, h, ss, hc.TABLES[table], content, seed=seed)
