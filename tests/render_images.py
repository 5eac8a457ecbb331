"""Coefficient images for the render tests: hard_content's samplings plus 4:1:1 (luma sampled
4x1), whose chroma libjpeg up-samples by box replication (int_upsample), and the further
geometries of hard_content.FACTORS that libjpeg writes in one scan (GEOMETRIES: grey, or at most
10 blocks per MCU; 3x3 and 4x4 luma over chroma only reach the smoothing, and files of one scan per
component)."""
import hard_content as hc

SAMPLINGS = hc.SAMPLINGS + ("411",)
GEOMETRIES = tuple(g for g in hc.GEOMETRIES if len(hc.factors(g)) == 1 or sum(h * v for h, v in hc.factors(g)) <= 10)


def make_411(width, height, tables, content="synth", seed=1):
    return hc.make_image(width, height, "411", tables, content, seed=seed)


def make(w, h, ss, table, content, seed):
    """An image of sampling ss (one of SAMPLINGS or GEOMETRIES), hard_content table `table` and
    content."""
    return hc.make_image(w, h, ss, hc.TABLES[table], content, seed=seed)
