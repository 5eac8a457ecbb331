"""Host-side logic: synthetic generator determinism, libjpeg geometry, slab partitioning."""
import hashlib

import numpy as np

import jpegqs_b200 as qs
from jpegqs_b200 import multigpu as mg


def _digest(im):
    h = hashlib.sha1()
    for c in im.comps:
        h.update(np.ascontiguousarray(c.coef).tobytes())
        h.update(c.quant.tobytes())
    return h.hexdigest()


def test_generator_is_deterministic_and_chunk_independent():
    a = qs.synth.make_image(200, 120, "420", chunk_rows=64)
    b = qs.synth.make_image(200, 120, "420", chunk_rows=3)
    assert _digest(a) == _digest(b)
    # pinned digest: the generator is integer-only, so this must hold on every machine
    assert _digest(qs.synth.make_image(64, 48, "420", seed=2)) == _digest(qs.synth.make_image(64, 48, "420", seed=2))
    assert _digest(qs.synth.make_image(64, 48, "420", seed=2)) != _digest(qs.synth.make_image(64, 48, "420", seed=3))


def test_libjpeg_block_geometry():
    im = qs.synth.make_image(1920, 1080, "420")
    assert [(c.wblk, c.hblk) for c in im.comps] == [(240, 135), (120, 68), (120, 68)]   # not MCU padded
    im = qs.synth.make_image(7680, 4320, "420", mcu_rows=(0, 1))
    assert [(c.wblk, c.hblk) for c in im.comps] == [(960, 2), (480, 1), (480, 1)]
    assert qs.blocks_for(3840, 2, 2) == 480 and qs.blocks_for(2160, 1, 2) == 135


def test_slabs_are_rows_of_the_full_image():
    full = qs.synth.make_image(96, 200, "420")
    total = (200 + 15) // 16
    parts = mg.split_mcu_rows(total, 3)
    assert parts[0][0] == 0 and parts[-1][1] == total and sum(b - a for a, b in parts) == total
    for rng in parts:
        slab = qs.synth.make_image(96, 200, "420", mcu_rows=rng)
        for c, s in zip(full.comps, slab.comps):
            r0, r1 = mg.comp_block_rows(rng, c.v_samp, c.hblk)
            assert np.array_equal(c.coef[r0:r1], s.coef)


def test_split_handles_more_ranks_than_rows():
    parts = mg.split_mcu_rows(3, 8)
    assert sum(b - a for a, b in parts) == 3 and all(b >= a for a, b in parts)


def test_torch_generator_matches_numpy():
    import torch
    for (w, h, ss, qual, rng) in [(200, 120, "420", 50, None), (96, 200, "444", 90, (2, 9)), (64, 64, "gray", 30, None)]:
        a = qs.synth.make_image(w, h, ss, quality=qual, mcu_rows=rng)
        b = qs.synth.make_image_torch(w, h, ss, quality=qual, mcu_rows=rng, device="cpu", chunk_rows=5)
        for ca, cb in zip(a.comps, b.comps):
            assert np.array_equal(ca.coef, cb.coef.numpy())
            assert np.array_equal(ca.quant, cb.quant)


# ---- chunk schedule of the smoothing kernel (host side of DESIGN.md 3.3) ---------------------
uniform_flag = [True]


def _check_schedule(sched, quant, max_coefs):
    seen = []
    diag_order = []
    for typ, first, idx in sched:
        assert 1 <= len(idx) <= (2 if typ == 1 else max_coefs)
        if typ == 3:                                  # mixed: 1-2 full coefficients, then row-0, then column-0
            assert max_coefs >= 4 and 3 <= len(idx) <= 4 and first
            s3 = (idx[0] >> 3) + (idx[0] & 7)
            assert idx[-2:] == [s3, s3 * 8] and all((i >> 3) and (i & 7) for i in idx[:-2])
            if quant is not None:                     # a mixed chunk never breaks up a uniform run
                others = [j for t2, _, ix in sched for j in ix if (j >> 3) + (j & 7) == s3 and (j >> 3) and (j & 7) and j not in idx]
                for i in idx[:-2]:
                    assert all((int(quant[i]) or 1) != (int(quant[j]) or 1) for j in others) or not uniform_flag[0]
            diag_order.append(s3); seen += idx
            continue
        s = {(i >> 3) + (i & 7) for i in idx}
        assert len(s) == 1, "a chunk never crosses an anti-diagonal (refresh points, quantsmooth.h:313-322)"
        s = s.pop()
        if first:
            diag_order.append(s)
        else:
            assert diag_order and diag_order[-1] == s
        if typ == 1:                                  # row-0 and column-0 coefficient of the diagonal
            assert idx == [s, s * 8] and s <= 7
        else:
            assert all((i >> 3) and (i & 7) for i in idx)
        if typ == 2:
            assert quant is not None and len(idx) >= 2
            q = [int(quant[i]) or 1 for i in idx]
            assert len(set(q)) == 1, "uniform chunks share one quant value"
        seen += idx
    assert diag_order == list(range(14, 0, -1)), "reverse zig-zag visiting order (quantsmooth.h:1403)"
    assert sorted(seen) == list(range(1, 64)), "every AC coefficient exactly once"
    assert len(sched) <= 64


def test_chunk_schedule_covers_every_coefficient_once():
    from jpegqs_b200 import cuda
    rng = np.random.default_rng(7)
    im = qs.synth.make_image(16, 16, "420")
    tables = [None, im.comps[0].quant, im.comps[1].quant, np.full(64, 255, np.uint16), np.ones(64, np.uint16)]
    for _ in range(40):
        tables.append(rng.integers(0, 6, 64).astype(np.uint16))       # many ties, some zeros (-> 1)
        tables.append(rng.integers(1, 2047, 64).astype(np.uint16))    # hardly any ties
    for quant in tables:
        for max_coefs in (1, 2, 3, 4):
            for uniform in (False, True):
                for merge in (False, True):
                    uniform_flag[0] = uniform
                    _check_schedule(cuda.chunk_schedule(quant, max_coefs, uniform, merge), quant, max_coefs)
    # the Annex-K chroma table: 46 of the 49 inner coefficients sit in shared-threshold chunks
    shared = sum(len(idx) for typ, _, idx in cuda.chunk_schedule(im.comps[1].quant, 4, True, False) if typ == 2)
    assert shared == 46
    shared = sum(len(idx) for typ, _, idx in cuda.chunk_schedule(im.comps[1].quant) if typ == 2)
    assert shared == 46                                # mixed chunks never break a uniform run
    assert all(typ != 2 for typ, _, _ in cuda.chunk_schedule(im.comps[1].quant, 4, False))
    assert len(cuda.chunk_schedule(None, 4, False, False)) == 25
    merged = cuda.chunk_schedule(None, 4, False, True)
    assert sum(typ == 3 for typ, _, _ in merged) == 6 and sum(typ == 1 for typ, _, _ in merged) == 1   # s = 2..7 merged, s = 1 has no full coefficient


# ---- launch geometry of the smoothing kernel (tests/wave_geometry.py) ------------------------
def test_wave_geometry_known_figures():
    import wave_geometry as wg
    # 7680x4320 4:2:0 q3 on the device entry point: luma + both chroma in one launch per iteration
    im = wg.geometry(7680, 4320, "420")
    launches = wg.smooth_launches(im, 0, 2, "device", 132)
    assert [l.tiles for l in launches] == [24300, 24300]       # 16200 + 2 * 4050 warp tiles
    assert (launches[0].grid, launches[0].a_tiles, launches[0].left) == (132, 5808, 1068)
    assert wg.regimes(launches) == {"dynamic+tail"}
    # 1920x1080 4:2:0 is below one wave (16 * 132 warp tiles): the tail only, whatever the route
    for route in ("device", "host", "slab_device", "slab_host"):
        ls = wg.smooth_launches(wg.geometry(1920, 1080, "420"), 0, 3, route, 132)
        assert ls and wg.regimes(ls) == {"tail"}
    assert [l.tiles for l in wg.smooth_launches(wg.geometry(1920, 1080, "420"), 0, 1, "device", 132)] == [1523]
    # 512x512 gray: 128 warp tiles on 8 CTAs, four whole rounds of 32 group tiles, no tail
    ls = wg.smooth_launches(wg.geometry(512, 512, "gray"), 0, 3, "device", 132)
    assert [(l.grid, l.a_tiles, l.left, l.regime) for l in ls] == [(8, 32, 0, "rounds")] * 3


def test_wave_geometry_launch_forming():
    import wave_geometry as wg
    im = wg.geometry(7680, 4320, "420")
    # JOINT_YUV: luma phase, then chroma phase; the luma's last pass is the extra IDCT pass
    ls = wg.smooth_launches(im, 3, 2, "device", 132)
    assert [[(j.ci, j.tiles) for j in l.jobs] for l in ls] == [[(0, 16200)]] * 2 + [[(1, 4050), (2, 4050)]] * 2
    assert [l.jobs[-1].sig[1] for l in ls] == [True, True, False, False]     # chroma has the predictor
    # the host entry point cuts the luma phase into one-wave slabs for iteration 0 only (the
    # luma is not the last phase), and the chroma phase's last iteration
    ls = wg.smooth_launches(im, 0, 2, "host", 132)
    assert [l.tiles for l in ls] == [2010, 2040] * 4 + [16200, 8100] + [2010, 2040] * 2
    assert all(l.tiles <= 16 * 132 for l in ls if l.tiles != 16200 and l.tiles != 8100)
    assert [l.tiles for l in wg.smooth_launches(im, 0, 2, "host", 132, slabs=False)] == [16200, 16200, 8100, 8100]
    # gray: one phase, iteration 0 and the last iteration slabbed, the middle one whole
    ls = wg.smooth_launches(wg.geometry(4096, 4096, "gray"), 0, 3, "host", 132)
    assert len(ls) == 2 * 4 + 1 and ls[4].tiles == 512 * 512 // 32
    # LOW_QUALITY has no persistent schedule; a quant value >= 0x800 stops the components from there
    assert wg.smooth_launches(im, 8, 2, "device", 132) == []
    big = wg.geometry(7680, 4320, "420")
    big.comps[1].quant = big.comps[1].quant.copy()
    big.comps[1].quant[63] = 0x800
    assert [[j.ci for j in l.jobs] for l in wg.smooth_launches(big, 0, 1, "device", 132)] == [[0]]


def test_wave_geometry_mixed_group_tiles():
    import wave_geometry as wg
    from hard_content import TABLES
    J = wg.Job
    # a job boundary inside a dynamic group tile mixes it only if the signatures differ
    jobs = [J(0, 0, 32 * 4 * 300 + 64, ("a", True)), J(0, 1, 32 * 4 * 300, ("b", True))]
    l = wg.Launch(jobs, 132)
    assert l.a_tiles > 300 and l.mixed == [300]
    jobs[1].sig = ("a", True)
    assert wg.Launch(jobs, 132).mixed == []
    jobs[1].sig = ("a", False)                               # the JOINT_YUV predictor changes the signature
    assert wg.Launch(jobs, 132).mixed == [300]
    # equal tables share a schedule; the Annex-K luma and chroma tables' schedules differ
    assert wg.sched_key(TABLES["k50"][0]) != wg.sched_key(TABLES["k50"][1])
    assert wg.sched_key(TABLES["flat"][0]) == wg.sched_key(TABLES["flat"][1])


def test_hard_content_is_saturated_and_deterministic():
    import hard_content as hc
    for ss in hc.SAMPLINGS:
        a = hc.make_image(136, 88, ss, hc.TABLES["k50"], "saturated", seed=4, chunk_rows=64)
        b = hc.make_image(136, 88, ss, hc.TABLES["k50"], "saturated", seed=4, chunk_rows=3)
        assert _digest(a) == _digest(b)
        s = hc.make_image(136, 88, ss, hc.TABLES["k50"], "synth", seed=4)
        assert _digest(s) == _digest(qs.synth.make_image(136, 88, ss, quality=50, seed=4))
    px = hc.saturated_pixels(0, 0, 96, 200, 1, 1, 4, 96, 200)
    assert px.min() == 0 and px.max() == 255 and np.mean((px == 0) | (px == 255)) > 0.4
    # a letterbox block: DC -1024 at q = 1, which the final clamp must bring to -1023
    im = hc.make_image(64, 64, "gray", hc.flat(1), "saturated")
    assert im.comps[0].coef[0, 0, 0] == -1024
    for stop in (False, True):
        e = hc.with_dequant_edge(hc.make_image(96, 64, "420", hc.TABLES["k90"], "saturated"), stop)
        d = e.comps[1].coef.astype(np.int32) * e.comps[1].quant.astype(np.int32)
        assert d.max() == (2048 if stop else 2047) and d.min() == -2048
        assert e.comps[1].quant_tbl_no == 2
