"""world_size 2 and 3 over gloo (CPU): the product's MCU-row sharding, halo exchange and
stop logic (jpegqs_b200/multigpu.py) with oracle passes must reproduce the whole-image
oracle bit for bit - shard-count invariance (SURVEY.md 8e)."""
import os
import socket
import sys
import tempfile

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
from hard_content import FACTORS  # noqa: E402


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, cfg, outdir):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, HERE)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import jpegqs_b200 as qs
    from jpegqs_b200 import multigpu as mg
    from oracle_passes import OraclePasses
    from golden_io import adversarial_image
    w, h, ss, flags, niter, kind = cfg
    if kind:
        full = adversarial_image(kind)
        w, h = full.width, full.height
    elif ss in FACTORS:
        full = _geometry_image(w, h, ss)
    total = (h + 15) // 16 if ss != "gray" and (kind or ss in ("420", "440")) else (h + 7) // 8
    if ss in FACTORS:
        total = -(-h // (8 * max(c.v_samp for c in full.comps)))
    rng = mg.split_mcu_rows(total, world)[rank]
    if kind or ss in FACTORS:
        comps_src = []
        for c in full.comps:
            r0, r1 = mg.comp_block_rows(rng, c.v_samp, c.hblk)
            comps_src.append((c.coef[r0:r1].copy(), c))
    else:
        slab = qs.synth.make_image(w, h, ss, mcu_rows=rng)
        comps_src = [(c.coef, c) for c in slab.comps]
    comps = []
    geom_src = full if kind or ss in FACTORS else qs.synth.make_image(w, h, ss, mcu_rows=(0, 0))
    fullh = [qs.blocks_for(h, c.v_samp, max(cc.v_samp for cc in geom_src.comps)) for c in geom_src.comps]
    for k, (coef, c) in enumerate(comps_src):
        rows = coef.shape[0]
        r0, _ = mg.comp_block_rows(rng, c.v_samp, fullh[k])
        comps.append(mg.SlabComp(torch.from_numpy(np.ascontiguousarray(coef)),
                                 torch.zeros((rows * 8 + 2, mg.plane_stride(c.wblk)), dtype=torch.uint8),
                                 c.wblk, rows, c.quant, k == 0 or ss == "gray", c.h_samp, c.v_samp, r0, fullh[k]))
    geom = mg.SlabGeom(ss != "gray", w, h)

    allreduce_flag = mg.make_flag_allreduce(dist, torch.device('cpu'))

    stop, ups = mg.run_slab(OraclePasses(flags), comps, flags, niter, rank, world, dist, allreduce_flag, geom)
    outs = {f"c{k}": (c.coef_up if ups and k in (1, 2) else c.coef).numpy() for k, c in enumerate(comps)}
    np.savez(os.path.join(outdir, f"r{rank}.npz"), stop=stop, ups=int(ups), **outs)
    dist.barrier()
    dist.destroy_process_group()


def _geometry_image(w, h, ss):
    import hard_content as hc
    return hc.make_image(w, h, ss, hc.TABLES["k50"], "saturated", seed=w + h)


CFGS = [
    (2, (96, 80, "420", 0, 2, None)),
    (3, (64, 112, "420", 1, 2, None)),         # DIAGONALS, uneven split
    (2, (48, 40, "gray", 16, 3, None)),        # NO_REBALANCE, 8-row MCUs
    (2, (0, 0, "420", 0, 2, "badcoef")),       # stop semantics across ranks
    (2, (64, 96, "420", 8, 2, None)),          # LOW_QUALITY
    (2, (96, 80, "420", 3, 2, None)),          # JOINT_YUV: luma plane handed to the chroma phase
    (3, (64, 112, "420", 7, 2, None)),         # + UPSAMPLE_UV, uneven split
    (2, (48, 64, "444", 7, 2, None)),          # 4:4:4: the luma plane itself is the predictor
    (2, (90, 72, "420", 7, 1, None)),          # ragged size: edge replication inside the last slab
    (2, (0, 0, "420", 7, 2, "badcoef")),       # stop in the chroma phase
    # hard_content.FACTORS: MCU rows of 3 and 4 block rows, down- / up-sampling by 3 and 4 across slab
    # boundaries, chroma with more block rows than luma
    (2, (121, 223, "13", 3, 2, None)), (3, (121, 223, "13", 7, 2, None)),
    (3, (64, 193, "14", 3, 2, None)), (2, (64, 193, "14", 7, 2, None)),
    (2, (121, 223, "24", 3, 2, None)), (3, (96, 190, "24", 7, 2, None)),
    (2, (121, 223, "11_22_22", 3, 2, None)), (3, (121, 223, "11_22_22", 7, 2, None)),
]


@pytest.mark.parametrize("world,cfg", CFGS)
def test_shard_count_invariance(world, cfg):
    sys.path.insert(0, HERE)
    import jpegqs_b200 as qs
    import oracle_lib as ol
    from golden_io import adversarial_image
    w, h, ss, flags, niter, kind = cfg
    full = adversarial_image(kind) if kind else _geometry_image(w, h, ss) if ss in FACTORS else qs.synth.make_image(w, h, ss)
    want_ret, want = ol.run_oracle(full, flags, niter)
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_worker, args=(world, _free_port(), cfg, d), nprocs=world, join=True)
        parts = [np.load(os.path.join(d, f"r{r}.npz")) for r in range(world)]
    assert all(int(p["stop"]) == want_ret for p in parts)
    for k, c in enumerate(want.comps):
        got = np.concatenate([p[f"c{k}"] for p in parts], axis=0)
        assert got.shape == c.coef.shape
        assert np.array_equal(got, c.coef), f"component {k}: {np.count_nonzero(got != c.coef)} differ"
