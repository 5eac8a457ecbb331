"""Which branch of the smoothing kernel's tile schedule a run reaches.

The persistent smoothing kernel (csrc/qs_kernels.cu `qs_smooth_kernel`, launched by
`qs_launch_smooth`) splits the warp tiles of a launch (32 blocks each) in two parts:

  * the first `a_tiles` group tiles (4 warp tiles each) are taken dynamically, one atomic per
    group tile, with the next one prefetched; a group whose warps sit in jobs with different
    chunk schedules switches to the table-independent schedule (`mixed`);
  * the left-over warp tiles are spread statically over all groups, idle warps leave and the
    named barrier is re-sized (the tail).

Which part a test exercises depends on how the driver (csrc/qs_cuda.cu) forms its launches:
which components share a launch, how many tiles each job has and in which order, and whether
the host entry point cuts a phase into one-wave slabs.  This module restates those decisions
so that a test can assert the regime its input was built for before it compares results.
Everything here is host arithmetic; the chunk schedules come from the library's host-only
`jpegqs_cuda_chunk_schedule`.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Callable, List, Optional, Sequence

import numpy as np

from jpegqs_b200.image import CoefImage, Component, JCS_GRAYSCALE, JCS_YCbCr, blocks_for

QS_DIAGONALS, QS_JOINT_YUV, QS_UPSAMPLE_UV, QS_LOW_QUALITY = 1, 2, 4, 8

TILE = 32                 # blocks per warp tile (one block per lane)
WPG = 4                   # warps per lock-step group: qs_launch_smooth forces wpg = 4
NG = 4                    # lock-step groups per CTA: NG = 4 * QS_SYNC_GS(2)
CTA_WARPS = WPG * NG      # qs_launch_smooth: `warps = wpg * 4`
MAX_SLABS = 16            # qs_cuda.cu QS_MAX_SLABS
MAX_JOBS = 1024           # qs_common.h QS_MAX_JOBS: components per batch launch


def tile_schedule(total_tiles: int, num_sms: int):
    """(grid, a_tiles, left) of one launch.
    qs_launch_smooth:    grid = min(ceil(tiles / warps), num_sms)
    qs_smooth_kernel:    G = gridDim.x * NG;  a_tiles = (tiles / (WPG * G)) * G;
                         left = tiles - a_tiles * WPG"""
    grid = min(-(-total_tiles // CTA_WARPS), num_sms)
    G = grid * NG
    a_tiles = (total_tiles // (WPG * G)) * G
    return grid, a_tiles, total_tiles - a_tiles * WPG


@dataclass
class Job:
    """One QsJob of a launch: `sig` stands for the kernel's per-warp signature
    `sched_slot * 2 + fresh_px` (equal chunk schedules share a sched_slot, assign_sched_slots)."""
    img: int
    ci: int
    nblocks: int
    sig: tuple

    @property
    def tiles(self) -> int:                 # upload_jobs: (nblocks + 31) / 32
        return -(-self.nblocks // TILE)


@dataclass
class Launch:
    jobs: List[Job]
    num_sms: int
    tiles: int = 0
    grid: int = 0
    a_tiles: int = 0
    left: int = 0
    mixed: List[int] = field(default_factory=list)     # dynamic group tiles with mixed warps

    def __post_init__(self):
        self.tiles = sum(j.tiles for j in self.jobs)
        self.grid, self.a_tiles, self.left = tile_schedule(self.tiles, self.num_sms)
        self.mixed = mixed_group_tiles(self.jobs, self.a_tiles)

    @property
    def regime(self) -> str:
        """'dynamic+tail' (i), 'rounds' (ii: dynamic only) or 'tail' (iii: no dynamic tile)."""
        if self.a_tiles == 0:
            return "tail"
        return "rounds" if self.left == 0 else "dynamic+tail"


def mixed_group_tiles(jobs: Sequence[Job], a_tiles: int) -> List[int]:
    """Dynamic group tiles gt < a_tiles whose warp tiles gt*WPG .. gt*WPG+WPG-1 lie in jobs with
    different signatures.  Jobs take consecutive tile ranges in launch order (upload_jobs
    tile_begin), so only a group tile that holds a job's first tile can be mixed."""
    begins = np.cumsum([0] + [j.tiles for j in jobs])
    out = set()
    for b in begins[1:-1]:
        gt = int(b) // WPG
        if gt >= a_tiles or b % WPG == 0:
            continue
        t0 = gt * WPG
        owners = np.searchsorted(begins, np.arange(t0, t0 + WPG), side="right") - 1
        if len({jobs[o].sig for o in owners if o < len(jobs)}) > 1:
            out.add(gt)
    return sorted(out)


# ---- the driver's decisions ----------------------------------------------------------------

def _chunk_sched(quant) -> tuple:
    """quant_prepare's chunk schedule (max 4 coefficients, uniform and merged chunks; a quant
    value 0 counts as 1) - tables with equal schedules run the same barrier sequence."""
    from jpegqs_b200 import cuda
    return tuple((t, f, tuple(ix)) for t, f, ix in cuda.chunk_schedule(quant, 4, True, True))


_SCHED_CACHE = {}


def sched_key(quant) -> tuple:
    k = np.asarray(quant, dtype=np.uint16).tobytes()
    if k not in _SCHED_CACHE:
        _SCHED_CACHE[k] = _chunk_sched(quant)
    return _SCHED_CACHE[k]


@dataclass
class _Work:
    img: int
    ci: int
    W: int
    H: int
    niter2: int
    extra: int
    sig: tuple
    alike: bool          # run_images slab plan: has a table, 1 < qval < 0x800, W, H > 0


def _image_works(n: int, im: CoefImage, flags: int, niter: int, on_device: bool, sched):
    """run_setup + comp_prelude for one image: (ngroups, works by component or None)."""
    ycc = im.colorspace == JCS_YCbCr
    nc = len(im.comps)
    need_ds = bool(flags & (QS_JOINT_YUV | QS_UPSAMPLE_UV)) and ycc and nc >= 3 and all(
        (im.comps[c].h_samp, im.comps[c].v_samp) == (1, 1) for c in (1, 2))      # run_setup 695-697
    if niter <= 0 and not ((flags & QS_UPSAMPLE_UV) and need_ds):                # 698 (skip)
        return 0, []
    sub = need_ds and (im.comps[0].h_samp, im.comps[0].v_samp) != (1, 1)        # 714
    ngroups = 2 if (need_ds or (not on_device and nc > 1)) else 1               # 728
    works, stop = [], False
    luma_iterates = False
    for ci, c in enumerate(im.comps):
        if c.quant is None:                                                      # comp_prelude 875
            works.append(None)
            continue
        qval = int(np.bitwise_or.reduce(np.asarray(c.quant, dtype=np.int64)))
        image1 = ci > 0 and luma_iterates and sub and bool(flags & QS_UPSAMPLE_UV)   # post_step 962
        extra = 1 if (image1 or (ci == 0 and need_ds)) else 0                  # 876
        niter2 = 0 if qval <= 1 else niter                                      # 877
        stop = stop or qval >= 0x800                                             # 878
        W, H = c.wblk, c.hblk
        if niter2 + extra == 0 or stop or not W * H:                             # 879-885
            works.append(None)
            continue
        if ci == 0:
            luma_iterates = True
        # plane2_of: the JOINT_YUV predictor (image2, set by the luma's post step) for chroma
        fresh_px = not ((flags & QS_JOINT_YUV) and need_ds and ci > 0 and luma_iterates)
        q = np.where(np.asarray(c.quant) == 0, 1, np.asarray(c.quant))
        works.append(_Work(n, ci, W, H, niter2, extra, (sched(q), fresh_px),
                           1 < qval < 0x800))
    return ngroups, works


def group_range(ngroups: int, nc: int, g: int):
    """qs_cuda.cu group_range: the whole image, or luma | chroma."""
    if ngroups == 1:
        return 0, nc
    if ngroups == nc:
        return g, g + 1
    return (1, nc) if g else (0, 1)


def _slab_plan(im: CoefImage, works, ngroups: int, g: int, num_sms: int):
    """run_images 1034-1058: the rows [r[k], r[k+1]) of each one-wave slab, or None."""
    c0, c1 = group_range(ngroups, len(im.comps), g)
    ws = works[c0:c1]
    if not ws or any(w is None or not w.alike or (w.W, w.H) != (ws[0].W, ws[0].H) for w in ws):
        return None
    Wb, Hb, nc = ws[0].W, ws[0].H, c1 - c0
    wave = num_sms * WPG * 4 * TILE                      # blocks in flight (tune_wave 0)
    rpw = wave // (nc * Wb)
    if rpw < 1:
        return None
    waves = -(-Hb // rpw)
    m = -(-waves // MAX_SLABS)
    K = -(-Hb // (m * rpw))
    if K < 2:
        return None
    return [k * Hb // K for k in range(K + 1)]


def _jobs(works, r0=None, r1=None):
    return [Job(w.img, w.ci, w.W * ((r1 - r0) if r0 is not None else w.H), w.sig) for w in works]


def _phase_launches(works: List[_Work], niter: int, num_sms: int, plan=None, slab_in=False,
                    slab_out=False) -> List[Launch]:
    out = []
    max_pass = max(w.niter2 + w.extra for w in works)
    for it in range(max_pass):
        if it == 0 and slab_in:                                   # run_images 1128-1166
            out += [Launch(_jobs(works, plan[k], plan[k + 1]), num_sms) for k in range(len(plan) - 1)]
            continue
        if slab_out and it == works[0].niter2 - 1:               # 1189-1207
            out += [Launch(_jobs(works, plan[k], plan[k + 1]), num_sms) for k in range(len(plan) - 1)]
            continue
        for clampv in (0, 1):                                     # smooth_pass 922-935
            js = [w for w in works if it < w.niter2 and int(it == w.niter2 - 1 and not w.extra) == clampv]
            if js:
                out.append(Launch(_jobs(js), num_sms))
    return out


def smooth_launches(images, flags: int, niter: int, route: str, num_sms: int, slabs: bool = True,
                    sched: Optional[Callable] = None) -> List[Launch]:
    """The smoothing-kernel launches of one call, in order, assuming no coefficient leaves
    the legal range (a runtime stop only removes components from later launches).

    route: 'device' (jpegqs_cuda_run_device), 'host' (jpegqs_cuda_run_host), 'batch_device' /
    'batch_host' (jpegqs_cuda_run_batch with on_device 1 / 0), 'slab_device' / 'slab_host'
    (jpegqs_cuda_run_slab, world 1).  slabs: tuning key 6 (the host entry point's slab pipeline).
    LOW_QUALITY runs another kernel without this schedule: no launches are returned."""
    if isinstance(images, CoefImage):
        images = [images]
    sched = sched or sched_key
    niter = max(0, min(int(niter), 100))                          # run_setup 682-683
    if flags & QS_LOW_QUALITY:
        return []
    on_device = route in ("device", "batch_device", "slab_device")
    if route.startswith("batch"):                                 # jpegqs_cuda_run_batch 1277-1285
        out, i = [], 0
        while i < len(images):
            n, jobs = 0, 0
            while i + n < len(images) and jobs + len(images[i + n].comps) <= MAX_JOBS:
                jobs += len(images[i + n].comps)
                n += 1
            out += _run_images(images[i:i + n], flags, niter, on_device, num_sms, False, sched)
            i += n
        return out
    assert len(images) == 1
    if route.startswith("slab"):
        on_device = route == "slab_device"
        ngroups, works = _image_works(0, images[0], flags, niter, on_device, sched)
        out = []
        for g in range(ngroups):                                  # run_slab 1519-1535
            c0, c1 = group_range(ngroups, len(images[0].comps), g)
            ws = [w for w in works[c0:c1] if w is not None]
            if ws:
                out += _phase_launches(ws, niter, num_sms)
        return out
    return _run_images(images, flags, niter, on_device, num_sms, slabs and route == "host", sched)


def _run_images(images, flags, niter, on_device, num_sms, slabs, sched) -> List[Launch]:
    per = [_image_works(n, im, flags, niter, on_device, sched) for n, im in enumerate(images)]
    max_groups = max([ng for ng, _ in per] + [0])
    out = []
    for g in range(max_groups):
        plan = None
        if slabs and len(images) == 1 and niter >= 1 and g < per[0][0] and not on_device:
            plan = _slab_plan(images[0], per[0][1], per[0][0], g, num_sms)
        works = []
        for (ng, ws), im in zip(per, images):
            if g >= ng:
                continue
            c0, c1 = group_range(ng, len(im.comps), g)
            works += [w for w in ws[c0:c1] if w is not None]
        if not works:
            continue
        slab_in = plan is not None
        if slab_in:                                               # run_images 1117-1122
            c0, c1 = group_range(per[0][0], len(images[0].comps), g)
            slab_in = len(works) == c1 - c0 and all(
                w.niter2 == works[0].niter2 and w.extra == works[0].extra and w.niter2 >= 1 for w in works)
        slab_out = slab_in and works[0].niter2 >= 2 and not works[0].extra and g == per[0][0] - 1
        if slab_in and g > 0:
            slab_in = False
        out += _phase_launches(works, niter, num_sms, plan, slab_in, slab_out)
    return out


def regimes(launches: Sequence[Launch]) -> set:
    """The regimes a run's launches reach: 'dynamic+tail', 'rounds', 'tail', and 'mixed' when
    a dynamic group tile spans jobs with different signatures."""
    out = {l.regime for l in launches}
    if any(l.mixed for l in launches):
        out.add("mixed")
    return out


def geometry(width: int, height: int, subsampling: str, quant=None) -> CoefImage:
    """An image of the given libjpeg geometry whose coefficient arrays are zero-strided views
    (nothing is allocated): enough for smooth_launches.  quant: (luma, chroma) tables."""
    from jpegqs_b200 import synth
    if quant is None:
        quant = (synth.quality_table(synth.ANNEX_K_LUMA, 50), synth.quality_table(synth.ANNEX_K_CHROMA, 50))
    if subsampling == "gray":
        samp, cs = [(1, 1)], JCS_GRAYSCALE
    else:
        samp = [{"444": (1, 1), "422": (2, 1), "420": (2, 2), "440": (1, 2)}[subsampling], (1, 1), (1, 1)]
        cs = JCS_YCbCr
    mh, mv = max(s[0] for s in samp), max(s[1] for s in samp)
    z = np.zeros((1, 1, 64), dtype=np.int16)
    comps = [Component(np.broadcast_to(z, (blocks_for(height, v, mv), blocks_for(width, h, mh), 64)),
                       np.asarray(quant[0 if c == 0 else 1], dtype=np.uint16), h, v, 0 if c == 0 else 1)
             for c, (h, v) in enumerate(samp)]
    return CoefImage(width, height, cs, comps)
