"""Host-side checks of the stream-ordered entry point (jpegqs_cuda_run_async): the workspace
size it asks for, the geometry it rejects, and the Python argument checks that run before the
library is called.  No device needed."""
import numpy as np
import pytest

import jpegqs_b200 as qs
import wave_geometry as wg
from jpegqs_b200 import cuda as qc

SAMPLINGS = ("gray", "420", "422", "444", "440")
FIXED = 4352 + 2 * 1024 * 80          # flags + tile counter, two job-list slots of QS_MAX_JOBS
QUANT_RECORD = 1544                   # sizeof(QsQuantDev)


def _a(x):
    return (x + 255) // 256 * 256


def _plane(wblk, hblk):
    return (wblk * 8 + 32) * (hblk * 8 + 2)


def documented_bytes(images, flags):
    """The sum stated in include/jpegqs_cuda.h for jpegqs_cuda_async_workspace_bytes."""
    ncomp = sum(len(im.comps) for im in images)
    total = FIXED + _a(QUANT_RECORD * ncomp)
    for im in images:
        cs = im.comps
        total += sum(_a(_plane(c.wblk, c.hblk)) for c in cs)
        down = (flags & 6) and im.colorspace == qs.JCS_YCbCr and len(cs) >= 3 and \
            all((c.h_samp, c.v_samp) == (1, 1) for c in cs[1:3]) and (cs[0].h_samp, cs[0].v_samp) != (1, 1)
        if down:
            total += _a(_plane(cs[1].wblk, cs[1].hblk))
            if flags & 4:
                total += 2 * _a(cs[0].wblk * cs[0].hblk * 64)
    return total


@pytest.mark.parametrize("flags", [0, 1, 2, 3, 4, 7, 8, 16 | 32])
@pytest.mark.parametrize("ss", SAMPLINGS)
def test_workspace_bytes_single_image(ss, flags):
    for w, h in ((208, 144), (1000, 333), (8, 8), (4096, 2160)):
        im = wg.geometry(w, h, ss)
        assert qc.async_workspace_bytes([im], flags) == documented_bytes([im], flags)


@pytest.mark.parametrize("flags", [0, 3, 7])
def test_workspace_bytes_batch(flags):
    ims = [wg.geometry(200 + 24 * k, 120 + 16 * k, ss) for k, ss in enumerate(SAMPLINGS * 2)]
    got = qc.async_workspace_bytes(ims, flags)
    assert got == documented_bytes(ims, flags)
    # the sum runs over the images: each image adds what it needs alone, less the fixed part
    assert got - FIXED - _a(QUANT_RECORD * sum(len(im.comps) for im in ims)) == sum(
        documented_bytes([im], flags) - FIXED - _a(QUANT_RECORD * len(im.comps)) for im in ims)


def test_workspace_bytes_of_no_image():
    assert qc.async_workspace_bytes([], 7) == FIXED


def test_upsampling_needs_the_down_sampled_luma_only_for_subsampled_luma():
    im444, im420 = wg.geometry(640, 480, "444"), wg.geometry(640, 480, "420")
    assert qc.async_workspace_bytes([im444], 7) == qc.async_workspace_bytes([im444], 0)
    assert qc.async_workspace_bytes([im420], 7) > qc.async_workspace_bytes([im420], 3) > \
        qc.async_workspace_bytes([im420], 0)
    assert qc.upsample_can_trigger(im420, 4) and not qc.upsample_can_trigger(im444, 4)
    assert not qc.upsample_can_trigger(im420, 3)


def _raw(images):
    return qc._image_array(images)


def test_workspace_bytes_rejects_malformed_images():
    lib = qc.load()
    im = wg.geometry(320, 240, "420")
    out = qc.C.c_size_t(0)
    for ncomp in (0, 11, -1):
        arr = _raw([im])
        arr[0].ncomp = ncomp
        assert lib.jpegqs_cuda_async_workspace_bytes(1, arr, 0, qc.C.byref(out)) == -2
    # unequal chroma components: rejected where JOINT_YUV / UPSAMPLE_UV down-sample the luma
    arr = _raw([im])
    arr[0].comp[2].wblk += 1
    for flags in (2, 4, 7):
        assert lib.jpegqs_cuda_async_workspace_bytes(1, arr, flags, qc.C.byref(out)) == -2
    assert lib.jpegqs_cuda_async_workspace_bytes(1, arr, 1, qc.C.byref(out)) == 0
    # a sampling factor outside 1..4
    arr = _raw([im])
    arr[0].comp[0].h_samp = 0
    assert lib.jpegqs_cuda_async_workspace_bytes(1, arr, 0, qc.C.byref(out)) == -2
    # one bad image spoils the batch; a NULL result pointer is an argument error too
    arr = _raw([im, im])
    arr[1].ncomp = 11
    assert lib.jpegqs_cuda_async_workspace_bytes(2, arr, 0, qc.C.byref(out)) == -2
    assert lib.jpegqs_cuda_async_workspace_bytes(1, _raw([im]), 0, None) == -2
    with pytest.raises(qc.QsError):
        bad = wg.geometry(320, 240, "420")
        bad.comps[0].h_samp = 5
        qc.async_workspace_bytes([bad], 0)


# ---- the Python argument checks of run_async -------------------------------------------------

class _Untouchable:
    """Stands in for the library: any use of it fails the test."""

    def __getattr__(self, name):
        raise AssertionError(f"the library was called ({name}) before the arguments were checked")


def _ctx():
    ctx = object.__new__(qc.QsContext)
    ctx.lib, ctx.h, ctx.device = _Untouchable(), None, 0
    return ctx


def _image():
    return wg.geometry(64, 48, "420")


def _tensors(im, dtype=None, shape=None, device="cpu"):
    import torch
    return [torch.zeros(shape or (c.hblk, c.wblk, 64), dtype=dtype or torch.int16, device=device)
            for c in im.comps]


def test_run_async_rejects_a_wrong_dtype():
    import torch
    im = _image()
    with pytest.raises(TypeError, match="dtype"):
        _ctx().run_async([im], [_tensors(im, dtype=torch.int32)], 0, 1)
    with pytest.raises(TypeError, match="torch.Tensor"):
        _ctx().run_async([im], [[np.zeros((c.hblk, c.wblk, 64), np.int16) for c in im.comps]], 0, 1)


def test_run_async_rejects_a_wrong_shape():
    im = _image()
    ts = _tensors(im)
    import torch
    ts[1] = torch.zeros((im.comps[1].hblk + 1, im.comps[1].wblk, 64), dtype=torch.int16)
    with pytest.raises(ValueError, match="shape"):
        _ctx().run_async([im], [ts], 0, 1)
    with pytest.raises(ValueError, match="coefficient tensors"):
        _ctx().run_async([im], [_tensors(im)[:2]], 0, 1)


def test_run_async_rejects_non_contiguous_tensors():
    import torch
    im = _image()
    ts = _tensors(im)
    c = im.comps[0]
    ts[0] = torch.zeros((c.wblk, c.hblk, 64), dtype=torch.int16).transpose(0, 1)
    with pytest.raises(ValueError, match="contiguous"):
        _ctx().run_async([im], [ts], 0, 1)


def test_run_async_rejects_cpu_tensors():
    im = _image()
    with pytest.raises(ValueError, match="expected cuda:0"):
        _ctx().run_async([im], [_tensors(im)], 0, 1)
    with pytest.raises(ValueError, match="CUDA tensors"):
        qs.run_async([im], [_tensors(im)], 0, 1)


def test_run_async_rejects_wrong_up_tensors():
    im = _image()
    with pytest.raises(ValueError, match="expected cuda:0"):
        _ctx().run_async([im], [_tensors(im, device="meta")], 7, 1)
    with pytest.raises(ValueError, match="one entry per image"):
        _ctx().run_async([im], [_tensors(im)], 7, 1, up=[None, None])
