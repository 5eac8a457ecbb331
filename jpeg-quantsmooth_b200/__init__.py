"""jpegqs_b200 - H100-native (sm_90a) implementation of jpeg-quantsmooth's
coefficient-smoothing hot path.  See DESIGN.md.

Host-side Python mirror of the reference's API surface for that path:
`do_quantsmooth(image, flags, niter)` (reference libjpegqs.h:47-48) over the
C-ABI shared library `csrc/libjpegqs_b200.so` (declared in include/jpegqs_cuda.h).
There is no CPU fallback: if the CUDA library is missing or no device is
usable the calls raise.
"""
from .image import (CoefImage, Component, JCS_GRAYSCALE, JCS_YCbCr, JCS_RGB,  # noqa: F401
                    JCS_UNKNOWN, JCS_CMYK, JCS_YCCK, blocks_for)
from . import synth  # noqa: F401

JPEGQS_ITER_MAX = 100
JPEGQS_DIAGONALS = 1
JPEGQS_JOINT_YUV = 2
JPEGQS_UPSAMPLE_UV = 4
JPEGQS_LOW_QUALITY = 8
JPEGQS_NO_REBALANCE = 16
JPEGQS_NO_REBALANCE_UV = 32
JPEGQS_TRANSCODE = 64


def quality_to_flags(quality: int) -> int:
    """The CLI's -q mapping (reference quantsmooth.c:380-393)."""
    flags = 0
    if quality < 3:
        flags |= JPEGQS_LOW_QUALITY
        quality += 4
    if quality >= 4:
        flags |= JPEGQS_DIAGONALS
    if quality >= 5:
        flags |= JPEGQS_JOINT_YUV
    if quality >= 6:
        flags |= JPEGQS_UPSAMPLE_UV
    return flags


def __getattr__(name):
    # the CUDA binding is imported lazily so that the host-only helpers
    # (synth, image) work on a machine without the built extension
    if name in ("cuda", "do_quantsmooth", "run_async", "render_async", "async_workspace_bytes", "QsContext", "lib_path",
                "parse_jpeg", "read_jpeg", "decode_async", "decode_workspace_bytes", "decode_model",
                "jpeg_prefix", "encode_bound", "encode_workspace_bytes", "encode_model", "encode_async",
                "parse_jpeg_scans", "decode_scans_async", "decode_scans_workspace_bytes", "decode_scans_model",
                "transcode_route", "transcode", "transcode_batch", "decode_pixels", "render_model", "resize_model",
                "compress_model", "compress_bound", "compress_async", "reencode", "exif_orientation",
                "thumbnail_geometry", "thumbnail_model", "reduce_model", "resize_model_box", "image_filter_model"):
        import importlib
        _cuda = importlib.import_module(__name__ + ".cuda")
        if name == "cuda":
            return _cuda
        return getattr(_cuda, name)
    raise AttributeError(name)
