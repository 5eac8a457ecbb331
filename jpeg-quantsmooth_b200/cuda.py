"""ctypes binding of the C ABI in include/jpegqs_cuda.h (csrc/libjpegqs_b200.so) and the
Python mirror of the reference's public call for this path:

    ret, out = do_quantsmooth(image, flags, niter)      # reference libjpegqs.h:47-48

`image` is the flat equivalent of (j_decompress_ptr, coef_arrays) - see image.py.
There is no CPU fallback: a missing library or device raises QsError.
"""
from __future__ import annotations

import ctypes as C
import math
import os
from typing import List, Optional, Sequence

import numpy as np

from .image import CoefImage, Component, JCS_YCbCr

_HERE = os.path.dirname(os.path.abspath(__file__))
MAX_COMP = 10


class QsError(RuntimeError):
    pass


def lib_path() -> str:
    # JPEGQS_B200_LIB: measurement builds of the same library (csrc/Makefile `experiments`,
    # `phase`) for tools/; never another implementation - there is no fallback of any kind
    return os.environ.get("JPEGQS_B200_LIB") or os.path.join(_HERE, "csrc", "libjpegqs_b200.so")


class _Comp(C.Structure):
    _fields_ = [("coef", C.c_void_p), ("wblk", C.c_uint32), ("hblk", C.c_uint32),
                ("h_samp", C.c_int32), ("v_samp", C.c_int32), ("has_qtbl", C.c_int32),
                ("quant", C.c_uint16 * 64), ("coef_up", C.c_void_p),
                ("rows", C.c_void_p), ("rows_up", C.c_void_p)]


class _Image(C.Structure):
    _fields_ = [("ncomp", C.c_int32), ("is_ycbcr", C.c_int32),
                ("image_width", C.c_uint32), ("image_height", C.c_uint32),
                ("comp", _Comp * MAX_COMP), ("upsampled", C.c_int32)]


class _Scan(C.Structure):
    """jpegqs_cuda_scan: what is in force at a file's first SOS (include/jpegqs_cuda.h)."""
    _fields_ = [("ncomp", C.c_int32), ("comp", C.c_int32 * 4), ("dc_tbl", C.c_int32 * 4), ("ac_tbl", C.c_int32 * 4),
                ("dc_present", C.c_int32 * 4), ("ac_present", C.c_int32 * 4),
                ("dc_bits", (C.c_uint8 * 17) * 4), ("dc_val", (C.c_uint8 * 256) * 4),
                ("ac_bits", (C.c_uint8 * 17) * 4), ("ac_val", (C.c_uint8 * 256) * 4),
                ("restart_interval", C.c_uint32), ("entropy_offset", C.c_uint64),
                ("jpeg_color_space", C.c_int32), ("sof", C.c_int32)]


class _ScanRec(C.Structure):
    """jpegqs_cuda_scan_rec: one scan of a file as the host marker walk found it (include/jpegqs_cuda.h)."""
    _fields_ = [("ncomp", C.c_int32), ("comp", C.c_int32 * 4), ("dc_tbl", C.c_int32 * 4), ("ac_tbl", C.c_int32 * 4),
                ("Ss", C.c_int32), ("Se", C.c_int32), ("Ah", C.c_int32), ("Al", C.c_int32), ("sof", C.c_int32),
                ("dc_present", C.c_int32 * 4), ("ac_present", C.c_int32 * 4),
                ("dc_bits", (C.c_uint8 * 17) * 4), ("dc_val", (C.c_uint8 * 256) * 4),
                ("ac_bits", (C.c_uint8 * 17) * 4), ("ac_val", (C.c_uint8 * 256) * 4),
                ("restart_interval", C.c_uint32), ("offset", C.c_uint64), ("end", C.c_uint64)]


MAX_SCANS = 64


class _Head(C.Structure):
    """jpegqs_cuda_jpeg_head: the prefix and frame identifiers of one encoded file (include/jpegqs_cuda.h)."""
    _fields_ = [("prefix_dev", C.c_void_p), ("prefix_len", C.c_uint32), ("comp_id", C.c_int32 * 4),
                ("quant_tbl", C.c_int32 * 4)]


class _FileInfo(C.Structure):
    """jpegqs_cuda_file_info: what the jpegqs tool's -v line shows of a file (include/jpegqs_cuda.h)."""
    _fields_ = [("image_width", C.c_uint32), ("image_height", C.c_uint32), ("ncomp", C.c_int32),
                ("progressive", C.c_int32), ("restart_interval", C.c_int32)]


class _TranscodeResult(C.Structure):
    """jpegqs_cuda_transcode_result (include/jpegqs_cuda.h)."""
    _fields_ = [("data", C.c_void_p), ("len", C.c_size_t), ("smoothed", C.c_int32), ("stop", C.c_int32),
                ("upsampled", C.c_int32), ("reason", C.c_char_p)]


class _PixelsResult(C.Structure):
    """jpegqs_cuda_pixels_result (include/jpegqs_cuda.h)."""
    _fields_ = [("channels", C.c_int32), ("host_decoded", C.c_int32), ("warnings", C.c_int32),
                ("smoothed", C.c_int32), ("stop", C.c_int32), ("upsampled", C.c_int32), ("reason", C.c_char_p)]


ROUTE_HOST, ROUTE_DEVICE = 0, 1
TRANSCODE_OK, TRANSCODE_FALLBACK = 0, 1


class _ResizeBox(C.Structure):
    _fields_ = [("left", C.c_int32), ("top", C.c_int32), ("right", C.c_int32), ("bottom", C.c_int32),
                ("width", C.c_int32), ("height", C.c_int32)]


class _ImageFilter(C.Structure):
    """jpegqs_cuda_image_filter (include/jpegqs_cuda.h)."""
    _fields_ = [("kind", C.c_int32), ("radius_x", C.c_float), ("radius_y", C.c_float), ("percent", C.c_int32),
                ("threshold", C.c_int32)]


class _JpegParams(C.Structure):
    """jpegqs_cuda_jpeg_params (include/jpegqs_cuda.h)."""
    _fields_ = [("quality", C.c_int32), ("subsampling", C.c_int32), ("optimize", C.c_int32)]


class _PixelsIn(C.Structure):
    """jpegqs_cuda_pixels_in (include/jpegqs_cuda.h)."""
    _fields_ = [("pixels_dev", C.c_void_p), ("width", C.c_int32), ("height", C.c_int32), ("channels", C.c_int32),
                ("row_bytes", C.c_size_t)]


class _Job(C.Structure):
    _fields_ = [("coef", C.c_void_p), ("plane", C.c_void_p), ("plane2", C.c_void_p),
                ("wblk", C.c_uint32), ("hblk", C.c_uint32), ("quant", C.c_uint16 * 64),
                ("luma", C.c_int32), ("top_edge", C.c_int32), ("bottom_edge", C.c_int32)]


class _Slab(C.Structure):
    _fields_ = [("rank", C.c_int32), ("world", C.c_int32),
                ("row0", C.c_uint32 * MAX_COMP), ("hblk_total", C.c_uint32 * MAX_COMP)]


PROGRESS_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int, C.c_int)
PASS_DEQUANT, PASS_CLAMP = 1, 2

_lib = None


def load():
    """Load the CUDA extension; raises QsError when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    p = lib_path()
    if not os.path.exists(p):
        raise QsError(f"{p} not built - run `python -c 'import __graft_entry__ as g; g.build()'` "
                      "(there is no CPU fallback)")
    lib = C.CDLL(p)
    lib.jpegqs_cuda_create.argtypes = [C.c_int, C.POINTER(C.c_void_p)]
    lib.jpegqs_cuda_destroy.argtypes = [C.c_void_p]
    lib.jpegqs_cuda_last_error.argtypes = [C.c_void_p]
    lib.jpegqs_cuda_last_error.restype = C.c_char_p
    lib.jpegqs_cuda_device_name.argtypes = [C.c_void_p]
    lib.jpegqs_cuda_device_name.restype = C.c_char_p
    lib.jpegqs_cuda_last_device_ms.argtypes = [C.c_void_p]
    lib.jpegqs_cuda_last_device_ms.restype = C.c_float
    lib.jpegqs_cuda_last_launches.argtypes = [C.c_void_p]
    lib.jpegqs_cuda_host_alloc.argtypes = [C.c_size_t]
    lib.jpegqs_cuda_host_alloc.restype = C.c_void_p
    lib.jpegqs_cuda_host_free.argtypes = [C.c_void_p]
    lib.jpegqs_cuda_run_host.argtypes = [C.c_void_p, C.POINTER(_Image), C.c_int, C.c_int, C.c_int,
                                         C.c_void_p, C.c_void_p]
    lib.jpegqs_cuda_run_device.argtypes = [C.c_void_p, C.POINTER(_Image), C.c_int, C.c_int, C.c_int,
                                           C.c_void_p, C.c_void_p, C.c_void_p]
    lib.jpegqs_cuda_run_batch.argtypes = [C.c_void_p, C.c_int, C.POINTER(_Image), C.c_int, C.c_int,
                                          C.c_int, C.POINTER(C.c_int), C.c_void_p]
    lib.jpegqs_cuda_plane_bytes.argtypes = [C.c_uint32, C.c_uint32]
    lib.jpegqs_cuda_plane_bytes.restype = C.c_size_t
    lib.jpegqs_cuda_plane_stride.argtypes = [C.c_uint32]
    lib.jpegqs_cuda_pass_idct.argtypes = [C.c_void_p, C.c_int, C.POINTER(_Job), C.c_int,
                                          C.POINTER(C.c_int), C.c_void_p]
    lib.jpegqs_cuda_pass_smooth.argtypes = [C.c_void_p, C.c_int, C.POINTER(_Job), C.c_int, C.c_int,
                                            C.c_void_p]
    lib.jpegqs_cuda_pass_downsample.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32,
                                                C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                                C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
    lib.jpegqs_cuda_pass_upsample.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p,
                                              C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p,
                                              C.c_int, C.c_int, C.c_uint32, C.c_uint32, C.c_void_p]
    lib.jpegqs_cuda_render_rgb.argtypes = [C.c_void_p, C.POINTER(_Image), C.c_int, C.c_void_p, C.c_void_p]
    lib.jpegqs_cuda_set_profiling.argtypes = [C.c_void_p, C.c_int]
    lib.jpegqs_cuda_kernel_stats.argtypes = [C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_int),
                                             C.POINTER(C.c_float), C.POINTER(C.c_int)]
    lib.jpegqs_cuda_set_tuning.argtypes = [C.c_void_p, C.c_int, C.c_int]
    lib.jpegqs_cuda_link_create.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_uint32, C.POINTER(C.c_void_p)]
    lib.jpegqs_cuda_link_destroy.argtypes = [C.c_void_p]
    lib.jpegqs_cuda_link_export.argtypes = [C.c_void_p, C.c_void_p]
    lib.jpegqs_cuda_link_connect_ipc.argtypes = [C.c_void_p, C.c_void_p]
    lib.jpegqs_cuda_link_connect_local.argtypes = [C.POINTER(C.c_void_p), C.c_int]
    lib.jpegqs_cuda_run_slab.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(_Image), C.POINTER(_Slab), C.c_int,
                                         C.c_int, C.c_int, C.c_void_p]
    lib.jpegqs_cuda_multi_create.argtypes = [C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_void_p)]
    lib.jpegqs_cuda_multi_destroy.argtypes = [C.c_void_p]
    lib.jpegqs_cuda_multi_devices.argtypes = [C.c_void_p]
    lib.jpegqs_cuda_multi_ctx.argtypes = [C.c_void_p, C.c_int]
    lib.jpegqs_cuda_multi_ctx.restype = C.c_void_p
    lib.jpegqs_cuda_multi_last_error.argtypes = [C.c_void_p]
    lib.jpegqs_cuda_multi_last_error.restype = C.c_char_p
    lib.jpegqs_cuda_multi_plan.argtypes = [C.c_void_p, C.POINTER(_Image)]
    lib.jpegqs_cuda_run_host_multi.argtypes = [C.c_void_p, C.POINTER(_Image), C.c_int, C.c_int]
    lib.jpegqs_cuda_async_workspace_bytes.argtypes = [C.c_int, C.POINTER(_Image), C.c_int, C.POINTER(C.c_size_t)]
    lib.jpegqs_cuda_run_async.argtypes = [C.c_void_p, C.c_int, C.POINTER(_Image), C.c_int, C.c_int, C.c_void_p,
                                          C.c_size_t, C.c_void_p, C.c_void_p]
    lib.jpegqs_cuda_render_async.argtypes = [C.c_void_p, C.c_int, C.POINTER(_Image), C.c_void_p, C.c_int,
                                             C.c_void_p, C.c_void_p]
    lib.jpegqs_cuda_render_scaled_async.argtypes = [C.c_void_p, C.c_int, C.POINTER(_Image), C.c_void_p, C.c_int,
                                                    C.c_int, C.c_void_p, C.c_void_p]
    lib.jpegqs_cuda_render_model.argtypes = [C.POINTER(_Image), C.c_int, C.c_int, C.c_int, C.c_void_p]
    lib.jpegqs_cuda_jpeg_parse.argtypes = [C.c_char_p, C.c_size_t, C.POINTER(_Image), C.POINTER(_Scan)]
    lib.jpegqs_cuda_jpeg_read.argtypes = [C.c_char_p, C.c_size_t, C.POINTER(_Image)]
    lib.jpegqs_cuda_decode_workspace_bytes.argtypes = [C.c_int, C.POINTER(_Image), C.POINTER(_Scan),
                                                       C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]
    lib.jpegqs_cuda_decode_async.argtypes = [C.c_void_p, C.c_int, C.POINTER(_Image), C.POINTER(_Scan), C.c_void_p,
                                             C.POINTER(C.c_size_t), C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
    lib.jpegqs_cuda_decode_model.argtypes = [C.POINTER(_Image), C.POINTER(_Scan), C.c_char_p, C.c_size_t, C.c_int,
                                             C.POINTER(C.c_int32), C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
    lib.jpegqs_cuda_jpeg_parse_scans.argtypes = [C.c_char_p, C.c_size_t, C.POINTER(_Image), C.POINTER(_ScanRec), C.c_int,
                                                 C.POINTER(C.c_int)]
    lib.jpegqs_cuda_decode_scans_workspace_bytes.argtypes = [C.c_int, C.POINTER(_Image), C.c_void_p, C.c_void_p,
                                                             C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]
    lib.jpegqs_cuda_decode_scans_async.argtypes = [C.c_void_p, C.c_int, C.POINTER(_Image), C.c_void_p, C.c_void_p,
                                                   C.c_void_p, C.POINTER(C.c_size_t), C.c_void_p, C.c_size_t, C.c_void_p,
                                                   C.c_void_p]
    lib.jpegqs_cuda_decode_scans_model.argtypes = [C.POINTER(_Image), C.POINTER(_ScanRec), C.c_int, C.c_char_p, C.c_size_t,
                                                   C.c_int, C.POINTER(C.c_int32)]
    lib.jpegqs_cuda_jpeg_prefix.argtypes = [C.c_char_p, C.c_size_t, C.c_int, C.c_void_p, C.c_size_t,
                                            C.POINTER(C.c_size_t), C.POINTER(C.c_int32), C.c_int32 * 4, C.c_int32 * 4]
    lib.jpegqs_cuda_encode_bound.argtypes = [C.POINTER(_Image), C.c_size_t, C.POINTER(C.c_size_t)]
    lib.jpegqs_cuda_encode_workspace_bytes.argtypes = [C.c_int, C.POINTER(_Image), C.c_int, C.POINTER(C.c_size_t)]
    lib.jpegqs_cuda_encode_async.argtypes = [C.c_void_p, C.c_int, C.POINTER(_Image), C.POINTER(_Head), C.c_int,
                                             C.c_void_p, C.c_void_p, C.POINTER(C.c_size_t), C.c_void_p, C.c_void_p,
                                             C.c_void_p, C.c_size_t, C.c_void_p]
    lib.jpegqs_cuda_encode_model.argtypes = [C.POINTER(_Image), C.POINTER(_Head), C.c_int, C.c_void_p, C.c_size_t,
                                             C.POINTER(C.c_uint64), C.POINTER(C.c_int32)]
    lib.jpegqs_cuda_transcode_route.argtypes = [C.c_char_p, C.c_size_t, C.POINTER(C.c_char_p), C.POINTER(_FileInfo)]
    lib.jpegqs_cuda_transcode.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_int,
                                          C.POINTER(_TranscodeResult)]
    lib.jpegqs_cuda_transcode_free.argtypes = [C.c_void_p]
    lib.jpegqs_cuda_transcode_batch.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_size_t), C.c_int,
                                                C.c_int, C.c_int, C.c_int, C.c_size_t, C.POINTER(C.c_int),
                                                C.POINTER(_TranscodeResult)]
    lib.jpegqs_cuda_pixels_batch.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_size_t), C.c_int,
                                             C.c_int, C.c_int, C.c_int, C.POINTER(C.c_void_p), C.c_size_t,
                                             C.POINTER(C.c_int), C.POINTER(_PixelsResult)]
    lib.jpegqs_cuda_pixels_batch_scaled.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_size_t),
                                                    C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_void_p),
                                                    C.c_size_t, C.POINTER(C.c_int), C.POINTER(_PixelsResult)]
    lib.jpegqs_cuda_pixels_batch_resized.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_size_t),
                                                     C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(_ResizeBox),
                                                     C.c_int, C.POINTER(C.c_void_p), C.c_size_t, C.POINTER(C.c_int),
                                                     C.POINTER(_PixelsResult)]
    lib.jpegqs_cuda_resize_model.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                             C.POINTER(_ResizeBox), C.c_void_p]
    lib.jpegqs_cuda_compress_bound.argtypes = [C.POINTER(_PixelsIn), C.POINTER(_JpegParams), C.POINTER(C.c_size_t)]
    lib.jpegqs_cuda_compress_workspace_bytes.argtypes = [C.c_int, C.POINTER(_PixelsIn), C.POINTER(_JpegParams),
                                                         C.POINTER(C.c_size_t)]
    lib.jpegqs_cuda_compress_async.argtypes = [C.c_void_p, C.c_int, C.POINTER(_PixelsIn), C.POINTER(_JpegParams),
                                               C.c_void_p, C.POINTER(C.c_size_t), C.c_void_p, C.c_void_p, C.c_void_p,
                                               C.c_size_t, C.c_void_p]
    lib.jpegqs_cuda_compress_model.argtypes = [C.POINTER(_PixelsIn), C.POINTER(_JpegParams), C.c_void_p, C.c_size_t,
                                               C.POINTER(C.c_uint64), C.POINTER(C.c_int32)]
    lib.jpegqs_cuda_pixels_batch_jpeg.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_size_t),
                                                  C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(_ResizeBox),
                                                  C.POINTER(_JpegParams), C.c_size_t, C.POINTER(C.c_int),
                                                  C.POINTER(_PixelsResult), C.POINTER(C.c_void_p),
                                                  C.POINTER(C.c_size_t)]
    lib.jpegqs_cuda_jpeg_orientation.argtypes = [C.c_char_p, C.c_size_t, C.POINTER(C.c_int32)]
    lib.jpegqs_cuda_render_oriented_async.argtypes = [C.c_void_p, C.c_int, C.POINTER(_Image), C.c_void_p, C.c_int, C.c_int,
                                                      C.POINTER(C.c_int32), C.POINTER(C.c_void_p), C.c_void_p]
    lib.jpegqs_cuda_pixels_batch_oriented.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_size_t),
                                                      C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(_ResizeBox),
                                                      C.POINTER(C.c_int32), C.c_int, C.POINTER(C.c_void_p), C.c_size_t,
                                                      C.POINTER(C.c_int), C.POINTER(_PixelsResult)]
    lib.jpegqs_cuda_pixels_batch_jpeg_oriented.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_char_p),
                                                           C.POINTER(C.c_size_t), C.c_int, C.c_int, C.c_int, C.c_int,
                                                           C.POINTER(_ResizeBox), C.POINTER(_JpegParams), C.c_size_t,
                                                           C.POINTER(C.c_int), C.POINTER(_PixelsResult),
                                                           C.POINTER(C.c_void_p), C.POINTER(C.c_size_t),
                                                           C.POINTER(C.c_int32)]
    lib.jpegqs_cuda_render_mode_async.argtypes = [C.c_void_p, C.c_int, C.POINTER(_Image), C.c_void_p, C.c_int, C.c_int,
                                                  C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_int,
                                                  C.POINTER(C.c_void_p), C.c_void_p]
    lib.jpegqs_cuda_render_model_mode.argtypes = [C.POINTER(_Image), C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                                  C.c_void_p]
    lib.jpegqs_cuda_pixels_batch_mode.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_size_t),
                                                  C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(_ResizeBox),
                                                  C.POINTER(C.c_int32), C.c_int, C.c_int, C.POINTER(C.c_void_p),
                                                  C.c_size_t, C.POINTER(C.c_int), C.POINTER(_PixelsResult)]
    lib.jpegqs_cuda_pixels_batch_jpeg_mode.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_char_p),
                                                       C.POINTER(C.c_size_t), C.c_int, C.c_int, C.c_int, C.c_int,
                                                       C.POINTER(_ResizeBox), C.POINTER(_JpegParams), C.c_size_t,
                                                       C.POINTER(C.c_int), C.POINTER(_PixelsResult),
                                                       C.POINTER(C.c_void_p), C.POINTER(C.c_size_t),
                                                       C.POINTER(C.c_int32), C.c_int]
    lib.jpegqs_cuda_thumbnail_geometry.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, C.c_int,
                                                   C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]
    lib.jpegqs_cuda_pixels_batch_reduced.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_size_t),
                                                     C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(_ResizeBox),
                                                     C.POINTER(C.c_int32), C.c_int, C.c_int, C.POINTER(C.c_void_p),
                                                     C.c_size_t, C.POINTER(C.c_int), C.POINTER(_PixelsResult), C.c_int,
                                                     C.c_double]
    lib.jpegqs_cuda_pixels_batch_jpeg_reduced.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_char_p),
                                                          C.POINTER(C.c_size_t), C.c_int, C.c_int, C.c_int, C.c_int,
                                                          C.POINTER(_ResizeBox), C.POINTER(_JpegParams), C.c_size_t,
                                                          C.POINTER(C.c_int), C.POINTER(_PixelsResult),
                                                          C.POINTER(C.c_void_p), C.POINTER(C.c_size_t),
                                                          C.POINTER(C.c_int32), C.c_int, C.c_int, C.c_double]
    lib.jpegqs_cuda_reduce_model.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                             C.POINTER(C.c_int32), C.c_void_p]
    lib.jpegqs_cuda_resize_model_box.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                                 C.POINTER(C.c_double), C.c_int, C.c_int, C.c_double, C.c_void_p]
    lib.jpegqs_cuda_pixels_batch_filtered.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_size_t),
                                                      C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(_ResizeBox),
                                                      C.POINTER(C.c_int32), C.c_int, C.c_int, C.POINTER(C.c_void_p),
                                                      C.c_size_t, C.POINTER(C.c_int), C.POINTER(_PixelsResult), C.c_int,
                                                      C.c_double, C.POINTER(_ImageFilter), C.c_int]
    lib.jpegqs_cuda_pixels_batch_jpeg_filtered.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_char_p),
                                                           C.POINTER(C.c_size_t), C.c_int, C.c_int, C.c_int, C.c_int,
                                                           C.POINTER(_ResizeBox), C.POINTER(_JpegParams), C.c_size_t,
                                                           C.POINTER(C.c_int), C.POINTER(_PixelsResult),
                                                           C.POINTER(C.c_void_p), C.POINTER(C.c_size_t),
                                                           C.POINTER(C.c_int32), C.c_int, C.c_int, C.c_double,
                                                           C.POINTER(_ImageFilter), C.c_int]
    lib.jpegqs_cuda_image_filter_model.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(_ImageFilter), C.c_int,
                                                   C.c_void_p]
    lib.jpegqs_cuda_tables.argtypes = [C.c_int, C.c_void_p]
    lib.jpegqs_cuda_orig_coef.argtypes = [C.c_int, C.c_int]
    _lib = lib
    return lib


def tables(flags: int) -> np.ndarray:
    """The weight tables the device uses (un-scaled), [64, 160|272] float32.  Host-only."""
    size = 272 if flags & 1 else 160
    out = np.zeros((64, size), dtype=np.float32)
    load().jpegqs_cuda_tables(flags, out.ctypes.data)
    return out


def orig_coef(coef: int, q: int) -> int:
    return load().jpegqs_cuda_orig_coef(coef, q)


def chunk_schedule(quant, max_coefs: int = 4, uniform: bool = True, merge: bool = True):
    """The smoothing kernel's chunk schedule for a quant table (or the table-independent one
    for quant=None): list of (type, first, [natural-order coefficient indices]).  Host-only."""
    lib = load()
    lib.jpegqs_cuda_chunk_schedule.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    out = np.zeros((64, 12), dtype=np.uint8)
    qp = None
    if quant is not None:
        qa = np.ascontiguousarray(quant, dtype=np.uint16).reshape(64)
        qp = qa.ctypes.data
    n = lib.jpegqs_cuda_chunk_schedule(qp, max_coefs, int(uniform) | (2 if merge else 0), out.ctypes.data)
    if n < 0:
        raise QsError(f"jpegqs_cuda_chunk_schedule: {n}")
    # type 3 ("mixed"): n full coefficients followed by the row-0 and the column-0 coefficient
    return [(int(r[0]), int(r[2]), [int(x) for x in r[4:4 + r[1] + (2 if r[0] == 3 else 0)]]) for r in out[:n]]


class PinnedArray:
    """int16 numpy view over pinned host memory from jpegqs_cuda_host_alloc."""

    def __init__(self, shape):
        n = int(np.prod(shape)) * 2
        self._lib = load()
        self._p = self._lib.jpegqs_cuda_host_alloc(max(n, 1))
        if not self._p:
            raise QsError("cudaMallocHost failed")
        buf = (C.c_int16 * (n // 2)).from_address(self._p)
        self.array = np.frombuffer(buf, dtype=np.int16).reshape(shape)

    def close(self):
        if self._p:
            self.array = None
            self._lib.jpegqs_cuda_host_free(self._p)
            self._p = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


SCALE_DENOMS = (1, 2, 4, 8)


def _scale_denom(d, who: str) -> int:
    if isinstance(d, bool) or not isinstance(d, (int, np.integer)) or int(d) not in SCALE_DENOMS:
        raise ValueError(f"{who}: scale_denom {d!r}: expected 1, 2, 4 or 8")
    return int(d)


def _scaled_shape(width: int, height: int, channels: int, layout: str, d: int):
    """libjpeg's output size at scale 1/d: ceil(width / d) x ceil(height / d)"""
    w, h = -(-int(width) // d), -(-int(height) // d)
    return (h, w, channels) if layout == "hwc" else (channels, h, w)


# Pillow's convolution filters, by name, with its Image.Resampling numbers (NEAREST, 0, is not one)
RESIZE_FILTERS = {"lanczos": 1, "bilinear": 2, "bicubic": 3, "box": 4, "hamming": 5}


def _resize_filter(f, who: str) -> int:
    """a filter name, or Pillow's Image.Resampling value of one of the five convolution filters"""
    if isinstance(f, str) and f.lower() in RESIZE_FILTERS:
        return RESIZE_FILTERS[f.lower()]
    if not isinstance(f, (str, bool)) and isinstance(f, (int, np.integer)) and int(f) in RESIZE_FILTERS.values():
        return int(f)
    raise ValueError(f"{who}: filter {f!r}: expected one of {', '.join(RESIZE_FILTERS)} (Pillow's BOX, BILINEAR, "
                     "HAMMING, BICUBIC, LANCZOS; NEAREST is not supported)")


def _int_tuple(v, k: int):
    if isinstance(v, (str, bytes)) or not hasattr(v, "__len__") or len(v) != k:
        return None
    if any(isinstance(x, bool) or not isinstance(x, (int, np.integer)) for x in v):
        return None
    return tuple(int(x) for x in v)


def _resize_boxes(n: int, size, crop, who: str):
    """Per file, (size, crop): size (width, height) or None, crop (left, top, right, bottom) or None,
    checked for form; ValueError names the file index"""
    def one_size(v, i):
        t = _int_tuple(v, 2)
        if t is None or not (1 <= t[0] <= 65535 and 1 <= t[1] <= 65535):
            raise ValueError(f"{who}: file {i}: size {v!r}: expected (width, height), each in 1..65535")
        return t
    if size is None:
        sizes = [None] * n
    elif _int_tuple(size, 2) is not None:
        sizes = [one_size(size, i) for i in range(n)]
    elif isinstance(size, (list, tuple)) and len(size) == n:
        sizes = [one_size(v, i) for i, v in enumerate(size)]
    else:
        raise ValueError(f"{who}: size must be (width, height) or a list of {n} of them")
    if crop is None:
        crops = [None] * n
    elif isinstance(crop, (list, tuple)) and len(crop) == n:
        crops = []
        for i, v in enumerate(crop):
            t = None if v is None else _int_tuple(v, 4)
            if v is not None and (t is None or min(t) < 0 or t[0] >= t[2] or t[1] >= t[3]):
                raise ValueError(f"{who}: file {i}: crop {v!r}: expected (left, top, right, bottom) with "
                                 "0 <= left < right and 0 <= top < bottom")
            crops.append(t)
    else:
        raise ValueError(f"{who}: crop must be None or a list of {n} (left, top, right, bottom) boxes or None")
    return sizes, crops


def _resize_box(pw: int, ph: int, size, crop, i: int, who: str) -> _ResizeBox:
    """the C box of file i, whose picture is pw x ph: crop None is the whole picture; size None is the crop's"""
    left, top, right, bottom = crop if crop is not None else (0, 0, pw, ph)
    if right > pw or bottom > ph:
        raise ValueError(f"{who}: file {i}: crop {crop!r} outside the {pw} x {ph} picture")
    w, h = size if size is not None else (right - left, bottom - top)
    return _ResizeBox(left, top, right, bottom, w, h)


class _GapDefault:
    """reducing_gap's default: Pillow's, 2.0 for thumbnail and None for size"""

    def __repr__(self):
        return "<Pillow's default>"


_GAP_DEFAULT = _GapDefault()


def _reducing_gap(gap, thumbnail: bool, who: str) -> float:
    """the C value of reducing_gap: 0.0 for None, else a finite value >= 1.0; the default is Pillow's"""
    if gap is _GAP_DEFAULT:
        return 2.0 if thumbnail else 0.0
    if gap is None:
        return 0.0
    if isinstance(gap, bool) or not isinstance(gap, (int, float, np.integer, np.floating)) or \
            not math.isfinite(float(gap)) or float(gap) < 1.0:
        raise ValueError(f"{who}: reducing_gap {gap!r}: expected None or a finite number of at least 1.0")
    return float(gap)


def _thumbnail_bounds(n: int, bound, who: str):
    """per file, a thumbnail bound (width, height), each 1..65535; ValueError names the file index"""
    def one(v, i):
        t = _int_tuple(v, 2)
        if t is None or not (1 <= t[0] <= 65535 and 1 <= t[1] <= 65535):
            raise ValueError(f"{who}: file {i}: thumbnail {v!r}: expected (width, height), each in 1..65535")
        return t
    if _int_tuple(bound, 2) is not None:
        return [one(bound, i) for i in range(n)]
    if isinstance(bound, (list, tuple)) and len(bound) == n:
        return [one(v, i) for i, v in enumerate(bound)]
    raise ValueError(f"{who}: thumbnail must be (width, height) or a list of {n} of them")


def thumbnail_geometry(width: int, height: int, bound, reducing_gap=2.0, loaded: bool = False):
    """Pillow's Image.thumbnail(bound, reducing_gap=reducing_gap) of a width x height JPEG file, host-only
    (jpegqs_cuda_thumbnail_geometry): (scale_denom, (out_width, out_height)).  scale_denom is the draft's
    libjpeg scale (1 when the bound covers the picture, for reducing_gap None, or loaded: the picture was
    decoded before, as exif_transpose and convert do); the size is the thumbnail's.  ValueError for a bad
    argument."""
    (bw, bh), = _thumbnail_bounds(1, bound, "thumbnail_geometry")
    gap = _reducing_gap(reducing_gap, True, "thumbnail_geometry")
    lib = load()
    s, w, h = C.c_int(), C.c_int(), C.c_int()
    if lib.jpegqs_cuda_thumbnail_geometry(int(width), int(height), bw, bh, gap, int(bool(loaded)), C.byref(s), C.byref(w),
                                          C.byref(h)) < 0:
        raise ValueError(f"thumbnail_geometry: {lib.jpegqs_cuda_last_error(None).decode()}")
    return s.value, (w.value, h.value)


def _host_pixels(pixels, who: str):
    a = np.asarray(pixels)
    if a.dtype != np.uint8 or a.ndim not in (2, 3) or (a.ndim == 3 and a.shape[2] not in (1, 3)) or 0 in a.shape:
        raise ValueError(f"{who}: pixels must be uint8 [H, W] or [H, W, 1|3], not {a.dtype} {a.shape}")
    return np.ascontiguousarray(a), (1 if a.ndim == 2 else a.shape[2])


def reduce_model(pixels, factor, box=None):
    """The device reduce on one CPU thread (jpegqs_cuda_reduce_model): byte for byte Pillow's
    Image.fromarray(pixels).reduce(factor, box).  pixels: uint8 [H, W] or [H, W, 1|3]; factor an int or
    (fx, fy); box (left, top, right, bottom) ints or None.  Returns [ceil(bh / fy), ceil(bw / fx)(, C)]."""
    a, c = _host_pixels(pixels, "reduce_model")
    f = _int_tuple((factor, factor) if _orient_int(factor) is not None else factor, 2)
    if f is None:
        raise ValueError(f"reduce_model: factor {factor!r}: expected an int or (fx, fy)")
    h, w = a.shape[:2]
    b = (0, 0, w, h) if box is None else _int_tuple(box, 4)
    if b is None:
        raise ValueError(f"reduce_model: box {box!r}: expected (left, top, right, bottom) ints")
    ow, oh = -(-(b[2] - b[0]) // max(f[0], 1)), -(-(b[3] - b[1]) // max(f[1], 1))
    out = np.zeros((max(oh, 0), max(ow, 0), c), dtype=np.uint8)
    lib = load()
    rc = lib.jpegqs_cuda_reduce_model(a.ctypes.data, w, h, c, f[0], f[1], (C.c_int32 * 4)(*b), out.ctypes.data)
    if rc < 0:
        raise ValueError(f"reduce_model: {lib.jpegqs_cuda_last_error(None).decode()} ({rc})")
    return out.reshape(oh, ow) if a.ndim == 2 else out


def resize_model_box(pixels, size, box=None, filter="bicubic", reducing_gap=None, layout: str = "hwc"):
    """The device reduce and resize on one CPU thread, planned as the batch plans them
    (jpegqs_cuda_resize_model_box): byte for byte Pillow's Image.fromarray(pixels).resize(size, filter,
    box=box, reducing_gap=reducing_gap), box (left, top, right, bottom) floats or None.  Returns
    [height, width] for a 2-D input, else [height, width, C] ("hwc") or [C, height, width] ("chw")."""
    if layout not in ("hwc", "chw"):
        raise ValueError(f"resize_model_box: layout {layout!r}: expected 'hwc' or 'chw'")
    a, c = _host_pixels(pixels, "resize_model_box")
    fcode = _resize_filter(filter, "resize_model_box")
    sz = _int_tuple(size, 2)
    if sz is None:
        raise ValueError(f"resize_model_box: size {size!r}: expected (width, height)")
    gap = _reducing_gap(reducing_gap, False, "resize_model_box")
    h, w = a.shape[:2]
    cbox = None
    if box is not None:
        if isinstance(box, (str, bytes)) or not hasattr(box, "__len__") or len(box) != 4:
            raise ValueError(f"resize_model_box: box {box!r}: expected (left, top, right, bottom)")
        cbox = (C.c_double * 4)(*[float(v) for v in box])
    shape = (max(sz[1], 0), max(sz[0], 0), c) if layout == "hwc" else (c, max(sz[1], 0), max(sz[0], 0))
    out = np.zeros(shape, dtype=np.uint8)
    lib = load()
    rc = lib.jpegqs_cuda_resize_model_box(a.ctypes.data, w, h, c, 0 if layout == "hwc" else 1, fcode, cbox, sz[0], sz[1],
                                          gap, out.ctypes.data)
    if rc < 0:
        raise ValueError(f"resize_model_box: {lib.jpegqs_cuda_last_error(None).decode()} ({rc})")
    return out.reshape(sz[1], sz[0]) if a.ndim == 2 else out


def thumbnail_model(pixels, full_size, bound, filter="bicubic", reducing_gap=2.0, loaded: bool = False):
    """Pillow's Image.thumbnail(bound, filter, reducing_gap) on one CPU thread, with the batch's planning:
    pixels is the picture thumbnail_geometry(W, H, bound, reducing_gap, loaded)'s draft gives, the
    W x H = full_size file at 1/scale_denom ([ceil(H / s), ceil(W / s)(, C)], as render_model gives it).
    Returns the thumbnail's pixels."""
    a, _ = _host_pixels(pixels, "thumbnail_model")
    W, H = (int(v) for v in full_size)
    s, (tw, th) = thumbnail_geometry(W, H, bound, reducing_gap, loaded)
    if a.shape[:2] != (-(-H // s), -(-W // s)):
        raise ValueError(f"thumbnail_model: pixels {a.shape[:2]}: expected the 1/{s} picture of {W} x {H}")
    if a.shape[:2] == (th, tw):
        return a.copy()
    gap = _reducing_gap(reducing_gap, True, "thumbnail_model")
    box = (0.0, 0.0, W / s, H / s) if gap and not loaded else None
    return resize_model_box(a, (tw, th), box, filter, gap or None)


# include/jpegqs_cuda.h: the largest radius magnitude (any axis, any filter) and UnsharpMask percent taken;
# beyond them Pillow's 32-bit sums would overflow
FILTER_MAX_RADIUS = 65535.0
FILTER_MAX_PERCENT = 8421504


def _filter_radius(v, who: str):
    import numbers
    if not isinstance(v, numbers.Real):
        raise ValueError(f"{who}: radius {v!r}: expected a number")
    r = float(v)
    if not abs(r) <= FILTER_MAX_RADIUS:
        raise ValueError(f"{who}: radius {v!r}: expected a finite value of magnitude at most {FILTER_MAX_RADIUS:g}")
    return r


def _filter_int(v, what: str, lim: int, who: str):
    import numbers
    if not isinstance(v, numbers.Integral) or not -lim <= int(v) <= lim:
        raise ValueError(f"{who}: {what} {v!r}: expected an int in -{lim}..{lim}")
    return int(v)


def _image_filters(image_filter, who: str):
    """image_filter (None, one filter or a sequence of them: Pillow's ImageFilter.GaussianBlur, BoxBlur or
    UnsharpMask, instances or classes) as a C array of jpegqs_cuda_image_filter, or None for no filter.
    ValueError names any other filter and a value Pillow's arithmetic cannot take."""
    if image_filter is None:
        return None
    seq = list(image_filter) if isinstance(image_filter, (list, tuple)) else [image_filter]
    if not seq:
        return None
    from PIL import ImageFilter
    kinds = {ImageFilter.BoxBlur: 1, ImageFilter.GaussianBlur: 2, ImageFilter.UnsharpMask: 3}
    out = (_ImageFilter * len(seq))()
    for k, f in enumerate(seq):
        w = f"{who}: image_filter {k}"
        if isinstance(f, type):
            if f not in kinds:
                raise ValueError(f"{w}: {f.__name__}: expected ImageFilter.GaussianBlur, BoxBlur or UnsharpMask")
            f = f()                                       # Image.filter's instance of a class: Pillow's defaults
        kind = kinds.get(type(f))
        if kind is None:
            raise ValueError(f"{w}: {type(f).__name__}: expected ImageFilter.GaussianBlur, BoxBlur or UnsharpMask")
        if kind == 3:
            r = _filter_radius(f.radius, w)
            out[k] = _ImageFilter(3, r, r, _filter_int(f.percent, "percent", FILTER_MAX_PERCENT, w),
                                  _filter_int(f.threshold, "threshold", 2 ** 31 - 1, w))
            continue
        xy = f.radius if isinstance(f.radius, (tuple, list)) else (f.radius, f.radius)
        if len(xy) != 2:
            raise ValueError(f"{w}: radius {f.radius!r}: expected a number or (x, y)")
        rx, ry = _filter_radius(xy[0], w), _filter_radius(xy[1], w)
        if kind == 1 and (rx < 0 or ry < 0):
            raise ValueError(f"{w}: radius {f.radius!r}: radius must be >= 0")
        out[k] = _ImageFilter(kind, rx, ry, 0, 0)
    return out


def image_filter_model(pixels, image_filter):
    """The device filters on one CPU thread, through the same pass plan (jpegqs_cuda_image_filter_model):
    byte for byte Pillow's Image.fromarray(pixels).filter(F1).filter(F2)... for image_filter F1 or
    [F1, F2, ...] (ImageFilter.GaussianBlur, BoxBlur or UnsharpMask).  pixels: uint8 [H, W] or
    [H, W, 1|3]; returns the same shape."""
    a, c = _host_pixels(pixels, "image_filter_model")
    filt = _image_filters(image_filter, "image_filter_model")
    h, w = a.shape[:2]
    out = np.empty_like(a)
    lib = load()
    rc = lib.jpegqs_cuda_image_filter_model(a.ctypes.data, w, h, c, filt, len(filt) if filt else 0, out.ctypes.data)
    if rc < 0:
        raise ValueError(f"image_filter_model: {lib.jpegqs_cuda_last_error(None).decode()} ({rc})")
    return out


def _fill_image(ci: _Image, image: CoefImage, coef_ptrs: Sequence[int], up_ptrs: Sequence[Optional[int]]):
    ci.ncomp = len(image.comps)
    ci.is_ycbcr = int(image.colorspace == JCS_YCbCr)
    ci.image_width, ci.image_height = image.width, image.height
    for i, c in enumerate(image.comps):
        cc = ci.comp[i]
        cc.coef = coef_ptrs[i]
        cc.wblk, cc.hblk, cc.h_samp, cc.v_samp = c.wblk, c.hblk, c.h_samp, c.v_samp
        cc.has_qtbl = int(c.quant is not None)
        if c.quant is not None:
            for k in range(64):
                cc.quant[k] = int(c.quant[k])
        cc.coef_up = up_ptrs[i] if i < len(up_ptrs) and up_ptrs[i] else None


def _image_array(images: Sequence[CoefImage], coef_ptrs=None, up_ptrs=None):
    arr = (_Image * max(len(images), 1))()
    for n, im in enumerate(images):
        _fill_image(arr[n], im, coef_ptrs[n] if coef_ptrs else [None] * len(im.comps),
                    up_ptrs[n] if up_ptrs else [])
    return arr


def upsample_can_trigger(image: CoefImage, flags: int) -> bool:
    """UPSAMPLE_UV replaces this image's chroma with luma-sized arrays unless the run stops
    (reference quantsmooth.h:2447-2453, 2691-2752)."""
    cs = image.comps
    return bool(flags & 4) and image.colorspace == JCS_YCbCr and len(cs) >= 3 and \
        all((c.h_samp, c.v_samp) == (1, 1) for c in cs[1:3]) and (cs[0].h_samp, cs[0].v_samp) != (1, 1)


def async_workspace_bytes(images: Sequence[CoefImage], flags: int) -> int:
    """Device bytes of workspace QsContext.run_async needs for these images (host-only)."""
    lib = load()
    out = C.c_size_t(0)
    arr = _image_array(images)
    rc = lib.jpegqs_cuda_async_workspace_bytes(len(images), arr, flags & 0x7f, C.byref(out))
    if rc < 0:
        raise QsError(f"jpegqs_cuda_async_workspace_bytes: malformed image ({rc})")
    return int(out.value)


# ---- JPEG files (include/jpegqs_cuda.h "JPEG files to quantized coefficients") ----
DECODE_BAD_CODE, DECODE_TRUNCATED, DECODE_RESTART, DECODE_AC_RUN, DECODE_UNITS = 1, 2, 4, 8, 16
DECODE_SUB_MIN, DECODE_SUB_DEFAULT = 32, 512


def _placeholder(shape):
    """An int16 array of this shape that costs no memory (all elements alias one zero)."""
    return np.broadcast_to(np.zeros((), dtype=np.int16), shape)


def _parse(data: bytes):
    lib = load()
    data = bytes(data)
    ci, sc = _Image(), _Scan()
    rc = lib.jpegqs_cuda_jpeg_parse(data, len(data), C.byref(ci), C.byref(sc))
    if rc not in (0, -3):
        raise QsError(f"parse_jpeg: {lib.jpegqs_cuda_last_error(None).decode()}")
    comps = []
    for c in range(ci.ncomp):
        cc = ci.comp[c]
        q = np.array(list(cc.quant), dtype=np.uint16) if cc.has_qtbl else None
        comps.append(Component(coef=_placeholder((cc.hblk, cc.wblk, 64)), quant=q, h_samp=cc.h_samp,
                               v_samp=cc.v_samp, quant_tbl_no=min(c, 1)))
    image = CoefImage(width=ci.image_width, height=ci.image_height, colorspace=int(sc.jpeg_color_space), comps=comps)
    return image, (sc if rc == 0 else None), sc


def parse_jpeg(data: bytes):
    """The header of a JPEG file, host-only: (CoefImage, scan).  The CoefImage carries the geometry,
    sampling, quant tables and colour space; its arrays are placeholders of the right shape that
    cost no memory.  scan (a jpegqs_cuda_scan) is what decode_async needs, or None when only
    read_jpeg takes the file (progressive, several scans).  Raises QsError for what the reader
    rejects (truncated headers, lossless / arithmetic / 12-bit files)."""
    image, scan, _ = _parse(data)
    return image, scan


def read_jpeg(data: bytes) -> CoefImage:
    """Host decode of any file the jpegqs tool reads, with its reader: the quantized coefficients
    jpeg_read_coefficients gives, as numpy int16 [hblk, wblk, 64] arrays."""
    lib = load()
    data = bytes(data)
    image, _, _ = _parse(data)
    ci = _Image()
    arrays = [np.zeros((c.hblk, c.wblk, 64), dtype=np.int16) for c in image.comps]
    for c, a in zip(image.comps, arrays):
        c.coef = a
    _fill_image(ci, image, [a.ctypes.data for a in arrays], [])
    rc = lib.jpegqs_cuda_jpeg_read(data, len(data), C.byref(ci))
    if rc < 0:
        raise QsError(f"read_jpeg: {lib.jpegqs_cuda_last_error(None).decode()}")
    return image


def decode_workspace_bytes(images: Sequence[CoefImage], scans, data_len: Sequence[int]) -> int:
    """Device bytes of workspace decode_async needs (host-only)."""
    lib = load()
    n = len(images)
    arr = _image_array(images)
    sc = (_Scan * max(n, 1))(*scans)
    lens = (C.c_size_t * max(n, 1))(*[int(x) for x in data_len])
    out = C.c_size_t(0)
    if lib.jpegqs_cuda_decode_workspace_bytes(n, arr, sc, lens, C.byref(out)) < 0:
        raise QsError(lib.jpegqs_cuda_last_error(None).decode())
    return int(out.value)


# Pillow's output modes (include/jpegqs_cuda.h JPEGQS_PIXELS_*): None keeps the file's own colour
_MODES = {None: 0, "RGB": 1, "L": 2}


def _mode(mode, who: str) -> int:
    if not isinstance(mode, (str, type(None))) or mode not in _MODES:
        raise ValueError(f"{who}: mode {mode!r}: expected None, 'RGB' or 'L'")
    return _MODES[mode]


def _mode_channels(ncomp: int, mode: int) -> int:
    """the output channels of an ncomp-component file in mode (0: the file's own, 3 for colour)"""
    return (1 if ncomp == 1 else 3) if mode == 0 else 3 if mode == 1 else 1


def render_model(image: CoefImage, upsampled=False, layout: str = "hwc", scale_denom: int = 1, mode=None):
    """render_async's algorithm on one CPU thread for one image (jpegqs_cuda_render_model): libjpeg's
    islow / reduced IDCTs, up-sampling and colour conversion at scale 1/scale_denom.  upsampled: None /
    False reads the image's own arrays; otherwise a pair of int16 numpy arrays [hblk, wblk, 64] at
    component 0's geometry, read for components 1 and 2.  Returns a uint8 numpy array [H, W, 3] ("hwc")
    or [3, H, W] ("chw"), H = ceil(height / d) and W = ceil(width / d).
    mode: None, or Pillow's "RGB" / "L" of the picture (jpegqs_cuda_render_model_mode), for any component
    count 1, 3 or 4, with image.colorspace deciding the conversion; the output then has 3 or 1 channels."""
    if layout not in ("hwc", "chw"):
        raise ValueError(f"render_model: layout {layout!r}: expected 'hwc' or 'chw'")
    d = _scale_denom(scale_denom, "render_model")
    m = _mode(mode, "render_model")
    lib = load()
    arrays = [np.ascontiguousarray(c.coef, dtype=np.int16) for c in image.comps]
    for c, a in zip(image.comps, arrays):
        if a.shape != (c.hblk, c.wblk, 64):
            raise ValueError(f"render_model: a coefficient array of shape {a.shape}, expected {(c.hblk, c.wblk, 64)}")
    ups = []
    if upsampled is not None and upsampled is not False:
        if len(upsampled) != 2 or len(image.comps) != 3:
            raise ValueError("render_model: upsampled must be two arrays for a three-component image")
        y = image.comps[0]
        ups = [np.ascontiguousarray(u, dtype=np.int16) for u in upsampled]
        if any(u.shape != (y.hblk, y.wblk, 64) for u in ups):
            raise ValueError(f"render_model: up-sampled arrays must have component 0's shape {(y.hblk, y.wblk, 64)}")
    ci = _Image()
    _fill_image(ci, image, [a.ctypes.data for a in arrays], [None] + [u.ctypes.data for u in ups] if ups else [])
    out = np.zeros(_scaled_shape(image.width, image.height, 3 if m < 2 else 1, layout, d), dtype=np.uint8)
    if m:
        rc = lib.jpegqs_cuda_render_model_mode(C.byref(ci), int(image.colorspace), int(bool(ups)),
                                               0 if layout == "hwc" else 1, d, m, out.ctypes.data)
    else:
        rc = lib.jpegqs_cuda_render_model(C.byref(ci), int(bool(ups)), 0 if layout == "hwc" else 1, d, out.ctypes.data)
    if rc < 0:
        raise QsError(f"render_model: {lib.jpegqs_cuda_last_error(None).decode()} ({rc})")
    return out


def resize_model(pixels, size, crop=None, filter="bicubic", layout: str = "hwc"):
    """The device resize on one CPU thread (jpegqs_cuda_resize_model): byte for byte Pillow's
    Image.fromarray(pixels).crop(crop).resize(size, filter).  pixels: uint8 [H, W] (grey, 'L') or
    [H, W, C] with C 1 or 3, as decode_pixels gives them in layout "hwc".  size (width, height) and
    crop (left, top, right, bottom) or None follow Pillow's conventions; filter as decode_pixels'.
    Returns [height, width] for a 2-D input, else [height, width, C] ("hwc") or [C, height, width]
    ("chw").  ValueError for a bad argument."""
    if layout not in ("hwc", "chw"):
        raise ValueError(f"resize_model: layout {layout!r}: expected 'hwc' or 'chw'")
    a = np.asarray(pixels)
    if a.dtype != np.uint8 or a.ndim not in (2, 3) or (a.ndim == 3 and a.shape[2] not in (1, 3)) or 0 in a.shape:
        raise ValueError(f"resize_model: pixels must be uint8 [H, W] or [H, W, 1|3], not {a.dtype} {a.shape}")
    a = np.ascontiguousarray(a)
    fcode = _resize_filter(filter, "resize_model")
    if size is None:
        raise ValueError("resize_model: size (width, height) is required")
    sizes, crops = _resize_boxes(1, size, None if crop is None else [crop], "resize_model")
    h, w = a.shape[:2]
    c = 1 if a.ndim == 2 else a.shape[2]
    box = _resize_box(w, h, sizes[0], crops[0], 0, "resize_model")
    shape = (box.height, box.width, c) if layout == "hwc" else (c, box.height, box.width)
    out = np.zeros(shape, dtype=np.uint8)
    lib = load()
    rc = lib.jpegqs_cuda_resize_model(a.ctypes.data, w, h, c, 0 if layout == "hwc" else 1, fcode, C.byref(box),
                                      out.ctypes.data)
    if rc < 0:
        raise ValueError(f"resize_model: {lib.jpegqs_cuda_last_error(None).decode()} ({rc})")
    return out.reshape(box.height, box.width) if a.ndim == 2 else out


def decode_model(image: CoefImage, scan, data: bytes, sub_bytes: int = DECODE_SUB_DEFAULT, out=None):
    """decode_async's algorithm run on the CPU for one file (jpegqs_cuda_decode_model).  out: numpy
    int16 arrays to write (default: new ones).  Returns (arrays, status, overrun), overrun the units
    the synchronisation decoded past each subsequence's end."""
    lib = load()
    data = bytes(data)
    if out is None:
        out = [np.zeros((c.hblk, c.wblk, 64), dtype=np.int16) for c in image.comps]
    ci = _Image()
    _fill_image(ci, image, [a.ctypes.data for a in out], [])
    cap = len(data) // DECODE_SUB_MIN + 1 + (image.comps[0].wblk * image.comps[0].hblk if scan.restart_interval else 1)
    over = np.zeros(cap, dtype=np.uint32)
    st, nsub = C.c_int32(0), C.c_size_t(0)
    if lib.jpegqs_cuda_decode_model(C.byref(ci), C.byref(scan), data, len(data), sub_bytes, C.byref(st),
                                    over.ctypes.data, cap, C.byref(nsub)) < 0:
        raise QsError(lib.jpegqs_cuda_last_error(None).decode())
    return out, int(st.value), over[:nsub.value]


def parse_jpeg_scans(data: bytes):
    """Every marker of a JPEG file, host-only, no entropy-coded data decoded: (CoefImage, scans).  The
    CoefImage is parse_jpeg's (placeholder arrays); scans is a ScanList of jpegqs_cuda_scan_rec, one per
    scan, what decode_scans_async needs, or None when only read_jpeg takes the file (more than 64 scans,
    tables libjpeg would reject, first scans after an overlapping refinement).  Raises QsError for
    what the reader rejects."""
    lib = load()
    data = bytes(data)
    image, _, _ = _parse(data)
    ci, recs, n = _Image(), (_ScanRec * MAX_SCANS)(), C.c_int(0)
    rc = lib.jpegqs_cuda_jpeg_parse_scans(data, len(data), C.byref(ci), recs, MAX_SCANS, C.byref(n))
    if rc not in (0, -3):
        raise QsError(f"parse_jpeg_scans: {lib.jpegqs_cuda_last_error(None).decode()}")
    return image, (ScanList(recs[:n.value]) if rc == 0 else None)


def exif_orientation(data: bytes) -> int:
    """The EXIF orientation 1..8 of a JPEG file (jpegqs_cuda_jpeg_orientation): the transform
    ImageOps.exif_transpose(Image.open(f)) applies, 1 for none.  QsError for a file the reader rejects."""
    lib = load()
    d = _file_bytes(data, "exif_orientation")
    o = C.c_int32()
    if lib.jpegqs_cuda_jpeg_orientation(d, len(d), C.byref(o)) < 0:
        raise QsError(f"exif_orientation: {lib.jpegqs_cuda_last_error(None).decode()}")
    return o.value


def _orient_int(v):
    return None if isinstance(v, bool) or not isinstance(v, (int, np.integer)) else int(v)


def _orientations(orientation, n: int, who: str, lo: int = 0):
    """None, or one value per file: "exif" gives 0 (the file's own) for every file, an int 1..8 that value
    for every file, a sequence one value lo..8 per file; ValueError otherwise"""
    if orientation is None:
        return None
    if isinstance(orientation, str):
        if orientation != "exif":
            raise ValueError(f"{who}: orientation {orientation!r}: expected 'exif', 1..8 or one value per file")
        return [0] * n
    v = _orient_int(orientation)
    if v is not None:
        if not 1 <= v <= 8:
            raise ValueError(f"{who}: orientation {v}: expected 1..8")
        return [v] * n
    if isinstance(orientation, (bytes, bytearray)) or not hasattr(orientation, "__len__") or len(orientation) != n:
        raise ValueError(f"{who}: orientation: expected 'exif', 1..8 or a sequence of {n} values")
    out = []
    for i, x in enumerate(orientation):
        v = _orient_int(x)
        if v is None or not lo <= v <= 8:
            raise ValueError(f"{who}: orientation[{i}] {x!r}: expected an int {lo}..8")
        out.append(v)
    return out


def _oriented_shape(shape, o: int, layout: str):
    """an unoriented picture's shape as orientation o gives it (5..8 swap width and height)"""
    if o < 5:
        return shape
    return (shape[1], shape[0], shape[2]) if layout == "hwc" else (shape[0], shape[2], shape[1])


def _file_bytes(data, what: str) -> bytes:
    if not isinstance(data, (bytes, bytearray, memoryview)):
        raise TypeError(f"{what}: data must be bytes-like, not {type(data).__name__}")
    return bytes(data)


def transcode_route(data: bytes):
    """Where the jpegqs tool transcodes this file, host-only: ("device", reason) or ("host", reason).
    The rule of jpegqs_cuda_transcode_route (include/jpegqs_cuda.h): the device when the whole file
    walks without a marker-level warning, one of the device decoders takes it, it is not a progressive
    file with an AC refinement scan without restart markers, and the encoder takes its geometry.
    Raises TypeError for data that is not bytes-like and QsError for a file the reader rejects."""
    lib = load()
    data = _file_bytes(data, "transcode_route")
    why = C.c_char_p()
    rc = lib.jpegqs_cuda_transcode_route(data, len(data), C.byref(why), None)
    reason = (why.value or b"").decode()
    if rc < 0:
        raise QsError(f"transcode_route: {reason}")
    return ("device" if rc == ROUTE_DEVICE else "host"), reason


class ScanList(list):
    """The jpegqs_cuda_scan_rec records of one file, in file order (parse_jpeg_scans)."""

    def array(self):
        return (_ScanRec * max(len(self), 1))(*self)


def _scan_arrays(scans):
    arrs = [s.array() for s in scans]
    ptrs = (C.c_void_p * max(len(arrs), 1))(*[C.addressof(a) for a in arrs])
    counts = (C.c_int * max(len(arrs), 1))(*[len(s) for s in scans])
    return arrs, ptrs, counts


def decode_scans_workspace_bytes(images: Sequence[CoefImage], scans, data_len: Sequence[int]) -> int:
    """Device bytes of workspace decode_scans_async needs (host-only)."""
    lib = load()
    n = len(images)
    arr = _image_array(images)
    keep, ptrs, counts = _scan_arrays(scans)
    lens = (C.c_size_t * max(n, 1))(*[int(x) for x in data_len])
    out = C.c_size_t(0)
    if lib.jpegqs_cuda_decode_scans_workspace_bytes(n, arr, ptrs, counts, lens, C.byref(out)) < 0:
        raise QsError(lib.jpegqs_cuda_last_error(None).decode())
    return int(out.value)


def decode_scans_model(image: CoefImage, scans, data: bytes, sub_bytes: int = DECODE_SUB_DEFAULT, out=None):
    """decode_scans_async's algorithm run on one CPU thread for one file (jpegqs_cuda_decode_scans_model).
    out: numpy int16 arrays to write (default: new ones).  Returns (arrays, status)."""
    lib = load()
    data = bytes(data)
    if out is None:
        out = [np.zeros((c.hblk, c.wblk, 64), dtype=np.int16) for c in image.comps]
    ci = _Image()
    _fill_image(ci, image, [a.ctypes.data for a in out], [])
    st = C.c_int32(0)
    recs = ScanList(scans).array()
    if lib.jpegqs_cuda_decode_scans_model(C.byref(ci), recs, len(scans), data, len(data), sub_bytes, C.byref(st)) < 0:
        raise QsError(lib.jpegqs_cuda_last_error(None).decode())
    return out, int(st.value)


# ---- coefficients to JPEG files (include/jpegqs_cuda.h "quantized coefficients to JPEG files") ----
ENCODE_RANGE, ENCODE_OVERFLOW, ENCODE_NO_UP = 1, 2, 4


def jpeg_prefix(data: bytes, copy: int = 2):
    """What the jpegqs tool's writer puts before its first DQT for this input file and marker copy
    level (the tool's -c): SOI, the JFIF APP0 or Adobe APP14, the copied APPn / COM markers.  Host-only,
    no entropy-coded data is decoded.  Returns (prefix bytes, component ids, quantization table
    numbers), one id and one table number per component: the frame identifiers encode_async writes in
    SOF / SOS and DQT, which a CoefImage does not carry."""
    lib = load()
    data = bytes(data)
    ids, tbls, n, nc = (C.c_int32 * 4)(), (C.c_int32 * 4)(), C.c_size_t(0), C.c_int32(0)
    if lib.jpegqs_cuda_jpeg_prefix(data, len(data), copy, None, 0, C.byref(n), C.byref(nc), ids, tbls) < 0:
        raise QsError(f"jpeg_prefix: {lib.jpegqs_cuda_last_error(None).decode()}")
    buf = (C.c_uint8 * max(n.value, 1))()
    if lib.jpegqs_cuda_jpeg_prefix(data, len(data), copy, buf, n.value, C.byref(n), C.byref(nc), ids, tbls) < 0:
        raise QsError(f"jpeg_prefix: {lib.jpegqs_cuda_last_error(None).decode()}")
    return bytes(buf)[:n.value], tuple(ids[:nc.value]), tuple(tbls[:nc.value])


def _head(prefix_ptr, prefix_len, comp_ids, quant_tbls, n):
    h = _Head()
    if len(comp_ids) != n or len(quant_tbls) != n:
        raise ValueError(f"expected {n} component ids and quantization table numbers")
    h.prefix_dev, h.prefix_len = prefix_ptr, prefix_len
    for k in range(n):
        h.comp_id[k], h.quant_tbl[k] = int(comp_ids[k]), int(quant_tbls[k])
    return h


def encode_bound(image: CoefImage, prefix_len: int) -> int:
    """Output bytes encode_async can never exceed for this image and prefix length (host-only)."""
    lib = load()
    ci, out = _Image(), C.c_size_t(0)
    _fill_image(ci, image, [None] * len(image.comps), [])
    if lib.jpegqs_cuda_encode_bound(C.byref(ci), int(prefix_len), C.byref(out)) < 0:
        raise QsError(lib.jpegqs_cuda_last_error(None).decode())
    return int(out.value)


def encode_workspace_bytes(images: Sequence[CoefImage], optimize: bool = False) -> int:
    """Device bytes of workspace encode_async needs for these images (host-only)."""
    lib = load()
    arr, out = _image_array(images), C.c_size_t(0)
    if lib.jpegqs_cuda_encode_workspace_bytes(len(images), arr, int(bool(optimize)), C.byref(out)) < 0:
        raise QsError(lib.jpegqs_cuda_last_error(None).decode())
    return int(out.value)


def encode_model(image: CoefImage, arrays, prefix: bytes, comp_ids, quant_tbls, optimize: bool = False, up=None,
                 capacity=None):
    """encode_async's algorithm run on the CPU for one image (jpegqs_cuda_encode_model).  arrays: numpy
    int16 [hblk, wblk, 64] per component; up: the two luma-sized arrays of up-sampled chroma, which
    makes the model write the up-sampled geometry.  capacity: output bytes (default encode_bound).
    Returns (file bytes, status).  On OVERFLOW the bytes are the first `capacity` bytes of the
    file, which is not complete."""
    lib = load()
    nc = len(image.comps)
    if len(arrays) != nc:
        raise ValueError(f"{len(arrays)} arrays for {nc} components")
    arrays = [np.ascontiguousarray(a, dtype=np.int16) for a in arrays]
    for c, (comp, a) in enumerate(zip(image.comps, arrays)):
        if a.shape != (comp.hblk, comp.wblk, 64):
            raise ValueError(f"arrays[{c}]: shape {a.shape}, expected {(comp.hblk, comp.wblk, 64)}")
    ups = [None, None]
    if up is not None:
        y = image.comps[0]
        ups = [np.ascontiguousarray(a, dtype=np.int16) for a in up]
        for a in ups:
            if a.shape != (y.hblk, y.wblk, 64):
                raise ValueError(f"up: shape {a.shape}, expected {(y.hblk, y.wblk, 64)}")
    ci = _Image()
    _fill_image(ci, image, [a.ctypes.data for a in arrays], [None] + [a.ctypes.data if a is not None else None for a in ups])
    ci.upsampled = int(up is not None)
    prefix = bytes(prefix)
    pbuf = (C.c_uint8 * max(len(prefix), 1)).from_buffer_copy(prefix or b"\0")
    head = _head(C.cast(pbuf, C.c_void_p), len(prefix), comp_ids, quant_tbls, nc)
    cap = int(capacity) if capacity is not None else encode_bound(image, len(prefix))
    out = np.zeros(max(cap, 1), dtype=np.uint8)
    n, st = C.c_uint64(0), C.c_int32(0)
    if lib.jpegqs_cuda_encode_model(C.byref(ci), C.byref(head), int(bool(optimize)), out.ctypes.data, cap,
                                    C.byref(n), C.byref(st)) < 0:
        raise QsError(lib.jpegqs_cuda_last_error(None).decode())
    return out[:min(n.value, cap)].tobytes(), int(st.value)


# ---- pictures to JPEG files (include/jpegqs_cuda.h "8-bit pictures -> JPEG files") ----
SUBSAMPLINGS = {"4:4:4": 0, "4:2:2": 1, "4:2:0": 2}
JPEG_PROGRESSIVE = 0x100       # JPEGQS_JPEG_PROGRESSIVE: ORed into jpegqs_cuda_jpeg_params.optimize


def _jpeg_params(quality, subsampling, optimize, who: str, progressive=False) -> _JpegParams:
    """Pillow's save keywords: quality 1..100; subsampling "4:4:4" / "4:2:2" / "4:2:0" or 0 / 1 / 2;
    progressive a bool (JPEGQS_JPEG_PROGRESSIVE ORed into optimize)"""
    if isinstance(quality, bool) or not isinstance(quality, (int, np.integer)) or not 1 <= int(quality) <= 100:
        raise ValueError(f"{who}: quality {quality!r}: expected an integer in 1..100")
    if isinstance(subsampling, str) and subsampling in SUBSAMPLINGS:
        s = SUBSAMPLINGS[subsampling]
    elif not isinstance(subsampling, (str, bool)) and isinstance(subsampling, (int, np.integer)) and int(subsampling) in (0, 1, 2):
        s = int(subsampling)
    else:
        raise ValueError(f"{who}: subsampling {subsampling!r}: expected '4:4:4', '4:2:2', '4:2:0' or 0, 1, 2")
    if not isinstance(progressive, (bool, np.bool_)):
        raise ValueError(f"{who}: progressive {progressive!r}: expected True or False")
    return _JpegParams(int(quality), s, int(bool(optimize)) | (JPEG_PROGRESSIVE if progressive else 0))


def _pixels_in(ptr, shape, row_bytes) -> _PixelsIn:
    h, w, c = shape
    return _PixelsIn(ptr, int(w), int(h), int(c), int(row_bytes))


def _host_picture(pixels, who: str) -> np.ndarray:
    a = np.asarray(pixels.cpu() if hasattr(pixels, "cpu") else pixels)
    if a.dtype != np.uint8:
        raise ValueError(f"{who}: dtype {a.dtype}, expected uint8")
    if a.ndim == 2:
        a = a[:, :, None]
    if a.ndim != 3 or a.shape[2] not in (1, 3):
        raise ValueError(f"{who}: shape {a.shape}, expected [H, W, 1] or [H, W, 3]")
    return np.ascontiguousarray(a)


def compress_bound(shape, quality=75, subsampling="4:2:0", optimize=False, progressive=False) -> int:
    """Output bytes compress_async never exceeds for an [H, W, C] picture (host-only)."""
    lib = load()
    pin, out = _pixels_in(None, shape, int(shape[1]) * int(shape[2])), C.c_size_t(0)
    jp = _jpeg_params(quality, subsampling, optimize, "compress_bound", progressive)
    if lib.jpegqs_cuda_compress_bound(C.byref(pin), C.byref(jp), C.byref(out)) < 0:
        raise QsError(lib.jpegqs_cuda_last_error(None).decode())
    return int(out.value)


def compress_model(pixels, quality=75, subsampling="4:2:0", optimize=False, capacity=None, progressive=False) -> bytes:
    """compress_async's algorithm on one CPU thread for one picture (jpegqs_cuda_compress_model): a uint8
    array [H, W, 3] (RGB), [H, W, 1] or [H, W] (grey) to the bytes of Pillow's
    Image.fromarray(P).save(f, "JPEG", quality=quality, subsampling=subsampling, optimize=optimize,
    progressive=progressive).  capacity: output bytes (default compress_bound); a file that does not fit
    raises QsError."""
    lib = load()
    a = _host_picture(pixels, "compress_model")
    jp = _jpeg_params(quality, subsampling, optimize, "compress_model", progressive)
    cap = int(capacity) if capacity is not None else compress_bound(a.shape, quality, subsampling, optimize, progressive)
    out = np.zeros(max(cap, 1), dtype=np.uint8)
    pin = _pixels_in(a.ctypes.data, a.shape, a.shape[1] * a.shape[2])
    n, st = C.c_uint64(0), C.c_int32(0)
    if lib.jpegqs_cuda_compress_model(C.byref(pin), C.byref(jp), out.ctypes.data, cap, C.byref(n), C.byref(st)) < 0:
        raise QsError(lib.jpegqs_cuda_last_error(None).decode())
    if st.value:
        raise QsError(f"compress_model: encoder status {st.value}, {n.value} bytes needed of {cap}")
    return out[:n.value].tobytes()


def _stream_handle(stream) -> C.c_void_p:
    """The cudaStream_t to pass for a torch.cuda.Stream.  torch's default stream is the legacy
    stream, handle 0; the library reads NULL as the context's own stream, which is not ordered with
    it, so the legacy stream goes in as cudaStreamLegacy (1)."""
    return C.c_void_p(stream.cuda_stream or 1)


def _check_tensor(t, shape, what: str):
    import torch
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{what}: expected a torch.Tensor, got {type(t).__name__}")
    if t.dtype != torch.int16:
        raise TypeError(f"{what}: dtype {t.dtype}, expected torch.int16")
    if tuple(t.shape) != tuple(shape):
        raise ValueError(f"{what}: shape {tuple(t.shape)}, expected {tuple(shape)}")
    if not t.is_contiguous():
        raise ValueError(f"{what}: not contiguous")


class QsContext:
    """One device context (stream, tables, scratch arena).  Mirrors the process-wide state
    the reference keeps implicitly (its tables are rebuilt per call, quantsmooth.h:2460-2464)."""

    def __init__(self, device: int = -1):
        self.lib = load()
        h = C.c_void_p()
        rc = self.lib.jpegqs_cuda_create(device, C.byref(h))
        if rc:
            raise QsError(f"jpegqs_cuda_create failed ({rc}): "
                          f"{self.lib.jpegqs_cuda_last_error(None).decode()}")
        self.h = h
        self.device = device

    def close(self):
        if getattr(self, "h", None):
            self.lib.jpegqs_cuda_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc < 0:
            raise QsError(f"CUDA back end error {rc}: {self.lib.jpegqs_cuda_last_error(self.h).decode()}")
        return rc

    @property
    def device_name(self) -> str:
        return self.lib.jpegqs_cuda_device_name(self.h).decode()

    @property
    def last_device_ms(self) -> float:
        return float(self.lib.jpegqs_cuda_last_device_ms(self.h))

    @property
    def last_launches(self) -> int:
        return int(self.lib.jpegqs_cuda_last_launches(self.h))

    def set_profiling(self, on: bool):
        self.lib.jpegqs_cuda_set_profiling(self.h, int(on))

    def set_tuning(self, key: int, value: int):
        self._check(self.lib.jpegqs_cuda_set_tuning(self.h, key, value))

    def kernel_stats(self):
        """(idct_ms, idct_launches, smooth_ms, smooth_launches) of the last run_* call."""
        a, b, c, d = C.c_float(), C.c_int(), C.c_float(), C.c_int()
        self.lib.jpegqs_cuda_kernel_stats(self.h, C.byref(a), C.byref(b), C.byref(c), C.byref(d))
        return a.value, b.value, c.value, d.value

    def transcode(self, data: bytes, flags: int, niter: int, optimize: bool = False, copy: int = 2):
        """One JPEG file to the file the jpegqs tool writes for it (read, do_quantsmooth(flags, niter),
        write with -o optimize and -c copy), decoded, smoothed and encoded on this context's device
        (jpegqs_cuda_transcode).  Returns (bytes, None), or (None, reason) when the file must take the
        host route: transcode_route says so, the device decoder flagged damaged data or the encoder met
        a coefficient it cannot code.  Device buffers stay with the context and only grow."""
        data = _file_bytes(data, "transcode")
        res = _TranscodeResult()
        rc = self._check(self.lib.jpegqs_cuda_transcode(self.h, data, len(data), int(flags), int(niter), int(bool(optimize)),
                                                        int(copy), C.byref(res)))
        if rc == TRANSCODE_FALLBACK:
            return None, (res.reason or b"").decode()
        try:
            return C.string_at(res.data, res.len), None
        finally:
            self.lib.jpegqs_cuda_transcode_free(res.data)

    def transcode_batch(self, datas, flags: int, niter: int, optimize: bool = False, copy: int = 2,
                        max_device_bytes: int = 0):
        """Many JPEG files, each to what transcode gives for it alone, in shared launches
        (jpegqs_cuda_transcode_batch): a list of (bytes, None) or (None, reason), in the order of datas.
        max_device_bytes bounds the device memory of one sub-batch (0: half of what is free plus what
        the context already holds).  Raises QsError naming the index of a file the reader rejects,
        ValueError for copy outside 0..2 or a negative max_device_bytes, TypeError for a non-bytes entry."""
        if isinstance(datas, (bytes, bytearray, memoryview, str)) or not hasattr(datas, "__len__"):
            raise TypeError("transcode_batch: datas must be a sequence of bytes-like files")
        files = [_file_bytes(d, f"transcode_batch: file {i}") for i, d in enumerate(datas)]
        if int(copy) not in (0, 1, 2):
            raise ValueError(f"transcode_batch: copy must be 0, 1 or 2, not {copy}")
        if int(max_device_bytes) < 0:
            raise ValueError("transcode_batch: max_device_bytes must be >= 0")
        n = len(files)
        if not n:
            return []
        ptrs = (C.c_char_p * n)(*files)
        lens = (C.c_size_t * n)(*[len(d) for d in files])
        rc = (C.c_int * n)()
        res = (_TranscodeResult * n)()
        self._check(self.lib.jpegqs_cuda_transcode_batch(self.h, n, ptrs, lens, int(flags), int(niter), int(bool(optimize)),
                                                         int(copy), int(max_device_bytes), rc, res))
        out, bad = [], None
        for i in range(n):
            if rc[i] == TRANSCODE_OK:
                out.append((C.string_at(res[i].data, res[i].len), None))
                self.lib.jpegqs_cuda_transcode_free(res[i].data)
            elif rc[i] == TRANSCODE_FALLBACK:
                out.append((None, (res[i].reason or b"").decode()))
            elif bad is None:
                bad = i
        if bad is not None:
            raise QsError(f"transcode_batch: file {bad}: {self.lib.jpegqs_cuda_last_error(self.h).decode()}")
        return out

    def decode_pixels(self, datas, flags: int, niter: int, layout: str = "hwc", device: str = "cuda",
                      max_device_bytes: int = 0, scale_denom: int = 1, size=None, crop=None, filter="bicubic",
                      orientation=None, mode=None, thumbnail=None, reducing_gap=_GAP_DEFAULT, image_filter=None):
        """Many JPEG files to the smoothed pixels the jpegqs tool's --ppm writes for them (islow, fancy
        up-sampling, after do_quantsmooth(flags, niter)), in shared launches (jpegqs_cuda_pixels_batch).
        Returns, in the order of datas, one record per file:
            (pixels, warnings, host_decoded, smoothed, stop, upsampled, reason)
        pixels is a uint8 tensor [H, W, C] for layout "hwc" or [C, H, W] for "chw", C = 1 for a grey
        file and 3 for a colour one; on cuda:<this context's device> for device="cuda", a CPU tensor for
        device="cpu".  warnings: the host reader's warning count (0 for a file the device decoded);
        host_decoded / reason: whether and why the host reader decoded the file.  Raises TypeError for a
        non-bytes entry or a bare bytes object, ValueError for an unknown layout or device or a negative
        max_device_bytes, and QsError naming the index of a file the reader rejects or the render
        cannot take (1 or 3 components, integral sampling ratios).
        scale_denom 2, 4 or 8: libjpeg's scaled decode of the same coefficients at 1/d size
        (jpegqs_cuda_pixels_batch_scaled); pixels are then [ceil(H/d), ceil(W/d), C] or
        [C, ceil(H/d), ceil(W/d)].  ValueError for any other value than 1, 2, 4 or 8.
        size / crop / filter: each file's pixels cropped and resized on the device, byte for byte
        Pillow's Image.fromarray(P).crop(crop).resize(size, filter) of the picture P the call gives
        without them (jpegqs_cuda_pixels_batch_resized).  The conventions are Pillow's, not torch's:
        size is (width, height), for every file or a list with one per file; crop is None or a list
        with one (left, top, right, bottom) box or None per file, in the 1/scale_denom picture.  filter
        is "bicubic" (Image.resize's default), "bilinear", "lanczos", "box" or "hamming", or Pillow's
        Image.Resampling value of one of them; NEAREST is not supported.  A crop without size returns
        the crop as it is.  Pixels are then [height, width, C] or [C, height, width].  ValueError
        naming the file index for a bad size, crop or filter, before anything runs.
        orientation: None (the pixels in the order the file stores them), "exif" (each file's own EXIF
        orientation, as Pillow's ImageOps.exif_transpose applies it), one int 1..8 for every file, or a
        sequence of ints 0..8, one per file, 0 meaning the file's own (jpegqs_cuda_pixels_batch_oriented).
        The picture is turned before the crop and the resize, so crop is in the oriented picture, and for
        5..8 the unresized pixels have width and height swapped.  ValueError for a bad value or length.
        mode: None (the file's own colour, as above), "RGB" or "L": Pillow's Image.convert(mode) of each
        file's picture, before the crop and the resize, so C is 3 or 1 for every file, and CMYK and YCCK
        files are decoded too (jpegqs_cuda_pixels_batch_mode).  ValueError for any other value.
        thumbnail: (width, height), or one per file: Pillow's Image.open(F) [exif_transpose] [convert(mode)]
        .thumbnail(bound, filter, reducing_gap) of the file F jpegqs writes (jpegqs_cuda_pixels_batch_reduced):
        each file is decoded at its own draft scale, reduced and resized as Pillow does; pixels are
        thumbnail_geometry's size.  An orientation (any value, 1 included) or a mode loads the picture
        first, as exif_transpose and convert do, so there is no draft.  reducing_gap: Pillow's, default 2.0 with thumbnail and None with size
        (an explicit None is None in both); with size, Image.resize(size, filter, reducing_gap=) of the
        crop.  ValueError naming the file for a bad bound, for thumbnail with size, crop or scale_denom
        other than 1, or for a reducing_gap below 1.0, before anything runs.
        image_filter: None, one of Pillow's ImageFilter.GaussianBlur, BoxBlur or UnsharpMask (an instance, or
        the class for Pillow's defaults), or a sequence of them: each file's picture as above, then
        .filter(F1).filter(F2)... on the device (jpegqs_cuda_pixels_batch_filtered), the last stage.  None
        and [] are the call without it.  ValueError naming any other filter, a negative BoxBlur radius, a
        radius above FILTER_MAX_RADIUS or a percent above FILTER_MAX_PERCENT in magnitude, or a non-int
        percent or threshold, before anything runs."""
        if isinstance(datas, (bytes, bytearray, memoryview, str)) or not hasattr(datas, "__len__"):
            raise TypeError("decode_pixels: datas must be a sequence of bytes-like files")
        files = [_file_bytes(d, f"decode_pixels: file {i}") for i, d in enumerate(datas)]
        if layout not in ("hwc", "chw"):
            raise ValueError(f"decode_pixels: layout {layout!r}: expected 'hwc' or 'chw'")
        if device not in ("cuda", "cpu"):
            raise ValueError(f"decode_pixels: device {device!r}: expected 'cuda' or 'cpu'")
        if int(max_device_bytes) < 0:
            raise ValueError("decode_pixels: max_device_bytes must be >= 0")
        scale = _scale_denom(scale_denom, "decode_pixels")
        n = len(files)
        resize = size is not None or crop is not None
        if resize:
            fcode = _resize_filter(filter, "decode_pixels")
            sizes, crops = _resize_boxes(n, size, crop, "decode_pixels")
        orient = _orientations(orientation, n, "decode_pixels")
        m = _mode(mode, "decode_pixels")
        bounds = self._thumbnail_args(n, thumbnail, resize, scale, "decode_pixels")
        # reducing_gap acts only in a resize
        gap = _reducing_gap(reducing_gap, bounds is not None, "decode_pixels") if resize or bounds is not None else 0.0
        if bounds is not None:
            fcode = _resize_filter(filter, "decode_pixels")
        filt = _image_filters(image_filter, "decode_pixels")
        if not n:
            return []
        # the output size rule of jpegqs_cuda_pixels_batch: transcode_route's width, height and ncomp
        shapes = []
        for i, d in enumerate(files):
            info = _FileInfo()
            if self.lib.jpegqs_cuda_transcode_route(d, len(d), None, C.byref(info)) < 0:
                raise QsError(f"decode_pixels: file {i}: the reader rejects the file")
            if info.ncomp not in ((1, 3) if not m else (1, 3, 4)):
                raise QsError(f"decode_pixels: file {i}: {info.ncomp} components; the render takes "
                              + ("1, 3 or 4" if m else "1 or 3 (4 with a mode)"))
            c, h, w = _mode_channels(info.ncomp, m), info.image_height, info.image_width
            shapes.append(_scaled_shape(w, h, c, layout, scale))
        if orient is not None:
            orient = [exif_orientation(d) if o == 0 else o for d, o in zip(files, orient)]
            shapes = [_oriented_shape(s, o, layout) for s, o in zip(shapes, orient)]
        if bounds is not None:
            boxes = self._thumbnail_boxes(shapes, bounds, layout, gap, orient is not None or m != 0)
            shapes = [s for s, _ in boxes]
            boxes = (_ResizeBox * n)(*[b for _, b in boxes])
        elif resize:
            boxes = (_ResizeBox * n)()
            for i, s in enumerate(shapes):
                ph, pw = (s[0], s[1]) if layout == "hwc" else (s[1], s[2])
                boxes[i] = _resize_box(pw, ph, sizes[i], crops[i], i, "decode_pixels")
                c = 1 if s[2 if layout == "hwc" else 0] == 1 else 3
                shapes[i] = (boxes[i].height, boxes[i].width, c) if layout == "hwc" else (c, boxes[i].height, boxes[i].width)
        import torch
        if device == "cuda":
            dev = self.device if self.device >= 0 else torch.cuda.current_device()
            outs = [torch.empty(s, dtype=torch.uint8, device=dev) for s in shapes]
            # the call writes on the context's stream: the memory must be free on the current one
            torch.cuda.current_stream(dev).synchronize()
        else:
            outs = [torch.empty(s, dtype=torch.uint8) for s in shapes]
        ptrs = (C.c_char_p * n)(*files)
        lens = (C.c_size_t * n)(*[len(d) for d in files])
        optrs = (C.c_void_p * n)(*[t.data_ptr() for t in outs])
        rc = (C.c_int * n)()
        res = (_PixelsResult * n)()
        if filt is not None:
            sized = bounds is not None or resize
            self._check(self.lib.jpegqs_cuda_pixels_batch_filtered(self.h, n, ptrs, lens, int(flags), int(niter),
                                                                  0 if layout == "hwc" else 1, scale,
                                                                  fcode if sized else 0, boxes if sized else None,
                                                                  None if orient is None else (C.c_int32 * n)(*orient),
                                                                  m, int(device == "cuda"), optrs, int(max_device_bytes),
                                                                  rc, res, int(bounds is not None), gap, filt, len(filt)))
        elif bounds is not None or gap:
            self._check(self.lib.jpegqs_cuda_pixels_batch_reduced(self.h, n, ptrs, lens, int(flags), int(niter),
                                                                  0 if layout == "hwc" else 1, scale, fcode, boxes,
                                                                  None if orient is None else (C.c_int32 * n)(*orient),
                                                                  m, int(device == "cuda"), optrs, int(max_device_bytes),
                                                                  rc, res, int(bounds is not None), gap))
        elif m:
            self._check(self.lib.jpegqs_cuda_pixels_batch_mode(self.h, n, ptrs, lens, int(flags), int(niter),
                                                               0 if layout == "hwc" else 1, scale,
                                                               fcode if resize else 0, boxes if resize else None,
                                                               None if orient is None else (C.c_int32 * n)(*orient), m,
                                                               int(device == "cuda"), optrs, int(max_device_bytes), rc,
                                                               res))
        elif orient is not None:
            self._check(self.lib.jpegqs_cuda_pixels_batch_oriented(self.h, n, ptrs, lens, int(flags), int(niter),
                                                                   0 if layout == "hwc" else 1, scale,
                                                                   fcode if resize else 0, boxes if resize else None,
                                                                   (C.c_int32 * n)(*orient), int(device == "cuda"),
                                                                   optrs, int(max_device_bytes), rc, res))
        elif resize:
            self._check(self.lib.jpegqs_cuda_pixels_batch_resized(self.h, n, ptrs, lens, int(flags), int(niter),
                                                                  0 if layout == "hwc" else 1, scale, fcode, boxes,
                                                                  int(device == "cuda"), optrs, int(max_device_bytes), rc,
                                                                  res))
        elif scale == 1:
            self._check(self.lib.jpegqs_cuda_pixels_batch(self.h, n, ptrs, lens, int(flags), int(niter),
                                                          0 if layout == "hwc" else 1, int(device == "cuda"), optrs,
                                                          int(max_device_bytes), rc, res))
        else:
            self._check(self.lib.jpegqs_cuda_pixels_batch_scaled(self.h, n, ptrs, lens, int(flags), int(niter),
                                                                 0 if layout == "hwc" else 1, scale, int(device == "cuda"),
                                                                 optrs, int(max_device_bytes), rc, res))
        for i in range(n):
            if rc[i] == -2:
                raise QsError(f"decode_pixels: file {i}: {self.lib.jpegqs_cuda_last_error(self.h).decode()}")
            if rc[i] < 0:
                raise QsError(f"decode_pixels: file {i}: the render takes 1 or 3 components with integral "
                              "sampling ratios only")
        return [(outs[i], res[i].warnings, res[i].host_decoded, res[i].smoothed, res[i].stop, res[i].upsampled,
                 (res[i].reason or b"").decode()) for i in range(n)]

    @staticmethod
    def _thumbnail_args(n: int, thumbnail, resize: bool, scale: int, who: str):
        """thumbnail's bounds per file, or None; ValueError with size, crop or scale_denom other than 1"""
        if thumbnail is None:
            return None
        if resize or scale != 1:
            raise ValueError(f"{who}: thumbnail takes no size, crop or scale_denom (thumbnail scales each file itself)")
        return _thumbnail_bounds(n, thumbnail, who)

    @staticmethod
    def _thumbnail_boxes(shapes, bounds, layout: str, gap: float, loaded: bool):
        """per file, the thumbnail's output shape and its C box (the bound): shapes are the full-size
        (oriented) pictures', read as thumbnail sees them"""
        lib = load()
        out = []
        for i, (sh, (bw, bh)) in enumerate(zip(shapes, bounds)):
            h, w, c = sh if layout == "hwc" else (sh[1], sh[2], sh[0])
            s, tw, th = C.c_int(), C.c_int(), C.c_int()
            if lib.jpegqs_cuda_thumbnail_geometry(w, h, bw, bh, gap, int(loaded), C.byref(s), C.byref(tw), C.byref(th)) < 0:
                raise ValueError(f"thumbnail: file {i}: {lib.jpegqs_cuda_last_error(None).decode()}")
            out.append(((th.value, tw.value, c) if layout == "hwc" else (c, th.value, tw.value), _ResizeBox(0, 0, 0, 0, bw, bh)))
        return out

    # ---- whole image, host buffers (the call a user of the reference makes) ----
    def do_quantsmooth(self, image: CoefImage, flags: int, niter: int, progprec: int = 0,
                       progress=None, inplace: bool = False, pinned: bool = False):
        """pinned=True stages the coefficient arrays in page-locked memory (what the C entry
        point do_quantsmooth does): only then the upload/download slab pipeline is used."""
        out = image if inplace else image.clone()
        keep = []
        ptrs, ups = [], []
        for c in out.comps:
            c.coef = np.ascontiguousarray(c.coef, dtype=np.int16)
            if pinned and c.coef.size:
                pa = PinnedArray(c.coef.shape)
                pa.array[...] = c.coef
                keep.append((pa, c))
                ptrs.append(pa.array.ctypes.data)
            else:
                ptrs.append(c.coef.ctypes.data)
        up_arrays = []
        if len(out.comps) >= 3:
            y = out.comps[0]
            ups.append(None)
            for _ in range(2):
                a = np.zeros((y.hblk, y.wblk, 64), dtype=np.int16)
                up_arrays.append(a)
                ups.append(a.ctypes.data)
        ci = _Image()
        _fill_image(ci, out, ptrs, ups)
        cb = None
        if progress is not None:
            cb = PROGRESS_FN(lambda d, cur, mx: int(progress(cur, mx)))
            keep.append(cb)
        ret = self._check(self.lib.jpegqs_cuda_run_host(
            self.h, C.byref(ci), flags & 0x7f, niter, progprec,
            C.cast(cb, C.c_void_p) if cb else None, None))
        for item in keep:
            if isinstance(item, tuple):
                pa, c = item
                c.coef[...] = pa.array
                pa.close()
        self._collect(out, ci, up_arrays)
        return ret, out

    @staticmethod
    def _collect(out: CoefImage, ci: _Image, up_arrays):
        for i, c in enumerate(out.comps):
            if ci.upsampled and i in (1, 2):
                c.coef = up_arrays[i - 1]
            if ci.upsampled:
                c.h_samp = c.v_samp = 1
            if c.quant is not None:
                c.quant = np.array(list(ci.comp[i].quant), dtype=np.uint16)

    def render_rgb(self, image: CoefImage) -> np.ndarray:
        """Decode a coefficient image (smoothed, or still quantized) to RGB [H, W, 3] uint8 the way
        libjpeg would (islow IDCT, fancy up-sampling, fixed-point YCbCr->RGB)."""
        ptrs = []
        keep = []
        for c in image.comps:
            a = np.ascontiguousarray(c.coef, dtype=np.int16)
            keep.append(a)
            ptrs.append(a.ctypes.data)
        ci = _Image()
        _fill_image(ci, image, ptrs, [])
        out = np.zeros((image.height, image.width, 3), dtype=np.uint8)
        self._check(self.lib.jpegqs_cuda_render_rgb(self.h, C.byref(ci), 0, out.ctypes.data, None))
        return out

    def run_batch_host(self, images: List[CoefImage], flags: int, niter: int):
        outs = [im.clone() for im in images]
        arr = (_Image * len(outs))()
        ups_all = []
        for n, out in enumerate(outs):
            ptrs, ups, up_arrays = [], [], []
            for c in out.comps:
                c.coef = np.ascontiguousarray(c.coef, dtype=np.int16)
                ptrs.append(c.coef.ctypes.data)
            if len(out.comps) >= 3:
                y = out.comps[0]
                ups.append(None)
                for _ in range(2):
                    a = np.zeros((y.hblk, y.wblk, 64), dtype=np.int16)
                    up_arrays.append(a)
                    ups.append(a.ctypes.data)
            _fill_image(arr[n], out, ptrs, ups)
            ups_all.append(up_arrays)
        rets = (C.c_int * len(outs))()
        self._check(self.lib.jpegqs_cuda_run_batch(self.h, len(outs), arr, flags & 0x7f, niter, 0, rets, None))
        for n, out in enumerate(outs):
            self._collect(out, arr[n], ups_all[n])
        return list(rets), outs

    # ---- device-resident buffers (torch tensors or raw pointers) ----
    def run_device(self, image: CoefImage, coef_ptrs: Sequence[int], up_ptrs: Sequence[Optional[int]],
                   flags: int, niter: int, stream: int = 0):
        """image carries geometry + quant tables; coef_ptrs/up_ptrs are device pointers.
        Returns (ret, upsampled)."""
        ci = _Image()
        _fill_image(ci, image, coef_ptrs, up_ptrs)
        ret = self._check(self.lib.jpegqs_cuda_run_device(self.h, C.byref(ci), flags & 0x7f, niter, 0,
                                                         None, None, C.c_void_p(stream or None)))
        return ret, bool(ci.upsampled)

    def run_batch_device(self, images: List[CoefImage], coef_ptrs: List[Sequence[int]],
                         up_ptrs: List[Sequence[Optional[int]]], flags: int, niter: int, stream: int = 0):
        arr = (_Image * len(images))()
        for n, im in enumerate(images):
            _fill_image(arr[n], im, coef_ptrs[n], up_ptrs[n] if up_ptrs else [])
        rets = (C.c_int * len(images))()
        self._check(self.lib.jpegqs_cuda_run_batch(self.h, len(images), arr, flags & 0x7f, niter, 1, rets,
                                                   C.c_void_p(stream or None)))
        return list(rets), [bool(a.upsampled) for a in arr]

    # ---- stream-ordered on torch tensors (include/jpegqs_cuda.h jpegqs_cuda_run_async) ----
    def run_async(self, images: Sequence[CoefImage], coefs, flags: int, niter: int, up=None, stream=None):
        """Smooth device-resident coefficients in place without blocking the calling thread.

        images: CoefImages carrying geometry and quant tables (their arrays are not read).
        coefs[i][c]: CUDA int16 contiguous tensors [hblk, wblk, 64] on this context's device.
        up[i]: the two luma-sized int16 tensors for image i's up-sampled chroma, or None; they are
        allocated when UPSAMPLE_UV can trigger and not given.  stream: a torch.cuda.Stream
        (default: the current one).  Everything, including the workspace, is enqueued on that
        stream; the call returns before the GPU has done anything.  The images' quant tables
        are set to ones on return, as do_quantsmooth does.

        Returns (status, up): status is an int32 device tensor [n, 2] of (stop, upsampled) per
        image, up the per-image pairs of up-sampled chroma tensors (None where UPSAMPLE_UV cannot
        trigger); they hold the result only where status[i, 1] is 1.  Capturable with
        torch.cuda.graph: a replay re-runs on the current contents of the same tensors."""
        import torch
        n = len(images)
        if len(coefs) != n or (up is not None and len(up) != n):
            raise ValueError("images, coefs and up must have one entry per image")
        ups, tensors = [], []
        for i, im in enumerate(images):
            if len(coefs[i]) != len(im.comps):
                raise ValueError(f"image {i}: {len(coefs[i])} coefficient tensors for {len(im.comps)} components")
            for c, (comp, t) in enumerate(zip(im.comps, coefs[i])):
                _check_tensor(t, (comp.hblk, comp.wblk, 64), f"coefs[{i}][{c}]")
                tensors.append((f"coefs[{i}][{c}]", t))
            given = up[i] if up is not None else None
            if given is not None:
                if len(given) != 2:
                    raise ValueError(f"up[{i}]: expected two tensors")
                y = im.comps[0]
                for j, t in enumerate(given):
                    _check_tensor(t, (y.hblk, y.wblk, 64), f"up[{i}][{j}]")
                    tensors.append((f"up[{i}][{j}]", t))
            ups.append(given)
        device = self.device if self.device >= 0 else torch.cuda.current_device()
        for what, t in tensors:
            if not t.is_cuda or t.device.index != device:
                raise ValueError(f"{what}: on {t.device}, expected cuda:{device}")
        stream = stream if stream is not None else torch.cuda.current_stream(device)
        with torch.cuda.device(device), torch.cuda.stream(stream):
            for i, im in enumerate(images):
                if ups[i] is None and upsample_can_trigger(im, flags):
                    y = im.comps[0]
                    ups[i] = tuple(torch.empty((y.hblk, y.wblk, 64), dtype=torch.int16, device=device)
                                   for _ in range(2))
            coef_ptrs = [[t.data_ptr() for t in coefs[i]] for i in range(n)]
            up_ptrs = [[None, ups[i][0].data_ptr(), ups[i][1].data_ptr()] if ups[i] is not None else []
                       for i in range(n)]
            arr = _image_array(images, coef_ptrs, up_ptrs)
            size = C.c_size_t(0)
            self._check(self.lib.jpegqs_cuda_async_workspace_bytes(n, arr, flags & 0x7f, C.byref(size)))
            # allocated on `stream`: the caching allocator hands the memory out again only to work
            # queued after this call's kernels on that stream, so it may be released at return
            ws = torch.empty(max(size.value, 1), dtype=torch.uint8, device=device)
            status = torch.empty((n, 2), dtype=torch.int32, device=device)
            self._check(self.lib.jpegqs_cuda_run_async(self.h, n, arr, flags & 0x7f, niter, ws.data_ptr(),
                                                       size.value, status.data_ptr() if n else None,
                                                       _stream_handle(stream)))
        for i, im in enumerate(images):
            for c, comp in enumerate(im.comps):
                if comp.quant is not None:
                    comp.quant = np.array(list(arr[i].comp[c].quant), dtype=np.uint16)
        return status, [tuple(u) if u is not None else None for u in ups]

    # ---- stream-ordered render to RGB (include/jpegqs_cuda.h jpegqs_cuda_render_async) ----
    def render_async(self, images: Sequence[CoefImage], coefs, status=None, up=None, layout: str = "hwc",
                     out=None, stream=None, scale_denom: int = 1, orientation=None, mode=None):
        """Decode device-resident coefficients to 8-bit RGB, as libjpeg would, without blocking the
        calling thread.  The coefficient tensors are only read.

        images, coefs, up: as for run_async; `status` and `up` are what run_async returned, so that
        up-sampled chroma is read from `up` exactly where status[i, 1] is 1 on the device.  status
        may also be a sequence of per-image booleans (the `upsampled` run_device and
        run_batch_device report), or None: every image reads `coefs`.
        layout: "hwc" gives uint8 [H, W, 3] per image, "chw" gives [3, H, W].  out: a sequence of
        per-image uint8 CUDA tensors of that shape to write (a batched tensor's unbind(0) will do);
        by default they are allocated on the stream.  stream: a torch.cuda.Stream (default: the
        current one).  scale_denom 2, 4 or 8: libjpeg's scaled decode (jpegqs_cuda_render_scaled_async),
        H and W then being ceil(height / d) and ceil(width / d).  orientation: None, or a sequence of
        one EXIF orientation 1..8 per image (jpegqs_cuda_render_oriented_async); each output is then the
        picture as Pillow's Image.transpose turns it, with H and W swapped for 5..8.  Capturable with
        torch.cuda.graph.  Returns the list of output tensors.
        mode: None, or "RGB" / "L": Pillow's Image.convert(mode) of the picture
        (jpegqs_cuda_render_mode_async), 3 or 1 channels for images of 1, 3 or 4 components, each
        image's CoefImage.colorspace deciding the conversion (4 components: JCS_CMYK or JCS_YCCK)."""
        import torch
        n = len(images)
        if layout not in ("hwc", "chw"):
            raise ValueError(f"layout {layout!r}: expected 'hwc' or 'chw'")
        d = _scale_denom(scale_denom, "render_async")
        m = _mode(mode, "render_async")
        if orientation is not None and (isinstance(orientation, (str, bytes)) or _orient_int(orientation) is not None):
            raise ValueError("render_async: orientation: expected a sequence of one value 1..8 per image")
        orient = _orientations(orientation, n, "render_async", lo=1)
        if len(coefs) != n or (up is not None and len(up) != n) or (out is not None and len(out) != n):
            raise ValueError("images, coefs, up and out must have one entry per image")
        host_up = None
        if status is not None and not isinstance(status, torch.Tensor):
            host_up = [bool(u) for u in status]
            if len(host_up) != n:
                raise ValueError("status must have one entry per image")
        tensors = []
        for i, im in enumerate(images):
            if len(coefs[i]) != len(im.comps):
                raise ValueError(f"image {i}: {len(coefs[i])} coefficient tensors for {len(im.comps)} components")
            for c, (comp, t) in enumerate(zip(im.comps, coefs[i])):
                _check_tensor(t, (comp.hblk, comp.wblk, 64), f"coefs[{i}][{c}]")
                tensors.append((f"coefs[{i}][{c}]", t))
            given = up[i] if up is not None else None
            if given is not None:
                if len(given) != 2 or len(im.comps) < 3:
                    raise ValueError(f"up[{i}]: expected two tensors for a three-component image")
                y = im.comps[0]
                for j, t in enumerate(given):
                    _check_tensor(t, (y.hblk, y.wblk, 64), f"up[{i}][{j}]")
                    tensors.append((f"up[{i}][{j}]", t))
            if host_up is not None and host_up[i] and given is None:
                raise ValueError(f"image {i} is up-sampled but up[{i}] is missing")
        if isinstance(status, torch.Tensor):
            if status.dtype != torch.int32 or tuple(status.shape) != (n, 2) or not status.is_contiguous():
                raise ValueError(f"status: expected a contiguous int32 tensor [{n}, 2]")
            tensors.append(("status", status))
        shapes = [_scaled_shape(im.width, im.height, 3 if m < 2 else 1, layout, d) for im in images]
        if orient is not None:
            shapes = [_oriented_shape(s, o, layout) for s, o in zip(shapes, orient)]
        if out is not None:
            for i, t in enumerate(out):
                if not isinstance(t, torch.Tensor):
                    raise TypeError(f"out[{i}]: expected a torch.Tensor, got {type(t).__name__}")
                if t.dtype != torch.uint8:
                    raise TypeError(f"out[{i}]: dtype {t.dtype}, expected torch.uint8")
                if tuple(t.shape) != shapes[i]:
                    raise ValueError(f"out[{i}]: shape {tuple(t.shape)}, expected {shapes[i]}")
                if not t.is_contiguous():
                    raise ValueError(f"out[{i}]: not contiguous")
                tensors.append((f"out[{i}]", t))
        device = self.device if self.device >= 0 else torch.cuda.current_device()
        for what, t in tensors:
            if not t.is_cuda or t.device.index != device:
                raise ValueError(f"{what}: on {t.device}, expected cuda:{device}")
        stream = stream if stream is not None else torch.cuda.current_stream(device)
        with torch.cuda.device(device), torch.cuda.stream(stream):
            if out is None:
                out = [torch.empty(s, dtype=torch.uint8, device=device) for s in shapes]
            out = list(out)
            coef_ptrs = [[t.data_ptr() for t in coefs[i]] for i in range(n)]
            up_ptrs = [[None, up[i][0].data_ptr(), up[i][1].data_ptr()] if up is not None and up[i] is not None else []
                       for i in range(n)]
            arr = _image_array(images, coef_ptrs, up_ptrs)
            for i in range(n):
                arr[i].upsampled = int(bool(host_up and host_up[i]))
            outs = (C.c_void_p * max(n, 1))(*[t.data_ptr() for t in out])
            st = status.data_ptr() if isinstance(status, torch.Tensor) else None
            if m:
                self._check(self.lib.jpegqs_cuda_render_mode_async(
                    self.h, n, arr, st, 0 if layout == "hwc" else 1, d,
                    None if orient is None else (C.c_int32 * max(n, 1))(*orient),
                    (C.c_int32 * max(n, 1))(*[int(im.colorspace) for im in images]), m, outs, _stream_handle(stream)))
            elif orient is not None:
                self._check(self.lib.jpegqs_cuda_render_oriented_async(self.h, n, arr, st, 0 if layout == "hwc" else 1, d,
                                                                       (C.c_int32 * max(n, 1))(*orient), outs,
                                                                       _stream_handle(stream)))
            elif d == 1:
                self._check(self.lib.jpegqs_cuda_render_async(self.h, n, arr, st, 0 if layout == "hwc" else 1, outs,
                                                              _stream_handle(stream)))
            else:
                self._check(self.lib.jpegqs_cuda_render_scaled_async(self.h, n, arr, st, 0 if layout == "hwc" else 1, d,
                                                                     outs, _stream_handle(stream)))
        return out

    # ---- JPEG bytes to coefficients (include/jpegqs_cuda.h jpegqs_cuda_decode_async) ----
    def decode_async(self, images: Sequence[CoefImage], scans, data, out=None, stream=None):
        """Decode JPEG files held in device memory to quantized coefficient tensors, without
        blocking the calling thread.

        images, scans: what parse_jpeg returned for each file (scan not None).  data[i]: a 1-D
        contiguous uint8 CUDA tensor with file i's bytes.  out[i][c] (optional): int16 CUDA tensors
        [hblk, wblk, 64] to write; by default they are allocated on the stream.  stream: a
        torch.cuda.Stream (default: the current one).  Returns (coefs, status): coefs[i][c] the
        tensors (run_async's and render_async's input), status an int32 device tensor [n], 0 where
        image i decoded cleanly, else DECODE_* bits.  Capturable with torch.cuda.graph: a replay
        decodes the current contents of the same data tensors."""
        import torch
        n = len(images)
        if len(scans) != n or len(data) != n or (out is not None and len(out) != n):
            raise ValueError("images, scans, data and out must have one entry per image")
        tensors = []
        for i, (im, sc) in enumerate(zip(images, scans)):
            if sc is None or not isinstance(sc, _Scan):
                raise ValueError(f"scans[{i}]: not a decodable scan (parse_jpeg gave None: use read_jpeg)")
            t = data[i]
            if not isinstance(t, torch.Tensor):
                raise TypeError(f"data[{i}]: expected a torch.Tensor, got {type(t).__name__}")
            if t.dtype != torch.uint8 or t.dim() != 1 or not t.is_contiguous():
                raise ValueError(f"data[{i}]: expected a contiguous 1-D uint8 tensor")
            if t.numel() <= sc.entropy_offset:
                raise ValueError(f"data[{i}]: {t.numel()} bytes, the entropy-coded data starts at {sc.entropy_offset}")
            tensors.append((f"data[{i}]", t))
            if out is not None:
                if len(out[i]) != len(im.comps):
                    raise ValueError(f"out[{i}]: {len(out[i])} tensors for {len(im.comps)} components")
                for c, (comp, o) in enumerate(zip(im.comps, out[i])):
                    _check_tensor(o, (comp.hblk, comp.wblk, 64), f"out[{i}][{c}]")
                    if o.data_ptr() % 16:
                        raise ValueError(f"out[{i}][{c}]: not 16-byte aligned")
                    tensors.append((f"out[{i}][{c}]", o))
        device = self.device if self.device >= 0 else torch.cuda.current_device()
        for what, t in tensors:
            if not t.is_cuda or t.device.index != device:
                raise ValueError(f"{what}: on {t.device}, expected cuda:{device}")
        stream = stream if stream is not None else torch.cuda.current_stream(device)
        with torch.cuda.device(device), torch.cuda.stream(stream):
            if out is None:
                out = [[torch.empty((c.hblk, c.wblk, 64), dtype=torch.int16, device=device) for c in im.comps]
                       for im in images]
            out = [list(o) for o in out]
            arr = _image_array(images, [[t.data_ptr() for t in out[i]] for i in range(n)])
            sc = (_Scan * max(n, 1))(*scans)
            lens = (C.c_size_t * max(n, 1))(*[int(t.numel()) for t in data])
            ptrs = (C.c_void_p * max(n, 1))(*[t.data_ptr() for t in data])
            size = C.c_size_t(0)
            if self.lib.jpegqs_cuda_decode_workspace_bytes(n, arr, sc, lens, C.byref(size)) < 0:
                raise QsError(self.lib.jpegqs_cuda_last_error(None).decode())
            # allocated on `stream`: reused only by work queued after this call's kernels
            ws = torch.empty(max(size.value, 1), dtype=torch.uint8, device=device)
            status = torch.empty((n,), dtype=torch.int32, device=device)
            self._check(self.lib.jpegqs_cuda_decode_async(self.h, n, arr, sc, ptrs, lens, ws.data_ptr(), size.value,
                                                          status.data_ptr() if n else None, _stream_handle(stream)))
        return out, status

    def decode_scans_async(self, images: Sequence[CoefImage], scans, data, out=None, stream=None):
        """decode_async for files of any scan script (progressive, several scans): the same tensor and
        stream conventions, scans[i] what parse_jpeg_scans returned for file i (not None).  The call
        zeroes the output tensors itself.  Returns (coefs, status).  Capturable with torch.cuda.graph:
        every scan's header, position and tables are fixed at capture, so a replay decodes the current
        contents of the same data tensors as a file with identical headers."""
        import torch
        n = len(images)
        if len(scans) != n or len(data) != n or (out is not None and len(out) != n):
            raise ValueError("images, scans, data and out must have one entry per image")
        tensors = []
        for i, (im, sc) in enumerate(zip(images, scans)):
            if not isinstance(sc, ScanList) or not sc:
                raise ValueError(f"scans[{i}]: not a scan list (parse_jpeg_scans gave None: use read_jpeg)")
            t = data[i]
            if not isinstance(t, torch.Tensor):
                raise TypeError(f"data[{i}]: expected a torch.Tensor, got {type(t).__name__}")
            if t.dtype != torch.uint8 or t.dim() != 1 or not t.is_contiguous():
                raise ValueError(f"data[{i}]: expected a contiguous 1-D uint8 tensor")
            if t.numel() < max(r.end for r in sc):
                raise ValueError(f"data[{i}]: {t.numel()} bytes, the last scan ends at {max(r.end for r in sc)}")
            tensors.append((f"data[{i}]", t))
            if out is not None:
                if len(out[i]) != len(im.comps):
                    raise ValueError(f"out[{i}]: {len(out[i])} tensors for {len(im.comps)} components")
                for c, (comp, o) in enumerate(zip(im.comps, out[i])):
                    _check_tensor(o, (comp.hblk, comp.wblk, 64), f"out[{i}][{c}]")
                    if o.data_ptr() % 16:
                        raise ValueError(f"out[{i}][{c}]: not 16-byte aligned")
                    tensors.append((f"out[{i}][{c}]", o))
        device = self.device if self.device >= 0 else torch.cuda.current_device()
        for what, t in tensors:
            if not t.is_cuda or t.device.index != device:
                raise ValueError(f"{what}: on {t.device}, expected cuda:{device}")
        stream = stream if stream is not None else torch.cuda.current_stream(device)
        with torch.cuda.device(device), torch.cuda.stream(stream):
            if out is None:
                out = [[torch.empty((c.hblk, c.wblk, 64), dtype=torch.int16, device=device) for c in im.comps]
                       for im in images]
            out = [list(o) for o in out]
            arr = _image_array(images, [[t.data_ptr() for t in out[i]] for i in range(n)])
            keep, ptrs, counts = _scan_arrays(scans)
            lens = (C.c_size_t * max(n, 1))(*[int(t.numel()) for t in data])
            dptrs = (C.c_void_p * max(n, 1))(*[t.data_ptr() for t in data])
            size = C.c_size_t(0)
            if self.lib.jpegqs_cuda_decode_scans_workspace_bytes(n, arr, ptrs, counts, lens, C.byref(size)) < 0:
                raise QsError(self.lib.jpegqs_cuda_last_error(None).decode())
            # allocated on `stream`: reused only by work queued after this call's kernels
            ws = torch.empty(max(size.value, 1), dtype=torch.uint8, device=device)
            status = torch.empty((n,), dtype=torch.int32, device=device)
            self._check(self.lib.jpegqs_cuda_decode_scans_async(self.h, n, arr, ptrs, counts, dptrs, lens, ws.data_ptr(),
                                                                size.value, status.data_ptr() if n else None,
                                                                _stream_handle(stream)))
        return out, status

    # ---- coefficients to JPEG bytes (include/jpegqs_cuda.h jpegqs_cuda_encode_async) ----
    def encode_async(self, images: Sequence[CoefImage], coefs, heads, optimize: bool = False, status=None, up=None,
                     out=None, capacity=None, stream=None):
        """Write device-resident coefficients as JPEG files in device memory - the bytes the jpegqs
        tool writes for them - without blocking the calling thread.  The coefficient tensors are
        only read.

        images, coefs, up, status: as for render_async (status / up what run_async returned, or
        host booleans).  heads[i]: (prefix, comp_ids, quant_tbls) with prefix a 1-D contiguous uint8
        CUDA tensor holding jpeg_prefix's bytes and the other two what jpeg_prefix returned.
        optimize: optimal Huffman tables (the tool's -o).  out[i] (optional): 1-D uint8 CUDA tensors
        to write, capacity[i] their usable bytes (default: their size); by default out[i] is
        allocated on the stream at encode_bound's size.  stream: a torch.cuda.Stream (default: the
        current one).  Returns (out, lengths, status): lengths an int64 device tensor [n] of file
        lengths, status an int32 device tensor [n], 0 or ENCODE_RANGE / ENCODE_OVERFLOW /
        ENCODE_NO_UP bits (NO_UP: status says image i was up-sampled but up[i] was not given, so it
        was written at its own sampling).
        Capturable with torch.cuda.graph: a replay encodes the current contents of the same tensors."""
        import torch
        n = len(images)
        if len(coefs) != n or len(heads) != n or (up is not None and len(up) != n) or (out is not None and len(out) != n):
            raise ValueError("images, coefs, heads, up and out must have one entry per image")
        if capacity is not None and (out is None or len(capacity) != n):
            raise ValueError("capacity needs out and one entry per image")
        host_up = None
        if status is not None and not isinstance(status, torch.Tensor):
            host_up = [bool(u) for u in status]
            if len(host_up) != n:
                raise ValueError("status must have one entry per image")
        tensors, prefixes = [], []
        for i, im in enumerate(images):
            if len(coefs[i]) != len(im.comps):
                raise ValueError(f"image {i}: {len(coefs[i])} coefficient tensors for {len(im.comps)} components")
            for c, (comp, t) in enumerate(zip(im.comps, coefs[i])):
                _check_tensor(t, (comp.hblk, comp.wblk, 64), f"coefs[{i}][{c}]")
                if t.data_ptr() % 16:
                    raise ValueError(f"coefs[{i}][{c}]: not 16-byte aligned")
                tensors.append((f"coefs[{i}][{c}]", t))
            given = up[i] if up is not None else None
            if given is not None:
                if len(given) != 2 or len(im.comps) != 3:
                    raise ValueError(f"up[{i}]: expected two tensors for a three-component image")
                y = im.comps[0]
                for j, t in enumerate(given):
                    _check_tensor(t, (y.hblk, y.wblk, 64), f"up[{i}][{j}]")
                    if t.data_ptr() % 16:
                        raise ValueError(f"up[{i}][{j}]: not 16-byte aligned")
                    tensors.append((f"up[{i}][{j}]", t))
            if host_up is not None and host_up[i] and given is None:
                raise ValueError(f"image {i} is up-sampled but up[{i}] is missing")
            if len(heads[i]) != 3:
                raise ValueError(f"heads[{i}]: expected (prefix tensor, comp_ids, quant_tbls)")
            p, ids, tbls = heads[i]
            if not isinstance(p, torch.Tensor) or p.dtype != torch.uint8 or p.dim() != 1 or not p.is_contiguous():
                raise ValueError(f"heads[{i}]: the prefix must be a contiguous 1-D uint8 tensor")
            if len(ids) != len(im.comps) or len(tbls) != len(im.comps):
                raise ValueError(f"heads[{i}]: {len(im.comps)} component ids and table numbers expected")
            tensors.append((f"heads[{i}] prefix", p))
            prefixes.append(p)
        if isinstance(status, torch.Tensor):
            if status.dtype != torch.int32 or tuple(status.shape) != (n, 2) or not status.is_contiguous():
                raise ValueError(f"status: expected a contiguous int32 tensor [{n}, 2]")
            tensors.append(("status", status))
        caps = None
        if out is not None:
            caps = []
            for i, t in enumerate(out):
                if not isinstance(t, torch.Tensor):
                    raise TypeError(f"out[{i}]: expected a torch.Tensor, got {type(t).__name__}")
                if t.dtype != torch.uint8 or t.dim() != 1 or not t.is_contiguous():
                    raise ValueError(f"out[{i}]: expected a contiguous 1-D uint8 tensor")
                cap = int(capacity[i]) if capacity is not None else t.numel()
                if cap > t.numel() or cap < prefixes[i].numel():
                    raise ValueError(f"out[{i}]: capacity {cap} outside [prefix length, {t.numel()}]")
                caps.append(cap)
                tensors.append((f"out[{i}]", t))
        device = self.device if self.device >= 0 else torch.cuda.current_device()
        for what, t in tensors:
            if not t.is_cuda or t.device.index != device:
                raise ValueError(f"{what}: on {t.device}, expected cuda:{device}")
        up_ptrs = [[None, up[i][0].data_ptr(), up[i][1].data_ptr()] if up is not None and up[i] is not None else []
                   for i in range(n)]
        arr = _image_array(images, [[t.data_ptr() for t in coefs[i]] for i in range(n)], up_ptrs)
        for i in range(n):
            arr[i].upsampled = int(bool(host_up and host_up[i]))
        if caps is None:
            caps = []
            for i in range(n):
                b = C.c_size_t(0)
                self._check(self.lib.jpegqs_cuda_encode_bound(C.byref(arr[i]), prefixes[i].numel(), C.byref(b)))
                caps.append(int(b.value))
        hs = (_Head * max(n, 1))()
        for i, (p, ids, tbls) in enumerate(heads):
            hs[i] = _head(p.data_ptr(), p.numel(), ids, tbls, len(images[i].comps))
        stream = stream if stream is not None else torch.cuda.current_stream(device)
        with torch.cuda.device(device), torch.cuda.stream(stream):
            if out is None:
                out = [torch.empty(c, dtype=torch.uint8, device=device) for c in caps]
            out = list(out)
            size = C.c_size_t(0)
            self._check(self.lib.jpegqs_cuda_encode_workspace_bytes(n, arr, int(bool(optimize)), C.byref(size)))
            # allocated on `stream`: reused only by work queued after this call's kernels
            ws = torch.empty(max(size.value, 1), dtype=torch.uint8, device=device)
            lengths = torch.empty((n,), dtype=torch.int64, device=device)
            st = torch.empty((n,), dtype=torch.int32, device=device)
            outs = (C.c_void_p * max(n, 1))(*[t.data_ptr() for t in out])
            capa = (C.c_size_t * max(n, 1))(*caps)
            self._check(self.lib.jpegqs_cuda_encode_async(
                self.h, n, arr, hs, int(bool(optimize)), status.data_ptr() if isinstance(status, torch.Tensor) else None,
                outs, capa, lengths.data_ptr() if n else None, st.data_ptr() if n else None, ws.data_ptr(), size.value,
                _stream_handle(stream)))
        return out, lengths, st

    def compress_async(self, pixels, quality=75, subsampling="4:2:0", optimize=False, out=None, stream=None,
                       progressive=False):
        """Write device pictures as the JPEG files Pillow's Image.save(quality=, subsampling=,
        optimize=) writes for them, without blocking the calling thread (jpegqs_cuda_compress_async).

        pixels: uint8 CUDA tensors [H, W, C], C = 3 (RGB) or 1 (grey), whose last two dimensions are
        contiguous (a row stride of at least W * C is taken, so crops of a bigger picture work).
        quality / subsampling / optimize: Pillow's keywords ("4:4:4", "4:2:2", "4:2:0" or 0, 1, 2;
        grey pictures ignore subsampling); progressive=True writes Pillow's progressive=True files
        (jpegqs_cuda_compress_async with JPEGQS_JPEG_PROGRESSIVE).  out[i] (optional): 1-D uint8 CUDA tensors to write, their
        size the capacity; by default allocated on the stream at compress_bound's size.  stream: a
        torch.cuda.Stream (default: the current one).  Returns (out, lengths [n] int64, status [n]
        int32), all on the device; status is 0, or ENCODE_OVERFLOW with lengths[i] the size needed.
        Capturable with torch.cuda.graph: a replay compresses the current contents of the same tensors."""
        import torch
        jp = _jpeg_params(quality, subsampling, optimize, "compress_async", progressive)
        n = len(pixels)
        if out is not None and len(out) != n:
            raise ValueError("compress_async: out must have one entry per picture")
        device = self.device if self.device >= 0 else torch.cuda.current_device()
        pins = (_PixelsIn * max(n, 1))()
        for i, t in enumerate(pixels):
            if not isinstance(t, torch.Tensor):
                raise TypeError(f"compress_async: pixels[{i}]: expected a torch.Tensor, got {type(t).__name__}")
            if t.dtype != torch.uint8 or t.dim() != 3 or t.shape[2] not in (1, 3):
                raise ValueError(f"compress_async: pixels[{i}]: expected a uint8 tensor [H, W, 1|3], got {t.dtype} "
                                 f"{tuple(t.shape)}")
            if t.stride(2) != 1 or t.stride(1) != t.shape[2] or t.stride(0) < t.shape[1] * t.shape[2]:
                raise ValueError(f"compress_async: pixels[{i}]: each row must be contiguous ([H, W, C] with strides "
                                 "(>= W * C, C, 1))")
            if not t.is_cuda or t.device.index != device:
                raise ValueError(f"compress_async: pixels[{i}]: on {t.device}, expected cuda:{device}")
            pins[i] = _pixels_in(t.data_ptr(), tuple(t.shape), t.stride(0))
        caps = []
        if out is not None:
            for i, t in enumerate(out):
                if not isinstance(t, torch.Tensor) or t.dtype != torch.uint8 or t.dim() != 1 or not t.is_contiguous():
                    raise ValueError(f"compress_async: out[{i}]: expected a contiguous 1-D uint8 tensor")
                if not t.is_cuda or t.device.index != device:
                    raise ValueError(f"compress_async: out[{i}]: on {t.device}, expected cuda:{device}")
                caps.append(t.numel())
        else:
            for i in range(n):
                b = C.c_size_t(0)
                self._check(self.lib.jpegqs_cuda_compress_bound(C.byref(pins[i]), C.byref(jp), C.byref(b)))
                caps.append(int(b.value))
        stream = stream if stream is not None else torch.cuda.current_stream(device)
        with torch.cuda.device(device), torch.cuda.stream(stream):
            if out is None:
                out = [torch.empty(c, dtype=torch.uint8, device=device) for c in caps]
            out = list(out)
            size = C.c_size_t(0)
            self._check(self.lib.jpegqs_cuda_compress_workspace_bytes(n, pins, C.byref(jp), C.byref(size)))
            # allocated on `stream`: reused only by work queued after this call's kernels
            ws = torch.empty(max(size.value, 1), dtype=torch.uint8, device=device)
            lengths = torch.empty((n,), dtype=torch.int64, device=device)
            st = torch.empty((n,), dtype=torch.int32, device=device)
            outs = (C.c_void_p * max(n, 1))(*[t.data_ptr() for t in out])
            capa = (C.c_size_t * max(n, 1))(*caps)
            self._check(self.lib.jpegqs_cuda_compress_async(
                self.h, n, pins, C.byref(jp), outs, capa, lengths.data_ptr() if n else None, st.data_ptr() if n else None,
                ws.data_ptr(), size.value, _stream_handle(stream)))
        return out, lengths, st

    def reencode(self, datas, flags: int, niter: int, quality=75, subsampling="4:2:0", optimize=False, scale_denom=1,
                 size=None, crop=None, filter="bicubic", max_device_bytes: int = 0, orientation=None, mode=None,
                 progressive=False, thumbnail=None, reducing_gap=_GAP_DEFAULT, image_filter=None):
        """Many JPEG files to JPEG files of their smoothed pixels (jpegqs_cuda_pixels_batch_jpeg): each
        file's output is exactly Pillow's Image.fromarray(P).save(f, "JPEG", quality=quality,
        subsampling=subsampling, optimize=optimize), where P is the picture decode_pixels gives for the
        same flags, niter, scale_denom, size, crop and filter (a grey file gives a grey JPEG).  Only the
        files cross the bus.  Returns, in the order of datas, one record per file:
            (data: bytes, warnings, host_decoded, smoothed, stop, upsampled, reason)
        with the fields of decode_pixels' records.  ValueError naming the file for a bad quality,
        subsampling, size, crop or filter, before anything runs; QsError naming a file the reader
        rejects, the render cannot take, or whose crop falls outside its picture.  orientation: as for
        decode_pixels (jpegqs_cuda_pixels_batch_jpeg_oriented); "exif" gives Pillow's
        ImageOps.exif_transpose(P).save(...): upright pixels in a JFIF file without the tag.  mode: as for
        decode_pixels (jpegqs_cuda_pixels_batch_jpeg_mode): Pillow's P.convert(mode).save(...), so CMYK
        and YCCK files give RGB files and "L" gives grey files.  progressive=True: Pillow's
        save(..., progressive=True) instead.  thumbnail / reducing_gap: as for decode_pixels
        (jpegqs_cuda_pixels_batch_jpeg_reduced): Pillow's thumbnail (or resize with reducing_gap), then
        save.  image_filter: as for decode_pixels (jpegqs_cuda_pixels_batch_jpeg_filtered): the picture is
        filtered on the device, then saved."""
        if isinstance(datas, (bytes, bytearray, memoryview, str)) or not hasattr(datas, "__len__"):
            raise TypeError("reencode: datas must be a sequence of bytes-like files")
        files = [_file_bytes(d, f"reencode: file {i}") for i, d in enumerate(datas)]
        jp = _jpeg_params(quality, subsampling, optimize, "reencode", progressive)
        if int(max_device_bytes) < 0:
            raise ValueError("reencode: max_device_bytes must be >= 0")
        scale = _scale_denom(scale_denom, "reencode")
        n = len(files)
        resize = size is not None or crop is not None
        fcode = _resize_filter(filter, "reencode")
        if resize:
            sizes, crops = _resize_boxes(n, size, crop, "reencode")
        orient = _orientations(orientation, n, "reencode")
        m = _mode(mode, "reencode")
        bounds = self._thumbnail_args(n, thumbnail, resize, scale, "reencode")
        gap = _reducing_gap(reducing_gap, bounds is not None, "reencode") if resize or bounds is not None else 0.0
        filt = _image_filters(image_filter, "reencode")
        if not n:
            return []
        boxes = None
        if orient is not None:
            orient = [exif_orientation(d) if o == 0 else o for d, o in zip(files, orient)]
        if bounds is not None:
            boxes = (_ResizeBox * n)(*[_ResizeBox(0, 0, 0, 0, bw, bh) for bw, bh in bounds])
        elif resize:
            boxes = (_ResizeBox * n)()
            for i, d in enumerate(files):
                info = _FileInfo()
                if self.lib.jpegqs_cuda_transcode_route(d, len(d), None, C.byref(info)) < 0:
                    raise QsError(f"reencode: file {i}: the reader rejects the file")
                h, w, _ = _oriented_shape(_scaled_shape(info.image_width, info.image_height, 1, "hwc", scale),
                                          orient[i] if orient is not None else 1, "hwc")
                boxes[i] = _resize_box(w, h, sizes[i], crops[i], i, "reencode")
        ptrs = (C.c_char_p * n)(*files)
        lens = (C.c_size_t * n)(*[len(d) for d in files])
        rc = (C.c_int * n)()
        res = (_PixelsResult * n)()
        outs = (C.c_void_p * n)()
        olen = (C.c_size_t * n)()
        if filt is not None:
            self._check(self.lib.jpegqs_cuda_pixels_batch_jpeg_filtered(
                self.h, n, ptrs, lens, int(flags), int(niter), scale, fcode, boxes, C.byref(jp), int(max_device_bytes),
                rc, res, outs, olen, None if orient is None else (C.c_int32 * n)(*orient), m, int(bounds is not None), gap,
                filt, len(filt)))
        elif bounds is not None or gap:
            self._check(self.lib.jpegqs_cuda_pixels_batch_jpeg_reduced(
                self.h, n, ptrs, lens, int(flags), int(niter), scale, fcode, boxes, C.byref(jp), int(max_device_bytes),
                rc, res, outs, olen, None if orient is None else (C.c_int32 * n)(*orient), m, int(bounds is not None), gap))
        elif m:
            self._check(self.lib.jpegqs_cuda_pixels_batch_jpeg_mode(
                self.h, n, ptrs, lens, int(flags), int(niter), scale, fcode, boxes, C.byref(jp), int(max_device_bytes),
                rc, res, outs, olen, None if orient is None else (C.c_int32 * n)(*orient), m))
        elif orient is not None:
            self._check(self.lib.jpegqs_cuda_pixels_batch_jpeg_oriented(self.h, n, ptrs, lens, int(flags), int(niter), scale,
                                                                        fcode, boxes, C.byref(jp), int(max_device_bytes),
                                                                        rc, res, outs, olen, (C.c_int32 * n)(*orient)))
        else:
            self._check(self.lib.jpegqs_cuda_pixels_batch_jpeg(self.h, n, ptrs, lens, int(flags), int(niter), scale, fcode,
                                                               boxes, C.byref(jp), int(max_device_bytes), rc, res, outs, olen))
        try:
            records, bad = [], None
            for i in range(n):
                if rc[i] < 0:
                    if bad is None:
                        bad = i
                    records.append(None)
                    continue
                records.append((C.string_at(outs[i], olen[i]), res[i].warnings, res[i].host_decoded, res[i].smoothed,
                                res[i].stop, res[i].upsampled, (res[i].reason or b"").decode()))
        finally:
            for i in range(n):
                if outs[i]:
                    self.lib.jpegqs_cuda_transcode_free(outs[i])
        if bad is not None:
            if rc[bad] == -2:
                raise QsError(f"reencode: file {bad}: {self.lib.jpegqs_cuda_last_error(self.h).decode()}")
            raise QsError(f"reencode: file {bad}: the render takes 1 or 3 components with integral sampling ratios only")
        return records

    # ---- one slab of a sharded image (include/jpegqs_cuda.h "one image sharded by MCU rows") ----
    def run_slab(self, link, slab: CoefImage, rank: int, world: int, row0: Sequence[int],
                 hblk_total: Sequence[int], flags: int, niter: int, coef_ptrs=None, up_ptrs=None, stream: int = 0):
        """slab: CoefImage whose components hold this rank's block rows (width / height = the
        WHOLE image's).  Host arrays (coef_ptrs None: slab.comps[].coef, modified IN PLACE, results
        for UPSAMPLE_UV in the returned arrays) or device pointers (coef_ptrs / up_ptrs).
        Returns (ret, upsampled, up_arrays)."""
        on_device = coef_ptrs is not None
        up_arrays = []
        if not on_device:
            coef_ptrs, up_ptrs = [], []
            for c in slab.comps:
                c.coef = np.ascontiguousarray(c.coef, dtype=np.int16)
                coef_ptrs.append(c.coef.ctypes.data)
            if len(slab.comps) >= 3:
                y = slab.comps[0]
                up_ptrs.append(None)
                for _ in range(2):
                    a = np.zeros((y.hblk, y.wblk, 64), dtype=np.int16)
                    up_arrays.append(a)
                    up_ptrs.append(a.ctypes.data)
        ci = _Image()
        _fill_image(ci, slab, coef_ptrs, up_ptrs or [])
        g = _Slab()
        g.rank, g.world = rank, world
        for k in range(len(slab.comps)):
            g.row0[k], g.hblk_total[k] = int(row0[k]), int(hblk_total[k])
        ret = self._check(self.lib.jpegqs_cuda_run_slab(self.h, link.h if link is not None else None, C.byref(ci),
                                                       C.byref(g), flags & 0x7f, niter, int(on_device),
                                                       C.c_void_p(stream or None)))
        if not on_device:
            for i, c in enumerate(slab.comps):
                if c.quant is not None:
                    c.quant = np.array(list(ci.comp[i].quant), dtype=np.uint16)
        return ret, bool(ci.upsampled), up_arrays

    # ---- pass level (multi-GPU slabs) ----
    @staticmethod
    def make_job(coef_ptr, plane_ptr, plane2_ptr, wblk, hblk, quant, luma, top_edge, bottom_edge) -> _Job:
        j = _Job()
        j.coef, j.plane, j.plane2 = coef_ptr, plane_ptr, plane2_ptr or None
        j.wblk, j.hblk = wblk, hblk
        for k in range(64):
            j.quant[k] = int(quant[k])
        j.luma, j.top_edge, j.bottom_edge = int(luma), int(top_edge), int(bottom_edge)
        return j

    def pass_idct(self, jobs: List[_Job], mode: int, want_bad: bool = False, stream: int = 0) -> int:
        arr = (_Job * len(jobs))(*jobs)
        bad = C.c_int(0)
        self._check(self.lib.jpegqs_cuda_pass_idct(self.h, len(jobs), arr, mode,
                                                   C.byref(bad) if want_bad else None,
                                                   C.c_void_p(stream or None)))
        return bad.value

    def pass_smooth(self, jobs: List[_Job], flags: int, clamp_out: bool, stream: int = 0):
        arr = (_Job * len(jobs))(*jobs)
        self._check(self.lib.jpegqs_cuda_pass_smooth(self.h, len(jobs), arr, flags & 0x7f, int(clamp_out),
                                                     C.c_void_p(stream or None)))

    def pass_downsample(self, yplane, y_wblk, y_row0, y_hblk_total, plane2, c_wblk, c_rows, c_row0,
                        c_hblk_total, ws, hs, top_edge, bottom_edge, stream: int = 0):
        self._check(self.lib.jpegqs_cuda_pass_downsample(
            self.h, yplane, y_wblk, y_row0, y_hblk_total, plane2, c_wblk, c_rows, c_row0, c_hblk_total,
            ws, hs, int(top_edge), int(bottom_edge), C.c_void_p(stream or None)))

    def pass_upsample(self, cplane, plane2, c_wblk, yplane, y_wblk, y_rows, y_row0, coef_up, scratch,
                      ws, hs, image_width, image_height, stream: int = 0):
        self._check(self.lib.jpegqs_cuda_pass_upsample(
            self.h, cplane, plane2, c_wblk, yplane, y_wblk, y_rows, y_row0, coef_up, scratch, ws, hs,
            image_width, image_height, C.c_void_p(stream or None)))

    def plane_bytes(self, wblk, hblk) -> int:
        return int(self.lib.jpegqs_cuda_plane_bytes(wblk, hblk))

    def plane_stride(self, wblk) -> int:
        return int(self.lib.jpegqs_cuda_plane_stride(wblk))

    def plane_pad(self) -> int:
        return int(self.lib.jpegqs_cuda_plane_pad())


class QsLink:
    """This rank's mailbox + its view of the other ranks' (jpegqs_cuda_link)."""

    def __init__(self, ctx: QsContext, rank: int, world: int, max_wblk: int):
        self.ctx, self.lib, self.rank, self.world = ctx, ctx.lib, rank, world
        h = C.c_void_p()
        ctx._check(self.lib.jpegqs_cuda_link_create(ctx.h, rank, world, max_wblk, C.byref(h)))
        self.h = h

    def export(self) -> bytes:
        n = self.lib.jpegqs_cuda_link_handle_bytes()
        buf = C.create_string_buffer(n)
        self.ctx._check(self.lib.jpegqs_cuda_link_export(self.h, buf))
        return buf.raw

    def connect_ipc(self, handles: Sequence[bytes]):
        blob = b"".join(handles)
        self.ctx._check(self.lib.jpegqs_cuda_link_connect_ipc(self.h, blob))

    @staticmethod
    def connect_local(links: Sequence["QsLink"]):
        arr = (C.c_void_p * len(links))(*[l.h for l in links])
        links[0].ctx._check(links[0].lib.jpegqs_cuda_link_connect_local(arr, len(links)))

    def close(self):
        if getattr(self, "h", None):
            self.lib.jpegqs_cuda_link_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class QsMulti:
    """Several devices of this process behind one call (jpegqs_cuda_multi): what the C entry
    point do_quantsmooth uses when JPEGQS_GPUS is set."""

    def __init__(self, devices):
        self.lib = load()
        if isinstance(devices, int):
            n, arr = devices, None
        else:
            n, arr = len(devices), (C.c_int * len(devices))(*devices)
        h = C.c_void_p()
        rc = self.lib.jpegqs_cuda_multi_create(n, arr, C.byref(h))
        if rc:
            raise QsError(f"jpegqs_cuda_multi_create failed ({rc}): {self.lib.jpegqs_cuda_last_error(None).decode()}")
        self.h = h

    def _image(self, out: CoefImage):
        ptrs, ups, up_arrays = [], [], []
        for c in out.comps:
            c.coef = np.ascontiguousarray(c.coef, dtype=np.int16)
            ptrs.append(c.coef.ctypes.data)
        if len(out.comps) >= 3:
            y = out.comps[0]
            ups.append(None)
            for _ in range(2):
                a = np.zeros((y.hblk, y.wblk, 64), dtype=np.int16)
                up_arrays.append(a)
                ups.append(a.ctypes.data)
        ci = _Image()
        _fill_image(ci, out, ptrs, ups)
        return ci, up_arrays

    def plan(self, image: CoefImage) -> int:
        ci, _ = self._image(image.clone())
        return int(self.lib.jpegqs_cuda_multi_plan(self.h, C.byref(ci)))

    def do_quantsmooth(self, image: CoefImage, flags: int, niter: int):
        out = image.clone()
        ci, up_arrays = self._image(out)
        rc = self.lib.jpegqs_cuda_run_host_multi(self.h, C.byref(ci), flags & 0x7f, niter)
        if rc < 0:
            raise QsError(f"CUDA back end error {rc}: {self.lib.jpegqs_cuda_multi_last_error(self.h).decode()}")
        QsContext._collect(out, ci, up_arrays)
        return rc, out

    def close(self):
        if getattr(self, "h", None):
            self.lib.jpegqs_cuda_multi_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


_default_ctx = {}


def default_context(device: int = -1) -> QsContext:
    if device not in _default_ctx:
        _default_ctx[device] = QsContext(device)
    return _default_ctx[device]


def do_quantsmooth(image: CoefImage, flags: int, niter: int, progprec: int = 0, progress=None,
                   device: int = -1):
    """Python mirror of `int do_quantsmooth(srcinfo, coef_arrays, opts)` (reference
    libjpegqs.h:47-48): returns (stop, smoothed image)."""
    return default_context(device).do_quantsmooth(image, flags, niter, progprec, progress)


def run_async(images: Sequence[CoefImage], coefs, flags: int, niter: int, up=None, stream=None):
    """QsContext.run_async on the default context of the tensors' device: smooths CUDA tensors
    in place, enqueued on `stream` (default: the current one) without waiting.  Returns
    (status [n, 2] int32 device tensor of (stop, upsampled), up-sampled chroma pairs)."""
    import torch
    first = next((t for ts in coefs for t in ts), None)
    if not isinstance(first, torch.Tensor) or not first.is_cuda:
        raise ValueError("run_async: the coefficient tensors must be CUDA tensors")
    return default_context(first.device.index).run_async(images, coefs, flags, niter, up, stream)


def decode_scans_async(images: Sequence[CoefImage], scans, data, out=None, stream=None):
    """QsContext.decode_scans_async on the default context of the data tensors' device: decodes JPEG
    files of any scan script in CUDA tensors to coefficient tensors; returns (coefs, status)."""
    if not data:
        raise ValueError("decode_scans_async: no images")
    first = data[0]
    if not getattr(first, "is_cuda", False):
        raise ValueError("decode_scans_async: the data tensors must be CUDA tensors")
    return default_context(first.device.index).decode_scans_async(images, scans, data, out, stream)


def decode_async(images: Sequence[CoefImage], scans, data, out=None, stream=None):
    """QsContext.decode_async on the default context of the data tensors' device: decodes JPEG
    files in CUDA uint8 tensors to int16 coefficient tensors, enqueued on `stream` (default: the
    current one) without waiting.  Returns (coefs, status [n] int32 device tensor)."""
    import torch
    first = next(iter(data), None)
    if not isinstance(first, torch.Tensor) or not first.is_cuda:
        raise ValueError("decode_async: the data tensors must be CUDA tensors")
    return default_context(first.device.index).decode_async(images, scans, data, out, stream)


def render_async(images: Sequence[CoefImage], coefs, status=None, up=None, layout: str = "hwc", out=None,
                 stream=None, scale_denom: int = 1, orientation=None, mode=None):
    """QsContext.render_async on the default context of the tensors' device: decodes CUDA
    coefficient tensors to uint8 RGB tensors ([H, W, 3] or [3, H, W], at 1/scale_denom size; one
    channel for mode "L"), enqueued on `stream` (default: the current one) without waiting."""
    import torch
    first = next((t for ts in coefs for t in ts), None)
    if not isinstance(first, torch.Tensor) or not first.is_cuda:
        raise ValueError("render_async: the coefficient tensors must be CUDA tensors")
    return default_context(first.device.index).render_async(images, coefs, status, up, layout, out, stream, scale_denom,
                                                            orientation, mode)


def encode_async(images: Sequence[CoefImage], coefs, heads, optimize: bool = False, status=None, up=None, out=None,
                 capacity=None, stream=None):
    """QsContext.encode_async on the default context of the tensors' device: writes CUDA coefficient
    tensors as JPEG files in CUDA uint8 tensors, enqueued on `stream` (default: the current one)
    without waiting.  Returns (out, lengths [n] int64, status [n] int32), all on the device."""
    import torch
    first = next((t for ts in coefs for t in ts), None)
    if not isinstance(first, torch.Tensor) or not first.is_cuda:
        raise ValueError("encode_async: the coefficient tensors must be CUDA tensors")
    return default_context(first.device.index).encode_async(images, coefs, heads, optimize, status, up, out,
                                                            capacity, stream)


def transcode(data: bytes, flags: int, niter: int, optimize: bool = False, copy: int = 2, device: int = -1):
    """QsContext.transcode on the default context of `device`: (bytes, None), or (None, reason) for a
    file the host route must take."""
    return default_context(device).transcode(data, flags, niter, optimize, copy)


def transcode_batch(datas, flags: int, niter: int, optimize: bool = False, copy: int = 2, max_device_bytes: int = 0,
                    device: int = -1):
    """QsContext.transcode_batch on the default context of `device`: a list of (bytes, None) or
    (None, reason), one per file."""
    return default_context(device).transcode_batch(datas, flags, niter, optimize, copy, max_device_bytes)


def decode_pixels(datas, flags: int, niter: int, layout: str = "hwc", device: str = "cuda", max_device_bytes: int = 0,
                  gpu: int = -1, scale_denom: int = 1, size=None, crop=None, filter="bicubic", orientation=None,
                  mode=None, thumbnail=None, reducing_gap=_GAP_DEFAULT, image_filter=None):
    """QsContext.decode_pixels on the default context of CUDA device `gpu`: one record (pixels, warnings,
    host_decoded, smoothed, stop, upsampled, reason) per file, at 1/scale_denom size, cropped and resized
    as Pillow would with size / crop / filter ((width, height) and (left, top, right, bottom), Pillow's
    conventions), turned by `orientation` ("exif", 1..8, or one value 0..8 per file) first and converted by
    `mode` (None, "RGB" or "L", Pillow's Image.convert) before the crop; or Pillow's thumbnail(bound, filter,
    reducing_gap) with `thumbnail`; then Pillow's Image.filter of each of `image_filter` (GaussianBlur, BoxBlur
    or UnsharpMask) in turn."""
    return default_context(gpu).decode_pixels(datas, flags, niter, layout, device, max_device_bytes, scale_denom,
                                              size, crop, filter, orientation, mode, thumbnail, reducing_gap,
                                              image_filter)


def compress_async(pixels, quality=75, subsampling="4:2:0", optimize=False, out=None, stream=None, progressive=False):
    """QsContext.compress_async on the default context of the tensors' device: writes uint8 CUDA pictures
    [H, W, C] as Pillow's JPEG files in CUDA uint8 tensors, enqueued on `stream` (default: the current
    one) without waiting.  Returns (out, lengths [n] int64, status [n] int32), all on the device."""
    import torch
    first = next(iter(pixels), None)
    if not isinstance(first, torch.Tensor) or not first.is_cuda:
        raise ValueError("compress_async: the pixel tensors must be CUDA tensors")
    return default_context(first.device.index).compress_async(pixels, quality, subsampling, optimize, out, stream,
                                                               progressive)


def reencode(datas, flags: int, niter: int, quality=75, subsampling="4:2:0", optimize=False, scale_denom=1, size=None,
             crop=None, filter="bicubic", max_device_bytes: int = 0, gpu: int = -1, orientation=None, mode=None,
             progressive=False, thumbnail=None, reducing_gap=_GAP_DEFAULT, image_filter=None):
    """QsContext.reencode on the default context of CUDA device `gpu`: one record (data, warnings,
    host_decoded, smoothed, stop, upsampled, reason) per file, data the JPEG file Pillow's save writes for
    the picture decode_pixels gives with the same arguments."""
    return default_context(gpu).reencode(datas, flags, niter, quality, subsampling, optimize, scale_denom, size, crop,
                                         filter, max_device_bytes, orientation, mode, progressive, thumbnail,
                                         reducing_gap, image_filter)
