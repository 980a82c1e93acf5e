"""ctypes binding of libfear_b200.so (the C ABI declared in include/fear_b200.h).

There is no fallback: if the shared object is missing or a call fails, a RuntimeError carrying
``fear_last_error()`` is raised.
"""
import ctypes
import os
from ctypes import POINTER, c_char_p, c_double, c_float, c_int, c_int32, c_int64, c_size_t, c_uint32, c_uint64, c_void_p

import numpy as np

from .build import LIB_PATH


class FearBox(ctypes.Structure):
    _fields_ = [
        ("x", c_double), ("y", c_double), ("w", c_double), ("h", c_double),
        ("score", c_float), ("row", c_int32), ("col", c_int32), ("flat", c_int32),
    ]


BOX_DTYPE = np.dtype(
    [("x", "<f8"), ("y", "<f8"), ("w", "<f8"), ("h", "<f8"), ("score", "<f4"), ("row", "<i4"), ("col", "<i4"),
     ("flat", "<i4")]
)
assert BOX_DTYPE.itemsize == ctypes.sizeof(FearBox) == 48

# FearFrame / FearTarget of the multi-target tracking loop (include/fear_b200.h)
FRAME_DTYPE = np.dtype([("offset", "<i8"), ("H", "<i4"), ("W", "<i4")])
TARGET_INTS = 16  # a FearTarget is 16 int32: frame, x, y, w, h, cx, cy, cw, ch, pad_r, pad_g, pad_b, 4 reserved
assert FRAME_DTYPE.itemsize == 16
# FearFrameView: a frame anywhere in device memory, with byte strides (include/fear_b200.h)
VIEW_DTYPE = np.dtype([("data", "<u8"), ("row_stride", "<i8"), ("pixel_stride", "<i8"), ("channel_stride", "<i8"),
                       ("H", "<i4"), ("W", "<i4")])
assert VIEW_DTYPE.itemsize == 40
# FearFrameYUV420: a YUV 4:2:0 frame (NV12, I420) anywhere in device memory, with byte strides (include/fear_b200.h)
YUV420_DTYPE = np.dtype([("y", "<u8"), ("u", "<u8"), ("v", "<u8"), ("y_row_stride", "<i8"), ("y_pixel_stride", "<i8"),
                         ("uv_row_stride", "<i8"), ("uv_pixel_stride", "<i8"), ("H", "<i4"), ("W", "<i4")])
assert YUV420_DTYPE.itemsize == 64
# FearFrameYUV: FearFrameYUV420 plus its colour format (matrix, range, bit depth, sample alignment)
YUV_DTYPE = np.dtype(YUV420_DTYPE.descr + [("matrix", "<i4"), ("full_range", "<i4"), ("bits", "<i4"),
                                           ("shift", "<i4")])
assert YUV_DTYPE.itemsize == 80
# FearFrameYCbCr: FearFrameYUV plus its chroma subsampling (4:2:0, 4:2:2, 4:4:4)
YCBCR_DTYPE = np.dtype(YUV_DTYPE.descr + [("chroma_shift_x", "<i4"), ("chroma_shift_y", "<i4")])
assert YCBCR_DTYPE.itemsize == 88
# FearFrameYCbCrV210: FearFrameYCbCr plus whether the entry is a v210 surface (10-bit 4:2:2, three codes per word)
YCBCR_V210_DTYPE = np.dtype(YCBCR_DTYPE.descr + [("v210", "<i4"), ("reserved", "<i4")])
assert YCBCR_V210_DTYPE.itemsize == 96
# FearFrameYCbCrHDR: FearFrameYCbCrV210 plus the H.273 transfer characteristics (0, PQ 16, HLG 18)
YCBCR_HDR_DTYPE = np.dtype(YCBCR_V210_DTYPE.descr + [("transfer", "<i4"), ("reserved_hdr", "<i4")])
assert YCBCR_HDR_DTYPE.itemsize == 104
# FearFrameBayer: a raw Bayer mosaic (unpacked 8 to 16 bits, MIPI RAW10 / RAW12) with its row pitch and CFA pattern
BAYER_DTYPE = np.dtype([("data", "<u8"), ("row_stride", "<i8"), ("H", "<i4"), ("W", "<i4"), ("pattern", "<i4"),
                        ("bits", "<i4"), ("shift", "<i4"), ("packing", "<i4")])
assert BAYER_DTYPE.itemsize == 40
# FearFrameMono: a single-channel frame (FearFrameBayer's containers), its gain control and the code range it uses
MONO_DTYPE = np.dtype([("data", "<u8"), ("row_stride", "<i8"), ("H", "<i4"), ("W", "<i4"), ("bits", "<i4"),
                       ("shift", "<i4"), ("packing", "<i4"), ("agc", "<i4"), ("lo", "<i4"), ("hi", "<i4")])
assert MONO_DTYPE.itemsize == 48
# FearFrameRGB: three channel addresses in one kind of little-endian container, shared strides, the code's depth and
# each channel's shift
RGB_DTYPE = np.dtype([("r", "<u8"), ("g", "<u8"), ("b", "<u8"), ("row_stride", "<i8"), ("pixel_stride", "<i8"),
                      ("H", "<i4"), ("W", "<i4"), ("container", "<i4"), ("bits", "<i4"), ("shift_r", "<i4"),
                      ("shift_g", "<i4"), ("shift_b", "<i4"), ("reserved", "<i4")])
assert RGB_DTYPE.itemsize == 72
# the `table` argument of fear_crop_targets_oriented_u8 / fear_advance_targets_oriented: FEAR_TABLE_* of the header,
# keyed by the name FEARMultiTracker gives each table
ORIENT_TABLES = {"views": 0, "yuv": 1, "ycbcr": 2, "ycbcr_v210": 3, "ycbcr_hdr": 4, "bayer": 5, "mono": 6, "rgb": 7}

_SIGNATURES = {
    # name: (restype, argtypes)
    "fear_init": (c_int, [c_int]),
    "fear_abi_version": (c_int, []),
    "fear_last_error": (c_char_p, []),
    "fear_weight_count": (c_int, []),
    "fear_weight_name": (c_char_p, [c_int]),
    "fear_weight_numel": (c_int64, [c_int]),
    "fear_pack_weights": (c_int, [c_void_p, POINTER(c_uint64), c_int, POINTER(c_void_p)]),
    "fear_reserve": (c_int, [c_void_p, c_int]),
    "fear_free": (None, [c_void_p]),
    "fear_get_features": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "fear_backbone": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "fear_head": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "fear_head_update": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "fear_track": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "fear_track_u8": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "fear_get_features_u8": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "fear_forward": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "fear_crop_resize_u8": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p]),
    "fear_crop_targets_u8": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_double, c_int, c_void_p, c_void_p]),
    "fear_advance_targets": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_void_p]),
    "fear_crop_targets_view_u8": (c_int, [c_void_p, c_int, c_void_p, c_int, c_double, c_int, c_void_p, c_void_p]),
    "fear_advance_targets_view": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_void_p]),
    "fear_frame_sums_u8": (c_int, [c_void_p, c_int, c_void_p, c_void_p]),
    "fear_crop_targets_yuv420_u8": (c_int, [c_void_p, c_int, c_void_p, c_int, c_double, c_int, c_void_p, c_void_p]),
    "fear_advance_targets_yuv420": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_void_p]),
    "fear_frame_sums_yuv420_u8": (c_int, [c_void_p, c_int, c_void_p, c_void_p]),
    "fear_crop_targets_yuv_u8": (c_int, [c_void_p, c_int, c_void_p, c_int, c_double, c_int, c_void_p, c_void_p]),
    "fear_advance_targets_yuv": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_void_p]),
    "fear_frame_sums_yuv_u8": (c_int, [c_void_p, c_int, c_void_p, c_void_p]),
    "fear_crop_targets_ycbcr_u8": (c_int, [c_void_p, c_int, c_void_p, c_int, c_double, c_int, c_void_p, c_void_p]),
    "fear_advance_targets_ycbcr": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_void_p]),
    "fear_frame_sums_ycbcr_u8": (c_int, [c_void_p, c_int, c_void_p, c_void_p]),
    "fear_crop_targets_ycbcr_v210_u8": (c_int, [c_void_p, c_int, c_void_p, c_int, c_double, c_int, c_void_p, c_void_p]),
    "fear_advance_targets_ycbcr_v210": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_void_p]),
    "fear_frame_sums_ycbcr_v210_u8": (c_int, [c_void_p, c_int, c_void_p, c_void_p]),
    "fear_crop_targets_ycbcr_hdr_u8": (c_int, [c_void_p, c_int, c_void_p, c_int, c_double, c_int, c_void_p, c_void_p]),
    "fear_advance_targets_ycbcr_hdr": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_void_p]),
    "fear_frame_sums_ycbcr_hdr_u8": (c_int, [c_void_p, c_int, c_void_p, c_void_p]),
    "fear_crop_targets_bayer_u8": (c_int, [c_void_p, c_int, c_void_p, c_int, c_double, c_int, c_void_p, c_void_p]),
    "fear_advance_targets_bayer": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_void_p]),
    "fear_frame_sums_bayer_u8": (c_int, [c_void_p, c_int, c_void_p, c_void_p]),
    "fear_frame_range_mono": (c_int, [c_void_p, c_int, c_void_p]),
    "fear_crop_targets_mono_u8": (c_int, [c_void_p, c_int, c_void_p, c_int, c_double, c_int, c_void_p, c_void_p]),
    "fear_advance_targets_mono": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_void_p]),
    "fear_frame_sums_mono_u8": (c_int, [c_void_p, c_int, c_void_p, c_void_p]),
    "fear_crop_targets_rgb_u8": (c_int, [c_void_p, c_int, c_void_p, c_int, c_double, c_int, c_void_p, c_void_p]),
    "fear_advance_targets_rgb": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_void_p]),
    "fear_frame_sums_rgb_u8": (c_int, [c_void_p, c_int, c_void_p, c_void_p]),
    "fear_crop_targets_oriented_u8": (c_int, [c_int, c_void_p, c_void_p, c_int, c_void_p, c_int, c_double, c_int,
                                              c_void_p, c_void_p]),
    "fear_advance_targets_oriented": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p, c_int, c_int,
                                              c_void_p]),
    "fear_gather_targets": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "fear_scatter_targets": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p]),
    "fear_decode": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "fear_decode_smooth": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "fear_head_sized": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_int, c_void_p, c_void_p,
                                c_void_p]),
    "fear_track_sized": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "fear_track_sized_u8": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                    c_void_p]),
    "fear_forward_sized": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "fear_decode_sized": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "fear_decode_smooth_sized": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "fear_corr_concat_f32": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p]),
    "fear_corr_concat_workspace_bytes": (c_size_t, [c_int, c_int]),
    "fear_corr_concat_ws_f32": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
    "fear_corr_nhwc_f32": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p]),
    "fear_debug_backbone_prefix": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "fear_debug_head_tensor": (c_int, [c_void_p, c_char_p, c_int, c_void_p, c_void_p]),
    "fear_debug_fill_workspace": (c_int, [c_void_p, c_uint32, c_void_p]),
    "fear_set_option": (c_int, [c_void_p, c_char_p, c_char_p]),
    "fear_launch_count": (c_int64, [c_void_p]),
    "fear_generation": (c_int64, [c_void_p]),
    "fear_profile": (c_int, [c_void_p, c_int]),
    "fear_stage_count": (c_int, []),
    "fear_stage_name": (c_char_p, [c_int]),
    "fear_stage_ms": (c_int, [c_void_p, c_int, POINTER(c_float), POINTER(c_int64)]),
}

_lib = None
_inited_devices = set()


def exported_symbols():
    return sorted(_SIGNATURES)


def load() -> ctypes.CDLL:
    """dlopen the library (no device needed) and attach signatures."""
    global _lib
    if _lib is None:
        if not os.path.isfile(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: build it with `python -m feartracker_b200.build` "
                "(there is no CPU / PyTorch fallback for the FEAR hot path)"
            )
        lib = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(lib, name)  # AttributeError if the .so does not export it
            fn.restype, fn.argtypes = res, args
        _lib = lib
    return _lib


def last_error() -> str:
    return load().fear_last_error().decode()


def check(code: int, what: str) -> None:
    if code != 0:
        raise RuntimeError(f"{what} failed ({code}): {last_error()}")


def init(device: int = 0) -> ctypes.CDLL:
    """Initialise the library's per-device state (once per device; several devices per process are fine).
    ``fear_init`` makes ``device`` current while a handle is packed; the caller's device is restored here."""
    lib = load()
    if device not in _inited_devices:
        check(lib.fear_init(device), "fear_init")
        _inited_devices.add(device)
    return lib


def weight_table():
    lib = load()
    return [(lib.fear_weight_name(i).decode(), int(lib.fear_weight_numel(i))) for i in range(lib.fear_weight_count())]


def stage_names():
    lib = load()
    return [lib.fear_stage_name(i).decode() for i in range(lib.fear_stage_count())]
