"""FEARMultiTracker: many targets, in one or several video streams, stepped together once per frame.

    trk = FEARMultiTracker(net, cuda_id=0, max_targets=64, **FEAR_XS_TRACKER_KWARGS)
    ids = trk.add(frames, rects, streams=None)   # frames: one HxWx3 uint8 array or a list of F; streams -> frame index
    out = trk.update(frames)                      # {"bbox": (N,4) int64, "score": (N,) float32, "ids": (N,) int64}
    out = trk.update({3: f3, 17: f17})            # only the streams that have a new frame: their M targets' results
    trk.remove(ids); trk.reset()

A list holds one frame of every stream.  Streams that do not tick together (cameras at different rates, a stalled or
reconnecting camera, frames batched as they arrive) pass a mapping {stream id: frame} of the streams at hand to update
and add: only the targets of those streams are stepped, and every other target's state and template stay as they were.

Frames are numpy arrays in host memory, uint8 (H, W, 3) CUDA tensors already on the tracker's device, strided views
included (t[..., :3] of an RGBA surface, t.permute(1, 2, 0) of a CHW tensor, t[y0:y1, x0:x1]), or YUV frames on the
device as a video decoder, webcam or capture card writes them: YUV420Frame (NV12 / I420, P010 / P016 / yuv420p10le),
YUV422Frame (YUYV / UYVY / YVYU, Y210, NV16 / P210, yuv422p) and YUV444Frame (yuv444p, NVDEC's 4:4:4 surfaces), in
BT.601, BT.709 or BT.2020, limited or full range, 8, 10 or 12 bits, converted to RGB inside the crop (8-bit BT.601
limited range exactly as cv2.cvtColor converts it), and V210Frame (SDI capture cards' packed 10-bit 4:2:2, unpacked
inside the crop); or raw Bayer mosaics as machine-vision and CSI-2 cameras send them: BayerFrame (RGGB / GRBG / GBRG /
BGGR at 8 to 16 bits, MIPI RAW10 / RAW12), demosaiced inside the crop exactly as cv2.cvtColor(COLOR_Bayer*2RGB)
demosaics them; or single-channel frames as mono cameras and thermal cores send them: MonoFrame (8 to 16 bits, MIPI
RAW10 / RAW12), mapped to grey inside the crop, optionally with per-frame min-max gain control (cv2.normalize
NORM_MINMAX); or RGB frames in any channel order and container: RGBFrame (OpenCV's BGR and BGRA, RGBA / ARGB / ABGR
and their X variants, 10-bit x2rgb10 / x2bgr10 words, 16-bit rgb48 / rgba64, planar gbrp at 8 to 16 bits), each tap's
channels fetched and mapped to 8 bits inside the crop.  Tensors, YUV planes, v210 surfaces, Bayer mosaics, mono frames
and RGB frames are read where they are, without a copy.  Any of them may be wrapped in Oriented(frame, rotate, mirror)
to track on the picture as it is shown (phone video's display rotation, cameras mounted upside down or mirrored):
rects and boxes are then in the turned picture's coordinates, and each display pixel is mapped to its stored pixel
inside the crop.

Every target behaves exactly like its own ``FEARTracker(gpu_crop=True)`` started on the same frame with the same
rect: the rect is clamped, the padding colour is the mean colour of the init frame, the template is the network
features of its 128 x 128 context crop, and each frame runs crop -> network -> decode -> rescale -> clamp.  Instead of
one batch-1 step and one host round trip per target, one step runs all N targets at batch N:

    fear_crop_targets_view_u8 (N search crops)  ->  fear_track_u8 (B = N, Bz = N)  ->  fear_advance_targets_view

on per-target state kept in device memory (an (N, 16) int32 tensor of FearTarget records, include/fear_b200.h), so the
step is captured once as a CUDA graph and replayed every frame.  The kernels find the frames through a table of
FearFrameView records (address, byte strides, H, W) in a fixed device buffer, written before every step: numpy frames
are packed into one pinned buffer and sent with one copy, and their views point into the packed device buffer; CUDA
tensors' views point at the tensors.  YUV420Frames go into a second fixed table of FearFrameYUV records (planes and colour
format), read by the *_yuv entry points; a call with any 4:2:2 or 4:4:4 frame puts all its frames into a third, of
FearFrameYCbCr records (the same plus the chroma subsampling), read by the *_ycbcr entry points; a call with any
V210Frame puts all its frames into a fourth, of FearFrameYCbCrV210 records (a FearFrameYCbCr or a v210 surface), read
by the *_ycbcr_v210 entry points; a call with any HDR frame (``transfer="pq"`` or ``"hlg"``) puts all its frames into
a sixth, of FearFrameYCbCrHDR records (a FearFrameYCbCrV210 and its transfer), read by the *_ycbcr_hdr entry points,
which tone-map HDR taps to SDR inside the crop.  BayerFrames go into a fifth, of FearFrameBayer records, read by the *_bayer entry
points; they cannot share a call with other kinds of frames.  MonoFrames go into a seventh, of FearFrameMono records,
read by the *_mono entry points, and cannot share a call with other kinds either; when any of a call's MonoFrames has
gain control, fear_frame_range_mono first writes each frame's code range into that table.  A call with any RGBFrame
puts all its frames, RGBFrames and CUDA tensors alike, into an eighth, of FearFrameRGB records, read by the *_rgb entry
points; RGBFrames cannot share a call with numpy arrays or YUV, Bayer or mono frames.  The host then reads back
the boxes and scores.  The launch count of a step depends neither on N nor on the kind of frames, with one exception:
a step on MonoFrames with gain control launches the range kernel too (49 launches instead of 48).  When any frame of a
call is Oriented, the call's F int32 orientation codes follow the records in the same table buffer and copy, and the
step runs fear_crop_targets_oriented_u8 / fear_advance_targets_oriented on the same table in place of its crop and
advance (the sums and the range kernel are unchanged: neither depends on orientation); the launch count is the same.

A step over the M targets of a mapping's streams runs on compact buffers of max_targets rows:

    fear_gather_targets -> [fear_frame_range_mono] -> crop (M) -> fear_track_u8 (B = M, Bz = M) -> advance (M)
                        -> fear_scatter_targets

The host writes the (target row, frame index) pair of each selected target into a fixed selection buffer, sent with the
frame table; gather copies those rows (frame replaced by the index) and their templates into the step buffers, and
scatter writes the new boxes and context boxes back.  The step is two launches longer than a list step whatever M is,
and is replayed from a small cache of captured graphs keyed by its shape, kept apart from the list step's graph.
"""
import math
import warnings
from collections import OrderedDict
from collections.abc import Mapping
from typing import Any, Dict, Optional, Sequence, Union

import numpy as np
import torch

from . import _lib, image_ops

_FRAME_ALIGN = 16  # byte alignment of each frame inside the packed buffer
_MAX_SIDE = 2 ** 31 - 1  # H and W are int32 in FearFrameView, FearFrameYUV and FearFrameYCbCr
_MAX_STREAM = 2 ** 31 - 1  # stream ids are int32 in FearTarget.frame
# Captured subset-step graphs kept per tracker.  A graph is keyed by the step's shape (step rows, frame count, table),
# not by which streams are in it, so a steady pattern of subsets uses one or two keys; 8 covers patterns whose subset
# sizes keep changing, and each graph holds little device memory (its box output; the network's workspace is shared).
SUBSET_GRAPHS = 8
# the entry points that read each frame table: frame sums, target crops, box advance
ENTRY_POINTS = {
    "views": ("fear_frame_sums_u8", "fear_crop_targets_view_u8", "fear_advance_targets_view"),
    "yuv": ("fear_frame_sums_yuv_u8", "fear_crop_targets_yuv_u8", "fear_advance_targets_yuv"),
    "ycbcr": ("fear_frame_sums_ycbcr_u8", "fear_crop_targets_ycbcr_u8", "fear_advance_targets_ycbcr"),
    "ycbcr_v210": ("fear_frame_sums_ycbcr_v210_u8", "fear_crop_targets_ycbcr_v210_u8",
                   "fear_advance_targets_ycbcr_v210"),
    "ycbcr_hdr": ("fear_frame_sums_ycbcr_hdr_u8", "fear_crop_targets_ycbcr_hdr_u8", "fear_advance_targets_ycbcr_hdr"),
    "bayer": ("fear_frame_sums_bayer_u8", "fear_crop_targets_bayer_u8", "fear_advance_targets_bayer"),
    "mono": ("fear_frame_sums_mono_u8", "fear_crop_targets_mono_u8", "fear_advance_targets_mono"),
    "rgb": ("fear_frame_sums_rgb_u8", "fear_crop_targets_rgb_u8", "fear_advance_targets_rgb"),
}
TABLE_DTYPES = {"views": _lib.VIEW_DTYPE, "yuv": _lib.YUV_DTYPE, "ycbcr": _lib.YCBCR_DTYPE,
                "ycbcr_v210": _lib.YCBCR_V210_DTYPE, "ycbcr_hdr": _lib.YCBCR_HDR_DTYPE, "bayer": _lib.BAYER_DTYPE,
                "mono": _lib.MONO_DTYPE, "rgb": _lib.RGB_DTYPE}
# the entry point that writes each frame's code range into a FearFrameMono table, for min-max gain control
RANGE_ENTRY_POINT = "fear_frame_range_mono"
# the crop and advance of any table on rotated and mirrored frames (Oriented), with the table named by
# _lib.ORIENT_TABLES and the call's orientation codes; the sums and the range do not depend on orientation
ORIENTED_ENTRY_POINTS = ("fear_crop_targets_oriented_u8", "fear_advance_targets_oriented")


def frame_view(frame: torch.Tensor) -> tuple:
    """The FearFrameView record (data, row_stride, pixel_stride, channel_stride, H, W) of a uint8 (H, W, 3) tensor, as
    it lies in memory: the address of pixel (0, 0) channel R and the byte strides (a uint8 stride is a byte stride)."""
    rs, ps, cs = frame.stride()
    return (frame.data_ptr(), rs, ps, cs, frame.shape[0], frame.shape[1])


class _YUVFrame:
    """What YUV420Frame, YUV422Frame and YUV444Frame share: three planes on the device, a colour format, the checks of
    both, and the FearFrameYCbCr record.  ``CHROMA_SHIFT`` (x, y) is the subsampling: chroma sample
    (r >> y, c >> x) belongs to pixel (r, c)."""
    CHROMA_SHIFT = (1, 1)
    _NAME = "4:2:0"
    _SIZES = "H and W even and >= 2"  # the luma sizes the subsampling allows, for error messages

    def __init__(self, y: torch.Tensor, u: torch.Tensor, v: torch.Tensor, *, matrix: str = "bt601",
                 full_range: bool = False, bits: int = 8, msb: bool = False, transfer: Optional[str] = None) -> None:
        cls = type(self).__name__
        self._check_format(matrix, full_range, bits, msb, transfer)
        dtype = self._dtype(bits)
        for name, p in (("y", y), ("u", u), ("v", v)):
            if not isinstance(p, torch.Tensor) or p.dtype != dtype or p.ndim != 2:
                what = f"{p.dtype} {tuple(p.shape)}" if isinstance(p, torch.Tensor) else type(p).__name__
                raise ValueError(f"{cls} plane {name} must be a 2-D {dtype} tensor at {bits} bits, got {what}")
            if min(p.stride()) < 0:
                raise ValueError(f"{cls} plane {name} has a negative stride {p.stride()}")
        h, w = y.shape
        sx, sy = self.CHROMA_SHIFT
        if not (1 << sy <= h <= _MAX_SIDE and 1 << sx <= w <= _MAX_SIDE) or h % (1 << sy) or w % (1 << sx):
            raise ValueError(f"YUV {self._NAME} luma must be (H, W) with {self._SIZES}, got {tuple(y.shape)}")
        ch, cw = h >> sy, w >> sx
        if tuple(u.shape) != (ch, cw) or tuple(v.shape) != (ch, cw):
            raise ValueError(f"YUV {self._NAME} chroma planes must be ({ch}, {cw}) for luma ({h}, {w}), got "
                             f"{tuple(u.shape)} and {tuple(v.shape)}")
        if u.stride() != v.stride():
            raise ValueError(f"{cls} u and v planes must share their strides, got {u.stride()} and {v.stride()}")
        self.y, self.u, self.v = y, u, v
        self.shape = (h, w, 3)
        self.matrix, self.full_range, self.bits = matrix, bool(full_range), int(bits)
        self.shift = 16 - self.bits if msb else 0
        self.transfer = transfer

    @classmethod
    def _check_format(cls, matrix, full_range, bits, msb, transfer=None) -> None:
        if matrix not in image_ops.YUV_MATRICES:
            raise ValueError(f"{cls.__name__} matrix must be one of {sorted(image_ops.YUV_MATRICES)}, got {matrix!r}")
        if isinstance(bits, bool) or bits not in (8, 10, 12):
            raise ValueError(f"{cls.__name__} bits must be 8, 10 or 12, got {bits!r}")
        if bits == 8 and msb:
            raise ValueError(f"{cls.__name__} msb applies to 10- and 12-bit samples, not 8-bit ones")
        image_ops.check_transfer(transfer, matrix, bits, f"{cls.__name__} transfer")

    @staticmethod
    def _dtype(bits: int) -> torch.dtype:
        return torch.uint8 if bits == 8 else torch.uint16

    @classmethod
    def _surface(cls, t, layout: str, bits: int, rows: int, cols: int, what: str) -> None:
        """Check that ``t`` is a 2-D tensor of the bit depth's sample type whose sides divide by ``rows``, ``cols``."""
        dtype = cls._dtype(bits)
        if not isinstance(t, torch.Tensor) or t.dtype != dtype or t.ndim != 2 or t.shape[0] % rows or t.shape[1] % cols:
            got = f"{t.dtype} {tuple(t.shape)}" if isinstance(t, torch.Tensor) else type(t).__name__
            raise ValueError(f"{cls.__name__}.{layout} takes a {dtype} {what} at {bits} bits, got {got}")

    @property
    def default_format(self) -> bool:
        """Whether the frame is 8-bit BT.601 limited range, the format FearFrameYUV420 records describe."""
        return self.matrix == "bt601" and not self.full_range and self.bits == 8

    def ycbcr_record(self) -> tuple:
        """The FearFrameYCbCr record (y, u, v, y_row_stride, y_pixel_stride, uv_row_stride, uv_pixel_stride, H, W,
        matrix, full_range, bits, shift, chroma_shift_x, chroma_shift_y): the addresses of luma sample (0, 0) and of
        the Cb and Cr samples (0, 0), byte strides (element strides times the sample size), the format, then the
        subsampling."""
        es = self.y.element_size()
        (yrs, yps), (uvrs, uvps) = self.y.stride(), self.u.stride()
        return (self.y.data_ptr(), self.u.data_ptr(), self.v.data_ptr(), yrs * es, yps * es, uvrs * es, uvps * es,
                *self.shape[:2], image_ops.YUV_MATRICES[self.matrix][0], int(self.full_range), self.bits, self.shift,
                *self.CHROMA_SHIFT)

    def ycbcr_v210_record(self) -> tuple:
        """The FearFrameYCbCrV210 record of a planar frame: ``ycbcr_record``, then v210 = 0 and the reserved 0."""
        return self.ycbcr_record() + (0, 0)

    def hdr_record(self) -> tuple:
        """The FearFrameYCbCrHDR record: ``ycbcr_v210_record``, then the H.273 transfer code (0 without a transfer,
        16 for "pq", 18 for "hlg") and the reserved 0."""
        return self.ycbcr_v210_record() + (image_ops.HDR_TRANSFERS.get(self.transfer, 0), 0)


class YUV420Frame(_YUVFrame):
    """A YUV 4:2:0 frame as a video decoder writes it: a luma plane ``y`` (H, W) and chroma planes ``u`` (Cb) and
    ``v`` (Cr) of (H/2, W/2), with H and W even.  Pixel (r, c) takes its chroma from sample (r // 2, c // 2).  The
    planes are tensors or views with any non-negative strides, and ``u`` and ``v`` share their strides.
    FEARMultiTracker reads the planes where they are and converts every pixel it reads, so no RGB copy of the frame is
    made.

    The colour format:
        matrix       "bt601" (Kr, Kb = 0.299, 0.114), "bt709" (0.2126, 0.0722; HD H.264 / HEVC) or "bt2020"
                     (0.2627, 0.0593, non-constant luminance; HDR / 10-bit content)
        full_range   False: limited range (Y in [16, 235] * 2^(bits-8)); True: full range (MJPEG's yuvj420p)
        bits         8: uint8 planes; 10 or 12: torch.uint16 planes (view byte surfaces as ``t.view(torch.uint16)``)
        msb          at 10 / 12 bits, whether samples sit in the high bits of their uint16 (P010 / P016) rather than
                     the low bits (yuv420p10le / yuv420p12le)
    The default (bt601, limited, 8 bits) is converted exactly as ``cv2.cvtColor(frame, cv2.COLOR_YUV2RGB_NV12 /
    COLOR_YUV2RGB_I420)`` converts it; every other format by the ITU-T H.273 inverse in float64 (include/fear_b200.h,
    FearFrameYUV).  ``image_ops.yuv420_to_rgb`` restates both in numpy: it gives the RGB frame the tracker sees.
    NV21 / YV12 are ``YUV420Frame(y, u, v)`` with the planes in the right order.

        transfer     None: the matrix only (SDR); "pq" or "hlg": HDR video (BT.2100 PQ as Android phones and HDR10
                     streams record it, HLG as iPhones and UHD broadcast do), BT.2020 at 10 / 12 bits only, tone-mapped
                     to SDR BT.709 inside the crop by ITU-R BT.2446-1 Method A at a 1000 cd/m² peak
                     (``image_ops.yuv_to_rgb(..., transfer=...)``, include/fear_b200.h FearFrameYCbCrHDR)

        YUV420Frame.nv12(t)    t (3H/2, W): H luma rows, then H/2 rows of interleaved (U, V) pairs; the rows may be
                               pitched (t = surface[:, :W]), as NVDEC and cv2 lay out NV12; at 10 / 12 bits a uint16
                               P010 / P016 surface (MSB-aligned)
        YUV420Frame.i420(t)    t contiguous (3H/2, W): the Y, U and V planes one after another (cv2's I420, ffmpeg's
                               yuv420p); at 10 / 12 bits uint16 yuv420p10le / yuv420p12le (LSB-aligned)
        YUV420Frame(y, u, v)   separate planes, regions of interest at even offsets

    ``shape`` is (H, W, 3), the shape of the RGB frame it stands for.  The constructors raise ValueError on a malformed
    frame or format; they do not look at the device (the tracker checks that).  YUV422Frame and YUV444Frame take the
    same colour formats and transfers."""

    @classmethod
    def nv12(cls, t: torch.Tensor, *, matrix: str = "bt601", full_range: bool = False, bits: int = 8,
             transfer: Optional[str] = None) -> "YUV420Frame":
        cls._check_format(matrix, full_range, bits, False, transfer)
        h = cls._luma_rows(t, "nv12", bits)
        uv = t[h:]
        return cls(t[:h], uv[:, 0::2], uv[:, 1::2], matrix=matrix, full_range=full_range, bits=bits, msb=bits > 8,
                   transfer=transfer)

    @classmethod
    def i420(cls, t: torch.Tensor, *, matrix: str = "bt601", full_range: bool = False, bits: int = 8,
             transfer: Optional[str] = None) -> "YUV420Frame":
        cls._check_format(matrix, full_range, bits, False, transfer)
        h, w = cls._luma_rows(t, "i420", bits), t.shape[1]
        if not t.is_contiguous():
            raise ValueError(f"YUV420Frame.i420 takes a contiguous tensor, got strides {t.stride()}")
        flat, luma, quarter = t.reshape(-1), h * w, h * w // 4
        return cls(flat[:luma].view(h, w), flat[luma:luma + quarter].view(h // 2, w // 2),
                   flat[luma + quarter:].view(h // 2, w // 2), matrix=matrix, full_range=full_range, bits=bits,
                   transfer=transfer)

    @classmethod
    def _luma_rows(cls, t, layout: str, bits: int = 8) -> int:
        cls._surface(t, layout, bits, 3, 2, "(3H/2, W) tensor with H and W even")
        return 2 * t.shape[0] // 3

    def record(self) -> tuple:
        """The FearFrameYUV420 record (y, u, v, y_row_stride, y_pixel_stride, uv_row_stride, uv_pixel_stride, H, W):
        the addresses of luma sample (0, 0) and of the Cb and Cr samples (0, 0), and the byte strides (a uint8 stride
        is a byte stride).  Only for the default format (8-bit BT.601 limited range); ``yuv_record`` describes any."""
        if not self.default_format:
            raise ValueError(f"a FearFrameYUV420 record describes 8-bit BT.601 limited range only, not this "
                             f"{self.matrix} {'full' if self.full_range else 'limited'} range {self.bits}-bit frame: "
                             "use yuv_record()")
        return self.yuv_record()[:9]

    def yuv_record(self) -> tuple:
        """The FearFrameYUV record (y, u, v, y_row_stride, y_pixel_stride, uv_row_stride, uv_pixel_stride, H, W,
        matrix, full_range, bits, shift): the FearFrameYUV420 fields, with byte strides (element strides times the
        sample size), then the format.  ``ycbcr_record`` adds the chroma shifts (1, 1)."""
        return self.ycbcr_record()[:13]


class YUV422Frame(_YUVFrame):
    """A YUV 4:2:2 frame: a luma plane ``y`` (H, W) and chroma planes ``u`` (Cb) and ``v`` (Cr) of (H, W/2), W even
    (H may be odd).  Pixel (r, c) takes its chroma from sample (r, c // 2).  Planes, strides and the colour format
    (matrix, full_range, bits, msb) are as for YUV420Frame; ``image_ops.yuv_to_rgb(..., chroma_shift=(1, 0))`` gives
    the RGB frame the tracker sees (for the default format, ``cv2.cvtColor(yuyv, cv2.COLOR_YUV2RGB_YUY2)``).

        YUV422Frame.yuyv(t)    t (H, 2W): each row Y0 U Y1 V ... (YUY2, what UVC webcams send); rows may be pitched;
                               at 10 / 12 bits a uint16 Y210 / Y212 / Y216 surface (MSB-aligned)
        YUV422Frame.uyvy(t)    t (H, 2W): each row U Y0 V Y1 ... (capture cards), as yuyv otherwise
        YUV422Frame.yvyu(t)    t (H, 2W): each row Y0 V Y1 U ..., as yuyv otherwise
        YUV422Frame.nv16(t)    t (2H, W): H luma rows, then H rows of interleaved (U, V) pairs; rows may be pitched;
                               at 10 / 12 bits a uint16 P210 / P216 surface (MSB-aligned)
        YUV422Frame.i422(t)    t contiguous (2H, W): the Y, U and V planes one after another (ffmpeg's yuv422p); at
                               10 / 12 bits uint16 yuv422p10le / yuv422p12le (LSB-aligned)
        YUV422Frame(y, u, v)   separate planes, regions of interest at even column offsets"""
    CHROMA_SHIFT = (1, 0)
    _NAME = "4:2:2"
    _SIZES = "W even and >= 2, H >= 1"

    @classmethod
    def _packed(cls, t, layout: str, order: tuple, matrix, full_range, bits, transfer) -> "YUV422Frame":
        cls._check_format(matrix, full_range, bits, False, transfer)
        cls._surface(t, layout, bits, 1, 4, "(H, 2W) tensor with W even")
        y0, u0, v0 = order  # sample offsets of Y0, U and V in each 4-sample group
        return cls(t[:, y0::2], t[:, u0::4], t[:, v0::4], matrix=matrix, full_range=full_range, bits=bits,
                   msb=bits > 8, transfer=transfer)

    @classmethod
    def yuyv(cls, t: torch.Tensor, *, matrix: str = "bt601", full_range: bool = False, bits: int = 8,
             transfer: Optional[str] = None) -> "YUV422Frame":
        return cls._packed(t, "yuyv", (0, 1, 3), matrix, full_range, bits, transfer)

    @classmethod
    def uyvy(cls, t: torch.Tensor, *, matrix: str = "bt601", full_range: bool = False, bits: int = 8,
             transfer: Optional[str] = None) -> "YUV422Frame":
        return cls._packed(t, "uyvy", (1, 0, 2), matrix, full_range, bits, transfer)

    @classmethod
    def yvyu(cls, t: torch.Tensor, *, matrix: str = "bt601", full_range: bool = False, bits: int = 8,
             transfer: Optional[str] = None) -> "YUV422Frame":
        return cls._packed(t, "yvyu", (0, 3, 1), matrix, full_range, bits, transfer)

    @classmethod
    def nv16(cls, t: torch.Tensor, *, matrix: str = "bt601", full_range: bool = False, bits: int = 8,
             transfer: Optional[str] = None) -> "YUV422Frame":
        cls._check_format(matrix, full_range, bits, False, transfer)
        cls._surface(t, "nv16", bits, 2, 2, "(2H, W) tensor with W even")
        h = t.shape[0] // 2
        uv = t[h:]
        return cls(t[:h], uv[:, 0::2], uv[:, 1::2], matrix=matrix, full_range=full_range, bits=bits, msb=bits > 8,
                   transfer=transfer)

    @classmethod
    def i422(cls, t: torch.Tensor, *, matrix: str = "bt601", full_range: bool = False, bits: int = 8,
             transfer: Optional[str] = None) -> "YUV422Frame":
        cls._check_format(matrix, full_range, bits, False, transfer)
        cls._surface(t, "i422", bits, 2, 2, "(2H, W) tensor with W even")
        if not t.is_contiguous():
            raise ValueError(f"YUV422Frame.i422 takes a contiguous tensor, got strides {t.stride()}")
        h, w = t.shape[0] // 2, t.shape[1]
        flat, luma, half = t.reshape(-1), h * w, h * w // 2
        return cls(flat[:luma].view(h, w), flat[luma:luma + half].view(h, w // 2), flat[luma + half:].view(h, w // 2),
                   matrix=matrix, full_range=full_range, bits=bits, transfer=transfer)


class YUV444Frame(_YUVFrame):
    """A YUV 4:4:4 frame: luma ``y``, chroma ``u`` (Cb) and ``v`` (Cr), three planes of the same shape (H, W), any
    size.  Planes, strides and the colour format (matrix, full_range, bits, msb) are as for YUV420Frame;
    ``image_ops.yuv_to_rgb(..., chroma_shift=(0, 0))`` gives the RGB frame the tracker sees.  Packed 4:4:4 layouts
    (AYUV, Y410, Y416) are ``YUV444Frame(y, u, v)`` of strided views.

        YUV444Frame.i444(t)    t (3H, W): the Y, U and V planes one after another, rows may be pitched (ffmpeg's
                               yuv444p, NVDEC's YUV444 surfaces); at 10 / 12 bits uint16, LSB-aligned
                               (yuv444p10le) unless ``msb=True`` (NVDEC's YUV444_16Bit surfaces)
        YUV444Frame(y, u, v)   separate planes, regions of interest at any offset"""
    CHROMA_SHIFT = (0, 0)
    _NAME = "4:4:4"
    _SIZES = "H, W >= 1"

    @classmethod
    def i444(cls, t: torch.Tensor, *, msb: bool = False, matrix: str = "bt601", full_range: bool = False,
             bits: int = 8, transfer: Optional[str] = None) -> "YUV444Frame":
        cls._check_format(matrix, full_range, bits, msb, transfer)
        cls._surface(t, "i444", bits, 3, 1, "(3H, W) tensor")
        h = t.shape[0] // 3
        return cls(t[:h], t[h:2 * h], t[2 * h:], matrix=matrix, full_range=full_range, bits=bits, msb=msb,
                   transfer=transfer)


class V210Frame:
    """A v210 frame (10-bit 4:2:2 packed three codes to a 32-bit word) as SDI capture cards (Blackmagic DeckLink's
    ``bmdFormat10BitYUV``, AJA, Magewell), ffmpeg's v210 decoder and QuickTime uncompressed 10-bit write it.  ``t`` is
    the capture buffer as bytes: a CUDA uint8 (H, row bytes) tensor whose rows are contiguous, any row pitch (a view
    ``surface[:, :n]`` of a pitched surface is fine); ``width`` is the picture width W (even).  A row needs
    ``16 * ceil(W / 6)`` bytes; capture cards pitch rows to ``128 * ceil(W / 48)``.  The buffer address and the row pitch
    must be multiples of 4 bytes.  ``matrix``, ``full_range`` and ``transfer`` are those of YUV420Frame; the depth is 10
    bits (``transfer`` "pq" or "hlg" with ``matrix="bt2020"`` reads 10-bit HLG or PQ from SDI: the tracker sees
    ``image_ops.yuv_to_rgb(..., bits=10, chroma_shift=(1, 0), transfer=...)`` of the unpacked planes).

    FEARMultiTracker and FEARTracker read the words where they are and unpack and convert every pixel they read, so no
    planes and no RGB copy are made: the RGB frame the tracker sees is ``image_ops.yuv_to_rgb(*image_ops.v210_unpack(
    rows, W), matrix, full_range, bits=10, chroma_shift=(1, 0))`` of the same bytes.  The constructor raises ValueError
    on a malformed buffer or format.  ``shape`` is (H, W, 3)."""
    CHROMA_SHIFT = (1, 0)
    bits = 10

    def __init__(self, t: torch.Tensor, width: int, *, matrix: str = "bt601", full_range: bool = False,
                 transfer: Optional[str] = None) -> None:
        if matrix not in image_ops.YUV_MATRICES:
            raise ValueError(f"V210Frame matrix must be one of {sorted(image_ops.YUV_MATRICES)}, got {matrix!r}")
        image_ops.check_transfer(transfer, matrix, self.bits, "V210Frame transfer")
        if not isinstance(t, torch.Tensor) or t.dtype != torch.uint8 or t.ndim != 2 or t.device.type != "cuda":
            what = f"{t.dtype} {tuple(t.shape)} on {t.device}" if isinstance(t, torch.Tensor) else type(t).__name__
            raise ValueError(f"V210Frame takes a 2-D CUDA uint8 (H, row bytes) tensor, got {what}")
        if isinstance(width, bool) or not isinstance(width, (int, np.integer)) or not (2 <= width <= _MAX_SIDE) \
                or width % 2:
            raise ValueError(f"V210Frame width must be an even int in [2, {_MAX_SIDE}], got {width!r}")
        h, need = t.shape[0], image_ops.v210_row_bytes(width)
        if not 1 <= h <= _MAX_SIDE:
            raise ValueError(f"V210Frame needs 1 to {_MAX_SIDE} rows, got {h}")
        if t.shape[1] < need:
            raise ValueError(f"a v210 row of {width} pixels needs {need} bytes, the tensor's rows have {t.shape[1]}")
        pitch = t.stride(0) if h > 1 else need  # one row: the pitch is never stepped
        if t.stride(1) != 1 or pitch < need:
            raise ValueError(f"V210Frame rows must be contiguous bytes at a pitch >= {need}, got strides {t.stride()}")
        if pitch % 4 or t.data_ptr() % 4:
            raise ValueError(f"V210Frame rows must start on 4-byte boundaries: pitch {pitch}, address offset "
                             f"{t.data_ptr() % 4}")
        self.t, self.width, self.pitch = t, int(width), int(pitch)
        self.shape = (h, self.width, 3)
        self.matrix, self.full_range = matrix, bool(full_range)
        self.transfer = transfer

    def ycbcr_v210_record(self) -> tuple:
        """The FearFrameYCbCrV210 record (y, u, v, y_row_stride, y_pixel_stride, uv_row_stride, uv_pixel_stride, H, W,
        matrix, full_range, bits, shift, chroma_shift_x, chroma_shift_y, v210, reserved) of the surface: its address and
        row pitch, the size and format, v210 = 1; the fields a v210 entry does not read are 0."""
        return (self.t.data_ptr(), 0, 0, self.pitch, 0, 0, 0, *self.shape[:2], image_ops.YUV_MATRICES[self.matrix][0],
                int(self.full_range), self.bits, 0, *self.CHROMA_SHIFT, 1, 0)

    def hdr_record(self) -> tuple:
        """The FearFrameYCbCrHDR record: ``ycbcr_v210_record``, then the H.273 transfer code (0, 16 for "pq", 18 for
        "hlg") and the reserved 0."""
        return self.ycbcr_v210_record() + (image_ops.HDR_TRANSFERS.get(self.transfer, 0), 0)


class _RawFrame:
    """What BayerFrame and MonoFrame share: a CUDA (H, W) tensor of unpacked samples, or an (H, row bytes) uint8 tensor
    of MIPI CSI-2 RAW10 / RAW12 rows, with its checks and row pitch.  ``_MIN_SIDE`` is the smallest H and W the kernels
    read and ``_SIZE_MSG`` names the frame in the size refusal."""
    _MIN_SIDE = 1
    _SIZE_MSG = "a frame needs at least 1 row and 1 column"

    @classmethod
    def _check_depth(cls, bits, msb) -> torch.dtype:
        if isinstance(bits, bool) or bits not in (8, 10, 12, 14, 16):
            raise ValueError(f"{cls.__name__} bits must be 8, 10, 12, 14 or 16, got {bits!r}")
        if bits == 8 and msb:
            raise ValueError(f"{cls.__name__} msb applies to samples wider than 8 bits, not 8-bit ones")
        return torch.uint8 if bits == 8 else torch.uint16

    @classmethod
    def _check_tensor(cls, t, dtype: torch.dtype, what: str) -> None:
        if not isinstance(t, torch.Tensor) or t.dtype != dtype or t.ndim != 2 or t.device.type != "cuda":
            got = f"{t.dtype} {tuple(t.shape)} on {t.device}" if isinstance(t, torch.Tensor) else type(t).__name__
            raise ValueError(f"{cls.__name__} takes a 2-D CUDA {dtype} {what}, got {got}")
        m = cls._MIN_SIDE
        if not (m <= t.shape[0] <= _MAX_SIDE and m <= t.shape[1] <= _MAX_SIDE):
            raise ValueError(f"{cls._SIZE_MSG}, got {tuple(t.shape)}")

    @classmethod
    def _check_packed(cls, t, width, bits: int) -> int:
        """The row bytes of RAW``bits`` rows of ``width`` pixels, after checking ``t`` and ``width``."""
        cls._check_tensor(t, torch.uint8, f"(H, row bytes) tensor of RAW{bits} rows")
        m = cls._MIN_SIDE
        if isinstance(width, bool) or not isinstance(width, (int, np.integer)) or not (m <= width <= _MAX_SIDE):
            raise ValueError(f"{cls.__name__} width must be an int in [{m}, {_MAX_SIDE}], got {width!r}")
        need = image_ops.mipi_row_bytes(width, bits)
        if t.shape[1] < need:
            raise ValueError(f"a RAW{bits} row of {width} pixels needs {need} bytes, the tensor's rows have "
                             f"{t.shape[1]}")
        return need

    def _init(self, t: torch.Tensor, bits: int, shift: int, packing: int, width: int, row_bytes: int) -> None:
        name = type(self).__name__
        es = t.element_size()
        pitch = t.stride(0) * es
        if t.stride(1) != 1 or pitch < row_bytes:
            raise ValueError(f"{name} rows must be contiguous samples at a pitch of at least {row_bytes} bytes, "
                             f"got strides {t.stride()}")
        if es == 2 and (pitch % 2 or t.data_ptr() % 2):
            raise ValueError(f"{name} uint16 rows must start on 2-byte boundaries: pitch {pitch}, address offset "
                             f"{t.data_ptr() % 2}")
        self.t, self.bits, self.shift, self.packing = t, bits, shift, packing
        self.pitch = int(pitch)
        self.shape = (t.shape[0], width, 3)


class BayerFrame(_RawFrame):
    """A raw Bayer mosaic as machine-vision cameras (GigE Vision / USB3 Vision PFNC ``BayerRG8``, ``BayerGR12`` ...),
    CSI-2 sensors under V4L2 or libcamera (``SRGGB10P`` / ``SRGGB12P``) and raw recorders deliver it.  ``pattern`` is
    the colours of the 2 x 2 block at pixel (0, 0), row by row: "RGGB", "GRBG", "GBRG" or "BGGR" (OpenCV 4.x's
    ``COLOR_Bayer{pattern}2RGB``; a region of interest at an odd offset names its own pattern).

        BayerFrame(t, pattern, bits=8, msb=False)   t a CUDA (H, W) tensor: uint8 at 8 bits, torch.uint16 at 10, 12,
                                                    14 or 16 bits, the code in the low bits (``msb=False``) or the
                                                    high bits (``msb=True``) of each sample; any row stride, column
                                                    stride 1 (a view ``surface[:, :W]`` of a pitched surface is fine)
        BayerFrame.raw10(t, width, pattern)         t a CUDA uint8 (H, row bytes) tensor of MIPI CSI-2 RAW10 rows
        BayerFrame.raw12(t, width, pattern)         t a CUDA uint8 (H, row bytes) tensor of MIPI CSI-2 RAW12 rows

    H and W must be at least 3.  FEARMultiTracker and FEARTracker read the samples where they are and demosaic every
    pixel they read, so no RGB copy is made: the RGB frame the tracker sees is ``image_ops.bayer_to_rgb(codes,
    pattern, bits)`` of the frame's codes (``image_ops.mipi_unpack`` for packed rows), which is ``cv2.cvtColor(raw,
    cv2.COLOR_Bayer{pattern}2RGB)`` at 8 bits.  The constructors raise ValueError on a malformed tensor or format.
    ``shape`` is (H, W, 3)."""
    _MIN_SIDE = 3
    _SIZE_MSG = "a Bayer mosaic needs at least 3 rows and 3 columns"

    def __init__(self, t: torch.Tensor, pattern: str = "RGGB", bits: int = 8, msb: bool = False) -> None:
        self._check_pattern(pattern)
        dtype = self._check_depth(bits, msb)
        self._check_tensor(t, dtype, f"(H, W) tensor at {bits} bits")
        self._init(t, int(bits), 16 - int(bits) if msb else 0, 0, t.shape[1], t.shape[1] * t.element_size())
        self.pattern = pattern

    @classmethod
    def raw10(cls, t: torch.Tensor, width: int, pattern: str = "RGGB") -> "BayerFrame":
        return cls._packed(t, width, pattern, 10, 1)

    @classmethod
    def raw12(cls, t: torch.Tensor, width: int, pattern: str = "RGGB") -> "BayerFrame":
        return cls._packed(t, width, pattern, 12, 2)

    @classmethod
    def _packed(cls, t, width, pattern, bits: int, packing: int) -> "BayerFrame":
        cls._check_pattern(pattern)
        need = cls._check_packed(t, width, bits)
        f = cls.__new__(cls)
        f._init(t, bits, 0, packing, int(width), need)
        f.pattern = pattern
        return f

    @staticmethod
    def _check_pattern(pattern) -> None:
        if pattern not in image_ops.BAYER_PATTERNS:
            raise ValueError(f"BayerFrame pattern must be one of {sorted(image_ops.BAYER_PATTERNS)}, got {pattern!r}")

    def bayer_record(self) -> tuple:
        """The FearFrameBayer record (data, row_stride, H, W, pattern, bits, shift, packing): the address of sample
        (0, 0) (packed: of row 0's first byte), the row pitch in bytes, the size and the format."""
        return (self.t.data_ptr(), self.pitch, *self.shape[:2], image_ops.BAYER_PATTERNS[self.pattern], self.bits,
                self.shift, self.packing)


class MonoFrame(_RawFrame):
    """A single-channel frame as mono machine-vision cameras (GigE Vision / USB3 Vision PFNC ``Mono8``, ``Mono10``,
    ``Mono12``, ``Mono16``), mono CSI-2 sensors under V4L2 (``GREY``, ``Y10``, ``Y12``, ``Y16``, ``Y10P``, ``Y12P``)
    and thermal cores (14- or 16-bit ``Y16``) deliver it.

        MonoFrame(t, bits=8, msb=False, agc=None)   t a CUDA (H, W) tensor: uint8 at 8 bits, torch.uint16 at 10, 12,
                                                    14 or 16 bits, the code in the low bits (``msb=False``) or the
                                                    high bits (``msb=True``) of each sample; any row stride, column
                                                    stride 1 (a view ``surface[:, :W]`` of a pitched surface is fine)
        MonoFrame.raw10(t, width, agc=None)         t a CUDA uint8 (H, row bytes) tensor of MIPI CSI-2 RAW10 rows (Y10P)
        MonoFrame.raw12(t, width, agc=None)         t a CUDA uint8 (H, row bytes) tensor of MIPI CSI-2 RAW12 rows (Y12P)

    ``agc`` is the gain control: None maps each code to 8 bits as a BayerFrame channel is mapped; ``"minmax"`` stretches
    the frame's own code range to [0, 255] as ``cv2.normalize(codes, None, 0, 255, cv2.NORM_MINMAX, cv2.CV_8U)`` does,
    which a thermal core's narrow band of codes needs.  FEARMultiTracker and FEARTracker read the samples where they are
    (with ``agc`` they first find the frame's range with one pass over it) and map every pixel they read to grey, so no
    RGB copy is made: the RGB frame the tracker sees is ``image_ops.mono_to_rgb(codes, bits, agc)`` of the frame's codes
    (``image_ops.mipi_unpack`` for packed rows).  The constructors raise ValueError on a malformed tensor or format.
    ``shape`` is (H, W, 3)."""
    _SIZE_MSG = "a mono frame needs at least 1 row and 1 column"

    def __init__(self, t: torch.Tensor, bits: int = 8, msb: bool = False, agc: Optional[str] = None) -> None:
        image_ops.check_agc(agc, "MonoFrame agc")
        dtype = self._check_depth(bits, msb)
        self._check_tensor(t, dtype, f"(H, W) tensor at {bits} bits")
        self._init(t, int(bits), 16 - int(bits) if msb else 0, 0, t.shape[1], t.shape[1] * t.element_size())
        self.agc = agc

    @classmethod
    def raw10(cls, t: torch.Tensor, width: int, agc: Optional[str] = None) -> "MonoFrame":
        return cls._packed(t, width, agc, 10, 1)

    @classmethod
    def raw12(cls, t: torch.Tensor, width: int, agc: Optional[str] = None) -> "MonoFrame":
        return cls._packed(t, width, agc, 12, 2)

    @classmethod
    def _packed(cls, t, width, agc, bits: int, packing: int) -> "MonoFrame":
        image_ops.check_agc(agc, "MonoFrame agc")
        need = cls._check_packed(t, width, bits)
        f = cls.__new__(cls)
        f._init(t, bits, 0, packing, int(width), need)
        f.agc = agc
        return f

    def mono_record(self) -> tuple:
        """The FearFrameMono record (data, row_stride, H, W, bits, shift, packing, agc, lo, hi): the address of sample
        (0, 0) (packed: of row 0's first byte), the row pitch in bytes, the size, the format and the gain control, then
        the empty range lo = INT32_MAX, hi = INT32_MIN that fear_frame_range_mono narrows to the frame's."""
        return (self.t.data_ptr(), self.pitch, *self.shape[:2], self.bits, self.shift, self.packing,
                image_ops.AGC_MODES[self.agc], 2 ** 31 - 1, -2 ** 31)


def _unstepped(t: torch.Tensor, *fixed) -> tuple:
    """``t``'s element strides, with the stride of each dimension of size 1 (never stepped, so torch may report any
    value) replaced by ``fixed[d]`` when given."""
    return tuple(f if n == 1 and f is not None else s for n, s, f in zip(t.shape, t.stride(), fixed))


class RGBFrame:
    """An RGB frame in device memory in any channel order and container, read where it is, as OpenCV and capture
    APIs hand it over.  Layout names are ffmpeg ``pix_fmt`` names:

        RGBFrame(t, layout)                 t a CUDA tensor whose rows may be pitched (any row stride >= W * C, a view
                                            ``surface[:, :W]`` is fine), channel stride 1, pixel stride C:
            uint8 (H, W, 3)                 "rgb24", "bgr24" (OpenCV's BGR)
            uint8 (H, W, 4)                 "rgba", "bgra", "argb", "abgr", "rgb0", "bgr0", "0rgb", "0bgr"
                                            (cv2.cudacodec's BGRA, DeckLink bmdFormat8BitBGRA, desktop duplication)
            torch.uint16 (H, W, 3 | 4)      "rgb48le", "bgr48le", "rgba64le", "bgra64le" (ProRes 4444, 16-bit PNG / TIFF)
            torch.int32 / torch.uint32      "x2rgb10le" (B in bits 0-9, G 10-19, R 20-29; DRM XRGB2101010), "x2bgr10le"
            (H, W), column stride 1         (R 0-9, G 10-19, B 20-29; DXGI R10G10B10A2_UNORM)
        RGBFrame.planar(r, g, b, bits=8)    three CUDA (H, W) planes of one shape, dtype and strides: uint8 at 8 bits,
                                            torch.uint16 with the code in the low bits at 10, 12 or 16; ffmpeg's gbrp*
                                            is ``planar(data[2], data[0], data[1], bits)`` and a (3, H, W) uint16
                                            tensor from torchvision's decode_png is ``planar(*t, bits=16)``

    Alpha and X samples and the spare bits of a word are never read.  Codes above 8 bits are mapped to 8 bits as a
    BayerFrame channel is, full range.  FEARMultiTracker and FEARTracker read each tap's channels where they are, so no
    RGB copy is made: the frame the tracker sees is ``image_ops.rgb_frame_to_rgb(data, layout)`` of the same samples
    (``"planar"`` with ``bits`` for planes), which at 8 bits is ``cv2.cvtColor(data, COLOR_BGR2RGB / COLOR_BGRA2RGB /
    COLOR_RGBA2RGB)`` for the layouts cv2 names.  The constructors raise ValueError on a malformed tensor or layout;
    they make no device call.  ``shape`` is (H, W, 3)."""

    def __init__(self, t: torch.Tensor, layout: str) -> None:
        if layout in image_ops.RGB_PACKED_LAYOUTS:
            np_dtype, n, idx = image_ops.RGB_PACKED_LAYOUTS[layout]
            dtype = torch.uint8 if np_dtype == np.uint8 else torch.uint16
            self._check_tensor(t, (dtype,), 3, f"(H, W, {n}) tensor for {layout!r}")
            if t.shape[2] != n:
                raise ValueError(f"RGBFrame {layout!r} takes (H, W, {n}) samples, got {tuple(t.shape)}")
            h, w = t.shape[:2]
            rs, ps, cs = _unstepped(t, w * n, n, None)
            if cs != 1 or ps != n or rs < w * n:
                raise ValueError(f"RGBFrame {layout!r} needs channel stride 1, pixel stride {n} and a row stride of at "
                                 f"least {w * n}, got strides {t.stride()}")
            es, base = t.element_size(), t.data_ptr()
            self._check_aligned(base, rs * es, es)
            self._record = (base + idx[0] * es, base + idx[1] * es, base + idx[2] * es, rs * es, n * es, h, w, es,
                            8 * es, 0, 0, 0, 0)
        elif layout in image_ops.X2RGB10_LAYOUTS:
            self._check_tensor(t, (torch.int32, torch.uint32), 2, f"(H, W) tensor of 32-bit words for {layout!r}")
            h, w = t.shape
            rs, ps = _unstepped(t, w, 1)
            if ps != 1 or rs < w:
                raise ValueError(f"RGBFrame {layout!r} needs column stride 1 and a row stride of at least {w}, got "
                                 f"strides {t.stride()}")
            base = t.data_ptr()
            self._check_aligned(base, rs * 4, 4)
            self._record = (base, base, base, rs * 4, 4, h, w, 4, 10, *image_ops.X2RGB10_LAYOUTS[layout], 0)
        else:
            raise ValueError(f"unknown RGBFrame layout {layout!r}: one of "
                             f"{sorted(image_ops.RGB_PACKED_LAYOUTS) + sorted(image_ops.X2RGB10_LAYOUTS)}")
        self.tensors = (t,)
        self.layout, self.bits = layout, self._record[8]
        self.shape = (h, w, 3)

    @classmethod
    def planar(cls, r: torch.Tensor, g: torch.Tensor, b: torch.Tensor, bits: int = 8) -> "RGBFrame":
        if isinstance(bits, bool) or bits not in image_ops.RGB_PLANAR_BITS:
            raise ValueError(f"RGBFrame.planar bits must be 8, 10, 12 or 16, got {bits!r}")
        dtype = torch.uint8 if bits == 8 else torch.uint16
        for p in (r, g, b):
            cls._check_tensor(p, (dtype,), 2, f"(H, W) plane at {bits} bits")
        if not (r.shape == g.shape == b.shape):
            raise ValueError(f"RGBFrame.planar planes must share one shape, got {tuple(r.shape)}, {tuple(g.shape)} "
                             f"and {tuple(b.shape)}")
        strides = [_unstepped(p, 0, 0) for p in (r, g, b)]
        if not (strides[0] == strides[1] == strides[2]):
            raise ValueError(f"RGBFrame.planar planes must share their strides, got {r.stride()}, {g.stride()} and "
                             f"{b.stride()}")
        es = r.element_size()
        rs, ps = strides[0]
        for p in (r, g, b):
            cls._check_aligned(p.data_ptr(), rs * es, es)
        f = cls.__new__(cls)
        h, w = r.shape
        f._record = (r.data_ptr(), g.data_ptr(), b.data_ptr(), rs * es, ps * es, h, w, es, int(bits), 0, 0, 0, 0)
        f.tensors = (r, g, b)
        f.layout, f.bits = "planar", int(bits)
        f.shape = (h, w, 3)
        return f

    @staticmethod
    def _check_tensor(t, dtypes: tuple, ndim: int, what: str) -> None:
        if not isinstance(t, torch.Tensor) or t.dtype not in dtypes or t.ndim != ndim or t.device.type != "cuda":
            got = f"{t.dtype} {tuple(t.shape)} on {t.device}" if isinstance(t, torch.Tensor) else type(t).__name__
            want = " or ".join(str(d) for d in dtypes)
            raise ValueError(f"RGBFrame takes a {ndim}-D CUDA {want} {what}, got {got}")
        if min(t.stride(), default=0) < 0:
            raise ValueError(f"RGBFrame tensors need non-negative strides, got {t.stride()}")
        if not (1 <= t.shape[0] <= _MAX_SIDE and 1 <= t.shape[1] <= _MAX_SIDE):
            raise ValueError(f"an RGB frame needs 1 to {_MAX_SIDE} rows and columns, got {tuple(t.shape)}")

    @staticmethod
    def _check_aligned(address: int, row_bytes: int, es: int) -> None:
        if es > 1 and (address % es or row_bytes % es):
            raise ValueError(f"RGBFrame {8 * es}-bit samples must start on {es}-byte boundaries: address offset "
                             f"{address % es}, row pitch {row_bytes}")

    def rgb_record(self) -> tuple:
        """The FearFrameRGB record (r, g, b, row_stride, pixel_stride, H, W, container, bits, shift_r, shift_g,
        shift_b, reserved): the addresses of the containers holding R, G and B of pixel (0, 0), the byte strides, the
        size, the container's bytes, the code depth and each channel's shift."""
        return self._record


def tensor_rgb_record(t: torch.Tensor) -> tuple:
    """The FearFrameRGB record of a uint8 (H, W, 3) RGB tensor (``frame_view`` as an 8-bit RGBFrame): channel c at
    data + c * channel_stride."""
    p, rs, ps, cs, h, w = frame_view(t)
    return (p, p + cs, p + 2 * cs, rs, ps, h, w, 1, 8, 0, 0, 0, 0)


_DEVICE_FRAMES = (_YUVFrame, V210Frame, _RawFrame, RGBFrame)


class Oriented:
    """A device frame as it is shown rather than as it is stored: ``frame`` turned ``rotate`` degrees clockwise (0, 90,
    180 or 270), after a left-right flip when ``mirror``.  For phone video (a portrait recording is coded in landscape
    and carries a display-matrix rotation) and for cameras mounted upside down or mirrored (ceiling CCTV, a rear
    camera, a mirrored selfie camera).  ffmpeg's autorotate convention: rotate = (-display-matrix rotation) mod 360,
    so ffprobe's ``rotation=-90`` is ``rotate=90``; nothing is read from containers.

        Oriented(frame, rotate=0, mirror=False)   frame: a CUDA uint8 (H, W, 3) tensor, YUV420Frame, YUV422Frame,
                                                  YUV444Frame, V210Frame, BayerFrame, MonoFrame or RGBFrame

    FEARMultiTracker and FEARTracker read the stored frame where it is and map each display pixel to its stored pixel
    inside the crop, so no turned copy is made: the frame the tracker sees is ``image_ops.orient(rgb, code)`` of the
    frame it sees for ``frame`` (``image_ops.yuv_to_rgb``, ``bayer_to_rgb``, ``mono_to_rgb``, ``rgb_frame_to_rgb`` or
    the tensor), and rects and boxes are in that frame's coordinates.  ``code`` is rotate / 90 + 4 * mirror
    (``image_ops.orient_code``); ``shape`` is the display shape, (W, H, 3) for 90 and 270 degrees.  The frame's kind
    (``frame_kind``) is the wrapped frame's, so the rules on mixing kinds in one call are unchanged, and oriented and
    plain frames, with different codes, may share a call.  The constructor raises ValueError on a bad rotation, a numpy
    array (turn host frames with ``image_ops.orient``: ``np.rot90`` is a free view there), a nested Oriented or
    anything that is not a device frame; the frame itself is checked by the tracker, as a plain one is."""

    def __init__(self, frame, rotate: int = 0, mirror: bool = False) -> None:
        code = image_ops.orient_code(rotate, mirror)
        if isinstance(frame, np.ndarray):
            raise ValueError("Oriented wraps device frames; turn a numpy frame with image_ops.orient(frame, code) "
                             "(np.rot90 and a flip are free views of a host frame) and pass the result")
        if isinstance(frame, Oriented):
            raise ValueError("Oriented frames cannot be nested: combine the turns into one rotate and mirror")
        if not isinstance(frame, _DEVICE_FRAMES + (torch.Tensor,)):
            raise ValueError(f"Oriented wraps a CUDA uint8 tensor, YUV420Frame, YUV422Frame, YUV444Frame, V210Frame, "
                             f"BayerFrame, MonoFrame or RGBFrame, got {type(frame).__name__}")
        self.frame, self.code = frame, code
        shape = tuple(frame.shape)
        self.shape = (shape[1], shape[0], *shape[2:]) if code & 1 and len(shape) >= 2 else shape

    def __repr__(self) -> str:
        return f"Oriented({type(self.frame).__name__}, code={self.code})"


def stored(frame):
    """The frame as it is stored: the wrapped frame of an ``Oriented``, any other frame itself."""
    return frame.frame if isinstance(frame, Oriented) else frame


def orient_codes(frames) -> Optional[np.ndarray]:
    """The (F,) int32 orientation codes of a call's frames (0 for a plain frame), or None when none is ``Oriented``: a
    call without Oriented frames launches the plain entry points."""
    if not any(isinstance(f, Oriented) for f in frames):
        return None
    return np.array([f.code if isinstance(f, Oriented) else 0 for f in frames], dtype=np.int32)


def frame_kind(frame) -> str:
    """"yuv" for a YUV420Frame, YUV422Frame, YUV444Frame or V210Frame, "bayer" for a BayerFrame, "mono" for a
    MonoFrame, "rgb" for an RGBFrame (any channel order and container: BGR, BGRA / ABGR, x2rgb10, rgb48 / rgba64, planar
    RGB; the kernels read its channels where they are), "cuda" for a torch tensor (checked by ``check_device_frame``),
    "numpy" for anything else.  Host frames are always H x W x 3 RGB.  An ``Oriented`` frame has its wrapped frame's
    kind."""
    frame = stored(frame)
    if isinstance(frame, RGBFrame):
        return "rgb"
    if isinstance(frame, (_YUVFrame, V210Frame)):
        return "yuv"
    if isinstance(frame, BayerFrame):
        return "bayer"
    if isinstance(frame, MonoFrame):
        return "mono"
    return "cuda" if isinstance(frame, torch.Tensor) else "numpy"


def _positions(keys: np.ndarray, streams: np.ndarray) -> np.ndarray:
    """The index in ``keys`` (distinct stream ids) of each of ``streams``, every one of which is in ``keys``."""
    order = np.argsort(keys)
    return order[np.searchsorted(keys[order], streams)]


def check_device(i: int, device, *tensors: torch.Tensor) -> None:
    """ValueError unless every tensor is on the tracker's CUDA device; ``device()`` gives that device and is called
    only once a tensor is known to be on some CUDA device."""
    for t in tensors:
        if t.device.type != "cuda":
            raise ValueError(f"frame {i} is in a {t.device} tensor: tensor frames and YUV planes must be on the "
                             "tracker's CUDA device (pass host frames as numpy arrays)")
        dev = device()
        if t.device != dev:
            raise ValueError(f"frame {i} is on {t.device}, the tracker on {dev}")


def check_tensor_frame(i: int, f: torch.Tensor, device) -> None:
    """ValueError unless ``f`` is a uint8 (H, W, 3) tensor with non-negative strides on the tracker's device."""
    if f.dtype != torch.uint8 or f.ndim != 3 or f.shape[2] != 3 or not (1 <= f.shape[0] <= _MAX_SIDE) \
            or not (1 <= f.shape[1] <= _MAX_SIDE):
        raise ValueError(f"frame {i} must be a uint8 HxWx3 RGB tensor, got {f.dtype} {tuple(f.shape)}")
    if min(f.stride()) < 0:
        raise ValueError(f"frame {i} has a negative stride {f.stride()}")
    check_device(i, device, f)


def uses_agc(frames, kind: str) -> bool:
    """Whether any of a call's frames of kind ``kind`` is a MonoFrame with gain control: its table needs
    fear_frame_range_mono before the sums or the crop read it."""
    return kind == "mono" and any(stored(f).agc is not None for f in frames)


def check_device_frame(i: int, f, kind: str, device) -> None:
    """The checks of a frame of kind "cuda", "yuv", "bayer", "mono" or "rgb" (``frame_kind``): ValueError before any
    device call.  An ``Oriented`` frame is checked as its wrapped frame."""
    f = stored(f)
    if kind == "rgb":
        check_device(i, device, *f.tensors)
    elif kind in ("bayer", "mono"):
        check_device(i, device, f.t)
    elif kind == "yuv":
        check_device(i, device, *((f.t,) if isinstance(f, V210Frame) else (f.y, f.u, f.v)))
    else:
        check_tensor_frame(i, f, device)


def write_records(table: np.ndarray, frames, name: str) -> None:
    """Write the records of device frames into rows of ``table`` (a numpy view of ``TABLE_DTYPES[name]``):
    FearFrameView records of CUDA tensors for "views", FearFrameYUV records for "yuv", FearFrameYCbCr for "ycbcr",
    FearFrameYCbCrV210 for "ycbcr_v210", FearFrameYCbCrHDR for "ycbcr_hdr", FearFrameBayer for "bayer", FearFrameMono
    for "mono", FearFrameRGB for "rgb" (of RGBFrames and of CUDA tensors, ``tensor_rgb_record``).  An ``Oriented``
    frame's record is its stored frame's: its code goes into a table of its own."""
    for i, f in enumerate(frames):
        f = stored(f)
        if name == "rgb":
            table[i] = f.rgb_record() if isinstance(f, RGBFrame) else tensor_rgb_record(f)
        elif name == "yuv":
            table[i] = f.yuv_record()
        elif name == "ycbcr":
            table[i] = f.ycbcr_record()
        elif name == "ycbcr_v210":
            table[i] = f.ycbcr_v210_record()
        elif name == "ycbcr_hdr":
            table[i] = f.hdr_record()
        elif name == "bayer":
            table[i] = f.bayer_record()
        elif name == "mono":
            table[i] = f.mono_record()
        else:
            table[i] = frame_view(f)


class FEARMultiTracker:
    def __init__(self, model, cuda_id: Union[int, str] = 0, max_targets: int = 64, **tracking_config: Any) -> None:
        cfg = tracking_config
        if cfg.get("smooth", False) or cfg.get("host_normalize", False):
            raise NotImplementedError("FEARMultiTracker covers the default uint8 RGB tracking path "
                                      "(no smooth / host_normalize)")
        for key in ("search_context", "template_bbox_offset"):
            v = float(cfg[key])
            if not math.isfinite(v) or v < 0:
                raise ValueError(f"{key} must be finite and >= 0, got {cfg[key]!r}")
        size = int(cfg["instance_size"])
        if size % 16 or not 16 <= size <= 256 or int(cfg["template_size"]) != 128:
            raise ValueError("FEAR-XS tracks S x S search crops, S a multiple of 16 in [16, 256], against 128 x 128 "
                             f"templates; got instance_size={cfg['instance_size']}, template_size={cfg['template_size']}")
        stride, score = cfg.get("total_stride", 16), cfg.get("score_size", size // 16)
        if int(stride) != 16 or int(score) != size // 16:
            raise ValueError(f"a {size} x {size} search gives a {size // 16} x {size // 16} score map at total_stride 16; "
                             f"got score_size={score}, total_stride={stride}")
        if int(max_targets) < 1:
            raise ValueError(f"max_targets must be >= 1, got {max_targets}")
        self.net = model
        self.cuda_id = cuda_id
        self.tracking_config = tracking_config
        self.max_targets = int(max_targets)
        self.net.reserve(self.max_targets)  # the whole batch fits the workspace: graph capture never allocates
        self._buf = None  # device buffers, allocated on first use
        self._frames_key = None  # numpy frame shapes the packed buffer is laid out for
        self._graph = None
        self._graph_key = None
        self._graph_gen = None
        self._graph_ok = True
        self._calls = 0
        self._subset_graphs = OrderedDict()  # subset step graphs: key -> {"calls", "graph", "boxes"}, LRU order
        self._subset_gen = None  # the net's generation the cached subset graphs were captured at
        self.reset()

    # ------------------------------------------------------------------ public API
    def reset(self) -> None:
        """Drop every target (ids start again from 0)."""
        self._ids = np.zeros(0, dtype=np.int64)
        self._streams = np.zeros(0, dtype=np.int64)
        self._next_id = 0

    def initialize(self, frames, rects, streams: Optional[Sequence[int]] = None) -> np.ndarray:
        self.reset()
        return self.add(frames, rects, streams)

    @property
    def ids(self) -> np.ndarray:
        return self._ids.copy()

    def __len__(self) -> int:
        return len(self._ids)

    def add(self, frames, rects, streams: Optional[Sequence[int]] = None) -> np.ndarray:
        """Start tracking ``rects`` ((n, 4) [x, y, w, h]); target i lives in stream ``streams[i]`` (default 0), whose
        current frame is ``frames[streams[i]]``.  Returns the new targets' ids.

        ``frames`` are all numpy arrays, all CUDA tensors, all YUV frames (YUV420Frame, YUV422Frame, YUV444Frame,
        V210Frame), all BayerFrames, all MonoFrames, or RGBFrames and CUDA tensors (see ``update``).  ``frames`` may
        also be a mapping {stream id: frame} of the streams at hand (ids ints in [0, 2^31 - 1], possibly sparse, such as
        cameras 3 and 17); ``streams[i]`` is then a key of it (the default stream 0 must be one), and only its frames
        are read.  A target's padding colour is the mean colour of its frame (of the converted RGB frame for a YUV
        frame, of the demosaiced 8-bit frame for a Bayer frame, of the grey frame after gain control for a mono frame,
        of the 8-bit RGB frame for an RGBFrame), from exact per-channel sums computed on the device."""
        keys = None
        if isinstance(frames, Mapping):
            keys, frames, kind = self._check_mapping(frames)
        else:
            frames, kind = self._check_frames(frames)
        rects = np.asarray(rects, dtype=np.float64)
        if rects.ndim == 1 and rects.size == 4:
            rects = rects[None]
        if rects.ndim != 2 or rects.shape[1] != 4:
            raise ValueError(f"rects must be (n, 4) [x, y, w, h], got shape {rects.shape}")
        n = rects.shape[0]
        streams = np.zeros(n, dtype=np.int64) if streams is None else streams
        if keys is None:
            streams = pos = self._check_streams(streams, n, len(frames))
        else:
            streams, pos = self._check_mapping_streams(streams, n, keys)
        if len(self._ids) + n > self.max_targets:
            raise ValueError(f"{len(self._ids)} + {n} targets exceed max_targets = {self.max_targets}")
        if n == 0:
            return np.zeros(0, dtype=np.int64)
        cfg = self.tracking_config
        recs = np.zeros((n, _lib.TARGET_INTS), dtype=np.int32)
        for i, (rect, s) in enumerate(zip(rects, pos)):  # the template crop reads frame index s of this call's table
            box = image_ops.clamp_bbox(rect, tuple(frames[s].shape))
            ctx = image_ops.context_box(box, cfg["template_bbox_offset"])
            inner = image_ops.trim_box([box[0] - ctx[0], box[1] - ctx[1], box[2], box[3]], (ctx[3], ctx[2]))
            if inner[2] * inner[3] == 0:
                raise IndexError("target box has zero area inside its context crop")
            recs[i, 0] = s
            recs[i, 1:5] = box
        dev = self._device()
        with torch.cuda.device(dev):
            b = self._buffers(dev)
            num_frames = len(frames)
            table = self._upload_frames(frames, kind, dev)
            sums_fn = ENTRY_POINTS[table][0]
            lib = _lib.load()
            stream = torch.cuda.current_stream(dev)
            if uses_agc(frames, kind):
                _lib.check(getattr(lib, RANGE_ENTRY_POINT)(b[table].data_ptr(), num_frames, stream.cuda_stream),
                           RANGE_ENTRY_POINT)
            _lib.check(getattr(lib, sums_fn)(b[table].data_ptr(), num_frames, b["sums"].data_ptr(), stream.cuda_stream),
                       sums_fn)
            b["sums_pin"][:num_frames].copy_(b["sums"][:num_frames], non_blocking=True)
            stream.synchronize()
            # numpy's mean of uint8 is an exact float64 sum of integers over H * W; then cv::saturate_cast, as
            # FEARTracker's padding
            sums = b["sums_pin"].numpy()[:num_frames].view(np.uint64)
            pixels = np.array([f.shape[0] * f.shape[1] for f in frames], dtype=np.float64)
            pads = np.clip(np.rint(sums / pixels[:, None]), 0, 255).astype(np.int32)
            recs[:, 9:12] = pads[pos]
            n0 = len(self._ids)
            b["state"][n0:n0 + n].copy_(torch.from_numpy(recs).pin_memory(), non_blocking=True)
            size = int(cfg["template_size"])
            crops = b["tcrops"][:n]
            self._crop(table, num_frames, orient_codes(frames) is not None, b["state"][n0].data_ptr(), n,
                       float(cfg["template_bbox_offset"]), size, crops.data_ptr(), stream.cuda_stream)
            b["zf"][n0:n0 + n].copy_(self.net.get_features(crops))
            if keys is not None:  # the rows keep their stream ids, not this call's frame indices
                b["state"][n0:n0 + n, 0].copy_(torch.from_numpy(streams.astype(np.int32)).pin_memory(),
                                               non_blocking=True)
            stream.synchronize()  # the pinned staging buffers are reused by the next call
        new_ids = np.arange(self._next_id, self._next_id + n, dtype=np.int64)
        self._next_id += n
        self._ids = np.concatenate([self._ids, new_ids])
        self._streams = np.concatenate([self._streams, streams])
        return new_ids

    def remove(self, ids) -> None:
        ids = np.atleast_1d(np.asarray(ids, dtype=np.int64))
        unknown = np.setdiff1d(ids, self._ids)
        if unknown.size:
            raise ValueError(f"unknown target ids {unknown.tolist()}")
        keep = np.flatnonzero(~np.isin(self._ids, ids))
        if self._buf is not None and keep.size:
            with torch.cuda.device(self._buf["device"]):
                idx = torch.from_numpy(keep).to(self._buf["device"])
                m = keep.size
                self._buf["state"][:m] = self._buf["state"][idx]
                self._buf["zf"][:m] = self._buf["zf"][idx]
        self._ids, self._streams = self._ids[keep], self._streams[keep]

    def update(self, frames) -> Dict[str, np.ndarray]:
        """One frame of every stream -> the new box and score of every target, in the order of ``ids``; or the frames
        of some streams -> the new boxes and scores of their targets only.

        ``frames`` is one frame, a list of F (stream i's frame at index i), or a mapping {stream id: frame} of the
        streams that have a new frame, for streams that do not tick together (cameras at different rates, a stalled
        stream, frames batched as they arrive).  With a mapping only the targets of its streams are stepped, and the
        result holds their "bbox", "score" and "ids" alone, in the order of ``ids``; every other target's state and
        template stay exactly as they were, so each target's trajectory is that of its own tracker fed the frames its
        stream delivered.  Keys are ints in [0, 2^31 - 1]; a key with no targets is allowed (its frame is checked, not
        read); a mapping that selects no target returns empty arrays without a device call.  The values follow the
        rules of a list below.

        The frames are all ``np.ndarray``, all
        ``torch.Tensor`` or all YUV frames (``YUV420Frame``, ``YUV422Frame``, ``YUV444Frame``, mixed freely); the kind
        may change from one call to the next.  A tensor frame is uint8 of shape (H, W, 3) on the tracker's CUDA device,
        with any non-negative strides: views are read as they are, nothing is copied.  A YUV frame's planes must be on
        the tracker's CUDA device; they are read in place too, and every target fed YUV frames gives exactly the ids,
        boxes and scores of the same tracker fed ``image_ops.yuv_to_rgb`` of the planes (with the frame's
        ``CHROMA_SHIFT``) as numpy arrays (for the default format that is ``cv2.cvtColor(frame,
        cv2.COLOR_YUV2RGB_NV12 / COLOR_YUV2RGB_I420 / COLOR_YUV2RGB_YUY2 / COLOR_YUV2RGB_UYVY)``).  A ``V210Frame``'s
        words are read in place as well and give what its ``image_ops.v210_unpack`` planes give at 10 bits, 4:2:2.
        Frames of one call may have different colour formats and subsamplings.  ``frames`` may also be all
        ``BayerFrame``s (any patterns, depths and packings), never mixed with other kinds; their samples are read in
        place and give exactly what ``image_ops.bayer_to_rgb`` of their codes gives as numpy arrays.  ``frames`` may
        also be all ``MonoFrame``s (any depths, packings and gain controls), never mixed with other kinds; they give
        exactly what ``image_ops.mono_to_rgb`` of their codes gives as numpy arrays.  ``frames`` may also be
        ``RGBFrame``s (any layouts and depths) mixed freely with CUDA tensors, never with other kinds; they give exactly
        what ``image_ops.rgb_frame_to_rgb`` of their samples gives as numpy arrays.  Any device frame may be an
        ``Oriented`` one, with its own code, alongside plain frames of kinds its frame may share a call with; it gives
        exactly what ``image_ops.orient`` of the frame it wraps gives as a numpy array, with boxes in the turned
        picture's coordinates.  Device frames must
        be ready on the current CUDA stream (write them on that stream, or make it wait for the stream that did, as for
        any torch op).  ``update`` synchronises that stream before it returns, so they only need to live until the
        call returns."""
        if isinstance(frames, Mapping):
            return self._update_streams(*self._check_mapping(frames))
        frames, kind = self._check_frames(frames)
        n = len(self._ids)
        if n and int(self._streams.max()) >= len(frames):
            raise ValueError(f"targets track stream {int(self._streams.max())} but only {len(frames)} frames were given")
        if n == 0:
            return dict(bbox=np.zeros((0, 4), dtype=np.int64), score=np.zeros(0, dtype=np.float32),
                        ids=self._ids.copy())
        dev = self._device()
        with torch.cuda.device(dev):
            b = self._buffers(dev)
            table = self._upload_frames(frames, kind, dev)
            boxes = self._run_step(n, len(frames), table, dev, uses_agc(frames, kind),
                                   orient_codes(frames) is not None)
            b["state_pin"][:n].copy_(b["state"][:n], non_blocking=True)
            b["box_pin"][:n].copy_(boxes, non_blocking=True)
            torch.cuda.current_stream(dev).synchronize()
        state = b["state_pin"].numpy()[:n]
        rec = b["box_pin"].numpy()[:n].view(_lib.BOX_DTYPE).reshape(-1)
        return dict(bbox=state[:, 1:5].astype(np.int64), score=rec["score"].astype(np.float32), ids=self._ids.copy())

    # ------------------------------------------------------------------ internals
    def _update_streams(self, keys: np.ndarray, frames: list, kind: str) -> Dict[str, np.ndarray]:
        """``update`` of a mapping: step the targets whose stream is in ``keys`` (the mapping's stream ids, in the order
        of ``frames``) on compact step rows, through the selection (target row, frame index) pairs."""
        rows = np.flatnonzero(np.isin(self._streams, keys))  # ascending: the order of ids
        m = rows.size
        if m == 0:
            return dict(bbox=np.zeros((0, 4), dtype=np.int64), score=np.zeros(0, dtype=np.float32),
                        ids=np.zeros(0, dtype=np.int64))
        dev = self._device()
        with torch.cuda.device(dev):
            b = self._buffers(dev)
            table = self._upload_frames(frames, kind, dev)
            sel = b["select_pin"].numpy()
            sel[:m, 0] = rows
            sel[:m, 1] = _positions(keys, self._streams[rows])
            b["select"][:m].copy_(b["select_pin"][:m], non_blocking=True)
            boxes = self._run_subset_step(m, len(frames), table, dev, uses_agc(frames, kind),
                                          orient_codes(frames) is not None)
            b["state_pin"][:m].copy_(b["step_state"][:m], non_blocking=True)
            b["box_pin"][:m].copy_(boxes, non_blocking=True)
            torch.cuda.current_stream(dev).synchronize()
        state = b["state_pin"].numpy()[:m]
        rec = b["box_pin"].numpy()[:m].view(_lib.BOX_DTYPE).reshape(-1)
        return dict(bbox=state[:, 1:5].astype(np.int64), score=rec["score"].astype(np.float32), ids=self._ids[rows])

    def _check_mapping(self, frames: Mapping):
        """-> (stream ids (F,) int64, list of frames, their kind) of a {stream id: frame} mapping, in its order.  Raises
        ValueError before any device call."""
        keys = list(frames)
        for k in keys:
            if isinstance(k, (bool, np.bool_)) or not isinstance(k, (int, np.integer)) or not 0 <= k <= _MAX_STREAM:
                raise ValueError(f"stream ids must be ints in [0, {_MAX_STREAM}], got {k!r}")
        if not keys:
            raise ValueError("no frames given")
        frames, kind = self._check_frames([frames[k] for k in keys])
        return np.array(keys, dtype=np.int64), frames, kind

    @staticmethod
    def _check_mapping_streams(streams, n: int, keys: np.ndarray):
        """-> (stream ids (n,) int64, their frame indices in the mapping) of ``add``'s ``streams`` for a mapping."""
        s = np.asarray(streams)
        if s.shape != (n,) or (s.size and not np.issubdtype(s.dtype, np.integer)):
            raise ValueError(f"streams must be ({n},) integer stream ids, got {s.dtype} {s.shape}")
        s = s.astype(np.int64)
        missing = np.setdiff1d(s, keys)
        if missing.size:
            raise ValueError(f"streams {missing.tolist()} are not keys of the frames mapping {keys.tolist()}")
        return s, _positions(keys, s)

    def _device(self) -> torch.device:
        if not torch.cuda.is_available():
            raise RuntimeError("FEARMultiTracker (H100) needs a CUDA device: there is no CPU path")
        if isinstance(self.cuda_id, int):
            return torch.device("cuda", self.cuda_id)
        dev = torch.device(self.cuda_id)
        if dev.type != "cuda":
            raise RuntimeError(f"FEARMultiTracker (H100) needs a CUDA device, got {self.cuda_id!r}: there is no CPU path")
        return torch.device("cuda", dev.index if dev.index is not None else torch.cuda.current_device())

    def _check_frames(self, frames):
        """-> (list of frames, their kind: "numpy", "cuda", "yuv", "bayer", "mono" or "rgb", the last for RGBFrames
        with or without CUDA tensors).  Raises ValueError before any device call."""
        if isinstance(frames, _DEVICE_FRAMES + (Oriented,)) or (isinstance(frames, (np.ndarray, torch.Tensor))
                                                                and frames.ndim == 3):
            frames = [frames]
        frames = list(frames)
        if not frames:
            raise ValueError("no frames given")
        kinds = [frame_kind(f) for f in frames]
        kind = kinds[0]
        if set(kinds) == {"rgb", "cuda"}:  # RGBFrames and RGB tensors share the rgb table
            kind = "rgb"
        elif any(k != kind for k in kinds):
            if any(frame_kind(f) == "bayer" for f in frames):
                raise ValueError("BayerFrames cannot share a call with other kinds of frames (numpy arrays, CUDA "
                                 "tensors, YUV frames): pass all of a call's frames as BayerFrames")
            if any(frame_kind(f) == "mono" for f in frames):
                raise ValueError("MonoFrames cannot share a call with other kinds of frames (numpy arrays, CUDA "
                                 "tensors, YUV frames): pass all of a call's frames as MonoFrames")
            if "rgb" in kinds:
                raise ValueError("RGBFrames can share a call only with CUDA uint8 RGB tensors, not with numpy arrays or "
                                 "YUV frames: pass the call's frames as RGBFrames or CUDA tensors")
            raise ValueError("frames of one call must be all numpy arrays, all CUDA tensors or all YUV frames "
                             "(YUV420Frame, YUV422Frame, YUV444Frame, V210Frame), not a mix")
        for i, f in enumerate(frames):
            if kind != "numpy":
                check_device_frame(i, f, kinds[i], self._device)
            elif not isinstance(f, np.ndarray) or f.dtype != np.uint8 or f.ndim != 3 or f.shape[2] != 3 \
                    or f.shape[0] < 1 or f.shape[1] < 1:
                what = f"{f.dtype} {f.shape}" if isinstance(f, np.ndarray) else type(f).__name__
                raise ValueError(f"frame {i} must be a uint8 HxWx3 RGB array, got {what}")
        return frames, kind

    @staticmethod
    def _check_streams(streams, n: int, num_frames: int) -> np.ndarray:
        s = np.asarray(streams)
        if s.shape != (n,) or (s.size and not np.issubdtype(s.dtype, np.integer)):
            raise ValueError(f"streams must be ({n},) integer frame indices, got {s.dtype} {s.shape}")
        s = s.astype(np.int64)
        if s.size and (s.min() < 0 or s.max() >= num_frames):
            raise ValueError(f"stream indices must be in [0, {num_frames}), got {s.tolist()}")
        return s

    def _buffers(self, dev: torch.device) -> dict:
        b = self._buf
        if b is not None and b["device"] == dev:
            return b
        if b is not None:  # moving to another device: the targets' state and templates do not follow
            raise RuntimeError(f"FEARMultiTracker state lives on {b['device']}, not {dev}")
        m, size = self.max_targets, int(self.tracking_config["instance_size"])
        tsize = int(self.tracking_config["template_size"])
        self._buf = b = dict(
            device=dev,
            state=torch.zeros((m, _lib.TARGET_INTS), dtype=torch.int32, device=dev),
            zf=torch.zeros((m, 256, 8, 8), dtype=torch.float32, device=dev),
            crops=torch.empty((m, size, size, 3), dtype=torch.uint8, device=dev),
            tcrops=torch.empty((m, tsize, tsize, 3), dtype=torch.uint8, device=dev),
            # the compact rows and templates of a subset step, and its selection: (target row, frame index) pairs
            step_state=torch.zeros((m, _lib.TARGET_INTS), dtype=torch.int32, device=dev),
            step_zf=torch.zeros((m, 256, 8, 8), dtype=torch.float32, device=dev),
            select=torch.zeros((m, 2), dtype=torch.int32, device=dev),
            select_pin=torch.zeros((m, 2), dtype=torch.int32).pin_memory(),
            state_pin=torch.empty((m, _lib.TARGET_INTS), dtype=torch.int32).pin_memory(),
            box_pin=torch.empty((m, _lib.BOX_DTYPE.itemsize), dtype=torch.uint8).pin_memory(),
            frames_pin=None, frames=None, views_pin=None, views=None, yuv_pin=None, yuv=None, ycbcr_pin=None,
            ycbcr=None, ycbcr_v210_pin=None, ycbcr_v210=None, ycbcr_hdr_pin=None, ycbcr_hdr=None, bayer_pin=None,
            bayer=None, mono_pin=None, mono=None, rgb_pin=None, rgb=None, sums_pin=None, sums=None)
        return b

    def _upload_frames(self, frames, kind: str, dev: torch.device) -> str:
        """Write the frame table of ``frames`` into the fixed device table the kernels read, and return its name:
        "yuv" (FearFrameYUV records) when every frame is a YUV420Frame, "ycbcr_hdr" (FearFrameYCbCrHDR records) for YUV
        frames of which any has a transfer (PQ, HLG), else "ycbcr_v210" (FearFrameYCbCrV210 records) for YUV frames of
        which any is a V210Frame, "ycbcr" (FearFrameYCbCr records) for other YUV frames of which any is
        4:2:2 or 4:4:4, "bayer" (FearFrameBayer records) for BayerFrames, "mono" (FearFrameMono records) for
        MonoFrames, "rgb" (FearFrameRGB records) for a call with any RGBFrame, "views" (FearFrameView records)
        otherwise.  Numpy frames are packed into the pinned staging buffer
        first and sent with one host-to-device copy (the packed layout is recomputed only when their shapes change);
        CUDA tensors, YUV planes, v210 surfaces, Bayer mosaics, mono frames and RGB frames are used where they are.
        When any frame is ``Oriented``, the F int32 orientation codes follow the F records in the same buffer and the
        same copy (``_orient_ptr``); otherwise the copy is the records alone, as it always was."""
        b, num_frames = self._buf, len(frames)
        plain = [stored(f) for f in frames]
        name = "views"
        if kind == "yuv":
            name = "yuv" if all(isinstance(f, YUV420Frame) for f in plain) else "ycbcr"
            if any(isinstance(f, V210Frame) for f in plain):
                name = "ycbcr_v210"
            if any(f.transfer is not None for f in plain):
                name = "ycbcr_hdr"
        elif kind in ("bayer", "mono", "rgb"):
            name = kind
        dtype = TABLE_DTYPES[name]
        nbytes = num_frames * dtype.itemsize
        codes = orient_codes(frames)
        room = nbytes + 4 * num_frames  # every table's record size is a multiple of 8: the codes stay aligned
        if b[name] is None or b[name].numel() < room:  # grows only: the step graph keys on it
            b[name + "_pin"] = torch.empty(room, dtype=torch.uint8).pin_memory()
            b[name] = torch.empty(room, dtype=torch.uint8, device=dev)
        if b["sums"] is None or b["sums"].shape[0] < num_frames:
            # the frame sums entry points write uint64; int64 storage, read back as uint64
            b["sums_pin"] = torch.empty((num_frames, 3), dtype=torch.int64).pin_memory()
            b["sums"] = torch.empty((num_frames, 3), dtype=torch.int64, device=dev)
        table = b[name + "_pin"].numpy()[:nbytes].view(dtype)
        if kind != "numpy":
            write_records(table, frames, name)
        else:
            key = tuple(f.shape for f in frames)
            if key != self._frames_key:
                offsets, off = [], 0
                for f in frames:
                    offsets.append(off)
                    off += -(-f.size // _FRAME_ALIGN) * _FRAME_ALIGN
                if b["frames"] is None or b["frames"].numel() < off:
                    b["frames_pin"] = torch.empty(off, dtype=torch.uint8).pin_memory()
                    b["frames"] = torch.empty(off, dtype=torch.uint8, device=dev)
                b["offsets"], b["nbytes"] = offsets, off
                self._frames_key = key
            pin, base = b["frames_pin"].numpy(), b["frames"].data_ptr()
            for i, (f, o) in enumerate(zip(frames, b["offsets"])):
                np.copyto(pin[o:o + f.size].reshape(f.shape), f)
                h, w = f.shape[:2]
                table[i] = (base + o, 3 * w, 3, 1, h, w)
            nb = b["nbytes"]
            b["frames"][:nb].copy_(b["frames_pin"][:nb], non_blocking=True)
        if codes is not None:
            b[name + "_pin"].numpy()[nbytes:nbytes + 4 * num_frames].view(np.int32)[:] = codes
            nbytes += 4 * num_frames
        b[name][:nbytes].copy_(b[name + "_pin"][:nbytes], non_blocking=True)
        return name

    def _orient_ptr(self, table: str, num_frames: int) -> int:
        """The device address of the orientation codes ``_upload_frames`` writes after the F records of ``table``."""
        return self._buf[table].data_ptr() + num_frames * TABLE_DTYPES[table].itemsize

    def _crop(self, table: str, num_frames: int, oriented: bool, state_ptr: int, n: int, offset: float, size: int,
              crops_ptr: int, s) -> None:
        """The crop entry point of ``table`` on ``n`` FearTarget rows, or with ``oriented`` the oriented one reading
        the call's codes."""
        lib, t = _lib.load(), self._buf[table].data_ptr()
        if oriented:
            fn = ORIENTED_ENTRY_POINTS[0]
            _lib.check(getattr(lib, fn)(_lib.ORIENT_TABLES[table], t, self._orient_ptr(table, num_frames), num_frames,
                                        state_ptr, n, offset, size, crops_ptr, s), fn)
        else:
            fn = ENTRY_POINTS[table][1]
            _lib.check(getattr(lib, fn)(t, num_frames, state_ptr, n, offset, size, crops_ptr, s), fn)

    def _step(self, n: int, num_frames: int, dev: torch.device, table: str = "views",
              agc: bool = False, state: str = "state", zf: str = "zf", oriented: bool = False) -> torch.Tensor:
        """crop -> network -> advance on the first ``n`` rows of the FearTarget buffer ``state`` and the templates
        ``zf`` (the targets' own rows, or the compact step rows of a subset step); with ``oriented`` the oriented crop
        and advance, the same number of launches."""
        b, cfg, lib = self._buf, self.tracking_config, _lib.load()
        size = int(cfg["instance_size"])
        s = torch.cuda.current_stream(dev).cuda_stream
        if agc:  # the frames' code ranges, written into the table the crop reads
            _lib.check(getattr(lib, RANGE_ENTRY_POINT)(b[table].data_ptr(), num_frames, s), RANGE_ENTRY_POINT)
        self._crop(table, num_frames, oriented, b[state].data_ptr(), n, float(cfg["search_context"]), size,
                   b["crops"].data_ptr(), s)
        boxes = self.net.track_boxes(b["crops"][:n], b[zf][:n])
        if oriented:
            fn = ORIENTED_ENTRY_POINTS[1]
            _lib.check(getattr(lib, fn)(boxes.data_ptr(), _lib.ORIENT_TABLES[table], b[table].data_ptr(),
                                        self._orient_ptr(table, num_frames), num_frames, b[state].data_ptr(), n, size,
                                        s), fn)
        else:
            advance_fn = ENTRY_POINTS[table][2]
            _lib.check(getattr(lib, advance_fn)(boxes.data_ptr(), b[table].data_ptr(), num_frames,
                                                b[state].data_ptr(), n, size, s), advance_fn)
        return boxes

    def _subset_step(self, m: int, num_frames: int, dev: torch.device, table: str, agc: bool,
                     oriented: bool = False) -> torch.Tensor:
        """One step of the ``m`` targets named by the selection buffer: gather their rows and templates into the
        compact step buffers, step those, and scatter the new boxes back.  Rows are bounded by ``max_targets`` (the
        buffer's size), not by the target count, so adding or removing targets does not change the captured graph."""
        b, lib, rows = self._buf, _lib.load(), self.max_targets
        s = torch.cuda.current_stream(dev).cuda_stream
        _lib.check(lib.fear_gather_targets(b["state"].data_ptr(), rows, b["zf"].data_ptr(), b["select"].data_ptr(), m,
                                           b["step_state"].data_ptr(), b["step_zf"].data_ptr(), s),
                   "fear_gather_targets")
        boxes = self._step(m, num_frames, dev, table, agc, state="step_state", zf="step_zf", oriented=oriented)
        _lib.check(lib.fear_scatter_targets(b["step_state"].data_ptr(), b["select"].data_ptr(), m,
                                            b["state"].data_ptr(), rows, s), "fear_scatter_targets")
        return boxes

    def _run_subset_step(self, m: int, num_frames: int, table: str, dev: torch.device, agc: bool,
                         oriented: bool = False) -> torch.Tensor:
        """One subset step, replayed from a cache of captured graphs kept apart from the list path's ``_graph``, so
        neither path recaptures the other's graph.  The selection is read from its buffer when the kernels run, so a
        graph is keyed by the step's shape only: the step row count, the frame count, the table and its buffer,
        ``agc``, the selection buffer and whether the step is ``oriented`` (not the codes, read when it runs).  A key is captured on its second call, as in ``_run_step``.  The cache holds
        at most ``SUBSET_GRAPHS`` keys (captured or counting calls) and evicts the least recently used one; a change of
        the net's generation drops every graph."""
        gen = self.net.generation()
        if gen != self._subset_gen:
            self._subset_graphs.clear()
            self._subset_gen = gen
        key = (m, num_frames, table, self._buf[table].data_ptr(), agc, self._buf["select"].data_ptr(), oriented)
        entry = self._subset_graphs.pop(key, None) or {"calls": 0, "graph": None, "boxes": None}
        self._subset_graphs[key] = entry  # most recently used last
        while len(self._subset_graphs) > SUBSET_GRAPHS:
            self._subset_graphs.popitem(last=False)
        use_graph = self.tracking_config.get("cuda_graph", True) and self._graph_ok
        if use_graph and entry["graph"] is None and entry["calls"] >= 1:
            try:
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    entry["boxes"] = self._subset_step(m, num_frames, dev, table, agc, oriented)
                entry["graph"] = g
            except RuntimeError as exc:
                warnings.warn(f"FEARMultiTracker: CUDA-graph capture of the step failed ({exc}); using eager launches")
                self._graph_ok = False
                torch.cuda.synchronize(dev)
        entry["calls"] += 1
        if use_graph and entry["graph"] is not None:
            entry["graph"].replay()
            return entry["boxes"]
        return self._subset_step(m, num_frames, dev, table, agc, oriented)

    def _run_step(self, n: int, num_frames: int, table: str, dev: torch.device, agc: bool = False,
                  oriented: bool = False) -> torch.Tensor:
        """One step, as a CUDA graph after one eager warm-up call (the pattern of FEARTracker's gpu_crop path).  The
        kernels read the frame table when they run, so frame addresses and shapes are not baked into the graph: it is
        keyed by the target count, the frame count, which table the step reads (RGB views, YUV 4:2:0 records, YCbCr
        records of any subsampling, YCbCr / v210 records, HDR records, Bayer records, mono records or RGB records) and
        its buffer, whether the step starts with the mono range kernel (``agc``), whether it runs the oriented crop
        and advance (``oriented``; the codes are read when the kernels run, so new codes replay the graph), and the
        net's generation.
        ``cuda_graph=False`` in the tracking config keeps eager launches."""
        key = (n, num_frames, table, self._buf[table].data_ptr(), agc, oriented)
        if key != self._graph_key or (self._graph is not None and self._graph_gen != self.net.generation()):
            # new target or frame count, another table or a new table buffer, or the net's workspace / weights /
            # options changed: the pointers and sizes baked into the captured graph are stale -> warm up eagerly and
            # capture again
            self._graph, self._graph_key, self._calls = None, key, 0
        use_graph = self.tracking_config.get("cuda_graph", True) and self._graph_ok
        if use_graph and self._graph is None and self._calls >= 1:
            try:
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    self._graph_boxes = self._step(n, num_frames, dev, table, agc, oriented=oriented)
                self._graph, self._graph_gen = g, self.net.generation()
            except RuntimeError as exc:
                warnings.warn(f"FEARMultiTracker: CUDA-graph capture of the step failed ({exc}); using eager launches")
                self._graph_ok = False
                torch.cuda.synchronize(dev)
        self._calls += 1
        if use_graph and self._graph is not None:
            self._graph.replay()
            return self._graph_boxes
        return self._step(n, num_frames, dev, table, agc, oriented=oriented)
