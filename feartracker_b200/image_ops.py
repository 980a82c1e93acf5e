"""Host-side crop / box helpers of the tracking loop (the CPU half of FEARTracker).

Behavioural mirror of the helpers the reference tracker calls (reference
model_training/utils/utils.py:29-71,202-253 and base_tracker.py:69-103): integer context
boxes, constant-colour padding, cv2 bilinear resize, ImageNet normalisation in float32.
``albumentations`` is not required: its Resize is ``cv2.resize(INTER_LINEAR)`` and its Normalize
is ``(img - mean*255) * (1/(std*255))`` in float32.
"""
import math
from typing import Optional, Sequence, Tuple

import cv2
import numpy as np

IMAGENET_MEAN = (0.485, 0.456, 0.406)
IMAGENET_STD = (0.229, 0.224, 0.225)
_MEAN255 = np.array(IMAGENET_MEAN, dtype=np.float32) * np.float32(255.0)
_INV_STD255 = np.reciprocal(np.array(IMAGENET_STD, dtype=np.float32) * np.float32(255.0), dtype=np.float32)


def context_box(bbox: Sequence[float], offset: float) -> np.ndarray:
    """Grow [x, y, w, h] by ``offset`` * side on every side, truncated to int32."""
    x, y, w, h = bbox
    return np.array([x - w * offset, y - h * offset, w * (1.0 + 2.0 * offset), h * (1.0 + 2.0 * offset)]).astype(
        "int32")


def trim_box(bbox: Sequence[float], img_shape: Sequence[int]) -> np.ndarray:
    """Clip [x, y, w, h] to an image of shape (h, w, ...)."""
    x1, y1, w, h = bbox
    x1, y1 = min(max(0, x1), img_shape[1]), min(max(0, y1), img_shape[0])
    x2, y2 = min(max(0, x1 + w), img_shape[1]), min(max(0, y1 + h), img_shape[0])
    return np.array([x1, y1, x2 - x1, y2 - y1]).astype("int32")


def clamp_bbox(bbox: Sequence[float], shape: Sequence[int], min_side: int = 3) -> np.ndarray:
    x, y, w, h = trim_box(bbox, shape)
    img_h, img_w = shape[0], shape[1]
    if w < min_side:
        w = min_side
        x -= max(0, x + w - img_w)
    if h < min_side:
        h = min_side
        y -= max(0, y + h - img_h)
    return np.array([x, y, w, h])


def extended_crop(image: np.ndarray, bbox: Sequence[float], crop_size: int, offset: float,
                  padding_value: Optional[np.ndarray] = None) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Square-resized context crop around ``bbox``.

    Returns (crop uint8 (crop_size, crop_size, 3), bbox inside the crop [x,y,w,h] float,
    context box in frame coordinates int32 [x,y,w,h])."""
    if padding_value is None:
        padding_value = np.mean(image, axis=(0, 1))
    ctx = context_box(bbox, offset)
    img_h, img_w = image.shape[:2]
    left, top = max(-ctx[0], 0), max(-ctx[1], 0)
    right, bottom = max(ctx[0] + ctx[2] - img_w, 0), max(ctx[1] + ctx[3] - img_h, 0)
    inner = image[ctx[1] + top: ctx[1] + ctx[3] - bottom, ctx[0] + left: ctx[0] + ctx[2] - right]
    padded = cv2.copyMakeBorder(inner, top, bottom, left, right, cv2.BORDER_CONSTANT, value=padding_value)
    rows, cols = padded.shape[:2]
    box = trim_box([bbox[0] - ctx[0], bbox[1] - ctx[1], bbox[2], bbox[3]], (rows, cols))
    if box[2] * box[3] == 0:
        raise IndexError("target box has zero area inside its context crop")
    crop = padded if (rows, cols) == (crop_size, crop_size) else cv2.resize(
        padded, dsize=(crop_size, crop_size), interpolation=cv2.INTER_LINEAR)
    x0, y0 = float(box[0]) / cols * crop_size, float(box[1]) / rows * crop_size
    x1, y1 = float(box[0] + box[2]) / cols * crop_size, float(box[1] + box[3]) / rows * crop_size
    return crop, np.array([x0, y0, x1 - x0, y1 - y0]), ctx


def normalize(image: np.ndarray) -> np.ndarray:
    """uint8 HWC -> float32 HWC, ImageNet statistics, same float32 operation order as the reference."""
    out = image.astype(np.float32)
    out -= _MEAN255
    out *= _INV_STD255
    return out


def rescale_bbox(bbox: Sequence[float], context: Sequence[float], instance_size: int) -> list:
    """Map a box from the 256x256 search crop back to frame pixels (python round, sides >= 3)."""
    sx, sy = context[2] / instance_size, context[3] / instance_size
    out = [round(bbox[0] * sx + context[0]), round(bbox[1] * sy + context[1]),
           max(3, round(bbox[2] * sx)), max(3, round(bbox[3] * sy))]
    return [int(v) for v in out]


# ---------------------------------------------------------------------------------------------- device crop
RESIZE_COEF_SCALE = np.float32(2048.0)  # cv::INTER_RESIZE_COEF_BITS = 11


def _axis_table(src: int, dst: int, clamp: bool):
    """Source offset + two fixed-point coefficients per destination index, as cv::resize (INTER_LINEAR, 8-bit)
    computes them: float32 position (dst + 0.5) * scale - 0.5, floor, fraction; along x the offset is clamped into
    the row and the fraction zeroed, along y only the ROW INDEX is clamped later (the kernel does that)."""
    d = np.arange(dst, dtype=np.float64)
    f = ((d + 0.5) * (float(src) / float(dst)) - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int32)
    f = (f - s.astype(np.float32)).astype(np.float32)
    if clamp:
        low, high = s < 0, s >= src - 1
        f = np.where(low | high, np.float32(0.0), f)
        s = np.where(low, 0, np.where(high, src - 1, s)).astype(np.int32)
    a0 = np.rint((np.float32(1.0) - f) * RESIZE_COEF_SCALE).astype(np.int32)
    a1 = np.rint(f * RESIZE_COEF_SCALE).astype(np.int32)
    return s, a0, a1


def resize_tables(src_w: int, src_h: int, dst: int) -> np.ndarray:
    """(6 * dst,) int32: xofs, xa0, xa1, yofs, ya0, ya1 -- the tail of fear_crop_resize_u8's parameter block."""
    return np.concatenate(_axis_table(src_w, dst, True) + _axis_table(src_h, dst, False)).astype(np.int32)


def crop_geometry(bbox: Sequence[float], crop_size: int, offset: float) -> Tuple[np.ndarray, np.ndarray]:
    """The two values ``extended_crop`` returns besides the image, without making the crop: the box inside the
    ``crop_size`` crop and the context box in frame coordinates."""
    ctx = context_box(bbox, offset)
    cols, rows = int(ctx[2]), int(ctx[3])
    box = trim_box([bbox[0] - ctx[0], bbox[1] - ctx[1], bbox[2], bbox[3]], (rows, cols))
    if box[2] * box[3] == 0:
        raise IndexError("target box has zero area inside its context crop")
    x0, y0 = float(box[0]) / cols * crop_size, float(box[1]) / rows * crop_size
    x1, y1 = float(box[0] + box[2]) / cols * crop_size, float(box[1] + box[3]) / rows * crop_size
    return np.array([x0, y0, x1 - x0, y1 - y0]), ctx


def padding_color(mean_color: np.ndarray) -> np.ndarray:
    """The int32 padding colour of a crop, cv::saturate_cast of the frame's mean colour, as copyMakeBorder takes it."""
    return np.clip(np.rint(np.asarray(mean_color, dtype=np.float64)), 0, 255).astype(np.int32)


def crop_params(bbox: Sequence[float], crop_size: int, offset: float, padding_value: np.ndarray) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Parameter block of fear_crop_resize_u8 for the context crop around ``bbox`` plus the two values
    ``extended_crop`` returns besides the image: the box inside the crop and the context box."""
    search_bbox, ctx = crop_geometry(bbox, crop_size, offset)
    cols, rows = int(ctx[2]), int(ctx[3])
    pad = padding_color(padding_value)
    head = np.array([ctx[0], ctx[1], cols, rows, pad[0], pad[1], pad[2], 0], dtype=np.int32)
    params = np.concatenate([head, resize_tables(cols, rows, crop_size)])
    return params, search_bbox, ctx


def crop_resize_reference(frame: np.ndarray, params: np.ndarray, crop_size: int) -> np.ndarray:
    """numpy model of crop_resize_u8_kernel (same integer arithmetic); used by the CPU tests to pin the kernel's
    formula to cv2.resize without a GPU."""
    cx, cy, cw, ch = (int(v) for v in params[:4])
    pad = params[4:7].astype(np.int64)
    t = params[8:].reshape(6, crop_size).astype(np.int64)
    xo, a0, a1, yo, b0, b1 = t
    h, w = frame.shape[:2]

    def px(ys, xs):
        fy, fx = cy + ys[:, None], cx + xs[None, :]
        inside = (fy >= 0) & (fy < h) & (fx >= 0) & (fx < w)
        vals = frame[np.clip(fy, 0, h - 1), np.clip(fx, 0, w - 1)].astype(np.int64)
        return np.where(inside[..., None], vals, pad[None, None, :])

    x1 = np.minimum(xo + 1, cw - 1)
    y0, y1 = np.clip(yo, 0, ch - 1), np.clip(yo + 1, 0, ch - 1)
    s0 = px(y0, xo) * a0[None, :, None] + px(y0, x1) * a1[None, :, None]
    s1 = px(y1, xo) * a0[None, :, None] + px(y1, x1) * a1[None, :, None]
    out = (((b0[:, None, None] * (s0 >> 4)) >> 16) + ((b1[:, None, None] * (s1 >> 4)) >> 16) + 2) >> 2
    return np.clip(out, 0, 255).astype(np.uint8)


# YUV matrices of YUV420Frame / FearFrameYUV: name -> (FEAR_YUV_* id, Kr, Kb)
YUV_MATRICES = {"bt601": (0, 0.299, 0.114), "bt709": (1, 0.2126, 0.0722), "bt2020": (2, 0.2627, 0.0593)}


def yuv420_to_rgb(y: np.ndarray, u: np.ndarray, v: np.ndarray, matrix: str = "bt601", full_range: bool = False,
                  bits: int = 8, shift: int = 0, transfer: Optional[str] = None) -> np.ndarray:
    """The (H, W, 3) uint8 RGB frame FEARMultiTracker sees for a YUV 4:2:0 frame: luma ``y`` (H, W), chroma ``u`` (Cb)
    and ``v`` (Cr) (H/2, W/2) of raw samples, pixel (r, c) taking chroma sample (r // 2, c // 2).  ``yuv_to_rgb`` with
    ``chroma_shift=(1, 1)``."""
    return yuv_to_rgb(y, u, v, matrix, full_range, bits, shift, (1, 1), transfer)


# HDR transfers of yuv_to_rgb and FearFrameYCbCrHDR: name -> ITU-T H.273 TransferCharacteristics code (None: 0, the
# matrix only)
HDR_TRANSFERS = {"pq": 16, "hlg": 18}

# SMPTE ST 2084 (PQ) constants; every one is exact in float64
PQ_M1, PQ_M2 = 2610.0 / 16384.0, 2523.0 / 4096.0 * 128.0
PQ_C1, PQ_C2, PQ_C3 = 3424.0 / 4096.0, 2413.0 / 4096.0 * 32.0, 2392.0 / 4096.0 * 32.0
HLG_A = 0.17883277
# The HDR chain's derived constants, folded: each is the float64 named by its hex string, which the crop kernel spells
# with the same hex literal (csrc/kernels_track_loop.cuh, kHdr*), so numpy and CUDA start from identical bits whatever
# either side's libm or constant folding would give.  HDR_CONSTANT_DERIVATIONS states how each was derived.
HDR_CONSTANTS = {
    "pq_inv_m1": float.fromhex("0x1.91c0d56e7162bp+2"),      # 1 / m1
    "pq_inv_m2": float.fromhex("0x1.9f9b5860989b1p-7"),      # 1 / m2
    "hlg_b": float.fromhex("0x1.23803fd659be6p-2"),          # 1 - 4a
    "hlg_c": float.fromhex("0x1.1eac9e800497cp-1"),          # 0.5 - a ln(4a)
    "inv_2_4": float.fromhex("0x1.aaaaaaaaaaaabp-2"),        # 1 / 2.4
    "rho_hdr_m1": float.fromhex("0x1.885043b97c4bap+3"),     # rho_HDR - 1, rho_HDR = 1 + 32 (1000 / 10000)^(1 / 2.4)
    "ln_rho_hdr": float.fromhex("0x1.4ad8a755a96c8p+1"),     # ln(rho_HDR)
    "rho_sdr": float.fromhex("0x1.6c9af449393ffp+2"),        # rho_SDR = 1 + 32 (100 / 10000)^(1 / 2.4)
    "rho_sdr_m1": float.fromhex("0x1.2c9af449393ffp+2"),     # rho_SDR - 1
}
HDR_CONSTANT_DERIVATIONS = {
    "pq_inv_m1": lambda: 1.0 / PQ_M1,
    "pq_inv_m2": lambda: 1.0 / PQ_M2,
    "hlg_b": lambda: 1.0 - 4.0 * HLG_A,
    "hlg_c": lambda: 0.5 - HLG_A * math.log(4.0 * HLG_A),
    "inv_2_4": lambda: 1.0 / 2.4,
    "rho_hdr_m1": lambda: (1.0 + 32.0 * (1000.0 / 10000.0) ** (1.0 / 2.4)) - 1.0,
    "ln_rho_hdr": lambda: math.log(1.0 + 32.0 * (1000.0 / 10000.0) ** (1.0 / 2.4)),
    "rho_sdr": lambda: 1.0 + 32.0 * (100.0 / 10000.0) ** (1.0 / 2.4),
    "rho_sdr_m1": lambda: (1.0 + 32.0 * (100.0 / 10000.0) ** (1.0 / 2.4)) - 1.0,
}

# CIE 1931 xy of the BT.2020 and BT.709 primaries (R, G, B) and of D65
BT2020_PRIMARIES = ((0.708, 0.292), (0.170, 0.797), (0.131, 0.046))
BT709_PRIMARIES = ((0.64, 0.33), (0.30, 0.60), (0.15, 0.06))
D65_WHITE = (0.3127, 0.3290)


def _inverse3(m):
    """The inverse of a 3 x 3 matrix (nested lists of Python floats) by the adjugate, each operation rounded on its
    own: no LAPACK, so every platform derives the same bits."""
    (a, b, c), (d, e, f), (g, h, i) = m
    adj = [[e * i - f * h, c * h - b * i, b * f - c * e],
           [f * g - d * i, a * i - c * g, c * d - a * f],
           [d * h - e * g, b * g - a * h, a * e - b * d]]
    det = (a * adj[0][0] + b * adj[1][0]) + c * adj[2][0]
    return [[v / det for v in row] for row in adj]


def _matmul3(p, q):
    return [[(p[r][0] * q[0][c] + p[r][1] * q[1][c]) + p[r][2] * q[2][c] for c in range(3)] for r in range(3)]


def _rgb_to_xyz(primaries, white):
    """The normalised primary matrix (SMPTE RP 177): linear RGB -> CIE XYZ for the primaries' xy and the white's xy."""
    cols = [[x / y, 1.0, ((1.0 - x) - y) / y] for x, y in primaries]
    p = [[cols[c][r] for c in range(3)] for r in range(3)]
    wx, wy = white
    w = [wx / wy, 1.0, ((1.0 - wx) - wy) / wy]
    s = [(pi[0] * w[0] + pi[1] * w[1]) + pi[2] * w[2] for pi in _inverse3(p)]
    return [[p[r][c] * s[c] for c in range(3)] for r in range(3)]


def bt2020_to_bt709_matrix() -> np.ndarray:
    """The (3, 3) float64 matrix taking linear BT.2020 RGB to linear BT.709 RGB (both D65):
    NPM(BT.709)^-1 NPM(BT.2020), derived from the primaries in Python floats in a fixed order (BT.2087's
    [[1.6605, -0.5876, -0.0728], [-0.1246, 1.1329, -0.0083], [-0.0182, -0.1006, 1.1187]] to 4 digits).  The crop
    kernel holds these nine values as hex literals (kHdrGamut)."""
    return np.array(_matmul3(_inverse3(_rgb_to_xyz(BT709_PRIMARIES, D65_WHITE)),
                             _rgb_to_xyz(BT2020_PRIMARIES, D65_WHITE)), dtype=np.float64)


def pq_eotf(e: np.ndarray) -> np.ndarray:
    """SMPTE ST 2084 EOTF: non-linear E' in [0, 1] -> display light in cd/m², each step rounded on its own."""
    k = HDR_CONSTANTS
    p = np.asarray(e, dtype=np.float64) ** k["pq_inv_m2"]
    return 10000.0 * (np.maximum(p - PQ_C1, 0.0) / (PQ_C2 - PQ_C3 * p)) ** k["pq_inv_m1"]


def hlg_inverse_oetf(e: np.ndarray) -> np.ndarray:
    """BT.2100 HLG inverse OETF: non-linear E' in [0, 1] -> normalised scene light E in [0, 1]."""
    e = np.asarray(e, dtype=np.float64)
    k = HDR_CONSTANTS
    with np.errstate(over="ignore"):  # the exp branch of codes below 1/2 is computed, then discarded
        hi = (np.exp((e - k["hlg_c"]) / HLG_A) + k["hlg_b"]) / 12.0
    return np.where(e <= 0.5, (e * e) / 3.0, hi)


def hlg_display_light(e_rgb) -> list:
    """BT.2100 HLG at Lw = 1000 cd/m², Lb = 0, system gamma 1.2: the three non-linear components -> display light in
    cd/m² per component, Fd = 1000 * Ys^0.2 * E."""
    er, eg, eb = (hlg_inverse_oetf(c) for c in e_rgb)
    ys = (0.2627 * er + 0.6780 * eg) + 0.0593 * eb
    scale = 1000.0 * ys ** 0.2
    return [scale * c for c in (er, eg, eb)]


def method_a_curve(yp: np.ndarray) -> np.ndarray:
    """BT.2446-1 Method A's tone curve Y'p -> Y'c (knots at 0.7399 and 0.9909)."""
    yp = np.asarray(yp, dtype=np.float64)
    mid = (-1.1510 * (yp * yp) + 2.7811 * yp) - 0.6302
    return np.where(yp <= 0.7399, 1.077 * yp, np.where(yp < 0.9909, mid, 0.5 * yp + 0.5))


def hdr_to_sdr(rgb, transfer: str) -> np.ndarray:
    """The (..., 3) uint8 SDR BT.709 pixels of unclamped float64 BT.2020 R'G'B' components ``rgb`` (three arrays, the
    H.273 inverse before rounding) under the HDR ``transfer`` ("pq" or "hlg"), each step rounded on its own:
    clamp to [0, 1]; display light (PQ EOTF, or HLG inverse OETF + OOTF at 1000 cd/m²); L = min(Fd / 1000, 1); BT.2446-1
    Method A tone mapping (L_HDR 1000, L_SDR 100) on L^(1/2.4); the BT.2020 inverse; clamp, ^2.4, the BT.2020 -> BT.709
    matrix, clamp, ^(1/2.4) (``hdr_to_sdr_unit``), then min(max(rint(255 v), 0), 255).  include/fear_b200.h
    (FearFrameYCbCrHDR) states the chain; the crop kernel restates this function."""
    return np.stack([np.clip(np.rint(255.0 * v), 0, 255) for v in hdr_to_sdr_unit(rgb, transfer)], -1).astype(np.uint8)


def hdr_to_sdr_unit(rgb, transfer: str) -> list:
    """``hdr_to_sdr`` before its last step: the three BT.709 R'G'B' components in [0, 1], float64."""
    k = HDR_CONSTANTS
    e = [np.clip(np.asarray(c, dtype=np.float64), 0.0, 1.0) for c in rgb]
    fd = [pq_eotf(c) for c in e] if transfer == "pq" else hlg_display_light(e)
    lin = [np.minimum(c / 1000.0, 1.0) for c in fd]
    r, g, b = (c ** k["inv_2_4"] for c in lin)
    y = (0.2627 * r + 0.6780 * g) + 0.0593 * b
    yp = np.log(1.0 + k["rho_hdr_m1"] * y) / k["ln_rho_hdr"]
    ysdr = (k["rho_sdr"] ** method_a_curve(yp) - 1.0) / k["rho_sdr_m1"]
    with np.errstate(divide="ignore", invalid="ignore"):
        f = np.where(y == 0.0, 0.0, ysdr / (1.1 * y))
    cb = (f * (b - y)) / 1.8814
    cr = (f * (r - y)) / 1.4746
    ytmo = ysdr - np.maximum(0.1 * cr, 0.0)
    r2 = ytmo + 1.4746 * cr
    b2 = ytmo + 1.8814 * cb
    g2 = ((ytmo - 0.2627 * r2) - 0.0593 * b2) / 0.6780
    lin = [np.clip(c, 0.0, 1.0) ** 2.4 for c in (r2, g2, b2)]
    m = bt2020_to_bt709_matrix()
    out = [(m[i, 0] * lin[0] + m[i, 1] * lin[1]) + m[i, 2] * lin[2] for i in range(3)]
    return [np.clip(c, 0.0, 1.0) ** k["inv_2_4"] for c in out]


def check_transfer(transfer, matrix: str, bits: int, what: str = "transfer") -> None:
    """ValueError unless ``transfer`` is None, "pq" or "hlg", and an HDR transfer comes with the BT.2020 matrix at 10
    or 12 bits."""
    if transfer is None:
        return
    if not isinstance(transfer, str) or transfer not in HDR_TRANSFERS:
        raise ValueError(f"{what} must be None, 'pq' or 'hlg', got {transfer!r}")
    if matrix != "bt2020":
        raise ValueError(f"{what} {transfer!r} needs the bt2020 matrix (BT.2100), got {matrix!r}")
    if bits == 8:
        raise ValueError(f"{what} {transfer!r} needs 10- or 12-bit samples, not 8-bit ones")


# (chroma_shift_x, chroma_shift_y) of the subsamplings FearFrameYCbCr describes: 4:2:0, 4:2:2, 4:4:4
CHROMA_SHIFTS = ((1, 1), (1, 0), (0, 0))


def yuv_to_rgb(y: np.ndarray, u: np.ndarray, v: np.ndarray, matrix: str = "bt601", full_range: bool = False,
               bits: int = 8, shift: int = 0, chroma_shift=(1, 1), transfer: Optional[str] = None) -> np.ndarray:
    """The (H, W, 3) uint8 RGB frame FEARMultiTracker sees for a YUV frame: luma ``y`` (H, W), chroma ``u`` (Cb) and
    ``v`` (Cr) of (H >> sy, W >> sx) raw samples (uint8, or uint16 at 10 / 12 bits, code = (sample >> shift) &
    (2^bits - 1)), where ``chroma_shift`` = (sx, sy) is (1, 1) for 4:2:0, (1, 0) for 4:2:2 and (0, 0) for 4:4:4, and
    pixel (r, c) takes chroma sample (r >> sy, c >> sx).  A numpy restatement of the crop kernel's conversion
    (include/fear_b200.h, FearFrameYUV and FearFrameYCbCr): for (bt601, limited, 8) cv2.cvtColor's fixed point, bit for
    bit; otherwise the ITU-T H.273 inverse in float64 with the same constants, derived in the same order, each
    operation rounded on its own, then rint (half to even) and saturation to [0, 255].

    ``transfer`` "pq" or "hlg" (BT.2020 at 10 or 12 bits only) reads the frame as HDR video: the unclamped R'G'B' of
    the H.273 inverse go through ``hdr_to_sdr`` instead of being rounded, giving the SDR BT.709 frame of BT.2446-1
    Method A tone mapping (include/fear_b200.h, FearFrameYCbCrHDR).  ``None`` is the matrix alone."""
    if matrix not in YUV_MATRICES:
        raise ValueError(f"matrix must be one of {sorted(YUV_MATRICES)}, got {matrix!r}")
    if bits not in (8, 10, 12) or not (0 <= shift <= 16 - bits) or (bits == 8 and shift):
        raise ValueError(f"bits must be 8, 10 or 12 with 0 <= shift <= 16 - bits (0 at 8 bits), got {bits}, {shift}")
    check_transfer(transfer, matrix, bits)
    sx, sy = chroma_shift
    if (sx, sy) not in CHROMA_SHIFTS:
        raise ValueError(f"chroma_shift must be one of {CHROMA_SHIFTS} (4:2:0, 4:2:2, 4:4:4), got {chroma_shift!r}")
    mask = (1 << bits) - 1
    Y = (np.asarray(y).astype(np.int64) >> shift) & mask
    U, V = ((np.asarray(c).astype(np.int64) >> shift) & mask for c in (u, v))
    U, V = (c.repeat(1 << sy, 0).repeat(1 << sx, 1) for c in (U, V))
    if U.shape != Y.shape or V.shape != Y.shape:
        raise ValueError(f"chroma of {np.shape(u)} and {np.shape(v)} does not cover luma of {Y.shape} at chroma "
                         f"shift {(sx, sy)}")
    if matrix == "bt601" and not full_range and bits == 8:  # yuv_to_rgb_bt601
        yy = np.maximum(Y - 16, 0) * 1220542 + (1 << 19)
        U, V = U - 128, V - 128
        rgb = [(yy + 1673527 * V) >> 20, (yy - 852492 * V - 409993 * U) >> 20, (yy + 2116026 * U) >> 20]
        return np.clip(np.stack(rgb, -1), 0, 255).astype(np.uint8)
    rgb = h273_rgb(Y, U, V, matrix, full_range, bits)
    if transfer is not None:
        return hdr_to_sdr(rgb, transfer)
    return np.stack([np.clip(np.rint(255.0 * c), 0, 255) for c in rgb], -1).astype(np.uint8)


def h273_rgb(Y: np.ndarray, U: np.ndarray, V: np.ndarray, matrix: str, full_range: bool, bits: int) -> list:
    """The unclamped float64 R', G', B' of the ITU-T H.273 inverse of integer codes (Y, U, V of one shape), before the
    rounding to 8 bits: the conversion of ``yuv_to_rgb`` for every format but (bt601, limited, 8)."""
    _, kr, kb = YUV_MATRICES[matrix]
    m = float(1 << (bits - 8))
    if full_range:
        y0, ys, c0 = 0.0, 1.0 / float((1 << bits) - 1), float(1 << (bits - 1))
        cs = ys
    else:
        y0, ys, c0, cs = 16.0 * m, 1.0 / (219.0 * m), 128.0 * m, 1.0 / (224.0 * m)
    kg = (1.0 - kr) - kb
    cr, cb = 2.0 * (1.0 - kr), 2.0 * (1.0 - kb)
    gb, gr = 2.0 * kb * (1.0 - kb) / kg, 2.0 * kr * (1.0 - kr) / kg
    yn = (np.asarray(Y).astype(np.float64) - y0) * ys
    pb = (np.asarray(U).astype(np.float64) - c0) * cs
    pr = (np.asarray(V).astype(np.float64) - c0) * cs
    return [yn + cr * pr, (yn - gb * pb) - gr * pr, yn + cb * pb]


def v210_row_bytes(width: int) -> int:
    """The bytes a v210 row of ``width`` pixels needs: 16 per group of 6 pixels, the last group possibly partial."""
    return 16 * -(-int(width) // 6)


def v210_pitch(width: int) -> int:
    """The row pitch capture cards and ffmpeg give a v210 row of ``width`` pixels: 128 * ceil(width / 48) bytes."""
    return 128 * -(-int(width) // 48)


def _v210_check_width(width, rows_bytes=None) -> int:
    if isinstance(width, bool) or not isinstance(width, (int, np.integer)) or width < 2 or width % 2:
        raise ValueError(f"a v210 width must be an even int >= 2, got {width!r}")
    width = int(width)
    if rows_bytes is not None and rows_bytes < v210_row_bytes(width):
        raise ValueError(f"a v210 row of {width} pixels needs {v210_row_bytes(width)} bytes, got {rows_bytes}")
    return width


def v210_unpack(words_u8: np.ndarray, width: int):
    """The (y, u, v) uint16 planes of a v210 frame: ``words_u8`` (H, pitch) uint8 are its rows as bytes, ``width`` the
    picture width (even).  y is (H, width), u (Cb) and v (Cr) are (H, width / 2) of 10-bit codes, the planes of a 4:2:2
    frame (``yuv_to_rgb(y, u, v, matrix, full_range, bits=10, chroma_shift=(1, 0))`` is the RGB frame the tracker sees
    for it).  A row is a run of 16-byte groups of four little-endian 32-bit words, each holding three 10-bit codes at bits
    0, 10 and 20 (bits 30-31 ignored); the twelve codes of a group are Cb0 Y0 Cr0 Y1 Cb1 Y2 Cr1 Y3 Cb2 Y4 Cr2 Y5 (ffmpeg's
    v210 order), pixels past ``width`` in the last group are dropped.  A numpy restatement of the crop kernel's reads
    (include/fear_b200.h, FearFrameYCbCrV210)."""
    a = np.asarray(words_u8)
    if a.dtype != np.uint8 or a.ndim != 2 or a.shape[0] < 1:
        raise ValueError(f"v210 rows must be a 2-D uint8 (H, pitch) array with H >= 1, got {a.dtype} {a.shape}")
    width = _v210_check_width(width, a.shape[1])
    groups = -(-width // 6)
    w = np.ascontiguousarray(a[:, :16 * groups]).view("<u4").reshape(a.shape[0], groups, 4)
    codes = np.stack([(w >> s) & 1023 for s in (0, 10, 20)], -1).reshape(a.shape[0], groups, 12).astype(np.uint16)
    y = codes[..., 1::2].reshape(a.shape[0], 6 * groups)[:, :width]
    u = codes[..., 0::4].reshape(a.shape[0], 3 * groups)[:, :width // 2]
    v = codes[..., 2::4].reshape(a.shape[0], 3 * groups)[:, :width // 2]
    return y, u, v


def v210_pack(y: np.ndarray, u: np.ndarray, v: np.ndarray, pitch: Optional[int] = None) -> np.ndarray:
    """The (H, pitch) uint8 v210 rows of 10-bit 4:2:2 planes: the inverse of ``v210_unpack``.  y is (H, W) with W even,
    u and v (H, W / 2), codes in [0, 1023]; ``pitch`` defaults to ``v210_pitch(W)``.  Codes of the pixels that fill out
    the last group, bits 30-31 and the bytes past the last group are 0."""
    Y, U, V = (np.asarray(p) for p in (y, u, v))
    if Y.ndim != 2 or Y.shape[0] < 1:
        raise ValueError(f"luma must be a 2-D (H, W) array with H >= 1, got shape {Y.shape}")
    h, width = Y.shape[0], _v210_check_width(Y.shape[1])
    if U.shape != (h, width // 2) or V.shape != (h, width // 2):
        raise ValueError(f"chroma must be ({h}, {width // 2}), got {U.shape} and {V.shape}")
    if any(p.size and (p.min() < 0 or p.max() > 1023) for p in (Y, U, V)):
        raise ValueError("v210 codes must be in [0, 1023]")
    pitch = v210_pitch(width) if pitch is None else int(pitch)
    if pitch < v210_row_bytes(width):
        raise ValueError(f"a v210 row of {width} pixels needs {v210_row_bytes(width)} bytes, got pitch {pitch}")
    groups = -(-width // 6)
    codes = np.zeros((h, groups, 12), dtype=np.uint32)
    for plane, first, step, n in ((Y, 1, 2, 6), (U, 0, 4, 3), (V, 2, 4, 3)):
        full = np.zeros((h, n * groups), dtype=np.uint32)
        full[:, :plane.shape[1]] = plane
        codes[..., first::step] = full.reshape(h, groups, n)
    c = codes.reshape(h, groups, 4, 3)
    words = (c[..., 0] | c[..., 1] << 10 | c[..., 2] << 20).astype("<u4")
    out = np.zeros((h, pitch), dtype=np.uint8)
    out[:, :16 * groups] = words.reshape(h, 4 * groups).view(np.uint8)
    return out


# Bayer colour filter arrays: the colours of the 2 x 2 block at pixel (0, 0), row by row (OpenCV 4.x's sensor-order
# COLOR_Bayer{RGGB,GRBG,GBRG,BGGR}2RGB) -> FearFrameBayer's pattern; pattern p has its R site at (p >> 1, p & 1)
BAYER_PATTERNS = {"RGGB": 0, "GRBG": 1, "GBRG": 2, "BGGR": 3}
# MIPI CSI-2 packings of FearFrameBayer: bits -> (pixels, bytes) per group
MIPI_GROUPS = {10: (4, 5), 12: (2, 3)}


def _bayer_pattern(pattern) -> int:
    if pattern not in BAYER_PATTERNS:
        raise ValueError(f"a Bayer pattern must be one of {sorted(BAYER_PATTERNS)}, got {pattern!r}")
    return BAYER_PATTERNS[pattern]


def bayer_demosaic(raw: np.ndarray, pattern: str = "RGGB") -> np.ndarray:
    """The (H, W, 3) RGB frame of a (H, W) Bayer mosaic at its own depth (uint8 or uint16 codes), as
    ``cv2.cvtColor(raw, cv2.COLOR_Bayer{pattern}2RGB)`` gives it for H, W >= 3.  A numpy restatement of the crop
    kernel's demosaic (include/fear_b200.h, FearFrameBayer): with N, S, W, E the neighbours and NW .. SE the diagonals,
    an R site takes G = (N + S + W + E + 2) >> 2 and B = (NW + NE + SW + SE + 2) >> 2, a B site alike with R and B
    swapped, a G site on an R row R = (W + E + 1) >> 1 and B = (N + S + 1) >> 1, on a B row the reverse; pixel (y, x) of
    the border takes the values of pixel (clamp(y, 1, H - 2), clamp(x, 1, W - 2))."""
    a = np.asarray(raw)
    if a.ndim != 2 or a.dtype not in (np.uint8, np.uint16) or a.shape[0] < 3 or a.shape[1] < 3:
        raise ValueError(f"a Bayer mosaic must be a 2-D uint8 or uint16 (H, W) array with H, W >= 3, got "
                         f"{a.dtype} {a.shape}")
    p = _bayer_pattern(pattern)
    ry, rx = p >> 1, p & 1
    h, w = a.shape
    s = a.astype(np.int64)
    c = s[1:-1, 1:-1]
    n, so, we, e = s[:-2, 1:-1], s[2:, 1:-1], s[1:-1, :-2], s[1:-1, 2:]
    cross = (n + so + we + e + 2) >> 2
    diag = (s[:-2, :-2] + s[:-2, 2:] + s[2:, :-2] + s[2:, 2:] + 2) >> 2
    hor, ver = (we + e + 1) >> 1, (n + so + 1) >> 1
    yy, xx = np.meshgrid(np.arange(1, h - 1), np.arange(1, w - 1), indexing="ij")
    r_row, r_col = ((yy ^ ry) & 1) == 0, ((xx ^ rx) & 1) == 0
    rb = r_row == r_col
    r = np.where(rb, np.where(r_row, c, diag), np.where(r_row, hor, ver))
    g = np.where(rb, cross, c)
    b = np.where(rb, np.where(r_row, diag, c), np.where(r_row, ver, hor))
    inner = np.stack([r, g, b], -1)
    rows = np.clip(np.arange(h), 1, h - 2) - 1
    cols = np.clip(np.arange(w), 1, w - 2) - 1
    return inner[rows][:, cols].astype(a.dtype)


def bayer_to_rgb(codes: np.ndarray, pattern: str = "RGGB", bits: int = 8) -> np.ndarray:
    """The (H, W, 3) uint8 RGB frame FEARMultiTracker sees for a Bayer mosaic of ``bits``-bit codes (uint8 at 8 bits,
    else uint16 codes in [0, 2^bits - 1], already unpacked and masked): ``bayer_demosaic`` at the codes' depth, then,
    above 8 bits, each channel value v mapped as full-range luma is, min(max(rint(255 * (v * (1 / (2^bits - 1)))), 0),
    255) in float64 (``yuv_to_rgb(v, c, c, full_range=True, bits=bits)`` at neutral chroma c = 2^(bits - 1))."""
    return raw_to_u8(bayer_demosaic(_raw_codes(codes, bits, "Bayer"), pattern), bits)


def _raw_codes(codes, bits: int, what: str) -> np.ndarray:
    """``codes`` as an array, checked to be ``bits``-bit codes: uint8 at 8 bits, else uint16 below 2^bits."""
    if isinstance(bits, bool) or bits not in (8, 10, 12, 14, 16):
        raise ValueError(f"{what} bits must be 8, 10, 12, 14 or 16, got {bits!r}")
    a = np.asarray(codes)
    if a.dtype != (np.uint8 if bits == 8 else np.uint16):
        raise ValueError(f"{bits}-bit {what} codes must be {'uint8' if bits == 8 else 'uint16'}, got {a.dtype}")
    if bits < 16 and a.size and int(a.max()) >= 1 << bits:
        raise ValueError(f"{bits}-bit {what} codes must be below {1 << bits}, got {int(a.max())}")
    return a


def raw_to_u8(v: np.ndarray, bits: int) -> np.ndarray:
    """``bits``-bit values v as uint8: v itself at 8 bits, above that min(max(rint(255 * (v * (1 / (2^bits - 1)))), 0),
    255) in float64, as full-range luma is mapped."""
    if bits == 8:
        return v
    ys = 1.0 / float((1 << bits) - 1)
    return np.clip(np.rint(255.0 * (v.astype(np.float64) * ys)), 0, 255).astype(np.uint8)


def mipi_row_bytes(width: int, bits: int) -> int:
    """The bytes a MIPI CSI-2 RAW10 (4 pixels in 5 bytes) or RAW12 (2 pixels in 3 bytes) row of ``width`` pixels
    needs, the last group possibly partial."""
    if bits not in MIPI_GROUPS:
        raise ValueError(f"MIPI packing is RAW10 or RAW12, got bits {bits!r}")
    px, nb = MIPI_GROUPS[bits]
    return nb * -(-int(width) // px)


def mipi_unpack(buf: np.ndarray, width: int, bits: int) -> np.ndarray:
    """The (H, width) uint16 codes of MIPI CSI-2 RAW10 / RAW12 rows ``buf`` ((H, pitch) uint8, pitch >= the row bytes;
    bytes past the last group are not read).  RAW10: bytes 0-3 of a group are bits 9..2 of pixels 0..3, byte 4 is
    P3[1:0] << 6 | P2[1:0] << 4 | P1[1:0] << 2 | P0[1:0]; RAW12: bytes 0-1 are bits 11..4 of pixels 0, 1, byte 2 is
    P1[3:0] << 4 | P0[3:0].  A numpy restatement of the crop kernel's reads (include/fear_b200.h, FearFrameBayer)."""
    a = np.asarray(buf)
    if a.dtype != np.uint8 or a.ndim != 2 or a.shape[0] < 1:
        raise ValueError(f"MIPI rows must be a 2-D uint8 (H, pitch) array, got {a.dtype} {a.shape}")
    if isinstance(width, bool) or not isinstance(width, (int, np.integer)) or width < 1:
        raise ValueError(f"a MIPI row width must be an int >= 1, got {width!r}")
    need = mipi_row_bytes(width, bits)
    if a.shape[1] < need:
        raise ValueError(f"a RAW{bits} row of {width} pixels needs {need} bytes, got {a.shape[1]}")
    px, nb = MIPI_GROUPS[bits]
    g = a[:, :need].reshape(a.shape[0], -1, nb).astype(np.uint16)
    lo_bits = bits - 8
    lo = np.stack([(g[..., px] >> (lo_bits * i)) & ((1 << lo_bits) - 1) for i in range(px)], -1)
    codes = (g[..., :px] << lo_bits) | lo
    return codes.reshape(a.shape[0], -1)[:, :int(width)]


def mipi_pack(codes: np.ndarray, bits: int, pitch: Optional[int] = None) -> np.ndarray:
    """The (H, pitch) uint8 MIPI CSI-2 RAW10 / RAW12 rows of (H, W) codes in [0, 2^bits): the inverse of
    ``mipi_unpack``.  ``pitch`` defaults to the row bytes; the pixels that fill out the last group and the bytes past
    it are 0."""
    c = np.asarray(codes)
    if c.ndim != 2 or c.shape[0] < 1 or c.shape[1] < 1:
        raise ValueError(f"codes must be a 2-D (H, W) array, got shape {c.shape}")
    need = mipi_row_bytes(c.shape[1], bits)
    if c.size and (c.min() < 0 or c.max() >= 1 << bits):
        raise ValueError(f"RAW{bits} codes must be in [0, {(1 << bits) - 1}]")
    pitch = need if pitch is None else int(pitch)
    if pitch < need:
        raise ValueError(f"a RAW{bits} row of {c.shape[1]} pixels needs {need} bytes, got pitch {pitch}")
    px, nb = MIPI_GROUPS[bits]
    h, groups, lo_bits = c.shape[0], need // nb, bits - 8
    full = np.zeros((h, groups * px), dtype=np.uint32)
    full[:, :c.shape[1]] = c
    full = full.reshape(h, groups, px)
    g = np.zeros((h, groups, nb), dtype=np.uint32)
    g[..., :px] = full >> lo_bits
    for i in range(px):
        g[..., px] |= (full[..., i] & ((1 << lo_bits) - 1)) << (lo_bits * i)
    out = np.zeros((h, pitch), dtype=np.uint8)
    out[:, :need] = g.reshape(h, need)
    return out


# FearFrameMono's gain control: None -> 0, "minmax" -> FEAR_AGC_MINMAX
AGC_MODES = {None: 0, "minmax": 1}


def check_agc(agc, what: str = "agc") -> None:
    if not isinstance(agc, (str, type(None))) or agc not in AGC_MODES:
        raise ValueError(f"{what} must be None or \"minmax\", got {agc!r}")


def fma_f32(v: np.ndarray, a: np.float32, b: np.float32) -> np.ndarray:
    """float32 fmaf(v, a, b) elementwise, rounded once (v integers below 2^24, a and b float32): v * a is exact in
    float64; the float64 sum s and its exact error e (TwoSum) fix the one case where rounding s to float32 differs from
    rounding v * a + b, an s that lies on a float32 midpoint while e != 0."""
    p = np.asarray(v).astype(np.float64) * np.float64(a)
    b64 = np.float64(b)
    s = p + b64
    bb = s - p
    e = (p - (s - bb)) + (b64 - bb)
    r = s.astype(np.float32)
    toward = np.nextafter(r, np.where(e > 0, np.float32(np.inf), np.float32(-np.inf)).astype(np.float32))
    tie = (e != 0) & ((r.astype(np.float64) + toward.astype(np.float64)) * 0.5 == s)
    return np.where(tie, toward, r)


def minmax_gain(lo: int, hi: int):
    """The float32 (a, b) that cv2.normalize(src, None, 0, 255, NORM_MINMAX, CV_8U) passes to convertTo for codes in
    [lo, hi]: OpenCV 4.13 computes scale = (dmax - dmin) * (smax - smin > DBL_EPSILON ? 1 / (smax - smin) : 0) and
    shift = dmin - smin * scale in float64 (dmin = 0, dmax = 255), and convertTo to uint8 takes them as float."""
    d = float(hi) - float(lo)
    scale = 255.0 * (1.0 / d if d > np.finfo(np.float64).eps else 0.0)
    shift = 0.0 - float(lo) * scale
    return np.float32(scale), np.float32(shift)


def minmax_normalize(codes: np.ndarray) -> np.ndarray:
    """cv2.normalize(codes, None, 0, 255, cv2.NORM_MINMAX, dtype=cv2.CV_8U) of uint8 or uint16 codes, bit for bit:
    with lo, hi the smallest and largest code and (a, b) = ``minmax_gain(lo, hi)``, each code v becomes
    saturate_cast<uchar>(fmaf(v, a, b)) = min(max(rint(fmaf(v, a, b)), 0), 255).  A constant frame gives 0."""
    a = np.asarray(codes)
    if a.size == 0:
        return np.zeros(a.shape, np.uint8)
    ga, gb = minmax_gain(int(a.min()), int(a.max()))
    return np.clip(np.rint(fma_f32(a, ga, gb)), 0, 255).astype(np.uint8)


def mono_to_rgb(codes: np.ndarray, bits: int = 8, agc: Optional[str] = None) -> np.ndarray:
    """The (H, W, 3) uint8 RGB frame FEARMultiTracker sees for a single-channel frame of ``bits``-bit codes (uint8 at 8
    bits, else uint16 codes in [0, 2^bits - 1], already unpacked and shifted: ``mipi_unpack`` for packed rows):
    ``cv2.cvtColor(g, cv2.COLOR_GRAY2RGB)`` of the 8-bit grey image g.  Without gain control g is the code at 8 bits,
    above it the code mapped as ``bayer_to_rgb`` maps a channel; with ``agc="minmax"`` g is ``minmax_normalize`` of the
    whole frame's codes, cv2.normalize(codes, None, 0, 255, NORM_MINMAX, CV_8U)."""
    check_agc(agc)
    a = _raw_codes(codes, bits, "mono")
    if a.ndim != 2:
        raise ValueError(f"mono codes must be a 2-D (H, W) array, got shape {a.shape}")
    g = minmax_normalize(a) if agc == "minmax" else raw_to_u8(a, bits)
    return np.repeat(g[..., None], 3, axis=-1)


# Packed RGB layouts by ffmpeg pix_fmt name: sample type, samples per pixel, and the sample indices of R, G and B
RGB_PACKED_LAYOUTS = {
    "rgb24": (np.uint8, 3, (0, 1, 2)), "bgr24": (np.uint8, 3, (2, 1, 0)),
    "rgba": (np.uint8, 4, (0, 1, 2)), "bgra": (np.uint8, 4, (2, 1, 0)), "argb": (np.uint8, 4, (1, 2, 3)),
    "abgr": (np.uint8, 4, (3, 2, 1)), "rgb0": (np.uint8, 4, (0, 1, 2)), "bgr0": (np.uint8, 4, (2, 1, 0)),
    "0rgb": (np.uint8, 4, (1, 2, 3)), "0bgr": (np.uint8, 4, (3, 2, 1)),
    "rgb48le": (np.uint16, 3, (0, 1, 2)), "bgr48le": (np.uint16, 3, (2, 1, 0)),
    "rgba64le": (np.uint16, 4, (0, 1, 2)), "bgra64le": (np.uint16, 4, (2, 1, 0)),
}
# 10-bit RGB in one little-endian 32-bit word (the top 2 bits spare): the bit offsets of R, G and B
X2RGB10_LAYOUTS = {"x2rgb10le": (20, 10, 0), "x2bgr10le": (0, 10, 20)}
# the depths of planar RGB (ffmpeg's gbrp, gbrp10le, gbrp12le, gbrp16le): uint8 at 8 bits, else LSB-aligned uint16
RGB_PLANAR_BITS = (8, 10, 12, 16)


def x2rgb10_pack(codes: np.ndarray, layout: str = "x2rgb10le", spare: Optional[np.ndarray] = None) -> np.ndarray:
    """The (H, W) uint32 words of (H, W, 3) RGB codes in [0, 1023] in ``layout`` ("x2rgb10le": B in bits 0-9, G in
    10-19, R in 20-29; "x2bgr10le": R, G, B from bit 0), with ``spare`` (values in [0, 3], default 0) in bits 30-31."""
    shifts = X2RGB10_LAYOUTS[layout]
    c = np.asarray(codes)
    if c.ndim != 3 or c.shape[2] != 3 or (c.size and (c.min() < 0 or c.max() > 1023)):
        raise ValueError(f"x2rgb10 codes must be an (H, W, 3) array in [0, 1023], got {c.dtype} {c.shape}")
    w = np.zeros(c.shape[:2], dtype=np.uint32)
    for ch, s in enumerate(shifts):
        w |= c[..., ch].astype(np.uint32) << np.uint32(s)
    if spare is not None:
        w |= (np.asarray(spare).astype(np.uint32) & np.uint32(3)) << np.uint32(30)
    return w


def x2rgb10_unpack(words: np.ndarray, layout: str = "x2rgb10le") -> np.ndarray:
    """The (H, W, 3) uint16 RGB codes of (H, W) 32-bit words in ``layout``; the 2 spare bits are not read."""
    shifts = X2RGB10_LAYOUTS[layout]
    w = np.asarray(words).view(np.uint32)
    return np.stack([(w >> np.uint32(s)) & np.uint32(1023) for s in shifts], -1).astype(np.uint16)


def rgb_frame_to_rgb(data, layout: str, bits: Optional[int] = None) -> np.ndarray:
    """The (H, W, 3) uint8 RGB frame FEARMultiTracker sees for an RGBFrame of ``layout`` holding ``data``:
        a packed layout (RGB_PACKED_LAYOUTS)   data (H, W, C) samples of the layout's type; R, G, B picked out, and at
                                               16 bits each mapped by ``raw_to_u8``
        "x2rgb10le" / "x2bgr10le"              data (H, W) 32-bit words: ``x2rgb10_unpack``, then ``raw_to_u8`` at 10
        "planar"                               data the R, G and B planes ((3, H, W) or three (H, W)), ``bits`` 8, 10,
                                               12 or 16: uint8 at 8 bits, else uint16 whose low ``bits`` bits are the
                                               code (the high bits are not read), mapped by ``raw_to_u8``
    At 8 bits this is cv2.cvtColor(data, COLOR_BGR2RGB / COLOR_BGRA2RGB / COLOR_RGBA2RGB) for the layouts cv2 names."""
    if layout in RGB_PACKED_LAYOUTS:
        dtype, n, idx = RGB_PACKED_LAYOUTS[layout]
        a = np.asarray(data)
        if a.dtype != dtype or a.ndim != 3 or a.shape[2] != n:
            raise ValueError(f"{layout} data must be (H, W, {n}) {np.dtype(dtype).name}, got {a.dtype} {a.shape}")
        return raw_to_u8(a[..., list(idx)], 8 if dtype == np.uint8 else 16)
    if layout in X2RGB10_LAYOUTS:
        a = np.asarray(data)
        if a.dtype not in (np.uint32, np.int32) or a.ndim != 2:
            raise ValueError(f"{layout} data must be (H, W) 32-bit words, got {a.dtype} {a.shape}")
        return raw_to_u8(x2rgb10_unpack(a, layout), 10)
    if layout == "planar":
        if isinstance(bits, bool) or bits not in RGB_PLANAR_BITS:
            raise ValueError(f"planar RGB bits must be 8, 10, 12 or 16, got {bits!r}")
        a = np.stack([np.asarray(p) for p in data])
        if a.dtype != (np.uint8 if bits == 8 else np.uint16) or a.ndim != 3 or a.shape[0] != 3:
            raise ValueError(f"planar RGB at {bits} bits takes three (H, W) {'uint8' if bits == 8 else 'uint16'} "
                             f"planes, got {a.dtype} {a.shape}")
        codes = np.moveaxis(a, 0, -1)
        if bits not in (8, 16):
            codes = codes & np.uint16((1 << bits) - 1)
        return raw_to_u8(codes, bits)
    raise ValueError(f"unknown RGB layout {layout!r}")


ORIENT_ROTATIONS = (0, 90, 180, 270)  # the clockwise turns of an orientation code, code & 3 = rotate / 90


def orient_code(rotate: int = 0, mirror: bool = False) -> int:
    """The orientation code of a clockwise turn by ``rotate`` degrees (0, 90, 180 or 270) after a left-right flip when
    ``mirror``: rotate / 90, plus 4 when mirrored.  ffmpeg's autorotate turns a display-matrix rotation of r degrees
    (ffprobe's ``rotation=-90``) by rotate = (-r) mod 360 (here 90)."""
    if isinstance(rotate, (bool, np.bool_)) or not isinstance(rotate, (int, np.integer)) \
            or int(rotate) not in ORIENT_ROTATIONS:
        raise ValueError(f"rotate must be 0, 90, 180 or 270 (degrees clockwise), got {rotate!r}")
    return int(rotate) // 90 + (4 if mirror else 0)


def orient(rgb: np.ndarray, code: int) -> np.ndarray:
    """The frame a tracker sees for orientation ``code`` in [0, 7]: ``rgb`` (H, W, ...) turned 90 * (code & 3) degrees
    clockwise, after a left-right flip when code & 4.  Display pixel (y, x) is stored pixel (ys, xs):
        code & 3 = 0: (y, x);  1: (H - 1 - x, y);  2: (H - 1 - y, W - 1 - x);  3: (x, W - 1 - y)
    then xs = W - 1 - xs when mirrored; the display is W x H for odd codes.  A view, no copy: for host frames this is
    the whole of orientation (pass ``np.ascontiguousarray`` of it, or the view, to a tracker)."""
    return np.rot90(rgb[:, ::-1] if code & 4 else rgb, -(code & 3))
