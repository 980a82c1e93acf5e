"""HDR test material: SDR RGB frames made into PQ or HLG BT.2020 code planes the BT.2408 way, and the frame wrappers the
HDR tests, the poison check and tools/bench_hdr.py feed the trackers.

    codes = hdr_codes(rgb, "pq", bits=10, full_range=False, sub="420")   # (y, u, v) integer code planes

SDR white goes to 203 cd/m²: the SDR frame is linearised (^2.4), taken from BT.709 to BT.2020 primaries, scaled to
203 cd/m² and encoded with the PQ inverse EOTF, or for HLG with BT.2100's inverse OOTF (1000 cd/m², gamma 1.2) and
the OETF; then the BT.2020 non-constant-luminance matrix, chroma averaged over each chroma sample's pixels."""
import numpy as np
import torch

import feartracker_b200 as fb
from feartracker_b200 import image_ops

SHIFTS = {"420": (1, 1), "422": (1, 0), "444": (0, 0)}
SDR_WHITE = 203.0


def pq_inverse_eotf(fd):
    y = (np.asarray(fd, dtype=np.float64) / 10000.0) ** image_ops.PQ_M1
    return ((image_ops.PQ_C1 + image_ops.PQ_C2 * y) / (1.0 + image_ops.PQ_C3 * y)) ** image_ops.PQ_M2


def hlg_oetf(e):
    e = np.asarray(e, dtype=np.float64)
    a, b, c = image_ops.HLG_A, image_ops.HDR_CONSTANTS["hlg_b"], image_ops.HDR_CONSTANTS["hlg_c"]
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(e <= 1.0 / 12.0, np.sqrt(3.0 * e), a * np.log(np.maximum(12.0 * e - b, 1e-300)) + c)


def hdr_rgb(rgb: np.ndarray, transfer: str) -> list:
    """The non-linear BT.2020 R'G'B' (three float64 planes in [0, 1]) of an SDR uint8 RGB frame, SDR white at 203
    cd/m²."""
    lin = [(rgb[..., c].astype(np.float64) / 255.0) ** 2.4 for c in range(3)]
    m = np.linalg.inv(image_ops.bt2020_to_bt709_matrix())
    fd = [SDR_WHITE * (m[i, 0] * lin[0] + m[i, 1] * lin[1] + m[i, 2] * lin[2]) for i in range(3)]
    fd = [np.clip(c, 0.0, 10000.0) for c in fd]
    if transfer == "pq":
        return [pq_inverse_eotf(c) for c in fd]
    yd = 0.2627 * fd[0] + 0.6780 * fd[1] + 0.0593 * fd[2]
    scale = np.where(yd > 0, (np.maximum(yd, 1e-300) / 1000.0) ** ((1.0 - 1.2) / 1.2), 0.0)
    return [hlg_oetf(np.clip(c / 1000.0 * scale, 0.0, 1.0)) for c in fd]


def encode_rgb(planes: list, bits: int, full_range: bool, sub: str) -> tuple:
    """Integer (y, u, v) code planes of non-linear BT.2020 R'G'B' planes: BT.2020 non-constant-luminance Y'CbCr,
    chroma the mean over each chroma sample's pixels."""
    r, g, b = planes
    yn = 0.2627 * r + 0.6780 * g + 0.0593 * b
    pb, pr = (b - yn) / 1.8814, (r - yn) / 1.4746
    h, w = yn.shape
    sx, sy = SHIFTS[sub]
    pb, pr = (p.reshape(h >> sy, 1 << sy, w >> sx, 1 << sx).mean(axis=(1, 3)) for p in (pb, pr))
    m, top = 1 << (bits - 8), (1 << bits) - 1
    if full_range:
        y, u, v = yn * top, (1 << (bits - 1)) + pb * top, (1 << (bits - 1)) + pr * top
    else:
        y, u, v = 16 * m + 219 * m * yn, 128 * m + 224 * m * pb, 128 * m + 224 * m * pr
    return tuple(np.clip(np.rint(p), 0, top).astype(np.int64) for p in (y, u, v))


def hdr_codes(rgb: np.ndarray, transfer: str, bits: int = 10, full_range: bool = False, sub: str = "420") -> tuple:
    return encode_rgb(hdr_rgb(rgb, transfer), bits, full_range, sub)


def p010_frame(y, u, v, bits: int = 10, pitch_pad: int = 64, **fmt) -> fb.YUV420Frame:
    """NVDEC's P010 / P016 layout: an MSB-aligned uint16 NV12 surface with ``pitch_pad`` samples of row pitch past the
    picture, 0xA5A5 there and noise in the low bits, wrapped by YUV420Frame.nv12."""
    h, w = y.shape
    surf = np.full((h * 3 // 2, w + pitch_pad), 0xA5A5, np.uint16)
    noise = np.random.default_rng(h * w).integers(0, 1 << (16 - bits), (h * 3 // 2, w))
    codes = np.concatenate([y, np.stack([u, v], -1).reshape(h // 2, w)]).astype(np.int64)
    surf[:, :w] = (codes << (16 - bits)) | noise
    t = torch.from_numpy(surf.view(np.int16)).view(torch.uint16).cuda()
    return fb.YUV420Frame.nv12(t[:, :w], bits=bits, **fmt)


def i420_frame(y, u, v, bits: int = 10, **fmt) -> fb.YUV420Frame:
    """ffmpeg's yuv420p10le / yuv420p12le: LSB-aligned contiguous planes, noise in the high bits."""
    flat = np.concatenate([np.asarray(p).reshape(-1) for p in (y, u, v)]).astype(np.int64)
    flat |= np.random.default_rng(flat.size).integers(0, 1 << (16 - bits), flat.size) << bits
    t = torch.from_numpy(flat.astype(np.uint16).view(np.int16).reshape(-1, y.shape[1])).view(torch.uint16).cuda()
    return fb.YUV420Frame.i420(t, bits=bits, **fmt)


def v210_frame(y, u, v, col: int = 0, **fmt) -> fb.V210Frame:
    """10-bit 4:2:2 code planes as a V210Frame at the capture cards' pitch, at byte column ``col`` of a larger surface."""
    rows = image_ops.v210_pack(np.asarray(y), np.asarray(u), np.asarray(v))
    h, pitch = rows.shape
    surf = np.full((h, pitch + col + 64), 0xA5, np.uint8)
    surf[:, col:col + pitch] = rows
    w = np.shape(y)[1]
    return fb.V210Frame(torch.from_numpy(surf).cuda()[:, col:col + image_ops.v210_row_bytes(w)], w, **fmt)
