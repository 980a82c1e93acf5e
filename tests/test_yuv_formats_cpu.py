"""CPU: YUV420Frame's colour formats, the FearFrameYUV records it builds, and image_ops.yuv420_to_rgb, the numpy
restatement of the kernels' conversion that the GPU tests compare against.

The restatement is pinned three ways: the default format against cv2.cvtColor on all 2^24 (Y, U, V) triples; every
other format against the exact rational value of the ITU-T H.273 equations (fractions, decimal Kr and Kb); and full
range BT.601 against PIL's independent YCbCr -> RGB conversion."""
import itertools
from fractions import Fraction

import cv2
import numpy as np
import pytest
import torch
from PIL import Image

import feartracker_b200 as fb
from feartracker_b200 import _lib, image_ops
from tests.test_yuv_frames_cpu import LAYOUTS, _tracker, split_i420, yuv_frame

MATRICES = ("bt601", "bt709", "bt2020")
FORMATS = [(m, f, b) for b in (8, 10, 12) for m in MATRICES for f in (False, True)]
NON_DEFAULT = [fmt for fmt in FORMATS if fmt != ("bt601", False, 8)]
WIDE_LAYOUTS = ("p010", "p010_pitched", "planes16", "i420_10le", "roi16")


def yuv16_frame(y: np.ndarray, u: np.ndarray, v: np.ndarray, layout: str, device="cuda", **fmt) -> fb.YUV420Frame:
    """uint16 sample planes (already aligned as the layout stores them) as a freshly allocated YUV420Frame on
    ``device``: contiguous P010 / P016 (NV12 layout), the same with a row pitch of 1024 samples or more, separate Y and
    interleaved UV allocations, contiguous yuv420p10le (I420 layout), or the region at luma offset (2, 4) of a larger
    P010 surface.  Samples outside the frame are 0xA5A5."""
    h, w = y.shape
    uv = np.stack([u, v], -1).reshape(h // 2, w)
    nv = np.concatenate([y, uv])

    def dev(a):
        return torch.from_numpy(np.ascontiguousarray(a).view(np.int16)).view(torch.uint16).to(device)

    def fill(shape):
        return torch.full(shape, 0xA5A5 - 65536, dtype=torch.int16, device=device).view(torch.uint16)

    if layout == "p010":
        return fb.YUV420Frame.nv12(dev(nv), **fmt)
    if layout == "p010_pitched":
        surface = fill((nv.shape[0], 1024 * (w // 1024 + 1)))
        surface[:, :w] = dev(nv)
        return fb.YUV420Frame.nv12(surface[:, :w], **fmt)
    if layout == "planes16":
        luma, chroma = dev(y), dev(uv)
        return fb.YUV420Frame(luma, chroma[:, 0::2], chroma[:, 1::2], msb=True, **fmt)
    if layout == "i420_10le":
        return fb.YUV420Frame.i420(dev(np.concatenate([y.reshape(-1), u.reshape(-1), v.reshape(-1)]).reshape(-1, w)),
                                   **fmt)
    if layout == "roi16":
        hb = h + 6
        big = fill((hb * 3 // 2, w + 10))
        big[2:2 + h, 4:4 + w] = dev(y)
        big[hb + 1:hb + 1 + h // 2, 4:4 + w] = dev(uv)
        c = big[hb + 1:hb + 1 + h // 2]
        return fb.YUV420Frame(big[2:2 + h, 4:4 + w], c[:, 4:4 + w:2], c[:, 5:5 + w:2], msb=True, **fmt)
    raise ValueError(layout)


def test_yuv_record_is_80_bytes():
    assert _lib.YUV_DTYPE.itemsize == 80
    assert _lib.YUV_DTYPE.names == ("y", "u", "v", "y_row_stride", "y_pixel_stride", "uv_row_stride",
                                    "uv_pixel_stride", "H", "W", "matrix", "full_range", "bits", "shift")


def _read_back(f: fb.YUV420Frame, want_planes, dtype):
    rec = np.array([f.yuv_record()], dtype=_lib.YUV_DTYPE)[0]
    assert (int(rec["H"]), int(rec["W"])) == f.shape[:2]
    strides = {"y": (rec["y_row_stride"], rec["y_pixel_stride"]), "u": (rec["uv_row_stride"], rec["uv_pixel_stride"]),
               "v": (rec["uv_row_stride"], rec["uv_pixel_stride"])}
    for name, want in zip("yuv", want_planes):
        plane = getattr(f, name)
        storage = np.frombuffer(bytes(plane.untyped_storage()), dtype=np.uint8)
        off = int(rec[name]) - plane.untyped_storage().data_ptr()
        rs, ps = (int(s) for s in strides[name])
        r, c = np.meshgrid(np.arange(want.shape[0]), np.arange(want.shape[1]), indexing="ij")
        at = off + r * rs + c * ps
        got = storage[at] if dtype == np.uint8 else storage[at] | (storage[at + 1].astype(np.uint16) << 8)
        assert np.array_equal(got, want), name
    return rec


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("hw", [(2, 2), (6, 10), (90, 334)])
def test_yuv_record_of_8_bit_frames_addresses_the_planes(layout, hw):
    h, w = hw
    i420 = np.random.default_rng(h * w).integers(0, 256, (h * 3 // 2, w), dtype=np.uint8)
    f = yuv_frame(i420, layout, device="cpu")
    rec = _read_back(f, split_i420(i420), np.uint8)
    assert tuple(int(rec[k]) for k in ("matrix", "full_range", "bits", "shift")) == (0, 0, 8, 0)
    assert f.yuv_record()[:9] == f.record()


@pytest.mark.parametrize("layout", WIDE_LAYOUTS)
@pytest.mark.parametrize("hw", [(2, 2), (6, 10), (90, 334)])
@pytest.mark.parametrize("bits", [10, 12])
def test_yuv_record_of_16_bit_frames_addresses_the_planes(layout, hw, bits):
    h, w = hw
    rng = np.random.default_rng(h * w + bits)
    planes = [rng.integers(0, 65536, s, dtype=np.uint16) for s in ((h, w), (h // 2, w // 2), (h // 2, w // 2))]
    f = yuv16_frame(*planes, layout, device="cpu", matrix="bt2020", full_range=True, bits=bits)
    rec = _read_back(f, planes, np.uint16)
    msb = layout not in ("i420_10le",)
    assert tuple(int(rec[k]) for k in ("matrix", "full_range", "bits", "shift")) == (2, 1, bits, 16 - bits if msb
                                                                                      else 0)
    assert all(int(rec[k]) % 2 == 0 for k in ("y", "u", "v", "y_row_stride", "y_pixel_stride", "uv_row_stride",
                                                 "uv_pixel_stride"))
    if layout == "p010_pitched":
        assert rec["y_row_stride"] >= 2048 and rec["uv_pixel_stride"] == 4 and int(rec["v"]) - int(rec["u"]) == 2


def test_p010_record_follows_the_documented_layout():
    h, w, p = 6, 10, 512  # p: row pitch in bytes
    surface = torch.zeros(h * 3 // 2, p // 2, dtype=torch.uint16)
    b = surface.data_ptr()
    assert fb.YUV420Frame.nv12(surface[:, :w], matrix="bt709", bits=10).yuv_record() == \
        (b, b + h * p, b + h * p + 2, p, 2, p, 4, h, w, 1, 0, 10, 6)
    packed = torch.zeros(h * 3 // 2, w, dtype=torch.uint16)
    b, q = packed.data_ptr(), h * w // 4
    assert fb.YUV420Frame.i420(packed, full_range=True, bits=12).yuv_record() == \
        (b, b + 2 * h * w, b + 2 * (h * w + q), 2 * w, 2, w, 2, h, w, 0, 1, 12, 0)


def _u8(h, w):
    return torch.zeros(h, w, dtype=torch.uint8)


def _u16(h, w):
    return torch.zeros(h, w, dtype=torch.uint16)


BAD_FORMATS = {
    "bits 10, uint8 planes": lambda: fb.YUV420Frame(_u8(64, 80), _u8(32, 40), _u8(32, 40), bits=10),
    "bits 10, uint8 nv12": lambda: fb.YUV420Frame.nv12(_u8(96, 80), bits=10),
    "bits 12, uint8 i420": lambda: fb.YUV420Frame.i420(_u8(96, 80), bits=12),
    "bits 8, uint16 planes": lambda: fb.YUV420Frame(_u16(64, 80), _u16(32, 40), _u16(32, 40)),
    "bits 8, uint16 nv12": lambda: fb.YUV420Frame.nv12(_u16(96, 80)),
    "bits 8, uint16 i420": lambda: fb.YUV420Frame.i420(_u16(96, 80)),
    "bits 10, int16 planes": lambda: fb.YUV420Frame(*(p.view(torch.int16) for p in (_u16(64, 80), _u16(32, 40),
                                                                                      _u16(32, 40))), bits=10),
    "bits 10, mixed dtypes": lambda: fb.YUV420Frame(_u16(64, 80), _u8(32, 40), _u8(32, 40), bits=10),
    "bits 9": lambda: fb.YUV420Frame(_u16(64, 80), _u16(32, 40), _u16(32, 40), bits=9),
    "bits 16": lambda: fb.YUV420Frame.nv12(_u16(96, 80), bits=16),
    "unknown matrix": lambda: fb.YUV420Frame.nv12(_u8(96, 80), matrix="bt470"),
    "matrix by number": lambda: fb.YUV420Frame.i420(_u8(96, 80), matrix=1),
    "msb at 8 bits": lambda: fb.YUV420Frame(_u8(64, 80), _u8(32, 40), _u8(32, 40), msb=True),
    "odd W at 10 bits": lambda: fb.YUV420Frame.nv12(_u16(96, 81), bits=10),
}


@pytest.mark.parametrize("what", list(BAD_FORMATS))
def test_bad_formats_are_refused_before_device_calls(what):
    make = BAD_FORMATS[what]
    trk = _tracker()
    with pytest.raises(ValueError):
        trk.add(make(), [[10, 10, 20, 20]])
    trk._ids, trk._streams = np.array([0]), np.array([0])
    with pytest.raises(ValueError):
        trk.update(make())


@pytest.mark.parametrize("fmt", NON_DEFAULT)
def test_record_of_non_default_format_is_refused(fmt):
    matrix, full, bits = fmt
    t = (_u8 if bits == 8 else _u16)(96, 80)
    f = fb.YUV420Frame.nv12(t, matrix=matrix, full_range=full, bits=bits)
    assert not f.default_format
    with pytest.raises(ValueError):
        f.record()
    assert f.yuv_record()[9:12] == (image_ops.YUV_MATRICES[matrix][0], int(full), bits)


# ---------------------------------------------------------------------------------------------------- the oracle
def test_oracle_refuses_unknown_formats():
    y, c = np.zeros((2, 2), np.uint8), np.zeros((1, 1), np.uint8)
    for kw in (dict(matrix="bt470"), dict(bits=9), dict(bits=8, shift=1), dict(bits=10, shift=7),
               dict(bits=12, shift=-1)):
        with pytest.raises(ValueError):
            image_ops.yuv420_to_rgb(y, c, c, **kw)


def _all_triple_frames():
    """64 frames of 512 x 512 that hold every 8-bit (Y, U, V) triple: chroma block (i, j) is (U, V) = (i, j), and the
    luma of 2 x 2 position (dy, dx) in frame k is 4k + 2dy + dx (the frames of test_gpu_yuv_frames)."""
    u, v = np.meshgrid(np.arange(256, dtype=np.uint8), np.arange(256, dtype=np.uint8), indexing="ij")
    for k in range(64):
        y = np.empty((512, 512), np.uint8)
        for dy in range(2):
            for dx in range(2):
                y[dy::2, dx::2] = 4 * k + 2 * dy + dx
        yield y, u, v


def test_oracle_default_format_is_cv2_on_every_triple():
    for y, u, v in _all_triple_frames():
        i420 = np.concatenate([y.reshape(-1), u.reshape(-1), v.reshape(-1)]).reshape(768, 512)
        assert np.array_equal(image_ops.yuv420_to_rgb(y, u, v), cv2.cvtColor(i420, cv2.COLOR_YUV2RGB_I420))


def test_oracle_full_range_bt601_is_within_one_of_pil_on_every_triple():
    """PIL's YCbCr -> RGB (JPEG's full-range BT.601, its own fixed point) is an independent implementation: a swapped
    or mis-signed coefficient would be far more than 1 away."""
    ones, total = 0, 0
    for y, u, v in _all_triple_frames():
        ycc = np.stack([y, u.repeat(2, 0).repeat(2, 1), v.repeat(2, 0).repeat(2, 1)], -1)
        want = np.asarray(Image.fromarray(ycc, "YCbCr").convert("RGB")).astype(np.int16)
        d = np.abs(image_ops.yuv420_to_rgb(y, u, v, full_range=True).astype(np.int16) - want)
        assert d.max() <= 1
        ones += int((d == 1).sum())
        total += d.size
    print(f"full-range BT.601 vs PIL: {ones / total:.1%} of channel values differ by 1, none by more")


def extreme_codes(bits):
    m = 1 << (bits - 8)
    return sorted({0, 16 * m, 128 * m, 235 * m, 240 * m, (1 << bits) - 1})


def format_codes(bits, n=100_000, seed=0):
    """n seeded (Y, U, V) code triples of a bit depth, then every triple of its range extremes."""
    rng = np.random.default_rng(seed + bits)
    ext = np.array(list(itertools.product(extreme_codes(bits), repeat=3)), dtype=np.int64)
    return np.concatenate([rng.integers(0, 1 << bits, (n, 3)), ext])


def exact_rgb(codes, matrix, full_range, bits):
    """(rgb, near_half): round-half-even of 255 x the exact rational H.273 value of each channel, saturated, and where
    that value lies within 1e-9 of a half-integer.  Python integers throughout."""
    _, kr, kb = image_ops.YUV_MATRICES[matrix]
    kr, kb = Fraction(str(kr)), Fraction(str(kb))
    m = 1 << (bits - 8)
    if full_range:
        y0, ys, c0, cs = 0, Fraction(1, (1 << bits) - 1), 1 << (bits - 1), Fraction(1, (1 << bits) - 1)
    else:
        y0, ys, c0, cs = 16 * m, Fraction(1, 219 * m), 128 * m, Fraction(1, 224 * m)
    kg = 1 - kr - kb
    cr, cb, gb, gr = 2 * (1 - kr), 2 * (1 - kb), 2 * kb * (1 - kb) / kg, 2 * kr * (1 - kr) / kg
    # channel = 255 * (ys * (Y - y0) + a * (U - c0) + b * (V - c0))
    rows = [(0, cr), (-gb, -gr), (cb, 0)]
    Y, U, V = (codes[:, i].astype(object) - off for i, off in ((0, y0), (1, c0), (2, c0)))
    out = np.empty((len(codes), 3), np.int64)
    near = np.zeros((len(codes), 3), bool)
    for c, (a, b) in enumerate(rows):
        ky, ku, kv = 255 * ys, 255 * cs * a, 255 * cs * b
        den = np.lcm.reduce([ky.denominator, Fraction(ku).denominator, Fraction(kv).denominator])
        den = int(den)
        num = Y * int(ky * den) + U * int(ku * den) + V * int(kv * den)
        q = num // den  # floor; 0 <= r < den
        r = num - q * den
        twice = 2 * r
        up = (twice > den) | ((twice == den) & (q % 2 == 1))
        out[:, c] = np.clip((q + up.astype(object)).astype(np.int64), 0, 255)
        near[:, c] = np.abs(twice - den).astype(object) * 10 ** 9 < 2 * den  # |frac - 1/2| < 1e-9
    return out, near


def oracle_on_codes(codes, matrix, full_range, bits, shift=0, noise=None):
    """image_ops.yuv420_to_rgb of code triples, each laid out as one 2 x 2 block (its chroma shared by four luma
    samples): samples are codes << shift, plus ``noise`` in the bits the reader must mask."""
    s = codes.astype(np.int64) << shift
    if noise is not None:
        s = s | noise
    dtype = np.uint8 if bits == 8 else np.uint16
    y = np.repeat(np.repeat(s[None, :, 0], 2, 1), 2, 0).astype(dtype)
    u, v = s[None, :, 1].astype(dtype), s[None, :, 2].astype(dtype)
    return image_ops.yuv420_to_rgb(y, u, v, matrix, full_range, bits, shift)[0, 0::2].astype(np.int64)


@pytest.mark.parametrize("fmt", NON_DEFAULT, ids=lambda f: f"{f}")
def test_oracle_equals_exact_rational_conversion(fmt):
    matrix, full, bits = fmt
    codes = format_codes(bits)
    want, near = exact_rgb(codes, matrix, full, bits)
    got = oracle_on_codes(codes, matrix, full, bits)
    ok = (got == want) | near
    assert ok.all(), (codes[~ok.all(1)][:5], got[~ok.all(1)][:5], want[~ok.all(1)][:5])
    print(f"{fmt}: {int(near.sum())} of {near.size} channel values within 1e-9 of a half-integer")
    if bits > 8:  # the same codes MSB-aligned with noise in the low bits, LSB-aligned with noise in the high bits
        rng = np.random.default_rng(bits)
        low = rng.integers(0, 1 << (16 - bits), codes.shape)
        assert np.array_equal(oracle_on_codes(codes, matrix, full, bits, 16 - bits, low), got)
        assert np.array_equal(oracle_on_codes(codes, matrix, full, bits, 0, low << bits), got)
