"""CPU: the numpy restatement of single-channel frames the GPU tests compare against -- image_ops.mono_to_rgb without
gain control (against cv2.cvtColor(GRAY2RGB) and bayer_to_rgb's per-channel mapping) and with min-max gain control
(against cv2.normalize(NORM_MINMAX, CV_8U), bit for bit, at every depth) -- plus packed round trips, the FearFrameMono
record, the new C ABI symbols and MonoFrame's refusals that need no device."""
import os

import cv2
import numpy as np
import pytest
import torch

import feartracker_b200 as fb
from feartracker_b200 import _lib, image_ops
from feartracker_b200 import multi_tracker as mt
from tests.test_yuv_frames_cpu import RGB, _tracker

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ("fear_frame_range_mono", "fear_crop_targets_mono_u8", "fear_advance_targets_mono",
               "fear_frame_sums_mono_u8")
DEPTHS = [8, 10, 12, 14, 16]


def _dtype(bits):
    return np.uint8 if bits == 8 else np.uint16


def test_mono_to_rgb_at_8_bits_is_gray2rgb():
    rng = np.random.default_rng(1)
    for h, w in ((1, 1), (1, 7), (5, 1), (31, 64)):
        g = rng.integers(0, 256, (h, w)).astype(np.uint8)
        assert np.array_equal(image_ops.mono_to_rgb(g), cv2.cvtColor(g, cv2.COLOR_GRAY2RGB))


@pytest.mark.parametrize("bits", [10, 12, 14, 16])
def test_mono_to_rgb_above_8_bits_maps_like_bayer_to_rgb(bits):
    """Every code of the depth, mapped as bayer_to_rgb maps each channel of a flat mosaic."""
    every = np.arange(1 << bits, dtype=np.uint16)
    rows = np.tile(every, (3, 1))
    want = image_ops.bayer_to_rgb(rows, "RGGB", bits)[1]  # a flat row demosaics to itself
    got = image_ops.mono_to_rgb(rows, bits)
    assert np.array_equal(got[1], want)
    assert np.array_equal(got[..., 0], got[..., 1]) and np.array_equal(got[..., 0], got[..., 2])


def _ranges(bits, rng, count):
    top = (1 << bits) - 1
    fixed = [(0, top), (0, 0), (top, top), (5, 5), (0, 1), (top - 1, top), (7, 8), (0, min(top, 300)),
             (top // 2, top // 2 + 1)]
    drawn = []
    for _ in range(count):
        lo = int(rng.integers(0, top + 1))
        drawn.append((lo, int(rng.integers(lo, top + 1))))
    return fixed + drawn


@pytest.mark.parametrize("bits", DEPTHS)
def test_minmax_agc_equals_cv2_normalize(bits):
    """Frames that hold every code of sampled (lo, hi) ranges (and random codes of the range after them), including
    hi == lo, hi - lo == 1, full scale and lo == 0: mono_to_rgb(agc="minmax") equals cv2.normalize(codes, None, 0, 255,
    NORM_MINMAX, CV_8U) on every value."""
    rng = np.random.default_rng(bits)
    dt = _dtype(bits)
    for lo, hi in _ranges(bits, rng, 60 if bits > 8 else 200):
        span = np.arange(lo, hi + 1, dtype=np.int64)
        n = max(span.size, 64)
        codes = np.concatenate([span, rng.integers(lo, hi + 1, n - span.size + 37)]).astype(dt)
        cols = 97
        codes = np.concatenate([codes, np.full(-codes.size % cols, lo, dt)]).reshape(-1, cols)
        want = cv2.normalize(codes, None, 0, 255, cv2.NORM_MINMAX, dtype=cv2.CV_8U)
        got = image_ops.mono_to_rgb(codes, bits, agc="minmax")
        assert np.array_equal(got[..., 0], want), (bits, lo, hi)
        assert np.array_equal(got, cv2.cvtColor(want, cv2.COLOR_GRAY2RGB))
        if lo == hi:
            assert not got.any()


def test_minmax_gain_is_opencv_arithmetic():
    """The float32 gain and offset are rounded from OpenCV's float64 scale = 255 * (1 / (hi - lo)) and
    shift = 0 - lo * scale, and the map rounds fmaf(v, a, b) once: on a range where the two roundings of v * a + b differ
    from one, the single rounding is what cv2 gives."""
    a, b = image_ops.minmax_gain(3, 1003)
    scale = 255.0 * (1.0 / 1000.0)
    assert a == np.float32(scale) and b == np.float32(0.0 - 3 * scale)
    assert image_ops.minmax_gain(9, 9) == (np.float32(0.0), np.float32(0.0))
    # fma_f32 against exact rational arithmetic on random float32 operands near integer + 1/2
    from fractions import Fraction
    rng = np.random.default_rng(4)
    for _ in range(2000):
        v = int(rng.integers(0, 1 << 16))
        a = np.float32(rng.uniform(0, 1))
        b = np.float32(-rng.uniform(0, 255))
        exact = Fraction(v) * Fraction(float(a)) + Fraction(float(b))
        got = image_ops.fma_f32(np.array([v]), a, b)[0]
        lo = np.float32(float(exact))
        cands = [lo, np.nextafter(lo, np.float32(np.inf)), np.nextafter(lo, np.float32(-np.inf))]
        best = min(cands, key=lambda c: (abs(Fraction(float(c)) - exact), int(np.float32(c).view(np.int32)) & 1))
        assert got == best, (v, a, b)


@pytest.mark.parametrize("bits", [10, 12])
def test_packed_round_trip_to_rgb(bits):
    rng = np.random.default_rng(bits + 100)
    for w in (1, 2, 3, 5, 1917, 1920):
        codes = rng.integers(0, 1 << bits, (4, w)).astype(np.uint16)
        rows = image_ops.mipi_pack(codes, bits, image_ops.mipi_row_bytes(w, bits) + 3)
        back = image_ops.mipi_unpack(rows, w, bits)
        assert np.array_equal(back, codes)
        for agc in (None, "minmax"):
            assert np.array_equal(image_ops.mono_to_rgb(back, bits, agc), image_ops.mono_to_rgb(codes, bits, agc))


def test_mono_to_rgb_refusals():
    g = np.zeros((4, 4), np.uint8)
    for args, kw in (((g, 9), {}), ((g, 10), {}), ((g.astype(np.uint16), 8), {}), ((np.full((2, 2), 1024, np.uint16), 10),
                     {}), ((g,), {"agc": "histogram"}), ((g,), {"agc": 1}), ((g[None],), {})):
        with pytest.raises(ValueError):
            image_ops.mono_to_rgb(*args, **kw)


def test_mono_record_is_48_bytes_and_matches_the_header():
    d = _lib.MONO_DTYPE
    assert d.itemsize == 48
    assert d.names == ("data", "row_stride", "H", "W", "bits", "shift", "packing", "agc", "lo", "hi")
    assert [d.fields[n][1] for n in d.names] == [0, 8, 16, 20, 24, 28, 32, 36, 40, 44]
    with open(os.path.join(ROOT, "include", "fear_b200.h")) as f:
        header = f.read()
    body = header[header.index("typedef struct FearFrameMono {"):header.index("} FearFrameMono;")]
    for field in ("const void* data;", "int64_t row_stride;", "int32_t H, W;", "int32_t bits, shift, packing;",
                  "int32_t agc;", "int32_t lo, hi;"):
        assert field in body
    assert "#define FEAR_AGC_MINMAX 1" in header and image_ops.AGC_MODES == {None: 0, "minmax": 1}


def test_new_symbols_are_declared_and_bound():
    with open(os.path.join(ROOT, "include", "fear_b200.h")) as f:
        header = f.read()
    for name in NEW_SYMBOLS:
        assert f"int {name}(" in header
        assert name in _lib.exported_symbols()
        assert getattr(_lib.load(), name).argtypes
    assert mt.ENTRY_POINTS["mono"] == ("fear_frame_sums_mono_u8", "fear_crop_targets_mono_u8",
                                        "fear_advance_targets_mono")
    assert mt.TABLE_DTYPES["mono"] is _lib.MONO_DTYPE
    assert mt.RANGE_ENTRY_POINT == "fear_frame_range_mono"


def _u8(*shape):
    return torch.zeros(*shape, dtype=torch.uint8)


BAD_FRAMES = {
    "host tensor": lambda: fb.MonoFrame(_u8(8, 8)),
    "numpy frame": lambda: fb.MonoFrame(np.zeros((8, 8), np.uint8)),
    "host uint16": lambda: fb.MonoFrame(torch.zeros(8, 8, dtype=torch.uint16), bits=12),
    "3-D frame": lambda: fb.MonoFrame(_u8(8, 8, 1)),
    "bits 9": lambda: fb.MonoFrame(_u8(8, 8), bits=9),
    "bits True": lambda: fb.MonoFrame(_u8(8, 8), bits=True),
    "msb at 8 bits": lambda: fb.MonoFrame(_u8(8, 8), msb=True),
    "unknown agc": lambda: fb.MonoFrame(_u8(8, 8), agc="clahe"),
    "agc True": lambda: fb.MonoFrame(_u8(8, 8), agc=True),
    "host raw10": lambda: fb.MonoFrame.raw10(_u8(8, 10), 8),
    "raw12 bad agc": lambda: fb.MonoFrame.raw12(_u8(8, 12), 8, agc="plateau"),
}


@pytest.mark.parametrize("what", list(BAD_FRAMES))
def test_bad_frames_are_refused_before_device_calls(what):
    """A MonoFrame must be a CUDA tensor of the depth's sample type with a known gain control: anything else is refused
    by the constructor, so add and update raise ValueError before any device call (there is no device here)."""
    make = BAD_FRAMES[what]
    trk = _tracker()
    with pytest.raises(ValueError):
        trk.add(make(), [[1, 1, 2, 2]])
    trk._ids, trk._streams = np.array([0]), np.array([0])
    with pytest.raises(ValueError):
        trk.update(make())


def _fake_mono():
    """A MonoFrame as the constructor leaves it, over a host tensor (the constructor itself needs a CUDA one)."""
    f = fb.MonoFrame.__new__(fb.MonoFrame)
    f.t, f.bits, f.shift, f.packing, f.agc, f.pitch, f.shape = _u8(8, 8), 8, 0, 0, "minmax", 8, (8, 8, 3)
    return f


def _fake_bayer():
    f = fb.BayerFrame.__new__(fb.BayerFrame)
    f.t, f.bits, f.shift, f.packing, f.pattern, f.pitch, f.shape = _u8(8, 8), 8, 0, 0, "RGGB", 8, (8, 8, 3)
    return f


def test_mixing_mono_with_other_kinds_is_refused_before_device_calls():
    trk = _tracker()
    for other in (RGB, torch.zeros(8, 8, 3, dtype=torch.uint8)):
        for frames in ([_fake_mono(), other], [other, _fake_mono()]):
            with pytest.raises(ValueError, match="MonoFrames cannot share"):
                trk.add(frames, [[1, 1, 2, 2]])
    # a call with a BayerFrame keeps the Bayer message, whatever else it holds
    with pytest.raises(ValueError, match="BayerFrames cannot share"):
        trk.add([_fake_mono(), _fake_bayer()], [[1, 1, 2, 2]])
    with pytest.raises(ValueError, match="BayerFrames cannot share"):
        trk.add([_fake_bayer(), RGB, _fake_mono()], [[1, 1, 2, 2]])


def test_frame_kind_and_records():
    f = _fake_mono()
    assert mt.frame_kind(f) == "mono" and mt.frame_kind(_fake_bayer()) == "bayer"
    assert mt.uses_agc([f], "mono") and not mt.uses_agc([f], "bayer")
    rec = f.mono_record()
    assert rec[2:] == (8, 8, 8, 0, 0, 1, 2 ** 31 - 1, -2 ** 31)
    table = np.zeros(1, _lib.MONO_DTYPE)
    mt.write_records(table, [f], "mono")
    assert table[0]["lo"] == 2 ** 31 - 1 and table[0]["hi"] == -2 ** 31 and table[0]["agc"] == 1
