"""CPU: the numpy restatement of RGB frames the GPU tests compare against -- image_ops.rgb_frame_to_rgb at 8 bits
(against cv2.cvtColor, bit for bit) and above 8 bits (against raw_to_u8 and bayer_to_rgb's per-channel mapping, on every
code), the x2rgb10 word pack / unpack pair -- plus the FearFrameRGB record, the new C ABI symbols, and RGBFrame's and the
trackers' refusals that need no device."""
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
NEW_SYMBOLS = ("fear_crop_targets_rgb_u8", "fear_advance_targets_rgb", "fear_frame_sums_rgb_u8")
# the 8-bit layouts cv2.cvtColor names, and its code for each
CV2_CODES = {"bgr24": cv2.COLOR_BGR2RGB, "bgra": cv2.COLOR_BGRA2RGB, "bgr0": cv2.COLOR_BGRA2RGB,
             "rgba": cv2.COLOR_RGBA2RGB, "rgb0": cv2.COLOR_RGBA2RGB}


@pytest.mark.parametrize("layout", [k for k, v in image_ops.RGB_PACKED_LAYOUTS.items() if v[0] == np.uint8])
def test_8_bit_layouts_equal_cv2(layout):
    """Every 8-bit packed layout: cv2.cvtColor where cv2 names the layout, the samples themselves for rgb24, and for
    ARGB / ABGR cv2.cvtColor of the same pixels with the leading sample moved last (cv2's RGBA / BGRA)."""
    rng = np.random.default_rng(len(layout))
    n = image_ops.RGB_PACKED_LAYOUTS[layout][1]
    for h, w in ((1, 1), (1, 7), (5, 1), (31, 64), (17, 333)):
        a = rng.integers(0, 256, (h, w, n)).astype(np.uint8)
        got = image_ops.rgb_frame_to_rgb(a, layout)
        assert got.dtype == np.uint8 and got.shape == (h, w, 3)
        if layout in CV2_CODES:
            want = cv2.cvtColor(a, CV2_CODES[layout])
        elif layout == "rgb24":
            want = a
        else:  # argb / 0rgb are rgba, abgr / 0bgr are bgra, with the alpha / X sample first
            code = cv2.COLOR_RGBA2RGB if layout in ("argb", "0rgb") else cv2.COLOR_BGRA2RGB
            want = cv2.cvtColor(np.ascontiguousarray(np.roll(a, -1, axis=-1)), code)
        assert np.array_equal(got, want), (layout, h, w)


def test_alpha_and_x_samples_are_not_read():
    rng = np.random.default_rng(2)
    for layout, (dtype, n, idx) in image_ops.RGB_PACKED_LAYOUTS.items():
        if n != 4:
            continue
        top = 255 if dtype == np.uint8 else 65535
        a = rng.integers(0, top + 1, (9, 13, 4)).astype(dtype)
        b = a.copy()
        spare = ({0, 1, 2, 3} - set(idx)).pop()
        b[..., spare] = rng.integers(0, top + 1, (9, 13))
        assert np.array_equal(image_ops.rgb_frame_to_rgb(a, layout), image_ops.rgb_frame_to_rgb(b, layout)), layout


@pytest.mark.parametrize("bits", [10, 12, 16])
def test_planar_above_8_bits_maps_every_code_like_raw_to_u8_and_bayer_to_rgb(bits):
    """Every code of the depth in each plane, with random bits above the code (not read): raw_to_u8 of the code, and
    the value bayer_to_rgb gives a flat mosaic of that code."""
    rng = np.random.default_rng(bits)
    every = np.arange(1 << bits, dtype=np.uint16)
    codes = np.stack([every, every[::-1], np.roll(every, 17)])[:, None, :]  # R, G, B planes of (1, 2^bits)
    noise = (rng.integers(0, 1 << (16 - bits), codes.shape) << bits).astype(np.uint16) if bits < 16 else 0
    got = image_ops.rgb_frame_to_rgb(codes | noise, "planar", bits)
    for c in range(3):
        assert np.array_equal(got[0, :, c], image_ops.raw_to_u8(codes[c, 0], bits))
    flat = image_ops.bayer_to_rgb(np.tile(every, (3, 1)), "RGGB", bits)[1, :, 1]
    assert np.array_equal(got[0, :, 0], flat)


def test_16_bit_packed_layouts_map_every_code():
    every = np.arange(1 << 16, dtype=np.uint16).reshape(256, 256)
    want = image_ops.raw_to_u8(every, 16)
    for layout in ("rgb48le", "bgr48le", "rgba64le", "bgra64le"):
        _, n, idx = image_ops.RGB_PACKED_LAYOUTS[layout]
        a = np.zeros((256, 256, n), np.uint16)
        a[..., idx[0]], a[..., idx[1]], a[..., idx[2]] = every, every.T, every[::-1]
        got = image_ops.rgb_frame_to_rgb(a, layout)
        assert np.array_equal(got[..., 0], want) and np.array_equal(got[..., 1], want.T)
        assert np.array_equal(got[..., 2], want[::-1]), layout


def test_8_bit_planar_is_the_planes_stacked():
    rng = np.random.default_rng(3)
    r, g, b = (rng.integers(0, 256, (7, 9)).astype(np.uint8) for _ in range(3))
    assert np.array_equal(image_ops.rgb_frame_to_rgb((r, g, b), "planar", 8), np.stack([r, g, b], -1))


@pytest.mark.parametrize("layout", list(image_ops.X2RGB10_LAYOUTS))
def test_x2rgb10_round_trip_ignores_spare_bits(layout):
    """pack / unpack round trips with random values in the 2 spare bits; every 10-bit code maps as raw_to_u8 does; and
    the field positions are those of DRM XRGB2101010 / DXGI R10G10B10A2 (x2rgb10le: B in the low bits)."""
    rng = np.random.default_rng(7)
    codes = rng.integers(0, 1024, (33, 65, 3)).astype(np.uint16)
    spare = rng.integers(0, 4, (33, 65))
    words = image_ops.x2rgb10_pack(codes, layout, spare)
    assert words.dtype == np.uint32 and np.array_equal(words >> 30, spare)
    assert np.array_equal(image_ops.x2rgb10_unpack(words, layout), codes)
    assert np.array_equal(image_ops.x2rgb10_unpack(words.view(np.int32), layout), codes)
    assert np.array_equal(image_ops.rgb_frame_to_rgb(words, layout), image_ops.raw_to_u8(codes, 10))
    assert np.array_equal(image_ops.rgb_frame_to_rgb(words.view(np.int32), layout), image_ops.raw_to_u8(codes, 10))
    one = image_ops.x2rgb10_pack(np.array([[[1, 2, 3]]]), layout)[0, 0]
    assert one == ((1 << 20) | (2 << 10) | 3 if layout == "x2rgb10le" else 1 | (2 << 10) | (3 << 20))
    every = np.arange(1024, dtype=np.uint16)
    w = image_ops.x2rgb10_pack(np.stack([every, every, every], -1)[None], layout, np.full((1, 1024), 3))
    assert np.array_equal(image_ops.rgb_frame_to_rgb(w, layout)[0, :, 1], image_ops.raw_to_u8(every, 10))


def test_rgb_frame_to_rgb_refusals():
    for args in ((np.zeros((4, 4, 3), np.uint16), "rgb24"), (np.zeros((4, 4, 3), np.uint8), "bgra"),
                 (np.zeros((4, 4, 4), np.uint8), "rgb48le"), (np.zeros((4, 4), np.uint16), "x2rgb10le"),
                 (np.zeros((4, 4, 3), np.uint8), "yuyv"), (np.zeros((3, 4, 4), np.uint8), "planar", 10),
                 (np.zeros((3, 4, 4), np.uint16), "planar", 8), (np.zeros((3, 4, 4), np.uint16), "planar", 14),
                 (np.zeros((2, 4, 4), np.uint8), "planar", 8)):
        with pytest.raises(ValueError):
            image_ops.rgb_frame_to_rgb(*args)
    with pytest.raises(ValueError):
        image_ops.x2rgb10_pack(np.full((1, 1, 3), 1024), "x2rgb10le")


def test_rgb_record_is_72_bytes_and_matches_the_header():
    d = _lib.RGB_DTYPE
    assert d.itemsize == 72
    assert d.names == ("r", "g", "b", "row_stride", "pixel_stride", "H", "W", "container", "bits", "shift_r",
                       "shift_g", "shift_b", "reserved")
    assert [d.fields[n][1] for n in d.names] == [0, 8, 16, 24, 32, 40, 44, 48, 52, 56, 60, 64, 68]
    with open(os.path.join(ROOT, "include", "fear_b200.h")) as f:
        header = f.read()
    body = header[header.index("typedef struct FearFrameRGB {"):header.index("} FearFrameRGB;")]
    for field in ("const uint8_t *r, *g, *b;", "int64_t row_stride, pixel_stride;", "int32_t H, W;",
                  "int32_t container;", "int32_t bits;", "int32_t shift_r, shift_g, shift_b;", "int32_t reserved;"):
        assert field in body
    from feartracker_b200 import tracker
    assert d.itemsize <= tracker._TARGET_OFFSET  # FEARTracker stages the record before its FearTarget


def test_new_symbols_are_declared_and_bound():
    with open(os.path.join(ROOT, "include", "fear_b200.h")) as f:
        header = f.read()
    for name in NEW_SYMBOLS:
        assert f"int {name}(" in header
        assert name in _lib.exported_symbols() and name in _lib._SIGNATURES
        assert getattr(_lib.load(), name).argtypes
    assert mt.ENTRY_POINTS["rgb"] == ("fear_frame_sums_rgb_u8", "fear_crop_targets_rgb_u8", "fear_advance_targets_rgb")
    assert mt.TABLE_DTYPES["rgb"] is _lib.RGB_DTYPE


def _u8(*shape):
    return torch.zeros(*shape, dtype=torch.uint8)


BAD_FRAMES = {
    "host tensor": lambda: fb.RGBFrame(_u8(8, 8, 3), "bgr24"),
    "numpy frame": lambda: fb.RGBFrame(np.zeros((8, 8, 3), np.uint8), "bgr24"),
    "unknown layout": lambda: fb.RGBFrame(_u8(8, 8, 3), "BGR"),
    "layout None": lambda: fb.RGBFrame(_u8(8, 8, 3), None),
    "host uint16": lambda: fb.RGBFrame(torch.zeros(8, 8, 3, dtype=torch.uint16), "rgb48le"),
    "host words": lambda: fb.RGBFrame(torch.zeros(8, 8, dtype=torch.int32), "x2rgb10le"),
    "host planes": lambda: fb.RGBFrame.planar(_u8(8, 8), _u8(8, 8), _u8(8, 8)),
    "planar bits 14": lambda: fb.RGBFrame.planar(_u8(8, 8), _u8(8, 8), _u8(8, 8), bits=14),
    "planar bits True": lambda: fb.RGBFrame.planar(_u8(8, 8), _u8(8, 8), _u8(8, 8), bits=True),
}


@pytest.mark.parametrize("what", list(BAD_FRAMES))
def test_bad_frames_are_refused_before_device_calls(what):
    """An RGBFrame must be a CUDA tensor of its layout's sample type: anything else is refused by the constructor, so
    add and update raise ValueError before any device call (there is no device here)."""
    make = BAD_FRAMES[what]
    trk = _tracker()
    with pytest.raises(ValueError):
        trk.add(make(), [[1, 1, 2, 2]])
    trk._ids, trk._streams = np.array([0]), np.array([0])
    with pytest.raises(ValueError):
        trk.update(make())


def _fake_rgb():
    """An RGBFrame as the constructor leaves it, over a host tensor (the constructor itself needs a CUDA one)."""
    f = fb.RGBFrame.__new__(fb.RGBFrame)
    t = _u8(8, 8, 4)
    f._record = (t.data_ptr() + 2, t.data_ptr() + 1, t.data_ptr(), 32, 4, 8, 8, 1, 8, 0, 0, 0, 0)
    f.tensors, f.layout, f.bits, f.shape = (t,), "bgra", 8, (8, 8, 3)
    return f


def _fake_mono():
    f = fb.MonoFrame.__new__(fb.MonoFrame)
    f.t, f.bits, f.shift, f.packing, f.agc, f.pitch, f.shape = _u8(8, 8), 8, 0, 0, None, 8, (8, 8, 3)
    return f


def _fake_bayer():
    f = fb.BayerFrame.__new__(fb.BayerFrame)
    f.t, f.bits, f.shift, f.packing, f.pattern, f.pitch, f.shape = _u8(8, 8), 8, 0, 0, "RGGB", 8, (8, 8, 3)
    return f


def test_mixing_rgb_frames_with_other_kinds_is_refused_before_device_calls():
    trk = _tracker()
    nv12 = fb.YUV420Frame.nv12(torch.zeros((12, 8), dtype=torch.uint8))
    for other in (RGB, nv12):
        for frames in ([_fake_rgb(), other], [other, _fake_rgb()], [_fake_rgb(), _u8(8, 8, 3), other]):
            with pytest.raises(ValueError, match="RGBFrames can share a call only with CUDA"):
                trk.add(frames, [[1, 1, 2, 2]])
            with pytest.raises(ValueError, match="RGBFrames can share a call only with CUDA"):
                trk.update(frames)
    # a call with a BayerFrame or a MonoFrame keeps its message
    with pytest.raises(ValueError, match="BayerFrames cannot share"):
        trk.add([_fake_rgb(), _fake_bayer()], [[1, 1, 2, 2]])
    with pytest.raises(ValueError, match="MonoFrames cannot share"):
        trk.add([_fake_mono(), _fake_rgb()], [[1, 1, 2, 2]])
    # RGBFrames with tensors pass the mixing check and reach the device checks (a host tensor is refused there)
    with pytest.raises(ValueError, match="cpu tensor"):
        trk.add([_fake_rgb(), _u8(8, 8, 3)], [[1, 1, 2, 2]])
    assert len(trk) == 0


def test_frame_kind_and_records():
    f = _fake_rgb()
    assert mt.frame_kind(f) == "rgb" and mt.frame_kind(_u8(8, 8, 3)) == "cuda"
    t = _u8(6, 10, 4)[:, 1:9, :3]  # a strided RGB view: channel c at data + c
    table = np.zeros(2, _lib.RGB_DTYPE)
    mt.write_records(table, [f, t], "rgb")
    assert tuple(table[0]) == f.rgb_record()
    p = t.data_ptr()
    assert tuple(table[1]) == (p, p + 1, p + 2, 40, 4, 6, 8, 1, 8, 0, 0, 0, 0)
    assert mt.tensor_rgb_record(t) == tuple(table[1])
