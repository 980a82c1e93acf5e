"""CPU: the numpy restatements of the Bayer reads the GPU tests compare against -- image_ops.bayer_demosaic (against
cv2.cvtColor), bayer_to_rgb (against yuv_to_rgb at neutral chroma), mipi_unpack (against hand-packed RAW10 / RAW12
groups) and its inverse mipi_pack -- plus the FearFrameBayer record, the new C ABI symbols and BayerFrame's refusals that
need no device."""
import os

import cv2
import numpy as np
import pytest
import torch

import feartracker_b200 as fb
from feartracker_b200 import _lib, image_ops
from tests.test_yuv_frames_cpu import RGB, _tracker

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ("fear_crop_targets_bayer_u8", "fear_advance_targets_bayer", "fear_frame_sums_bayer_u8")
CV2_CODES = {"RGGB": cv2.COLOR_BayerRGGB2RGB, "GRBG": cv2.COLOR_BayerGRBG2RGB, "GBRG": cv2.COLOR_BayerGBRG2RGB,
             "BGGR": cv2.COLOR_BayerBGGR2RGB}
SIZES = [(3, 3), (3, 4), (4, 3), (4, 5), (5, 5), (9, 13), (10, 12), (31, 64), (64, 31)]


@pytest.mark.parametrize("dtype", [np.uint8, np.uint16], ids=["u8", "u16"])
@pytest.mark.parametrize("pattern", list(CV2_CODES))
def test_demosaic_equals_cv2(pattern, dtype):
    """Every size from 3 x 3 up, odd and even, on random codes over the whole range and on all-0, all-max and
    0 / max checkerboards and stripes."""
    rng = np.random.default_rng(list(CV2_CODES).index(pattern) + 10 * (dtype == np.uint16))
    top = np.iinfo(dtype).max
    for h, w in SIZES:
        yy, xx = np.indices((h, w))
        cases = [rng.integers(0, top + 1, (h, w)), np.zeros((h, w)), np.full((h, w), top), ((yy + xx) % 2) * top,
                 (yy % 2) * top, (xx % 3 == 0) * top, rng.choice([0, 1, top - 1, top], (h, w))]
        for raw in cases:
            raw = raw.astype(dtype)
            assert np.array_equal(image_ops.bayer_demosaic(raw, pattern), cv2.cvtColor(raw, CV2_CODES[pattern])), \
                (pattern, dtype, h, w)


@pytest.mark.parametrize("bits", [10, 12])
def test_bayer_to_rgb_maps_like_full_range_luma(bits):
    """Above 8 bits each demosaiced channel maps to 8 bits as yuv_to_rgb maps full-range luma at neutral chroma."""
    rng = np.random.default_rng(bits)
    top = (1 << bits) - 1
    codes = rng.integers(0, top + 1, (17, 22)).astype(np.uint16)
    codes[0, :4] = [0, 1, top - 1, top]
    neutral = np.full(codes.shape, 1 << (bits - 1), np.uint16)
    for p in CV2_CODES:
        d = image_ops.bayer_demosaic(codes, p)
        want = np.stack([image_ops.yuv_to_rgb(d[..., c], neutral, neutral, full_range=True, bits=bits,
                                              chroma_shift=(0, 0))[..., 0] for c in range(3)], -1)
        assert np.array_equal(image_ops.bayer_to_rgb(codes, p, bits), want), (p, bits)
    every = np.arange(top + 1, dtype=np.uint16)
    neutral = np.full(every.shape, 1 << (bits - 1), np.uint16)
    assert np.array_equal(image_ops.bayer_to_rgb(np.tile(every, (3, 1)), "RGGB", bits)[1, :, 1],
                          image_ops.yuv_to_rgb(every[None], neutral[None], neutral[None], full_range=True, bits=bits,
                                               chroma_shift=(0, 0))[0, :, 1])


def test_bayer_to_rgb_at_8_bits_is_the_demosaic_and_refuses_bad_codes():
    raw = np.random.default_rng(3).integers(0, 256, (7, 9)).astype(np.uint8)
    assert np.array_equal(image_ops.bayer_to_rgb(raw, "GBRG", 8), cv2.cvtColor(raw, cv2.COLOR_BayerGBRG2RGB))
    for args in ((raw, "RGGB", 9), (raw, "RGGB", 10), (raw.astype(np.uint16), "RGGB", 8),
                 (np.full((4, 4), 1024, np.uint16), "RGGB", 10), (raw, "BayerRG", 8), (raw[:2], "RGGB", 8)):
        with pytest.raises(ValueError):
            image_ops.bayer_to_rgb(*args)


def hand_raw10(codes) -> bytes:
    """One RAW10 row spelled out from the CSI-2 table: per 4 pixels, P0[9:2] P1[9:2] P2[9:2] P3[9:2], then
    P3[1:0] << 6 | P2[1:0] << 4 | P1[1:0] << 2 | P0[1:0]; pixels past the row are 0."""
    c = [int(x) for x in codes] + [0] * (-len(codes) % 4)
    out = b""
    for g in range(0, len(c), 4):
        p = c[g:g + 4]
        out += bytes([x >> 2 for x in p] + [(p[3] & 3) << 6 | (p[2] & 3) << 4 | (p[1] & 3) << 2 | (p[0] & 3)])
    return out


def hand_raw12(codes) -> bytes:
    """One RAW12 row: per 2 pixels, P0[11:4] P1[11:4], then P1[3:0] << 4 | P0[3:0]."""
    c = [int(x) for x in codes] + [0] * (-len(codes) % 2)
    out = b""
    for g in range(0, len(c), 2):
        out += bytes([c[g] >> 4, c[g + 1] >> 4, (c[g + 1] & 15) << 4 | (c[g] & 15)])
    return out


@pytest.mark.parametrize("bits", [10, 12])
@pytest.mark.parametrize("width", [3, 4, 5, 6, 7, 8, 9, 1917, 1918, 1919, 1920])
def test_mipi_unpack_reads_hand_packed_groups(bits, width):
    """W % 4 in {0, 1, 2, 3} (RAW10) and W % 2 in {0, 1} (RAW12): whole groups and partial last groups, at a pitch
    with 0xA5 past the groups."""
    rng = np.random.default_rng(width + bits)
    codes = rng.integers(0, 1 << bits, (3, width))
    codes[0, :3] = [0, (1 << bits) - 1, 0b1010101010 if bits == 10 else 0xA5A]
    hand = hand_raw10 if bits == 10 else hand_raw12
    need = image_ops.mipi_row_bytes(width, bits)
    rows = np.full((3, need + 13), 0xA5, np.uint8)
    for r in range(3):
        rows[r, :need] = np.frombuffer(hand(codes[r]), np.uint8)
    assert np.array_equal(image_ops.mipi_unpack(rows, width, bits), codes)
    packed = image_ops.mipi_pack(codes, bits, need + 13)
    assert np.array_equal(packed[:, :need], rows[:, :need]) and (packed[:, need:] == 0).all()
    assert np.array_equal(image_ops.mipi_unpack(packed, width, bits), codes)


def test_mipi_row_bytes_and_refusals():
    assert [image_ops.mipi_row_bytes(w, 10) for w in (1, 4, 5, 1920)] == [5, 5, 10, 2400]
    assert [image_ops.mipi_row_bytes(w, 12) for w in (1, 2, 3, 1920)] == [3, 3, 6, 2880]
    codes = np.zeros((2, 8), np.uint16)
    for call in (lambda: image_ops.mipi_row_bytes(8, 8), lambda: image_ops.mipi_pack(codes, 14),
                 lambda: image_ops.mipi_pack(codes + 1024, 10), lambda: image_ops.mipi_pack(codes, 10, pitch=9),
                 lambda: image_ops.mipi_unpack(np.zeros((2, 9), np.uint8), 8, 10),
                 lambda: image_ops.mipi_unpack(np.zeros((2, 10), np.uint16), 8, 10),
                 lambda: image_ops.mipi_unpack(np.zeros((2, 10), np.uint8), 0, 10)):
        with pytest.raises(ValueError):
            call()


def test_bayer_record_is_40_bytes():
    d = _lib.BAYER_DTYPE
    assert d.itemsize == 40
    assert d.names == ("data", "row_stride", "H", "W", "pattern", "bits", "shift", "packing")
    assert [d.fields[n][1] for n in d.names] == [0, 8, 16, 20, 24, 28, 32, 36]
    assert image_ops.BAYER_PATTERNS == {"RGGB": 0, "GRBG": 1, "GBRG": 2, "BGGR": 3}


def test_new_symbols_are_declared_and_bound():
    with open(os.path.join(ROOT, "include", "fear_b200.h")) as f:
        header = f.read()
    assert "typedef struct FearFrameBayer" in header
    for name in NEW_SYMBOLS:
        assert f"int {name}(" in header
        assert name in _lib.exported_symbols()
        assert getattr(_lib.load(), name).argtypes  # bound with a signature
    from feartracker_b200 import multi_tracker as mt

    assert mt.ENTRY_POINTS["bayer"] == ("fear_frame_sums_bayer_u8", "fear_crop_targets_bayer_u8",
                                         "fear_advance_targets_bayer")
    assert mt.TABLE_DTYPES["bayer"] is _lib.BAYER_DTYPE


def _u8(*shape):
    return torch.zeros(*shape, dtype=torch.uint8)


BAD_FRAMES = {
    "host tensor": lambda: fb.BayerFrame(_u8(8, 8)),
    "numpy mosaic": lambda: fb.BayerFrame(np.zeros((8, 8), np.uint8)),
    "host uint16": lambda: fb.BayerFrame(torch.zeros(8, 8, dtype=torch.uint16), bits=12),
    "3-D mosaic": lambda: fb.BayerFrame(_u8(8, 8, 1)),
    "unknown pattern": lambda: fb.BayerFrame(_u8(8, 8), "RGBG"),
    "old cv2 name": lambda: fb.BayerFrame(_u8(8, 8), "BayerRG"),
    "bits 9": lambda: fb.BayerFrame(_u8(8, 8), bits=9),
    "bits True": lambda: fb.BayerFrame(_u8(8, 8), bits=True),
    "msb at 8 bits": lambda: fb.BayerFrame(_u8(8, 8), msb=True),
    "host raw10": lambda: fb.BayerFrame.raw10(_u8(8, 10), 8),
    "raw12 bad pattern": lambda: fb.BayerFrame.raw12(_u8(8, 12), 8, "GGRB"),
    "host bayer then RGB": lambda: [fb.BayerFrame(_u8(8, 8)), RGB],
}


@pytest.mark.parametrize("what", list(BAD_FRAMES))
def test_bad_frames_are_refused_before_device_calls(what):
    """A BayerFrame must be a CUDA tensor of the depth's sample type with a known pattern: a host tensor or array, another
    rank, an unknown pattern or a bad depth is refused by the constructor, so add and update raise ValueError before any
    device call (there is no device here).  The refusals that need a CUDA tensor (size, row, pitch, alignment) are in
    tests/test_gpu_bayer.py."""
    make = BAD_FRAMES[what]
    trk = _tracker()
    with pytest.raises(ValueError):
        trk.add(make(), [[1, 1, 2, 2]])
    trk._ids, trk._streams = np.array([0]), np.array([0])
    with pytest.raises(ValueError):
        trk.update(make())


def test_frame_kind_of_existing_frames_is_unchanged():
    from feartracker_b200 import multi_tracker as mt

    assert mt.frame_kind(RGB) == "numpy"
    assert mt.frame_kind(torch.zeros(4, 4, 3, dtype=torch.uint8)) == "cuda"
    assert mt.frame_kind(fb.YUV420Frame.nv12(torch.zeros(96, 80, dtype=torch.uint8))) == "yuv"
