"""CPU: image_ops.v210_unpack, the numpy restatement of the v210 reads the GPU tests compare against, its inverse
image_ops.v210_pack, the FearFrameYCbCrV210 record, V210Frame's refusals and the new C ABI symbols.

The unpacker is pinned to groups packed by hand from the format's word layout (ffmpeg's v210 order), including the
partial last group of widths that are not a multiple of 6."""
import os

import numpy as np
import pytest
import torch

import feartracker_b200 as fb
from feartracker_b200 import _lib, image_ops
from tests.test_yuv_frames_cpu import RGB, _tracker

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ("fear_crop_targets_ycbcr_v210_u8", "fear_advance_targets_ycbcr_v210", "fear_frame_sums_ycbcr_v210_u8")


def hand_packed_row(y, u, v) -> bytes:
    """One v210 row spelled out word by word from the format's table: w0 = Cb0 | Y0 << 10 | Cr0 << 20, w1 = Y1 |
    Cb1 << 10 | Y2 << 20, w2 = Cr1 | Y3 << 10 | Cb2 << 20, w3 = Y4 | Cr2 << 10 | Y5 << 20; codes past the row are 0,
    bits 30-31 are set in every word (readers ignore them)."""
    groups = -(-len(y) // 6)
    y = [int(c) for c in y] + [0] * (6 * groups - len(y))
    u = [int(c) for c in u] + [0] * (3 * groups - len(u))
    v = [int(c) for c in v] + [0] * (3 * groups - len(v))
    out = b""
    for g in range(groups):
        Y, U, V = y[6 * g:6 * g + 6], u[3 * g:3 * g + 3], v[3 * g:3 * g + 3]
        words = [U[0] | Y[0] << 10 | V[0] << 20, Y[1] | U[1] << 10 | Y[2] << 20,
                 V[1] | Y[3] << 10 | U[2] << 20, Y[4] | V[2] << 10 | Y[5] << 20]
        out += b"".join(int(w | 3 << 30).to_bytes(4, "little") for w in words)
    return out


@pytest.mark.parametrize("width", [2, 4, 6, 8, 10, 12, 720, 1280, 1918, 1920])
def test_unpack_reads_hand_packed_groups(width):
    """W % 6 in {0, 2, 4}: whole groups, and a last group with 2 or 4 of its 6 pixels (W = 2, 4, 8, 10, 1918)."""
    rng = np.random.default_rng(width)
    h = 3
    y = rng.integers(0, 1024, (h, width))
    u, v = rng.integers(0, 1024, (2, h, width // 2))
    pitch = image_ops.v210_pitch(width) + 32
    rows = np.zeros((h, pitch), np.uint8)
    for r in range(h):
        b = hand_packed_row(y[r], u[r], v[r])
        rows[r, :len(b)] = np.frombuffer(b, np.uint8)
        rows[r, len(b):] = 0xA5  # past the groups: never read
    gy, gu, gv = image_ops.v210_unpack(rows, width)
    assert gy.dtype == gu.dtype == gv.dtype == np.uint16
    assert gy.shape == (h, width) and gu.shape == gv.shape == (h, width // 2)
    assert np.array_equal(gy, y) and np.array_equal(gu, u) and np.array_equal(gv, v)


def test_unpack_of_one_group_names_each_code():
    codes = list(range(1, 13))  # Cb0 Y0 Cr0 Y1 Cb1 Y2 Cr1 Y3 Cb2 Y4 Cr2 Y5 = 1 .. 12
    words = [codes[3 * i] | codes[3 * i + 1] << 10 | codes[3 * i + 2] << 20 for i in range(4)]
    row = np.frombuffer(b"".join(w.to_bytes(4, "little") for w in words), np.uint8)[None]
    y, u, v = image_ops.v210_unpack(row, 6)
    assert y.tolist() == [[2, 4, 6, 8, 10, 12]] and u.tolist() == [[1, 5, 9]] and v.tolist() == [[3, 7, 11]]
    y, u, v = image_ops.v210_unpack(row, 4)
    assert y.tolist() == [[2, 4, 6, 8]] and u.tolist() == [[1, 5]] and v.tolist() == [[3, 7]]


@pytest.mark.parametrize("hw", [(1, 2), (5, 4), (7, 722), (4, 1280), (2, 3840)])
def test_pack_unpack_round_trip_and_pack_matches_hand_packing(hw):
    h, w = hw
    rng = np.random.default_rng(h * w)
    y = rng.integers(0, 1024, (h, w)).astype(np.uint16)
    u, v = rng.integers(0, 1024, (2, h, w // 2)).astype(np.uint16)
    for pitch in (None, image_ops.v210_row_bytes(w), image_ops.v210_pitch(w) + 64):
        rows = image_ops.v210_pack(y, u, v, pitch)
        assert rows.dtype == np.uint8
        assert rows.shape == (h, image_ops.v210_pitch(w) if pitch is None else pitch)
        back = image_ops.v210_unpack(rows, w)
        assert all(np.array_equal(a, b) for a, b in zip(back, (y, u, v)))
        hand = np.frombuffer(hand_packed_row(y[0], u[0], v[0]), np.uint8)
        assert np.array_equal(rows[0, :len(hand)] | 0xC0 * ((np.arange(len(hand)) % 4) == 3), hand)


def test_pitch_helpers_follow_the_capture_card_rule():
    assert [image_ops.v210_row_bytes(w) for w in (2, 6, 8, 720, 1280, 1920, 3840)] == [16, 16, 32, 1920, 3424, 5120,
                                                                                           10240]
    assert [image_ops.v210_pitch(w) for w in (2, 48, 50, 720, 1280, 1920, 3840)] == [128, 128, 256, 1920, 3456, 5120,
                                                                                     10240]


@pytest.mark.parametrize("args", [
    (np.zeros((2, 16), np.uint8), 3), (np.zeros((2, 16), np.uint8), 0), (np.zeros((2, 16), np.uint8), 8),
    (np.zeros((2, 16), np.uint16), 2), (np.zeros((2, 4, 4), np.uint8), 2), (np.zeros((0, 16), np.uint8), 2),
    (np.zeros((2, 16), np.uint8), 2.0), (np.zeros((2, 16), np.uint8), True)], ids=str)
def test_unpack_refuses_bad_input(args):
    with pytest.raises(ValueError):
        image_ops.v210_unpack(*args)


def test_pack_refuses_bad_input():
    y, c = np.zeros((2, 4), np.uint16), np.zeros((2, 2), np.uint16)
    for bad in ((y[:, :3], c, c), (y, c[:1], c), (y, c, c[:, :1]), (y + 1024, c, c), (y, c - 1.0, c)):
        with pytest.raises(ValueError):
            image_ops.v210_pack(*bad)
    with pytest.raises(ValueError):
        image_ops.v210_pack(y, c, c, pitch=15)


def test_v210_record_is_96_bytes_after_the_ycbcr_fields():
    assert _lib.YCBCR_V210_DTYPE.itemsize == 96
    assert _lib.YCBCR_V210_DTYPE.names == _lib.YCBCR_DTYPE.names + ("v210", "reserved")
    assert _lib.YCBCR_V210_DTYPE.fields["v210"][1] == 88


def test_new_symbols_are_declared_and_bound():
    with open(os.path.join(ROOT, "include", "fear_b200.h")) as f:
        header = f.read()
    assert "typedef struct FearFrameYCbCrV210" in header
    for name in NEW_SYMBOLS:
        assert f"int {name}(" in header
        assert name in _lib.exported_symbols()
        assert getattr(_lib.load(), name).argtypes  # bound with a signature
    assert fb.V210Frame.CHROMA_SHIFT == (1, 0) and fb.V210Frame.bits == 10


def test_planar_frames_give_their_ycbcr_record_with_v210_0():
    for f in (fb.YUV420Frame.nv12(torch.zeros(96, 80, dtype=torch.uint8)),
              fb.YUV422Frame.nv16(torch.zeros(96, 80, dtype=torch.uint16), matrix="bt709", bits=10),
              fb.YUV444Frame.i444(torch.zeros(9, 6, dtype=torch.uint8))):
        rec = f.ycbcr_v210_record()
        assert rec == f.ycbcr_record() + (0, 0)
        assert np.array([rec], dtype=_lib.YCBCR_V210_DTYPE)["v210"][0] == 0


def _u8(*shape):
    return torch.zeros(*shape, dtype=torch.uint8)


BAD_FRAMES = {
    "host tensor": lambda: fb.V210Frame(_u8(4, 128), 48),
    "numpy rows": lambda: fb.V210Frame(np.zeros((4, 128), np.uint8), 48),
    "uint16 rows": lambda: fb.V210Frame(torch.zeros(4, 64, dtype=torch.uint16), 48),
    "3-D rows": lambda: fb.V210Frame(_u8(4, 128, 1), 48),
    "unknown matrix": lambda: fb.V210Frame(_u8(4, 128), 48, matrix="bt470"),
    "host tensor then RGB": lambda: [fb.V210Frame(_u8(4, 128), 48), RGB],
    "tensor then host v210": lambda: [torch.zeros(4, 8, 3, dtype=torch.uint8), fb.V210Frame(_u8(4, 128), 48)],
}


@pytest.mark.parametrize("what", list(BAD_FRAMES))
def test_bad_frames_are_refused_before_device_calls(what):
    """A V210Frame must be a CUDA uint8 (H, row bytes) tensor: a host tensor or array, another dtype or rank, or an
    unknown matrix is refused by the constructor, so add and update raise ValueError before any device call (there is no
    device here).  The refusals that need a CUDA tensor (width, pitch, alignment) are in tests/test_gpu_v210.py."""
    make = BAD_FRAMES[what]
    trk = _tracker()
    with pytest.raises(ValueError):
        trk.add(make(), [[1, 1, 2, 2]])
    trk._ids, trk._streams = np.array([0]), np.array([0])
    with pytest.raises(ValueError):
        trk.update(make())
