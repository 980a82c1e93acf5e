"""GPU tests of raw Bayer frames: the FearFrameBayer entry points (fear_crop_targets_bayer_u8,
fear_advance_targets_bayer, fear_frame_sums_bayer_u8), BayerFrame, and FEARMultiTracker / FEARTracker fed Bayer
mosaics.

Every comparison is exact, against image_ops.bayer_to_rgb of the frame's codes (pinned to cv2.cvtColor and to
yuv_to_rgb by tests/test_bayer_cpu.py): identity crops against the demosaiced frame itself, general crops against cv2
on it, boxes against the host rescale + clamp, sums against numpy, and every tracker output against the same tracker
fed the demosaiced frames as numpy arrays.  uint16 samples carry noise in the bits the reader masks, and the samples or
bytes around each frame (past each row, above and below it) hold 0xA5, so a reader that does not mask or that strays
outside the frame is caught."""
import json
import os
import subprocess
import sys

import cv2
import numpy as np
import pytest
import torch

import feartracker_b200 as fb
from feartracker_b200 import _lib, image_ops
from oracle import fear_oracle as fo
from tests import test_gpu_multi_tracker as base
from tests.helpers import GOLDEN, load_full_state
from tests.test_gpu_yuv_formats import code_frame
from tests.test_gpu_yuv_subsampling import encode

pytestmark = pytest.mark.gpu
CFG = fb.FEAR_XS_TRACKER_KWARGS
HERE = os.path.dirname(os.path.abspath(__file__))
PATTERNS = list(image_ops.BAYER_PATTERNS)


@pytest.fixture(scope="module")
def net():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    n = fb.FEARNet(**fb.FEAR_XS_MODEL_KWARGS)
    n.load_state_dict(load_full_state(), strict=True)
    return n.cuda().eval()


@pytest.fixture(scope="module")
def clip():
    return fo.read_video_rgb(os.path.join(GOLDEN, "test.mp4"))


def stream():
    return torch.cuda.current_stream().cuda_stream


# ---------------------------------------------------------------------------------------------------- frames
def samples(codes: np.ndarray, bits: int, msb: bool, rng) -> np.ndarray:
    """The samples that hold ``codes``: uint8 at 8 bits; else uint16, MSB-aligned with random low bits or LSB-aligned
    with random high bits (none at 16 bits)."""
    codes = np.asarray(codes)
    if bits == 8:
        return codes.astype(np.uint8)
    c = codes.astype(np.int64)
    noise = rng.integers(0, 1 << (16 - bits), c.shape) if bits < 16 else np.zeros_like(c)
    return ((c << (16 - bits)) | noise if msb else c | (noise << bits)).astype(np.uint16)


def device(a: np.ndarray) -> torch.Tensor:
    if a.dtype == np.uint16:
        return torch.from_numpy(np.ascontiguousarray(a).view(np.int16)).cuda().view(torch.uint16)
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def place(a: np.ndarray, col: int = 0, extra: int = 0) -> torch.Tensor:
    """``a`` (H, C) at row 1, column ``col`` of a device surface filled with 0xA5 bytes whose rows are ``extra``
    elements longer: the view of ``a`` in it (pitch (col + C + extra) elements)."""
    h, c = a.shape
    surf = np.full((h + 2, col + c + extra), 0xA5A5 if a.dtype == np.uint16 else 0xA5, a.dtype)
    surf[1:h + 1, col:col + c] = a
    return device(surf)[1:h + 1, col:col + c]


def unpacked_frame(codes, pattern, bits, msb=False, col=0, extra=0, rng=None) -> fb.BayerFrame:
    rng = rng or np.random.default_rng(0)
    return fb.BayerFrame(place(samples(codes, bits, msb, rng), col, extra), pattern, bits=bits, msb=msb)


def mipi_rows(codes, bits, pitch=None) -> np.ndarray:
    """RAW10 / RAW12 rows of ``codes`` at ``pitch`` (default: the row bytes), 0xA5 in the bytes past the groups."""
    need = image_ops.mipi_row_bytes(np.shape(codes)[1], bits)
    rows = image_ops.mipi_pack(codes, bits, pitch)
    rows[:, need:] = 0xA5
    return rows


def packed_frame(codes, pattern, bits, pitch=None, col=0) -> fb.BayerFrame:
    w = np.shape(codes)[1]
    rows = mipi_rows(codes, bits, pitch)
    need = image_ops.mipi_row_bytes(w, bits)
    t = place(rows, col)[:, :need]
    return (fb.BayerFrame.raw10 if bits == 10 else fb.BayerFrame.raw12)(t, w, pattern)


def bayer_table(records) -> torch.Tensor:
    return torch.from_numpy(np.array(records, dtype=_lib.BAYER_DTYPE).view(np.uint8).copy()).cuda()


def unreadable_records(rec, wide_rec):
    """Entries the kernels must treat as empty, from a valid 8-bit record ``rec`` and a valid 12-bit uint16 one
    ``wide_rec``: a null address, H or W below 3, a pattern or packing outside its range, bad bits or
    shifts unpacked, a uint16 entry at an odd address or pitch, RAW10 / RAW12 at the wrong depth, and pitches one byte
    short of a row in each packing."""
    d, rs, h, w, pat, bits, shift, pk = rec
    wd, wrs, wh, ww = wide_rec[:4]
    return [
        (0, rs, h, w, pat, 8, 0, 0), (d, rs, 2, w, pat, 8, 0, 0), (d, rs, h, 2, pat, 8, 0, 0),
        (d, rs, 0, w, pat, 8, 0, 0), (d, rs, h, -5, pat, 8, 0, 0),
        (d, rs, h, w, 4, 8, 0, 0), (d, rs, h, w, -1, 8, 0, 0), (d, rs, h, w, pat, 8, 0, 3), (d, rs, h, w, pat, 8, 0, -1),
        (d, rs, h, w, pat, 9, 0, 0), (d, rs, h, w, pat, 11, 0, 0), (d, rs, h, w, pat, 0, 0, 0),
        (d, rs, h, w, pat, 8, 1, 0), (wd, wrs, wh, ww, pat, 12, 5, 0), (wd, wrs, wh, ww, pat, 12, -1, 0),
        (wd, wrs, wh, ww, pat, 16, 1, 0), (wd + 1, wrs, wh, ww, pat, 12, 0, 0), (wd, wrs + 1, wh, ww, pat, 12, 0, 0),
        (d, rs, h, w, pat, 12, 0, 1), (d, rs, h, w, pat, 8, 0, 1), (d, rs, h, w, pat, 10, 0, 2),
        (d, w - 1, h, w, pat, 8, 0, 0), (wd, 2 * ww - 2, wh, ww, pat, 12, 0, 0),
        (d, image_ops.mipi_row_bytes(w, 10) - 1, h, w, pat, 10, 0, 1),
        (d, image_ops.mipi_row_bytes(w, 12) - 1, h, w, pat, 12, 0, 2), (d, -rs, h, w, pat, 8, 0, 0),
    ]


# ---------------------------------------------------------------------------------------------------- kernels
def crop_all(lib, table, F, recs, size, off):
    n = len(recs)
    state = torch.from_numpy(np.asarray(recs, dtype=np.int32)).cuda()
    crops = torch.empty((n, size, size, 3), dtype=torch.uint8, device="cuda")
    _lib.check(lib.fear_crop_targets_bayer_u8(table.data_ptr(), F, state.data_ptr(), n, off, size, crops.data_ptr(),
                                              stream()), "fear_crop_targets_bayer_u8")
    return crops.cpu().numpy(), state.cpu().numpy()


IDENTITY_DEPTHS = [(8, False, "random"), (8, False, "extreme"), (10, False, "random"), (10, True, "random"),
                   (12, False, "random"), (12, True, "extreme"), (14, False, "random"), (14, True, "random"),
                   (16, False, "random"), (16, True, "extreme")]


@pytest.mark.parametrize("depth", IDENTITY_DEPTHS, ids=lambda d: f"{d[0]}-{'msb' if d[1] else 'lsb'}-{d[2]}")
def test_identity_crop_equals_bayer_to_rgb(depth):
    """A 256 x 256 frame whose crop is the frame itself (box [0, 0, 256, 256], offset 0, size 256), once per pattern in
    one table: every pixel, so every site kind and the whole border, equals bayer_to_rgb.  Random codes over the whole
    range, or extreme ones (0, 1, max - 1, max in blocks and alone), with noise in the masked bits."""
    bits, msb, kind = depth
    lib = _lib.init(0)
    rng = np.random.default_rng(bits * 10 + msb)
    top = (1 << bits) - 1
    frames, rgbs = [], []
    for p in PATTERNS:
        if kind == "random":
            codes = rng.integers(0, top + 1, (256, 256))
        else:
            codes = rng.choice([0, 1, top - 1, top], (256, 256))
            codes[::7] = top
            codes[:, 3::11] = 0
        codes = codes.astype(np.uint8 if bits == 8 else np.uint16)
        frames.append(unpacked_frame(codes, p, bits, msb, col=1, extra=5, rng=rng))
        rgbs.append(image_ops.bayer_to_rgb(codes, p, bits))
    table = bayer_table([f.bayer_record() for f in frames])
    recs = np.zeros((4, _lib.TARGET_INTS), dtype=np.int32)
    recs[:, 0] = np.arange(4)
    recs[:, 3:5] = 256
    got, _ = crop_all(lib, table, 4, recs, 256, 0.0)
    for i, p in enumerate(PATTERNS):
        assert np.array_equal(got[i], rgbs[i]), (depth, p)


def test_identity_crop_of_packed_rows_equals_bayer_to_rgb():
    """RAW10 and RAW12 at widths that end in a partial group (W % 4 = 1, 2, 3; W % 2 = 1), tight and pitched: every
    pixel of a 1:1 crop equals bayer_to_rgb of mipi_unpack's codes."""
    lib = _lib.init(0)
    rng = np.random.default_rng(8)
    for bits, w, pitch_extra in ((10, 256, 0), (10, 253, 0), (10, 254, 3), (10, 255, 64), (12, 256, 0), (12, 255, 0),
                                 (12, 253, 7)):
        frames, rgbs = [], []
        for p in PATTERNS:
            codes = rng.integers(0, 1 << bits, (256, w)).astype(np.uint16)
            need = image_ops.mipi_row_bytes(w, bits)
            frames.append(packed_frame(codes, p, bits, need + pitch_extra, col=3))
            assert np.array_equal(image_ops.mipi_unpack(mipi_rows(codes, bits, need + pitch_extra), w, bits), codes)
            rgbs.append(image_ops.bayer_to_rgb(codes, p, bits))
        table = bayer_table([f.bayer_record() for f in frames])
        recs = np.zeros((4, _lib.TARGET_INTS), dtype=np.int32)
        recs[:, 0] = np.arange(4)
        recs[:, 3], recs[:, 4] = w, 256
        got, _ = crop_all(lib, table, 4, recs, 256, 0.0)
        for i, p in enumerate(PATTERNS):
            if w == 256:
                assert np.array_equal(got[i], rgbs[i]), (bits, w, p)
            else:  # a w x 256 box resized to 256 x 256: compare with cv2 on the demosaiced frame
                want = base._cv2_crop(rgbs[i], [0, 0, w, 256], 256, 0.0, np.mean(rgbs[i], axis=(0, 1)))
                assert np.array_equal(got[i], want), (bits, w, p)


# (H, W, container, pattern, pitch extra (elements / bytes), column offset): tight and pitched rows, odd sizes
SHAPES = [(255, 480, ("u8", 8, False), "RGGB", 32, 0), (183, 98, ("u16", 12, True), "GRBG", 0, 0),
          (91, 334, ("raw10", 10, False), "GBRG", 0, 1), (3, 3, ("u8", 8, False), "BGGR", 0, 0),
          (64, 1283, ("raw12", 12, False), "RGGB", 9, 2), (100, 203, ("u16", 10, False), "BGGR", 3, 1)]
TARGETS = [(0, [163, 53, 45, 174]), (0, [-10, 100, 40, 30]), (0, [450, 20, 60, 40]), (0, [200, -15, 30, 50]),
           (0, [0, 0, 3, 3]), (0, [476, 252, 3, 3]), (0, [-50, 30, 600, 100]), (0, [0, 240, 480, 30]),
           (1, [-300, -200, 900, 500]), (1, [95, 180, 3, 3]), (2, [5, 40, 320, 20]), (2, [330, 87, 3, 3]),
           (3, [0, 0, 3, 3]), (3, [-20, -20, 40, 40]), (4, [1270, 30, 40, 40]), (4, [600, 10, 300, 50]),
           (5, [-1, -1, 205, 102]), (5, [100, 50, 50, 50]), (0, [2000, 900, 30, 30])]


def make_frame(codes, container, pattern, extra, col, rng):
    kind, bits, msb = container
    if kind in ("raw10", "raw12"):
        return packed_frame(codes, pattern, bits, image_ops.mipi_row_bytes(codes.shape[1], bits) + extra, col)
    return unpacked_frame(codes, pattern, bits, msb, col, extra, rng)


def kernel_frames(rng):
    frames, rgbs = [], []
    for h, w, container, p, extra, col in SHAPES:
        bits = container[1]
        codes = rng.integers(0, 1 << bits, (h, w)).astype(np.uint8 if bits == 8 else np.uint16)
        frames.append(make_frame(codes, container, p, extra, col, rng))
        rgbs.append(image_ops.bayer_to_rgb(codes, p, bits))
    return frames, rgbs


def test_crop_bayer_kernel_matches_cv2_on_demosaiced_frame():
    """Targets inside, across and touching every border, tiny, huge and outside the frame, on tight and pitched
    uint8 / uint16 rows and RAW10 / RAW12 rows; every unreadable entry and an out-of-range frame index give a
    padding-colour crop."""
    lib = _lib.init(0)
    rng = np.random.default_rng(17)
    frames, rgbs = kernel_frames(rng)
    means = [np.mean(f, axis=(0, 1)) for f in rgbs]
    targets = list(TARGETS)
    for side in (1, 3, 9, 33, 120, 200):
        targets.append((1, [48 - side // 2, 90 - side // 2, side, side]))
    records = [f.bayer_record() for f in frames]
    bad = unreadable_records(records[0], records[1])
    extra = [(9999, [12, 200, 255]), (-1, [1, 2, 3])] + [(len(records) + i, [i, 128, 7]) for i in range(len(bad))]
    recs = np.zeros((len(targets) + len(extra), _lib.TARGET_INTS), dtype=np.int32)
    for i, (f, box) in enumerate(targets):
        recs[i, 0], recs[i, 1:5] = f, box
        recs[i, 9:12] = np.clip(np.rint(means[f]), 0, 255)
    for i, (f, pad) in enumerate(extra):
        recs[len(targets) + i, 0], recs[len(targets) + i, 1:5], recs[len(targets) + i, 9:12] = f, [10, 10, 20, 20], pad
    table = bayer_table(records + bad)
    for size, off in ((256, 2.0), (128, 0.2)):
        got, state = crop_all(lib, table, len(records) + len(bad), recs, size, off)
        for i, (f, box) in enumerate(targets):
            assert np.array_equal(state[i, 5:9], image_ops.context_box(box, off)), (size, off, box)
            assert np.array_equal(got[i], base._cv2_crop(rgbs[f], box, size, off, means[f])), (size, off, f, box)
        for i, (_, pad) in enumerate(extra):
            assert (got[len(targets) + i] == np.array(pad, dtype=np.uint8)).all(), (i, bad[i - 2] if i >= 2 else i)


def test_odd_offset_region_of_interest_names_its_own_pattern():
    """A region of interest of an RGGB mosaic at row 1, column 3 is a BGGR mosaic (and at (0, 1) GRBG, at (1, 0)
    GBRG): its crops equal cv2 on bayer_to_rgb of the region's codes in that pattern."""
    lib = _lib.init(0)
    rng = np.random.default_rng(23)
    full = rng.integers(0, 4096, (260, 500)).astype(np.uint16)
    t = place(samples(full, 12, True, rng))
    frames, rgbs = [], []
    for (r0, c0), p in (((0, 0), "RGGB"), ((0, 1), "GRBG"), ((1, 0), "GBRG"), ((1, 3), "BGGR")):
        frames.append(fb.BayerFrame(t[r0:r0 + 251, c0:c0 + 487], p, bits=12, msb=True))
        rgbs.append(image_ops.bayer_to_rgb(full[r0:r0 + 251, c0:c0 + 487], p, 12))
    table = bayer_table([f.bayer_record() for f in frames])
    boxes = [[163, 53, 45, 174], [-10, -10, 60, 60], [440, 200, 47, 51], [0, 0, 487, 251]]
    recs = np.zeros((16, _lib.TARGET_INTS), dtype=np.int32)
    for i in range(16):
        f, box = i // 4, boxes[i % 4]
        recs[i, 0], recs[i, 1:5], recs[i, 9:12] = f, box, np.clip(np.rint(np.mean(rgbs[f], axis=(0, 1))), 0, 255)
    got, _ = crop_all(lib, table, 4, recs, 256, 2.0)
    for i in range(16):
        f, box = i // 4, boxes[i % 4]
        assert np.array_equal(got[i], base._cv2_crop(rgbs[f], box, 256, 2.0, np.mean(rgbs[f], axis=(0, 1)))), (f, box)


def test_advance_bayer_kernel_matches_host_rescale_and_clamp():
    """12 000 records on Bayer frames of three sizes and packings; unreadable entries and out-of-range frame indices
    keep their boxes."""
    lib = _lib.init(0)
    rng = np.random.default_rng(5)
    shapes = [(255, 480, ("u8", 8, False)), (183, 98, ("u16", 12, True)), (3, 5, ("raw10", 10, False))]
    n = 12000
    boxes = np.zeros(n, dtype=_lib.BOX_DTYPE)
    recs = np.zeros((n, _lib.TARGET_INTS), dtype=np.int32)
    recs[:, 0] = rng.integers(0, 3, n)
    recs[:, 5:7] = rng.integers(-600, 700, (n, 2))
    recs[:, 7:9] = rng.integers(1, 2000, (n, 2))
    boxes["x"], boxes["y"] = rng.uniform(-300, 600, n), rng.uniform(-300, 600, n)
    boxes["w"], boxes["h"] = rng.uniform(0, 300, n), rng.uniform(0, 300, n)
    boxes["w"][:n // 4], boxes["h"][:n // 4] = rng.uniform(0, 3, n // 4), rng.uniform(0, 3, n // 4)
    frames = []
    for h, w, container in shapes:
        codes = rng.integers(0, 1 << container[1], (h, w)).astype(np.uint8 if container[1] == 8 else np.uint16)
        frames.append(make_frame(codes, container, "RGGB", 0, 0, rng))
    records = [f.bayer_record() for f in frames]
    bad = unreadable_records(records[0], records[1])
    table = bayer_table(records + bad)
    recs[-len(bad) - 4:-len(bad), 0] = 999
    recs[-len(bad):, 0] = 3 + np.arange(len(bad))
    kept = len(bad) + 4
    recs[-kept:, 1:5] = [7, 8, 9, 10]
    state = torch.from_numpy(recs).cuda()
    dboxes = torch.from_numpy(boxes.view(np.uint8).copy()).cuda()
    _lib.check(lib.fear_advance_targets_bayer(dboxes.data_ptr(), table.data_ptr(), 3 + len(bad), state.data_ptr(), n,
                                              256, stream()), "fear_advance_targets_bayer")
    got = state.cpu().numpy()
    for i in range(n - kept):
        b = np.array([boxes["x"][i], boxes["y"][i], boxes["w"][i], boxes["h"][i]])
        h, w, _ = shapes[recs[i, 0]]
        want = image_ops.clamp_bbox(image_ops.rescale_bbox(b, recs[i, 5:9], 256), (h, w, 3))
        assert np.array_equal(got[i, 1:5], want), (i, b.tolist(), recs[i, 5:9].tolist(), (h, w), got[i, 1:5], want)
    assert (got[-kept:, 1:5] == [7, 8, 9, 10]).all()
    assert np.array_equal(np.delete(got, np.s_[1:5], axis=1), np.delete(recs, np.s_[1:5], axis=1))


def test_frame_sums_bayer_give_numpy_sums_of_demosaiced_frame():
    lib = _lib.init(0)
    rng = np.random.default_rng(11)
    cases = [((3, 3), ("u8", 8, False), "RGGB"), ((3, 4), ("u16", 16, True), "GRBG"),
             ((5, 3), ("raw12", 12, False), "GBRG"), ((183, 98), ("raw10", 10, False), "BGGR"),
             ((37, 1005), ("u16", 14, False), "RGGB"), ((1080, 1920), ("u8", 8, False), "GRBG"),
             ((1081, 1918), ("raw10", 10, False), "RGGB"), ((2160, 3840), ("u16", 12, True), "BGGR")]
    frames, rgbs = [], []
    for (h, w), container, p in cases:
        bits = container[1]
        codes = rng.integers(0, 1 << bits, (h, w)).astype(np.uint8 if bits == 8 else np.uint16)
        frames.append(make_frame(codes, container, p, 4, 0, rng))
        rgbs.append(image_ops.bayer_to_rgb(codes, p, bits))
    records = [f.bayer_record() for f in frames]
    bad = unreadable_records(records[0], records[1])
    table = bayer_table(records + bad)
    F = len(records) + len(bad)
    sums = torch.full((F, 3), -1, dtype=torch.int64, device="cuda")  # zeroed by the call
    _lib.check(lib.fear_frame_sums_bayer_u8(table.data_ptr(), F, sums.data_ptr(), stream()), "fear_frame_sums_bayer_u8")
    got = sums.cpu().numpy().view(np.uint64)
    for i, rgb in enumerate(rgbs):
        assert np.array_equal(got[i], rgb.sum(axis=(0, 1), dtype=np.uint64)), (i, cases[i])
        assert np.array_equal(np.clip(np.rint(got[i] / (rgb.shape[0] * rgb.shape[1])), 0, 255),
                              np.clip(np.rint(np.mean(rgb, axis=(0, 1))), 0, 255))
    assert (got[len(records):] == 0).all()


def test_c_abi_rejects_bad_arguments_and_launches_nothing():
    lib = _lib.init(0)
    t = torch.full((1 << 16,), 0x5A, dtype=torch.uint8, device="cuda")
    p = t.data_ptr()
    good = dict(views=p, F=1, targets=p, N=1, offset=2.0, size=256, crops=p)

    def crop(**kw):
        a = dict(good, **kw)
        return lib.fear_crop_targets_bayer_u8(a["views"], a["F"], a["targets"], a["N"], a["offset"], a["size"],
                                              a["crops"], None)

    bad = [dict(views=None), dict(targets=None), dict(crops=None), dict(N=0), dict(N=-1), dict(N=65536), dict(F=0),
           dict(F=-3), dict(size=0), dict(size=257), dict(offset=-0.5), dict(offset=float("nan")),
           dict(offset=float("inf"))]
    for kw in bad:
        assert crop(**kw) == -1, kw
        assert _lib.last_error(), kw
    for args in [(None, p, 1, p, 1, 256), (p, None, 1, p, 1, 256), (p, p, 1, None, 1, 256), (p, p, 1, p, 0, 256),
                 (p, p, 0, p, 1, 256), (p, p, 1, p, 1, 0)]:
        assert lib.fear_advance_targets_bayer(*args, None) == -1, args
        assert _lib.last_error(), args
    for args in [(None, 1, p), (p, 1, None), (p, 0, p), (p, 65536, p), (p, -1, p)]:
        assert lib.fear_frame_sums_bayer_u8(*args, None) == -1, args
        assert _lib.last_error(), args
    torch.cuda.synchronize()
    assert (t == 0x5A).all()  # no kernel and no memset ran


# ---------------------------------------------------------------------------------------------------- BayerFrame
def _dev(h, w, dtype=torch.uint8):
    return torch.zeros((h, w), dtype=dtype, device="cuda")


def test_bayer_frame_records_its_mosaic():
    surf = _dev(8, 2000, torch.uint16)
    f = fb.BayerFrame(surf[1:7, 3:1923], "GRBG", bits=12, msb=True)
    assert f.shape == (6, 1920, 3) and f.pitch == 4000
    rec = np.array([f.bayer_record()], dtype=_lib.BAYER_DTYPE)[0]
    assert rec["data"] == surf.data_ptr() + 4000 + 6 and rec["row_stride"] == 4000
    assert (rec["H"], rec["W"], rec["pattern"], rec["bits"], rec["shift"], rec["packing"]) == (6, 1920, 1, 12, 4, 0)
    assert fb.BayerFrame(surf[:, :5], bits=16, msb=True).bayer_record()[4:] == (0, 16, 0, 0)
    assert fb.BayerFrame(_dev(3, 3)).bayer_record()[1:] == (3, 3, 3, 0, 8, 0, 0)
    raw = _dev(5, 3000)
    r10 = fb.BayerFrame.raw10(raw[1:4, 7:7 + 2400], 1920, "BGGR")
    assert r10.shape == (3, 1920, 3) and r10.bayer_record() == (raw.data_ptr() + 3007, 3000, 3, 1920, 3, 10, 0, 1)
    r12 = fb.BayerFrame.raw12(raw[:, :6], 3, "GBRG")
    assert r12.shape == (5, 3, 3) and r12.bayer_record()[1:] == (3000, 5, 3, 2, 12, 0, 2)


BAD_BAYER = {
    "2 rows": lambda: fb.BayerFrame(_dev(2, 8)),
    "2 columns": lambda: fb.BayerFrame(_dev(8, 2)),
    "uint8 at 12 bits": lambda: fb.BayerFrame(_dev(8, 8), bits=12),
    "uint16 at 8 bits": lambda: fb.BayerFrame(_dev(8, 8, torch.uint16)),
    "int16 samples": lambda: fb.BayerFrame(_dev(8, 8, torch.int16), bits=12),
    "strided columns": lambda: fb.BayerFrame(_dev(8, 16)[:, ::2]),
    "rows overlap": lambda: fb.BayerFrame(_dev(8, 16).as_strided((8, 16), (8, 1))),
    "transposed": lambda: fb.BayerFrame(_dev(16, 8).t()),
    "raw10 short row": lambda: fb.BayerFrame.raw10(_dev(8, 9), 8),
    "raw12 short row": lambda: fb.BayerFrame.raw12(_dev(8, 11), 7),
    "raw10 width 2": lambda: fb.BayerFrame.raw10(_dev(8, 10), 2),
    "raw10 width float": lambda: fb.BayerFrame.raw10(_dev(8, 10), 8.0),
    "raw10 uint16": lambda: fb.BayerFrame.raw10(_dev(8, 10, torch.uint16), 8),
    "raw12 pitch below the row": lambda: fb.BayerFrame.raw12(_dev(8, 24).view(-1)[:96].as_strided((8, 12), (11, 1)),
                                                             8),
    "misaligned uint16": lambda: fb.BayerFrame(_dev(8, 34)[:, 1:33].view(torch.uint16), bits=10),
}


@pytest.mark.parametrize("what", list(BAD_BAYER))
def test_bayer_frame_refuses_malformed_tensors(what):
    with pytest.raises((ValueError, RuntimeError)) as e:
        BAD_BAYER[what]()
    if what != "misaligned uint16":  # torch itself may refuse that view
        assert e.type is ValueError


def test_tracker_refuses_bayer_mixed_with_other_kinds(net):
    trk = fb.FEARMultiTracker(net, cuda_id=0, max_targets=4, **CFG)
    f = fb.BayerFrame(torch.zeros((64, 80), dtype=torch.uint8, device="cuda"))
    rgb = torch.zeros((64, 80, 3), dtype=torch.uint8, device="cuda")
    nv12 = fb.YUV420Frame.nv12(torch.zeros((96, 80), dtype=torch.uint8, device="cuda"))
    for frames in ([f, np.zeros((64, 80, 3), np.uint8)], [rgb, f], [nv12, f]):
        with pytest.raises(ValueError, match="BayerFrames cannot share"):
            trk.add(frames, [[1, 1, 20, 20]])
    with pytest.raises(ValueError, match="not a mix"):  # the other mixes keep their message
        trk.add([rgb, nv12], [[1, 1, 20, 20]])
    assert len(trk) == 0


# ---------------------------------------------------------------------------------------------------- trackers
def mosaic(rgb: np.ndarray, pattern: str, bits: int, rng) -> np.ndarray:
    """The Bayer codes a sensor with ``pattern`` would give for an RGB frame: each site's colour, scaled to ``bits``,
    plus uniform noise of +-2 codes, clipped."""
    p = image_ops.BAYER_PATTERNS[pattern]
    ry, rx = p >> 1, p & 1
    h, w = rgb.shape[:2]
    yy, xx = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    r_row, r_col = ((yy ^ ry) & 1) == 0, ((xx ^ rx) & 1) == 0
    ch = np.where(r_row & r_col, 0, np.where(~r_row & ~r_col, 2, 1))
    v = np.take_along_axis(rgb, ch[..., None], 2)[..., 0].astype(np.float64) * ((1 << bits) - 1) / 255.0
    v = np.clip(np.rint(v + rng.uniform(-2, 2, v.shape)), 0, (1 << bits) - 1)
    return v.astype(np.uint8 if bits == 8 else np.uint16)


# stream: (size (W, H), container, pattern, pitch extra): pitched 1080p RGGB8, BayerGR12 MSB, RAW10 with a pitch
BAYER_STREAMS = [((1920, 1080), ("u8", 8, False), "RGGB", 128), ((1920, 1080), ("u16", 12, True), "GRBG", 64),
                 ((1920, 1080), ("raw10", 10, False), "BGGR", 80)]


def bayer_clip(clip, T, rng):
    codes, rgb = [], []
    for size, container, p, _ in BAYER_STREAMS:
        c = [mosaic(cv2.resize(clip[t], size), p, container[1], rng) for t in range(T + 1)]
        codes.append(c)
        rgb.append([image_ops.bayer_to_rgb(x, p, container[1]) for x in c])
    return codes, rgb


def bayer_frames(codes, t, rng):
    return [make_frame(codes[s][t], c, p, extra, 2 * s, rng) for s, (_, c, p, extra) in enumerate(BAYER_STREAMS)]


def test_multi_tracker_on_bayer_matches_numpy_rgb(net, clip):
    """Three 1080p Bayer streams (pitched RGGB8, BayerGR12 MSB, RAW10), several targets each, with add / remove part way
    and calls on numpy, CUDA RGB and NV12 frames of the same pixels in between.  Every output equals a tracker fed the
    demosaiced frames as numpy arrays; steady Bayer calls replay one captured graph of the bayer table, of 48 launches,
    and the graph is captured again after the net's workspace grows."""
    T = 40
    rng = np.random.default_rng(97)
    codes, rgb = bayer_clip(clip, T, rng)
    n2 = fb.FEARNet(**fb.FEAR_XS_MODEL_KWARGS)
    n2.load_state_dict(load_full_state(), strict=True)
    n2 = n2.cuda().eval()
    ref = fb.FEARMultiTracker(n2, cuda_id=0, max_targets=12, **CFG)
    trk = fb.FEARMultiTracker(n2, cuda_id=0, max_targets=12, **CFG)
    start = [[[652, 211, 180, 696], [1700, 840, 160, 224]], [[900, 400, 120, 300]], [[0, 0, 60, 60], [1800, 1000,
                                                                                                      120, 80]]]
    late = [[[400, 600, 120, 120]], [[100, 150, 30, 30]], []]

    def rects(d):
        return [r for s in d for r in s], [k for k, s in enumerate(d) for _ in s]

    def other(t, kind):
        """The demosaiced frames of time t as another kind of frame: CUDA RGB tensors, or NV12 frames whose
        yuv_to_rgb the reference is fed instead."""
        if kind == "cuda":
            return [torch.from_numpy(rgb[s][t]).cuda() for s in range(3)], [rgb[s][t] for s in range(3)]
        planes = [encode(rgb[s][t], "bt601", False, 8, "420", rng) for s in range(3)]
        return ([code_frame(*pl, "nv12", "bt601", False, 8, rng) for pl in planes],
                [image_ops.yuv_to_rgb(*pl) for pl in planes])

    r, s = rects(start)
    assert np.array_equal(trk.add(bayer_frames(codes, 0, rng), r, s), ref.add([x[0] for x in rgb], r, s))
    graphs = []
    for t in range(1, T + 1):
        if t == 12:
            r, s = rects(late)
            assert np.array_equal(trk.add(bayer_frames(codes, t - 1, rng), r, s),
                                  ref.add([x[t - 1] for x in rgb], r, s))
        if t == 22:
            for x in (ref, trk):
                x.remove([1, 2])
        if t == 30:
            gen = n2.generation()
            zt, xt, _, _ = fo.synthetic_crops(16)
            n2.track(xt.cuda(), n2.get_features(zt.cuda()))  # batch 16 > reserved 12: the workspace grows
            assert n2.generation() != gen
        if t in (8, 18, 27):  # another kind of frame in between: its own table, then back to the Bayer graph
            frames, want_frames = other(t, "cuda" if t != 18 else "nv12")
            if t == 27:
                frames, want_frames = [x[t] for x in rgb], [x[t] for x in rgb]
            expect, out = ref.update(want_frames), trk.update(frames)
            assert trk._graph_key[2] != "bayer"
        else:
            expect = ref.update([x[t] for x in rgb])
            out = trk.update(bayer_frames(codes, t, rng))
            assert trk._graph_key[2] == "bayer"
        assert np.array_equal(out["ids"], expect["ids"]), t
        assert np.array_equal(out["bbox"], expect["bbox"]), (t, out["bbox"], expect["bbox"])
        assert np.array_equal(out["score"], expect["score"]), t
        if t in (3, 10, 14, 20, 24, 29, 32):  # two Bayer updates after the start, each switch, add, remove, growth
            assert trk._graph is not None and all(trk._graph is not g for g in graphs), t
            graphs.append(trk._graph)
            if t == 32:
                assert trk._graph_gen == n2.generation()
        if t in (7, 17, 21, 26, T):
            assert trk._graph is graphs[-1], t  # replayed with new surface addresses every update
    # the step's launches: the crop and advance entry points around the network's own
    eager = fb.FEARMultiTracker(n2, cuda_id=0, max_targets=12, cuda_graph=False, **CFG)
    eager.add(bayer_frames(codes, 0, rng), *rects(start))
    eager.update(bayer_frames(codes, 1, rng))
    torch.cuda.synchronize()
    c0 = n2.launch_count()
    eager.update(bayer_frames(codes, 2, rng))
    assert n2.launch_count() - c0 + 2 == 48


@pytest.mark.parametrize("smooth", [False, True], ids=["plain", "smooth"])
def test_fear_tracker_on_bayer_matches_numpy_rgb(net, clip, smooth):
    """FEARTracker on pitched 1080p BayerGR12 MSB frames (graphed, and eager), with RAW10 and RGGB8 frames and a numpy
    frame part way, gives the trajectory and tracking_state of the same tracker on the demosaiced frames as numpy
    arrays."""
    T = 25
    rng = np.random.default_rng(61)
    codes, rgb = bayer_clip(clip, T, rng)
    init = np.array([652, 211, 180, 696])
    for extra in ({}, {"cuda_graph": False}):
        cfg = dict(CFG, smooth=smooth, **extra)
        ref, trk = fb.FEARTracker(net, cuda_id=0, **cfg), fb.FEARTracker(net, cuda_id=0, **cfg)
        ref.initialize(rgb[1][0], init)
        trk.initialize(bayer_frames(codes, 0, rng)[1], init)
        assert np.array_equal(trk.tracking_state.mean_color, ref.tracking_state.mean_color)
        for t in range(1, T + 1):
            s = 1 if t < 10 else (0 if t < 15 else 2)  # same pixels up to the codes' noise: a stream switch
            want = ref.update(rgb[s][t])["bbox"]
            frame = rgb[s][t] if t == 20 else bayer_frames(codes, t, rng)[s]
            got = trk.update(frame)["bbox"]
            assert np.array_equal(got, want), (smooth, extra, t, got, want)
            for key in ("bbox", "mapping", "prev_size"):
                assert np.array_equal(getattr(trk.tracking_state, key), getattr(ref.tracking_state, key)), (key, t)
        assert [list(p) for p in trk.tracking_state.paths] == [list(p) for p in ref.tracking_state.paths]
        z_ref = ref.get_template_features(rgb[0][3], [600, 200, 100, 300])
        z_trk = trk.get_template_features(bayer_frames(codes, 3, rng)[0], [600, 200, 100, 300])
        assert torch.equal(z_ref, z_trk)


# ---------------------------------------------------------------------------------------------------- poison
def test_bayer_entry_points_and_trackers_on_poisoned_memory():
    """tests/poison_bayer_check.py in its own process: guarded, poisoned tables, crops, sums, boxes and mosaics."""
    proc = subprocess.run([sys.executable, os.path.join(HERE, "poison_bayer_check.py")], capture_output=True, text=True,
                          timeout=1200)
    lines = [l for l in proc.stdout.splitlines() if l.startswith("POISON_CHECK ")]
    assert proc.returncode == 0 and lines, f"poison_bayer_check failed: {proc.stderr[-3000:]}"
    res = json.loads(lines[-1][len("POISON_CHECK "):])
    assert res["checked_calls"] > 0
    assert res["n_failures"] == 0, res["failures"]
