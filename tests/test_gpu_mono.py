"""GPU tests of single-channel frames: the FearFrameMono entry points (fear_frame_range_mono, fear_crop_targets_mono_u8,
fear_advance_targets_mono, fear_frame_sums_mono_u8), MonoFrame, and FEARMultiTracker / FEARTracker fed mono frames
with and without min-max gain control.

Every comparison is exact, against image_ops.mono_to_rgb of the frame's codes (pinned to cv2.cvtColor(GRAY2RGB) and
cv2.normalize(NORM_MINMAX, CV_8U) by tests/test_mono_cpu.py): identity crops against the grey frame itself, general
crops against cv2 on it, ranges against torch.aminmax, boxes against the host rescale + clamp, sums against numpy, and
every tracker output against the same tracker fed the grey frames as numpy arrays.  As in tests/test_gpu_bayer.py,
uint16 samples carry noise in the bits the reader masks and the memory around each frame holds 0xA5."""
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
from tests.test_gpu_bayer import mipi_rows, place, samples

pytestmark = pytest.mark.gpu
CFG = fb.FEAR_XS_TRACKER_KWARGS
HERE = os.path.dirname(os.path.abspath(__file__))
INT_MAX, INT_MIN = 2 ** 31 - 1, -2 ** 31


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


def _dt(bits):
    return np.uint8 if bits == 8 else np.uint16


# ---------------------------------------------------------------------------------------------------- frames
def make_frame(codes, container, agc=None, extra=0, col=0, rng=None) -> fb.MonoFrame:
    """A MonoFrame holding ``codes`` in ``container`` ("u8", "u16", "raw10", "raw12", bits, msb) at row 1, column
    ``col`` of a 0xA5 surface with ``extra`` elements / bytes of pitch past each row."""
    kind, bits, msb = container
    rng = rng or np.random.default_rng(0)
    if kind in ("raw10", "raw12"):
        w = np.shape(codes)[1]
        need = image_ops.mipi_row_bytes(w, bits)
        t = place(mipi_rows(codes, bits, need + extra), col)[:, :need]
        return (fb.MonoFrame.raw10 if bits == 10 else fb.MonoFrame.raw12)(t, w, agc=agc)
    return fb.MonoFrame(place(samples(codes, bits, msb, rng), col, extra), bits=bits, msb=msb, agc=agc)


def mono_table(records) -> torch.Tensor:
    return torch.from_numpy(np.array(records, dtype=_lib.MONO_DTYPE).view(np.uint8).copy()).cuda()


def table_records(table: torch.Tensor) -> np.ndarray:
    return table.cpu().numpy().view(_lib.MONO_DTYPE)


def run_range(lib, table, F):
    _lib.check(lib.fear_frame_range_mono(table.data_ptr(), F, stream()), "fear_frame_range_mono")


def unreadable_records(rec, wide_rec):
    """Entries the kernels must treat as empty, from a valid 8-bit record ``rec`` and a valid 12-bit uint16 one
    ``wide_rec`` (both with agc): a null address, H or W below 1, a packing or agc outside its range, bad bits or shifts
    unpacked, a uint16 entry at an odd address or pitch, RAW10 / RAW12 at the wrong depth, and pitches one byte short of
    a row in each packing."""
    d, rs, h, w, bits, shift, pk, agc, lo, hi = rec
    wd, wrs, wh, ww = wide_rec[:4]
    e = (lo, hi)
    return [
        (0, rs, h, w, 8, 0, 0, 1) + e, (d, rs, 0, w, 8, 0, 0, 1) + e, (d, rs, h, 0, 8, 0, 0, 1) + e,
        (d, rs, h, -5, 8, 0, 0, 1) + e, (d, rs, h, w, 8, 0, 3, 1) + e, (d, rs, h, w, 8, 0, -1, 1) + e,
        (d, rs, h, w, 8, 0, 0, 2) + e, (d, rs, h, w, 8, 0, 0, -1) + e,
        (d, rs, h, w, 9, 0, 0, 1) + e, (d, rs, h, w, 11, 0, 0, 1) + e, (d, rs, h, w, 0, 0, 0, 1) + e,
        (d, rs, h, w, 8, 1, 0, 1) + e, (wd, wrs, wh, ww, 12, 5, 0, 1) + e, (wd, wrs, wh, ww, 12, -1, 0, 1) + e,
        (wd, wrs, wh, ww, 16, 1, 0, 1) + e, (wd + 1, wrs, wh, ww, 12, 0, 0, 1) + e, (wd, wrs + 1, wh, ww, 12, 0, 0, 1) + e,
        (d, rs, h, w, 12, 0, 1, 1) + e, (d, rs, h, w, 8, 0, 1, 1) + e, (d, rs, h, w, 10, 0, 2, 1) + e,
        (d, w - 1, h, w, 8, 0, 0, 1) + e, (wd, 2 * ww - 2, wh, ww, 12, 0, 0, 1) + e,
        (d, image_ops.mipi_row_bytes(w, 10) - 1, h, w, 10, 0, 1, 1) + e,
        (d, image_ops.mipi_row_bytes(w, 12) - 1, h, w, 12, 0, 2, 1) + e, (d, -rs, h, w, 8, 0, 0, 1) + e,
    ]


def crop_all(lib, table, F, recs, size, off):
    n = len(recs)
    state = torch.from_numpy(np.asarray(recs, dtype=np.int32)).cuda()
    crops = torch.empty((n, size, size, 3), dtype=torch.uint8, device="cuda")
    _lib.check(lib.fear_crop_targets_mono_u8(table.data_ptr(), F, state.data_ptr(), n, off, size, crops.data_ptr(),
                                             stream()), "fear_crop_targets_mono_u8")
    return crops.cpu().numpy(), state.cpu().numpy()


# ---------------------------------------------------------------------------------------------------- kernels
DEPTHS = [(8, False), (10, False), (10, True), (12, False), (12, True), (14, False), (14, True), (16, False),
          (16, True)]


@pytest.mark.parametrize("agc", [None, "minmax"], ids=["plain", "agc"])
@pytest.mark.parametrize("depth", DEPTHS, ids=lambda d: f"{d[0]}-{'msb' if d[1] else 'lsb'}")
def test_identity_crop_equals_mono_to_rgb(depth, agc):
    """256 x 256 frames cropped 1:1 (box [0, 0, 256, 256], offset 0, size 256) after the range kernel: every pixel
    equals mono_to_rgb.  One frame of random codes over the whole range, one of a narrow band, one of extremes."""
    bits, msb = depth
    lib = _lib.init(0)
    rng = np.random.default_rng(bits * 10 + msb + (agc is not None))
    top = (1 << bits) - 1
    lo = int(rng.integers(0, top - 40))
    sets = [rng.integers(0, top + 1, (256, 256)), rng.integers(lo, lo + 41, (256, 256)),
            rng.choice([0, 1, top - 1, top], (256, 256))]
    frames, rgbs = [], []
    for codes in sets:
        codes = codes.astype(_dt(bits))
        frames.append(make_frame(codes, ("u8" if bits == 8 else "u16", bits, msb), agc, extra=5, col=1, rng=rng))
        rgbs.append(image_ops.mono_to_rgb(codes, bits, agc))
    table = mono_table([f.mono_record() for f in frames])
    run_range(lib, table, len(frames))
    recs = np.zeros((len(frames), _lib.TARGET_INTS), dtype=np.int32)
    recs[:, 0] = np.arange(len(frames))
    recs[:, 3:5] = 256
    got, _ = crop_all(lib, table, len(frames), recs, 256, 0.0)
    for i, rgb in enumerate(rgbs):
        assert np.array_equal(got[i], rgb), (depth, agc, i)


@pytest.mark.parametrize("agc", [None, "minmax"], ids=["plain", "agc"])
def test_identity_crop_of_packed_rows_equals_mono_to_rgb(agc):
    """RAW10 / RAW12 rows ending in a partial group, tight and pitched; 1:1 crops equal mono_to_rgb of the codes, and
    crops of the narrower frames equal cv2 on it."""
    lib = _lib.init(0)
    rng = np.random.default_rng(8 + (agc is not None))
    for bits, w, extra in ((10, 256, 0), (10, 253, 0), (10, 254, 3), (10, 255, 64), (12, 256, 0), (12, 255, 7)):
        codes = rng.integers(0, 1 << bits, (256, w)).astype(np.uint16)
        if agc:
            codes = (codes % 97 + 300).astype(np.uint16)
        f = make_frame(codes, (f"raw{bits}", bits, False), agc, extra=extra, col=3)
        rgb = image_ops.mono_to_rgb(codes, bits, agc)
        table = mono_table([f.mono_record()])
        run_range(lib, table, 1)
        recs = np.zeros((1, _lib.TARGET_INTS), dtype=np.int32)
        recs[:, 3], recs[:, 4] = w, 256
        got, _ = crop_all(lib, table, 1, recs, 256, 0.0)
        want = rgb if w == 256 else base._cv2_crop(rgb, [0, 0, w, 256], 256, 0.0, np.mean(rgb, axis=(0, 1)))
        assert np.array_equal(got[0], want), (bits, w, extra)


# frame: (H, W), container, agc, pitch extra, column offset: tight, pitched, regions of interest, packed, 1-pixel sides
SHAPES = [((255, 480), ("u8", 8, False), None, 32, 0), ((183, 98), ("u16", 12, True), "minmax", 0, 0),
          ((91, 334), ("raw10", 10, False), "minmax", 0, 1), ((1, 1), ("u8", 8, False), None, 0, 0),
          ((64, 1283), ("raw12", 12, False), None, 9, 2), ((100, 203), ("u16", 16, False), "minmax", 3, 1),
          ((1, 57), ("u16", 14, False), "minmax", 0, 0), ((43, 1), ("raw10", 10, False), None, 0, 0)]
TARGETS = [(0, [163, 53, 45, 174]), (0, [-10, 100, 40, 30]), (0, [450, 20, 60, 40]), (0, [200, -15, 30, 50]),
           (0, [0, 0, 3, 3]), (1, [-300, -200, 900, 500]), (1, [95, 180, 3, 3]), (2, [5, 40, 320, 20]),
           (2, [330, 87, 3, 3]), (3, [0, 0, 1, 1]), (3, [-20, -20, 40, 40]), (4, [1270, 30, 40, 40]),
           (4, [600, 10, 300, 50]), (5, [-1, -1, 205, 102]), (5, [100, 50, 50, 50]), (6, [0, 0, 57, 1]),
           (6, [20, -5, 10, 10]), (7, [0, 0, 1, 43]), (7, [-3, 10, 5, 5]), (0, [2000, 900, 30, 30])]


def shape_frames(rng):
    frames, rgbs = [], []
    for (h, w), container, agc, extra, col in SHAPES:
        bits = container[1]
        codes = rng.integers(0, 1 << bits, (h, w))
        if agc:
            codes = codes % 500 + (1 << bits) // 3
        codes = codes.astype(_dt(bits))
        frames.append(make_frame(codes, container, agc, extra, col, rng))
        rgbs.append(image_ops.mono_to_rgb(codes, bits, agc))
    return frames, rgbs


@pytest.mark.parametrize("size,off", [(256, 2.0), (128, 0.2)])
def test_general_crops_equal_cv2(size, off):
    """Targets inside, across and outside frames of every container, with and without gain control, against the cv2
    crop of the grey RGB frame; targets past F or on unreadable entries get their padding colour."""
    lib = _lib.init(0)
    rng = np.random.default_rng(3)
    frames, rgbs = shape_frames(rng)
    records = [f.mono_record() for f in frames]
    bad = unreadable_records(records[0], records[1])
    table = mono_table(records + bad)
    F = len(records) + len(bad)
    run_range(lib, table, F)
    means = [np.mean(f, axis=(0, 1)) for f in rgbs]
    extra = [(9999, [12, 200, 255]), (-1, [1, 2, 3])] + [(len(records) + i, [i, 128, 7]) for i in range(len(bad))]
    recs = np.zeros((len(TARGETS) + len(extra), _lib.TARGET_INTS), dtype=np.int32)
    for i, (f, box) in enumerate(TARGETS):
        recs[i, 0], recs[i, 1:5] = f, box
        recs[i, 9:12] = np.clip(np.rint(means[f]), 0, 255)
    for j, (f, pad) in enumerate(extra):
        recs[len(TARGETS) + j, 0], recs[len(TARGETS) + j, 1:5] = f, [5, 5, 30, 30]
        recs[len(TARGETS) + j, 9:12] = pad
    got, state = crop_all(lib, table, F, recs, size, off)
    for i, (f, box) in enumerate(TARGETS):
        want = base._cv2_crop(rgbs[f], box, size, off, means[f])
        assert np.array_equal(got[i], want), (i, f, box)
        assert np.array_equal(state[i, 5:9], image_ops.context_box(box, off))
    for j, (f, pad) in enumerate(extra):
        assert (got[len(TARGETS) + j] == np.array(pad, np.uint8)).all(), (f, pad)


def test_range_kernel_equals_aminmax():
    """lo / hi against torch.aminmax of the unpacked codes, up to 2160 x 3840, with the extremes alone at the first
    pixel, at the last pixel and in a packed tail group, on constant frames, and with entries without agc and
    unreadable entries left untouched."""
    lib = _lib.init(0)
    rng = np.random.default_rng(21)
    cases = []
    for (h, w), container in (((2160, 3840), ("u16", 16, False)), ((2160, 3840), ("u16", 12, True)),
                              ((1080, 1920), ("u8", 8, False)), ((1081, 1917), ("raw10", 10, False)),
                              ((1079, 1919), ("raw12", 12, False)), ((1, 1), ("u16", 14, False)),
                              ((3, 5), ("raw10", 10, False)), ((7, 1), ("raw12", 12, False))):
        bits = container[1]
        top = (1 << bits) - 1
        mid = top // 2
        body = rng.integers(mid - 50, mid + 51, (h, w))
        first, last, tail = body.copy(), body.copy(), body.copy()
        first[0, 0] = 0
        first[-1, -1] = top
        last[-1, -1] = 0
        last[0, 0] = top if h * w > 1 else 0
        tail[h // 2, w - 1] = top  # in the last, possibly partial, group of a packed row
        tail[h - 1, w - 1 - (w > 1)] = 1
        const = np.full((h, w), mid)
        for codes in (body, first, last, tail, const):
            cases.append((codes.astype(_dt(bits)), container))
    frames = [make_frame(c, container, "minmax", extra=3, col=1, rng=rng) for c, container in cases]
    records = [f.mono_record() for f in frames]
    plain = list(records[0])
    plain[7] = 0  # agc 0: not read, not written
    bad = unreadable_records(records[10], records[5])
    table = mono_table(records + [tuple(plain)] + bad)
    F = len(records) + 1 + len(bad)
    run_range(lib, table, F)
    torch.cuda.synchronize()
    got = table_records(table)
    for i, (codes, container) in enumerate(cases):
        lo, hi = torch.aminmax(torch.from_numpy(codes.astype(np.int32)))
        assert (got[i]["lo"], got[i]["hi"]) == (int(lo), int(hi)), (i, container, codes.shape)
    for r in got[len(records):]:
        assert (r["lo"], r["hi"]) == (INT_MAX, INT_MIN)
    # run again on the written table: min and max are idempotent
    run_range(lib, table, F)
    assert np.array_equal(table_records(table), got)


def test_advance_keeps_boxes_of_unreadable_entries():
    lib = _lib.init(0)
    rng = np.random.default_rng(5)
    shapes = [(255, 480, ("u8", 8, False)), (183, 98, ("u16", 12, True)), (1, 5, ("raw10", 10, False))]
    frames = [make_frame(rng.integers(0, 1 << c[1], (h, w)).astype(_dt(c[1])), c, "minmax", rng=rng)
              for h, w, c in shapes]
    records = [f.mono_record() for f in frames]
    bad = unreadable_records(records[0], records[1])
    table = mono_table(records + bad)
    n = 12000
    boxes = np.zeros(n, dtype=_lib.BOX_DTYPE)
    boxes["x"], boxes["y"] = rng.uniform(-300, 600, n), rng.uniform(-300, 600, n)
    boxes["w"], boxes["h"] = rng.uniform(0, 400, n), rng.uniform(0, 400, n)
    recs = np.zeros((n, _lib.TARGET_INTS), dtype=np.int32)
    recs[:, 0] = rng.integers(0, 3, n)
    recs[:, 5:7] = rng.integers(-600, 700, (n, 2))
    recs[:, 7:9] = rng.integers(1, 2000, (n, 2))
    recs[-len(bad):, 0] = 3 + np.arange(len(bad))
    kept = len(bad) + 4
    recs[-4 - len(bad):-len(bad), 0] = [-1, 3 + len(bad), 9999, INT_MIN]
    recs[-kept:, 1:5] = [7, 8, 9, 10]
    state = torch.from_numpy(recs).cuda()
    dboxes = torch.from_numpy(boxes.view(np.uint8).copy()).cuda()
    _lib.check(lib.fear_advance_targets_mono(dboxes.data_ptr(), table.data_ptr(), 3 + len(bad), state.data_ptr(), n,
                                             256, stream()), "fear_advance_targets_mono")
    got = state.cpu().numpy()
    for i in range(n - kept):
        b = np.array([boxes["x"][i], boxes["y"][i], boxes["w"][i], boxes["h"][i]])
        h, w, _ = shapes[recs[i, 0]]
        want = image_ops.clamp_bbox(image_ops.rescale_bbox(b, recs[i, 5:9], 256), (h, w, 3))
        assert np.array_equal(got[i, 1:5], want), (i, (h, w))
    assert (got[-kept:, 1:5] == [7, 8, 9, 10]).all()
    assert np.array_equal(np.delete(got, np.s_[1:5], axis=1), np.delete(recs, np.s_[1:5], axis=1))


def test_frame_sums_mono_give_numpy_sums_of_grey_frame():
    """Sums up to 2160 x 3840 with and without gain control, and 0 for unreadable entries."""
    lib = _lib.init(0)
    rng = np.random.default_rng(11)
    cases = [((1, 1), ("u8", 8, False), None), ((3, 4), ("u16", 16, True), "minmax"),
             ((5, 3), ("raw12", 12, False), "minmax"), ((183, 98), ("raw10", 10, False), None),
             ((37, 1005), ("u16", 14, False), "minmax"), ((1080, 1920), ("u8", 8, False), "minmax"),
             ((1081, 1918), ("raw10", 10, False), "minmax"), ((2160, 3840), ("u16", 16, False), "minmax"),
             ((2160, 3840), ("u16", 12, True), None)]
    frames, rgbs = [], []
    for (h, w), container, agc in cases:
        bits = container[1]
        codes = rng.integers(0, 1 << bits, (h, w))
        if agc and h * w > 100:
            codes = codes % 900 + 17
        codes = codes.astype(_dt(bits))
        frames.append(make_frame(codes, container, agc, 4, 0, rng))
        rgbs.append(image_ops.mono_to_rgb(codes, bits, agc))
    records = [f.mono_record() for f in frames]
    bad = unreadable_records(records[0], records[1])
    table = mono_table(records + bad)
    F = len(records) + len(bad)
    run_range(lib, table, F)
    sums = torch.full((F, 3), -1, dtype=torch.int64, device="cuda")
    _lib.check(lib.fear_frame_sums_mono_u8(table.data_ptr(), F, sums.data_ptr(), stream()), "fear_frame_sums_mono_u8")
    got = sums.cpu().numpy().view(np.uint64)
    for i, rgb in enumerate(rgbs):
        assert np.array_equal(got[i], rgb.sum(axis=(0, 1), dtype=np.uint64)), (i, cases[i])
    assert (got[len(records):] == 0).all()


def test_c_abi_rejects_bad_arguments_and_launches_nothing():
    lib = _lib.init(0)
    t = torch.full((1 << 16,), 0x5A, dtype=torch.uint8, device="cuda")
    p = t.data_ptr()
    good = dict(views=p, F=1, targets=p, N=1, offset=2.0, size=256, crops=p)

    def crop(**kw):
        a = dict(good, **kw)
        return lib.fear_crop_targets_mono_u8(a["views"], a["F"], a["targets"], a["N"], a["offset"], a["size"],
                                             a["crops"], None)

    for kw in [dict(views=None), dict(targets=None), dict(crops=None), dict(N=0), dict(N=-1), dict(N=65536),
               dict(F=0), dict(F=-3), dict(size=0), dict(size=257), dict(offset=-0.5), dict(offset=float("nan")),
               dict(offset=float("inf"))]:
        assert crop(**kw) == -1, kw
        assert _lib.last_error(), kw
    for args in [(None, p, 1, p, 1, 256), (p, None, 1, p, 1, 256), (p, p, 1, None, 1, 256), (p, p, 1, p, 0, 256),
                 (p, p, 0, p, 1, 256), (p, p, 1, p, 1, 0)]:
        assert lib.fear_advance_targets_mono(*args, None) == -1, args
    for args in [(None, 1, p), (p, 1, None), (p, 0, p), (p, 65536, p), (p, -1, p)]:
        assert lib.fear_frame_sums_mono_u8(*args, None) == -1, args
    for args in [(None, 1), (p, 0), (p, -1), (p, 65536)]:
        assert lib.fear_frame_range_mono(*args, None) == -1, args
        assert _lib.last_error(), args
    torch.cuda.synchronize()
    assert (t == 0x5A).all()


# ---------------------------------------------------------------------------------------------------- MonoFrame
def _dev(h, w, dtype=torch.uint8):
    return torch.zeros((h, w), dtype=dtype, device="cuda")


def test_mono_frame_records_its_samples():
    surf = _dev(8, 2000, torch.uint16)
    f = fb.MonoFrame(surf[1:7, 3:1923], bits=12, msb=True, agc="minmax")
    assert f.shape == (6, 1920, 3) and f.pitch == 4000
    assert f.mono_record() == (surf.data_ptr() + 4006, 4000, 6, 1920, 12, 4, 0, 1, INT_MAX, INT_MIN)
    assert fb.MonoFrame(_dev(1, 1)).mono_record()[1:] == (1, 1, 1, 8, 0, 0, 0, INT_MAX, INT_MIN)
    raw = _dev(5, 3000)
    r10 = fb.MonoFrame.raw10(raw[1:4, 7:7 + 2400], 1920)
    assert r10.shape == (3, 1920, 3) and r10.mono_record()[:8] == (raw.data_ptr() + 3007, 3000, 3, 1920, 10, 0, 1, 0)
    r12 = fb.MonoFrame.raw12(raw[:, :3], 1, agc="minmax")
    assert r12.shape == (5, 1, 3) and r12.mono_record()[1:8] == (3000, 5, 1, 12, 0, 2, 1)


BAD_MONO = {
    "0 rows": lambda: fb.MonoFrame(_dev(0, 8)),
    "0 columns": lambda: fb.MonoFrame(_dev(8, 0)),
    "uint8 at 12 bits": lambda: fb.MonoFrame(_dev(8, 8), bits=12),
    "uint16 at 8 bits": lambda: fb.MonoFrame(_dev(8, 8, torch.uint16)),
    "int16 samples": lambda: fb.MonoFrame(_dev(8, 8, torch.int16), bits=12),
    "strided columns": lambda: fb.MonoFrame(_dev(8, 16)[:, ::2]),
    "rows overlap": lambda: fb.MonoFrame(_dev(8, 16).as_strided((8, 16), (8, 1))),
    "raw10 short row": lambda: fb.MonoFrame.raw10(_dev(8, 9), 8),
    "raw12 short row": lambda: fb.MonoFrame.raw12(_dev(8, 11), 7),
    "raw10 width 0": lambda: fb.MonoFrame.raw10(_dev(8, 10), 0),
    "raw10 width float": lambda: fb.MonoFrame.raw10(_dev(8, 10), 8.0),
    "raw10 uint16": lambda: fb.MonoFrame.raw10(_dev(8, 10, torch.uint16), 8),
    "unknown agc": lambda: fb.MonoFrame(_dev(8, 8), agc="MINMAX"),
    "misaligned uint16": lambda: fb.MonoFrame(_dev(8, 34)[:, 1:33].view(torch.uint16), bits=10),
}


@pytest.mark.parametrize("what", list(BAD_MONO))
def test_mono_frame_refuses_malformed_tensors(what):
    with pytest.raises((ValueError, RuntimeError)) as e:
        BAD_MONO[what]()
    if what != "misaligned uint16":  # torch itself may refuse that view
        assert e.type is ValueError


def test_tracker_refuses_mono_mixed_with_other_kinds(net):
    trk = fb.FEARMultiTracker(net, cuda_id=0, max_targets=4, **CFG)
    f = fb.MonoFrame(torch.zeros((64, 80), dtype=torch.uint8, device="cuda"), agc="minmax")
    rgb = torch.zeros((64, 80, 3), dtype=torch.uint8, device="cuda")
    nv12 = fb.YUV420Frame.nv12(torch.zeros((96, 80), dtype=torch.uint8, device="cuda"))
    bayer = fb.BayerFrame(torch.zeros((64, 80), dtype=torch.uint8, device="cuda"))
    for frames in ([f, np.zeros((64, 80, 3), np.uint8)], [rgb, f], [nv12, f]):
        with pytest.raises(ValueError, match="MonoFrames cannot share"):
            trk.add(frames, [[1, 1, 20, 20]])
    for frames in ([f, bayer], [bayer, rgb]):  # a call with a BayerFrame keeps the Bayer message
        with pytest.raises(ValueError, match="BayerFrames cannot share"):
            trk.add(frames, [[1, 1, 20, 20]])
    assert len(trk) == 0


# ---------------------------------------------------------------------------------------------------- trackers
def gray(rgb: np.ndarray) -> np.ndarray:
    return cv2.cvtColor(rgb, cv2.COLOR_RGB2GRAY)


def thermal(rgb: np.ndarray, rng) -> np.ndarray:
    """A thermal core's 16-bit codes: a narrow band 30000 + 8 * gray with seeded noise, from a half-size picture
    upscaled to 1080p with cv2 (a thermal sensor's resolution is low)."""
    g = cv2.resize(gray(rgb), (960, 540)).astype(np.float64)
    v = 30000 + 8 * g + rng.normal(0, 3, g.shape)
    return cv2.resize(np.clip(np.rint(v), 0, 65535).astype(np.uint16), (1920, 1080), interpolation=cv2.INTER_LINEAR)


# stream: container, agc, pitch extra; the codes of each are built from the demo clip by ``stream_codes``
MONO_STREAMS = [(("u8", 8, False), None, 128), (("u16", 12, True), None, 64), (("raw10", 10, False), None, 80),
                (("raw12", 12, False), None, 0), (("u16", 16, False), "minmax", 32)]


def stream_codes(rgb, s, rng):
    container = MONO_STREAMS[s][0]
    if MONO_STREAMS[s][1]:
        return thermal(rgb, rng)
    g = gray(cv2.resize(rgb, (1920, 1080))).astype(np.int64)
    bits = container[1]
    return ((g * ((1 << bits) - 1) + 127) // 255).astype(_dt(bits))


def mono_clip(clip, T, rng):
    codes = [[stream_codes(clip[t], s, rng) for t in range(T + 1)] for s in range(len(MONO_STREAMS))]
    rgb = [[image_ops.mono_to_rgb(c, MONO_STREAMS[s][0][1], MONO_STREAMS[s][1]) for c in codes[s]]
           for s in range(len(MONO_STREAMS))]
    return codes, rgb


def mono_frames(codes, t, rng, streams=None):
    streams = range(len(MONO_STREAMS)) if streams is None else streams
    return [make_frame(codes[s][t], MONO_STREAMS[s][0], MONO_STREAMS[s][1], MONO_STREAMS[s][2], s, rng)
            for s in streams]


def test_multi_tracker_on_mono_matches_numpy_rgb(net, clip):
    """Five 1080p mono streams (pitched Mono8, 12-bit MSB, RAW10, RAW12, thermal Y16 with AGC), several targets, with
    add / remove part way, a call on numpy frames in between, and calls without the thermal stream (no AGC).  Every
    output equals a tracker fed the grey frames as numpy arrays; steady calls replay one graph per AGC setting, and the
    graph is captured again after the net's workspace grows.  A step is 49 launches with AGC, 48 without."""
    T = 32
    rng = np.random.default_rng(97)
    codes, rgb = mono_clip(clip, T, rng)
    n2 = fb.FEARNet(**fb.FEAR_XS_MODEL_KWARGS)
    n2.load_state_dict(load_full_state(), strict=True)
    n2 = n2.cuda().eval()
    ref = fb.FEARMultiTracker(n2, cuda_id=0, max_targets=12, **CFG)
    trk = fb.FEARMultiTracker(n2, cuda_id=0, max_targets=12, **CFG)
    start = [[[652, 211, 180, 696]], [[900, 400, 120, 300]], [[0, 0, 60, 60]], [[1700, 840, 160, 224]],
             [[600, 200, 200, 600], [1800, 1000, 120, 80]]]
    late = [[[400, 600, 120, 120]], [], [[100, 150, 30, 30]], [], []]

    def rects(d):
        return [r for s in d for r in s], [k for k, s in enumerate(d) for _ in s]

    r, s = rects(start)
    assert np.array_equal(trk.add(mono_frames(codes, 0, rng), r, s), ref.add([x[0] for x in rgb], r, s))
    graphs = []
    for t in range(1, T + 1):
        if t == 12:
            r, s = rects(late)
            assert np.array_equal(trk.add(mono_frames(codes, t - 1, rng), r, s), ref.add([x[t - 1] for x in rgb], r, s))
        if t == 22:
            for x in (ref, trk):
                x.remove([1, 2])
        if t == 27:
            gen = n2.generation()
            zt, xt, _, _ = fo.synthetic_crops(16)
            n2.track(xt.cuda(), n2.get_features(zt.cuda()))  # batch 16 > reserved 12: the workspace grows
            assert n2.generation() != gen
        if t == 8:  # numpy frames in between: their own table, then back to the mono graph
            expect, out = ref.update([x[t] for x in rgb]), trk.update([x[t] for x in rgb])
            assert trk._graph_key[2] == "views"
        else:
            expect = ref.update([x[t] for x in rgb])
            out = trk.update(mono_frames(codes, t, rng))
            assert trk._graph_key[2] == "mono" and trk._graph_key[4] is True
        assert np.array_equal(out["ids"], expect["ids"]), t
        assert np.array_equal(out["bbox"], expect["bbox"]), (t, out["bbox"], expect["bbox"])
        assert np.array_equal(out["score"], expect["score"]), t
        if t in (3, 10, 14, 24, 28):  # two updates after the start, the switch back, add, remove, growth
            assert trk._graph is not None and all(trk._graph is not g for g in graphs), t
            graphs.append(trk._graph)
        if t in (7, 11, 21, 26, T):  # replayed with new frame addresses every update
            assert trk._graph is graphs[-1], t
    # without the thermal stream: no AGC, another graph key (streams 0..3 only track targets of streams 0..3)
    only = fb.FEARMultiTracker(n2, cuda_id=0, max_targets=12, **CFG)
    oref = fb.FEARMultiTracker(n2, cuda_id=0, max_targets=12, **CFG)
    r, s = rects(start[:4])
    only.add(mono_frames(codes, 0, rng, range(4)), r, s)
    oref.add([x[0] for x in rgb[:4]], r, s)
    for t in range(1, 6):
        out, expect = only.update(mono_frames(codes, t, rng, range(4))), oref.update([x[t] for x in rgb[:4]])
        assert np.array_equal(out["bbox"], expect["bbox"]) and np.array_equal(out["score"], expect["score"]), t
        assert only._graph_key[2] == "mono" and only._graph_key[4] is False
    # the step's launches: the range kernel (with AGC), the crop and advance entry points around the network's own
    for streams, launches in ((range(5), 49), (range(4), 48)):
        eager = fb.FEARMultiTracker(n2, cuda_id=0, max_targets=12, cuda_graph=False, **CFG)
        eager.add(mono_frames(codes, 0, rng, streams), [[600, 200, 200, 300]] * len(streams), list(range(len(streams))))
        eager.update(mono_frames(codes, 1, rng, streams))
        torch.cuda.synchronize()
        c0 = n2.launch_count()
        eager.update(mono_frames(codes, 2, rng, streams))
        extra = 3 if launches == 49 else 2
        assert n2.launch_count() - c0 + extra == launches


@pytest.mark.parametrize("smooth", [False, True], ids=["plain", "smooth"])
def test_fear_tracker_on_mono_matches_numpy_rgb(net, clip, smooth):
    """FEARTracker on the thermal stream with AGC (graphed, and eager), with 12-bit MSB, RAW12 and a numpy frame part
    way, gives the trajectory and tracking_state of the same tracker on the grey frames as numpy arrays."""
    T = 25
    rng = np.random.default_rng(61)
    codes, rgb = mono_clip(clip, T, rng)
    init = np.array([600, 200, 200, 600])
    for extra in ({}, {"cuda_graph": False}):
        cfg = dict(CFG, smooth=smooth, **extra)
        ref, trk = fb.FEARTracker(net, cuda_id=0, **cfg), fb.FEARTracker(net, cuda_id=0, **cfg)
        ref.initialize(rgb[4][0], init)
        trk.initialize(mono_frames(codes, 0, rng, [4])[0], init)
        assert np.array_equal(trk.tracking_state.mean_color, ref.tracking_state.mean_color)
        for t in range(1, T + 1):
            s = 4 if t < 10 else (1 if t < 15 else (3 if t < 19 else 4))
            want = ref.update(rgb[s][t])["bbox"]
            frame = rgb[s][t] if t == 20 else mono_frames(codes, t, rng, [s])[0]
            got = trk.update(frame)["bbox"]
            assert np.array_equal(got, want), (smooth, extra, t, got, want)
            for key in ("bbox", "mapping", "prev_size"):
                assert np.array_equal(getattr(trk.tracking_state, key), getattr(ref.tracking_state, key)), (key, t)
        assert [list(p) for p in trk.tracking_state.paths] == [list(p) for p in ref.tracking_state.paths]
        for s in (4, 0):
            z_ref = ref.get_template_features(rgb[s][3], [600, 200, 100, 300])
            z_trk = trk.get_template_features(mono_frames(codes, 3, rng, [s])[0], [600, 200, 100, 300])
            assert torch.equal(z_ref, z_trk), s


# ---------------------------------------------------------------------------------------------------- poison
def test_mono_entry_points_and_trackers_on_poisoned_memory():
    """tests/poison_mono_check.py in its own process: guarded, poisoned tables, crops, sums, ranges, boxes and frames."""
    proc = subprocess.run([sys.executable, os.path.join(HERE, "poison_mono_check.py")], capture_output=True, text=True,
                          timeout=1200)
    lines = [l for l in proc.stdout.splitlines() if l.startswith("POISON_CHECK ")]
    assert proc.returncode == 0 and lines, f"poison_mono_check failed: {proc.stderr[-3000:]}"
    res = json.loads(lines[-1][len("POISON_CHECK "):])
    assert res["checked_calls"] > 0
    assert res["n_failures"] == 0, res["failures"]
