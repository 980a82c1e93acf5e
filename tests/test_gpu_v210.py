"""GPU tests of v210 frames: the FearFrameYCbCrV210 entry points (fear_crop_targets_ycbcr_v210_u8,
fear_advance_targets_ycbcr_v210, fear_frame_sums_ycbcr_v210_u8), V210Frame, and FEARMultiTracker / FEARTracker fed
v210 surfaces.

Every comparison is exact, against image_ops.yuv_to_rgb of image_ops.v210_unpack's planes (both pinned on the CPU by
tests/test_v210_cpu.py and tests/test_yuv_subsampling_cpu.py): crops against cv2 on the unpacked and converted frame,
boxes against the host rescale + clamp, sums against numpy, and every tracker output against the same tracker fed the
converted frames as numpy arrays.  The v210 words carry noise in bits 30-31 and the bytes past each row's groups hold
0xA5, so a reader that does not mask or that strays past the row is caught."""
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
from tests.test_yuv_subsampling_cpu import ycbcr_frame

pytestmark = pytest.mark.gpu
CFG = fb.FEAR_XS_TRACKER_KWARGS
HERE = os.path.dirname(os.path.abspath(__file__))
MATRIX_RANGES = [(m, f) for m in ("bt601", "bt709", "bt2020") for f in (False, True)]


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


def pitch_of(kind: str, w: int) -> int:
    """The row pitches a v210 surface may have: exactly 16 * ceil(W / 6) ("tight"), the capture cards' 128 * ceil(W /
    48) ("card"), that plus 256 ("wide"), or the tight pitch plus 4, a multiple of 4 but not of 16 ("odd4")."""
    return {"tight": image_ops.v210_row_bytes(w), "card": image_ops.v210_pitch(w),
            "wide": image_ops.v210_pitch(w) + 256, "odd4": image_ops.v210_row_bytes(w) + 4}[kind]


def v210_rows(y, u, v, pitch: int, rng) -> np.ndarray:
    """The (H, pitch) bytes of code planes packed to v210, with random bits 30-31 in every word and 0xA5 in the bytes
    past the last group of each row."""
    rows = image_ops.v210_pack(np.asarray(y), np.asarray(u), np.asarray(v), pitch)
    need = image_ops.v210_row_bytes(np.shape(y)[1])
    words = np.ascontiguousarray(rows[:, :need]).view("<u4")
    words |= (rng.integers(0, 4, words.shape) << 30).astype(np.uint32)
    rows[:, :need] = words.view(np.uint8)
    rows[:, need:] = 0xA5
    return rows


def v210_surface(rows: np.ndarray, w: int, col: int = 0, **fmt) -> fb.V210Frame:
    """``rows`` at row 1, byte column ``col`` (a multiple of 4) of a 0xA5-filled device surface, as a V210Frame of the
    view that holds each row's groups: the frame's pitch is the surface's."""
    h, pitch = rows.shape
    surf = np.full((h + 2, pitch + col), 0xA5, np.uint8)
    surf[1:h + 1, col:col + pitch] = rows
    return fb.V210Frame(torch.from_numpy(surf).cuda()[1:h + 1, col:col + image_ops.v210_row_bytes(w)], w, **fmt)


def oracle(rows: np.ndarray, w: int, matrix="bt601", full_range=False) -> np.ndarray:
    """The RGB frame the tracker sees for v210 bytes: yuv_to_rgb of their unpacked planes at 10 bits, 4:2:2."""
    return image_ops.yuv_to_rgb(*image_ops.v210_unpack(rows, w), matrix, full_range, 10, 0, (1, 0))


def random_planes(rng, h, w):
    return rng.integers(0, 1024, (h, w)), rng.integers(0, 1024, (h, w // 2)), rng.integers(0, 1024, (h, w // 2))


def v210_table(records) -> torch.Tensor:
    return torch.from_numpy(np.array(records, dtype=_lib.YCBCR_V210_DTYPE).view(np.uint8).copy()).cuda()


def unreadable_records(rec):
    """Entries the kernels must treat as empty, from a valid v210 record (W >= 6): a null or misaligned address, a pitch
    not a multiple of 4 or one below 16 * ceil(W / 6), an odd W, W = 0, H = 0, bits 8 or 12, shifts other than (1, 0),
    an unknown matrix, full_range 2, and a v210 value other than 0 and 1."""
    rec = list(rec)
    w = rec[8]
    edits = [(0, 0), (0, rec[0] + 2), (3, rec[3] + 2), (3, image_ops.v210_row_bytes(w) - 4), (8, w - 1), (8, 0),
             (7, 0), (11, 8), (11, 12), (13, 0), (14, 1), (9, 3), (9, -1), (10, 2), (15, 2), (15, -1)]
    out = []
    for field, value in edits:
        r = list(rec)
        r[field] = value
        out.append(tuple(r))
    return out


# ---------------------------------------------------------------------------------------------------- kernels
SHAPES = [(255, 480, "card", 0), (183, 98, "tight", 4), (91, 334, "wide", 0), (1, 4, "odd4", 0), (64, 1282, "tight", 8)]
TARGETS = [(0, [163, 53, 45, 174]), (0, [-10, 100, 40, 30]), (0, [450, 20, 60, 40]), (0, [200, -15, 30, 50]),
           (0, [0, 0, 3, 3]), (0, [476, 252, 3, 3]), (0, [-50, 30, 600, 100]), (2, [-300, -200, 900, 500]),
           (2, [330, 87, 3, 3]), (2, [5, 40, 320, 20]), (3, [0, 0, 3, 3]), (3, [-20, -20, 40, 40]),
           (4, [1270, 30, 40, 40]), (4, [600, 10, 300, 50]), (0, [2000, 900, 30, 30])]


def kernel_frames(rng, matrix, full):
    """SHAPES as v210 surfaces: W % 6 = 0, 2, 4, 4, 4 (partial last groups), odd H, every pitch kind, addresses at byte
    4 and 8 of a row."""
    rows = [v210_rows(*random_planes(rng, h, w), pitch_of(kind, w), rng) for h, w, kind, _ in SHAPES]
    frames = [v210_surface(r, w, col, matrix=matrix, full_range=full) for r, (_, w, _, col) in zip(rows, SHAPES)]
    rgbs = [oracle(r, w, matrix, full) for r, (_, w, _, _) in zip(rows, SHAPES)]
    return frames, rgbs


@pytest.mark.parametrize("fmt", MATRIX_RANGES, ids=lambda f: f"{f[0]}-{'full' if f[1] else 'limited'}")
def test_crop_v210_kernel_matches_cv2_on_unpacked_frame(fmt):
    """Random codes over the whole 10-bit range (outside the nominal range too); targets inside, across every border,
    tiny, huge and outside the frame; every unreadable entry and an out-of-range frame index give a padding-colour
    crop."""
    matrix, full = fmt
    lib = _lib.init(0)
    rng = np.random.default_rng(sum(map(ord, matrix)) + full)
    frames, rgbs = kernel_frames(rng, matrix, full)
    means = [np.mean(f, axis=(0, 1)) for f in rgbs]
    targets = list(TARGETS)
    for side in (1, 3, 9, 33, 120, 200):
        targets.append((1, [48 - side // 2, 90 - side // 2, side, side]))
    records = [f.ycbcr_v210_record() for f in frames]
    bad = unreadable_records(records[0])
    extra = [(9999, [12, 200, 255]), (-1, [1, 2, 3])] + [(len(records) + i, [i, 128, 7]) for i in range(len(bad))]
    recs = np.zeros((len(targets) + len(extra), _lib.TARGET_INTS), dtype=np.int32)
    for i, (f, box) in enumerate(targets):
        recs[i, 0], recs[i, 1:5] = f, box
        recs[i, 9:12] = np.clip(np.rint(means[f]), 0, 255)
    for i, (f, pad) in enumerate(extra):
        recs[len(targets) + i, 0], recs[len(targets) + i, 1:5], recs[len(targets) + i, 9:12] = f, [10, 10, 20, 20], pad
    table = v210_table(records + bad)
    n = len(recs)
    for size, off in ((256, 2.0), (128, 0.2)):
        state = torch.from_numpy(recs).cuda()
        crops = torch.empty((n, size, size, 3), dtype=torch.uint8, device="cuda")
        _lib.check(lib.fear_crop_targets_ycbcr_v210_u8(table.data_ptr(), len(records) + len(bad), state.data_ptr(), n,
                                                       off, size, crops.data_ptr(), stream()),
                   "fear_crop_targets_ycbcr_v210_u8")
        got, ctxs = crops.cpu().numpy(), state.cpu().numpy()[:, 5:9]
        for i, (f, box) in enumerate(targets):
            assert np.array_equal(ctxs[i], image_ops.context_box(box, off)), (fmt, size, off, box)
            assert np.array_equal(got[i], base._cv2_crop(rgbs[f], box, size, off, means[f])), (fmt, size, off, f, box)
        for i, (_, pad) in enumerate(extra):
            assert (got[len(targets) + i] == np.array(pad, dtype=np.uint8)).all(), (fmt, i)


def test_identity_crop_reads_every_pixel_of_every_group_position():
    """A 256 x 1536 frame at offset 0, cropped 1:1 in six 256 x 256 tiles: every pixel, so every (x % 6) position and
    every code slot, equals the unpacked frame's RGB."""
    lib = _lib.init(0)
    rng = np.random.default_rng(2)
    h, w = 256, 1536
    rows = v210_rows(*random_planes(rng, h, w), pitch_of("card", w), rng)
    frame = v210_surface(rows, w, matrix="bt709")
    table = v210_table([frame.ycbcr_v210_record()])
    recs = np.zeros((6, _lib.TARGET_INTS), dtype=np.int32)
    recs[:, 1] = 256 * np.arange(6)
    recs[:, 3:5] = 256
    state = torch.from_numpy(recs).cuda()
    crops = torch.empty((6, 256, 256, 3), dtype=torch.uint8, device="cuda")
    _lib.check(lib.fear_crop_targets_ycbcr_v210_u8(table.data_ptr(), 1, state.data_ptr(), 6, 0.0, 256,
                                                   crops.data_ptr(), stream()), "fear_crop_targets_ycbcr_v210_u8")
    got = crops.cpu().numpy().transpose(1, 0, 2, 3).reshape(h, w, 3)
    assert np.array_equal(got, oracle(rows, w, "bt709"))


def test_v210_0_entries_equal_the_ycbcr_entry_points():
    """FearFrameYCbCr records followed by v210 = 0 give bit-identical crops, advances and sums through the v210 entry
    points and through the *_ycbcr ones."""
    lib = _lib.init(0)
    rng = np.random.default_rng(43)
    kinds = [((255, 480), "yuyv_pitched", 8, "bt601", False, 1), ((183, 98), "nv16", 10, "bt709", False, 1),
             ((90, 334), "i444_pitched", 8, "bt2020", True, 0), ((1080, 1920), "i422", 12, "bt709", True, 1),
             ((256, 480), "planes444", 10, "bt601", False, 0)]
    frames = []
    for (h, w), layout, b, m, f, sx in kinds:
        y, u, v = rng.integers(0, 1 << b, (h, w)), rng.integers(0, 1 << b, (h, w >> sx)), \
            rng.integers(0, 1 << b, (h, w >> sx))
        frames.append(ycbcr_frame(y, u, v, layout, b, rng=rng, matrix=m, full_range=f))
    old = torch.from_numpy(np.array([f.ycbcr_record() for f in frames], dtype=_lib.YCBCR_DTYPE)
                           .view(np.uint8).copy()).cuda()
    new = v210_table([f.ycbcr_v210_record() for f in frames])
    F, n = len(frames), 1000
    recs = np.zeros((n, _lib.TARGET_INTS), dtype=np.int32)
    recs[:, 0] = rng.integers(-1, F + 1, n)
    recs[:, 1:3] = rng.integers(-300, 1900, (n, 2))
    recs[:, 3:5] = rng.integers(1, 600, (n, 2))
    recs[:, 9:12] = rng.integers(0, 256, (n, 3))
    boxes = np.zeros(n, dtype=_lib.BOX_DTYPE)
    for k in ("x", "y"):
        boxes[k] = rng.uniform(-50, 300, n)
    for k in ("w", "h"):
        boxes[k] = rng.uniform(0, 300, n)
    dboxes = torch.from_numpy(boxes.view(np.uint8).copy()).cuda()
    out = {}
    for name, table, crop, adv, sums in (
            ("ycbcr", old, lib.fear_crop_targets_ycbcr_u8, lib.fear_advance_targets_ycbcr,
             lib.fear_frame_sums_ycbcr_u8),
            ("v210", new, lib.fear_crop_targets_ycbcr_v210_u8, lib.fear_advance_targets_ycbcr_v210,
             lib.fear_frame_sums_ycbcr_v210_u8)):
        state = torch.from_numpy(recs).cuda()
        crops = torch.empty((n, 256, 256, 3), dtype=torch.uint8, device="cuda")
        s = torch.empty((F, 3), dtype=torch.int64, device="cuda")
        _lib.check(crop(table.data_ptr(), F, state.data_ptr(), n, 2.0, 256, crops.data_ptr(), stream()), name)
        _lib.check(adv(dboxes.data_ptr(), table.data_ptr(), F, state.data_ptr(), n, 256, stream()), name)
        _lib.check(sums(table.data_ptr(), F, s.data_ptr(), stream()), name)
        out[name] = (crops.cpu().numpy(), state.cpu().numpy(), s.cpu().numpy())
    for a, b in zip(out["ycbcr"], out["v210"]):
        assert np.array_equal(a, b)


def test_advance_v210_kernel_matches_host_rescale_and_clamp():
    """12 000 records on v210 frames of three sizes; unreadable entries and out-of-range frame indices keep their
    boxes."""
    lib = _lib.init(0)
    rng = np.random.default_rng(5)
    shapes = [(255, 480), (183, 98), (1, 2)]
    n = 12000
    boxes = np.zeros(n, dtype=_lib.BOX_DTYPE)
    recs = np.zeros((n, _lib.TARGET_INTS), dtype=np.int32)
    recs[:, 0] = rng.integers(0, 3, n)
    recs[:, 5:7] = rng.integers(-600, 700, (n, 2))
    recs[:, 7:9] = rng.integers(1, 2000, (n, 2))
    boxes["x"], boxes["y"] = rng.uniform(-300, 600, n), rng.uniform(-300, 600, n)
    boxes["w"], boxes["h"] = rng.uniform(0, 300, n), rng.uniform(0, 300, n)
    boxes["w"][:n // 4], boxes["h"][:n // 4] = rng.uniform(0, 3, n // 4), rng.uniform(0, 3, n // 4)
    frames = [v210_surface(v210_rows(*random_planes(rng, h, w), pitch_of("card", w), rng), w) for h, w in shapes]
    records = [f.ycbcr_v210_record() for f in frames]
    bad = unreadable_records(records[0])
    table = v210_table(records + bad)
    recs[-len(bad) - 4:-len(bad), 0] = 999
    recs[-len(bad):, 0] = 3 + np.arange(len(bad))
    kept = len(bad) + 4
    recs[-kept:, 1:5] = [7, 8, 9, 10]
    state = torch.from_numpy(recs).cuda()
    dboxes = torch.from_numpy(boxes.view(np.uint8).copy()).cuda()
    _lib.check(lib.fear_advance_targets_ycbcr_v210(dboxes.data_ptr(), table.data_ptr(), 3 + len(bad),
                                                   state.data_ptr(), n, 256, stream()),
               "fear_advance_targets_ycbcr_v210")
    got = state.cpu().numpy()
    for i in range(n - kept):
        b = np.array([boxes["x"][i], boxes["y"][i], boxes["w"][i], boxes["h"][i]])
        h, w = shapes[recs[i, 0]]
        want = image_ops.clamp_bbox(image_ops.rescale_bbox(b, recs[i, 5:9], 256), (h, w, 3))
        assert np.array_equal(got[i, 1:5], want), (i, b.tolist(), recs[i, 5:9].tolist(), (h, w), got[i, 1:5], want)
    assert (got[-kept:, 1:5] == [7, 8, 9, 10]).all()
    assert np.array_equal(np.delete(got, np.s_[1:5], axis=1), np.delete(recs, np.s_[1:5], axis=1))


def test_frame_sums_v210_give_numpy_sums_of_unpacked_frame():
    lib = _lib.init(0)
    rng = np.random.default_rng(11)
    cases = [((1, 2), "tight", "bt601", False), ((3, 4), "odd4", "bt709", True), ((183, 98), "card", "bt2020", True),
             ((37, 1004), "wide", "bt601", True), ((1080, 1920), "card", "bt709", False),
             ((1081, 1918), "tight", "bt2020", False), ((2160, 3840), "card", "bt709", True)]
    rows = [v210_rows(*random_planes(rng, h, w), pitch_of(kind, w), rng) for (h, w), kind, _, _ in cases]
    frames = [v210_surface(r, w, matrix=m, full_range=f) for r, ((_, w), _, m, f) in zip(rows, cases)]
    records = [f.ycbcr_v210_record() for f in frames]
    bad = unreadable_records(records[2])
    table = v210_table(records + bad)
    F = len(records) + len(bad)
    sums = torch.full((F, 3), -1, dtype=torch.int64, device="cuda")  # zeroed by the call
    _lib.check(lib.fear_frame_sums_ycbcr_v210_u8(table.data_ptr(), F, sums.data_ptr(), stream()),
               "fear_frame_sums_ycbcr_v210_u8")
    got = sums.cpu().numpy().view(np.uint64)
    for i, (r, ((_, w), _, m, f)) in enumerate(zip(rows, cases)):
        assert np.array_equal(got[i], oracle(r, w, m, f).sum(axis=(0, 1), dtype=np.uint64)), (i, cases[i])
    assert (got[len(records):] == 0).all()


def test_c_abi_rejects_bad_arguments_and_launches_nothing():
    lib = _lib.init(0)
    t = torch.full((1 << 16,), 0x5A, dtype=torch.uint8, device="cuda")
    p = t.data_ptr()
    good = dict(views=p, F=1, targets=p, N=1, offset=2.0, size=256, crops=p)

    def crop(**kw):
        a = dict(good, **kw)
        return lib.fear_crop_targets_ycbcr_v210_u8(a["views"], a["F"], a["targets"], a["N"], a["offset"], a["size"],
                                                   a["crops"], None)

    bad = [dict(views=None), dict(targets=None), dict(crops=None), dict(N=0), dict(N=-1), dict(N=65536), dict(F=0),
           dict(F=-3), dict(size=0), dict(size=257), dict(offset=-0.5), dict(offset=float("nan")),
           dict(offset=float("inf"))]
    for kw in bad:
        assert crop(**kw) == -1, kw
        assert _lib.last_error(), kw
    for args in [(None, p, 1, p, 1, 256), (p, None, 1, p, 1, 256), (p, p, 1, None, 1, 256), (p, p, 1, p, 0, 256),
                 (p, p, 0, p, 1, 256), (p, p, 1, p, 1, 0)]:
        assert lib.fear_advance_targets_ycbcr_v210(*args, None) == -1, args
        assert _lib.last_error(), args
    for args in [(None, 1, p), (p, 1, None), (p, 0, p), (p, 65536, p), (p, -1, p)]:
        assert lib.fear_frame_sums_ycbcr_v210_u8(*args, None) == -1, args
        assert _lib.last_error(), args
    torch.cuda.synchronize()
    assert (t == 0x5A).all()  # no kernel and no memset ran


# ---------------------------------------------------------------------------------------------------- V210Frame
def _dev(h, w):
    return torch.zeros((h, w), dtype=torch.uint8, device="cuda")


def test_v210_frame_records_its_surface():
    surf = _dev(6, 5120 + 128)
    f = fb.V210Frame(surf[1:5, 64:64 + 5120], 1920, matrix="bt2020", full_range=True)
    assert f.shape == (4, 1920, 3) and f.pitch == 5248
    rec = np.array([f.ycbcr_v210_record()], dtype=_lib.YCBCR_V210_DTYPE)[0]
    assert rec["y"] == surf.data_ptr() + 5248 + 64 and rec["y_row_stride"] == 5248
    assert (rec["H"], rec["W"], rec["matrix"], rec["full_range"], rec["bits"], rec["shift"]) == (4, 1920, 2, 1, 10, 0)
    assert (rec["chroma_shift_x"], rec["chroma_shift_y"], rec["v210"], rec["reserved"]) == (1, 0, 1, 0)
    one = fb.V210Frame(_dev(8, 256)[3:4, :20], 6)  # one row: its pitch is never stepped
    assert one.shape == (1, 6, 3) and one.pitch == 16


BAD_FRAMES = {
    "odd width": lambda: fb.V210Frame(_dev(4, 128), 47),
    "width 0": lambda: fb.V210Frame(_dev(4, 128), 0),
    "width float": lambda: fb.V210Frame(_dev(4, 128), 48.0),
    "rows too short": lambda: fb.V210Frame(_dev(4, 128), 50),
    "no rows": lambda: fb.V210Frame(_dev(0, 128), 48),
    "pitch not a multiple of 4": lambda: fb.V210Frame(_dev(4, 130)[:, :128], 48),
    "misaligned address": lambda: fb.V210Frame(_dev(4, 256)[:, 2:130], 48),
    "strided bytes": lambda: fb.V210Frame(_dev(4, 256)[:, ::2], 48),
    "pitch below the row": lambda: fb.V210Frame(_dev(8, 64).view(4, 128)[:, :128].as_strided((4, 128), (64, 1)), 48),
    "int16 rows": lambda: fb.V210Frame(torch.zeros((4, 64), dtype=torch.int16, device="cuda"), 48),
}


@pytest.mark.parametrize("what", list(BAD_FRAMES))
def test_v210_frame_refuses_malformed_buffers(what):
    with pytest.raises(ValueError):
        BAD_FRAMES[what]()


def test_tracker_refuses_v210_mixed_with_rgb(net):
    trk = fb.FEARMultiTracker(net, cuda_id=0, max_targets=4, **CFG)
    f = fb.V210Frame(_dev(64, 256), 80)
    for frames in ([f, np.zeros((64, 80, 3), np.uint8)], [torch.zeros((64, 80, 3), dtype=torch.uint8,
                                                                      device="cuda"), f]):
        with pytest.raises(ValueError):
            trk.add(frames, [[1, 1, 20, 20]])
    assert len(trk) == 0


# ---------------------------------------------------------------------------------------------------- trackers
def clip_codes(clip, size, matrix, full, T, rng):
    """10-bit 4:2:2 code planes of the first T + 1 clip frames resized to ``size`` (W, H)."""
    out = []
    for t in range(T + 1):
        rgb = cv2.resize(clip[t], size) if size != clip.shape[2:0:-1] else clip[t]
        out.append(encode(rgb, matrix, full, 10, "422", rng))
    return out


V210_STREAMS = [((1920, 1080), "card", "bt709", False), ((478, 256), "tight", "bt601", True)]
OTHER_STREAMS = [((480, 256), "nv12", "bt601", False, 8), ((480, 256), "nv16", "bt709", False, 10),
                 ((480, 256), "i444_pitched", "bt2020", True, 8)]


def test_multi_tracker_on_v210_alone_and_mixed_matches_numpy_rgb(net, clip):
    """Two v210 streams (pitched 1080p BT.709 and a 478-wide full-range stream whose rows end in a partial group), alone
    and in one call with NV12, P210 and I444 streams, several targets each, add / remove part way.  Every output equals a
    tracker fed the unpacked and converted frames as numpy arrays; steady calls replay one captured graph of the
    ycbcr_v210 table, and a new target count captures a new one."""
    T = 30
    rng = np.random.default_rng(97)
    rows, rgb = [], []
    for size, kind, m, f in V210_STREAMS:
        codes = clip_codes(clip, size, m, f, T, rng)
        rows.append([v210_rows(*c, pitch_of(kind, size[0]), rng) for c in codes])
        rgb.append([oracle(r, size[0], m, f) for r in rows[-1]])
    planes = []
    for size, layout, m, f, b in OTHER_STREAMS:
        sub = "420" if layout == "nv12" else "444" if "444" in layout else "422"
        planes.append([encode(cv2.resize(clip[t], size), m, f, b, sub, rng) for t in range(T + 1)])
        rgb.append([image_ops.yuv_to_rgb(*p, m, f, b, 0, {"420": (1, 1), "422": (1, 0), "444": (0, 0)}[sub])
                    for p in planes[-1]])

    def v210(t):
        return [v210_surface(rows[s][t], size[0], col=4 * s, matrix=m, full_range=f)
                for s, (size, _, m, f) in enumerate(V210_STREAMS)]

    def others(t):
        out = []
        for s, (_, layout, m, f, b) in enumerate(OTHER_STREAMS):
            if layout == "nv12":
                out.append(code_frame(*planes[s][t], layout, m, f, b, rng))
            else:
                out.append(ycbcr_frame(*planes[s][t], layout, b, rng=rng, matrix=m, full_range=f))
        return out

    start = [[[652, 211, 180, 696], [1700, 840, 160, 224]], [base.GOLDEN_BOX, [-10, 100, 50, 50]],
             [[300, 80, 60, 90]], [base.GOLDEN_BOX], [[168, 50, 40, 170]]]
    late = [[[400, 600, 120, 120]], [[100, 150, 30, 30]], [], [[0, 0, 40, 60]], []]

    def rects(d):
        return [r for s in d for r in s], [k for k, s in enumerate(d) for _ in s]

    runs = {"only": (lambda t: v210(t), 2), "mixed": (lambda t: v210(t) + others(t), 5)}
    for name, (frames, ns) in runs.items():
        ref = fb.FEARMultiTracker(net, cuda_id=0, max_targets=12, **CFG)
        trk = fb.FEARMultiTracker(net, cuda_id=0, max_targets=12, **CFG)
        r, s = rects(start[:ns])
        assert np.array_equal(trk.add(frames(0), r, s), ref.add([rgb[k][0] for k in range(ns)], r, s))
        graphs = []
        for t in range(1, T + 1):
            if t == 12:
                r, s = rects(late[:ns])
                assert np.array_equal(trk.add(frames(t - 1), r, s), ref.add([rgb[k][t - 1] for k in range(ns)], r, s))
            if t == 22:
                for x in (ref, trk):
                    x.remove([1, 2])
            expect = ref.update([rgb[k][t] for k in range(ns)])
            out = trk.update(frames(t))
            assert np.array_equal(out["ids"], expect["ids"]), (name, t)
            assert np.array_equal(out["bbox"], expect["bbox"]), (name, t, out["bbox"], expect["bbox"])
            assert np.array_equal(out["score"], expect["score"]), (name, t)
            assert trk._graph_key[2] == "ycbcr_v210"
            if t in (3, 14, 24):  # two updates after the start, the add and the remove: captured
                assert trk._graph is not None and all(trk._graph is not g for g in graphs)
                graphs.append(trk._graph)
            if t in (11, 21, T):
                assert trk._graph is graphs[-1]  # replayed with new surface addresses every update


def test_calls_without_v210_keep_their_tables(net, clip):
    rng = np.random.default_rng(4)
    rgb = cv2.resize(clip[0], (480, 256))
    c420, c422 = encode(rgb, "bt601", False, 8, "420", rng), encode(rgb, "bt601", False, 10, "422", rng)
    trk = fb.FEARMultiTracker(net, cuda_id=0, max_targets=4, cuda_graph=False, **CFG)
    nv12 = code_frame(*c420, "nv12", "bt601", False, 8, rng)
    v210 = v210_surface(v210_rows(*c422, pitch_of("card", 480), rng), 480)
    trk.add([nv12, v210], [base.GOLDEN_BOX, [10, 10, 40, 40]], [0, 1])
    for frames, table in (([nv12, nv12], "yuv"), ([nv12, v210], "ycbcr_v210"),
                          ([ycbcr_frame(*c422, "nv16", 10), nv12], "ycbcr"), ([v210, v210], "ycbcr_v210"),
                          ([nv12, nv12], "yuv")):
        trk.update(frames)
        assert trk._graph_key[2] == table


@pytest.mark.parametrize("smooth", [False, True], ids=["plain", "smooth"])
def test_fear_tracker_on_v210_matches_numpy_rgb(net, clip, smooth):
    """FEARTracker on pitched v210 surfaces (graphed, and eager) gives the trajectory and tracking_state of the same
    tracker on the unpacked, converted frames as numpy arrays."""
    T = 25
    rng = np.random.default_rng(61)
    rows = [v210_rows(*c, pitch_of("card", 480), rng) for c in clip_codes(clip, (480, 256), "bt709", False, T, rng)]
    rgb = [oracle(r, 480, "bt709") for r in rows]
    init = np.array(base.GOLDEN_BOX)
    for extra in ({}, {"cuda_graph": False}):
        cfg = dict(CFG, smooth=smooth, **extra)
        ref, trk = fb.FEARTracker(net, cuda_id=0, **cfg), fb.FEARTracker(net, cuda_id=0, **cfg)
        ref.initialize(rgb[0], init)
        trk.initialize(v210_surface(rows[0], 480, matrix="bt709"), init)
        assert np.array_equal(trk.tracking_state.mean_color, ref.tracking_state.mean_color)
        for t in range(1, T + 1):
            want = ref.update(rgb[t])["bbox"]
            got = trk.update(v210_surface(rows[t], 480, col=4 * (t % 3), matrix="bt709"))["bbox"]
            assert np.array_equal(got, want), (smooth, extra, t, got, want)
            for key in ("bbox", "mapping", "prev_size"):
                assert np.array_equal(getattr(trk.tracking_state, key), getattr(ref.tracking_state, key)), (key, t)
        assert [list(p) for p in trk.tracking_state.paths] == [list(p) for p in ref.tracking_state.paths]


# ---------------------------------------------------------------------------------------------------- poison
def test_v210_entry_points_and_trackers_on_poisoned_memory():
    """tests/poison_v210_check.py in its own process: guarded, poisoned tables, crops, sums, boxes and surfaces."""
    proc = subprocess.run([sys.executable, os.path.join(HERE, "poison_v210_check.py")], capture_output=True, text=True,
                          timeout=1200)
    lines = [l for l in proc.stdout.splitlines() if l.startswith("POISON_CHECK ")]
    assert proc.returncode == 0 and lines, f"poison_v210_check failed: {proc.stderr[-3000:]}"
    res = json.loads(lines[-1][len("POISON_CHECK "):])
    assert res["checked_calls"] > 0
    assert res["n_failures"] == 0, res["failures"]
