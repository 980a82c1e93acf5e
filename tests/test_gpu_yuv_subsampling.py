"""GPU tests of YUV 4:2:2 and 4:4:4 frames: the FearFrameYCbCr entry points (fear_crop_targets_ycbcr_u8,
fear_advance_targets_ycbcr, fear_frame_sums_ycbcr_u8) and FEARMultiTracker fed YUV422Frames and YUV444Frames.

Every comparison is exact, against image_ops.yuv_to_rgb (pinned to cv2 and to yuv420_to_rgb by
tests/test_yuv_subsampling_cpu.py) or cv2 itself: identity-resample crops against the converted frames, crops against
cv2 on the converted frame, boxes against the host rescale + clamp, sums against numpy, and every tracker output
against the same tracker fed the converted frames as numpy arrays."""
import os

import cv2
import numpy as np
import pytest
import torch

import feartracker_b200 as fb
from feartracker_b200 import _lib, image_ops
from oracle import fear_oracle as fo
from tests import test_gpu_multi_tracker as base
from tests.helpers import GOLDEN, load_full_state
from tests.test_gpu_yuv_formats import code_frame, invalid_records, pair_frames, random_frames
from tests.test_yuv_subsampling_cpu import CV2_PACKED, PACKED, ycbcr_frame

pytestmark = pytest.mark.gpu
CFG = fb.FEAR_XS_TRACKER_KWARGS
SHIFTS = {"422": (1, 0), "444": (0, 0), "420": (1, 1)}


@pytest.fixture(scope="module")
def net():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    n = fb.FEARNet(**fb.FEAR_XS_MODEL_KWARGS)
    n.load_state_dict(load_full_state(), strict=True)
    return n.cuda().eval()


@pytest.fixture(scope="module")
def clip():
    return fo.read_video_rgb(os.path.join(GOLDEN, "test.mp4"))


def ycbcr_table(records) -> torch.Tensor:
    return torch.from_numpy(np.array(records, dtype=_lib.YCBCR_DTYPE).view(np.uint8).copy()).cuda()


def stream():
    return torch.cuda.current_stream().cuda_stream


def oracle(y, u, v, sub, matrix="bt601", full_range=False, bits=8) -> np.ndarray:
    return image_ops.yuv_to_rgb(y, u, v, matrix, full_range, bits, 0, SHIFTS[sub])


def sub_of(layout: str) -> str:
    return "444" if "444" in layout else "422"


def chroma_of(u, sub):
    """4:2:0 chroma planes (H/2, W/2) as the chroma of a 4:2:2 (rows repeated) or 4:4:4 (nearest upsampled) frame."""
    u = np.asarray(u).repeat(2, 0)
    return u if sub == "422" else u.repeat(2, 1)


def unreadable_records(rec):
    """Entries the kernels must treat as empty, from a valid FearFrameYCbCr record: FearFrameYUV's refusals, each shift
    pair outside (1, 1), (1, 0), (0, 0), and an odd W at chroma_shift_x 1 or an odd H at chroma_shift_y 1."""
    rec = tuple(rec)
    out = [r + rec[13:] for r in invalid_records(rec[:13])]
    out += [rec[:13] + s for s in ((0, 1), (2, 1), (1, 2), (-1, 0), (0, -1), (2, 0))]
    out.append(rec[:8] + (rec[8] | 1,) + rec[9:13] + (1, 0))  # odd W at 4:2:2
    out.append(rec[:7] + (rec[7] | 1,) + rec[8:13] + (1, 1))  # odd H at 4:2:0
    return out


# ---------------------------------------------------------------------------------------------------- conversion
def identity_crops(frames) -> np.ndarray:
    """The four 256 x 256 quadrants of every 512 x 512 frame cropped at offset 0 to 256 x 256 (an identity resample),
    through the ycbcr table, reassembled: (K, 512, 512, 3), the RGB frames the kernels see."""
    lib = _lib.init(0)
    quads = [(0, 0), (256, 0), (0, 256), (256, 256)]
    k = len(frames)
    recs = np.zeros((4 * k, _lib.TARGET_INTS), dtype=np.int32)
    for i in range(k):
        for q, (x, y) in enumerate(quads):
            recs[4 * i + q, 0], recs[4 * i + q, 1:5] = i, [x, y, 256, 256]
    state = torch.from_numpy(recs).cuda()
    crops = torch.empty((4 * k, 256, 256, 3), dtype=torch.uint8, device="cuda")
    table = ycbcr_table([f.ycbcr_record() for f in frames])
    _lib.check(lib.fear_crop_targets_ycbcr_u8(table.data_ptr(), k, state.data_ptr(), 4 * k, 0.0, 256,
                                              crops.data_ptr(), stream()), "fear_crop_targets_ycbcr_u8")
    got = crops.cpu().numpy().reshape(k, 2, 2, 256, 256, 3)
    return got.transpose(0, 1, 3, 2, 4, 5).reshape(k, 512, 512, 3)


def test_packed_422_crops_are_cv2_on_every_8_bit_triple():
    """64 frames of 512 x 512: chroma sample (i, j) is (U, V) = (i mod 256, j) and its two luma samples in frame k are
    4k + 2 (i // 256) and that + 1, so every (Y, U, V) triple occurs.  YUYV, UYVY and YVYU crops equal
    cv2.cvtColor(COLOR_YUV2RGB_YUY2 / UYVY / YVYU) of the same bytes."""
    i, j = np.meshgrid(np.arange(512), np.arange(256), indexing="ij")
    u, v = (i % 256).astype(np.uint8), j.astype(np.uint8)
    for k0 in range(0, 64, 16):
        ys = []
        for k in range(k0, k0 + 16):
            y = np.empty((512, 512), np.uint8)
            y[:, 0::2], y[:, 1::2] = 4 * k + 2 * (i // 256), 4 * k + 2 * (i // 256) + 1
            ys.append(y)
        for layout, code in CV2_PACKED.items():
            got = identity_crops([ycbcr_frame(y, u, v, layout if k % 2 else layout + "_pitched")
                                  for k, y in enumerate(ys)])
            (yo, ysx), (uo, us), (vo, vs) = PACKED[layout]
            for k, y in enumerate(ys):
                row = np.empty((512, 1024), np.uint8)
                row[:, yo::ysx], row[:, uo::us], row[:, vo::vs] = y, u, v
                assert np.array_equal(got[k], cv2.cvtColor(row.reshape(512, 512, 2), code)), (layout, k0 + k)


@pytest.mark.parametrize("fmt", [("bt601", False), ("bt709", True)], ids=str)
def test_444_crops_are_the_oracle_on_every_8_bit_triple(fmt):
    """64 frames of 512 x 512: pixel (i, j) of frame k is (Y, U, V) = (4k + 2 (i // 256) + j // 256, i mod 256,
    j mod 256)."""
    matrix, full = fmt
    i, j = np.meshgrid(np.arange(512), np.arange(512), indexing="ij")
    u, v = (i % 256).astype(np.uint8), (j % 256).astype(np.uint8)
    for k0 in range(0, 64, 16):
        ys = [(4 * k + 2 * (i // 256) + j // 256).astype(np.uint8) for k in range(k0, k0 + 16)]
        got = identity_crops([ycbcr_frame(y, u, v, ("i444", "i444_pitched", "roi444")[k % 3], matrix=matrix,
                                          full_range=full) for k, y in enumerate(ys)])
        for k, y in enumerate(ys):
            assert np.array_equal(got[k], oracle(y, u, v, "444", matrix, full)), (fmt, k0 + k)


WIDE_CASES = [  # (layout, matrix, full_range): MSB-aligned Y210 and 16-bit 4:4:4, LSB-aligned yuv422p10le / yuv444p10le
    ("yuyv", "bt709", False), ("i422", "bt2020", True), ("i444", "bt601", True), ("i444_msb_pitched", "bt2020", False),
]


@pytest.mark.parametrize("bits", [10, 12])
def test_wide_crops_are_the_oracle_on_every_pair_and_random_triples(bits):
    """The frames of test_gpu_yuv_formats (every (Y, V) and (Y, U) pair, then 2^22 seeded triples and the range
    extremes) with their 4:2:0 chroma repeated to 4:2:2 / 4:4:4, noise in the bits the reader masks."""
    py, pu, pv = pair_frames(bits)
    ry, ru, rv = random_frames(bits)
    ys, us, vs = py + ry, pu + ru, pv + rv
    rng = np.random.default_rng(bits)
    for layout, matrix, full in WIDE_CASES:
        sub = sub_of(layout)
        for i in range(0, len(ys), 16):
            part = range(i, min(i + 16, len(ys)))
            planes = [(ys[k], chroma_of(us[k], sub), chroma_of(vs[k], sub)) for k in part]
            got = identity_crops([ycbcr_frame(*p, layout, bits, rng=rng, matrix=matrix, full_range=full)
                                  for p in planes])
            for g, p, k in zip(got, planes, part):
                assert np.array_equal(g, oracle(*p, sub, matrix, full, bits)), (bits, layout, k)


# ---------------------------------------------------------------------------------------------------- kernels
CROP_CASES = [  # (layout, bits, matrix, full_range)
    ("yuyv_pitched", 8, "bt601", False), ("uyvy", 8, "bt709", False), ("yvyu", 8, "bt601", True),
    ("yuyv", 10, "bt2020", False), ("nv16_pitched", 8, "bt709", True), ("nv16", 10, "bt709", False),
    ("i422", 8, "bt601", False), ("i422", 10, "bt2020", True), ("roi422", 12, "bt709", False),
    ("i444_pitched", 8, "bt709", False), ("i444", 10, "bt2020", False), ("i444_msb_pitched", 12, "bt601", True),
    ("roi444", 8, "bt601", False), ("planes444", 12, "bt709", True), ("planes422", 8, "bt2020", False),
]


def random_planes(rng, h, w, bits, sub):
    sx = 1 if sub == "422" else 0
    return (rng.integers(0, 1 << bits, (h, w)), rng.integers(0, 1 << bits, (h, w >> sx)),
            rng.integers(0, 1 << bits, (h, w >> sx)))


@pytest.mark.parametrize("case", CROP_CASES, ids=lambda c: "-".join(map(str, c)))
def test_crop_ycbcr_kernel_matches_cv2_on_oracle_frame(case):
    """Frames with an odd H (4:2:2) or odd H and W (4:4:4); targets inside, across every border, tiny and huge; every
    unreadable entry and an out-of-range frame index give a padding-colour crop."""
    layout, bits, matrix, full = case
    sub = sub_of(layout)
    lib = _lib.init(0)
    rng = np.random.default_rng(37)
    shapes = [(255, 480), (183, 98), (91, 334)] if sub == "422" else [(255, 479), (183, 97), (90, 334)]
    planes = [random_planes(rng, h, w, bits, sub) for h, w in shapes]
    rgbs = [oracle(*p, sub, matrix, full, bits) for p in planes]
    means = [np.mean(f, axis=(0, 1)) for f in rgbs]
    targets = [(0, [163, 53, 45, 174]), (0, [-10, 100, 40, 30]), (0, [450, 20, 60, 40]), (0, [200, -15, 30, 50]),
               (0, [0, 0, 3, 3]), (0, [476, 252, 3, 3]), (0, [-50, 30, 600, 100]), (2, [-300, -200, 900, 500]),
               (2, [330, 87, 3, 3]), (2, [5, 40, 320, 20])]
    for side in (1, 3, 9, 33, 120, 200):
        targets.append((1, [48 - side // 2, 90 - side // 2, side, side]))
    frames = [ycbcr_frame(*p, layout, bits, rng=rng, matrix=matrix, full_range=full) for p in planes]
    records = [f.ycbcr_record() for f in frames]
    bad = unreadable_records(records[0])
    extra = [(9999, [12, 200, 255])] + [(len(records) + i, [i, 128, 7]) for i in range(len(bad))]
    recs = np.zeros((len(targets) + len(extra), _lib.TARGET_INTS), dtype=np.int32)
    for i, (f, box) in enumerate(targets):
        recs[i, 0], recs[i, 1:5] = f, box
        recs[i, 9:12] = np.clip(np.rint(means[f]), 0, 255)
    for i, (f, pad) in enumerate(extra):
        recs[len(targets) + i, 0], recs[len(targets) + i, 1:5], recs[len(targets) + i, 9:12] = f, [10, 10, 20, 20], pad
    table = ycbcr_table(records + bad)
    n = len(recs)
    for size, off in ((256, 2.0), (128, 0.2)):
        state = torch.from_numpy(recs).cuda()
        crops = torch.empty((n, size, size, 3), dtype=torch.uint8, device="cuda")
        _lib.check(lib.fear_crop_targets_ycbcr_u8(table.data_ptr(), len(records) + len(bad), state.data_ptr(), n, off,
                                                  size, crops.data_ptr(), stream()), "fear_crop_targets_ycbcr_u8")
        got, ctxs = crops.cpu().numpy(), state.cpu().numpy()[:, 5:9]
        for i, (f, box) in enumerate(targets):
            assert np.array_equal(ctxs[i], image_ops.context_box(box, off)), (case, size, off, box)
            assert np.array_equal(got[i], base._cv2_crop(rgbs[f], box, size, off, means[f])), (case, size, off, f, box)
        for i, (_, pad) in enumerate(extra):
            assert (got[len(targets) + i] == np.array(pad, dtype=np.uint8)).all(), (case, i)


def test_yuv420_frames_through_ycbcr_table_equal_yuv_table():
    """YUV420Frames of several formats give bit-identical crops, advances and sums through FearFrameYCbCr and
    FearFrameYUV."""
    lib = _lib.init(0)
    rng = np.random.default_rng(43)
    kinds = [((256, 480), "nv12", "bt601", False, 8), ((182, 98), "p010_pitched", "bt709", False, 10),
             ((2, 2), "i420", "bt2020", True, 8), ((90, 334), "i420_10le", "bt709", True, 12),
             ((1080, 1920), "pitched", "bt601", False, 8)]
    frames = []
    for (h, w), layout, m, f, b in kinds:
        y, u, v = (rng.integers(0, 1 << b, s) for s in ((h, w), (h // 2, w // 2), (h // 2, w // 2)))
        frames.append(code_frame(y, u, v, layout, m, f, b, rng))
    old = torch.from_numpy(np.array([f.yuv_record() for f in frames], dtype=_lib.YUV_DTYPE).view(np.uint8).copy()).cuda()
    new = ycbcr_table([f.ycbcr_record() for f in frames])
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
            ("yuv", old, lib.fear_crop_targets_yuv_u8, lib.fear_advance_targets_yuv, lib.fear_frame_sums_yuv_u8),
            ("ycbcr", new, lib.fear_crop_targets_ycbcr_u8, lib.fear_advance_targets_ycbcr,
             lib.fear_frame_sums_ycbcr_u8)):
        state = torch.from_numpy(recs).cuda()
        crops = torch.empty((n, 256, 256, 3), dtype=torch.uint8, device="cuda")
        s = torch.empty((F, 3), dtype=torch.int64, device="cuda")
        _lib.check(crop(table.data_ptr(), F, state.data_ptr(), n, 2.0, 256, crops.data_ptr(), stream()), name)
        _lib.check(adv(dboxes.data_ptr(), table.data_ptr(), F, state.data_ptr(), n, 256, stream()), name)
        _lib.check(sums(table.data_ptr(), F, s.data_ptr(), stream()), name)
        out[name] = (crops.cpu().numpy(), state.cpu().numpy(), s.cpu().numpy())
    for a, b in zip(out["yuv"], out["ycbcr"]):
        assert np.array_equal(a, b)


def test_advance_ycbcr_kernel_matches_host_rescale_and_clamp():
    """The 12 000 records of test_gpu_yuv_formats' advance test, on 4:2:2 and 4:4:4 frames of odd sizes; unreadable
    entries and out-of-range frame indices keep their boxes."""
    lib = _lib.init(0)
    rng = np.random.default_rng(5)
    shapes = [(255, 480), (183, 97), (1, 2)]
    n = 12000
    boxes = np.zeros(n, dtype=_lib.BOX_DTYPE)
    recs = np.zeros((n, _lib.TARGET_INTS), dtype=np.int32)
    recs[:, 0] = rng.integers(0, 3, n)
    recs[:, 5:7] = rng.integers(-600, 700, (n, 2))
    recs[:, 7:9] = rng.integers(1, 2000, (n, 2))
    xy = rng.uniform(-300, 600, (n, 2))
    wh = rng.uniform(0, 300, (n, 2))
    wh[n // 4:n // 2] = rng.uniform(0, 3, (n // 4, 2))
    half = slice(n // 2, 3 * n // 4)
    side = rng.choice([256, 512], n // 4)
    recs[half, 7] = recs[half, 8] = side
    v = rng.integers(-200, 300, (n // 4, 4)) + np.where(side == 512, 0.25, 0.5)[:, None]
    xy[half], wh[half] = v[:, :2], np.abs(v[:, 2:])
    boxes["x"], boxes["y"], boxes["w"], boxes["h"] = xy[:, 0], xy[:, 1], wh[:, 0], wh[:, 1]
    kinds = [("yuyv_pitched", 8, "bt709", False), ("i444", 10, "bt2020", True), ("nv16", 12, "bt601", False)]
    frames = [ycbcr_frame(*random_planes(rng, h, w, k[1], sub_of(k[0])), *k[:2], rng=rng, matrix=k[2],
                          full_range=k[3]) for (h, w), k in zip(shapes, kinds)]
    records = [f.ycbcr_record() for f in frames]
    bad = unreadable_records(records[1])
    table = ycbcr_table(records + bad)
    recs[-len(bad) - 4:-len(bad), 0] = 999
    recs[-len(bad):, 0] = 3 + np.arange(len(bad))
    kept = len(bad) + 4
    recs[-kept:, 1:5] = [7, 8, 9, 10]
    state = torch.from_numpy(recs).cuda()
    dboxes = torch.from_numpy(boxes.view(np.uint8).copy()).cuda()
    _lib.check(lib.fear_advance_targets_ycbcr(dboxes.data_ptr(), table.data_ptr(), 3 + len(bad), state.data_ptr(), n,
                                              256, stream()), "fear_advance_targets_ycbcr")
    got = state.cpu().numpy()
    for i in range(n - kept):
        b = np.array([boxes["x"][i], boxes["y"][i], boxes["w"][i], boxes["h"][i]])
        h, w = shapes[recs[i, 0]]
        want = image_ops.clamp_bbox(image_ops.rescale_bbox(b, recs[i, 5:9], 256), (h, w, 3))
        assert np.array_equal(got[i, 1:5], want), (i, b.tolist(), recs[i, 5:9].tolist(), (h, w), got[i, 1:5], want)
    assert (got[-kept:, 1:5] == [7, 8, 9, 10]).all()
    assert np.array_equal(np.delete(got, np.s_[1:5], axis=1), np.delete(recs, np.s_[1:5], axis=1))


def test_frame_sums_ycbcr_give_numpy_sums_of_oracle_frame():
    lib = _lib.init(0)
    rng = np.random.default_rng(11)
    cases = [((1, 2), "yuyv", 8, "bt601", False), ((1, 1), "i444", 8, "bt709", True),
             ((3, 2), "uyvy", 10, "bt709", False), ((183, 98), "i422", 10, "bt2020", True),
             ((37, 1003), "roi444", 12, "bt601", True), ((91, 334), "roi422", 8, "bt709", False),
             ((1081, 1920), "nv16_pitched", 10, "bt2020", False), ((1080, 1920), "yuyv_pitched", 8, "bt601", False),
             ((2160, 3840), "i444_msb_pitched", 10, "bt2020", False), ((2160, 3840), "yvyu", 8, "bt709", False)]
    planes = [random_planes(rng, h, w, b, sub_of(layout)) for (h, w), layout, b, _, _ in cases]
    frames = [ycbcr_frame(*p, layout, b, rng=rng, matrix=m, full_range=f)
              for p, (_, layout, b, m, f) in zip(planes, cases)]
    records = [f.ycbcr_record() for f in frames]
    bad = unreadable_records(records[3])
    table = ycbcr_table(records + bad)
    F = len(records) + len(bad)
    sums = torch.full((F, 3), -1, dtype=torch.int64, device="cuda")  # zeroed by the call
    _lib.check(lib.fear_frame_sums_ycbcr_u8(table.data_ptr(), F, sums.data_ptr(), stream()),
               "fear_frame_sums_ycbcr_u8")
    got = sums.cpu().numpy().view(np.uint64)
    for i, (p, (_, layout, b, m, f)) in enumerate(zip(planes, cases)):
        rgb = oracle(*p, sub_of(layout), m, f, b)
        assert np.array_equal(got[i], rgb.sum(axis=(0, 1), dtype=np.uint64)), (i, cases[i])
    assert (got[len(records):] == 0).all()


# ---------------------------------------------------------------------------------------------------- tracker
def encode(rgb: np.ndarray, matrix: str, full_range: bool, bits: int, sub: str, rng) -> tuple:
    """Code planes of an RGB frame by the forward H.273 equations (chroma: mean over each chroma sample's pixels),
    plus uniform noise of +-2 codes, clipped to the sample range."""
    _, kr, kb = image_ops.YUV_MATRICES[matrix]
    kg = 1.0 - kr - kb
    r, g, b = (rgb[..., c].astype(np.float64) / 255.0 for c in range(3))
    yn = kr * r + kg * g + kb * b
    pb, pr = (b - yn) / (2.0 * (1.0 - kb)), (r - yn) / (2.0 * (1.0 - kr))
    h, w = yn.shape
    sx, sy = SHIFTS[sub]
    pb, pr = (p.reshape(h >> sy, 1 << sy, w >> sx, 1 << sx).mean(axis=(1, 3)) for p in (pb, pr))
    m, top = 1 << (bits - 8), (1 << bits) - 1
    if full_range:
        y, u, v = yn * top, (1 << (bits - 1)) + pb * top, (1 << (bits - 1)) + pr * top
    else:
        y, u, v = 16 * m + 219 * m * yn, 128 * m + 224 * m * pb, 128 * m + 224 * m * pr
    return tuple(np.clip(np.rint(p + rng.uniform(-2, 2, p.shape)), 0, top).astype(np.int64) for p in (y, u, v))


STREAMS = [  # (size, layout, matrix, full_range, bits, subsampling)
    ((1920, 1080), "yuyv_pitched", "bt601", False, 8, "422"),
    ((480, 256), "nv16", "bt709", False, 10, "422"),
    ((480, 256), "i444_pitched", "bt709", False, 8, "444"),
    ((480, 256), "nv12", "bt601", False, 8, "420"),
]


def test_mixed_subsampling_streams_match_trackers_fed_oracle_frames(net, clip):
    """Pitched 1080p YUYV, P210, pitched BT.709 I444 and an NV12 YUV420Frame in one call, several targets each, add /
    remove part way.  One tracker gets fresh YUV frames every update; another alternates them with numpy-RGB, CUDA-RGB
    and 4:2:0-only calls.  Both give every output of a tracker fed image_ops.yuv_to_rgb's frames as numpy arrays, and
    the first replays one captured graph of the ycbcr table.  Every fourth frame is encoded at 4:2:0 and its chroma
    repeated to the stream's subsampling, so that the 4:2:0-only call (NV12 / P010 of the 4:2:0 codes) shows the
    tracker the same RGB frame."""
    T = 45
    rng = np.random.default_rng(79)
    planes, p420 = [], []
    for (w, h), _, matrix, full, bits, sub in STREAMS:
        planes.append([]), p420.append({})
        for t in range(T + 1):
            rgb_t = cv2.resize(clip[t], (w, h)) if (w, h) != clip.shape[2:0:-1] else clip[t]
            if t % 4 == 3:
                c = encode(rgb_t, matrix, full, bits, "420", rng)
                p420[-1][t] = c
                planes[-1].append(c if sub == "420" else (c[0], chroma_of(c[1], sub), chroma_of(c[2], sub)))
            else:
                planes[-1].append(encode(rgb_t, matrix, full, bits, sub, rng))
    rgb = [[oracle(*p, sub, m, f, b) for p in planes[s]] for s, (_, _, m, f, b, sub) in enumerate(STREAMS)]
    start = [[[652, 211, 180, 696], [1760, 840, 160, 224]], [base.GOLDEN_BOX, [300, 80, 60, 90]],
             [[168, 50, 40, 170], [-10, 100, 50, 50]], [base.GOLDEN_BOX, [440, 200, 40, 56]]]
    late = [[[400, 600, 120, 120]], [[100, 150, 30, 30]], [], [[0, 0, 40, 60]]]

    def rects(d):
        return [r for s in d for r in s], [k for k, s in enumerate(d) for _ in s]

    def yuv(t):
        out = []
        for s, (_, layout, m, f, b, sub) in enumerate(STREAMS):
            if sub == "420":
                out.append(code_frame(*planes[s][t], layout, m, f, b, rng))
            else:
                out.append(ycbcr_frame(*planes[s][t], layout, b, rng=rng, matrix=m, full_range=f))
        return out

    def frames(mode, t):
        if mode == "yuv":
            return yuv(t)
        if mode == "numpy":
            return [rgb[s][t] for s in range(len(STREAMS))]
        if mode == "yuv420":
            return [code_frame(*p420[s][t], "nv12" if b == 8 else "p010", m, f, b, rng)
                    for s, (_, _, m, f, b, _) in enumerate(STREAMS)]
        return [torch.from_numpy(rgb[s][t]).cuda() for s in range(len(STREAMS))]

    ref = fb.FEARMultiTracker(net, cuda_id=0, max_targets=12, **CFG)
    only = fb.FEARMultiTracker(net, cuda_id=0, max_targets=12, **CFG)
    mixed = fb.FEARMultiTracker(net, cuda_id=0, max_targets=12, **CFG)
    r, s = rects(start)
    want = ref.add(frames("numpy", 0), r, s)
    assert np.array_equal(only.add(yuv(0), r, s), want)
    assert np.array_equal(mixed.add(yuv(0), r, s), want)
    graph = None
    for t in range(1, T + 1):
        if t == 15:
            r, s = rects(late)
            want = ref.add(frames("numpy", t - 1), r, s)
            assert np.array_equal(only.add(yuv(t - 1), r, s), want)
            assert np.array_equal(mixed.add(frames("cuda", t - 1), r, s), want)
        if t == 30:
            for trk in (ref, only, mixed):
                trk.remove([1, 4])
        expect = ref.update(frames("numpy", t))
        for trk, mode in ((only, "yuv"), (mixed, ("yuv", "numpy", "cuda", "yuv420")[t % 4])):
            out = trk.update(frames(mode, t))
            assert np.array_equal(out["ids"], expect["ids"]), (mode, t)
            assert np.array_equal(out["bbox"], expect["bbox"]), (mode, t, out["bbox"], expect["bbox"])
            assert np.array_equal(out["score"], expect["score"]), (mode, t)
        if t in (17, 32):  # two updates after the add (warm-up + capture) and after the remove
            graph = only._graph
            assert graph is not None and only._graph_key[2] == "ycbcr"
        if t in (29, T):
            assert only._graph is graph  # replayed with new frame addresses, layouts and subsamplings every update
    assert len(only) == 9


def test_yuv420_only_calls_keep_the_yuv_table_and_any_422_or_444_frame_selects_ycbcr(net, clip):
    rng = np.random.default_rng(4)
    rgb = cv2.resize(clip[0], (480, 256))
    c420 = encode(rgb, "bt601", False, 8, "420", rng)
    c422 = encode(rgb, "bt601", False, 8, "422", rng)
    trk = fb.FEARMultiTracker(net, cuda_id=0, max_targets=4, cuda_graph=False, **CFG)
    nv12 = code_frame(*c420, "nv12", "bt601", False, 8, rng)
    trk.add([nv12, nv12], [base.GOLDEN_BOX, [10, 10, 40, 40]], [0, 1])
    for frames, table in (([nv12, nv12], "yuv"), ([nv12, ycbcr_frame(*c422, "yuyv")], "ycbcr"),
                          ([ycbcr_frame(*c422, "nv16"), ycbcr_frame(*c422, "i422")], "ycbcr"), ([nv12, nv12], "yuv")):
        trk.update(frames)
        assert trk._graph_key[2] == table


def test_launch_count_of_ycbcr_step_equals_rgb_step(net, clip):
    rgb = [np.stack([cv2.resize(f, (480, 256)) for f in clip[:4]]), np.ascontiguousarray(clip[:4, 30:201, 50:351])]
    rng = np.random.default_rng(3)
    codes = [[encode(f, "bt709", False, 10, "422", rng) for f in rgb[0]],
             [encode(f, "bt601", True, 8, "444", rng) for f in rgb[1]]]
    layouts = [("yuyv_pitched", 10, "bt709", False), ("i444_pitched", 8, "bt601", True)]
    deltas = {}
    for n in (1, 16):
        for kind in ("cuda", "ycbcr"):
            def frames(t):
                if kind == "cuda":
                    return [torch.from_numpy(np.ascontiguousarray(a[t])).cuda() for a in rgb]
                return [ycbcr_frame(*c[t], lay, b, rng=rng, matrix=m, full_range=f)
                        for c, (lay, b, m, f) in zip(codes, layouts)]

            trk = fb.FEARMultiTracker(net, cuda_id=0, max_targets=16, cuda_graph=False, **CFG)
            trk.initialize(frames(0), [base.GOLDEN_BOX] * n, [i % 2 for i in range(n)])
            trk.update(frames(1))
            torch.cuda.synchronize()
            c0 = net.launch_count()
            trk.update(frames(2))
            trk.update(frames(3))
            deltas[(n, kind)] = (net.launch_count() - c0) / 2
    # the net counts its own launches; the step adds the crop and advance kernels: 48 in all
    assert len(set(deltas.values())) == 1 and deltas[(1, "cuda")] + 2 == 48, deltas


def test_c_abi_rejects_bad_arguments_and_launches_nothing():
    lib = _lib.init(0)
    t = torch.full((1 << 16,), 0x5A, dtype=torch.uint8, device="cuda")
    p = t.data_ptr()
    good = dict(views=p, F=1, targets=p, N=1, offset=2.0, size=256, crops=p)

    def crop(**kw):
        a = dict(good, **kw)
        return lib.fear_crop_targets_ycbcr_u8(a["views"], a["F"], a["targets"], a["N"], a["offset"], a["size"],
                                              a["crops"], None)

    bad = [dict(views=None), dict(targets=None), dict(crops=None), dict(N=0), dict(N=-1), dict(N=65536), dict(F=0),
           dict(F=-3), dict(size=0), dict(size=257), dict(offset=-0.5), dict(offset=float("nan")),
           dict(offset=float("inf"))]
    for kw in bad:
        assert crop(**kw) == -1, kw
        assert _lib.last_error(), kw
    for args in [(None, p, 1, p, 1, 256), (p, None, 1, p, 1, 256), (p, p, 1, None, 1, 256), (p, p, 1, p, 0, 256),
                 (p, p, 0, p, 1, 256), (p, p, 1, p, 1, 0)]:
        assert lib.fear_advance_targets_ycbcr(*args, None) == -1, args
        assert _lib.last_error(), args
    for args in [(None, 1, p), (p, 1, None), (p, 0, p), (p, 65536, p), (p, -1, p)]:
        assert lib.fear_frame_sums_ycbcr_u8(*args, None) == -1, args
        assert _lib.last_error(), args
    torch.cuda.synchronize()
    assert (t == 0x5A).all()  # no kernel and no memset ran
