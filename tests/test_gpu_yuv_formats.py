"""GPU tests of YUV 4:2:0 frames in every colour format: the FearFrameYUV entry points (fear_crop_targets_yuv_u8,
fear_advance_targets_yuv, fear_frame_sums_yuv_u8) and FEARMultiTracker fed BT.709, BT.2020, full-range and 10 / 12-bit
YUV420Frames.

Every comparison is exact, against image_ops.yuv420_to_rgb (the numpy restatement of the conversion, itself pinned to
cv2, to exact rationals and to PIL by tests/test_yuv_formats_cpu.py): identity-resample crops against the converted
frames, crops against cv2 on the converted frame, boxes against the host rescale + clamp, sums against numpy, and every
tracker output against the same tracker fed the converted frames as numpy arrays."""
import itertools
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
from tests.test_yuv_formats_cpu import NON_DEFAULT, extreme_codes, yuv16_frame
from tests.test_yuv_frames_cpu import LAYOUTS, yuv_frame

pytestmark = pytest.mark.gpu
CFG = fb.FEAR_XS_TRACKER_KWARGS
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


def yuv_table(records) -> torch.Tensor:
    return torch.from_numpy(np.array(records, dtype=_lib.YUV_DTYPE).view(np.uint8).copy()).cuda()


def stream():
    return torch.cuda.current_stream().cuda_stream


def samples(codes: np.ndarray, bits: int, msb: bool, rng) -> np.ndarray:
    """uint16 samples holding ``codes``: MSB-aligned with random low bits, or LSB-aligned with random high bits (the
    kernels must mask both away)."""
    codes = codes.astype(np.int64)
    noise = rng.integers(0, 1 << (16 - bits), codes.shape)
    return ((codes << (16 - bits)) | noise if msb else codes | (noise << bits)).astype(np.uint16)


def code_frame(y, u, v, layout, matrix="bt601", full_range=False, bits=8, rng=None) -> fb.YUV420Frame:
    """Code planes (Y (H, W), U and V (H/2, W/2)) as a fresh YUV420Frame on the device.  8-bit layouts are those of
    tests/test_yuv_frames_cpu.yuv_frame; 16-bit ones those of tests/test_yuv_formats_cpu.yuv16_frame, the samples
    aligned as the layout stores them, with noise in the bits the reader masks."""
    fmt = dict(matrix=matrix, full_range=full_range, bits=bits)
    if bits == 8:
        i420 = np.concatenate([np.asarray(p, np.uint8).reshape(-1) for p in (y, u, v)]).reshape(-1, y.shape[1])
        f = yuv_frame(i420, layout)
        return fb.YUV420Frame(f.y, f.u, f.v, **fmt)
    rng = rng if rng is not None else np.random.default_rng(0)
    msb = layout != "i420_10le"
    return yuv16_frame(*(samples(p, bits, msb, rng) for p in (y, u, v)), layout, **fmt)


def oracle(y, u, v, matrix="bt601", full_range=False, bits=8) -> np.ndarray:
    return image_ops.yuv420_to_rgb(y, u, v, matrix, full_range, bits, 0)


def invalid_records(rec):
    """Entries the kernels must treat as empty, derived from a valid record: an unknown matrix, full_range 2, bits 9,
    a shift past 16 - bits (any shift at 8 bits), a negative shift, a null plane, H = 0; and for a 16-bit record an odd
    plane address, an odd row stride and an odd pixel stride (8-bit samples may sit at any address)."""
    rec = list(rec)
    out = []
    edits = [(9, 3), (10, 2), (11, 9), (12, 17 - rec[11]), (12, -1), (2, 0), (7, 0)]
    if rec[11] > 8:
        edits += [(1, rec[1] + 1), (3, rec[3] + 1), (6, rec[6] - 1)]
    for field, value in edits:
        r = list(rec)
        r[field] = value
        out.append(tuple(r))
    return out


# ---------------------------------------------------------------------------------------------------- conversion
def identity_crops(frames) -> np.ndarray:
    """The four 256 x 256 quadrants of every 512 x 512 frame cropped at offset 0 to 256 x 256 (an identity resample:
    coefficients (2048, 0)), reassembled: (K, 512, 512, 3), the RGB frames the kernels see."""
    lib = _lib.init(0)
    quads = [(0, 0), (256, 0), (0, 256), (256, 256)]
    k = len(frames)
    recs = np.zeros((4 * k, _lib.TARGET_INTS), dtype=np.int32)
    for i in range(k):
        for q, (x, y) in enumerate(quads):
            recs[4 * i + q, 0], recs[4 * i + q, 1:5] = i, [x, y, 256, 256]
    state = torch.from_numpy(recs).cuda()
    crops = torch.empty((4 * k, 256, 256, 3), dtype=torch.uint8, device="cuda")
    table = yuv_table([f.yuv_record() for f in frames])
    _lib.check(lib.fear_crop_targets_yuv_u8(table.data_ptr(), k, state.data_ptr(), 4 * k, 0.0, 256, crops.data_ptr(),
                                            stream()), "fear_crop_targets_yuv_u8")
    got = crops.cpu().numpy().reshape(k, 2, 2, 256, 256, 3)  # (frame, y half, x half, row, column, channel)
    return got.transpose(0, 1, 3, 2, 4, 5).reshape(k, 512, 512, 3)


def all_8_bit_triples():
    """64 frames of 512 x 512 holding every 8-bit (Y, U, V) triple (as tests/test_gpu_yuv_frames)."""
    u, v = np.meshgrid(np.arange(256), np.arange(256), indexing="ij")
    ys = []
    for k in range(64):
        y = np.empty((512, 512), np.int64)
        for dy in range(2):
            for dx in range(2):
                y[dy::2, dx::2] = 4 * k + 2 * dy + dx
        ys.append(y)
    return ys, u, v


@pytest.mark.parametrize("fmt", [f for f in NON_DEFAULT if f[2] == 8], ids=str)
def test_8_bit_formats_match_oracle_on_every_triple(fmt):
    matrix, full, _ = fmt
    ys, u, v = all_8_bit_triples()
    frames = [code_frame(y, u, v, "i420" if k % 2 else "pitched", matrix, full) for k, y in enumerate(ys)]
    got = identity_crops(frames)
    for k, y in enumerate(ys):
        assert np.array_equal(got[k], oracle(y, u, v, matrix, full)), (fmt, k)


def pair_frames(bits):
    """Frames of 512 x 512 code planes holding every (Y, V) pair and every (Y, U) pair of a bit depth: 2 x 2 block g
    holds the pairs 4g .. 4g + 3 of (V, Y) in row-major order, and U = (1237 V + 517) mod 2^bits (a bijection)."""
    mask = (1 << bits) - 1
    per_frame = 256 * 256
    ys, us, vs = [], [], []
    for k in range((1 << (2 * bits)) // (4 * per_frame)):
        g = k * per_frame + np.arange(per_frame).reshape(256, 256)
        v = (4 * g) >> bits
        y = np.empty((512, 512), np.int64)
        for dy in range(2):
            for dx in range(2):
                y[dy::2, dx::2] = (4 * g + 2 * dy + dx) & mask
        ys.append(y), us.append((1237 * v + 517) & mask), vs.append(v)
    return ys, us, vs


def random_frames(bits, count=16, seed=0):
    """count frames of 512 x 512 of seeded random codes (2^22 luma samples at 16 frames); the first 216 blocks of frame
    0 hold every triple of the range extremes (0, 16m, 128m, 235m, 240m, max), four equal luma samples each."""
    rng = np.random.default_rng(seed + bits)
    ys = [rng.integers(0, 1 << bits, (512, 512)) for _ in range(count)]
    us = [rng.integers(0, 1 << bits, (256, 256)) for _ in range(count)]
    vs = [rng.integers(0, 1 << bits, (256, 256)) for _ in range(count)]
    ext = np.array(list(itertools.product(extreme_codes(bits), repeat=3)))
    r, c = np.divmod(np.arange(len(ext)), 256)
    for dy in range(2):
        for dx in range(2):
            ys[0][2 * r + dy, 2 * c + dx] = ext[:, 0]
    us[0][r, c], vs[0][r, c] = ext[:, 1], ext[:, 2]
    return ys, us, vs


@pytest.mark.parametrize("bits", [10, 12])
def test_wide_formats_match_oracle_on_every_pair_and_random_triples(bits):
    """Every matrix and range, MSB-aligned (P010 / P016 layout, noise in the low bits) and LSB-aligned (yuv420p10le,
    noise in the high bits): R over all (Y, V) pairs, B over all (Y, U) pairs, G over those pixels and 2^22 seeded
    triples plus the range extremes; all three channels are compared on every pixel."""
    py, pu, pv = pair_frames(bits)
    ry, ru, rv = random_frames(bits)
    ys, us, vs = py + ry, pu + ru, pv + rv
    rng = np.random.default_rng(bits)
    for matrix, full in MATRIX_RANGES:
        want = [oracle(y, u, v, matrix, full, bits) for y, u, v in zip(ys, us, vs)]
        for layout in ("p010", "i420_10le"):
            got = np.concatenate([identity_crops([code_frame(y, u, v, layout, matrix, full, bits, rng)
                                                  for y, u, v in zip(ys[i:i + 16], us[i:i + 16], vs[i:i + 16])])
                                  for i in range(0, len(ys), 16)])
            for k in range(len(ys)):
                assert np.array_equal(got[k], want[k]), (bits, matrix, full, layout, k)


# ---------------------------------------------------------------------------------------------------- kernels
FORMAT_LAYOUTS = [  # (layout, matrix, full_range, bits)
    ("p010", "bt2020", False, 10), ("p010_pitched", "bt709", False, 10), ("planes16", "bt2020", True, 12),
    ("i420_10le", "bt709", True, 10), ("roi16", "bt601", False, 12), ("pitched", "bt709", False, 8),
    ("i420", "bt601", True, 8), ("roi", "bt2020", False, 8),
]


def random_code_planes(rng, h, w, bits):
    return (rng.integers(0, 1 << bits, (h, w)), rng.integers(0, 1 << bits, (h // 2, w // 2)),
            rng.integers(0, 1 << bits, (h // 2, w // 2)))


@pytest.mark.parametrize("case", FORMAT_LAYOUTS, ids=lambda c: "-".join(map(str, c)))
def test_crop_yuv_kernel_matches_cv2_on_oracle_frame(case):
    layout, matrix, full, bits = case
    lib = _lib.init(0)
    rng = np.random.default_rng(31)
    planes = [random_code_planes(rng, h, w, bits) for h, w in ((256, 480), (182, 98), (90, 334))]
    rgbs = [oracle(*p, matrix, full, bits) for p in planes]
    means = [np.mean(f, axis=(0, 1)) for f in rgbs]
    targets = [(0, [163, 53, 45, 174]), (0, [-10, 100, 40, 30]), (0, [450, 20, 60, 40]), (0, [200, -15, 30, 50]),
               (0, [0, 0, 3, 3]), (0, [477, 253, 3, 3]), (0, [-50, 30, 600, 100]), (2, [-300, -200, 900, 500]),
               (2, [330, 87, 3, 3]), (2, [5, 40, 320, 20])]
    for side in (1, 3, 9, 33, 120, 200):
        targets.append((1, [48 - side // 2, 90 - side // 2, side, side]))
    frames = [code_frame(*p, layout, matrix, full, bits, rng) for p in planes]
    records = [f.yuv_record() for f in frames]
    bad = invalid_records(records[0])
    extra = [(9999, [12, 200, 255])] + [(len(records) + i, [i, 128, 7]) for i in range(len(bad))]
    recs = np.zeros((len(targets) + len(extra), _lib.TARGET_INTS), dtype=np.int32)
    for i, (f, box) in enumerate(targets):
        recs[i, 0], recs[i, 1:5] = f, box
        recs[i, 9:12] = np.clip(np.rint(means[f]), 0, 255)
    for i, (f, pad) in enumerate(extra):
        recs[len(targets) + i, 0], recs[len(targets) + i, 1:5], recs[len(targets) + i, 9:12] = f, [10, 10, 20, 20], pad
    table = yuv_table(records + bad)
    n = len(recs)
    for size, off in ((256, 2.0), (128, 0.2), (256, 0.5)):
        state = torch.from_numpy(recs).cuda()
        crops = torch.empty((n, size, size, 3), dtype=torch.uint8, device="cuda")
        _lib.check(lib.fear_crop_targets_yuv_u8(table.data_ptr(), len(records) + len(bad), state.data_ptr(), n, off,
                                                size, crops.data_ptr(), stream()), "fear_crop_targets_yuv_u8")
        got, ctxs = crops.cpu().numpy(), state.cpu().numpy()[:, 5:9]
        for i, (f, box) in enumerate(targets):
            assert np.array_equal(ctxs[i], image_ops.context_box(box, off)), (case, size, off, box)
            assert np.array_equal(got[i], base._cv2_crop(rgbs[f], box, size, off, means[f])), (case, size, off, f, box)
        for i, (_, pad) in enumerate(extra):
            assert (got[len(targets) + i] == np.array(pad, dtype=np.uint8)).all(), (case, i)


def test_default_format_through_yuv_table_equals_yuv420_entry_points():
    """Default-format frames give the same crops, advances and sums through FearFrameYUV and FearFrameYUV420."""
    lib = _lib.init(0)
    rng = np.random.default_rng(41)
    shapes = [(256, 480), (182, 98), (2, 2), (90, 334), (1080, 1920)]
    frames = [yuv_frame(rng.integers(0, 256, (h * 3 // 2, w), dtype=np.uint8), LAYOUTS[i % len(LAYOUTS)])
              for i, (h, w) in enumerate(shapes)]
    old = torch.from_numpy(np.array([f.record() for f in frames], dtype=_lib.YUV420_DTYPE).view(np.uint8).copy()).cuda()
    new = yuv_table([f.yuv_record() for f in frames])
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
            ("yuv420", old, lib.fear_crop_targets_yuv420_u8, lib.fear_advance_targets_yuv420,
             lib.fear_frame_sums_yuv420_u8),
            ("yuv", new, lib.fear_crop_targets_yuv_u8, lib.fear_advance_targets_yuv, lib.fear_frame_sums_yuv_u8)):
        state = torch.from_numpy(recs).cuda()
        crops = torch.empty((n, 256, 256, 3), dtype=torch.uint8, device="cuda")
        s = torch.empty((F, 3), dtype=torch.int64, device="cuda")
        _lib.check(crop(table.data_ptr(), F, state.data_ptr(), n, 2.0, 256, crops.data_ptr(), stream()), name)
        _lib.check(adv(dboxes.data_ptr(), table.data_ptr(), F, state.data_ptr(), n, 256, stream()), name)
        _lib.check(sums(table.data_ptr(), F, s.data_ptr(), stream()), name)
        out[name] = (crops.cpu().numpy(), state.cpu().numpy(), s.cpu().numpy())
    for a, b in zip(out["yuv420"], out["yuv"]):
        assert np.array_equal(a, b)


def test_advance_yuv_kernel_matches_host_rescale_and_clamp():
    """The 12 000 records of test_gpu_yuv_frames' advance test, on frames of several formats; entries the kernels
    cannot read keep their boxes."""
    lib = _lib.init(0)
    rng = np.random.default_rng(5)
    shapes = [(256, 480), (182, 98), (2, 2)]
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
    kinds = [("p010_pitched", "bt709", False, 10), ("i420_10le", "bt2020", True, 12), ("nv12", "bt709", True, 8)]
    frames = [code_frame(*random_code_planes(rng, h, w, k[3]), *k, rng) for (h, w), k in zip(shapes, kinds)]
    records = [f.yuv_record() for f in frames]
    bad = invalid_records(records[0])
    table = yuv_table(records + bad)
    recs[-len(bad) - 4:-len(bad), 0] = 999  # frame index out of range: the box is kept
    recs[-len(bad):, 0] = 3 + np.arange(len(bad))  # entries the kernels cannot read: the box is kept
    kept = len(bad) + 4
    recs[-kept:, 1:5] = [7, 8, 9, 10]
    state = torch.from_numpy(recs).cuda()
    dboxes = torch.from_numpy(boxes.view(np.uint8).copy()).cuda()
    _lib.check(lib.fear_advance_targets_yuv(dboxes.data_ptr(), table.data_ptr(), 3 + len(bad), state.data_ptr(), n,
                                            256, stream()), "fear_advance_targets_yuv")
    got = state.cpu().numpy()
    for i in range(n - kept):
        b = np.array([boxes["x"][i], boxes["y"][i], boxes["w"][i], boxes["h"][i]])
        h, w = shapes[recs[i, 0]]
        want = image_ops.clamp_bbox(image_ops.rescale_bbox(b, recs[i, 5:9], 256), (h, w, 3))
        assert np.array_equal(got[i, 1:5], want), (i, b.tolist(), recs[i, 5:9].tolist(), (h, w), got[i, 1:5], want)
    assert (got[-kept:, 1:5] == [7, 8, 9, 10]).all()
    assert np.array_equal(np.delete(got, np.s_[1:5], axis=1), np.delete(recs, np.s_[1:5], axis=1))


def test_frame_sums_yuv_give_numpy_sums_of_oracle_frame():
    lib = _lib.init(0)
    rng = np.random.default_rng(9)
    cases = [((2, 2), "p010", "bt2020", False, 10), ((182, 98), "i420_10le", "bt709", True, 10),
             ((38, 1002), "roi16", "bt601", True, 12), ((2, 514), "planes16", "bt2020", True, 12),
             ((2160, 3840), "p010_pitched", "bt2020", False, 10), ((4, 6), "i420", "bt709", False, 8),
             ((90, 334), "roi", "bt601", True, 8), ((1080, 1920), "pitched", "bt709", False, 8),
             ((1080, 1920), "nv12", "bt601", False, 8)]
    planes = [random_code_planes(rng, h, w, c[3]) for (h, w), *c in cases]
    frames = [code_frame(*p, layout, m, f, b, rng) for p, (_, layout, m, f, b) in zip(planes, cases)]
    records = [f.yuv_record() for f in frames]
    bad = invalid_records(records[1])
    table = yuv_table(records + bad)
    F = len(records) + len(bad)
    sums = torch.full((F, 3), -1, dtype=torch.int64, device="cuda")  # zeroed by the call
    _lib.check(lib.fear_frame_sums_yuv_u8(table.data_ptr(), F, sums.data_ptr(), stream()), "fear_frame_sums_yuv_u8")
    got = sums.cpu().numpy().view(np.uint64)
    for i, (p, (hw, _, m, f, b)) in enumerate(zip(planes, cases)):
        rgb = oracle(*p, m, f, b)
        assert np.array_equal(got[i], rgb.sum(axis=(0, 1), dtype=np.uint64)), (i, cases[i])
    assert (got[len(records):] == 0).all()


# ---------------------------------------------------------------------------------------------------- tracker
def encode(rgb: np.ndarray, matrix: str, full_range: bool, bits: int, rng) -> tuple:
    """Code planes of an RGB frame by the forward H.273 equations (chroma: mean of each 2 x 2 block), plus uniform noise
    of +-2 codes so that every code occurs, clipped to the sample range."""
    _, kr, kb = image_ops.YUV_MATRICES[matrix]
    kg = 1.0 - kr - kb
    r, g, b = (rgb[..., c].astype(np.float64) / 255.0 for c in range(3))
    yn = kr * r + kg * g + kb * b
    pb, pr = (b - yn) / (2.0 * (1.0 - kb)), (r - yn) / (2.0 * (1.0 - kr))
    h, w = yn.shape
    pb, pr = (p.reshape(h // 2, 2, w // 2, 2).mean(axis=(1, 3)) for p in (pb, pr))
    m, top = 1 << (bits - 8), (1 << bits) - 1
    if full_range:
        y, u, v = yn * top, (1 << (bits - 1)) + pb * top, (1 << (bits - 1)) + pr * top
    else:
        y, u, v = 16 * m + 219 * m * yn, 128 * m + 224 * m * pb, 128 * m + 224 * m * pr
    return tuple(np.clip(np.rint(p + rng.uniform(-2, 2, p.shape)), 0, top).astype(np.uint16) for p in (y, u, v))


STREAMS = [  # (size, layout, matrix, full_range, bits)
    ((1920, 1080), "pitched", "bt709", False, 8),
    ((480, 256), "p010", "bt2020", False, 10),
    ((480, 256), "i420_10le", "bt709", True, 10),
    ((480, 256), "nv12", "bt601", False, 8),
]


def test_four_format_streams_match_trackers_fed_oracle_frames(net, clip):
    """Pitched BT.709 NV12 at 1080p, BT.2020 P010, full-range BT.709 yuv420p10le and default NV12 in one call, several
    targets each, add / remove part way.  One tracker gets fresh YUV420Frames every update, another alternates YUV,
    numpy-RGB and CUDA-RGB calls; both must give every output of a tracker fed image_ops.yuv420_to_rgb's frames as
    numpy arrays, and the YUV-only tracker replays one captured graph."""
    T = 45
    rng = np.random.default_rng(77)
    planes = []
    for (w, h), _, matrix, full, bits in STREAMS:
        planes.append([encode(cv2.resize(clip[t], (w, h)) if (w, h) != clip.shape[2:0:-1] else clip[t],
                              matrix, full, bits, rng) for t in range(T + 1)])
    rgb = [[oracle(*p, m, f, b) for p in planes[s]] for s, (_, _, m, f, b) in enumerate(STREAMS)]
    start = [[[652, 211, 180, 696], [1760, 840, 160, 224]], [base.GOLDEN_BOX, [300, 80, 60, 90]],
             [[168, 50, 40, 170], [-10, 100, 50, 50]], [base.GOLDEN_BOX, [440, 200, 40, 56]]]
    late = [[[400, 600, 120, 120]], [[100, 150, 30, 30]], [], [[0, 0, 40, 60]]]

    def rects(d):
        return [r for s in d for r in s], [k for k, s in enumerate(d) for _ in s]

    def yuv(t):
        return [code_frame(*planes[s][t], layout, m, f, b, rng) for s, (_, layout, m, f, b) in enumerate(STREAMS)]

    def frames(mode, t):
        if mode == "yuv":
            return yuv(t)
        if mode == "numpy":
            return [rgb[s][t] for s in range(len(STREAMS))]
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
        for trk, mode in ((only, "yuv"), (mixed, ("yuv", "numpy", "cuda")[t % 3])):
            out = trk.update(frames(mode, t))
            assert np.array_equal(out["ids"], expect["ids"]), (mode, t)
            assert np.array_equal(out["bbox"], expect["bbox"]), (mode, t, out["bbox"], expect["bbox"])
            assert np.array_equal(out["score"], expect["score"]), (mode, t)
        if t in (17, 32):  # two updates after the add (warm-up + capture) and after the remove
            graph = only._graph
            assert graph is not None
        if t in (29, T):
            assert only._graph is graph  # replayed with new frame addresses and mixed formats every update
    assert len(only) == 9


def test_launch_count_of_format_step_equals_rgb_step(net, clip):
    rgb = [clip[:4], np.ascontiguousarray(clip[:4, 30:200, 50:350])]
    rng = np.random.default_rng(3)
    codes = [[encode(f, "bt2020", False, 10, rng) for f in rgb[0]], [encode(f, "bt709", True, 8, rng) for f in rgb[1]]]
    layouts = [("p010", "bt2020", False, 10), ("i420", "bt709", True, 8)]
    deltas = {}
    for n in (1, 16):
        for kind in ("cuda", "yuv"):
            def frames(t):
                if kind == "cuda":
                    return [torch.from_numpy(np.ascontiguousarray(a[t])).cuda() for a in rgb]
                return [code_frame(*c[t], *lay, rng) for c, lay in zip(codes, layouts)]

            trk = fb.FEARMultiTracker(net, cuda_id=0, max_targets=16, cuda_graph=False, **CFG)
            trk.initialize(frames(0), [base.GOLDEN_BOX] * n, [i % 2 for i in range(n)])
            trk.update(frames(1))
            torch.cuda.synchronize()
            c0 = net.launch_count()
            trk.update(frames(2))
            trk.update(frames(3))
            deltas[(n, kind)] = (net.launch_count() - c0) / 2
    assert len(set(deltas.values())) == 1 and deltas[(1, "cuda")] > 0, deltas
    print(f"launches per step: {deltas[(1, 'cuda')]}")


def test_c_abi_rejects_bad_arguments_and_launches_nothing():
    lib = _lib.init(0)
    t = torch.full((1 << 16,), 0x5A, dtype=torch.uint8, device="cuda")
    p = t.data_ptr()
    good = dict(views=p, F=1, targets=p, N=1, offset=2.0, size=256, crops=p)

    def crop(**kw):
        a = dict(good, **kw)
        return lib.fear_crop_targets_yuv_u8(a["views"], a["F"], a["targets"], a["N"], a["offset"], a["size"],
                                            a["crops"], None)

    bad = [dict(views=None), dict(targets=None), dict(crops=None), dict(N=0), dict(N=-1), dict(N=65536), dict(F=0),
           dict(F=-3), dict(size=0), dict(size=257), dict(offset=-0.5), dict(offset=float("nan")),
           dict(offset=float("inf"))]
    for kw in bad:
        assert crop(**kw) == -1, kw
        assert _lib.last_error(), kw
    for args in [(None, p, 1, p, 1, 256), (p, None, 1, p, 1, 256), (p, p, 1, None, 1, 256), (p, p, 1, p, 0, 256),
                 (p, p, 0, p, 1, 256), (p, p, 1, p, 1, 0)]:
        assert lib.fear_advance_targets_yuv(*args, None) == -1, args
        assert _lib.last_error(), args
    for args in [(None, 1, p), (p, 1, None), (p, 0, p), (p, 65536, p), (p, -1, p)]:
        assert lib.fear_frame_sums_yuv_u8(*args, None) == -1, args
        assert _lib.last_error(), args
    torch.cuda.synchronize()
    assert (t == 0x5A).all()  # no kernel and no memset ran
