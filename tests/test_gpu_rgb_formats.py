"""GPU tests of RGB frames in any channel order and container: the FearFrameRGB entry points (fear_crop_targets_rgb_u8,
fear_advance_targets_rgb, fear_frame_sums_rgb_u8), RGBFrame, and FEARMultiTracker / FEARTracker fed BGR, BGRA / ABGR,
x2rgb10, rgb48 / rgba64 and planar frames, alone and mixed with CUDA RGB tensors.

Every comparison is exact, against image_ops.rgb_frame_to_rgb of the frame's samples (pinned to cv2.cvtColor and
raw_to_u8 by tests/test_rgb_formats_cpu.py): identity crops against the RGB frame itself, general crops against cv2 on
it, boxes against the host rescale + clamp, sums against numpy, and every tracker output against the same tracker fed the
RGB frames as numpy arrays.  Alpha and X samples, the spare bits of x2rgb10 words and the bits above a planar code are
random, and the memory around each frame holds 0xA5."""
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
from feartracker_b200 import multi_tracker as mt
from oracle import fear_oracle as fo
from tests import test_gpu_multi_tracker as base
from tests.helpers import GOLDEN, load_full_state

pytestmark = pytest.mark.gpu
CFG = fb.FEAR_XS_TRACKER_KWARGS
HERE = os.path.dirname(os.path.abspath(__file__))
# (layout, bits): every packed layout and every planar depth
LAYOUTS = [(k, 8 if v[0] == np.uint8 else 16) for k, v in image_ops.RGB_PACKED_LAYOUTS.items()] + \
          [(k, 10) for k in image_ops.X2RGB10_LAYOUTS] + [("planar", b) for b in image_ops.RGB_PLANAR_BITS]


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


def code_dtype(bits):
    return np.uint8 if bits == 8 else np.uint16


# ---------------------------------------------------------------------------------------------------- frames
def layout_data(codes: np.ndarray, layout: str, bits: int, rng) -> np.ndarray:
    """The samples of RGB ``codes`` ((H, W, 3) at ``bits``) in ``layout``: (H, W, C) packed samples with random alpha /
    X samples, (H, W) int32 x2rgb10 words with random spare bits, or (3, H, W) R, G, B planes with random bits above
    the code."""
    h, w, _ = codes.shape
    if layout in image_ops.RGB_PACKED_LAYOUTS:
        dtype, n, idx = image_ops.RGB_PACKED_LAYOUTS[layout]
        a = rng.integers(0, np.iinfo(dtype).max + 1, (h, w, n)).astype(dtype)
        for c in range(3):
            a[..., idx[c]] = codes[..., c]
        return a
    if layout in image_ops.X2RGB10_LAYOUTS:
        return image_ops.x2rgb10_pack(codes, layout, rng.integers(0, 4, (h, w))).view(np.int32)
    planes = np.moveaxis(codes, -1, 0).astype(code_dtype(bits))
    if bits not in (8, 16):
        planes = planes | (rng.integers(0, 1 << (16 - bits), planes.shape) << bits).astype(np.uint16)
    return planes


def device(a: np.ndarray) -> torch.Tensor:
    a = np.ascontiguousarray(a)
    if a.dtype == np.uint16:
        return torch.from_numpy(a.view(np.int16)).cuda().view(torch.uint16)
    return torch.from_numpy(a).cuda()


def place(a: np.ndarray, col: int = 0, extra: int = 0, planar: bool = False) -> torch.Tensor:
    """``a`` ((H, W, ...) samples, or with ``planar`` (3, H, W) planes) at row 1, column ``col`` of a device surface of
    0xA5 bytes whose rows are ``extra`` pixels longer: the view of ``a`` in it."""
    if planar:
        a = np.moveaxis(a, 0, -1)
    h, w = a.shape[:2]
    fill = {1: 0xA5, 2: 0xA5A5, 4: -0x5A5A5A5B}[a.dtype.itemsize]
    surf = np.full((h + 2, col + w + extra) + a.shape[2:], fill, a.dtype)
    surf[1:h + 1, col:col + w] = a
    if planar:
        surf = np.moveaxis(surf, -1, 0)  # each plane its own surface of the same pitch
    t = device(surf)
    return t[:, 1:h + 1, col:col + w] if planar else t[1:h + 1, col:col + w]


def make_frame(codes, layout, bits, rng, col=0, extra=0, uint32=False, chw=False):
    """(RGBFrame of ``codes`` in ``layout`` at column ``col`` of a pitched 0xA5 surface, the numpy RGB frame it stands
    for).  ``uint32``: x2rgb10 words as a torch.uint32 tensor; ``chw``: planes as one contiguous (3, H, W) tensor, as
    torchvision's decode_png returns a 16-bit PNG."""
    data = layout_data(codes, layout, bits, rng)
    want = image_ops.rgb_frame_to_rgb(data, layout, bits)
    if layout == "planar":
        t = device(data) if chw else place(data, col, extra, planar=True)
        return fb.RGBFrame.planar(*t, bits=bits), want
    t = place(data, col, extra)
    if uint32:
        t = t.view(torch.uint32)
    return fb.RGBFrame(t, layout), want


def rgb_table(records) -> torch.Tensor:
    return torch.from_numpy(np.array(records, dtype=_lib.RGB_DTYPE).view(np.uint8).copy()).cuda()


def unreadable_records(rec8, rec16, rec32):
    """Entries the kernels must treat as empty, from valid records of an 8-bit, a uint16 and an x2rgb10 frame: every
    rule of FearFrameRGB broken once."""
    def edit(rec, **kw):
        r = np.array(rec, dtype=_lib.RGB_DTYPE)
        for k, v in kw.items():
            r[k] = v
        return tuple(r.tolist())

    return [
        edit(rec8, r=0), edit(rec8, g=0), edit(rec8, b=0), edit(rec8, H=0), edit(rec8, W=0), edit(rec8, W=-5),
        edit(rec8, H=-1), edit(rec8, container=0), edit(rec8, container=3), edit(rec8, container=8),
        edit(rec8, container=-1), edit(rec8, bits=10), edit(rec8, bits=16), edit(rec8, shift_g=1),
        edit(rec8, shift_b=-1), edit(rec8, row_stride=-rec8[3]), edit(rec8, pixel_stride=-3),
        edit(rec16, bits=8), edit(rec16, bits=14), edit(rec16, bits=11), edit(rec16, bits=0), edit(rec16, shift_r=1),
        edit(rec16, bits=12, shift_g=5), edit(rec16, bits=10, shift_b=-1), edit(rec16, bits=10, shift_r=7),
        edit(rec16, r=rec16[0] + 1), edit(rec16, b=rec16[2] + 1), edit(rec16, row_stride=rec16[3] + 1),
        edit(rec16, pixel_stride=rec16[4] + 1), edit(rec16, container=4),
        edit(rec32, bits=12), edit(rec32, bits=8), edit(rec32, g=rec32[1] + 4), edit(rec32, b=rec32[2] + 4),
        edit(rec32, shift_r=0, shift_g=10, shift_b=10), edit(rec32, shift_r=0, shift_g=10, shift_b=21),
        edit(rec32, shift_r=0, shift_g=10, shift_b=30), edit(rec32, shift_r=-10, shift_g=10, shift_b=20),
        edit(rec32, r=rec32[0] + 2, g=rec32[0] + 2, b=rec32[0] + 2), edit(rec32, row_stride=rec32[3] + 2),
        edit(rec32, pixel_stride=2), edit(rec32, container=2),
    ]


def crop_all(lib, table, F, recs, size, off):
    n = len(recs)
    state = torch.from_numpy(np.asarray(recs, dtype=np.int32)).cuda()
    crops = torch.empty((n, size, size, 3), dtype=torch.uint8, device="cuda")
    _lib.check(lib.fear_crop_targets_rgb_u8(table.data_ptr(), F, state.data_ptr(), n, off, size, crops.data_ptr(),
                                            stream()), "fear_crop_targets_rgb_u8")
    return crops.cpu().numpy(), state.cpu().numpy()


def identity_crop(lib, frame, size):
    recs = np.zeros((1, _lib.TARGET_INTS), dtype=np.int32)
    recs[0, 3:5] = size
    return crop_all(lib, rgb_table([frame.rgb_record()]), 1, recs, size, 0.0)[0][0]


def random_codes(rng, shape, bits):
    return rng.integers(0, 1 << bits, shape).astype(code_dtype(bits))


# ---------------------------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("layout,bits", LAYOUTS, ids=[f"{k}-{b}" for k, b in LAYOUTS])
def test_identity_crop_equals_rgb_frame_to_rgb(layout, bits):
    """Whole frames cropped at their own size (box [0, 0, W, H], offset 0): a 256 x 256 region of interest of a pitched
    surface, a tight 255 x 255 frame (odd W) of extreme codes, and for x2rgb10 a torch.uint32 view; every pixel equals
    rgb_frame_to_rgb of the samples."""
    lib = _lib.init(0)
    rng = np.random.default_rng(len(layout) * 31 + bits)
    top = (1 << bits) - 1
    cases = [(random_codes(rng, (256, 256, 3), bits), dict(col=1, extra=5)),
             (rng.choice([0, 1, top - 1, top], (255, 255, 3)).astype(code_dtype(bits)), {})]
    if layout in image_ops.X2RGB10_LAYOUTS:
        cases.append((random_codes(rng, (256, 256, 3), bits), dict(col=3, extra=1, uint32=True)))
    if layout == "planar":
        cases.append((random_codes(rng, (255, 255, 3), bits), dict(chw=True)))
    for codes, kw in cases:
        frame, want = make_frame(codes, layout, bits, rng, **kw)
        assert frame.shape == codes.shape
        got = identity_crop(lib, frame, codes.shape[0])
        assert np.array_equal(got, want), (layout, bits, kw)
        if bits == 8:
            assert np.array_equal(want, codes)


def test_alpha_x_and_spare_bits_change_nothing():
    """The same codes with different random alpha / X samples, spare bits of x2rgb10 words and bits above planar codes
    give the same crops and sums."""
    lib = _lib.init(0)
    for layout, bits in LAYOUTS:
        if layout in ("rgb24", "bgr24", "rgb48le", "bgr48le") or (layout == "planar" and bits in (8, 16)):
            continue  # nothing spare to vary
        codes = random_codes(np.random.default_rng(5), (97, 131, 3), bits)
        frames = [make_frame(codes, layout, bits, np.random.default_rng(s))[0] for s in (1, 2)]
        crops = [identity_crop(lib, f, 97) for f in frames]  # the top-left 97 x 97 region, 1:1
        assert np.array_equal(crops[0], crops[1]), layout
        table = rgb_table([f.rgb_record() for f in frames])
        sums = torch.full((2, 3), -1, dtype=torch.int64, device="cuda")
        _lib.check(lib.fear_frame_sums_rgb_u8(table.data_ptr(), 2, sums.data_ptr(), stream()), "sums")
        got = sums.cpu().numpy()
        assert np.array_equal(got[0], got[1]), layout


# frame: (H, W), layout, bits, column offset, pitch extra -- tight, pitched, regions of interest, 1-pixel sides -- and
# plain CUDA RGB tensors ("tensor": a strided rgba[..., :3] view), as they share a call's table with RGBFrames
SHAPES = [((255, 480), "bgra", 8, 0, 32), ((183, 98), "rgb48le", 16, 1, 0), ((91, 334), "x2rgb10le", 10, 1, 3),
          ((1, 1), "bgr24", 8, 0, 0), ((64, 1283), "planar", 12, 2, 9), ((100, 203), "abgr", 8, 1, 3),
          ((1, 57), "x2bgr10le", 10, 0, 0), ((43, 1), "planar", 16, 0, 0), ((120, 160), "tensor", 8, 4, 2)]
TARGETS = [(0, [163, 53, 45, 174]), (0, [-10, 100, 40, 30]), (0, [450, 20, 60, 40]), (0, [200, -15, 30, 50]),
           (0, [0, 0, 3, 3]), (1, [-300, -200, 900, 500]), (1, [95, 180, 3, 3]), (2, [5, 40, 320, 20]),
           (2, [330, 87, 3, 3]), (3, [0, 0, 1, 1]), (3, [-20, -20, 40, 40]), (4, [1270, 30, 40, 40]),
           (4, [600, 10, 300, 50]), (5, [-1, -1, 205, 102]), (5, [100, 50, 50, 50]), (6, [0, 0, 57, 1]),
           (6, [20, -5, 10, 10]), (7, [0, 0, 1, 43]), (7, [-3, 10, 5, 5]), (8, [30, 20, 50, 60]),
           (8, [-40, 100, 120, 90]), (0, [2000, 900, 30, 30])]


def shape_frames(rng):
    frames, rgbs = [], []
    for (h, w), layout, bits, col, extra in SHAPES:
        codes = random_codes(rng, (h, w, 3), bits)
        if layout == "tensor":
            alpha = rng.integers(0, 256, (h, w, 1)).astype(np.uint8)
            frames.append(place(np.concatenate([codes, alpha], -1), col, extra)[..., :3])
            rgbs.append(codes)
            continue
        f, want = make_frame(codes, layout, bits, rng, col, extra)
        frames.append(f)
        rgbs.append(want)
    return frames, rgbs


def records_of(frames):
    table = np.zeros(len(frames), _lib.RGB_DTYPE)
    mt.write_records(table, frames, "rgb")
    return [tuple(r.tolist()) for r in table]


def bad_entries(records):
    return unreadable_records(records[0], records[1], records[2])


@pytest.mark.parametrize("size,off", [(256, 2.0), (128, 0.2)])
def test_general_crops_equal_cv2(size, off):
    """Targets inside, across and outside frames of every container and of a strided CUDA tensor, against the cv2 crop
    of the RGB frame; targets past F or on unreadable entries get their padding colour and keep their box."""
    lib = _lib.init(0)
    rng = np.random.default_rng(3)
    frames, rgbs = shape_frames(rng)
    records = records_of(frames)
    bad = bad_entries(records)
    table = rgb_table(records + bad)
    F = len(records) + len(bad)
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
        assert (got[len(TARGETS) + j] == np.array(pad, np.uint8)).all(), (j, f, pad)
        assert np.array_equal(state[len(TARGETS) + j, 1:5], [5, 5, 30, 30])


def test_advance_keeps_boxes_of_unreadable_entries():
    lib = _lib.init(0)
    rng = np.random.default_rng(5)
    frames, _ = shape_frames(rng)
    shapes = [s[0] for s in SHAPES]
    records = records_of(frames)
    bad = bad_entries(records)
    table = rgb_table(records + bad)
    nf = len(records)
    n = 12000
    boxes = np.zeros(n, dtype=_lib.BOX_DTYPE)
    boxes["x"], boxes["y"] = rng.uniform(-300, 600, n), rng.uniform(-300, 600, n)
    boxes["w"], boxes["h"] = rng.uniform(0, 400, n), rng.uniform(0, 400, n)
    recs = np.zeros((n, _lib.TARGET_INTS), dtype=np.int32)
    recs[:, 0] = rng.integers(0, nf, n)
    recs[:, 5:7] = rng.integers(-600, 700, (n, 2))
    recs[:, 7:9] = rng.integers(1, 2000, (n, 2))
    recs[-len(bad):, 0] = nf + np.arange(len(bad))
    kept = len(bad) + 4
    recs[-4 - len(bad):-len(bad), 0] = [-1, nf + len(bad), 9999, -2 ** 31]
    recs[-kept:, 1:5] = [7, 8, 9, 10]
    state = torch.from_numpy(recs).cuda()
    dboxes = torch.from_numpy(boxes.view(np.uint8).copy()).cuda()
    _lib.check(lib.fear_advance_targets_rgb(dboxes.data_ptr(), table.data_ptr(), nf + len(bad), state.data_ptr(), n,
                                            256, stream()), "fear_advance_targets_rgb")
    got = state.cpu().numpy()
    for i in range(n - kept):
        b = np.array([boxes["x"][i], boxes["y"][i], boxes["w"][i], boxes["h"][i]])
        h, w = shapes[recs[i, 0]]
        want = image_ops.clamp_bbox(image_ops.rescale_bbox(b, recs[i, 5:9], 256), (h, w, 3))
        assert np.array_equal(got[i, 1:5], want), (i, (h, w))
    assert (got[-kept:, 1:5] == [7, 8, 9, 10]).all()
    assert np.array_equal(np.delete(got, np.s_[1:5], axis=1), np.delete(recs, np.s_[1:5], axis=1))


def test_frame_sums_rgb_give_numpy_sums():
    """Sums up to 2160 x 3840 in every container, and 0 for unreadable entries."""
    lib = _lib.init(0)
    rng = np.random.default_rng(11)
    cases = [((1, 1), "bgr24", 8), ((3, 4), "rgba64le", 16), ((5, 3), "x2rgb10le", 10), ((183, 98), "planar", 10),
             ((37, 1005), "0bgr", 8), ((1080, 1920), "bgra", 8), ((1081, 1918), "x2bgr10le", 10),
             ((2160, 3840), "rgb48le", 16), ((2160, 3840), "planar", 12), ((2160, 3840), "bgra", 8)]
    frames, rgbs = [], []
    for (h, w), layout, bits in cases:
        f, want = make_frame(random_codes(rng, (h, w, 3), bits), layout, bits, rng, 1, 3)
        frames.append(f)
        rgbs.append(want)
    records = [f.rgb_record() for f in frames]
    bad = unreadable_records(records[5], records[1], records[2])
    table = rgb_table(records + bad)
    F = len(records) + len(bad)
    sums = torch.full((F, 3), -1, dtype=torch.int64, device="cuda")
    _lib.check(lib.fear_frame_sums_rgb_u8(table.data_ptr(), F, sums.data_ptr(), stream()), "fear_frame_sums_rgb_u8")
    got = sums.cpu().numpy().view(np.uint64)
    for i, rgb in enumerate(rgbs):
        assert np.array_equal(got[i], rgb.sum(axis=(0, 1), dtype=np.uint64)), (i, cases[i])
        assert np.array_equal(got[i] / (rgb.shape[0] * rgb.shape[1]), np.mean(rgb, axis=(0, 1)))
    assert (got[len(records):] == 0).all()


def test_c_abi_rejects_bad_arguments_and_launches_nothing():
    lib = _lib.init(0)
    t = torch.full((1 << 16,), 0x5A, dtype=torch.uint8, device="cuda")
    p = t.data_ptr()
    good = dict(views=p, F=1, targets=p, N=1, offset=2.0, size=256, crops=p)

    def crop(**kw):
        a = dict(good, **kw)
        return lib.fear_crop_targets_rgb_u8(a["views"], a["F"], a["targets"], a["N"], a["offset"], a["size"],
                                            a["crops"], None)

    for kw in [dict(views=None), dict(targets=None), dict(crops=None), dict(N=0), dict(N=-1), dict(N=65536),
               dict(F=0), dict(F=-3), dict(size=0), dict(size=257), dict(offset=-0.5), dict(offset=float("nan")),
               dict(offset=float("inf"))]:
        assert crop(**kw) == -1, kw
        assert _lib.last_error(), kw
    for args in [(None, p, 1, p, 1, 256), (p, None, 1, p, 1, 256), (p, p, 1, None, 1, 256), (p, p, 1, p, 0, 256),
                 (p, p, 0, p, 1, 256), (p, p, 1, p, 1, 0)]:
        assert lib.fear_advance_targets_rgb(*args, None) == -1, args
    for args in [(None, 1, p), (p, 1, None), (p, 0, p), (p, 65536, p), (p, -1, p)]:
        assert lib.fear_frame_sums_rgb_u8(*args, None) == -1, args
        assert _lib.last_error(), args
    torch.cuda.synchronize()
    assert (t == 0x5A).all()


# ---------------------------------------------------------------------------------------------------- RGBFrame
def _dev(*shape, dtype=torch.uint8):
    return torch.zeros(shape, dtype=dtype, device="cuda")


def test_rgb_frame_records_its_samples():
    surf = _dev(8, 2000, 4)
    p = surf.data_ptr()
    f = fb.RGBFrame(surf[1:7, 3:1923], "bgra")
    assert f.shape == (6, 1920, 3)
    assert f.rgb_record() == (p + 8012 + 2, p + 8012 + 1, p + 8012, 8000, 4, 6, 1920, 1, 8, 0, 0, 0, 0)
    assert fb.RGBFrame(surf, "argb").rgb_record()[:3] == (p + 1, p + 2, p + 3)
    assert fb.RGBFrame(surf, "0bgr").rgb_record()[:3] == (p + 3, p + 2, p + 1)
    assert fb.RGBFrame(_dev(1, 1, 3), "bgr24").rgb_record()[3:] == (3, 3, 1, 1, 1, 8, 0, 0, 0, 0)
    s16 = _dev(4, 10, 4, dtype=torch.uint16)
    q = s16.data_ptr()
    assert fb.RGBFrame(s16[:, 2:], "bgra64le").rgb_record() == (q + 20, q + 18, q + 16, 80, 8, 4, 8, 2, 16, 0, 0, 0, 0)
    words = _dev(5, 64, dtype=torch.int32)
    w = words.data_ptr()
    assert fb.RGBFrame(words[1:, :60], "x2rgb10le").rgb_record() == (w + 256, w + 256, w + 256, 256, 4, 4, 60, 4, 10,
                                                                       20, 10, 0, 0)
    assert fb.RGBFrame(words.view(torch.uint32), "x2bgr10le").rgb_record()[9:12] == (0, 10, 20)
    chw = _dev(3, 6, 7, dtype=torch.uint16)
    c = chw.data_ptr()
    f = fb.RGBFrame.planar(*chw, bits=16)
    assert f.shape == (6, 7, 3) and f.rgb_record() == (c, c + 84, c + 168, 14, 2, 6, 7, 2, 16, 0, 0, 0, 0)
    gbrp = _dev(3, 6, 8)  # ffmpeg's gbrp: data[0] G, data[1] B, data[2] R
    g = gbrp.data_ptr()
    assert fb.RGBFrame.planar(gbrp[2], gbrp[0], gbrp[1]).rgb_record()[:3] == (g + 96, g, g + 48)


BAD_RGB = {
    "0 rows": lambda: fb.RGBFrame(_dev(0, 8, 3), "bgr24"),
    "0 columns": lambda: fb.RGBFrame(_dev(8, 0, 4), "bgra"),
    "4 channels as bgr24": lambda: fb.RGBFrame(_dev(8, 8, 4), "bgr24"),
    "3 channels as bgra": lambda: fb.RGBFrame(_dev(8, 8, 3), "bgra"),
    "uint16 as bgra": lambda: fb.RGBFrame(_dev(8, 8, 4, dtype=torch.uint16), "bgra"),
    "uint8 as rgb48le": lambda: fb.RGBFrame(_dev(8, 8, 3), "rgb48le"),
    "int16 as rgb48le": lambda: fb.RGBFrame(_dev(8, 8, 3, dtype=torch.int16), "rgb48le"),
    "2-D as bgr24": lambda: fb.RGBFrame(_dev(8, 24), "bgr24"),
    "unknown layout": lambda: fb.RGBFrame(_dev(8, 8, 3), "bgr"),
    "ffmpeg name of planar": lambda: fb.RGBFrame(_dev(8, 8, 3), "gbrp"),
    "channel stride 2": lambda: fb.RGBFrame(_dev(8, 8, 6)[..., ::2], "bgr24"),
    "pixel stride 4 for bgr24": lambda: fb.RGBFrame(_dev(8, 8, 4)[..., :3], "bgr24"),
    "planar chw as bgr24": lambda: fb.RGBFrame(_dev(3, 8, 8).permute(1, 2, 0), "bgr24"),
    "rows overlap": lambda: fb.RGBFrame(_dev(8, 16, 3).as_strided((8, 16, 3), (24, 3, 1)), "bgr24"),
    "misaligned uint16": lambda: fb.RGBFrame(_dev(8, 8 * 6 + 1)[:, 1:].view(torch.uint16).view(8, 8, 3), "rgb48le"),
    "int64 words": lambda: fb.RGBFrame(_dev(8, 8, dtype=torch.int64), "x2rgb10le"),
    "uint16 words": lambda: fb.RGBFrame(_dev(8, 8, dtype=torch.uint16), "x2rgb10le"),
    "3-D words": lambda: fb.RGBFrame(_dev(8, 8, 1, dtype=torch.int32), "x2rgb10le"),
    "strided words": lambda: fb.RGBFrame(_dev(8, 16, dtype=torch.int32)[:, ::2], "x2rgb10le"),
    "misaligned words": lambda: fb.RGBFrame(_dev(8, 35)[:, 1:33].view(torch.int32), "x2rgb10le"),
    "planar bits 9": lambda: fb.RGBFrame.planar(_dev(8, 8), _dev(8, 8), _dev(8, 8), bits=9),
    "planar uint8 at 10 bits": lambda: fb.RGBFrame.planar(_dev(8, 8), _dev(8, 8), _dev(8, 8), bits=10),
    "planar uint16 at 8 bits": lambda: fb.RGBFrame.planar(*_dev(3, 8, 8, dtype=torch.uint16)),
    "planar shapes differ": lambda: fb.RGBFrame.planar(_dev(8, 8), _dev(8, 8), _dev(8, 9)),
    "planar dtypes differ": lambda: fb.RGBFrame.planar(_dev(8, 8, dtype=torch.uint16), _dev(8, 8),
                                                       _dev(8, 8, dtype=torch.uint16), bits=16),
    "planar strides differ": lambda: fb.RGBFrame.planar(_dev(8, 8), _dev(8, 16)[:, :8], _dev(8, 8)),
    "planar 3-D": lambda: fb.RGBFrame.planar(_dev(8, 8, 1), _dev(8, 8, 1), _dev(8, 8, 1)),
    "planar 0 rows": lambda: fb.RGBFrame.planar(_dev(0, 8), _dev(0, 8), _dev(0, 8)),
}


@pytest.mark.parametrize("what", list(BAD_RGB))
def test_rgb_frame_refuses_malformed_tensors(what):
    with pytest.raises((ValueError, RuntimeError)) as e:
        BAD_RGB[what]()
    if not what.startswith("misaligned"):  # torch itself may refuse those views
        assert e.type is ValueError


def test_tracker_refuses_rgb_frames_mixed_with_other_kinds(net):
    trk = fb.FEARMultiTracker(net, cuda_id=0, max_targets=4, **CFG)
    f = fb.RGBFrame(_dev(64, 80, 4), "bgra")
    nv12 = fb.YUV420Frame.nv12(_dev(96, 80))
    mono = fb.MonoFrame(_dev(64, 80))
    bayer = fb.BayerFrame(_dev(64, 80))
    for frames in ([f, np.zeros((64, 80, 3), np.uint8)], [nv12, f], [f, _dev(64, 80, 3), nv12]):
        with pytest.raises(ValueError, match="RGBFrames can share a call only with CUDA"):
            trk.add(frames, [[1, 1, 20, 20]])
    with pytest.raises(ValueError, match="MonoFrames cannot share"):
        trk.add([f, mono], [[1, 1, 20, 20]])
    with pytest.raises(ValueError, match="BayerFrames cannot share"):
        trk.add([bayer, f, mono], [[1, 1, 20, 20]])
    other = torch.zeros((64, 80, 4), dtype=torch.uint8)  # a host tensor behind an RGBFrame's checks
    with pytest.raises(ValueError):
        trk.add([f, fb.RGBFrame(other.cuda(), "bgra"), other[..., :3]], [[1, 1, 20, 20]])
    assert len(trk) == 0


# ---------------------------------------------------------------------------------------------------- trackers
def codes_of(rgb: np.ndarray, bits: int) -> np.ndarray:
    """8-bit RGB as ``bits``-bit codes, rounded to the nearest code."""
    if bits == 8:
        return rgb
    return ((rgb.astype(np.int64) * ((1 << bits) - 1) + 127) // 255).astype(np.uint16)


# stream: layout, bits, column offset, pitch extra, options of make_frame
STREAMS = [("bgr24", 8, 0, 0, {}), ("bgra", 8, 2, 64, {}), ("abgr", 8, 0, 0, {}), ("x2rgb10le", 10, 1, 32, {}),
           ("x2bgr10le", 10, 0, 0, {"uint32": True}), ("rgb48le", 16, 3, 16, {}), ("rgba64le", 16, 0, 0, {}),
           ("planar", 10, 0, 0, {}), ("planar", 12, 1, 8, {}), ("planar", 16, 0, 0, {"chw": True})]


def hd(clip, t):
    return cv2.resize(clip[t], (1920, 1080))


def stream_frames(clip, t, rng, streams=None):
    """The RGBFrames of update ``t`` of ``streams`` (default: all) and the numpy RGB frames they stand for."""
    out = []
    rgb = hd(clip, t)
    for s in (range(len(STREAMS)) if streams is None else streams):
        layout, bits, col, extra, kw = STREAMS[s]
        out.append(make_frame(codes_of(rgb, bits), layout, bits, rng, col, extra, **kw))
    return [f for f, _ in out], [w for _, w in out]


def _net():
    n = fb.FEARNet(**fb.FEAR_XS_MODEL_KWARGS)
    n.load_state_dict(load_full_state(), strict=True)
    return n.cuda().eval()


def test_multi_tracker_on_rgb_frames_matches_numpy_rgb(clip):
    """Ten 1080p streams, one per layout family (BGR, BGRA, ABGR, x2rgb10, x2bgr10 as uint32, rgb48, rgba64, planar 10
    / 12 bits, a (3, H, W) uint16 tensor), with add / remove part way, a call mixing RGBFrames with CUDA tensors (the
    same graph), a call on CUDA tensors alone (the views table, then a new graph back on the rgb table) and the net's
    workspace growing.  Every output equals a tracker fed the RGB frames as numpy arrays; a step is 48 launches."""
    T = 24
    rng = np.random.default_rng(97)
    n2 = _net()
    ref = fb.FEARMultiTracker(n2, cuda_id=0, max_targets=16, **CFG)
    trk = fb.FEARMultiTracker(n2, cuda_id=0, max_targets=16, **CFG)
    start = [[[652, 211, 180, 696]], [[900, 400, 120, 300]], [[0, 0, 60, 60]], [[1700, 840, 160, 224]],
             [[600, 200, 200, 600]], [[1800, 1000, 120, 80]], [[300, 100, 300, 500]], [[640, 300, 160, 400]],
             [[1000, 500, 90, 90]], [[620, 220, 190, 640], [50, 900, 100, 100]]]
    late = [[[400, 600, 120, 120]], [], [[100, 150, 30, 30]], [], [], [], [], [], [], []]

    def rects(d):
        return [r for s in d for r in s], [k for k, s in enumerate(d) for _ in s]

    frames, rgbs = stream_frames(clip, 0, rng)
    r, s = rects(start)
    assert np.array_equal(trk.add(frames, r, s), ref.add(rgbs, r, s))
    graphs = []
    for t in range(1, T + 1):
        if t == 12:
            r, s = rects(late)
            frames, rgbs = stream_frames(clip, t - 1, rng)
            assert np.array_equal(trk.add(frames, r, s), ref.add(rgbs, r, s))
        if t == 18:
            for x in (ref, trk):
                x.remove([1, 2, 11])
        if t == 21:
            gen = n2.generation()
            zt, xt, _, _ = fo.synthetic_crops(20)
            n2.track(xt.cuda(), n2.get_features(zt.cuda()))  # batch 20 > reserved 16: the workspace grows
            assert n2.generation() != gen
        frames, rgbs = stream_frames(clip, t, rng)
        if t == 6:  # RGBFrames and CUDA tensors in one call: the rgb table, the same graph
            rgba = np.concatenate([rgbs[5], rgbs[5][..., :1]], -1)
            frames[0], frames[5] = torch.from_numpy(rgbs[0]).cuda(), torch.from_numpy(rgba).cuda()[..., :3]
        if t == 8:  # CUDA tensors alone: the views table
            frames = [torch.from_numpy(x).cuda() for x in rgbs]
        expect, out = ref.update(rgbs), trk.update(frames)
        assert trk._graph_key[2] == ("views" if t == 8 else "rgb"), t
        assert np.array_equal(out["ids"], expect["ids"]), t
        assert np.array_equal(out["bbox"], expect["bbox"]), (t, out["bbox"], expect["bbox"])
        assert np.array_equal(out["score"], expect["score"]), t
        if t in (3, 10, 14, 20, 23):  # two updates after the start, the switch back, add, remove, growth
            assert trk._graph is not None and all(trk._graph is not g for g in graphs), t
            graphs.append(trk._graph)
        if t in (6, 7, 11, 17, 24):  # replayed with new frame addresses every update, mixed call included
            assert trk._graph is graphs[-1], t
    # the step's launches: the crop and advance entry points around the network's own
    eager = fb.FEARMultiTracker(n2, cuda_id=0, max_targets=16, cuda_graph=False, **CFG)
    frames, _ = stream_frames(clip, 0, rng)
    eager.add(frames, [[600, 200, 200, 300]] * len(frames), list(range(len(frames))))
    eager.update(stream_frames(clip, 1, rng)[0])
    torch.cuda.synchronize()
    c0 = n2.launch_count()
    eager.update(stream_frames(clip, 2, rng)[0])
    assert n2.launch_count() - c0 + 2 == 48


def test_multi_tracker_at_instance_size_192(clip):
    cfg = dict(CFG, instance_size=192, score_size=12)
    n2 = _net()
    rng = np.random.default_rng(7)
    ref = fb.FEARMultiTracker(n2, cuda_id=0, max_targets=4, **cfg)
    trk = fb.FEARMultiTracker(n2, cuda_id=0, max_targets=4, **cfg)
    streams = [1, 3, 9]
    frames, rgbs = stream_frames(clip, 0, rng, streams)
    rects = [[652, 211, 180, 696], [900, 400, 120, 300], [600, 200, 200, 600]]
    assert np.array_equal(trk.add(frames, rects, [0, 1, 2]), ref.add(rgbs, rects, [0, 1, 2]))
    for t in range(1, 9):
        frames, rgbs = stream_frames(clip, t, rng, streams)
        out, expect = trk.update(frames), ref.update(rgbs)
        for k in ("ids", "bbox", "score"):
            assert np.array_equal(out[k], expect[k]), (t, k)


@pytest.mark.parametrize("smooth", [False, True], ids=["plain", "smooth"])
def test_fear_tracker_on_rgb_frames_matches_numpy_rgb(net, clip, smooth):
    """FEARTracker on streams of several layouts (graphed, eager, and with gpu_crop), with a numpy frame and a CUDA
    tensor part way, gives the trajectory and tracking_state of the same tracker on the RGB frames as numpy arrays;
    templates made from RGBFrames equal those made from numpy frames."""
    T = 18
    rng = np.random.default_rng(61)
    init = np.array([600, 200, 200, 600])
    for extra in ({}, {"cuda_graph": False}, {"gpu_crop": True}):
        cfg = dict(CFG, smooth=smooth, **extra)
        ref, trk = fb.FEARTracker(net, cuda_id=0, **cfg), fb.FEARTracker(net, cuda_id=0, **cfg)
        frames, rgbs = stream_frames(clip, 0, rng, [1])
        ref.initialize(rgbs[0], init)
        trk.initialize(frames[0], init)
        assert np.array_equal(trk.tracking_state.mean_color, ref.tracking_state.mean_color)
        for t in range(1, T + 1):
            s = 1 if t < 6 else (3 if t < 10 else (5 if t < 13 else 9))
            frames, rgbs = stream_frames(clip, t, rng, [s])
            want = ref.update(rgbs[0])["bbox"]
            frame = rgbs[0] if t == 7 else (torch.from_numpy(rgbs[0]).cuda() if t == 11 else frames[0])
            got = trk.update(frame)["bbox"]
            assert np.array_equal(got, want), (smooth, extra, t, got, want)
            for key in ("bbox", "mapping", "prev_size"):
                assert np.array_equal(getattr(trk.tracking_state, key), getattr(ref.tracking_state, key)), (key, t)
        assert [list(p) for p in trk.tracking_state.paths] == [list(p) for p in ref.tracking_state.paths]
        for s in (4, 8):
            frames, rgbs = stream_frames(clip, 3, rng, [s])
            z_ref = ref.get_template_features(rgbs[0], [600, 200, 100, 300])
            z_trk = trk.get_template_features(frames[0], [600, 200, 100, 300])
            assert torch.equal(z_ref, z_trk), s


def test_fear_tracker_at_instance_size_192(net, clip):
    cfg = dict(CFG, instance_size=192, score_size=12)
    rng = np.random.default_rng(8)
    ref, trk = fb.FEARTracker(net, cuda_id=0, **cfg), fb.FEARTracker(net, cuda_id=0, **cfg)
    frames, rgbs = stream_frames(clip, 0, rng, [6])
    ref.initialize(rgbs[0], [600, 200, 200, 600])
    trk.initialize(frames[0], [600, 200, 200, 600])
    for t in range(1, 9):
        frames, rgbs = stream_frames(clip, t, rng, [6])
        assert np.array_equal(trk.update(frames[0])["bbox"], ref.update(rgbs[0])["bbox"]), t


# ---------------------------------------------------------------------------------------------------- poison
def test_rgb_entry_points_and_trackers_on_poisoned_memory():
    """tests/poison_rgb_check.py in its own process: guarded, poisoned tables, crops, sums, boxes and frames."""
    proc = subprocess.run([sys.executable, os.path.join(HERE, "poison_rgb_check.py")], capture_output=True, text=True,
                          timeout=1200)
    lines = [l for l in proc.stdout.splitlines() if l.startswith("POISON_CHECK ")]
    assert proc.returncode == 0 and lines, f"poison_rgb_check failed: {proc.stderr[-3000:]}"
    res = json.loads(lines[-1][len("POISON_CHECK "):])
    assert res["checked_calls"] > 0
    assert res["n_failures"] == 0, res["failures"]
