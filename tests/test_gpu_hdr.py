"""GPU tests of HDR frames: the FearFrameYCbCrHDR entry points (fear_crop_targets_ycbcr_hdr_u8,
fear_advance_targets_ycbcr_hdr, fear_frame_sums_ycbcr_hdr_u8), the frames' ``transfer``, and FEARMultiTracker /
FEARTracker fed PQ and HLG video.

The conversion is compared with image_ops.yuv_to_rgb(..., transfer=...) (pinned on the CPU by tests/test_hdr_cpu.py)
under one rule: equal, except that an output may differ by exactly 1 where numpy's 255 * v before rounding lies within
1e-9 of k + 1/2 (CUDA's exp / log / pow may differ from numpy's in the last ulp).  The tests count those cases and
print the count.  Everything downstream of the conversion (crops, boxes, sums, trajectories) is compared exactly, on
frames whose conversion was first checked to be exact."""
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
from tests.hdr_frames import SHIFTS, hdr_codes, i420_frame, p010_frame, v210_frame
from tests.helpers import GOLDEN, load_full_state
from tests.test_yuv_subsampling_cpu import ycbcr_frame

pytestmark = pytest.mark.gpu
CFG = fb.FEAR_XS_TRACKER_KWARGS
HERE = os.path.dirname(os.path.abspath(__file__))
TIES = {"count": 0}  # outputs that differ by 1 at a k + 1/2 tie of numpy's value, over the whole module


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


def hdr_table(records) -> torch.Tensor:
    return torch.from_numpy(np.array(records, dtype=_lib.YCBCR_HDR_DTYPE).view(np.uint8).copy()).cuda()


def unit_values(y, u, v, sub, full, bits, transfer):
    """numpy's 255 * v before rounding, (H, W, 3), for the exactness rule."""
    sx, sy = SHIFTS[sub]
    U, V = (np.asarray(c).repeat(1 << sy, 0).repeat(1 << sx, 1) for c in (u, v))
    rgb = image_ops.h273_rgb(np.asarray(y), U, V, "bt2020", full, bits)
    return np.stack([255.0 * c for c in image_ops.hdr_to_sdr_unit(rgb, transfer)], -1)


def assert_conversion(got, want, y, u, v, sub, full, bits, transfer, what):
    """The exactness rule: equal, or off by exactly 1 where numpy's 255 * v is within 1e-9 of k + 1/2."""
    diff = got.astype(np.int32) - want.astype(np.int32)
    bad = diff != 0
    if not bad.any():
        return
    idx = np.argwhere(bad.any(-1))
    units = unit_values(y[idx[:, 0], idx[:, 1]][None], *(unit_sample(c, idx, sub) for c in (u, v)),
                        "444", full, bits, transfer)[0]
    d = diff[idx[:, 0], idx[:, 1]]
    tie = np.abs(units - np.floor(units) - 0.5) <= 1e-9
    ok = (d == 0) | ((np.abs(d) == 1) & tie)
    assert ok.all(), (what, idx[~ok.all(-1)][:5].tolist(), d[~ok.all(-1)][:5].tolist())
    TIES["count"] += int((d != 0).sum())
    print(f"{what}: {int((d != 0).sum())} outputs off by 1 at a k + 1/2 tie")


def unit_sample(c, idx, sub):
    sx, sy = SHIFTS[sub]
    return np.asarray(c)[idx[:, 0] >> sy, idx[:, 1] >> sx][None]


def identity_crops(frame, h, w):
    """The frame cropped 1:1 in 256 x 256 tiles (H and W multiples of 256) through the HDR crop entry point."""
    lib = _lib.init(0)
    table = hdr_table([frame.hdr_record()])
    ty, tx = h // 256, w // 256
    recs = np.zeros((ty * tx, _lib.TARGET_INTS), dtype=np.int32)
    recs[:, 1] = 256 * np.tile(np.arange(tx), ty)
    recs[:, 2] = 256 * np.repeat(np.arange(ty), tx)
    recs[:, 3:5] = 256
    state = torch.from_numpy(recs).cuda()
    crops = torch.empty((ty * tx, 256, 256, 3), dtype=torch.uint8, device="cuda")
    _lib.check(lib.fear_crop_targets_ycbcr_hdr_u8(table.data_ptr(), 1, state.data_ptr(), ty * tx, 0.0, 256,
                                                  crops.data_ptr(), stream()), "fear_crop_targets_ycbcr_hdr_u8")
    return crops.cpu().numpy().reshape(ty, tx, 256, 256, 3).transpose(0, 2, 1, 3, 4).reshape(h, w, 3)


# ---------------------------------------------------------------------------------------------------- conversion
@pytest.mark.parametrize("transfer", ["pq", "hlg"])
@pytest.mark.parametrize("bits", [10, 12])
@pytest.mark.parametrize("full", [False, True], ids=["limited", "full"])
def test_conversion_of_every_code_pair_and_random_triples(transfer, bits, full):
    """4:4:4 frames of every (Y, U) pair (V seeded) and every (Y, V) pair (U seeded) at 10 bits, and 2^22 seeded
    triples at both depths, against yuv_to_rgb by the exactness rule.  (At 12 bits the 2^25 pairs would take the numpy
    side minutes per case; every 12-bit Y code is in the triples' luma, which runs over the whole range.)"""
    rng = np.random.default_rng(bits * 10 + full + (transfer == "hlg") * 100)
    top = 1 << bits
    planes = []
    if bits == 10:
        yy, cc = np.meshgrid(np.arange(top), np.arange(top), indexing="ij")
        other = rng.integers(0, top, yy.shape)
        planes += [(yy, cc, other), (yy, other, cc)]
    n = 1 << 22
    planes.append((np.tile(np.arange(top), n // top), rng.integers(0, top, n), rng.integers(0, top, n)))
    for k, (y, u, v) in enumerate(planes):
        y, u, v = (np.asarray(p).reshape(-1, 2048) for p in (y, u, v))
        h, w = y.shape
        frame = ycbcr_frame(y, u, v, "i444", bits, rng=rng, matrix="bt2020", full_range=full, transfer=transfer)
        got = identity_crops(frame, h, w)
        want = image_ops.yuv_to_rgb(y, u, v, "bt2020", full, bits, 0, (0, 0), transfer)
        assert_conversion(got, want, y, u, v, "444", full, bits, transfer, f"{transfer} {bits} full={full} set {k}")


LAYOUTS = [("p010", "420"), ("i420", "420"), ("nv16", "422"), ("i422", "422"), ("yuyv_pitched", "422"),
           ("i444_msb_pitched", "444"), ("v210", "422")]


@pytest.mark.parametrize("layout,sub", LAYOUTS, ids=[l[0] for l in LAYOUTS])
@pytest.mark.parametrize("bits", [10, 12])
@pytest.mark.parametrize("transfer", ["pq", "hlg"])
def test_conversion_in_every_layout(layout, sub, bits, transfer):
    """MSB- and LSB-aligned samples, 4:2:0, 4:2:2, 4:4:4 and v210, limited and full range, seeded codes."""
    if layout == "v210" and bits == 12:
        pytest.skip("v210 is 10-bit")
    rng = np.random.default_rng(len(layout) * 31 + bits + (transfer == "hlg"))
    h, w = 512, 1024
    sx, sy = SHIFTS[sub]
    for full in (False, True):
        y = rng.integers(0, 1 << bits, (h, w))
        u, v = rng.integers(0, 1 << bits, (2, h >> sy, w >> sx))
        fmt = dict(matrix="bt2020", full_range=full, transfer=transfer)
        if layout == "p010":
            frame = p010_frame(y, u, v, bits, **fmt)
        elif layout == "i420":
            frame = i420_frame(y, u, v, bits, **fmt)
        elif layout == "v210":
            frame = v210_frame(y, u, v, col=8, **fmt)
        else:
            frame = ycbcr_frame(y, u, v, layout, bits, rng=rng, **fmt)
        got = identity_crops(frame, h, w)
        want = image_ops.yuv_to_rgb(y, u, v, "bt2020", full, bits, 0, (sx, sy), transfer)
        assert_conversion(got, want, y, u, v, sub, full, bits, transfer, f"{layout} {bits} {transfer} full={full}")


# ---------------------------------------------------------------------------------------------------- kernels
def kernel_frames(rng):
    """Five HDR frames of several layouts and sizes, and their converted RGB frames (image_ops.yuv_to_rgb)."""
    specs = [((256, 480), "p010", "pq", 10, False), ((183, 98), "nv16", "hlg", 12, True),
             ((91, 334), "v210", "hlg", 10, False), ((64, 1282), "i444_msb_pitched", "pq", 12, True),
             ((256, 480), "roi422", "hlg", 10, False)]
    frames, rgbs = [], []
    for (h, w), layout, transfer, bits, full in specs:
        sub = "420" if layout == "p010" else "444" if "444" in layout else "422"
        sx, sy = SHIFTS[sub]
        y, (u, v) = rng.integers(0, 1 << bits, (h, w)), rng.integers(0, 1 << bits, (2, h >> sy, w >> sx))
        fmt = dict(matrix="bt2020", full_range=full, transfer=transfer)
        f = p010_frame(y, u, v, bits, **fmt) if layout == "p010" else v210_frame(y, u, v, col=4, **fmt) \
            if layout == "v210" else ycbcr_frame(y, u, v, layout, bits, rng=rng, **fmt)
        frames.append(f)
        rgbs.append(image_ops.yuv_to_rgb(y, u, v, "bt2020", full, bits, 0, (sx, sy), transfer))
    return frames, rgbs


def unreadable_records(pq_rec, sdr8_rec):
    """Entries the kernels must treat as empty: transfers other than 0, 16 and 18, an HDR transfer with the BT.709 or
    BT.601 matrix or at 8 bits, and a v210 field of 2 (FearFrameYCbCrV210's own rules)."""
    out = []
    for field, value in ((17, 1), (17, 17), (17, -1), (17, 14), (9, 1), (9, 0), (15, 2)):
        r = list(pq_rec)
        r[field] = value
        out.append(tuple(r))
    for t in (16, 18):
        r = list(sdr8_rec)
        r[17] = t
        out.append(tuple(r))
    return out


TARGETS = [(0, [163, 53, 45, 174]), (0, [-10, 100, 40, 30]), (0, [450, 20, 60, 40]), (1, [0, 0, 3, 3]),
           (1, [-300, -200, 900, 500]), (2, [330, 87, 3, 3]), (2, [5, 40, 320, 20]), (3, [1270, 30, 40, 40]),
           (3, [600, 10, 300, 50]), (4, [100, 100, 200, 120]), (4, [2000, 900, 30, 30])]


def test_crops_match_cv2_on_the_converted_frame_and_unreadable_entries_pad():
    lib = _lib.init(0)
    rng = np.random.default_rng(7)
    frames, rgbs = kernel_frames(rng)
    means = [np.mean(f, axis=(0, 1)) for f in rgbs]
    sdr8 = fb.YUV420Frame.nv12(torch.zeros((96, 80), dtype=torch.uint8, device="cuda"), matrix="bt2020")
    records = [f.hdr_record() for f in frames]
    bad = unreadable_records(records[0], sdr8.hdr_record())
    extra = [(9999, [12, 200, 255]), (-1, [1, 2, 3])] + [(len(records) + i, [i, 128, 7]) for i in range(len(bad))]
    recs = np.zeros((len(TARGETS) + len(extra), _lib.TARGET_INTS), dtype=np.int32)
    for i, (f, box) in enumerate(TARGETS):
        recs[i, 0], recs[i, 1:5], recs[i, 9:12] = f, box, np.clip(np.rint(means[f]), 0, 255)
    for i, (f, pad) in enumerate(extra):
        recs[len(TARGETS) + i, 0], recs[len(TARGETS) + i, 1:5], recs[len(TARGETS) + i, 9:12] = f, [10, 10, 20, 20], pad
    table = hdr_table(records + bad)
    n = len(recs)
    for size, off in ((256, 2.0), (128, 0.2)):
        state = torch.from_numpy(recs).cuda()
        crops = torch.empty((n, size, size, 3), dtype=torch.uint8, device="cuda")
        _lib.check(lib.fear_crop_targets_ycbcr_hdr_u8(table.data_ptr(), len(records) + len(bad), state.data_ptr(), n,
                                                      off, size, crops.data_ptr(), stream()), "crop")
        got, ctxs = crops.cpu().numpy(), state.cpu().numpy()[:, 5:9]
        for i, (f, box) in enumerate(TARGETS):
            assert np.array_equal(ctxs[i], image_ops.context_box(box, off)), (size, box)
            assert np.array_equal(got[i], base._cv2_crop(rgbs[f], box, size, off, means[f])), (size, off, f, box)
        for i, (_, pad) in enumerate(extra):
            assert (got[len(TARGETS) + i] == np.array(pad, dtype=np.uint8)).all(), (size, i)


def test_transfer_0_entries_equal_the_v210_entry_points():
    """SDR frames of every kind (planar 8 / 10 / 12-bit, every matrix, and v210) through the HDR entry points with
    transfer 0 give bit-identical crops, advances and sums to the *_ycbcr_v210 ones."""
    lib = _lib.init(0)
    rng = np.random.default_rng(43)
    frames = []
    for (h, w), layout, b, m, f, sx in [((255, 480), "yuyv_pitched", 8, "bt601", False, 1),
                                        ((183, 98), "nv16", 10, "bt2020", False, 1),
                                        ((90, 334), "i444_pitched", 12, "bt2020", True, 0),
                                        ((256, 480), "planes444", 10, "bt709", False, 0)]:
        frames.append(ycbcr_frame(rng.integers(0, 1 << b, (h, w)), rng.integers(0, 1 << b, (h, w >> sx)),
                                  rng.integers(0, 1 << b, (h, w >> sx)), layout, b, rng=rng, matrix=m, full_range=f))
    frames.append(v210_frame(rng.integers(0, 1024, (120, 300)), *rng.integers(0, 1024, (2, 120, 150)), col=4,
                             matrix="bt2020"))
    old = torch.from_numpy(np.array([f.ycbcr_v210_record() for f in frames], dtype=_lib.YCBCR_V210_DTYPE)
                           .view(np.uint8).copy()).cuda()
    new = hdr_table([f.hdr_record() for f in frames])
    F, n = len(frames), 1000
    recs = np.zeros((n, _lib.TARGET_INTS), dtype=np.int32)
    recs[:, 0] = rng.integers(-1, F + 1, n)
    recs[:, 1:3] = rng.integers(-300, 600, (n, 2))
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
            ("v210", old, lib.fear_crop_targets_ycbcr_v210_u8, lib.fear_advance_targets_ycbcr_v210,
             lib.fear_frame_sums_ycbcr_v210_u8),
            ("hdr", new, lib.fear_crop_targets_ycbcr_hdr_u8, lib.fear_advance_targets_ycbcr_hdr,
             lib.fear_frame_sums_ycbcr_hdr_u8)):
        state = torch.from_numpy(recs).cuda()
        crops = torch.empty((n, 256, 256, 3), dtype=torch.uint8, device="cuda")
        s = torch.empty((F, 3), dtype=torch.int64, device="cuda")
        _lib.check(crop(table.data_ptr(), F, state.data_ptr(), n, 2.0, 256, crops.data_ptr(), stream()), name)
        _lib.check(adv(dboxes.data_ptr(), table.data_ptr(), F, state.data_ptr(), n, 256, stream()), name)
        _lib.check(sums(table.data_ptr(), F, s.data_ptr(), stream()), name)
        out[name] = (crops.cpu().numpy(), state.cpu().numpy(), s.cpu().numpy())
    for a, b in zip(out["v210"], out["hdr"]):
        assert np.array_equal(a, b)


def test_advance_matches_host_rescale_and_clamp():
    """12 000 records on HDR frames of three sizes; unreadable entries and out-of-range indices keep their boxes."""
    lib = _lib.init(0)
    rng = np.random.default_rng(5)
    frames = [p010_frame(rng.integers(0, 1024, (h, w)), *rng.integers(0, 1024, (2, h // 2, w // 2)),
                         matrix="bt2020", transfer="pq") for h, w in ((256, 480), (184, 98), (2, 2))]
    shapes = [(256, 480), (184, 98), (2, 2)]
    sdr8 = fb.YUV420Frame.nv12(torch.zeros((96, 80), dtype=torch.uint8, device="cuda"), matrix="bt2020")
    records = [f.hdr_record() for f in frames]
    bad = unreadable_records(records[0], sdr8.hdr_record())
    table = hdr_table(records + bad)
    n = 12000
    boxes = np.zeros(n, dtype=_lib.BOX_DTYPE)
    recs = np.zeros((n, _lib.TARGET_INTS), dtype=np.int32)
    recs[:, 0] = rng.integers(0, 3, n)
    recs[:, 5:7] = rng.integers(-600, 700, (n, 2))
    recs[:, 7:9] = rng.integers(1, 2000, (n, 2))
    boxes["x"], boxes["y"] = rng.uniform(-300, 600, n), rng.uniform(-300, 600, n)
    boxes["w"], boxes["h"] = rng.uniform(0, 300, n), rng.uniform(0, 300, n)
    boxes["w"][:n // 4], boxes["h"][:n // 4] = rng.uniform(0, 3, n // 4), rng.uniform(0, 3, n // 4)
    recs[-len(bad) - 4:-len(bad), 0] = 999
    recs[-len(bad):, 0] = 3 + np.arange(len(bad))
    kept = len(bad) + 4
    recs[-kept:, 1:5] = [7, 8, 9, 10]
    state = torch.from_numpy(recs).cuda()
    dboxes = torch.from_numpy(boxes.view(np.uint8).copy()).cuda()
    _lib.check(lib.fear_advance_targets_ycbcr_hdr(dboxes.data_ptr(), table.data_ptr(), 3 + len(bad), state.data_ptr(),
                                                  n, 256, stream()), "fear_advance_targets_ycbcr_hdr")
    got = state.cpu().numpy()
    for i in range(n - kept):
        b = np.array([boxes["x"][i], boxes["y"][i], boxes["w"][i], boxes["h"][i]])
        h, w = shapes[recs[i, 0]]
        want = image_ops.clamp_bbox(image_ops.rescale_bbox(b, recs[i, 5:9], 256), (h, w, 3))
        assert np.array_equal(got[i, 1:5], want), (i, got[i, 1:5], want)
    assert (got[-kept:, 1:5] == [7, 8, 9, 10]).all()
    assert np.array_equal(np.delete(got, np.s_[1:5], axis=1), np.delete(recs, np.s_[1:5], axis=1))


def test_frame_sums_give_numpy_sums_of_the_converted_frame():
    lib = _lib.init(0)
    rng = np.random.default_rng(11)
    frames, rgbs = kernel_frames(rng)
    hd = hdr_codes(cv2.resize(rng.integers(0, 256, (54, 96, 3), dtype=np.uint8), (1920, 1080)), "pq", 10, False, "420")
    frames.append(p010_frame(*hd, matrix="bt2020", transfer="pq"))
    rgbs.append(image_ops.yuv_to_rgb(*hd, "bt2020", False, 10, 0, (1, 1), "pq"))
    sdr8 = fb.YUV420Frame.nv12(torch.zeros((96, 80), dtype=torch.uint8, device="cuda"), matrix="bt2020")
    records = [f.hdr_record() for f in frames]
    bad = unreadable_records(records[0], sdr8.hdr_record())
    table = hdr_table(records + bad)
    F = len(records) + len(bad)
    sums = torch.full((F, 3), -1, dtype=torch.int64, device="cuda")
    _lib.check(lib.fear_frame_sums_ycbcr_hdr_u8(table.data_ptr(), F, sums.data_ptr(), stream()), "sums")
    got = sums.cpu().numpy().view(np.uint64)
    for i, rgb in enumerate(rgbs):
        assert np.array_equal(got[i], rgb.sum(axis=(0, 1), dtype=np.uint64)), i
    assert (got[len(records):] == 0).all()


def test_c_abi_rejects_bad_arguments_and_launches_nothing():
    lib = _lib.init(0)
    t = torch.full((1 << 16,), 0x5A, dtype=torch.uint8, device="cuda")
    p = t.data_ptr()
    good = dict(views=p, F=1, targets=p, N=1, offset=2.0, size=256, crops=p)

    def crop(**kw):
        a = dict(good, **kw)
        return lib.fear_crop_targets_ycbcr_hdr_u8(a["views"], a["F"], a["targets"], a["N"], a["offset"], a["size"],
                                                  a["crops"], None)

    for kw in [dict(views=None), dict(targets=None), dict(crops=None), dict(N=0), dict(N=65536), dict(F=0),
               dict(size=0), dict(size=257), dict(offset=-0.5), dict(offset=float("nan")), dict(offset=float("inf"))]:
        assert crop(**kw) == -1, kw
        assert _lib.last_error(), kw
    for args in [(None, p, 1, p, 1, 256), (p, None, 1, p, 1, 256), (p, p, 1, None, 1, 256), (p, p, 1, p, 0, 256),
                 (p, p, 0, p, 1, 256), (p, p, 1, p, 1, 0)]:
        assert lib.fear_advance_targets_ycbcr_hdr(*args, None) == -1, args
    for args in [(None, 1, p), (p, 1, None), (p, 0, p), (p, 65536, p), (p, -1, p)]:
        assert lib.fear_frame_sums_ycbcr_hdr_u8(*args, None) == -1, args
    torch.cuda.synchronize()
    assert (t == 0x5A).all()  # no kernel and no memset ran


# ---------------------------------------------------------------------------------------------------- trackers
def stream_codes(clip, T, size, transfer, bits, full, sub):
    out = []
    for t in range(T + 1):
        rgb = cv2.resize(clip[t], size)
        out.append(hdr_codes(rgb, transfer, bits, full, sub) if transfer else None)
    return out


STREAMS = [  # (size, layout, transfer, bits, full_range, subsampling)
    ((1920, 1080), "p010", "pq", 10, False, "420"),
    ((480, 256), "nv16", "hlg", 10, False, "422"),
    ((478, 256), "v210", "hlg", 10, True, "422"),
]


def test_multi_tracker_on_hdr_streams_matches_numpy_rgb(net, clip):
    """Pitched 1080p PQ P010, HLG P210 and full-range HLG v210 streams with an SDR NV12 stream in one call, several
    targets each, add / remove part way, and SDR-only calls in between.  Every output equals a tracker fed the converted
    frames as numpy arrays; HDR calls replay one captured graph of the ycbcr_hdr table, SDR-only calls keep the yuv
    table, and the eager step's launch count is that of the other tables."""
    T = 24
    rng = np.random.default_rng(97)
    codes, rgb = [], []
    for size, layout, transfer, bits, full, sub in STREAMS:
        codes.append(stream_codes(clip, T, size, transfer, bits, full, sub))
        rgb.append([image_ops.yuv_to_rgb(*c, "bt2020", full, bits, 0, SHIFTS[sub], transfer) for c in codes[-1]])
    sdr = [cv2.cvtColor(cv2.resize(clip[t], (480, 256)), cv2.COLOR_RGB2YUV_I420) for t in range(T + 1)]
    rgb.append([cv2.cvtColor(f, cv2.COLOR_YUV2RGB_I420) for f in sdr])

    def frames(t, hdr=True):
        out = []
        for s, (size, layout, transfer, bits, full, sub) in enumerate(STREAMS):
            fmt = dict(matrix="bt2020", full_range=full, transfer=transfer if hdr else None)
            if layout == "p010":
                out.append(p010_frame(*codes[s][t], bits, **fmt))
            elif layout == "v210":
                out.append(v210_frame(*codes[s][t], col=4 * s, **fmt))
            else:
                out.append(ycbcr_frame(*codes[s][t], layout, bits, rng=rng, **fmt))
        y = torch.from_numpy(sdr[t]).cuda()
        out.append(fb.YUV420Frame.i420(y))
        return out

    # the identity-crop conversion of every HDR frame the trajectories use is exact
    for s, (size, layout, transfer, bits, full, sub) in enumerate(STREAMS):
        for t in (0, T // 2, T):
            w, h = size
            f = frames(t)[s]
            hh, ww = -(-h // 256) * 256, -(-w // 256) * 256
            got = identity_crops(f, hh, ww)[:h, :w]
            assert np.array_equal(got, rgb[s][t]), (layout, t)

    start = [[[652, 211, 180, 696], [1700, 840, 160, 224]], [base.GOLDEN_BOX, [-10, 100, 50, 50]],
             [[300, 80, 60, 90]], [base.GOLDEN_BOX]]
    late = [[[400, 600, 120, 120]], [[100, 150, 30, 30]], [], [[0, 0, 40, 60]]]

    def rects(d):
        return [r for s in d for r in s], [k for k, s in enumerate(d) for _ in s]

    ref = fb.FEARMultiTracker(net, cuda_id=0, max_targets=12, **CFG)
    trk = fb.FEARMultiTracker(net, cuda_id=0, max_targets=12, **CFG)
    r, s = rects(start)
    assert np.array_equal(trk.add(frames(0), r, s), ref.add([x[0] for x in rgb], r, s))
    hdr_graphs = []
    for t in range(1, T + 1):
        if t == 10:
            r, s = rects(late)
            assert np.array_equal(trk.add(frames(t - 1), r, s), ref.add([x[t - 1] for x in rgb], r, s))
        if t == 18:
            for x in (ref, trk):
                x.remove([1, 2])
        hdr = t % 5 != 0
        if hdr:
            expect = ref.update([x[t] for x in rgb])
            out = trk.update(frames(t))
            assert trk._graph_key[2] == "ycbcr_hdr"
        else:  # SDR only: the NV12 stream's frame for every stream, through the yuv table
            one = [fb.YUV420Frame.i420(torch.from_numpy(sdr[t]).cuda()) for _ in range(4)]
            expect = ref.update([rgb[-1][t]] * 4)
            out = trk.update(one)
            assert trk._graph_key[2] == "yuv"
        assert np.array_equal(out["ids"], expect["ids"]), t
        assert np.array_equal(out["bbox"], expect["bbox"]), (t, out["bbox"], expect["bbox"])
        assert np.array_equal(out["score"], expect["score"]), t
        if hdr and trk._graph is not None:
            hdr_graphs.append(trk._graph)
    assert len({id(g) for g in hdr_graphs}) >= 2  # captured again after the add and the remove
    # one step: the crop and advance entry points around the network's own launches, as on every other table
    counts = {}
    for name, make in (("hdr", lambda t: frames(t)), ("yuv", lambda t: [frames(t)[-1]] * 4)):
        eager = fb.FEARMultiTracker(net, cuda_id=0, max_targets=12, cuda_graph=False, **CFG)
        eager.add(make(0), *rects(start))
        eager.update(make(1))
        torch.cuda.synchronize()
        c0 = net.launch_count()
        eager.update(make(2))
        counts[name] = net.launch_count() - c0
    assert counts["hdr"] == counts["yuv"], counts


def test_sdr_calls_keep_their_tables(net, clip):
    rng = np.random.default_rng(4)
    rgb = cv2.resize(clip[0], (480, 256))
    c420 = hdr_codes(rgb, "pq", 10, False, "420")
    trk = fb.FEARMultiTracker(net, cuda_id=0, max_targets=4, cuda_graph=False, **CFG)
    p010 = p010_frame(*c420, matrix="bt2020")
    pq = p010_frame(*c420, matrix="bt2020", transfer="pq")
    v210 = v210_frame(*hdr_codes(rgb, "hlg", 10, False, "422"), matrix="bt2020")
    nv16 = ycbcr_frame(*hdr_codes(rgb, "hlg", 10, False, "422"), "nv16", 10, rng=rng, matrix="bt2020")
    trk.add([p010, p010], [base.GOLDEN_BOX, [10, 10, 40, 40]], [0, 1])
    for frames, table in (([p010, p010], "yuv"), ([p010, pq], "ycbcr_hdr"), ([nv16, p010], "ycbcr"),
                          ([v210, p010], "ycbcr_v210"), ([v210, pq], "ycbcr_hdr"), ([p010, p010], "yuv")):
        trk.update(frames)
        assert trk._graph_key[2] == table


@pytest.mark.parametrize("smooth", [False, True], ids=["plain", "smooth"])
@pytest.mark.parametrize("transfer", ["pq", "hlg"])
def test_fear_tracker_on_hdr_matches_numpy_rgb(net, clip, smooth, transfer):
    T = 20
    codes = stream_codes(clip, T, (480, 256), transfer, 10, False, "420")
    rgb = [image_ops.yuv_to_rgb(*c, "bt2020", False, 10, 0, (1, 1), transfer) for c in codes]
    init = np.array(base.GOLDEN_BOX)
    for extra in ({}, {"cuda_graph": False}):
        cfg = dict(CFG, smooth=smooth, **extra)
        ref, trk = fb.FEARTracker(net, cuda_id=0, **cfg), fb.FEARTracker(net, cuda_id=0, **cfg)
        ref.initialize(rgb[0], init)
        trk.initialize(p010_frame(*codes[0], matrix="bt2020", transfer=transfer), init)
        assert np.array_equal(trk.tracking_state.mean_color, ref.tracking_state.mean_color)
        for t in range(1, T + 1):
            want = ref.update(rgb[t])["bbox"]
            got = trk.update(p010_frame(*codes[t], matrix="bt2020", transfer=transfer))["bbox"]
            assert np.array_equal(got, want), (smooth, extra, t, got, want)
            for key in ("bbox", "mapping", "prev_size"):
                assert np.array_equal(getattr(trk.tracking_state, key), getattr(ref.tracking_state, key)), (key, t)


def test_hdr_entry_points_and_trackers_on_poisoned_memory():
    """tests/poison_hdr_check.py in its own process: guarded, poisoned tables, crops, sums, boxes and surfaces."""
    proc = subprocess.run([sys.executable, os.path.join(HERE, "poison_hdr_check.py")], capture_output=True, text=True,
                          timeout=1200)
    lines = [l for l in proc.stdout.splitlines() if l.startswith("POISON_CHECK ")]
    assert proc.returncode == 0 and lines, f"poison_hdr_check failed: {proc.stderr[-3000:]}"
    res = json.loads(lines[-1][len("POISON_CHECK "):])
    assert res["checked_calls"] > 0
    assert res["n_failures"] == 0, res["failures"]


def test_report_tie_count():
    """Prints how many outputs the conversion tests found off by 1 at a k + 1/2 tie (none are expected)."""
    print(f"HDR conversion: {TIES['count']} outputs off by 1 at a k + 1/2 tie")
