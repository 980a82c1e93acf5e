"""CPU: the orientation of rotated and mirrored frames (``image_ops.orient``, ``fb.Oriented``) agrees with the
documented index table, is refused before any device call when malformed, keeps the kinds' mixing rules, and the two
oriented entry points are declared, bound, check their arguments and fail cleanly without a driver."""
import os
import re

import numpy as np
import pytest
import torch

import feartracker_b200 as fb
from feartracker_b200 import _lib, image_ops
from feartracker_b200 import multi_tracker as mt
from tests.test_rgb_formats_cpu import _fake_bayer, _fake_mono, _fake_rgb
from tests.test_yuv_frames_cpu import RGB, _tracker

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ("fear_crop_targets_oriented_u8", "fear_advance_targets_oriented")
TABLES = ("VIEW", "YUV", "YCBCR", "YCBCR_V210", "YCBCR_HDR", "BAYER", "MONO", "RGB")


def _stored(y, x, H, W, code):
    """The stored pixel of display pixel (y, x) for ``code``, as include/fear_b200.h tabulates it."""
    ys, xs = [(y, x), (H - 1 - x, y), (H - 1 - y, W - 1 - x), (x, W - 1 - y)][code & 3]
    return ys, (W - 1 - xs if code & 4 else xs)


@pytest.mark.parametrize("shape", [(3, 5), (7, 4), (1, 6), (5, 1), (1, 1), (37, 53)])
def test_orient_agrees_with_the_index_table(shape):
    H, W = shape
    a = np.arange(H * W * 3, dtype=np.int64).reshape(H, W, 3)
    for code in range(8):
        d = image_ops.orient(a, code)
        assert d.shape == ((W, H, 3) if code & 1 else (H, W, 3)), code
        for y in range(d.shape[0]):
            for x in range(d.shape[1]):
                assert np.array_equal(d[y, x], a[_stored(y, x, H, W, code)]), (code, y, x)


def test_orient_codes_are_distinct_and_compose_as_documented():
    a = np.arange(15).reshape(3, 5)
    outs = [image_ops.orient(a, c) for c in range(8)]
    for i in range(8):
        for j in range(i):
            assert outs[i].shape != outs[j].shape or not np.array_equal(outs[i], outs[j]), (i, j)
    assert np.array_equal(image_ops.orient(a, 1), np.rot90(a, -1))  # 90 degrees clockwise
    assert np.array_equal(image_ops.orient(a, 4), a[:, ::-1])
    assert np.array_equal(image_ops.orient(a, 5), np.rot90(a[:, ::-1], -1))


def test_orient_code_of_rotate_and_mirror():
    assert [image_ops.orient_code(r, m) for m in (False, True) for r in (0, 90, 180, 270)] == list(range(8))
    assert image_ops.orient_code(np.int64(270)) == 3
    # ffprobe's rotation=-90 (a portrait phone clip) is rotate = 90: code 1
    assert image_ops.orient_code((90) % 360) == 1


BAD_ROTATIONS = [45, -90, 360, 1, 90.0, "90", None, True]


@pytest.mark.parametrize("rotate", BAD_ROTATIONS, ids=[repr(r) for r in BAD_ROTATIONS])
def test_bad_rotation_is_refused(rotate):
    with pytest.raises(ValueError, match="rotate must be 0, 90, 180 or 270"):
        fb.Oriented(torch.zeros((4, 6, 3), dtype=torch.uint8), rotate)


def test_numpy_nested_and_non_frames_are_refused():
    with pytest.raises(ValueError, match=r"image_ops\.orient"):
        fb.Oriented(RGB, 90)
    inner = fb.Oriented(torch.zeros((4, 6, 3), dtype=torch.uint8), 90)
    with pytest.raises(ValueError, match="cannot be nested"):
        fb.Oriented(inner, 90)
    for bad in ("frame", None, 3, [torch.zeros((4, 6, 3), dtype=torch.uint8)]):
        with pytest.raises(ValueError, match="Oriented wraps a CUDA uint8 tensor"):
            fb.Oriented(bad)


def test_attributes_and_display_shape():
    t = torch.zeros((4, 6, 3), dtype=torch.uint8)
    for rotate in (0, 90, 180, 270):
        for mirror in (False, True):
            o = fb.Oriented(t, rotate, mirror)
            assert o.frame is t and o.code == rotate // 90 + 4 * mirror
            assert o.shape == ((6, 4, 3) if rotate % 180 else (4, 6, 3))
    for f in (_fake_rgb(), _fake_mono(), _fake_bayer()):
        assert fb.Oriented(f, 270).shape == (f.shape[1], f.shape[0], 3)
    nv12 = fb.YUV420Frame.nv12(torch.zeros((12, 10), dtype=torch.uint8))
    assert fb.Oriented(nv12, 90).shape == (10, 8, 3) and nv12.shape == (8, 10, 3)


def test_frame_kind_and_codes_through_the_wrapper():
    nv12 = fb.YUV420Frame.nv12(torch.zeros((12, 8), dtype=torch.uint8))
    t = torch.zeros((4, 6, 3), dtype=torch.uint8)
    for f in (nv12, t, _fake_rgb(), _fake_mono(), _fake_bayer()):
        assert mt.frame_kind(fb.Oriented(f, 180, True)) == mt.frame_kind(f)
        assert mt.stored(fb.Oriented(f, 90)) is f and mt.stored(f) is f
    assert mt.orient_codes([t, t]) is None
    assert mt.orient_codes([t, fb.Oriented(t, 270, True), fb.Oriented(t)]).tolist() == [0, 7, 0]
    assert mt.orient_codes([t, fb.Oriented(t, 270)]).dtype == np.int32
    mono = _fake_mono()
    mono.agc = "minmax"
    assert mt.uses_agc([fb.Oriented(mono, 90)], "mono") and not mt.uses_agc([fb.Oriented(_fake_mono(), 90)], "mono")


def test_mixing_rules_hold_through_the_wrapper():
    trk = _tracker()
    nv12 = fb.YUV420Frame.nv12(torch.zeros((12, 8), dtype=torch.uint8))
    t = torch.zeros((8, 8, 3), dtype=torch.uint8)
    O = fb.Oriented
    cases = [
        ([O(_fake_bayer(), 90), nv12], "BayerFrames cannot share a call"),
        ([O(_fake_mono(), 90), O(t, 180)], "MonoFrames cannot share a call"),
        ([O(_fake_rgb(), 90), O(nv12, 90)], "RGBFrames can share a call only with CUDA uint8 RGB tensors"),
        ([O(t, 90), RGB], "frames of one call must be all numpy arrays"),
        ([O(nv12, 270), O(t, 90)], "frames of one call must be all numpy arrays"),
    ]
    for frames, msg in cases:
        with pytest.raises(ValueError, match=msg):
            trk.update(frames)
        with pytest.raises(ValueError, match=msg):
            trk.update(dict(enumerate(frames)))
        with pytest.raises(ValueError, match=msg):
            trk.add(frames, [[1, 1, 2, 2]])
    # frames the kinds allow together pass the checks; the device is checked as for plain frames
    for frames in ([O(t, 90), t, O(t, 180, True)], [O(_fake_rgb(), 270), O(t, 90)], O(t, 90), {5: O(t, 90)}):
        with pytest.raises(ValueError, match="cpu tensor"):
            trk.update(frames)
    assert len(trk) == 0


def test_new_symbols_and_table_enum_are_declared_and_bound():
    with open(os.path.join(ROOT, "include", "fear_b200.h")) as f:
        header = f.read()
    for name in NEW_SYMBOLS:
        assert f"int {name}(" in header
        assert name in _lib.exported_symbols() and name in _lib._SIGNATURES
        assert getattr(_lib.load(), name).argtypes
    enum = dict((k, int(v)) for k, v in re.findall(r"\bFEAR_TABLE_([A-Z0-9_]+)\s*=\s*(\d+)", header))
    assert enum == {name: i for i, name in enumerate(TABLES)}
    # every table FEARMultiTracker names has its enum value, and the oriented pair covers all of them
    assert set(_lib.ORIENT_TABLES) == set(mt.ENTRY_POINTS) == set(mt.TABLE_DTYPES)
    assert sorted(_lib.ORIENT_TABLES.values()) == list(range(8))
    families = {"views": "VIEW", "yuv": "YUV", "ycbcr": "YCBCR", "ycbcr_v210": "YCBCR_V210", "ycbcr_hdr": "YCBCR_HDR",
                "bayer": "BAYER", "mono": "MONO", "rgb": "RGB"}
    for name, code in _lib.ORIENT_TABLES.items():
        assert enum[families[name]] == code, name
    assert _lib.load().fear_abi_version() == 1


def test_entry_points_check_arguments_without_a_device():
    lib = _lib.load()
    p = 1 << 20  # never dereferenced: every call below is refused before a launch

    def crop(table=0, d_table=p, orient=p, F=2, targets=p, N=4, offset=2.0, size=256, crops=p):
        return lib.fear_crop_targets_oriented_u8(table, d_table, orient, F, targets, N, offset, size, crops, None)

    def advance(boxes=p, table=0, d_table=p, orient=p, F=2, targets=p, N=4, size=256):
        return lib.fear_advance_targets_oriented(boxes, table, d_table, orient, F, targets, N, size, None)

    for kw in [dict(table=-1), dict(table=8), dict(table=1 << 20), dict(d_table=None), dict(targets=None),
               dict(crops=None), dict(F=0), dict(N=0), dict(N=65536), dict(size=0), dict(size=257),
               dict(offset=-1.0), dict(offset=float("nan"))]:
        assert crop(**kw) == -1, kw
        assert _lib.last_error(), kw
    assert crop(table=9) == -1 and "unknown frame table 9" in _lib.last_error()
    for kw in [dict(table=-1), dict(table=8), dict(boxes=None), dict(d_table=None), dict(targets=None), dict(F=0),
               dict(N=0), dict(size=0)]:
        assert advance(**kw) == -1, kw
        assert _lib.last_error(), kw


def test_entry_points_fail_without_a_driver():
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    lib = _lib.load()
    p = 1 << 20
    for table in range(8):
        # a null code array is allowed: every code 0
        for orient in (p, None):
            assert lib.fear_crop_targets_oriented_u8(table, p, orient, 2, p, 4, 2.0, 256, p, None) > 0
            assert "crop_targets_u8_kernel" in _lib.last_error()
            assert lib.fear_advance_targets_oriented(p, table, p, orient, 2, p, 4, 256, None) > 0
            assert "advance_targets_kernel" in _lib.last_error()
