"""CPU: FEARMultiTracker's {stream id: frame} mappings are refused before any device call when malformed, select the
right targets, and the gather / scatter entry points of a subset step are declared, bound and fail cleanly without a
driver."""
import os

import numpy as np
import pytest
import torch

import feartracker_b200 as fb
from feartracker_b200 import _lib
from feartracker_b200 import multi_tracker as mt
from tests.test_rgb_formats_cpu import _fake_bayer, _fake_mono, _fake_rgb
from tests.test_yuv_frames_cpu import RGB, _tracker

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ("fear_gather_targets", "fear_scatter_targets")


def _with_targets(streams):
    """A tracker on "cpu" (every device call raises RuntimeError) that believes it tracks targets in ``streams``."""
    trk = _tracker()
    trk._ids, trk._streams = np.arange(len(streams), dtype=np.int64), np.asarray(streams, dtype=np.int64)
    return trk


BAD_KEYS = ["a", 1.0, None, (0,), True, False, np.bool_(True), -1, 2 ** 31, np.int64(-3), np.uint64(2 ** 32)]


@pytest.mark.parametrize("key", BAD_KEYS, ids=[repr(k) for k in BAD_KEYS])
def test_bad_stream_ids_are_refused_before_device_calls(key):
    trk = _with_targets([0])
    with pytest.raises(ValueError, match="stream ids must be ints"):
        trk.update({key: RGB})
    with pytest.raises(ValueError, match="stream ids must be ints"):
        trk.update({5: RGB, key: RGB})
    with pytest.raises(ValueError, match="stream ids must be ints"):
        _tracker().add({key: RGB}, [[1, 1, 2, 2]])


def test_extreme_stream_ids_pass_the_checks():
    # the checks pass and the call reaches the device, which this tracker does not have
    for key in (0, 2 ** 31 - 1, np.int32(17), np.uint8(3)):
        trk = _with_targets([int(key)])
        with pytest.raises(RuntimeError, match="needs a CUDA device"):
            trk.update({key: RGB})
        with pytest.raises(RuntimeError, match="needs a CUDA device"):
            _tracker().add({key: RGB}, [[1, 1, 2, 2]], [int(key)])


def test_empty_mapping_is_refused_like_an_empty_list():
    trk = _with_targets([0])
    for call in (lambda: trk.update({}), lambda: trk.add({}, [[1, 1, 2, 2]]), lambda: trk.update([])):
        with pytest.raises(ValueError, match="no frames given"):
            call()


def test_add_streams_must_be_keys():
    trk = _tracker()
    with pytest.raises(ValueError, match=r"streams \[0\] are not keys"):
        trk.add({3: RGB, 17: RGB}, [[1, 1, 2, 2]])  # the default stream 0
    with pytest.raises(ValueError, match=r"streams \[5\] are not keys"):
        trk.add({3: RGB, 17: RGB}, [[1, 1, 2, 2]] * 3, [3, 5, 17])
    with pytest.raises(ValueError, match="integer stream ids"):
        trk.add({3: RGB}, [[1, 1, 2, 2]], [3.0])
    with pytest.raises(ValueError, match="integer stream ids"):
        trk.add({3: RGB}, [[1, 1, 2, 2]] * 2, [3])
    with pytest.raises(ValueError, match="integer stream ids"):
        trk.add({0: RGB}, [[1, 1, 2, 2]], [False])
    assert len(trk) == 0


def test_malformed_frames_are_refused_as_in_a_list():
    trk = _with_targets([0, 1])
    cases = [
        ({0: RGB, 1: np.zeros((8, 8), np.uint8)}, "frame 1 must be a uint8 HxWx3 RGB array"),
        ({0: RGB, 1: RGB.astype(np.float32)}, "frame 1 must be a uint8 HxWx3 RGB array"),
        ({0: "frame"}, "frame 0 must be a uint8 HxWx3 RGB array"),
        ({0: torch.zeros((8, 8, 3), dtype=torch.uint8)}, "cpu tensor"),
        ({0: RGB, 1: torch.zeros((8, 8, 3), dtype=torch.uint8)}, "frames of one call must be all numpy arrays"),
        ({0: _fake_rgb(), 1: RGB}, "RGBFrames can share a call only with CUDA"),
        ({0: _fake_bayer(), 1: RGB}, "BayerFrames cannot share"),
        ({0: RGB, 1: _fake_mono()}, "MonoFrames cannot share"),
    ]
    for frames, msg in cases:
        with pytest.raises(ValueError, match=msg):
            trk.update(frames)
        with pytest.raises(ValueError, match=msg):
            _tracker().add(frames, [[1, 1, 2, 2]])
        # the same values as a list give the same message
        with pytest.raises(ValueError, match=msg):
            trk.update(list(frames.values()))


def test_a_key_without_targets_is_checked_but_not_read():
    trk = _with_targets([0, 5])
    with pytest.raises(ValueError, match="frame 1 must be"):
        trk.update({3: RGB, 4: np.zeros((2, 2), np.uint8)})
    out = trk.update({3: RGB, 4: RGB})  # no target selected: empty results, no device call
    assert out["bbox"].shape == (0, 4) and out["bbox"].dtype == np.int64
    assert out["score"].shape == (0,) and out["score"].dtype == np.float32
    assert out["ids"].shape == (0,) and out["ids"].dtype == np.int64
    with pytest.raises(RuntimeError, match="needs a CUDA device"):
        trk.update({3: RGB, 5: RGB})  # selects target 1: the call reaches the device
    assert _tracker().update({0: RGB})["ids"].size == 0  # no targets at all


def test_list_update_after_sparse_stream_ids_raises_the_stream_error():
    trk = _with_targets([3, 17])
    with pytest.raises(ValueError, match="targets track stream 17 but only 2 frames were given"):
        trk.update([RGB, RGB])


def test_positions_of_streams_in_a_mapping():
    keys = np.array([17, 3, 40, 0], dtype=np.int64)
    assert mt._positions(keys, np.array([3, 3, 17, 0, 40])).tolist() == [1, 1, 0, 3, 2]
    s, pos = fb.FEARMultiTracker._check_mapping_streams([40, 17], 2, keys)
    assert s.tolist() == [40, 17] and pos.tolist() == [2, 0]


def test_new_symbols_are_declared_and_bound():
    with open(os.path.join(ROOT, "include", "fear_b200.h")) as f:
        header = f.read()
    for name in NEW_SYMBOLS:
        assert f"int {name}(" in header
        assert name in _lib.exported_symbols() and name in _lib._SIGNATURES
        assert getattr(_lib.load(), name).argtypes
    assert _lib.load().fear_abi_version() == 1


def test_entry_points_check_arguments_without_a_device():
    lib = _lib.load()
    p = 1 << 20  # never dereferenced: every call below is refused before a launch
    good = dict(targets=p, N=4, templates=p, select=p, M=2, step_targets=p, step_templates=p)

    def gather(**kw):
        a = dict(good, **kw)
        return lib.fear_gather_targets(a["targets"], a["N"], a["templates"], a["select"], a["M"], a["step_targets"],
                                       a["step_templates"], None)

    for kw in [dict(targets=None), dict(templates=None), dict(select=None), dict(step_targets=None),
               dict(step_templates=None), dict(N=0), dict(N=-1), dict(M=0), dict(M=65536), dict(templates=p + 4),
               dict(step_templates=p + 8)]:
        assert gather(**kw) == -1, kw
        assert _lib.last_error(), kw
    for args in [(None, p, 2, p, 4), (p, None, 2, p, 4), (p, p, 2, None, 4), (p, p, 0, p, 4), (p, p, 65536, p, 4),
                 (p, p, 2, p, 0)]:
        assert lib.fear_scatter_targets(*args, None) == -1, args
        assert _lib.last_error(), args


def test_entry_points_fail_without_a_driver():
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    lib = _lib.load()
    p = 1 << 20
    assert lib.fear_gather_targets(p, 4, p, p, 2, p, p, None) > 0
    assert "gather_targets_kernel" in _lib.last_error()
    assert lib.fear_scatter_targets(p, p, 2, p, 4, None) > 0
    assert "scatter_targets_kernel" in _lib.last_error()
