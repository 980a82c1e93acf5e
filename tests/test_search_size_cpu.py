"""CPU: search crops of side S (instance_size = S, score_size = S / 16) -- the geometry the trackers accept, what they
refuse before any device call, and the sized entry points of the C ABI."""
import os
import re

import numpy as np
import pytest
import torch

import feartracker_b200 as fb
from feartracker_b200 import _lib
from feartracker_b200.box_coder import FEARBoxCoder
from feartracker_b200.fear_net import search_side

CFG = fb.FEAR_XS_TRACKER_KWARGS
SIZES = list(range(16, 257, 16))
HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "fear_b200.h")
SIZED = ["fear_track_sized", "fear_track_sized_u8", "fear_forward_sized", "fear_head_sized", "fear_decode_sized",
         "fear_decode_smooth_sized"]


def _cfg(size, **kw):
    return dict(CFG, instance_size=size, score_size=size // 16, **kw)


def _net():
    return fb.FEARNet(**fb.FEAR_XS_MODEL_KWARGS).eval()


@pytest.mark.parametrize("size", SIZES)
def test_every_size_in_the_contract_is_accepted(size):
    s = size // 16
    coder = FEARBoxCoder(_cfg(size))
    ax = (np.arange(s) - s // 2) * 16.0 + size // 2  # reference utils/utils.py:183-199
    assert np.array_equal(coder.grid_x.numpy()[0], np.tile(ax, (s, 1)))
    assert np.array_equal(coder.grid_y.numpy()[0], np.tile(ax[:, None], (1, s)))
    trk = fb.FEARTracker(_net(), cuda_id="cpu", **_cfg(size))
    assert trk.window.shape == (s, s)
    multi = fb.FEARMultiTracker(_net(), cuda_id="cpu", max_targets=2, **_cfg(size))
    assert len(multi) == 0


@pytest.mark.parametrize("size", [255, 272, 320, 8, 0, 24])
def test_sizes_outside_the_contract_are_refused(size):
    cfg = dict(CFG, instance_size=size, score_size=size // 16)
    with pytest.raises(NotImplementedError):
        FEARBoxCoder(cfg)
    with pytest.raises((NotImplementedError, ValueError)):
        fb.FEARTracker(_net(), cuda_id="cpu", **cfg)
    with pytest.raises(ValueError):
        fb.FEARMultiTracker(_net(), cuda_id="cpu", max_targets=2, **cfg)


@pytest.mark.parametrize("size,score", [(192, 16), (192, 11), (256, 12), (128, 16), (16, 2)])
def test_mismatched_score_size_is_refused(size, score):
    cfg = dict(CFG, instance_size=size, score_size=score)
    with pytest.raises(NotImplementedError):
        FEARBoxCoder(cfg)
    with pytest.raises(ValueError, match="score_size"):
        fb.FEARTracker(_net(), cuda_id="cpu", **cfg)
    with pytest.raises(ValueError, match="score_size"):
        fb.FEARMultiTracker(_net(), cuda_id="cpu", max_targets=2, **cfg)


@pytest.mark.parametrize("stride", [8, 32])
def test_other_strides_are_refused(stride):
    cfg = dict(CFG, instance_size=192, score_size=192 // stride, total_stride=stride)
    with pytest.raises(NotImplementedError):
        FEARBoxCoder(cfg)
    with pytest.raises(NotImplementedError):
        fb.FEARTracker(_net(), cuda_id="cpu", **cfg)
    with pytest.raises(ValueError, match="total_stride"):
        fb.FEARMultiTracker(_net(), cuda_id="cpu", max_targets=2, **cfg)


def test_template_size_stays_128():
    with pytest.raises(ValueError):
        fb.FEARMultiTracker(_net(), cuda_id="cpu", max_targets=2, **_cfg(192, template_size=96))


@pytest.mark.parametrize("size", SIZES)
def test_search_side_accepts_square_searches(size):
    assert search_side((3, 3, size, size), u8=False) == size
    assert search_side((1, size, size, 3), u8=True) == size


@pytest.mark.parametrize("shape,u8", [
    ((1, 3, 192, 128), False), ((1, 3, 255, 255), False), ((1, 3, 272, 272), False), ((1, 3, 8, 8), False),
    ((1, 4, 192, 192), False), ((3, 192, 192), False), ((1, 192, 128, 3), True), ((1, 192, 192, 4), True),
    ((1, 320, 320, 3), True), ((1, 3, 192, 192), True),
])
def test_search_side_refuses_other_shapes(shape, u8):
    with pytest.raises(ValueError, match="multiple of 16"):
        search_side(shape, u8)


def test_fearnet_refuses_bad_searches_before_device_calls():
    net = _net()
    for x in (torch.zeros(1, 3, 192, 128), torch.zeros(1, 3, 272, 272)):
        with pytest.raises((ValueError, RuntimeError)):
            net.track(x, torch.zeros(1, 256, 8, 8))
    with pytest.raises(ValueError, match="multiple of 16"):
        net.track_boxes_from_host(torch.zeros(2, 3, 200, 200), torch.zeros(1, 256, 8, 8))


def test_sized_entry_points_are_declared_exported_and_bound():
    with open(HEADER) as f:
        header = f.read()
    assert re.search(r"#define FEAR_ABI_VERSION 1\b", header)
    for name in SIZED:
        assert re.search(r"\b%s\(" % name, header), name
        assert name in _lib.exported_symbols(), name
    if os.path.isfile(_lib.LIB_PATH):
        lib = _lib.load()
        assert lib.fear_abi_version() == 1
        for name in SIZED:
            assert getattr(lib, name) is not None


def test_sized_entry_points_refuse_sizes_without_a_device():
    """Size checks of the handle-free decode entry points come before any launch (non-null dummy pointers)."""
    if not os.path.isfile(_lib.LIB_PATH):
        pytest.skip("library not built")
    lib = _lib.load()
    p = 16  # never dereferenced: the refusal comes first
    for s in (0, 17, -1):
        assert lib.fear_decode_sized(p, p, 1, s, 1, p, None) == -1
        assert "score-map side" in _lib.last_error()
        assert lib.fear_decode_smooth_sized(p, p, 1, s, p, p, p, None) == -1


@pytest.mark.parametrize("drop,kw", [("total_stride", dict(score_size=11)), ("score_size", dict(total_stride=8))])
def test_multi_tracker_refuses_a_partial_geometry_with_value_error(drop, kw):
    cfg = {k: v for k, v in _cfg(192).items() if k != drop}
    cfg.update(kw)
    with pytest.raises(ValueError, match="score map"):
        fb.FEARMultiTracker(_net(), cuda_id="cpu", max_targets=2, **cfg)
