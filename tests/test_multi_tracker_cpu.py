"""CPU: FEARMultiTracker construction and the input checks that run before any device call."""
import numpy as np
import pytest
import torch

import feartracker_b200 as fb

CFG = fb.FEAR_XS_TRACKER_KWARGS
FRAME = np.zeros((64, 80, 3), np.uint8)


def _tracker(**kw):
    net = fb.FEARNet(**fb.FEAR_XS_MODEL_KWARGS).eval()
    return fb.FEARMultiTracker(net, cuda_id="cpu", max_targets=kw.pop("max_targets", 4), **dict(CFG, **kw))


def test_constructs_without_gpu_and_fails_loudly():
    trk = _tracker()
    assert len(trk) == 0 and trk.net._reserved == 4
    out = trk.update(FRAME)  # nothing to track: no device needed
    assert out["bbox"].shape == (0, 4) and out["score"].shape == (0,) and out["ids"].shape == (0,)
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError):
            trk.add(FRAME, [[10, 10, 20, 20]])
        assert len(trk) == 0


@pytest.mark.parametrize("key", ["smooth", "host_normalize"])
def test_unsupported_options_are_refused(key):
    with pytest.raises(NotImplementedError, match="no smooth / host_normalize"):
        _tracker(**{key: True})


@pytest.mark.parametrize("kw", [dict(search_context=-1), dict(template_bbox_offset=-0.1),
                                dict(search_context=float("nan")), dict(template_bbox_offset=float("inf")),
                                dict(instance_size=255), dict(template_size=127), dict(max_targets=0)])
def test_bad_config_is_refused(kw):
    with pytest.raises(ValueError):
        _tracker(**kw)


@pytest.mark.parametrize("frames", [
    np.zeros((64, 80), np.uint8), np.zeros((64, 80, 4), np.uint8), np.zeros((64, 80, 3), np.float32),
    np.zeros((0, 80, 3), np.uint8), [FRAME, np.zeros((8, 8, 3), np.int16)], [], [torch.zeros(64, 80, 3)],
])
def test_bad_frames_are_refused_before_device_calls(frames):
    trk = _tracker()
    with pytest.raises(ValueError):
        trk.add(frames, [[10, 10, 20, 20]])
    with pytest.raises(ValueError):
        trk.update(frames)


@pytest.mark.parametrize("rects,streams", [
    ([[10, 10, 20, 20]], [1]), ([[10, 10, 20, 20]], [-1]), ([[10, 10, 20, 20]], [0, 0]),
    ([[10, 10, 20, 20]], [0.0]), ([[10, 10, 20]], None), (np.zeros((2, 2, 4)), None),
    ([[10, 10, 20, 20]] * 5, None),  # more than max_targets
])
def test_bad_targets_are_refused_before_device_calls(rects, streams):
    with pytest.raises(ValueError):
        _tracker().add(FRAME, rects, streams)


def test_update_checks_stream_indices_of_live_targets():
    trk = _tracker()
    trk._ids, trk._streams = np.array([0, 1]), np.array([0, 2])  # two targets, the second in stream 2
    with pytest.raises(ValueError, match="stream 2"):
        trk.update([FRAME, FRAME])
    with pytest.raises(ValueError, match="unknown target ids"):
        trk.remove([5])
