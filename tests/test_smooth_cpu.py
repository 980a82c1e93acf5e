"""CPU: FEARTracker(gpu_crop=True, smooth=True) is accepted (it fails only for want of a CUDA device), host_normalize
with gpu_crop is still refused, and fear_decode_smooth is declared and bound."""
import numpy as np
import pytest
import torch

import feartracker_b200 as fb
from feartracker_b200 import _lib


def _tracker(**extra):
    trk = fb.FEARTracker(None, cuda_id=0, gpu_crop=True, **dict(fb.FEAR_XS_TRACKER_KWARGS, **extra))
    st = trk.tracking_state
    st.bbox = np.array([163, 53, 45, 174])
    st.mean_color = np.array([90.0, 100.0, 110.0])
    st.paths = [st.bbox]
    return trk


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the behaviour without a GPU")
def test_gpu_crop_smooth_needs_only_a_device():
    trk = _tracker(smooth=True)
    with pytest.raises(RuntimeError, match="needs a CUDA device"):
        trk.update(np.zeros((256, 480, 3), dtype=np.uint8))
    assert trk.tracking_state.prev_size is not None and len(trk.tracking_state.prev_size) == 2


@pytest.mark.parametrize("extra", [dict(host_normalize=True), dict(host_normalize=True, smooth=True)])
def test_gpu_crop_still_refuses_host_normalize(extra):
    with pytest.raises(NotImplementedError, match="host_normalize"):
        _tracker(**extra).update(np.zeros((256, 480, 3), dtype=np.uint8))


def test_gpu_crop_still_refuses_non_rgb_frames():
    with pytest.raises(NotImplementedError, match="host_normalize"):
        _tracker(smooth=True).update(np.zeros((256, 480, 4), dtype=np.uint8))


def test_decode_smooth_is_bound():
    assert "fear_decode_smooth" in _lib.exported_symbols()
