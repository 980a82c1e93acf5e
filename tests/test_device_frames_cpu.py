"""CPU: FEARMultiTracker's tensor-frame checks and the FearFrameView records it builds for tensors."""
import numpy as np
import pytest
import torch

import feartracker_b200 as fb
from feartracker_b200 import _lib
from feartracker_b200.multi_tracker import frame_view

CFG = fb.FEAR_XS_TRACKER_KWARGS
FRAME = np.zeros((64, 80, 3), np.uint8)


def _tracker():
    net = fb.FEARNet(**fb.FEAR_XS_MODEL_KWARGS).eval()
    return fb.FEARMultiTracker(net, cuda_id="cpu", max_targets=4, **CFG)


def test_view_record_is_40_bytes():
    assert _lib.VIEW_DTYPE.itemsize == 40
    assert _lib.VIEW_DTYPE.names == ("data", "row_stride", "pixel_stride", "channel_stride", "H", "W")


@pytest.mark.parametrize("frames", [
    torch.zeros(64, 80, 3, dtype=torch.uint8),  # a CPU tensor
    [torch.zeros(64, 80, 3, dtype=torch.uint8)],
    [torch.zeros(64, 80, 3, dtype=torch.float32)],
    [torch.zeros(64, 80, 4, dtype=torch.uint8)],
    [torch.zeros(3, 64, 80, 3, dtype=torch.uint8)[0, :, :, :2]],
    [torch.zeros(64, 80, dtype=torch.uint8)],
    [torch.zeros(0, 80, 3, dtype=torch.uint8)],
    [torch.zeros(64, 0, 3, dtype=torch.uint8)],
    [FRAME, torch.zeros(64, 80, 3, dtype=torch.uint8)],  # numpy and tensor frames mixed in one call
    [torch.zeros(64, 80, 3, dtype=torch.uint8), FRAME],
])
def test_bad_tensor_frames_are_refused_before_device_calls(frames):
    trk = _tracker()
    with pytest.raises(ValueError):
        trk.add(frames, [[10, 10, 20, 20]])
    with pytest.raises(ValueError):
        trk.update(frames)
    trk._ids, trk._streams = np.array([0]), np.array([0])  # a live target: update reaches the frame checks the same way
    with pytest.raises(ValueError):
        trk.update(frames)


def _expect(t, offset, strides, h, w):
    base = t.untyped_storage().data_ptr()
    assert frame_view(t) == (base + offset, *strides, h, w)
    rec = np.array([frame_view(t)], dtype=_lib.VIEW_DTYPE)[0]
    assert (int(rec["data"]), int(rec["H"]), int(rec["W"])) == (base + offset, h, w)


def test_view_of_contiguous_hwc():
    t = torch.arange(6 * 7 * 3, dtype=torch.uint8).reshape(6, 7, 3)
    _expect(t, 0, (21, 3, 1), 6, 7)


def test_view_of_roi():
    t = torch.zeros(40, 50, 3, dtype=torch.uint8)
    _expect(t[5:25, 10:45], 5 * 150 + 10 * 3, (150, 3, 1), 20, 35)


def test_view_of_chw_permuted_to_hwc():
    t = torch.zeros(3, 40, 50, dtype=torch.uint8)
    _expect(t.permute(1, 2, 0), 0, (50, 1, 2000), 40, 50)


def test_view_of_rgba_sliced_to_rgb():
    t = torch.zeros(40, 50, 4, dtype=torch.uint8)
    _expect(t[..., :3], 0, (200, 4, 1), 40, 50)
    _expect(t[2:, 3:, :3], 2 * 200 + 3 * 4, (200, 4, 1), 38, 47)


def test_view_addresses_pixels():
    """Reading through the record's strides gives the tensor's pixels, for every kind of view."""
    g = torch.Generator().manual_seed(3)
    rgba = torch.randint(0, 256, (9, 11, 4), dtype=torch.uint8, generator=g)
    chw = torch.randint(0, 256, (3, 9, 11), dtype=torch.uint8, generator=g)
    for t in (rgba[..., :3].contiguous(), rgba[2:7, 1:10, :3], chw.permute(1, 2, 0), rgba[..., :3]):
        data, rs, ps, cs, h, w = frame_view(t)
        storage = np.frombuffer(bytes(t.untyped_storage()), dtype=np.uint8)
        off = data - t.untyped_storage().data_ptr()
        y, x, c = np.meshgrid(np.arange(h), np.arange(w), np.arange(3), indexing="ij")
        assert np.array_equal(storage[off + y * rs + x * ps + c * cs], t.numpy())
