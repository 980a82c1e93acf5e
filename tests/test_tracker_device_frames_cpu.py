"""CPU: FEARTracker's checks of device frames (CUDA tensors, YUV frames), which run before any device call or state
change, and the frame helpers it shares with FEARMultiTracker."""
import numpy as np
import pytest
import torch

import feartracker_b200 as fb
from feartracker_b200 import image_ops, multi_tracker

CFG = fb.FEAR_XS_TRACKER_KWARGS
BOX = np.array([163, 53, 45, 174])


def _tracker(**extra):
    return fb.FEARTracker(None, cuda_id=0, **dict(CFG, **extra))


def _tracking(trk):
    st = trk.tracking_state
    st.bbox, st.mean_color, st.paths = BOX.copy(), np.array([90.0, 100.0, 110.0]), [BOX.copy()]
    st.mapping, st.prev_size = np.array([1, 2, 3, 4], dtype=np.int32), np.array([40.0, 50.0])
    return trk


def _snapshot(trk):
    st = trk.tracking_state
    return (repr(st.bbox), repr(st.mapping), repr(st.prev_size), repr(st.mean_color), repr(st.paths),
            trk._template_features, getattr(trk, "_device_state", None), getattr(trk, "_gpu_crop_state", None))


def _planes(h=64, w=80):
    return torch.zeros(h, w, dtype=torch.uint8), torch.zeros(h // 2, w // 2, dtype=torch.uint8)


BAD_FRAMES = {
    "cpu_tensor": torch.zeros(64, 80, 3, dtype=torch.uint8),
    "float_tensor": torch.zeros(64, 80, 3, dtype=torch.float32),
    "four_channels": torch.zeros(64, 80, 4, dtype=torch.uint8),
    "two_channels": torch.zeros(3, 64, 80, 3, dtype=torch.uint8)[0, :, :, :2],
    "2d_tensor": torch.zeros(64, 80, dtype=torch.uint8),
    "4d_tensor": torch.zeros(1, 64, 80, 3, dtype=torch.uint8),
    "empty_tensor": torch.zeros(0, 80, 3, dtype=torch.uint8),
    "nv12_on_cpu": fb.YUV420Frame.nv12(torch.zeros(96, 80, dtype=torch.uint8)),
    "planes_on_cpu": fb.YUV420Frame(_planes()[0], _planes()[1], _planes()[1]),
    "yuyv_on_cpu": fb.YUV422Frame.yuyv(torch.zeros(64, 160, dtype=torch.uint8)),
    "i444_on_cpu": fb.YUV444Frame.i444(torch.zeros(192, 80, dtype=torch.uint8)),
}


@pytest.mark.parametrize("extra", [{}, dict(smooth=True), dict(gpu_crop=True), dict(gpu_crop=True, smooth=True)])
@pytest.mark.parametrize("name", sorted(BAD_FRAMES))
def test_malformed_device_frames_are_refused_before_any_state_change(name, extra):
    frame = BAD_FRAMES[name]
    trk = _tracker(**extra)
    before = _snapshot(trk)
    with pytest.raises(ValueError):
        trk.initialize(frame, BOX)
    with pytest.raises(ValueError):
        trk.get_template_features(frame, BOX)
    assert _snapshot(trk) == before and trk.tracking_state.bbox is None
    _tracking(trk)
    before = _snapshot(trk)
    with pytest.raises(ValueError):
        trk.update(frame)
    assert _snapshot(trk) == before


@pytest.mark.parametrize("name", ["cpu_tensor", "nv12_on_cpu", "planes_on_cpu", "yuyv_on_cpu", "i444_on_cpu"])
def test_host_memory_frames_point_to_numpy(name):
    with pytest.raises(ValueError, match="pass host frames as numpy arrays"):
        _tracking(_tracker()).update(BAD_FRAMES[name])


@pytest.mark.parametrize("extra", [{}, dict(smooth=True), dict(gpu_crop=True)])
@pytest.mark.parametrize("name", ["cpu_tensor", "four_channels", "nv12_on_cpu", "yuyv_on_cpu"])
def test_host_normalize_refuses_device_frames(name, extra):
    """Refused for any tensor or YUV frame, before its checks: no device is needed to see it."""
    trk = _tracker(host_normalize=True, **extra)
    for call in (lambda: trk.initialize(BAD_FRAMES[name], BOX), lambda: trk.get_template_features(BAD_FRAMES[name], BOX)):
        with pytest.raises(NotImplementedError, match="host_normalize"):
            call()
    assert trk.tracking_state.bbox is None and getattr(trk, "_device_state", None) is None
    _tracking(trk)
    before = _snapshot(trk)
    with pytest.raises(NotImplementedError, match="host_normalize"):
        trk.update(BAD_FRAMES[name])
    assert _snapshot(trk) == before


@pytest.mark.parametrize("name", sorted(BAD_FRAMES))
def test_messages_are_those_of_the_multi_tracker(name):
    multi = fb.FEARMultiTracker(fb.FEARNet(**fb.FEAR_XS_MODEL_KWARGS).eval(), cuda_id="cpu", max_targets=1, **CFG)
    frame = BAD_FRAMES[name]
    with pytest.raises(ValueError) as want:
        multi.update([frame])
    with pytest.raises(ValueError) as got:
        _tracking(_tracker()).update(frame)
    assert str(got.value) == str(want.value)


def test_shared_helpers():
    assert multi_tracker.frame_kind(np.zeros((2, 2, 3), np.uint8)) == "numpy"
    assert multi_tracker.frame_kind(torch.zeros(2, 2, 3, dtype=torch.uint8)) == "cuda"
    assert multi_tracker.frame_kind(BAD_FRAMES["yuyv_on_cpu"]) == "yuv"
    assert multi_tracker.frame_kind([np.zeros((2, 2, 3), np.uint8)]) == "numpy"

    def no_device():
        raise AssertionError("the device is looked up only for a CUDA tensor")

    with pytest.raises(ValueError, match=r"^frame 3 is in a cpu tensor"):
        multi_tracker.check_device_frame(3, BAD_FRAMES["cpu_tensor"], "cuda", no_device)
    with pytest.raises(ValueError, match=r"^frame 0 must be a uint8 HxWx3 RGB tensor, got torch.uint8 \(64, 80, 4\)"):
        multi_tracker.check_device_frame(0, BAD_FRAMES["four_channels"], "cuda", no_device)
    with pytest.raises(ValueError, match=r"^frame 1 is in a cpu tensor"):
        multi_tracker.check_device_frame(1, BAD_FRAMES["i444_on_cpu"], "yuv", no_device)
    frames = [torch.zeros(6, 7, 3, dtype=torch.uint8), torch.zeros(3, 6, 7, dtype=torch.uint8).permute(1, 2, 0)]
    table = np.zeros(2, multi_tracker.TABLE_DTYPES["views"])
    multi_tracker.write_records(table, frames, "views")
    assert table.tolist() == [multi_tracker.frame_view(f) for f in frames]
    yuv = [BAD_FRAMES["nv12_on_cpu"], BAD_FRAMES["yuyv_on_cpu"]]
    table = np.zeros(2, multi_tracker.TABLE_DTYPES["ycbcr"])
    multi_tracker.write_records(table, yuv, "ycbcr")
    assert table.tolist() == [f.ycbcr_record() for f in yuv]
    table = np.zeros(1, multi_tracker.TABLE_DTYPES["yuv"])
    multi_tracker.write_records(table, yuv[:1], "yuv")
    assert table.tolist() == [yuv[0].yuv_record()]


@pytest.mark.parametrize("bbox", [[163, 53, 45, 174], [-30, -20, 50, 40], [470, 250, 30, 30], [0, 0, 3, 3]])
@pytest.mark.parametrize("size,offset", [(256, 2.0), (128, 0.2)])
def test_crop_geometry_is_that_of_the_crops(bbox, size, offset):
    frame = np.random.default_rng(0).integers(0, 256, (256, 480, 3), dtype=np.uint8)
    mean = np.mean(frame, axis=(0, 1))
    _, box, ctx = image_ops.extended_crop(frame, bbox, size, offset, mean)
    params, box2, ctx2 = image_ops.crop_params(bbox, size, offset, mean)
    box3, ctx3 = image_ops.crop_geometry(bbox, size, offset)
    assert np.array_equal(box, box3) and np.array_equal(box2, box3)
    assert np.array_equal(ctx, ctx3) and np.array_equal(ctx2, ctx3)
    assert np.array_equal(params[4:7], image_ops.padding_color(mean))


def test_crop_geometry_refuses_zero_area():
    with pytest.raises(IndexError, match="zero area"):
        image_ops.crop_geometry([10, 10, 0, 5], 256, 2.0)


def test_padding_color_rounds_half_to_even_and_saturates():
    assert image_ops.padding_color([100.5, 101.5, -3.0]).tolist() == [100, 102, 0]
    assert image_ops.padding_color([255.5, 254.5, 0.5]).tolist() == [255, 254, 0]
