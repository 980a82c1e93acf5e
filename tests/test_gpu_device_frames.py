"""GPU tests of frames that are already in device memory: the FearFrameView entry points (fear_crop_targets_view_u8,
fear_advance_targets_view, fear_frame_sums_u8) and FEARMultiTracker fed CUDA tensors, strided views included.

Every comparison is exact: crops against cv2, boxes against the host rescale + clamp, padding colours against numpy's
mean, and every tracker output against the same tracker fed the same frames as numpy arrays."""
import os

import numpy as np
import pytest
import torch

import feartracker_b200 as fb
from feartracker_b200 import _lib, image_ops
from feartracker_b200.multi_tracker import frame_view
from oracle import fear_oracle as fo
from tests import test_gpu_multi_tracker as base
from tests.helpers import GOLDEN, golden, load_full_state

pytestmark = pytest.mark.gpu
CFG = fb.FEAR_XS_TRACKER_KWARGS
KINDS = ("hwc", "roi", "chw", "rgba")


@pytest.fixture(scope="module")
def net():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    n = fb.FEARNet(**fb.FEAR_XS_MODEL_KWARGS)
    n.load_state_dict(load_full_state(), strict=True)
    return n.cuda().eval()


@pytest.fixture(scope="module")
def clip():
    return fo.read_video_rgb(os.path.join(GOLDEN, "test.mp4"))


def as_view(frame: np.ndarray, kind: str) -> torch.Tensor:
    """A CUDA uint8 (H, W, 3) tensor equal to ``frame``: contiguous HWC, a region of interest of a larger frame,
    a CHW tensor permuted to HWC, or the RGB channels of an RGBA surface.  Freshly allocated on every call."""
    h, w = frame.shape[:2]
    t = torch.from_numpy(np.ascontiguousarray(frame)).cuda()
    if kind == "hwc":
        return t
    if kind == "roi":
        big = torch.full((h + 7, w + 9, 3), 77, dtype=torch.uint8, device="cuda")
        big[3:3 + h, 5:5 + w] = t
        return big[3:3 + h, 5:5 + w]
    if kind == "chw":
        return t.permute(2, 0, 1).contiguous().permute(1, 2, 0)
    if kind == "rgba":
        rgba = torch.full((h, w, 4), 201, dtype=torch.uint8, device="cuda")
        rgba[..., :3] = t
        return rgba[..., :3]
    raise ValueError(kind)


def view_table(records) -> torch.Tensor:
    return torch.from_numpy(np.array(records, dtype=_lib.VIEW_DTYPE).view(np.uint8).copy()).cuda()


# ---------------------------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("kind", KINDS)
def test_crop_view_kernel_matches_cv2(kind):
    lib = _lib.init(0)
    rng = np.random.default_rng(21)
    frames = [rng.integers(0, 256, s, dtype=np.uint8) for s in ((256, 480, 3), (181, 97, 3), (90, 333, 3))]
    means = [np.mean(f, axis=(0, 1)) for f in frames]
    targets = [
        (0, [163, 53, 45, 174]), (0, [-10, 100, 40, 30]), (0, [450, 20, 60, 40]), (0, [200, -15, 30, 50]),
        (0, [100, 240, 50, 40]), (0, [0, 0, 3, 3]), (0, [477, 253, 3, 3]), (0, [-50, 30, 600, 100]),  # wider than frame
        (2, [-300, -200, 900, 500]), (2, [330, 87, 3, 3]), (2, [5, 40, 320, 20]),
    ]
    for side in (1, 2, 3, 5, 9, 17, 33, 64, 120, 200):  # context sides from 1 px (offset 0.2) to 1000 px (offset 2)
        targets.append((1, [48 - side // 2, 90 - side // 2, side, side]))
    recs = np.zeros((len(targets) + 2, _lib.TARGET_INTS), dtype=np.int32)
    for i, (f, box) in enumerate(targets):
        recs[i, 0], recs[i, 1:5] = f, box
        recs[i, 9:12] = np.clip(np.rint(means[f]), 0, 255)
    recs[-2, 0], recs[-2, 1:5], recs[-2, 9:12] = 7, [10, 10, 20, 20], [12, 200, 255]  # frame index out of range
    recs[-1, 0], recs[-1, 1:5], recs[-1, 9:12] = 3, [10, 10, 20, 20], [99, 0, 31]  # view entry with H = 0
    tensors = [as_view(f, kind) for f in frames]
    views = [frame_view(t) for t in tensors]
    data, rs, ps, cs, h, w = views[0]
    table = view_table(views + [(data, rs, ps, cs, 0, w)])
    st = torch.cuda.current_stream().cuda_stream
    n = len(recs)
    for size, off in ((256, 2.0), (128, 0.2), (256, 0.5), (128, 2.0)):
        state = torch.from_numpy(recs).cuda()
        crops = torch.empty((n, size, size, 3), dtype=torch.uint8, device="cuda")
        _lib.check(lib.fear_crop_targets_view_u8(table.data_ptr(), len(views) + 1, state.data_ptr(), n, off, size,
                                                 crops.data_ptr(), st), "fear_crop_targets_view_u8")
        got, ctxs = crops.cpu().numpy(), state.cpu().numpy()[:, 5:9]
        for i, (f, box) in enumerate(targets):
            assert np.array_equal(ctxs[i], image_ops.context_box(box, off)), (kind, size, off, box)
            want = base._cv2_crop(frames[f], box, size, off, means[f])
            assert np.array_equal(got[i], want), (kind, size, off, f, box)
        assert (got[-2] == np.array([12, 200, 255], dtype=np.uint8)).all()
        assert (got[-1] == np.array([99, 0, 31], dtype=np.uint8)).all()
        assert np.array_equal(ctxs[-1], image_ops.context_box([10, 10, 20, 20], off))


def test_advance_view_kernel_matches_host_rescale_and_clamp():
    lib = _lib.init(0)
    rng = np.random.default_rng(5)
    shapes = [(256, 480), (181, 97), (2, 2)]  # the last frame is smaller than the minimum side
    n = 12000
    boxes = np.zeros(n, dtype=_lib.BOX_DTYPE)
    recs = np.zeros((n, _lib.TARGET_INTS), dtype=np.int32)
    recs[:, 0] = rng.integers(0, 3, n)
    recs[:, 5:7] = rng.integers(-600, 700, (n, 2))
    recs[:, 7:9] = rng.integers(1, 2000, (n, 2))
    xy = rng.uniform(-300, 600, (n, 2))
    wh = rng.uniform(0, 300, (n, 2))
    wh[n // 4:n // 2] = rng.uniform(0, 3, (n // 4, 2))  # sides below 3
    # exact .5 after scaling: cw = 512 (scale 2) with x = k + 0.25, cw = 256 (scale 1) with x = k + 0.5
    half = slice(n // 2, 3 * n // 4)
    side = rng.choice([256, 512], n // 4)
    recs[half, 7] = recs[half, 8] = side
    v = rng.integers(-200, 300, (n // 4, 4)) + np.where(side == 512, 0.25, 0.5)[:, None]
    xy[half], wh[half] = v[:, :2], np.abs(v[:, 2:])
    boxes["x"], boxes["y"], boxes["w"], boxes["h"] = xy[:, 0], xy[:, 1], wh[:, 0], wh[:, 1]
    recs[-10:-5, 0] = 9  # frame index out of range: the box is kept
    recs[-5:, 0] = 3  # view entry with data == NULL: the box is kept
    recs[-10:, 1:5] = [7, 8, 9, 10]
    kinds = ["rgba", "chw", "roi"]
    tensors = [as_view(np.zeros(s + (3,), np.uint8), k) for s, k in zip(shapes, kinds)]
    table = view_table([frame_view(t) for t in tensors] + [(0, 3 * 480, 3, 1, 256, 480)])
    state = torch.from_numpy(recs).cuda()
    dboxes = torch.from_numpy(boxes.view(np.uint8).copy()).cuda()
    _lib.check(lib.fear_advance_targets_view(dboxes.data_ptr(), table.data_ptr(), 4, state.data_ptr(), n, 256,
                                             torch.cuda.current_stream().cuda_stream), "fear_advance_targets_view")
    got = state.cpu().numpy()
    for i in range(n - 10):
        b = np.array([boxes["x"][i], boxes["y"][i], boxes["w"][i], boxes["h"][i]])
        h, w = shapes[recs[i, 0]]
        want = image_ops.clamp_bbox(image_ops.rescale_bbox(b, recs[i, 5:9], 256), (h, w, 3))
        assert np.array_equal(got[i, 1:5], want), (i, b.tolist(), recs[i, 5:9].tolist(), (h, w), got[i, 1:5], want)
    assert (got[-10:, 1:5] == [7, 8, 9, 10]).all()
    assert np.array_equal(np.delete(got, np.s_[1:5], axis=1), np.delete(recs, np.s_[1:5], axis=1))


def test_frame_sums_give_numpy_mean_padding():
    lib = _lib.init(0)
    rng = np.random.default_rng(8)
    half = np.zeros((2, 2, 3), np.uint8)  # means exactly 0.5, 2.5 and 254.5: rint rounds half to even
    half[..., 0] = [[0, 1], [0, 1]]
    half[..., 1] = [[2, 3], [3, 2]]
    half[..., 2] = [[254, 255], [255, 254]]
    frames = [np.full((1, 1, 3), [7, 0, 255], np.uint8), rng.integers(0, 256, (181, 97, 3), dtype=np.uint8),
              rng.integers(0, 256, (37, 1001, 3), dtype=np.uint8), rng.integers(0, 256, (1, 513, 3), dtype=np.uint8),
              rng.integers(0, 256, (2160, 3840, 3), dtype=np.uint8), half,
              rng.integers(0, 256, (3, 5, 3), dtype=np.uint8)]
    kinds = ["hwc", "rgba", "chw", "roi", "hwc", "roi", "chw"]
    tensors = [as_view(f, k) for f, k in zip(frames, kinds)]
    views = [frame_view(t) for t in tensors]
    views += [(0, 0, 0, 0, 4, 4), views[1][:4] + (0, 97)]  # data == NULL, H = 0: both sum to 0
    table = view_table(views)
    sums = torch.full((len(views), 3), -1, dtype=torch.int64, device="cuda")  # zeroed by the call
    _lib.check(lib.fear_frame_sums_u8(table.data_ptr(), len(views), sums.data_ptr(),
                                      torch.cuda.current_stream().cuda_stream), "fear_frame_sums_u8")
    got = sums.cpu().numpy().view(np.uint64)
    for i, f in enumerate(frames):
        assert np.array_equal(got[i], f.sum(axis=(0, 1), dtype=np.uint64)), (i, f.shape)
        pad = np.clip(np.rint(got[i] / np.float64(f.shape[0] * f.shape[1])), 0, 255)
        assert np.array_equal(pad, np.clip(np.rint(np.mean(f, axis=(0, 1))), 0, 255)), (i, f.shape)
    assert np.array_equal(np.clip(np.rint(got[5] / 4.0), 0, 255), [0, 2, 254])
    assert (got[-2:] == 0).all()


# ---------------------------------------------------------------------------------------------------- tracker
def _assert_same(out, want, what):
    assert np.array_equal(out["ids"], want["ids"]), what
    assert np.array_equal(out["bbox"], want["bbox"]), (what, out["bbox"], want["bbox"])
    assert np.array_equal(out["score"], want["score"]), what


def test_several_streams_of_cuda_views_match_numpy_frames(net, clip):
    T = 150
    streams = {"clip": clip[:T + 1], "mirror": np.ascontiguousarray(clip[:T + 1, :, ::-1]),
               "window": np.ascontiguousarray(clip[:T + 1, 30:200, 50:350])}
    rects = {"clip": [base.GOLDEN_BOX, [420, 10, 50, 60]], "mirror": [[272, 53, 45, 174], [0, 180, 40, 70]],
             "window": [[113, 23, 45, 120], [250, 140, 60, 40]]}
    names = list(streams)
    all_rects = [r for s in names for r in rects[s]]
    stream_idx = [names.index(s) for s in names for _ in rects[s]]
    ref = fb.FEARMultiTracker(net, cuda_id=0, max_targets=8, **CFG)
    dev = fb.FEARMultiTracker(net, cuda_id=0, max_targets=8, **CFG)
    ref.add([streams[s][0] for s in names], all_rects, stream_idx)
    dev.add([as_view(streams[s][0], KINDS[j]) for j, s in enumerate(names)], all_rects, stream_idx)
    graph, held, golden_boxes = None, None, []
    for t in range(1, T + 1):
        frames = [as_view(streams[s][t], KINDS[(j + t) % 4]) for j, s in enumerate(names)]
        if held is not None:  # the previous update's tensors are still alive: these frames lie elsewhere
            assert all(a.data_ptr() != b.data_ptr() for a, b in zip(frames, held))
        out = dev.update(frames)
        _assert_same(out, ref.update([streams[s][t] for s in names]), t)
        golden_boxes.append(out["bbox"][0])
        held = frames
        if t == 2:
            graph = dev._graph
            assert graph is not None
    assert dev._graph is graph  # captured once, replayed with new frame addresses every update
    assert np.array_equal(np.array(golden_boxes), golden("video_teacher.npz")["trajectory"][:T])


def test_alternating_kinds_and_add_remove_with_cuda_frames(net, clip):
    start_rects = base.CLIP_TARGETS[:4]
    late_rects = [[300, 80, 60, 90], [100, 150, 30, 30]]
    ref = fb.FEARMultiTracker(net, cuda_id=0, max_targets=8, **CFG)
    dev = fb.FEARMultiTracker(net, cuda_id=0, max_targets=8, **CFG)
    assert np.array_equal(ref.initialize(clip[0], start_rects), dev.initialize(as_view(clip[0], "chw"), start_rects))
    for f in range(1, 161):
        if f == 120:
            ref.remove([1])
            dev.remove([1])
        frame = clip[f] if f % 2 else as_view(clip[f], KINDS[(f // 2) % 4])
        _assert_same(dev.update(frame), ref.update(clip[f]), f)
        if f == 60:
            assert np.array_equal(ref.add(clip[60], late_rects), dev.add([as_view(clip[60], "rgba")], late_rects))
    assert len(dev) == 5


def test_launch_count_same_for_both_kinds_and_does_not_grow(net, clip):
    window = np.ascontiguousarray(clip[:4, 30:200, 50:350])
    deltas = {}
    for n in (1, 16):
        for num_frames in (1, 3):
            for kind in ("numpy", "cuda"):
                def frames(t):
                    fs = [clip[t], window[t], clip[t]][:num_frames]
                    return fs if kind == "numpy" else [as_view(f, "roi") for f in fs]

                trk = fb.FEARMultiTracker(net, cuda_id=0, max_targets=16, cuda_graph=False, **CFG)
                trk.initialize(frames(0), [base.GOLDEN_BOX] * n, [i % num_frames for i in range(n)])
                trk.update(frames(1))
                torch.cuda.synchronize()
                c0 = net.launch_count()
                trk.update(frames(2))
                trk.update(frames(3))
                deltas[(n, num_frames, kind)] = (net.launch_count() - c0) / 2
    assert len(set(deltas.values())) == 1 and deltas[(1, 1, "numpy")] > 0, deltas


def test_c_abi_rejects_bad_arguments():
    lib = _lib.load()
    t = torch.zeros(4096, dtype=torch.uint8, device="cuda")
    p = t.data_ptr()
    good = dict(views=p, F=1, targets=p, N=1, offset=2.0, size=256, crops=p)

    def crop(**kw):
        a = dict(good, **kw)
        return lib.fear_crop_targets_view_u8(a["views"], a["F"], a["targets"], a["N"], a["offset"], a["size"],
                                             a["crops"], None)

    bad = [dict(views=None), dict(targets=None), dict(crops=None), dict(N=0), dict(N=65536), dict(F=0), dict(size=0),
           dict(size=257), dict(offset=-0.5), dict(offset=float("nan")), dict(offset=float("inf"))]
    for kw in bad:
        assert crop(**kw) == -1, kw
        assert _lib.last_error(), kw
    for args in [(None, p, 1, p, 1, 256), (p, None, 1, p, 1, 256), (p, p, 1, None, 1, 256), (p, p, 1, p, 0, 256),
                 (p, p, 0, p, 1, 256), (p, p, 1, p, 1, 0)]:
        assert lib.fear_advance_targets_view(*args, None) == -1, args
        assert _lib.last_error(), args
    for args in [(None, 1, p), (p, 1, None), (p, 0, p), (p, 65536, p), (p, -1, p)]:
        assert lib.fear_frame_sums_u8(*args, None) == -1, args
        assert _lib.last_error(), args
