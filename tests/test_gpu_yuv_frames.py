"""GPU tests of YUV 4:2:0 frames: the FearFrameYUV420 entry points (fear_crop_targets_yuv420_u8,
fear_advance_targets_yuv420, fear_frame_sums_yuv420_u8) and FEARMultiTracker fed YUV420Frames.

Every comparison is exact: the conversion against cv2.cvtColor over all 2^24 (Y, U, V) triples, crops against cv2 on
the cv2-converted frame, boxes against the host rescale + clamp, padding colours against numpy's mean, and every
tracker output against the same tracker fed the cv2-converted frames as numpy arrays."""
import os

import cv2
import numpy as np
import pytest
import torch

import feartracker_b200 as fb
from feartracker_b200 import _lib, image_ops
from oracle import fear_oracle as fo
from tests import test_gpu_multi_tracker as base
from tests.helpers import GOLDEN, load_full_state
from tests.test_yuv_frames_cpu import LAYOUTS, yuv_frame

pytestmark = pytest.mark.gpu
CFG = fb.FEAR_XS_TRACKER_KWARGS


@pytest.fixture(scope="module")
def net():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    n = fb.FEARNet(**fb.FEAR_XS_MODEL_KWARGS)
    n.load_state_dict(load_full_state(), strict=True)
    return n.cuda().eval()


@pytest.fixture(scope="module")
def clip():
    return fo.read_video_rgb(os.path.join(GOLDEN, "test.mp4"))


def yuv_table(records) -> torch.Tensor:
    return torch.from_numpy(np.array(records, dtype=_lib.YUV420_DTYPE).view(np.uint8).copy()).cuda()


def to_rgb(i420: np.ndarray) -> np.ndarray:
    return cv2.cvtColor(i420, cv2.COLOR_YUV2RGB_I420)


def random_i420(rng, h, w) -> np.ndarray:
    return rng.integers(0, 256, (h * 3 // 2, w), dtype=np.uint8)


def empty_records(rec):
    """Entries the kernels treat as empty, derived from a valid record: a null plane, H = 0, an odd W."""
    null_u, no_rows, odd_w = list(rec), list(rec), list(rec)
    null_u[1], no_rows[7], odd_w[8] = 0, 0, rec[8] - 1
    return [tuple(null_u), tuple(no_rows), tuple(odd_w)]


# ---------------------------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("layout", ["nv12", "i420"])
def test_conversion_matches_cv2_on_every_yuv_triple(layout):
    """64 frames of 512 x 512: chroma block (i, j) holds (U, V) = (i, j), and the luma of 2 x 2 position (dy, dx) in
    frame k is 4k + 2dy + dx, so the frames hold every (Y, U, V) triple.  Offset 0 and out_size 256 on the four
    256 x 256 quadrants make the crop an identity resample (coefficients (2048, 0)): crop = converted frame."""
    lib = _lib.init(0)
    i, j = np.meshgrid(np.arange(256, dtype=np.uint8), np.arange(256, dtype=np.uint8), indexing="ij")
    frames, want = [], []
    for k in range(64):
        y = np.empty((512, 512), np.uint8)
        for dy in range(2):
            for dx in range(2):
                y[dy::2, dx::2] = 4 * k + 2 * dy + dx
        i420 = np.concatenate([y.reshape(-1), i.reshape(-1), j.reshape(-1)]).reshape(768, 512)
        frames.append(yuv_frame(i420, layout))
        want.append(to_rgb(i420) if layout == "i420" else
                    cv2.cvtColor(np.concatenate([y, np.stack([i, j], -1).reshape(256, 512)]), cv2.COLOR_YUV2RGB_NV12))
    quads = [(0, 0), (256, 0), (0, 256), (256, 256)]
    recs = np.zeros((64 * 4, _lib.TARGET_INTS), dtype=np.int32)
    for k in range(64):
        for q, (x, y) in enumerate(quads):
            recs[4 * k + q, 0], recs[4 * k + q, 1:5] = k, [x, y, 256, 256]
    state = torch.from_numpy(recs).cuda()
    crops = torch.empty((len(recs), 256, 256, 3), dtype=torch.uint8, device="cuda")
    table = yuv_table([f.record() for f in frames])
    _lib.check(lib.fear_crop_targets_yuv420_u8(table.data_ptr(), 64, state.data_ptr(), len(recs), 0.0, 256,
                                               crops.data_ptr(), torch.cuda.current_stream().cuda_stream),
               "fear_crop_targets_yuv420_u8")
    got = crops.cpu().numpy()
    for k in range(64):
        for q, (x, y) in enumerate(quads):
            assert np.array_equal(got[4 * k + q], want[k][y:y + 256, x:x + 256]), (layout, k, q)


@pytest.mark.parametrize("layout", LAYOUTS)
def test_crop_yuv420_kernel_matches_cv2(layout):
    lib = _lib.init(0)
    rng = np.random.default_rng(23)
    i420s = [random_i420(rng, h, w) for h, w in ((256, 480), (182, 98), (90, 334))]
    rgbs = [to_rgb(f) for f in i420s]
    means = [np.mean(f, axis=(0, 1)) for f in rgbs]
    targets = [  # the targets of test_gpu_device_frames.test_crop_view_kernel_matches_cv2
        (0, [163, 53, 45, 174]), (0, [-10, 100, 40, 30]), (0, [450, 20, 60, 40]), (0, [200, -15, 30, 50]),
        (0, [100, 240, 50, 40]), (0, [0, 0, 3, 3]), (0, [477, 253, 3, 3]), (0, [-50, 30, 600, 100]),
        (2, [-300, -200, 900, 500]), (2, [330, 87, 3, 3]), (2, [5, 40, 320, 20]),
    ]
    for side in (1, 2, 3, 5, 9, 17, 33, 64, 120, 200):
        targets.append((1, [48 - side // 2, 90 - side // 2, side, side]))
    # frame index out of range, then the three empty entries (null plane, H = 0, odd W)
    extra = [(7, [12, 200, 255]), (3, [99, 0, 31]), (4, [1, 2, 3]), (5, [250, 128, 7])]
    recs = np.zeros((len(targets) + len(extra), _lib.TARGET_INTS), dtype=np.int32)
    for i, (f, box) in enumerate(targets):
        recs[i, 0], recs[i, 1:5] = f, box
        recs[i, 9:12] = np.clip(np.rint(means[f]), 0, 255)
    for i, (f, pad) in enumerate(extra):
        recs[len(targets) + i, 0], recs[len(targets) + i, 1:5], recs[len(targets) + i, 9:12] = f, [10, 10, 20, 20], pad
    frames = [yuv_frame(f, layout) for f in i420s]
    records = [f.record() for f in frames]
    table = yuv_table(records + empty_records(records[0]))
    st = torch.cuda.current_stream().cuda_stream
    n = len(recs)
    for size, off in ((256, 2.0), (128, 0.2), (256, 0.5), (128, 2.0)):
        state = torch.from_numpy(recs).cuda()
        crops = torch.empty((n, size, size, 3), dtype=torch.uint8, device="cuda")
        _lib.check(lib.fear_crop_targets_yuv420_u8(table.data_ptr(), len(records) + 3, state.data_ptr(), n, off, size,
                                                   crops.data_ptr(), st), "fear_crop_targets_yuv420_u8")
        got, ctxs = crops.cpu().numpy(), state.cpu().numpy()[:, 5:9]
        for i, (f, box) in enumerate(targets):
            assert np.array_equal(ctxs[i], image_ops.context_box(box, off)), (layout, size, off, box)
            want = base._cv2_crop(rgbs[f], box, size, off, means[f])
            assert np.array_equal(got[i], want), (layout, size, off, f, box)
        for i, (_, pad) in enumerate(extra):
            assert (got[len(targets) + i] == np.array(pad, dtype=np.uint8)).all(), (layout, i)
            assert np.array_equal(ctxs[len(targets) + i], image_ops.context_box([10, 10, 20, 20], off))


def test_advance_yuv420_kernel_matches_host_rescale_and_clamp():
    """The records of test_gpu_device_frames.test_advance_view_kernel_matches_host_rescale_and_clamp, on YUV frames
    (even sizes)."""
    lib = _lib.init(0)
    rng = np.random.default_rng(5)
    shapes = [(256, 480), (182, 98), (2, 2)]  # the last frame is smaller than the minimum side
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
    recs[-16:-12, 0] = 9  # frame index out of range: the box is kept
    recs[-12:, 0] = np.repeat([3, 4, 5], 4)  # empty entries (null plane, H = 0, odd W): the box is kept
    recs[-16:, 1:5] = [7, 8, 9, 10]
    frames = [yuv_frame(np.zeros((h * 3 // 2, w), np.uint8), k) for (h, w), k in zip(shapes, ["pitched", "roi", "i420"])]
    records = [f.record() for f in frames]
    table = yuv_table(records + empty_records(records[0]))
    state = torch.from_numpy(recs).cuda()
    dboxes = torch.from_numpy(boxes.view(np.uint8).copy()).cuda()
    _lib.check(lib.fear_advance_targets_yuv420(dboxes.data_ptr(), table.data_ptr(), 6, state.data_ptr(), n, 256,
                                               torch.cuda.current_stream().cuda_stream), "fear_advance_targets_yuv420")
    got = state.cpu().numpy()
    for i in range(n - 16):
        b = np.array([boxes["x"][i], boxes["y"][i], boxes["w"][i], boxes["h"][i]])
        h, w = shapes[recs[i, 0]]
        want = image_ops.clamp_bbox(image_ops.rescale_bbox(b, recs[i, 5:9], 256), (h, w, 3))
        assert np.array_equal(got[i, 1:5], want), (i, b.tolist(), recs[i, 5:9].tolist(), (h, w), got[i, 1:5], want)
    assert (got[-16:, 1:5] == [7, 8, 9, 10]).all()
    assert np.array_equal(np.delete(got, np.s_[1:5], axis=1), np.delete(recs, np.s_[1:5], axis=1))


def test_frame_sums_yuv420_give_numpy_mean_of_converted_frame():
    lib = _lib.init(0)
    rng = np.random.default_rng(9)
    sizes = [(2, 2), (182, 98), (38, 1002), (2, 514), (2160, 3840), (4, 6), (90, 334), (1080, 1920)]
    i420s = [random_i420(rng, h, w) for h, w in sizes]
    layouts = ["nv12", "pitched", "roi", "planes", "pitched", "i420", "roi", "nv12"]
    frames = [yuv_frame(f, k) for f, k in zip(i420s, layouts)]
    records = [f.record() for f in frames]
    table = yuv_table(records + empty_records(records[1]))
    sums = torch.full((len(records) + 3, 3), -1, dtype=torch.int64, device="cuda")  # zeroed by the call
    _lib.check(lib.fear_frame_sums_yuv420_u8(table.data_ptr(), len(records) + 3, sums.data_ptr(),
                                             torch.cuda.current_stream().cuda_stream), "fear_frame_sums_yuv420_u8")
    got = sums.cpu().numpy().view(np.uint64)
    for i, f in enumerate(i420s):
        rgb = to_rgb(f)
        assert np.array_equal(got[i], rgb.sum(axis=(0, 1), dtype=np.uint64)), (i, sizes[i])
        pad = np.clip(np.rint(got[i] / np.float64(rgb.shape[0] * rgb.shape[1])), 0, 255)
        assert np.array_equal(pad, np.clip(np.rint(np.mean(rgb, axis=(0, 1))), 0, 255)), (i, sizes[i])
    assert (got[-3:] == 0).all()


# ---------------------------------------------------------------------------------------------------- tracker
def _assert_same(out, want, what):
    assert np.array_equal(out["ids"], want["ids"]), what
    assert np.array_equal(out["bbox"], want["bbox"]), (what, out["bbox"], want["bbox"])
    assert np.array_equal(out["score"], want["score"]), what


def test_yuv_streams_match_trackers_fed_cv2_converted_frames(net, clip):
    """A pitched-NV12 stream of the demo clip (480 x 256) and a 1920 x 1080 I420 stream, several targets each, add /
    remove part way.  One tracker gets YUV420Frames every update, another alternates YUV, numpy-RGB and CUDA-RGB
    calls; both must give every output of a tracker fed cv2.cvtColor's RGB frames as numpy arrays.  Every frame is
    freshly allocated, and the YUV-only tracker replays one captured graph."""
    T = 60
    i420 = {"clip": [cv2.cvtColor(clip[t], cv2.COLOR_RGB2YUV_I420) for t in range(T + 1)],
            "hd": [cv2.cvtColor(cv2.resize(clip[t], (1920, 1080)), cv2.COLOR_RGB2YUV_I420) for t in range(T + 1)]}
    layouts = {"clip": "pitched", "hd": "i420"}
    names = list(i420)
    rgb = {s: [to_rgb(f) for f in i420[s]] for s in names}
    start = {"clip": [base.GOLDEN_BOX, [168, 50, 40, 170], [300, 80, 60, 90], [-10, 100, 50, 50]],
             "hd": [[652, 211, 180, 696], [640, 230, 200, 650], [1760, 840, 160, 224]]}
    late = {"clip": [[100, 150, 30, 30]], "hd": [[400, 600, 120, 120]]}

    def rects(d):
        return [r for s in names for r in d[s]], [k for k, s in enumerate(names) for _ in d[s]]

    def yuv(t):
        return [yuv_frame(i420[s][t], layouts[s]) for s in names]

    def frames(mode, t):
        if mode == "yuv":
            return yuv(t)
        if mode == "numpy":
            return [rgb[s][t] for s in names]
        return [torch.from_numpy(rgb[s][t]).cuda() for s in names]

    ref = fb.FEARMultiTracker(net, cuda_id=0, max_targets=12, **CFG)
    only = fb.FEARMultiTracker(net, cuda_id=0, max_targets=12, **CFG)
    mixed = fb.FEARMultiTracker(net, cuda_id=0, max_targets=12, **CFG)
    r, s = rects(start)
    want = ref.add(frames("numpy", 0), r, s)
    assert np.array_equal(only.add(yuv(0), r, s), want)
    assert np.array_equal(mixed.add(yuv(0), r, s), want)
    graph, held = None, None
    for t in range(1, T + 1):
        if t == 25:
            r, s = rects(late)
            want = ref.add(frames("numpy", t - 1), r, s)
            assert np.array_equal(only.add(yuv(t - 1), r, s), want)
            assert np.array_equal(mixed.add(frames("cuda", t - 1), r, s), want)
        if t == 40:
            for trk in (ref, only, mixed):
                trk.remove([2, 5])
        expect = ref.update(frames("numpy", t))
        fresh = yuv(t)
        if held is not None:  # the previous update's planes are still alive: these frames lie elsewhere
            assert all(a.y.data_ptr() != b.y.data_ptr() for a, b in zip(fresh, held))
        _assert_same(only.update(fresh), expect, ("yuv", t))
        held = fresh
        _assert_same(mixed.update(frames(("yuv", "numpy", "cuda")[t % 3], t)), expect, ("mixed", t))
        if t in (27, 42):  # two updates after the add (warm-up + capture) and after the remove
            graph = only._graph
            assert graph is not None
        if t in (39, T):
            assert only._graph is graph  # replayed with new frame addresses every update
    assert len(only) == 7


def test_launch_count_of_yuv_step_equals_rgb_step_and_does_not_grow(net, clip):
    rgb = [clip[:4], np.ascontiguousarray(clip[:4, 30:200, 50:350]), clip[:4]]
    i420 = [[cv2.cvtColor(f, cv2.COLOR_RGB2YUV_I420) for f in a] for a in rgb]
    deltas = {}
    for n in (1, 16):
        for num_frames in (1, 3):
            for kind in ("cuda", "yuv"):
                def frames(t):
                    if kind == "cuda":
                        return [torch.from_numpy(np.ascontiguousarray(a[t])).cuda() for a in rgb[:num_frames]]
                    return [yuv_frame(a[t], "pitched") for a in i420[:num_frames]]

                trk = fb.FEARMultiTracker(net, cuda_id=0, max_targets=16, cuda_graph=False, **CFG)
                trk.initialize(frames(0), [base.GOLDEN_BOX] * n, [i % num_frames for i in range(n)])
                trk.update(frames(1))
                torch.cuda.synchronize()
                c0 = net.launch_count()
                trk.update(frames(2))
                trk.update(frames(3))
                deltas[(n, num_frames, kind)] = (net.launch_count() - c0) / 2
    assert len(set(deltas.values())) == 1 and deltas[(1, 1, "cuda")] > 0, deltas


def test_c_abi_rejects_bad_arguments_and_launches_nothing():
    lib = _lib.init(0)
    t = torch.full((1 << 16,), 0x5A, dtype=torch.uint8, device="cuda")
    p = t.data_ptr()
    good = dict(views=p, F=1, targets=p, N=1, offset=2.0, size=256, crops=p)

    def crop(**kw):
        a = dict(good, **kw)
        return lib.fear_crop_targets_yuv420_u8(a["views"], a["F"], a["targets"], a["N"], a["offset"], a["size"],
                                               a["crops"], None)

    bad = [dict(views=None), dict(targets=None), dict(crops=None), dict(N=0), dict(N=-1), dict(N=65536), dict(F=0),
           dict(F=-3), dict(size=0), dict(size=257), dict(offset=-0.5), dict(offset=float("nan")),
           dict(offset=float("inf"))]
    for kw in bad:
        assert crop(**kw) == -1, kw
        assert _lib.last_error(), kw
    for args in [(None, p, 1, p, 1, 256), (p, None, 1, p, 1, 256), (p, p, 1, None, 1, 256), (p, p, 1, p, 0, 256),
                 (p, p, 0, p, 1, 256), (p, p, 1, p, 1, 0)]:
        assert lib.fear_advance_targets_yuv420(*args, None) == -1, args
        assert _lib.last_error(), args
    for args in [(None, 1, p), (p, 1, None), (p, 0, p), (p, 65536, p), (p, -1, p)]:
        assert lib.fear_frame_sums_yuv420_u8(*args, None) == -1, args
        assert _lib.last_error(), args
    torch.cuda.synchronize()
    assert (t == 0x5A).all()  # no kernel and no memset ran
