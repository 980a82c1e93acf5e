"""GPU tests of FEARMultiTracker and its two device kernels (fear_crop_targets_u8, fear_advance_targets).

Every comparison is exact: the crop kernel against cv2 (image_ops.extended_crop), the advance kernel against the host
rescale + clamp, and every tracked target against its own FEARTracker(gpu_crop=True) on every frame."""
import os

import cv2
import numpy as np
import pytest
import torch

import feartracker_b200 as fb
from feartracker_b200 import _lib, image_ops
from oracle import fear_oracle as fo
from tests.helpers import GOLDEN, golden, load_full_state

pytestmark = pytest.mark.gpu
CFG = fb.FEAR_XS_TRACKER_KWARGS
GOLDEN_BOX = [163, 53, 45, 174]
# 8 targets on the demo clip (480 x 256): the golden one, targets at / beyond every edge, a duplicate of the golden one
CLIP_TARGETS = [GOLDEN_BOX, [0, 0, 40, 60], [440, 200, 40, 56], [-10, 100, 50, 50], [470, 250, 30, 30],
                GOLDEN_BOX, [300, 80, 60, 90], [100, 150, 30, 30]]


@pytest.fixture(scope="module")
def net():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    n = fb.FEARNet(**fb.FEAR_XS_MODEL_KWARGS)
    n.load_state_dict(load_full_state(), strict=True)
    return n.cuda().eval()


@pytest.fixture(scope="module")
def clip():
    return fo.read_video_rgb(os.path.join(GOLDEN, "test.mp4"))


_INDEPENDENT = {}


def independent(net, stream, frames, rect, start=0, stop=None):
    """(boxes (T, 4) int64, scores (T,) float32) of FEARTracker(gpu_crop=True) initialised on frames[start] and
    updated on frames[start + 1:stop]; cached per (stream name, start, stop, rect)."""
    key = (stream, start, stop, tuple(rect))
    if key not in _INDEPENDENT:
        trk = fb.FEARTracker(net, cuda_id=0, gpu_crop=True, **CFG)
        trk.initialize(frames[start], np.asarray(rect))
        scores = []
        record = trk._track_record_gpu_crop

        def keep_score(image, params):  # FEARTracker.track's score, which update() does not return
            rec = record(image, params)
            scores.append(np.float32(rec["score"]))
            return rec

        trk._track_record_gpu_crop = keep_score
        boxes = [trk.update(f)["bbox"] for f in frames[start + 1:stop]]
        _INDEPENDENT[key] = (np.array(boxes, dtype=np.int64).reshape(-1, 4), np.array(scores, dtype=np.float32))
    return _INDEPENDENT[key]


def run_multi(trk, frame_lists):
    """update() over a list of per-step frame lists -> (boxes (T, N, 4), scores (T, N))."""
    outs = [trk.update(fr) for fr in frame_lists]
    return np.stack([o["bbox"] for o in outs]), np.stack([o["score"] for o in outs])


def assert_matches_independent(net, stream, frames, rects, boxes, scores, start=0):
    for i, rect in enumerate(rects):
        want_b, want_s = independent(net, stream, frames, rect, start, start + 1 + boxes.shape[0])
        same = (boxes[:, i] == want_b).all(1)
        assert same.all(), (stream, i, rect, int(np.argmin(same)), boxes[np.argmin(same), i], want_b[np.argmin(same)])
        assert np.array_equal(scores[:, i], want_s), (stream, i, rect, int(np.argmin(scores[:, i] == want_s)))


# ---------------------------------------------------------------------------------------------------- kernels
def _cv2_crop(frame, box, size, off, mean):
    """image_ops.extended_crop's image; boxes with no area inside their context (which extended_crop refuses) take
    the same copyMakeBorder + resize steps directly."""
    try:
        return image_ops.extended_crop(frame, box, size, off, mean)[0]
    except IndexError:
        ctx = image_ops.context_box(box, off)
        h, w = frame.shape[:2]
        left, top = max(-ctx[0], 0), max(-ctx[1], 0)
        right, bottom = max(ctx[0] + ctx[2] - w, 0), max(ctx[1] + ctx[3] - h, 0)
        inner = frame[ctx[1] + top: ctx[1] + ctx[3] - bottom, ctx[0] + left: ctx[0] + ctx[2] - right]
        padded = cv2.copyMakeBorder(inner, top, bottom, left, right, cv2.BORDER_CONSTANT, value=mean)
        if padded.shape[:2] == (size, size):
            return padded
        return cv2.resize(padded, dsize=(size, size), interpolation=cv2.INTER_LINEAR)


def _pack_frames(frames):
    table = np.zeros(len(frames), dtype=_lib.FRAME_DTYPE)
    off, parts = 0, []
    for i, f in enumerate(frames):
        table[i] = (off, f.shape[0], f.shape[1])
        n = -(-f.size // 16) * 16
        parts.append(np.pad(f.reshape(-1), (0, n - f.size)))
        off += n
    return (torch.from_numpy(np.concatenate(parts)).cuda(), torch.from_numpy(table.view(np.uint8).copy()).cuda())


def test_crop_kernel_matches_cv2():
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
    recs = np.zeros((len(targets) + 1, _lib.TARGET_INTS), dtype=np.int32)
    for i, (f, box) in enumerate(targets):
        recs[i, 0], recs[i, 1:5] = f, box
        recs[i, 9:12] = np.clip(np.rint(means[f]), 0, 255)
    recs[-1, 0], recs[-1, 1:5], recs[-1, 9:12] = 7, [10, 10, 20, 20], [12, 200, 255]  # frame index out of range
    fbuf, table = _pack_frames(frames)
    st = torch.cuda.current_stream().cuda_stream
    n = len(recs)
    for size, off in ((256, 2.0), (128, 0.2), (256, 0.5), (128, 2.0)):
        state = torch.from_numpy(recs).cuda()
        crops = torch.empty((n, size, size, 3), dtype=torch.uint8, device="cuda")
        _lib.check(lib.fear_crop_targets_u8(fbuf.data_ptr(), table.data_ptr(), len(frames), state.data_ptr(), n, off,
                                            size, crops.data_ptr(), st), "fear_crop_targets_u8")
        got, ctxs = crops.cpu().numpy(), state.cpu().numpy()[:, 5:9]
        for i, (f, box) in enumerate(targets):
            assert np.array_equal(ctxs[i], image_ops.context_box(box, off)), (size, off, box)
            assert np.array_equal(got[i], _cv2_crop(frames[f], box, size, off, means[f])), (size, off, f, box)
        assert (got[-1] == np.array([12, 200, 255], dtype=np.uint8)).all()


def test_advance_kernel_matches_host_rescale_and_clamp():
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
    recs[-5:, 0] = 9  # frame index out of range: the box is kept
    recs[-5:, 1:5] = [7, 8, 9, 10]
    frames = [np.zeros(s + (3,), np.uint8) for s in shapes]
    fbuf, table = _pack_frames(frames)
    state = torch.from_numpy(recs).cuda()
    dboxes = torch.from_numpy(boxes.view(np.uint8).copy()).cuda()
    _lib.check(lib.fear_advance_targets(dboxes.data_ptr(), table.data_ptr(), len(frames), state.data_ptr(), n, 256,
                                        torch.cuda.current_stream().cuda_stream), "fear_advance_targets")
    got = state.cpu().numpy()
    for i in range(n - 5):
        b = np.array([boxes["x"][i], boxes["y"][i], boxes["w"][i], boxes["h"][i]])
        h, w = shapes[recs[i, 0]]
        want = image_ops.clamp_bbox(image_ops.rescale_bbox(b, recs[i, 5:9], 256), (h, w, 3))
        assert np.array_equal(got[i, 1:5], want), (i, b.tolist(), recs[i, 5:9].tolist(), (h, w), got[i, 1:5], want)
    assert (got[-5:, 1:5] == [7, 8, 9, 10]).all()
    assert np.array_equal(np.delete(got, np.s_[1:5], axis=1), np.delete(recs, np.s_[1:5], axis=1))


# ---------------------------------------------------------------------------------------------------- tracker
def test_one_stream_matches_golden_and_independent_trackers(net, clip):
    trk = fb.FEARMultiTracker(net, cuda_id=0, max_targets=16, **CFG)
    ids = trk.initialize(clip[0], CLIP_TARGETS)
    assert ids.tolist() == list(range(len(CLIP_TARGETS)))
    boxes, scores = run_multi(trk, [[f] for f in clip[1:]])
    assert np.array_equal(boxes[:, 0], golden("video_teacher.npz")["trajectory"])
    assert np.array_equal(boxes[:, 0], boxes[:, 5]) and np.array_equal(scores[:, 0], scores[:, 5])
    assert_matches_independent(net, "clip", clip, CLIP_TARGETS, boxes, scores)


def test_several_streams_of_different_shapes(net, clip):
    T = 150
    streams = {"clip": clip[:T + 1], "mirror": np.ascontiguousarray(clip[:T + 1, :, ::-1]),
               "window": np.ascontiguousarray(clip[:T + 1, 30:200, 50:350])}
    rects = {"clip": [GOLDEN_BOX, [420, 10, 50, 60]], "mirror": [[272, 53, 45, 174], [0, 180, 40, 70]],
             "window": [[113, 23, 45, 120], [250, 140, 60, 40]]}
    names = list(streams)
    trk = fb.FEARMultiTracker(net, cuda_id=0, max_targets=8, **CFG)
    first = [streams[s][0] for s in names]
    trk.add(first, [r for s in names for r in rects[s]], [names.index(s) for s in names for _ in rects[s]])
    boxes, scores = run_multi(trk, [[streams[s][t] for s in names] for t in range(1, T + 1)])
    for j, s in enumerate(names):
        assert_matches_independent(net, s, streams[s], rects[s], boxes[:, 2 * j:2 * j + 2], scores[:, 2 * j:2 * j + 2])


@pytest.mark.parametrize("case", ["reversed", "single", "eager"])
def test_invariance(net, clip, case):
    T = 100
    rects = {"reversed": CLIP_TARGETS[::-1], "single": [GOLDEN_BOX], "eager": CLIP_TARGETS}[case]
    cfg = dict(CFG, cuda_graph=False) if case == "eager" else CFG
    trk = fb.FEARMultiTracker(net, cuda_id=0, max_targets=16, **cfg)
    trk.initialize(clip[0], rects)
    boxes, scores = run_multi(trk, [[f] for f in clip[1:T + 1]])
    assert (trk._graph is None) == (case == "eager")
    assert_matches_independent(net, "clip", clip, rects, boxes, scores)


def test_graph_recaptured_after_workspace_growth(net, clip):
    n2 = fb.FEARNet(**fb.FEAR_XS_MODEL_KWARGS)
    n2.load_state_dict(load_full_state(), strict=True)
    n2 = n2.cuda().eval()
    trk = fb.FEARMultiTracker(n2, cuda_id=0, max_targets=8, **CFG)
    trk.initialize(clip[0], CLIP_TARGETS)
    b1, s1 = run_multi(trk, [[f] for f in clip[1:6]])
    assert trk._graph is not None
    gen = n2.generation()
    zt, xt, _, _ = fo.synthetic_crops(12)
    n2.track(xt.cuda(), n2.get_features(zt.cuda()))  # batch 12 > reserved 8: the workspace is re-allocated
    assert n2.generation() != gen
    b2, s2 = run_multi(trk, [[f] for f in clip[6:40]])
    assert trk._graph is not None and trk._graph_gen == n2.generation()
    assert_matches_independent(net, "clip", clip, CLIP_TARGETS, np.concatenate([b1, b2]), np.concatenate([s1, s2]))


def test_add_and_remove(net, clip):
    start_rects = CLIP_TARGETS[:4]
    late_rects = [[300, 80, 60, 90], [100, 150, 30, 30]]
    trk = fb.FEARMultiTracker(net, cuda_id=0, max_targets=8, **CFG)
    trk.initialize(clip[0], start_rects)
    hist = {}  # id -> list of (box, score)
    for f in range(1, 401):
        if f == 300:
            trk.remove([1])
        out = trk.update(clip[f])
        for i, tid in enumerate(out["ids"]):
            hist.setdefault(int(tid), []).append((out["bbox"][i], out["score"][i]))
        if f == 100:
            assert trk.add(clip[100], late_rects).tolist() == [4, 5]
    assert sorted(hist) == [0, 1, 2, 3, 4, 5] and len(trk) == 5
    for tid, rect, start in [(0, start_rects[0], 0), (1, start_rects[1], 0), (2, start_rects[2], 0),
                             (3, start_rects[3], 0), (4, late_rects[0], 100), (5, late_rects[1], 100)]:
        boxes = np.array([b for b, _ in hist[tid]])[:, None]
        scores = np.array([s for _, s in hist[tid]])[:, None]
        assert boxes.shape[0] == (299 if tid == 1 else 400 - start)
        assert_matches_independent(net, "clip", clip, [rect], boxes, scores, start=start)


def test_launch_count_does_not_grow_with_targets(net, clip):
    deltas = {}
    for n in (1, 16):
        trk = fb.FEARMultiTracker(net, cuda_id=0, max_targets=16, cuda_graph=False, **CFG)
        trk.initialize(clip[0], [GOLDEN_BOX] * n)
        trk.update(clip[1])
        torch.cuda.synchronize()
        c0 = net.launch_count()
        trk.update(clip[2])
        trk.update(clip[3])
        deltas[n] = (net.launch_count() - c0) / 2
    assert deltas[1] == deltas[16] > 0, deltas


def test_c_abi_rejects_bad_arguments():
    lib = _lib.load()
    t = torch.zeros(4096, dtype=torch.uint8, device="cuda")
    p = t.data_ptr()
    good = dict(frames=p, table=p, F=1, targets=p, N=1, offset=2.0, size=256, crops=p)

    def crop(**kw):
        a = dict(good, **kw)
        return lib.fear_crop_targets_u8(a["frames"], a["table"], a["F"], a["targets"], a["N"], a["offset"], a["size"],
                                        a["crops"], None)

    bad = [dict(frames=None), dict(table=None), dict(targets=None), dict(crops=None), dict(N=0), dict(N=65536),
           dict(F=0), dict(size=0), dict(size=257), dict(offset=-0.5), dict(offset=float("nan")),
           dict(offset=float("inf"))]
    for kw in bad:
        assert crop(**kw) == -1, kw
        assert _lib.last_error(), kw
    for args in [(None, p, 1, p, 1, 256), (p, None, 1, p, 1, 256), (p, p, 1, None, 1, 256), (p, p, 1, p, 0, 256),
                 (p, p, 0, p, 1, 256), (p, p, 1, p, 1, 0)]:
        assert lib.fear_advance_targets(*args, None) == -1, args
        assert _lib.last_error(), args
