"""GPU: FEARTracker on frames already in GPU memory -- CUDA tensors (contiguous and strided views) and YUV frames --
against a second FEARTracker with the same config fed the same pixels as numpy arrays (``image_ops.yuv_to_rgb`` of a
YUV frame's planes), on the demo clip.  Every update must give the same box and the same whole ``tracking_state``
(bbox, mapping, prev_size, paths and a bitwise-equal mean_color), with and without ``smooth``."""
import json
import os
import subprocess
import sys

import cv2
import numpy as np
import pytest
import torch

import feartracker_b200 as fb
from feartracker_b200 import image_ops
from oracle import fear_oracle as fo
from tests.helpers import GOLDEN, golden, load_full_state

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
CFG = fb.FEAR_XS_TRACKER_KWARGS
SMOOTH = {"plain": {}, "smooth": {"smooth": True}}
OUT = None  # dump directory of this run (set by _dump_dir)


@pytest.fixture(scope="module", autouse=True)
def _dump_dir(tmp_path_factory):
    global OUT
    OUT = str(tmp_path_factory.mktemp("gpu_tracker_device_frames"))


def _dump(name, obj):
    with open(os.path.join(OUT, name), "w") as f:
        json.dump(obj, f, indent=1)


def _make_net(reserve=1):
    n = fb.FEARNet(**fb.FEAR_XS_MODEL_KWARGS)
    n.load_state_dict(load_full_state(), strict=True)
    n = n.cuda().eval()
    n.reserve(reserve)
    return n


@pytest.fixture(scope="module")
def net():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return _make_net(1)


@pytest.fixture(scope="module")
def clip():
    return fo.read_video_rgb(os.path.join(GOLDEN, "test.mp4"))


@pytest.fixture(scope="module")
def init_box():
    return golden("video_teacher.npz")["init_bbox"]


# ------------------------------------------------------------------------------------------------------------- frames
def _rgba(f, alpha):
    t = torch.empty(f.shape[:2] + (4,), dtype=torch.uint8)
    t[..., :3] = torch.from_numpy(f)
    t[..., 3] = alpha
    return t.cuda()[..., :3]


def _chw(f):
    return torch.from_numpy(np.ascontiguousarray(f.transpose(2, 0, 1))).cuda().permute(1, 2, 0)


def _roi(f):
    """A region of interest inside a larger canvas whose border holds other content (the frame, mirrored)."""
    h, w = f.shape[:2]
    canvas = np.pad(f[::-1, ::-1], ((17, 23), (29, 35), (0, 0)), mode="reflect")
    canvas[17:17 + h, 29:29 + w] = f
    return torch.from_numpy(canvas).cuda()[17:17 + h, 29:29 + w]


VIEWS = {"rgba": lambda f: _rgba(f, 77), "chw": _chw, "roi": _roi}


def _codes(f, bits, sub):
    """Y, Cb, Cr codes (numpy, LSB-aligned) of an RGB frame at ``bits`` and chroma subsampling ``sub`` = (sx, sy): a
    limited-range BT.601 forward transform (any codes would do: the reference converts these very codes back)."""
    x = f.astype(np.float64)
    m = float(1 << (bits - 8))
    y = (16 + (0.257 * x[..., 0] + 0.504 * x[..., 1] + 0.098 * x[..., 2])) * m
    cb = (128 + (-0.148 * x[..., 0] - 0.291 * x[..., 1] + 0.439 * x[..., 2])) * m
    cr = (128 + (0.439 * x[..., 0] - 0.368 * x[..., 1] - 0.071 * x[..., 2])) * m
    sx, sy = sub
    dt = np.uint8 if bits == 8 else np.uint16
    return tuple(np.clip(np.rint(c), 0, (1 << bits) - 1).astype(dt) for c in (y, cb[::1 << sy, ::1 << sx],
                                                                                cr[::1 << sy, ::1 << sx]))


def _nv12(f, bits=8, matrix="bt601", pitch=0):
    y, u, v = _codes(f, bits, (1, 1))
    h, w = y.shape
    sh = 16 - bits if bits > 8 else 0
    surf = np.full((h + h // 2, w + pitch), 0xA5, dtype=y.dtype)
    surf[:h, :w] = y << sh
    surf[h:, :w:2], surf[h:, 1:w:2] = u << sh, v << sh
    return fb.YUV420Frame.nv12(torch.from_numpy(surf).cuda()[:, :w], matrix=matrix, bits=bits)


def _i420(f, bits=8, matrix="bt601"):
    y, u, v = _codes(f, bits, (1, 1))
    h, w = y.shape
    flat = np.concatenate([y.reshape(-1), u.reshape(-1), v.reshape(-1)]).reshape(h + h // 2, w)
    return fb.YUV420Frame.i420(torch.from_numpy(flat).cuda(), matrix=matrix, bits=bits)


def _yuyv(f):
    y, u, v = _codes(f, 8, (1, 0))
    h, w = y.shape
    surf = np.empty((h, 2 * w), np.uint8)
    surf[:, 0::2], surf[:, 1::4], surf[:, 3::4] = y, u, v
    return fb.YUV422Frame.yuyv(torch.from_numpy(surf).cuda())


def _p210(f):
    y, u, v = _codes(f, 10, (1, 0))
    h, w = y.shape
    surf = np.empty((2 * h, w), np.uint16)
    surf[:h] = y << 6
    surf[h:, 0::2], surf[h:, 1::2] = u << 6, v << 6
    return fb.YUV422Frame.nv16(torch.from_numpy(surf).cuda(), matrix="bt709", bits=10)


def _i444(f, pitch=48):
    y, u, v = _codes(f, 8, (0, 0))
    h, w = y.shape
    surf = np.full((3 * h, w + pitch), 0x5A, np.uint8)
    surf[:h, :w], surf[h:2 * h, :w], surf[2 * h:, :w] = y, u, v
    return fb.YUV444Frame.i444(torch.from_numpy(surf).cuda()[:, :w])


YUV = {
    "nv12_pitched": lambda f: _nv12(f, pitch=32),
    "i420": _i420,
    "p010_bt709": lambda f: _nv12(f, bits=10, matrix="bt709"),
    "yuv420p10le_bt2020": lambda f: _i420(f, bits=10, matrix="bt2020"),
    "yuyv": _yuyv,
    "p210": _p210,
    "i444_pitched": _i444,
}


def as_rgb(frame):
    """The numpy frame a device frame stands for."""
    if isinstance(frame, torch.Tensor):
        return frame.cpu().numpy()
    y, u, v = (p.cpu().numpy() for p in (frame.y, frame.u, frame.v))
    return image_ops.yuv_to_rgb(y, u, v, frame.matrix, frame.full_range, frame.bits, frame.shift, frame.CHROMA_SHIFT)


# --------------------------------------------------------------------------------------------------------- comparison
def assert_same_state(a, b, where):
    sa, sb = a.tracking_state, b.tracking_state
    assert np.array_equal(sa.bbox, sb.bbox), (where, sa.bbox, sb.bbox)
    assert np.array_equal(sa.mapping, sb.mapping), (where, sa.mapping, sb.mapping)
    assert np.array_equal(np.asarray(sa.prev_size), np.asarray(sb.prev_size)), (where, sa.prev_size, sb.prev_size)
    assert [list(p) for p in sa.paths] == [list(p) for p in sb.paths], where
    assert sa.mean_color.dtype == sb.mean_color.dtype and sa.mean_color.tobytes() == sb.mean_color.tobytes(), \
        (where, sa.mean_color, sb.mean_color)


def run_pair(net, frames, make, init_box, extra=None):
    """``make(t, frame)`` -> the frame fed to the device tracker at index t (a numpy frame feeds both unchanged);
    the reference is fed ``as_rgb`` of it.  Compares every box and the whole tracking_state after every call."""
    cfg = dict(CFG, **(extra or {}))
    dev_trk = fb.FEARTracker(net, cuda_id=0, **cfg)
    ref_trk = fb.FEARTracker(net, cuda_id=0, **cfg)
    f0 = make(0, frames[0])
    dev_trk.initialize(f0, init_box)
    ref_trk.initialize(f0 if isinstance(f0, np.ndarray) else as_rgb(f0), init_box)
    assert_same_state(dev_trk, ref_trk, "initialize")
    boxes = []
    for t in range(1, len(frames)):
        f = make(t, frames[t])
        got = dev_trk.update(f)["bbox"]
        want = ref_trk.update(f if isinstance(f, np.ndarray) else as_rgb(f))["bbox"]
        assert list(got) == list(want), (t, got, want)
        assert_same_state(dev_trk, ref_trk, t)
        boxes.append(list(map(int, got)))
    return dev_trk, np.array(boxes)


# ------------------------------------------------------------------------------------------------------------ 1. clip
@pytest.mark.parametrize("mode", list(SMOOTH))
def test_whole_clip_contiguous_tensors(net, clip, init_box, mode):
    dev = torch.from_numpy(clip).cuda()
    trk, boxes = run_pair(net, clip, lambda t, f: dev[t], init_box, SMOOTH[mode])
    st = trk._device_state
    assert st["graph"] is not None and st["key"][0] == "views" and getattr(trk, "_gpu_crop_state", None) is None
    if mode == "plain":  # the host path's trajectory is the reference's own
        assert np.array_equal(boxes, golden("video_teacher.npz")["trajectory"])
    _dump(f"clip_{mode}.json", {"updates": len(boxes)})


# ------------------------------------------------------------------------------------------------ 2. strided views
@pytest.mark.parametrize("mode", list(SMOOTH))
@pytest.mark.parametrize("view", ["rgba", "chw", "roi"])
def test_strided_views(net, clip, init_box, view, mode):
    run_pair(net, clip[:121], lambda t, f: VIEWS[view](f), init_box, SMOOTH[mode])


# ---------------------------------------------------------------------------------------------------------- 3. YUV
@pytest.mark.parametrize("mode", list(SMOOTH))
@pytest.mark.parametrize("fmt", list(YUV))
def test_yuv_frames(net, clip, init_box, fmt, mode):
    frames = clip if fmt == "nv12_pitched" else clip[:121]
    trk, _ = run_pair(net, frames, lambda t, f: YUV[fmt](f), init_box, SMOOTH[mode])
    assert trk._device_state["key"][0] == "ycbcr" and trk._device_state["graph"] is not None


# ------------------------------------------------------------------------------------------------- 4. mixed kinds
@pytest.mark.parametrize("extra", [{}, dict(smooth=True), dict(gpu_crop=True), dict(gpu_crop=True, smooth=True)])
def test_mixed_kinds(net, clip, init_box, extra):
    """Init on NV12, then updates cycling numpy -> CUDA view -> YUYV -> NV12."""
    kinds = [lambda f: f, VIEWS["rgba"], _yuyv, _nv12]
    trk, _ = run_pair(net, clip[:81], lambda t, f: _nv12(f) if t == 0 else kinds[(t - 1) % 4](f), init_box, extra)
    if extra.get("gpu_crop"):
        assert trk._gpu_crop_state["graph"] is not None  # numpy updates kept their own graph


def _resized(clip, t, switch):
    return clip[t] if t < switch else np.ascontiguousarray(cv2.resize(clip[t], (640, 360)))


@pytest.mark.parametrize("mode", list(SMOOTH))
def test_resolution_change(net, clip, init_box, mode):
    """Frames grow from 480 x 256 to 640 x 360 partway (a CUDA view, then NV12 and numpy at the new size)."""
    frames = [_resized(clip, t, 40) for t in range(81)]
    kinds = [VIEWS["chw"], _nv12, lambda f: f]
    run_pair(net, frames, lambda t, f: kinds[t % 3](f), init_box, SMOOTH[mode])


# ---------------------------------------------------------------------------------------------------- 5. mean colour
def _half_means(h, w):
    """A frame whose channel means are exactly 100.5, 101.5 and 7.5 (half to even: 100, 102, 8)."""
    f = np.empty((h, w, 3), np.uint8)
    f[:, :w // 2] = (100, 101, 7)
    f[:, w // 2:] = (101, 102, 8)
    return f


@pytest.mark.parametrize("mode", list(SMOOTH))
def test_mean_colour_half_integers_and_4k(net, clip, mode):
    rng = np.random.default_rng(5)
    big = rng.integers(0, 256, (2160, 3840, 3), dtype=np.uint8)
    big[500:1500, 1000:2500] = cv2.resize(clip[0], (1500, 1000))
    cases = {"half": (_half_means(256, 480), [200, 100, 60, 50]), "4k": (big, [1000, 500, 600, 700])}
    for name, (frame, box) in cases.items():
        cfg = dict(CFG, **SMOOTH[mode])
        dev_trk, ref_trk = fb.FEARTracker(net, cuda_id=0, **cfg), fb.FEARTracker(net, cuda_id=0, **cfg)
        for trk, f in ((dev_trk, torch.from_numpy(frame).cuda()), (ref_trk, frame)):
            trk.initialize(f, box)
        assert_same_state(dev_trk, ref_trk, name)
        assert dev_trk.tracking_state.mean_color.tobytes() == np.mean(frame, axis=(0, 1)).tobytes()
        assert torch.equal(dev_trk._template_features, ref_trk._template_features), name
        assert torch.equal(dev_trk.get_template_features(torch.from_numpy(frame).cuda(), box),
                           ref_trk.get_template_features(frame, box)), name
        for t in range(3):
            assert list(dev_trk.update(torch.from_numpy(frame).cuda())["bbox"]) == list(ref_trk.update(frame)["bbox"])
            assert_same_state(dev_trk, ref_trk, (name, t))
    assert image_ops.padding_color(np.mean(cases["half"][0], axis=(0, 1))).tolist() == [100, 102, 8]


# ----------------------------------------------------------------------------------------------- 6. graph, launches
def test_graph_replay_launches_and_no_recapture(clip, init_box, monkeypatch):
    """The first device update runs eagerly, then each update is one replay with no handle launch outside it; fresh
    frames (new addresses) and a resolution change replay the same graph."""
    n = _make_net(1)
    replays = []
    real_replay = torch.cuda.CUDAGraph.replay
    monkeypatch.setattr(torch.cuda.CUDAGraph, "replay", lambda self: (replays.append(1), real_replay(self))[1])
    for mode, extra in SMOOTH.items():
        replays.clear()
        trk = fb.FEARTracker(n, cuda_id=0, **dict(CFG, **extra))
        trk.initialize(torch.from_numpy(clip[0]).cuda(), init_box)
        trk.update(torch.from_numpy(clip[1]).cuda())
        assert trk._device_state["graph"] is None and not replays
        graph = None
        for k, t in enumerate(range(2, 40), 1):
            f = _resized(clip, t, 20)
            frame = torch.from_numpy(f).cuda() if t % 2 else VIEWS["roi"](f)
            c0 = n.launch_count() if k > 1 else None
            trk.update(frame)
            assert len(replays) == k, mode
            if graph is None:
                graph = trk._device_state["graph"]
            assert trk._device_state["graph"] is graph, (mode, t)  # never re-captured
            if c0 is not None:
                assert n.launch_count() == c0, mode
        # YUV frames go through the other entry point: re-captured, and back again
        trk.update(_nv12(clip[40]))
        trk.update(_nv12(clip[41]))
        assert trk._device_state["graph"] is not graph and trk._device_state["key"][0] == "ycbcr"
        ycbcr_graph = trk._device_state["graph"]
        trk.update(torch.from_numpy(clip[42]).cuda())
        trk.update(torch.from_numpy(clip[43]).cuda())
        assert trk._device_state["graph"] not in (graph, ycbcr_graph) and trk._device_state["key"][0] == "views"


@pytest.mark.parametrize("mode", list(SMOOTH))
def test_eager_launches_equal_gpu_crop(clip, init_box, mode):
    """An eager device update launches on the handle what a numpy gpu_crop update launches (the crop kernels and
    fear_decode_smooth are handle-free)."""
    n = _make_net(1)
    per_update = {}
    for name, frames in (("gpu_crop", clip[:6]), ("device", torch.from_numpy(clip[:6]).cuda())):
        trk = fb.FEARTracker(n, cuda_id=0, gpu_crop=True, cuda_graph=False, **dict(CFG, **SMOOTH[mode]))
        trk.initialize(frames[0], init_box)
        trk.update(frames[1])
        c0 = n.launch_count()
        for f in frames[2:5]:
            trk.update(f)
        per_update[name] = (n.launch_count() - c0) / 3
    _dump(f"launches_{mode}.json", per_update)
    assert per_update["device"] == per_update["gpu_crop"] > 0, per_update


@pytest.mark.parametrize("mode", list(SMOOTH))
def test_workspace_growth_recaptures(clip, init_box, mode):
    frames = torch.from_numpy(clip[:16]).cuda()
    cfg = dict(CFG, **SMOOTH[mode])
    want = [list(map(int, b)) for b in _traj(fb.FEARTracker(_make_net(1), cuda_id=0, **cfg), frames, init_box)]
    n = _make_net(1)
    trk = fb.FEARTracker(n, cuda_id=0, **cfg)
    trk.initialize(frames[0], init_box)
    out = [list(map(int, trk.update(f)["bbox"])) for f in frames[1:6]]
    graph, gen = trk._device_state["graph"], n.generation()
    assert graph is not None
    zt, xt, _, _ = fo.synthetic_crops(12)
    n.track(xt.cuda(), n.get_features(zt.cuda()))  # batch 12 > reserved: workspace freed and re-allocated
    assert n.generation() != gen
    out += [list(map(int, trk.update(f)["bbox"])) for f in frames[6:]]
    st = trk._device_state
    assert st["graph"] is not None and st["graph"] is not graph and st["key"][3] == n.generation()
    assert out == want


def _traj(trk, frames, init_box):
    trk.initialize(frames[0], init_box)
    return [trk.update(f)["bbox"] for f in frames[1:]]


@pytest.mark.parametrize("mode", list(SMOOTH))
def test_eager_equals_graph(net, clip, init_box, mode):
    frames = clip[:60]  # the last 10 updates are one kind: the graphed tracker ends on a graph
    eager = fb.FEARTracker(net, cuda_id=0, cuda_graph=False, **dict(CFG, **SMOOTH[mode]))
    graphed = fb.FEARTracker(net, cuda_id=0, **dict(CFG, **SMOOTH[mode]))
    for trk in (eager, graphed):
        trk.initialize(_nv12(frames[0]), init_box)
    for t in range(1, len(frames)):
        f = _nv12(frames[t]) if (t // 10) % 2 else VIEWS["chw"](frames[t])  # each kind in runs of 10 updates
        assert list(eager.update(f)["bbox"]) == list(graphed.update(f)["bbox"]), t
        assert_same_state(eager, graphed, t)
    assert eager._device_state["graph"] is None and graphed._device_state["graph"] is not None


def test_refusals_on_the_device(net, clip, init_box):
    """Planes or tensors on another device than the tracker's, and host_normalize, are refused before any device
    call or state change."""
    frame = torch.from_numpy(clip[0]).cuda()
    trk = fb.FEARTracker(net, cuda_id=0, **CFG)
    trk.cuda_id = 1  # a tracker on cuda:1 (set after construction: cuda:1 need not exist, the check compares devices)
    for f in (frame, _nv12(clip[0])):
        with pytest.raises(ValueError, match="the tracker on cuda:1"):
            trk.initialize(f, init_box)
    assert trk.tracking_state.bbox is None and getattr(trk, "_device_state", None) is None
    trk = fb.FEARTracker(net, cuda_id=0, host_normalize=True, **CFG)
    with pytest.raises(NotImplementedError, match="host_normalize"):
        trk.initialize(frame, init_box)
    trk.initialize(clip[0], init_box)  # numpy frames still work with host_normalize
    with pytest.raises(NotImplementedError, match="host_normalize"):
        trk.update(_yuyv(clip[1]))
    assert getattr(trk, "_device_state", None) is None


# ---------------------------------------------------------------------------------------------- 7. poisoned memory
def test_poisoned_memory():
    proc = subprocess.run([sys.executable, os.path.join(HERE, "poison_tracker_device_check.py")],
                          capture_output=True, text=True, timeout=1200)
    with open(os.path.join(OUT, "poison_tracker_device_check.log"), "w") as f:
        f.write(proc.stdout + "\n--- stderr ---\n" + proc.stderr)
    lines = [l for l in proc.stdout.splitlines() if l.startswith("POISON_CHECK ")]
    assert proc.returncode == 0 and lines, proc.stderr[-3000:]
    res = json.loads(lines[-1][len("POISON_CHECK "):])
    assert res["checked_calls"] > 0
    assert res["n_failures"] == 0, res["failures"]
