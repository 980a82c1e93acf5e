"""GPU: fear_decode_smooth (the ``smooth: true`` post-processing of FEARTracker on the device) against the host's
FEARTracker._smooth_postprocess, the reference's recorded cases and trajectory, and FEARTracker(gpu_crop=True,
smooth=True) against FEARTracker(smooth=True)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import feartracker_b200 as fb
from feartracker_b200 import _lib
from oracle import fear_oracle as fo
from tests.helpers import GOLDEN, golden, load_full_state

pytestmark = pytest.mark.gpu
R, C = fo.TARGET_REGRESSION_LABEL_KEY, fo.TARGET_CLASSIFICATION_KEY
HERE = os.path.dirname(os.path.abspath(__file__))
CFG = dict(fb.FEAR_XS_TRACKER_KWARGS, smooth=True)
OUT = None  # dump directory of this run (set by _dump_dir)


@pytest.fixture(scope="module", autouse=True)
def _dump_dir(tmp_path_factory):
    global OUT
    OUT = str(tmp_path_factory.mktemp("gpu_smooth"))


def _dump(name, obj):
    with open(os.path.join(OUT, name), "w") as f:
        json.dump(obj, f, indent=1)


def _make_net(reserve=8):
    n = fb.FEARNet(**fb.FEAR_XS_MODEL_KWARGS)
    n.load_state_dict(load_full_state(), strict=True)
    n = n.cuda().eval()
    n.reserve(reserve)
    return n


@pytest.fixture(scope="module")
def net():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return _make_net(8)


@pytest.fixture(scope="module")
def clip():
    return fo.read_video_rgb(os.path.join(GOLDEN, "test.mp4"))


def _host(**over):
    """A FEARTracker whose _smooth_postprocess is the reference for one config (the net is never called)."""
    cfg = dict(CFG, **over)
    return fb.FEARTracker(None, cuda_id=0, **cfg), cfg


def _params(trk, cfg):
    window = np.asarray(trk.window, dtype=np.float64).reshape(256)
    return torch.from_numpy(np.concatenate([[cfg["penalty_k"], cfg["window_influence"], cfg["lr"]], window])).cuda()


def _decode_smooth(reg, cls, prev, params):
    """fear_decode_smooth on CUDA maps (B,4,16,16) / (B,1,16,16), prev (B,2) float64 -> BOX_DTYPE records."""
    reg, cls = reg.float().contiguous(), cls.float().contiguous()
    prev = torch.as_tensor(np.asarray(prev, dtype=np.float64)).cuda().contiguous()
    b = reg.shape[0]
    boxes = torch.full((b, 48), 0xA5, dtype=torch.uint8, device="cuda")
    _lib.check(_lib.load().fear_decode_smooth(reg.data_ptr(), cls.data_ptr(), b, prev.data_ptr(), params.data_ptr(),
                                              boxes.data_ptr(), torch.cuda.current_stream().cuda_stream),
               "fear_decode_smooth")
    return boxes.cpu().numpy().view(_lib.BOX_DTYPE).reshape(-1)


def _pscore(trk, reg, score):
    """The penalised score map of _smooth_postprocess (its argmax is the cell the host picks)."""
    cfg, (pw, ph) = trk.tracking_config, trk.tracking_state.prev_size
    gx, gy = trk.box_coder.grid_x.cpu().numpy()[0], trk.box_coder.grid_y.cpu().numpy()[0]
    x1, y1, x2, y2 = gx - reg[0], gy - reg[1], gx + reg[2], gy + reg[3]

    def limit(r):
        return np.maximum(r, 1.0 / r)

    def sq(w, h):
        pad = (w + h) * 0.5
        return np.sqrt((w + pad) * (h + pad))

    with np.errstate(all="ignore"):
        s_c = limit(sq(x2 - x1, y2 - y1) / sq(pw, ph))
        r_c = limit((pw / ph) / ((x2 - x1) / (y2 - y1)))
        penalty = np.exp(-(r_c * s_c - 1) * cfg["penalty_k"])
        return (penalty * score) * (1 - cfg["window_influence"]) + trk.window * cfg["window_influence"]


def _host_case(trk, reg_cuda, cls_cuda, prev):
    """(box, score, flat, relative gap of the top two pscores) of the host path on one frame's CUDA maps."""
    trk.tracking_state.prev_size = np.asarray(prev, dtype=np.float64)
    with np.errstate(all="ignore"):
        box, score = trk._postprocess({R: reg_cuda[None], C: cls_cuda[None]})
    reg = reg_cuda.float().cpu().numpy().astype(np.float64)
    p = _pscore(trk, reg, cls_cuda.float().sigmoid().cpu().numpy()[0]).reshape(-1)
    flat = int(np.argmax(p))
    top = np.sort(p[~np.isnan(p)])[-2:] if not np.isnan(p).any() else np.array([np.nan, np.nan])
    gap = float(abs(top[1] - top[0]) / max(abs(top[1]), 1e-300)) if len(top) == 2 and np.isfinite(top).all() else 1.0
    return np.asarray(box, dtype=np.float64), np.float32(score), flat, gap


def _rec_box(rec):
    return np.array([rec["x"], rec["y"], rec["w"], rec["h"]], dtype=np.float64)


def _same_box(got, want, rtol=1e-12):
    return np.allclose(got, want, rtol=rtol, atol=1e-12, equal_nan=True)


# --------------------------------------------------------------------------------------------------- golden cases
def test_golden_cases():
    """The reference's recorded per-frame cases at B = 7 and B = 1: against the golden (whose sigmoid ran on the CPU)
    and, strictly, against _postprocess on the same CUDA maps (torch's device sigmoid)."""
    g = golden("smooth_tracker.npz")
    trk, cfg = _host()
    params = _params(trk, cfg)
    reg, cls = torch.from_numpy(g["reg"]).cuda(), torch.from_numpy(g["cls"]).cuda()
    batched = _decode_smooth(reg, cls, g["prev_size"], params)
    singles = np.concatenate([_decode_smooth(reg[i:i + 1], cls[i:i + 1], g["prev_size"][i:i + 1], params)
                              for i in range(len(reg))])
    assert batched.tobytes() == singles.tobytes()
    for i, rec in enumerate(batched):
        assert [int(rec["row"]), int(rec["col"])] == g["coords"][i].tolist() and rec["flat"] == rec["row"] * 16 + rec["col"]
        np.testing.assert_allclose([rec["x"], rec["y"]], g["box"][i][:2], rtol=1e-12)
        assert abs(int(np.float32(rec["score"]).view(np.int32)) - int(g["score"][i].view(np.int32))) <= 1, i
        np.testing.assert_allclose([rec["w"], rec["h"]], g["box"][i][2:], rtol=1e-6)
        box, score, flat, _ = _host_case(trk, reg[i], cls[i], g["prev_size"][i])
        assert int(rec["flat"]) == flat
        assert np.float32(rec["score"]).view(np.uint32) == score.view(np.uint32)
        np.testing.assert_allclose(_rec_box(rec), box, rtol=1e-12, atol=0)


# ------------------------------------------------------------------------------------------------ real maps, batched
@pytest.fixture(scope="module")
def real_maps(net, clip):
    """Maps of net.track on 256 search crops of the demo clip (targets around the reference's smooth trajectory,
    with jittered boxes) and a prev_size per crop that varies around each target's size."""
    from feartracker_b200 import image_ops

    g = golden("smooth_tracker.npz")
    rng = np.random.default_rng(11)
    traj = g["trajectory"]
    frame0 = clip[0]
    zf = net.get_features(torch.from_numpy(image_ops.extended_crop(frame0, g["init_bbox"], 128, 0.2)[0][None]).cuda())
    crops, prev = [], []
    for k in range(256):
        i = int(rng.integers(0, len(traj)))
        box = traj[i].astype(np.float64)
        box[:2] += rng.normal(0, 6, 2)
        box[2:] *= np.exp(rng.normal(0, 0.2, 2))
        box = image_ops.clamp_bbox(np.rint(box).astype(np.int64), clip[i + 1].shape)
        crop, search_bbox, _ = image_ops.extended_crop(clip[i + 1], box, 256, 2, np.mean(clip[0], axis=(0, 1)))
        crops.append(crop)
        prev.append(search_bbox[2:] * np.exp(rng.normal(0, 0.3, 2)) if k % 4 else search_bbox[2:])
    net.reserve(256)
    maps = net.track(torch.from_numpy(np.stack(crops)).cuda(), zf)
    torch.cuda.synchronize()
    return maps[R], maps[C], np.array(prev, dtype=np.float64)


CONFIGS = [dict(), dict(windowing="uniform"), dict(window_influence=0.0), dict(window_influence=1.0), dict(lr=0.0),
           dict(penalty_k=0.5, windowing="uniform", window_influence=0.2)]


@pytest.mark.parametrize("B", [1, 3, 64, 256])
@pytest.mark.parametrize("over", CONFIGS, ids=lambda o: ",".join(f"{k}={v}" for k, v in o.items()) or "default")
def test_real_maps_batched(real_maps, B, over):
    reg, cls, prev = real_maps
    trk, cfg = _host(**over)
    recs = _decode_smooth(reg[:B], cls[:B], prev[:B], _params(trk, cfg))
    near_ties = 0
    for i, rec in enumerate(recs):
        box, score, flat, gap = _host_case(trk, reg[i], cls[i], prev[i])
        if int(rec["flat"]) != flat:
            assert gap <= 1e-12, (i, int(rec["flat"]), flat, gap)
            near_ties += 1
            continue
        assert (rec["row"], rec["col"]) == (flat // 16, flat % 16)
        assert np.float32(rec["score"]).view(np.uint32) == score.view(np.uint32), i
        assert _same_box(_rec_box(rec), box), (i, _rec_box(rec), box)
    tag = "_".join(f"{k}={v}" for k, v in over.items()) or "default"
    _dump(f"real_maps_B{B}_{tag}.json", {"items": B, "near_ties": near_ties})


# -------------------------------------------------------------------------------------------------- adversarial maps
def test_adversarial_maps():
    """NaN and +-inf logits and distances, constant maps (first index wins), one NaN among equal values, zero and
    negative sizes: the argmax and the record follow the host's numpy rules."""
    trk, cfg = _host()
    params = _params(trk, cfg)
    gen = torch.Generator().manual_seed(7)
    base_reg = 20 + 40 * torch.rand(4, 16, 16, generator=gen)
    base_cls = torch.randn(1, 16, 16, generator=gen)
    cases = []

    def add(reg=None, cls=None, prev=(51.2, 51.2)):
        cases.append((base_reg.clone() if reg is None else reg, base_cls.clone() if cls is None else cls, prev))

    add()
    add(cls=torch.full((1, 16, 16), 0.7))                                   # constant: window decides
    add(reg=torch.full((4, 16, 16), 25.0), cls=torch.full((1, 16, 16), 0.7))  # all equal but the window
    c = torch.full((1, 16, 16), 0.7)
    c[0, 9, 4] = float("nan")
    add(reg=torch.full((4, 16, 16), 25.0), cls=c)                            # one NaN score
    c = base_cls.clone()
    c[0, 3, 3] = c[0, 12, 12] = float("nan")
    add(cls=c)                                                              # first NaN wins
    c = base_cls.clone()
    c[0, 5, 6] = float("inf")
    c[0, 7, 2] = float("-inf")
    add(cls=c)
    r = base_reg.clone()
    r[0, 8, 8] = float("nan")
    r[2, 4, 4] = float("inf")
    r[1, 6, 9] = float("-inf")
    add(reg=r)
    r = base_reg.clone()
    r[:, 8, 8] = 0.0                                                        # zero-size box: inf / NaN ratios
    r[0, 2, 3], r[2, 2, 3] = 10.0, -10.0                                    # negative width
    add(reg=r)
    add(prev=(0.0, 51.2))
    add(prev=(float("nan"), 40.0))
    add(reg=torch.full((4, 16, 16), float("nan")))
    add(cls=torch.full((1, 16, 16), float("nan")))
    # equal pscore everywhere (uniform window, no window weight, constant maps): flat index 0
    for over in (dict(), dict(windowing="uniform", window_influence=0.0)):
        t, cf = _host(**over)
        p = _params(t, cf)
        for reg, cls, prev in cases + [(torch.full((4, 16, 16), 25.0), torch.full((1, 16, 16), 0.0), (51.2, 51.2))]:
            rec = _decode_smooth(reg[None].cuda(), cls[None].cuda(), [prev], p)[0]
            box, score, flat, gap = _host_case(t, reg.cuda(), cls.cuda(), prev)
            assert int(rec["flat"]) == flat or gap <= 1e-12, (over, prev, int(rec["flat"]), flat)
            assert np.float32(rec["score"]).view(np.uint32) == score.view(np.uint32) or (np.isnan(rec["score"])
                                                                                          and np.isnan(score))
            assert _same_box(_rec_box(rec), box), (over, prev, _rec_box(rec), box)
    rec = _decode_smooth(torch.full((1, 4, 16, 16), 25.0).cuda(), torch.zeros(1, 1, 16, 16).cuda(), [(51.2, 51.2)],
                         _params(*_host(windowing="uniform", window_influence=0.0)))[0]
    assert int(rec["flat"]) == 0


# ------------------------------------------------------------------------------------------------------ trajectories
def _run(tracker, frames, init):
    tracker.initialize(frames[0], init)
    return np.array([list(map(int, tracker.update(f)["bbox"])) for f in frames[1:]], dtype=np.int64)


def test_trajectory_matches_host_smooth_path(net, clip):
    """FEARTracker(gpu_crop=True, smooth=True) over the whole clip == FEARTracker(smooth=True), and against the
    reference's own trajectory the bar of the host path: the first 20 frames identical and > 90 % overall."""
    g = golden("smooth_tracker.npz")
    host = _run(fb.FEARTracker(net, cuda_id=0, **CFG), clip, g["init_bbox"])
    dev_trk = fb.FEARTracker(net, cuda_id=0, gpu_crop=True, **CFG)
    dev = _run(dev_trk, clip, g["init_bbox"])
    assert dev_trk._gpu_crop_state["graph"] is not None
    same = (dev == host).all(1)
    ref = (dev[:len(g["trajectory"])] == g["trajectory"]).all(1)
    _dump("trajectory.json", {"frames": int(len(dev)), "identical_to_host": int(same.sum()),
                              "identical_to_reference": int(ref.sum()), "reference_frames": int(len(ref))})
    assert same.all(), (int(same.sum()), int(np.argmin(same)))
    assert ref[:20].all() and ref.mean() > 0.9, (int(ref.sum()), int(np.argmin(ref)))


# ------------------------------------------------------------------------------------------------------------- graph
def test_graph_replay_and_launch_count(clip, monkeypatch):
    """From the second update on, an update is one graph replay; an eager update launches one kernel fewer on the
    handle than plain gpu_crop (the decode is skipped; fear_decode_smooth and the crop are handle-free)."""
    g = golden("smooth_tracker.npz")
    n = _make_net(1)
    frames = clip[:12]
    per_update = {}
    for name, extra in (("plain", {}), ("smooth", {"smooth": True})):
        trk = fb.FEARTracker(n, cuda_id=0, gpu_crop=True, cuda_graph=False, **dict(fb.FEAR_XS_TRACKER_KWARGS, **extra))
        trk.initialize(frames[0], g["init_bbox"])
        trk.update(frames[1])
        c0 = n.launch_count()
        for f in frames[2:5]:
            trk.update(f)
        per_update[name] = (n.launch_count() - c0) / 3
    assert per_update["smooth"] == per_update["plain"] - 1, per_update

    replays = []
    real_replay = torch.cuda.CUDAGraph.replay
    monkeypatch.setattr(torch.cuda.CUDAGraph, "replay", lambda self: (replays.append(1), real_replay(self))[1])
    trk = fb.FEARTracker(n, cuda_id=0, gpu_crop=True, **CFG)
    trk.initialize(frames[0], g["init_bbox"])
    trk.update(frames[1])
    assert trk._gpu_crop_state["graph"] is None and not replays  # the first update runs eagerly
    for k, f in enumerate(frames[2:], 1):
        c0 = n.launch_count() if k > 1 else None
        trk.update(f)
        assert len(replays) == k
        if c0 is not None:
            assert n.launch_count() == c0  # nothing launched on the handle outside the replay
    _dump("launches.json", per_update)


def test_graph_recaptured_after_workspace_growth(clip):
    """A larger batch on the same net re-allocates the workspace (generation changes): the tracker re-captures its
    graph and the trajectory stays that of an undisturbed tracker."""
    g = golden("smooth_tracker.npz")
    frames = clip[:16]
    want = _run(fb.FEARTracker(_make_net(1), cuda_id=0, gpu_crop=True, **CFG), frames, g["init_bbox"])
    n = _make_net(1)
    trk = fb.FEARTracker(n, cuda_id=0, gpu_crop=True, **CFG)
    trk.initialize(frames[0], g["init_bbox"])
    out = [list(map(int, trk.update(f)["bbox"])) for f in frames[1:6]]
    graph, gen = trk._gpu_crop_state["graph"], n.generation()
    assert graph is not None
    zt, xt, _, _ = fo.synthetic_crops(12)
    n.track(xt.cuda(), n.get_features(zt.cuda()))  # batch 12 > reserved: workspace freed and re-allocated
    assert n.generation() != gen
    out += [list(map(int, trk.update(f)["bbox"])) for f in frames[6:]]
    st = trk._gpu_crop_state
    assert st["graph"] is not None and st["graph"] is not graph and st["generation"] == n.generation()
    assert np.array_equal(np.array(out), want)


# ------------------------------------------------------------------------------------------------------------- C ABI
def test_c_abi_errors():
    lib = _lib.load()
    reg = torch.zeros(2, 4, 16, 16, device="cuda")
    cls = torch.zeros(2, 1, 16, 16, device="cuda")
    prev = torch.ones(2, 2, dtype=torch.float64, device="cuda")
    params = torch.zeros(259, dtype=torch.float64, device="cuda")
    boxes = torch.zeros(2, 48, dtype=torch.uint8, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    ptrs = [reg.data_ptr(), cls.data_ptr(), prev.data_ptr(), params.data_ptr(), boxes.data_ptr()]

    def call(p, b):
        return lib.fear_decode_smooth(p[0], p[1], b, p[2], p[3], p[4], s)

    for k in range(5):
        p = list(ptrs)
        p[k] = None
        assert call(p, 2) == -1  # FEAR_EINVAL
    assert call(ptrs, 0) == -1 and call(ptrs, -3) == -1
    assert "bad argument" in _lib.last_error()
    torch.cuda.synchronize()
    assert not boxes.any()  # a refused call launches nothing
    assert call(ptrs, 2) == 0
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------ poisoned memory
def test_poisoned_memory():
    proc = subprocess.run([sys.executable, os.path.join(HERE, "poison_smooth_check.py")], capture_output=True,
                          text=True, timeout=1200)
    with open(os.path.join(OUT, "poison_smooth_check.log"), "w") as f:
        f.write(proc.stdout + "\n--- stderr ---\n" + proc.stderr)
    lines = [l for l in proc.stdout.splitlines() if l.startswith("POISON_CHECK ")]
    assert proc.returncode == 0 and lines, proc.stderr[-3000:]
    res = json.loads(lines[-1][len("POISON_CHECK "):])
    assert res["checked_calls"] > 0
    assert res["n_failures"] == 0, res["failures"]
