"""GPU tests of rotated and mirrored frames (fb.Oriented, fear_crop_targets_oriented_u8, fear_advance_targets_oriented).

Every comparison is exact: the oriented entry points on each of the eight frame tables against the plain view entry
points on ``image_ops.orient`` of the frame the table's kernels see; FEARMultiTracker and FEARTracker on Oriented device
frames against the same trackers fed those oriented frames as numpy arrays; graph replays against eager launches."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import feartracker_b200 as fb
from feartracker_b200 import _lib, image_ops
from feartracker_b200 import multi_tracker as mt
from tests import hdr_frames
from tests.test_gpu_multi_tracker import clip, net  # noqa: F401  (fixtures)
from tests.test_gpu_stream_subsets import bayer, bgra, planes, u8, u16

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
CFG = fb.FEAR_XS_TRACKER_KWARGS
CFG192 = dict(CFG, instance_size=192, score_size=12)


# ------------------------------------------------------------------------------------------------ what the kernels see
def host(t: torch.Tensor) -> np.ndarray:
    if t.dtype == torch.uint16:
        return t.view(torch.int16).cpu().numpy().view(np.uint16)
    return t.cpu().numpy()


def seen(f) -> np.ndarray:
    """The RGB frame the tracker sees for device frame ``f``, from its samples read back (image_ops' statements)."""
    if isinstance(f, fb.Oriented):
        return np.ascontiguousarray(image_ops.orient(seen(f.frame), f.code))
    if isinstance(f, torch.Tensor):
        return host(f)
    if isinstance(f, fb.V210Frame):
        y, u, v = image_ops.v210_unpack(host(f.t), f.width)
        return image_ops.yuv_to_rgb(y, u, v, f.matrix, f.full_range, bits=10, chroma_shift=(1, 0), transfer=f.transfer)
    if isinstance(f, mt._YUVFrame):
        return image_ops.yuv_to_rgb(host(f.y), host(f.u), host(f.v), f.matrix, f.full_range, f.bits, f.shift,
                                    f.CHROMA_SHIFT, f.transfer)
    if isinstance(f, (fb.BayerFrame, fb.MonoFrame)):
        if f.packing:
            codes = image_ops.mipi_unpack(host(f.t), f.shape[1], f.bits)
        else:
            codes = host(f.t)
            if f.bits > 8:
                codes = (codes >> f.shift) & np.uint16((1 << f.bits) - 1)
        if isinstance(f, fb.BayerFrame):
            return image_ops.bayer_to_rgb(codes, f.pattern, f.bits)
        return image_ops.mono_to_rgb(codes, f.bits, f.agc)
    assert isinstance(f, fb.RGBFrame) and f.layout != "planar"
    return image_ops.rgb_frame_to_rgb(host(f.tensors[0]), f.layout)


def even(rgb, rows=True):
    return rgb[:rgb.shape[0] & ~1 if rows else rgb.shape[0], :rgb.shape[1] & ~1]


# table -> two frames of it, from two RGB sources (odd sizes wherever the format allows them)
TABLE_FRAMES = {
    "views": lambda a, b: [u8(a.transpose(2, 0, 1)).permute(1, 2, 0), u8(b)],
    "yuv": lambda a, b: [fb.YUV420Frame(*(u8(p) for p in planes(even(a), 8, "420"))),
                         hdr_frames.p010_frame(*planes(even(b), 10, "420"), matrix="bt709")],
    "ycbcr": lambda a, b: [fb.YUV422Frame(*(u16(p) for p in planes(even(a, False), 10, "422")), bits=10),
                           fb.YUV444Frame(*(u8(p) for p in planes(b, 8, "444")), matrix="bt709", full_range=True)],
    "ycbcr_v210": lambda a, b: [hdr_frames.v210_frame(*planes(even(a, False), 10, "422"), col=16),
                                fb.YUV444Frame(*(u8(p) for p in planes(b, 8, "444")))],
    "ycbcr_hdr": lambda a, b: [hdr_frames.p010_frame(*hdr_frames.hdr_codes(even(a), "pq"), matrix="bt2020",
                                                     transfer="pq"),
                               hdr_frames.v210_frame(*hdr_frames.hdr_codes(even(b, False), "hlg", sub="422"),
                                                     matrix="bt2020", transfer="hlg")],
    "bayer": lambda a, b: [bayer(a), fb.BayerFrame(u16(b[..., 1].astype(np.int64) * 16), "GRBG", bits=12)],
    "mono": lambda a, b: [fb.MonoFrame(u16(a[..., 1].astype(np.int64) * 7 + 300), bits=16, agc="minmax"),
                          fb.MonoFrame(u8(b[..., 0]))],
    "rgb": lambda a, b: [bgra(a), u8(b)],
}


def table_of(frames, name):
    dtype = mt.TABLE_DTYPES[name]
    rec = np.zeros(len(frames), dtype)
    mt.write_records(rec, frames, name)
    return torch.from_numpy(rec.view(np.uint8).copy()).cuda()


def targets_for(shapes, pad=(17, 99, 201)):
    """FearTarget rows on frames of display ``shapes``: boxes overhanging each display edge, inside, tiny, huge."""
    rows = []
    for i, (h, w) in enumerate(shapes):
        for box in ([-5, 3, 20, 15], [w - 10, 5, 20, 12], [4, -6, 14, 20], [6, h - 8, 16, 20],
                    [w // 3, h // 3, w // 3 + 1, h // 3 + 2], [0, 0, 3, 3], [-w, -h, 3 * w, 3 * h]):
            r = np.zeros(16, np.int32)
            r[0], r[1:5], r[9:12] = i, box, pad
            rows.append(r)
    return torch.from_numpy(np.stack(rows)).cuda()


def boxes_for(n, seed):
    rng = np.random.default_rng(seed)
    rec = np.zeros(n, _lib.BOX_DTYPE)
    rec["x"], rec["y"] = rng.uniform(-80, 300, n), rng.uniform(-80, 300, n)
    rec["w"], rec["h"] = rng.uniform(-5, 300, n), rng.uniform(-5, 300, n)
    return torch.from_numpy(rec.view(np.uint8).copy()).cuda()


def view_step(rgbs, targets, boxes, offset, size):
    """Plain view crop + advance on numpy RGB frames -> (crops, targets)."""
    lib, n = _lib.load(), targets.shape[0]
    ts = [torch.from_numpy(r).cuda() for r in rgbs]
    table = table_of(ts, "views")
    t, crops = targets.clone(), torch.empty((n, size, size, 3), dtype=torch.uint8, device="cuda")
    _lib.check(lib.fear_crop_targets_view_u8(table.data_ptr(), len(ts), t.data_ptr(), n, offset, size,
                                             crops.data_ptr(), None), "crop")
    _lib.check(lib.fear_advance_targets_view(boxes.data_ptr(), table.data_ptr(), len(ts), t.data_ptr(), n, 256, None),
               "advance")
    torch.cuda.synchronize()
    return crops.cpu().numpy(), t.cpu().numpy()


def oriented_step(name, frames, codes, targets, boxes, offset, size):
    lib, n = _lib.load(), targets.shape[0]
    table = table_of(frames, name)
    if name == "mono":
        _lib.check(lib.fear_frame_range_mono(table.data_ptr(), len(frames), None), "range")
    d_codes = None if codes is None else torch.tensor(codes, dtype=torch.int32, device="cuda")
    cp = None if d_codes is None else d_codes.data_ptr()
    t, crops = targets.clone(), torch.empty((n, size, size, 3), dtype=torch.uint8, device="cuda")
    code = _lib.ORIENT_TABLES[name]
    _lib.check(lib.fear_crop_targets_oriented_u8(code, table.data_ptr(), cp, len(frames), t.data_ptr(), n, offset,
                                                 size, crops.data_ptr(), None), "oriented crop")
    _lib.check(lib.fear_advance_targets_oriented(boxes.data_ptr(), code, table.data_ptr(), cp, len(frames),
                                                 t.data_ptr(), n, 256, None), "oriented advance")
    torch.cuda.synchronize()
    return crops.cpu().numpy(), t.cpu().numpy()


def plain_step(name, frames, targets, boxes, offset, size):
    lib, n = _lib.load(), targets.shape[0]
    _, crop_fn, advance_fn = mt.ENTRY_POINTS[name]
    table = table_of(frames, name)
    if name == "mono":
        _lib.check(lib.fear_frame_range_mono(table.data_ptr(), len(frames), None), "range")
    t, crops = targets.clone(), torch.empty((n, size, size, 3), dtype=torch.uint8, device="cuda")
    _lib.check(getattr(lib, crop_fn)(table.data_ptr(), len(frames), t.data_ptr(), n, offset, size, crops.data_ptr(),
                                     None), crop_fn)
    _lib.check(getattr(lib, advance_fn)(boxes.data_ptr(), table.data_ptr(), len(frames), t.data_ptr(), n, 256, None),
               advance_fn)
    torch.cuda.synchronize()
    return crops.cpu().numpy(), t.cpu().numpy()


@pytest.mark.parametrize("name", list(TABLE_FRAMES))
def test_oriented_entry_points_equal_the_view_entry_points_on_oriented_frames(clip, name):  # noqa: F811
    rng = np.random.default_rng(7)
    small = rng.integers(0, 256, (37, 53, 3), dtype=np.uint8)
    frames = TABLE_FRAMES[name](small, clip[5])
    rgbs = [seen(f) for f in frames]
    for codes in [(c, (c + 3) % 8) for c in range(8)]:
        shapes = [image_ops.orient(r, c).shape[:2] for r, c in zip(rgbs, codes)]
        targets = targets_for(shapes)
        boxes = boxes_for(targets.shape[0], sum(codes))
        want_rgbs = [np.ascontiguousarray(image_ops.orient(r, c)) for r, c in zip(rgbs, codes)]
        for offset, size in ((2.0, 96), (0.2, 128)):
            want = view_step(want_rgbs, targets, boxes, offset, size)
            got = oriented_step(name, frames, codes, targets, boxes, offset, size)
            assert np.array_equal(got[0], want[0]), (name, codes, offset)
            assert np.array_equal(got[1], want[1]), (name, codes, offset)
    # a null code array, and codes of 0, are the table's plain entry points
    targets = targets_for([r.shape[:2] for r in rgbs])
    boxes = boxes_for(targets.shape[0], 3)
    want = plain_step(name, frames, targets, boxes, 2.0, 64)
    for codes in (None, (0, 0)):
        got = oriented_step(name, frames, codes, targets, boxes, 2.0, 64)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), (name, codes)
    # a code outside [0, 7]: a padding crop, and the box is kept (its context box is still written)
    for bad in (8, -1, 1 << 30, -(1 << 31)):
        crops, rows = oriented_step(name, frames, (bad, 1), targets, boxes, 2.0, 64)
        first = targets.cpu().numpy()[:, 0] == 0
        assert (crops[first] == np.array([17, 99, 201], np.uint8)).all(), (name, bad)
        assert np.array_equal(rows[first][:, 1:5], targets.cpu().numpy()[first][:, 1:5]), (name, bad)


def test_c_abi_rejects_bad_arguments():
    lib = _lib.load()
    t = torch.zeros(4096, dtype=torch.uint8, device="cuda")
    p = t.data_ptr()

    def crop(table=0, d_table=p, orient=p, F=1, targets=p, N=1, size=256, crops=p):
        return lib.fear_crop_targets_oriented_u8(table, d_table, orient, F, targets, N, 2.0, size, crops, None)

    def advance(boxes=p, table=0, d_table=p, orient=p, F=1, targets=p, N=1, size=256):
        return lib.fear_advance_targets_oriented(boxes, table, d_table, orient, F, targets, N, size, None)

    for kw in [dict(table=-1), dict(table=8), dict(d_table=None), dict(targets=None), dict(crops=None), dict(F=0),
               dict(F=-3), dict(N=0), dict(N=-1), dict(N=65536), dict(size=0)]:
        assert crop(**kw) == -1, kw
        assert _lib.last_error(), kw
    for kw in [dict(table=-1), dict(table=8), dict(boxes=None), dict(d_table=None), dict(targets=None), dict(F=0),
               dict(N=0), dict(size=0)]:
        assert advance(**kw) == -1, kw
    torch.cuda.synchronize()
    assert not t.any()  # nothing was launched


# ------------------------------------------------------------------------------------------------ trackers
def _yuyv10(rgb):
    y, u, v = planes(rgb, 10, "422")
    h, w = y.shape
    surf = np.zeros((h, 2 * w), np.int64)
    surf[:, 0::2], surf[:, 1::4], surf[:, 3::4] = y, u, v
    return fb.YUV422Frame.yuyv(u16(surf << 6), bits=10)


# kind -> device frame of stream j from its RGB frame
KINDS = {
    "cuda": lambda rgb, j: u8(rgb.transpose(2, 0, 1)).permute(1, 2, 0) if j % 2 else u8(rgb),
    "nv12": lambda rgb, j: fb.YUV420Frame.nv12(u8(np.concatenate(
        [planes(rgb, 8, "420")[0], np.stack(planes(rgb, 8, "420")[1:], -1).reshape(rgb.shape[0] // 2, -1)]))),
    "yuyv10": lambda rgb, j: _yuyv10(rgb),
    "v210": lambda rgb, j: hdr_frames.v210_frame(*planes(rgb, 10, "422"), col=32 * j),
    "bayer": lambda rgb, j: bayer(rgb),
    "mono_y16_agc": lambda rgb, j: fb.MonoFrame(u16(rgb[..., 1].astype(np.int64) * 40 + 1000 * j), bits=16,
                                                agc="minmax"),
    "bgra": lambda rgb, j: bgra(rgb),
}
STREAMS = 4
CODES = [(0, 1, 6, 3), (5, 2, 7, 4), (1, 3, 1, 3)]  # per stream, cycling through the updates; 0 as Oriented(f, 0)
RECTS = [[60, 150, 45, 80], [0, 0, 40, 60], [200, 120, 60, 90], [-10, 400, 50, 50]]


def stream_rgb(clip, j, t):
    c = clip[t]
    return [c, np.ascontiguousarray(c[:, ::-1]), np.ascontiguousarray(np.roll(c, (17, 40), axis=(0, 1))),
            np.ascontiguousarray(c[::-1])][j]


def oriented_frames(clip, kind, t, codes, plain=()):
    frames = [KINDS[kind](stream_rgb(clip, j, t), j) for j in range(STREAMS)]
    return [f if j in plain else fb.Oriented(f, 90 * (c & 3), bool(c & 4)) for j, (f, c) in enumerate(zip(frames, codes))]


@pytest.mark.parametrize("cfg", [CFG, CFG192], ids=["256", "192"])
@pytest.mark.parametrize("kind", list(KINDS))
def test_multi_tracker_on_oriented_frames_matches_oriented_numpy(net, clip, kind, cfg):  # noqa: F811
    T = 10
    got_trk, ref_trk = (fb.FEARMultiTracker(net, cuda_id=0, max_targets=8, **cfg) for _ in range(2))
    rects = RECTS + [[30, 30, 80, 40]] * 2
    streams = [0, 1, 2, 3, 1, 2]
    frames = oriented_frames(clip, kind, 0, CODES[0], plain=(0,))
    got_trk.add(frames, rects, streams)
    ref_trk.add([seen(f) for f in frames], rects, streams)
    for t in range(1, T + 1):
        frames = oriented_frames(clip, kind, t, CODES[t % 3], plain=(0,) if t % 2 else ())
        rgbs = [seen(f) for f in frames]
        if t % 3 == 2:  # a mapping of some streams
            live = [3, 1] if t % 2 else [0, 2]
            a = got_trk.update({j: frames[j] for j in live})
            b = ref_trk.update({j: rgbs[j] for j in live})
        else:
            a, b = got_trk.update(frames), ref_trk.update(rgbs)
        for key in ("bbox", "score", "ids"):
            assert a[key].dtype == b[key].dtype and np.array_equal(a[key], b[key]), (kind, t, key)
        assert np.array_equal(got_trk._buf["state"][:6].cpu(), ref_trk._buf["state"][:6].cpu()), (kind, t)
    assert got_trk._graph_key[-1] is True


def test_code_zero_is_the_plain_frame_with_the_same_launches(net, clip):  # noqa: F811
    plain, wrapped = (fb.FEARMultiTracker(net, cuda_id=0, max_targets=4, **CFG) for _ in range(2))
    frames = [KINDS["nv12"](stream_rgb(clip, j, 0), j) for j in range(2)]
    plain.add(frames, RECTS[:2], [0, 1])
    wrapped.add([fb.Oriented(f) for f in frames], RECTS[:2], [0, 1])
    deltas = {}
    for t in range(1, 8):
        frames = [KINDS["nv12"](stream_rgb(clip, j, t), j) for j in range(2)]
        for name, trk, fr in (("plain", plain, frames), ("wrapped", wrapped, [fb.Oriented(f, 0) for f in frames])):
            c0 = net.launch_count()
            out = trk.update(fr)
            deltas.setdefault(name, []).append(net.launch_count() - c0)
            deltas.setdefault(name + "_out", []).append(out)
    for a, b in zip(deltas["plain_out"], deltas["wrapped_out"]):
        for key in ("bbox", "score", "ids"):
            assert np.array_equal(a[key], b[key])
    assert deltas["plain"] == deltas["wrapped"]
    key, wkey = plain._graph_key, wrapped._graph_key
    assert key[:3] == wkey[:3] and key[4] == wkey[4] and key[5] is False and wkey[5] is True


class OrientCountingGraph(torch.cuda.CUDAGraph):
    """A CUDAGraph that counts the graphs made while it is patched in, in a counter of its own (other modules' counting
    graphs keep theirs)."""
    made = 0

    def __new__(cls, *args, **kwargs):
        OrientCountingGraph.made += 1
        return super().__new__(cls, *args, **kwargs)


def test_new_codes_replay_without_recapture(net, clip, monkeypatch):  # noqa: F811
    monkeypatch.setattr(torch.cuda, "CUDAGraph", OrientCountingGraph)
    made0 = OrientCountingGraph.made
    graph = fb.FEARMultiTracker(net, cuda_id=0, max_targets=8, **CFG)
    eager = fb.FEARMultiTracker(net, cuda_id=0, max_targets=8, **dict(CFG, cuda_graph=False))
    for trk in (graph, eager):
        trk.add(oriented_frames(clip, "cuda", 0, CODES[0]), RECTS, [0, 1, 2, 3])
    outs = {id(graph): [], id(eager): []}
    made = None
    for t in range(1, 16):
        codes = [(t * (j + 1)) % 8 for j in range(STREAMS)]
        for trk in (graph, eager):
            outs[id(trk)].append(trk.update(oriented_frames(clip, "cuda", t, codes)))
            sub = {j: fb.Oriented(u8(stream_rgb(clip, j, t)), 90 * ((t + j) % 4)) for j in (1, 3)}
            outs[id(trk)].append(trk.update(sub))
        if t == 3:
            made = OrientCountingGraph.made - made0
            g = graph._graph
    # the list graph and one subset graph, captured on their second calls; new codes replay them
    assert made == 2 and OrientCountingGraph.made - made0 == made and graph._graph is g
    for a, b in zip(outs[id(graph)], outs[id(eager)]):
        for key in ("bbox", "score", "ids"):
            assert np.array_equal(a[key], b[key])


def fear_tracker_run(net, cfg, frames, rect, smooth):
    trk = fb.FEARTracker(net, cuda_id=0, smooth=smooth, **cfg)
    trk.initialize(frames[0], np.asarray(rect))
    return [trk.update(f)["bbox"] for f in frames[1:]], trk.tracking_state


@pytest.mark.parametrize("smooth", [False, True], ids=["plain", "smooth"])
@pytest.mark.parametrize("kind", ["cuda", "nv12", "v210", "mono_y16_agc", "bgra", "bayer"])
def test_fear_tracker_on_oriented_frames_matches_oriented_numpy(net, clip, kind, smooth):  # noqa: F811
    T = 10
    frames = [fb.Oriented(KINDS[kind](stream_rgb(clip, 0, t), 1), 90 * (t % 4), t % 3 == 1) for t in range(T)]
    rgbs = [seen(f) for f in frames]
    rect = [100, 200, 60, 90]
    got, gst = fear_tracker_run(net, CFG, frames, rect, smooth)
    want, wst = fear_tracker_run(net, dict(CFG, gpu_crop=True), rgbs, rect, smooth)
    assert np.array_equal(np.array(got), np.array(want)), kind
    assert np.array_equal(gst.mean_color, wst.mean_color)
    dev = fb.FEARTracker(net, cuda_id=0, **CFG)
    host = fb.FEARTracker(net, cuda_id=0, gpu_crop=True, **CFG)
    zf_dev = dev.get_template_features(frames[1], np.array(rect))
    zf_host = host.get_template_features(rgbs[1], np.array(rect))
    assert torch.equal(zf_dev, zf_host)


def test_fear_tracker_at_instance_size_192(net, clip):  # noqa: F811
    frames = [fb.Oriented(KINDS["nv12"](stream_rgb(clip, 2, t), 0), 270, True) for t in range(8)]
    got, _ = fear_tracker_run(net, CFG192, frames, [50, 300, 60, 90], False)
    want, _ = fear_tracker_run(net, dict(CFG192, gpu_crop=True), [seen(f) for f in frames], [50, 300, 60, 90], False)
    assert np.array_equal(np.array(got), np.array(want))


# ---------------------------------------------------------------------------------------------------- poison
def test_oriented_entry_points_on_poisoned_memory():
    """tests/poison_orientation_check.py in its own process: guarded, poisoned tables, codes, targets and crops."""
    proc = subprocess.run([sys.executable, os.path.join(HERE, "poison_orientation_check.py")], capture_output=True,
                          text=True, timeout=1200)
    lines = [l for l in proc.stdout.splitlines() if l.startswith("POISON_CHECK ")]
    assert proc.returncode == 0 and lines, f"poison_orientation_check failed: {proc.stderr[-3000:]}"
    res = json.loads(lines[-1][len("POISON_CHECK "):])
    assert res["checked_calls"] > 0
    assert res["n_failures"] == 0, res["failures"]
