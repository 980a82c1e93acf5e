"""GPU tests of FEARMultiTracker.update / add on {stream id: frame} mappings (a step over the targets of some streams
only) and of fear_gather_targets / fear_scatter_targets.

Every comparison is exact: a mapping of every stream against the list on each frame table; every target of streams
ticking at different rates against its own FEARTracker(gpu_crop=True) fed only the frames its stream delivered; the
device rows and templates of the targets not stepped against their previous bits; the kernels against numpy."""
import numpy as np
import pytest
import torch

import feartracker_b200 as fb
from feartracker_b200 import _lib
from feartracker_b200 import multi_tracker as mt
from oracle import fear_oracle as fo
from tests import hdr_frames
from tests.helpers import load_full_state
from tests.test_gpu_multi_tracker import clip, net  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu
CFG = fb.FEAR_XS_TRACKER_KWARGS
CFG192 = dict(CFG, instance_size=192, score_size=12)
NAMES = ("clip", "mirror", "window", "shifted")
# two targets per stream, at and beyond the frame edges among them
RECTS = {"clip": [[163, 53, 45, 174], [0, 0, 40, 60]], "mirror": [[272, 53, 45, 174], [440, 200, 40, 56]],
         "window": [[113, 23, 45, 120], [250, 140, 60, 40]], "shifted": [[180, 70, 45, 174], [-10, 100, 50, 50]]}


def sources(clip, T):
    """The four streams of the demo clip (480 x 256): the clip, its mirror, a window and a shifted copy."""
    c = clip[:T]
    return {"clip": c, "mirror": np.ascontiguousarray(c[:, :, ::-1]),
            "window": np.ascontiguousarray(c[:, 30:200, 50:350]),
            "shifted": np.ascontiguousarray(np.roll(c, (17, 40), axis=(1, 2)))}


def fear_tracker_run(net, cfg, frames, rect):
    """(boxes (T - 1, 4) int64, scores (T - 1,) float32) of FEARTracker(gpu_crop=True) initialised on frames[0] and
    updated on the rest."""
    trk = fb.FEARTracker(net, cuda_id=0, gpu_crop=True, **cfg)
    trk.initialize(frames[0], np.asarray(rect))
    scores, record = [], trk._track_record_gpu_crop

    def keep_score(image, params):
        rec = record(image, params)
        scores.append(np.float32(rec["score"]))
        return rec

    trk._track_record_gpu_crop = keep_score
    boxes = [trk.update(f)["bbox"] for f in frames[1:]]
    return np.array(boxes, dtype=np.int64).reshape(-1, 4), np.array(scores, dtype=np.float32)


class History:
    """Per target id: the frames its own tracker sees (its add frame, then every frame its stream delivered while it
    lived) and the (box, score) FEARMultiTracker gave it on each."""

    def __init__(self):
        self.rect, self.frames, self.out = {}, {}, {}

    def added(self, ids, rects, frames):
        for tid, rect, f in zip(ids, rects, frames):
            self.rect[int(tid)], self.frames[int(tid)], self.out[int(tid)] = rect, [f], []

    def stepped(self, out, frame_of):
        assert np.all(np.diff(out["ids"]) > 0)  # in the order of ids
        for i, tid in enumerate(out["ids"]):
            self.frames[int(tid)].append(frame_of(int(tid)))
            self.out[int(tid)].append((out["bbox"][i], out["score"][i]))

    def check(self, net, cfg):
        for tid, frames in self.frames.items():
            want_b, want_s = fear_tracker_run(net, cfg, frames, self.rect[tid])
            got_b = np.array([b for b, _ in self.out[tid]], dtype=np.int64).reshape(-1, 4)
            got_s = np.array([s for _, s in self.out[tid]], dtype=np.float32)
            assert np.array_equal(got_b, want_b), (tid, self.rect[tid])
            assert np.array_equal(got_s, want_s), (tid, self.rect[tid])


def device_rows(trk):
    n = len(trk)
    return trk._buf["state"][:n].cpu().numpy().copy(), trk._buf["zf"][:n].view(torch.int32).cpu().numpy().copy()


def subset_update(trk, frames, before=None):
    """trk.update(frames) of a mapping; checks that the rows and templates of the targets not stepped, and the frame,
    padding colour and reserved words of the stepped ones, keep their bits."""
    state0, zf0 = device_rows(trk) if before is None else before
    out = trk.update(frames)
    state1, zf1 = device_rows(trk)
    stepped = np.isin(trk.ids, out["ids"])
    assert np.array_equal(zf1, zf0)
    assert np.array_equal(state1[~stepped], state0[~stepped])
    keep = [0] + list(range(9, 16))
    assert np.array_equal(state1[stepped][:, keep], state0[stepped][:, keep])
    return out


# ------------------------------------------------------------------------------------------------ frame tables
def u8(a) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint8)).cuda()


def u16(a) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint16).view(np.int16)).cuda().view(torch.uint16)


def planes(rgb, bits, sub):
    return hdr_frames.encode_rgb([c / 255.0 for c in np.moveaxis(rgb.astype(np.float64), -1, 0)], bits, False, sub)


def bayer(rgb):
    raw = rgb[..., 1].copy()
    raw[0::2, 0::2], raw[1::2, 1::2] = rgb[0::2, 0::2, 0], rgb[1::2, 1::2, 2]
    return fb.BayerFrame(u8(raw), "RGGB")


def bgra(rgb):
    surf = np.full(rgb.shape[:2] + (4,), 255, np.uint8)
    surf[..., :3] = rgb[..., ::-1]
    return fb.RGBFrame(u8(surf), "bgra")


# kind -> (frame of stream j from its RGB frame, the table the step reads)
KINDS = {
    "numpy": (lambda rgb, j: rgb, "views"),
    "views": (lambda rgb, j: u8(rgb.transpose(2, 0, 1)).permute(1, 2, 0), "views"),
    "yuv": (lambda rgb, j: fb.YUV420Frame(*(u8(p) for p in planes(rgb, 8, "420"))), "yuv"),
    "ycbcr": (lambda rgb, j: (fb.YUV422Frame if j % 2 else fb.YUV444Frame)(
        *(u8(p) for p in planes(rgb, 8, "422" if j % 2 else "444"))), "ycbcr"),
    "v210": (lambda rgb, j: hdr_frames.v210_frame(*planes(rgb, 10, "422")) if j % 2 else
             fb.YUV420Frame(*(u8(p) for p in planes(rgb, 8, "420"))), "ycbcr_v210"),
    "ycbcr_hdr": (lambda rgb, j: hdr_frames.p010_frame(*hdr_frames.hdr_codes(rgb, "pq"), matrix="bt2020",
                                                       transfer="pq") if j % 2 else
                  hdr_frames.i420_frame(*hdr_frames.hdr_codes(rgb, "hlg"), matrix="bt2020", transfer="hlg"),
                  "ycbcr_hdr"),
    "bayer": (lambda rgb, j: bayer(rgb), "bayer"),
    "mono": (lambda rgb, j: fb.MonoFrame(u16(rgb[..., 1].astype(np.int64) * 16 + j), bits=12, agc="minmax"), "mono"),
    "rgb": (lambda rgb, j: bgra(rgb) if j % 2 else u8(rgb), "rgb"),
}


@pytest.mark.parametrize("kind", list(KINDS))
def test_mapping_of_every_stream_equals_the_list(net, clip, kind):  # noqa: F811
    T = 20
    make, table = KINDS[kind]
    src = sources(clip, T + 1)
    rects = [r for s in NAMES for r in RECTS[s]]
    streams = [j for j, s in enumerate(NAMES) for _ in RECTS[s]]
    lst, mp = (fb.FEARMultiTracker(net, cuda_id=0, max_targets=8, **CFG) for _ in range(2))
    frames = [make(src[s][0], j) for j, s in enumerate(NAMES)]
    lst.add(frames, rects, streams)
    mp.add(dict(enumerate(frames)), rects, streams)
    for t in range(1, T + 1):
        frames = [make(src[s][t], j) for j, s in enumerate(NAMES)]
        a = lst.update(frames)
        pairs = list(enumerate(frames))
        b = mp.update(dict(pairs[::-1] if t % 2 else pairs))  # the mapping's order does not matter
        for key in ("bbox", "score", "ids"):
            assert a[key].dtype == b[key].dtype and np.array_equal(a[key], b[key]), (kind, t, key)
        assert all(np.array_equal(x, y) for x, y in zip(device_rows(lst), device_rows(mp))), (kind, t)
    assert lst._graph_key[2] == table
    assert [k[2] for k in mp._subset_graphs] == [table]


# ------------------------------------------------------------------------------------------------ different rates
def delivers(name, t):
    """Whether stream ``name`` has a frame at tick t: periods 1, 2 and 3, and an irregular stream stalled for 40."""
    if name == "clip":
        return True
    if name == "mirror":
        return t % 2 == 0
    if name == "window":
        return t % 3 == 0
    return t % 5 in (0, 1, 3) and not 30 <= t < 70


@pytest.mark.parametrize("cfg,device_frames", [(CFG, False), (CFG192, True)], ids=["256", "192"])
def test_streams_at_different_rates_match_their_own_trackers(net, clip, cfg, device_frames):  # noqa: F811
    T = 120
    src = sources(clip, T + 1)
    as_frame = u8 if device_frames else (lambda a: a)
    trk = fb.FEARMultiTracker(net, cuda_id=0, max_targets=8, **cfg)
    hist = History()
    rects = [r for s in NAMES for r in RECTS[s]]
    streams = [j for j, s in enumerate(NAMES) for _ in RECTS[s]]
    ids = trk.add({j: as_frame(src[s][0]) for j, s in enumerate(NAMES)}, rects, streams)
    hist.added(ids, rects, [src[NAMES[j]][0] for j in streams])
    for t in range(1, T + 1):
        live = [j for j, s in enumerate(NAMES) if delivers(s, t)]
        out = subset_update(trk, {j: as_frame(src[NAMES[j]][t]) for j in live})
        assert sorted(set(np.asarray(streams)[out["ids"]])) == live
        hist.stepped(out, lambda tid: src[NAMES[streams[tid]]][t])
    hist.check(net, cfg)


# ------------------------------------------------------------------------------------------------ add and remove
def test_add_and_remove_with_sparse_stream_ids(net, clip):  # noqa: F811
    src = sources(clip, 41)
    a, b = src["clip"], src["mirror"]
    trk = fb.FEARMultiTracker(net, cuda_id=0, max_targets=8, **CFG)
    hist, stream_of = History(), {}

    def add(frames, rects, streams):
        ids = trk.add(frames, rects, streams)
        hist.added(ids, rects, [frames[s] for s in streams])
        stream_of.update({int(i): s for i, s in zip(ids, streams)})
        assert np.all(np.diff(trk.ids) > 0)

    add({3: a[0]}, RECTS["clip"], [3, 3])
    for t in range(1, 41):
        frames = {3: a[t]} if t < 6 or t % 2 else {3: a[t], 17: b[t]}
        if t == 33:
            frames = {17: b[t], 3: a[t], 5: src["window"][t]}  # a key without targets
        out = subset_update(trk, frames)
        hist.stepped(out, lambda tid: frames[stream_of[tid]])
        if t == 5:
            add({3: a[5], 17: b[5]}, RECTS["mirror"], [17, 17])
        if t == 20:
            trk.remove([1])
        if t == 25:
            add({17: b[25]}, [[300, 80, 60, 90]], [17])
        if t == 30:
            with pytest.raises(ValueError, match="targets track stream 17 but only 2 frames were given"):
                trk.update([a[t], b[t]])
    assert trk.ids.tolist() == [0, 2, 3, 4]
    hist.check(net, CFG)


def test_list_and_mapping_updates_interleaved_with_add_and_remove(net, clip):  # noqa: F811
    T = 30
    src = sources(clip, T + 1)
    seq = [src["clip"], src["mirror"], src["window"]]
    trk = fb.FEARMultiTracker(net, cuda_id=0, max_targets=8, **CFG)
    hist, stream_of = History(), {}

    def add(frames, rects, streams):
        ids = trk.add(frames, rects, streams)
        hist.added(ids, rects, [frames[s] for s in streams])
        stream_of.update({int(i): s for i, s in zip(ids, streams)})

    add([s[0] for s in seq], RECTS["clip"] + RECTS["mirror"][:1] + RECTS["window"][:1], [0, 0, 1, 2])
    for t in range(1, T + 1):
        frames = [s[t] for s in seq] if t % 2 else {2: seq[2][t], 0: seq[0][t]}
        out = trk.update(frames) if t % 2 else subset_update(trk, frames)
        hist.stepped(out, lambda tid: frames[stream_of[tid]])
        if t == 8:
            add({1: seq[1][8]}, RECTS["mirror"][1:], [1])
        if t == 12:
            trk.remove([0])
        if t == 15:
            add([s[15] for s in seq], RECTS["window"][1:], [2])
    assert trk.ids.tolist() == [1, 2, 3, 4, 5]
    hist.check(net, CFG)


# ------------------------------------------------------------------------------------------------ graphs
class CountingGraph(torch.cuda.CUDAGraph):
    made = 0

    def __new__(cls, *args, **kwargs):
        CountingGraph.made += 1
        return super().__new__(cls, *args, **kwargs)


def _four_streams(net, cfg=CFG, max_targets=8):
    trk = fb.FEARMultiTracker(net, cuda_id=0, max_targets=max_targets, **cfg)
    return trk


PATTERN = [(0, 1), (2, 3), (0, 2, 3), (1,)]


def _run_pattern(trk, src, t0, rounds):
    outs = []
    for r in range(rounds):
        for k, live in enumerate(PATTERN):
            t = t0 + r * len(PATTERN) + k
            outs.append(trk.update({j: src[NAMES[j]][t] for j in live}))
    return outs


def test_repeating_subset_pattern_replays_without_recapture(net, clip, monkeypatch):  # noqa: F811
    src = sources(clip, 40)
    rects = [r for s in NAMES for r in RECTS[s]]
    streams = [j for j, s in enumerate(NAMES) for _ in RECTS[s]]
    monkeypatch.setattr(torch.cuda, "CUDAGraph", CountingGraph)
    graph, eager = _four_streams(net), _four_streams(net, dict(CFG, cuda_graph=False))
    for trk in (graph, eager):
        trk.add([src[s][0] for s in NAMES], rects, streams)
    first = _run_pattern(graph, src, 1, 3)  # every key seen three times: captured on its second call
    captured = CountingGraph.made
    assert captured == 3  # keys (M, F) = (4, 2), (6, 3), (2, 1)
    cached = {k: e["graph"] for k, e in graph._subset_graphs.items()}
    second = _run_pattern(graph, src, 13, 5)
    assert CountingGraph.made == captured
    assert {k: e["graph"] for k, e in graph._subset_graphs.items()} == cached
    assert all(g is not None for g in cached.values())
    want = _run_pattern(eager, src, 1, 8)
    assert all(e["graph"] is None for e in eager._subset_graphs.values())
    for got, exp in zip(first + second, want):
        for key in ("bbox", "score", "ids"):
            assert np.array_equal(got[key], exp[key])


def test_list_graph_survives_subset_steps(net, clip):  # noqa: F811
    src = sources(clip, 30)
    rects = [r for s in NAMES for r in RECTS[s]]
    streams = [j for j, s in enumerate(NAMES) for _ in RECTS[s]]
    trk = _four_streams(net)
    hist = History()
    hist.added(trk.add([src[s][0] for s in NAMES], rects, streams), rects, [src[NAMES[j]][0] for j in streams])
    for t in range(1, 30):
        if t % 6 < 3:
            frames = [src[s][t] for s in NAMES]
            out = trk.update(frames)
        else:
            frames = {j: src[NAMES[j]][t] for j in PATTERN[t % 4]}
            out = subset_update(trk, frames)
        hist.stepped(out, lambda tid: frames[streams[tid]])
        if t == 3:
            g = trk._graph
            assert g is not None
        if t > 3 and t % 6 < 3:
            assert trk._graph is g
    hist.check(net, CFG)


def test_workspace_growth_recaptures_subset_graphs(clip, monkeypatch):  # noqa: F811
    n2 = fb.FEARNet(**fb.FEAR_XS_MODEL_KWARGS)
    n2.load_state_dict(load_full_state(), strict=True)
    n2 = n2.cuda().eval()
    src = sources(clip, 40)
    rects = [r for s in NAMES for r in RECTS[s]]
    streams = [j for j, s in enumerate(NAMES) for _ in RECTS[s]]
    monkeypatch.setattr(torch.cuda, "CUDAGraph", CountingGraph)
    trk = _four_streams(n2)
    hist = History()
    hist.added(trk.add([src[s][0] for s in NAMES], rects, streams), rects, [src[NAMES[j]][0] for j in streams])

    def run(t0, t1):
        for t in range(t0, t1):
            frames = {j: src[NAMES[j]][t] for j in PATTERN[t % 2]}
            hist.stepped(trk.update(frames), lambda tid: frames[streams[tid]])

    run(1, 10)
    old = [e["graph"] for e in trk._subset_graphs.values()]
    assert len(old) == 1 and old[0] is not None  # both halves have (M, F) = (4, 2)
    made, gen = CountingGraph.made, n2.generation()
    zt, xt, _, _ = fo.synthetic_crops(12)
    n2.track(xt.cuda(), n2.get_features(zt.cuda()))  # batch 12 > reserved 8: the workspace is re-allocated
    assert n2.generation() != gen
    run(10, 40)
    assert CountingGraph.made == made + 1
    new = [e["graph"] for e in trk._subset_graphs.values()]
    assert len(new) == 1 and new[0] is not None and new[0] is not old[0]
    assert trk._subset_gen == n2.generation()
    hist.check(n2, CFG)


def test_subset_graph_cache_is_bounded_and_least_recently_used_goes_first(net, clip):  # noqa: F811
    frame = clip[0]
    trk = fb.FEARMultiTracker(net, cuda_id=0, max_targets=mt.SUBSET_GRAPHS + 2, **CFG)
    n = mt.SUBSET_GRAPHS + 2
    trk.add(list(np.repeat(frame[None], n, 0)), [[163, 53, 45, 174]] * n, list(range(n)))
    for m in range(1, n + 1):  # n keys (M = m, F = m), each called twice
        for _ in range(2):
            trk.update({j: clip[1] for j in range(m)})
    keys = list(trk._subset_graphs)
    assert len(keys) == mt.SUBSET_GRAPHS
    assert [k[0] for k in keys] == list(range(3, n + 1))


def test_launch_counts_of_subset_and_list_steps(net, clip):  # noqa: F811
    """Handle launches per subset step equal those per list step at M = 1 and M = 16, and a subset step runs exactly
    two kernels more (gather and scatter)."""
    src = sources(clip, 8)
    for m in (1, 16):
        trk = fb.FEARMultiTracker(net, cuda_id=0, max_targets=32, cuda_graph=False, **CFG)
        trk.add([src["clip"][0], src["mirror"][0]], [[163, 53, 45, 174]] * 2 * m, [0] * m + [1] * m)
        trk.update([src["clip"][1], src["mirror"][1]])
        trk.update({1: src["mirror"][1]})
        torch.cuda.synchronize()
        c0 = net.launch_count()
        trk.update([src["clip"][2], src["mirror"][2]])
        c1 = net.launch_count()
        out = trk.update({1: src["mirror"][2]})
        c2 = net.launch_count()
        assert out["ids"].tolist() == list(range(m, 2 * m))
        assert c1 - c0 == c2 - c1 > 0, (m, c1 - c0, c2 - c1)

        def kernels(call):
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                call()
                torch.cuda.synchronize()
            names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
            return [n for n in names if "memcpy" not in n.lower() and "memset" not in n.lower()]

        lst = kernels(lambda: trk.update([src["clip"][3], src["mirror"][3]]))
        sub = kernels(lambda: trk.update({1: src["mirror"][3]}))
        assert len(sub) == len(lst) + 2, (m, len(lst), len(sub))
        assert sum("gather_targets_kernel" in n for n in sub) == 1
        assert sum("scatter_targets_kernel" in n for n in sub) == 1


# ------------------------------------------------------------------------------------------------ kernels
GUARD = 4096  # int32 words of guard band on each side of every buffer
FILLS = {"zero": 0, "nan": 0x7FC00001, "finite": 0x3F8CCCCD}
TEMPLATE_INTS = 256 * 8 * 8


def guarded(n_words, fill):
    """An int32 device buffer of n_words with GUARD words on each side, every word ``fill``; -> (whole, interior)."""
    whole = torch.full((n_words + 2 * GUARD,), fill, dtype=torch.int32, device="cuda")
    return whole, whole[GUARD:GUARD + n_words]


def selections(rng, N):
    bad = [-1, N, N + 7, -2 ** 31, 2 ** 31 - 1]
    rows = rng.integers(0, N, 3000)
    rows[rng.choice(3000, len(bad), replace=False)] = bad
    distinct = rng.permutation(N)[:2500].astype(np.int64)
    distinct_bad = np.concatenate([distinct, bad])
    rng.shuffle(distinct_bad)
    return {"random": (rows, False), "all": (rng.permutation(N), True), "distinct_with_bad": (distinct_bad, True)}


@pytest.mark.parametrize("fill", list(FILLS))
def test_gather_and_scatter_equal_numpy_on_poisoned_buffers(fill):
    lib = _lib.load()
    rng = np.random.default_rng(12000 + FILLS[fill] % 97)
    N = 12000
    targets_np = rng.integers(-2 ** 31, 2 ** 31, (N, 16), dtype=np.int64).astype(np.int32)
    t_whole, targets = guarded(N * 16, FILLS[fill])
    targets.copy_(torch.from_numpy(targets_np.reshape(-1)))
    z_whole, templates = guarded(N * TEMPLATE_INTS, FILLS[fill])
    templates.copy_(torch.randint(-2 ** 31, 2 ** 31 - 1, (N * TEMPLATE_INTS,), dtype=torch.int32, device="cuda"))
    z_before = z_whole.clone()
    for name, (rows, distinct) in selections(rng, N).items():
        M = rows.size
        frames = rng.integers(-2 ** 31, 2 ** 31, M, dtype=np.int64).astype(np.int32)
        sel_np = np.stack([rows.astype(np.int32), frames], 1)
        s_whole, sel = guarded(2 * M, FILLS[fill])
        sel.copy_(torch.from_numpy(sel_np.reshape(-1)))
        st_whole, step_t = guarded(M * 16, FILLS[fill])
        sz_whole, step_z = guarded(M * TEMPLATE_INTS, FILLS[fill])
        t_before = t_whole.clone()
        _lib.check(lib.fear_gather_targets(targets.data_ptr(), N, templates.data_ptr(), sel.data_ptr(), M,
                                           step_t.data_ptr(), step_z.data_ptr(), None), "fear_gather_targets")
        torch.cuda.synchronize()
        valid = (rows >= 0) & (rows < N)
        want = np.zeros((M, 16), np.int32)
        want[valid] = targets_np[rows[valid]]
        want[:, 0] = np.where(valid, frames, -1)
        assert np.array_equal(step_t.view(M, 16).cpu().numpy(), want), name
        got_z = step_z.view(M, TEMPLATE_INTS)
        idx = torch.from_numpy(np.where(valid, rows, 0)).cuda()
        want_z = templates.view(N, TEMPLATE_INTS)[idx]
        want_z[torch.from_numpy(~valid).cuda()] = 0
        assert torch.equal(got_z, want_z), name
        for whole in (st_whole, sz_whole):
            assert bool((whole[:GUARD] == FILLS[fill]).all()) and bool((whole[-GUARD:] == FILLS[fill]).all()), name
        assert torch.equal(t_whole, t_before) and torch.equal(z_whole, z_before), name
        assert bool((s_whole[:GUARD] == FILLS[fill]).all()) and bool((s_whole[-GUARD:] == FILLS[fill]).all())
        if not distinct:
            continue
        # scatter random step rows back: only x .. ch of the in-range rows change
        step_np = rng.integers(-2 ** 31, 2 ** 31, (M, 16), dtype=np.int64).astype(np.int32)
        step_t.copy_(torch.from_numpy(step_np.reshape(-1)))
        st_before = st_whole.clone()
        _lib.check(lib.fear_scatter_targets(step_t.data_ptr(), sel.data_ptr(), M, targets.data_ptr(), N, None),
                   "fear_scatter_targets")
        torch.cuda.synchronize()
        targets_np[rows[valid], 1:9] = step_np[valid, 1:9]
        assert np.array_equal(targets.view(N, 16).cpu().numpy(), targets_np), name
        assert bool((t_whole[:GUARD] == FILLS[fill]).all()) and bool((t_whole[-GUARD:] == FILLS[fill]).all())
        assert torch.equal(st_whole, st_before)
        del s_whole, sel, st_whole, step_t, sz_whole, step_z, got_z, want_z


def test_gather_and_scatter_reject_bad_arguments():
    lib = _lib.load()
    t = torch.zeros(16 * TEMPLATE_INTS, dtype=torch.int32, device="cuda")
    p = t.data_ptr()
    good = dict(targets=p, N=4, templates=p, select=p, M=2, step_targets=p, step_templates=p)

    def gather(**kw):
        a = dict(good, **kw)
        return lib.fear_gather_targets(a["targets"], a["N"], a["templates"], a["select"], a["M"], a["step_targets"],
                                       a["step_templates"], None)

    for kw in [dict(targets=None), dict(templates=None), dict(select=None), dict(step_targets=None),
               dict(step_templates=None), dict(N=0), dict(M=0), dict(M=65536), dict(M=-1), dict(templates=p + 4),
               dict(step_templates=p + 8)]:
        assert gather(**kw) == -1, kw
        assert _lib.last_error(), kw
    for args in [(None, p, 2, p, 4), (p, None, 2, p, 4), (p, p, 2, None, 4), (p, p, 0, p, 4), (p, p, 65536, p, 4),
                 (p, p, 2, p, 0)]:
        assert lib.fear_scatter_targets(*args, None) == -1, args
        assert _lib.last_error(), args
    torch.cuda.synchronize()
    assert bool((t == 0).all())  # nothing was launched
