"""The mono entry points and trackers on poisoned memory, in their own process (as tests/poison_check.py, whose guarded
buffers, fills and checker it reuses).  Prints one JSON line.

    python tests/poison_mono_check.py

Kernels: mono frames of three containers (uint8, MSB-aligned 12-bit uint16, MIPI RAW10 whose rows end in a partial
group; tight and pitched rows, with and without gain control) live in guarded allocations whose guard bands and whose
bytes past each row are filled with 0, fill A and fill B in turn.  fear_frame_range_mono writes the lo / hi of a
guarded FearFrameMono table with decoy entries past F; fear_crop_targets_mono_u8, fear_advance_targets_mono and
fear_frame_sums_mono_u8 read that table and write guarded crops, state rows and sums.  Every result must be the same
under every fill and equal aminmax / cv2 / the host rescale / numpy on the grey frames; no guard band, sample byte,
record field or state field the call does not own may change.

Trackers: FEARMultiTracker (graphed and eager) and FEARTracker (plain and smooth) on 16-bit frames with gain control
made from the demo clip, with the net's workspace, the trackers' own buffers and the frames' pitch bytes poisoned
before every call, must give what the same trackers give unpoisoned.
"""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import feartracker_b200 as fb  # noqa: E402
from feartracker_b200 import _lib, image_ops  # noqa: E402
from oracle import fear_oracle as fo  # noqa: E402
from tests.helpers import GOLDEN, golden  # noqa: E402
from tests.poison_check import FILLS, Checker, Guarded, as_i32, make_net, stream  # noqa: E402
from tests.poison_tracker_device_check import poison as poison_single, state as single_state  # noqa: E402

# (H, W), container (kind, bits, shift), agc, pitch bytes past the row
SHAPES = [((255, 480), ("u8", 8, 0), 1, 32), ((91, 334), ("u16", 12, 4), 0, 0),
          ((37, 1005), ("raw10", 10, 0), 1, 11)]
TARGETS = [(0, [163, 53, 45, 174]), (0, [-10, 100, 40, 30]), (0, [450, 200, 60, 90]), (1, [0, 0, 3, 3]),
           (1, [-300, -200, 900, 500]), (2, [990, 20, 30, 30]), (2, [400, 5, 200, 20]), (3, [10, 10, 20, 20])]
N_DECOY_ROWS = 5
MONO_INTS = _lib.MONO_DTYPE.itemsize // 4  # a FearFrameMono as int32 fields; lo and hi are fields 10 and 11


def row_bytes(w, kind):
    return {"u8": w, "u16": 2 * w, "raw10": image_ops.mipi_row_bytes(w, 10)}[kind]


class Surface:
    """One mono frame in a guarded allocation: ``rows`` (H, pitch) bytes, the bytes past each row poisoned by every
    fill and checked never to be written."""

    def __init__(self, codes: np.ndarray, container, agc: int, extra: int, rng):
        kind, bits, shift = container
        h, w = codes.shape
        self.need = row_bytes(w, kind)
        if kind == "raw10":
            rows = image_ops.mipi_pack(codes, 10, self.need + extra)
        else:
            smp = codes.astype(np.uint8) if bits == 8 else \
                ((codes.astype(np.int64) << shift) | rng.integers(0, 1 << shift, codes.shape)).astype("<u2")
            rows = np.zeros((h, self.need + extra), np.uint8)
            rows[:, :self.need] = smp.view(np.uint8).reshape(h, self.need)
        self.rows, self.w, self.container, self.agc = rows, w, container, agc
        self.g = Guarded(rows.size, frame=rows.size, words=False, data=torch.from_numpy(rows.reshape(-1)).cuda())
        c = codes.astype(np.uint8 if bits == 8 else np.uint16)
        self.range = (int(c.min()), int(c.max())) if agc else (2 ** 31 - 1, -2 ** 31)
        self.rgb = image_ops.mono_to_rgb(c, bits, "minmax" if agc else None)

    def record(self):
        kind, bits, shift = self.container
        return (self.g.ptr(), self.rows.shape[1], self.rows.shape[0], self.w, bits, shift, 1 if kind == "raw10" else 0,
                self.agc, 2 ** 31 - 1, -2 ** 31)

    def fill(self, fill):
        self.g.fill(fill)
        self.g.raw.view(self.rows.shape)[:, self.need:] = FILLS[fill][1]

    def ok(self, fill):
        body = self.g.raw.view(self.rows.shape)[:, :self.need]
        return self.g.guards_ok(fill) and bool(torch.equal(body, self.g.data.view(self.rows.shape)[:, :self.need]))


def group_kernels(chk, rng):
    from tests.test_gpu_multi_tracker import _cv2_crop

    lib = _lib.load()
    surfaces = []
    for (h, w), container, agc, extra in SHAPES:
        codes = rng.integers(0, 1 << container[1], (h, w))
        if agc:
            codes = codes % 300 + 21
        surfaces.append(Surface(codes, container, agc, extra, rng))
    F = len(surfaces)
    decoys = [surfaces[0].record()[:6] + (0, 1, 5, 9), surfaces[1].record()[:7] + (1, 0, 1)]  # past F: never read
    table = np.array([s.record() for s in surfaces] + decoys, dtype=_lib.MONO_DTYPE)
    gtable = Guarded.of(torch.from_numpy(table.view(np.int32).reshape(-1, MONO_INTS).copy()), MONO_INTS)
    fills = []

    def on_fill(fill):
        for s in surfaces:
            s.fill(fill)
        fills[:] = [fill]

    def surfaces_ok(tag):
        if not all(s.ok(fills[0]) for s in surfaces):
            chk.fail(f"{tag}: a mono frame or its guard band was written")

    tag = "mono range"
    ranged = chk.run(tag, lambda: _lib.check(lib.fear_frame_range_mono(gtable.ptr(), F, stream()), tag), [], [],
                     owned={gtable: (F, slice(10, 12))}, on_fill=on_fill)[0].cpu().numpy()
    surfaces_ok(tag)
    for i, s in enumerate(surfaces):
        if tuple(ranged[i, 10:12]) != s.range:
            chk.fail(f"{tag} frame {i}: {tuple(ranged[i, 10:12])} is not the frame's range {s.range}")
    # the kernels below read the ranged table, guarded as an input
    gtable = Guarded.of(torch.from_numpy(ranged.copy()), MONO_INTS)
    means = [np.mean(s.rgb, axis=(0, 1)) for s in surfaces]
    targets = [(f if f < F else F, box) for f, box in TARGETS]  # frame F: out of range (a decoy entry sits there)
    N = len(targets)
    recs = np.zeros((N + N_DECOY_ROWS, _lib.TARGET_INTS), dtype=np.int32)
    for i, (f, box) in enumerate(targets + [(k % F, [20 + k, 30, 40, 50]) for k in range(N_DECOY_ROWS)]):
        recs[i, 0], recs[i, 1:5] = f, box
        recs[i, 9:12] = np.clip(np.rint(means[f % F]), 0, 255)
        recs[i, 12:16] = [1000 + i, -7, 12345, i]  # reserved fields: kept
    gstate = Guarded.of(torch.from_numpy(recs), recs.size)
    for size, off in ((256, 2.0), (128, 0.2)):
        gcrops = Guarded.out((N, size, size, 3), torch.uint8, size * size * 3)
        tag = f"mono crop {size} {off}"
        crops, st = chk.run(tag, lambda: _lib.check(lib.fear_crop_targets_mono_u8(
            gtable.ptr(), F, gstate.ptr(), N, off, size, gcrops.ptr(), stream()), tag), [gtable], [gcrops],
            owned={gstate: (N, slice(5, 9))}, on_fill=on_fill)
        surfaces_ok(tag)
        got, ctx = crops.cpu().numpy(), st.cpu().numpy()[:, 5:9]
        for i, (f, box) in enumerate(targets):
            if not np.array_equal(ctx[i], image_ops.context_box(box, off)):
                chk.fail(f"{tag} target {i}: context box")
            want = np.broadcast_to(recs[i, 9:12].astype(np.uint8), got[i].shape) if f == F else \
                _cv2_crop(surfaces[f].rgb, box, size, off, means[f])
            if not np.array_equal(got[i], want):
                chk.fail(f"{tag} target {i} frame {f} {box}: crop differs from cv2")
    nb = 2000
    arecs = np.zeros((nb + N_DECOY_ROWS, _lib.TARGET_INTS), dtype=np.int32)
    arecs[:, 0] = rng.integers(0, F, nb + N_DECOY_ROWS)
    arecs[:, 1:5] = rng.integers(0, 50, (nb + N_DECOY_ROWS, 4))
    arecs[:, 5:7] = rng.integers(-600, 700, (nb + N_DECOY_ROWS, 2))
    arecs[:, 7:9] = rng.integers(1, 2000, (nb + N_DECOY_ROWS, 2))
    arecs[:, 9:16] = rng.integers(-99, 999, (nb + N_DECOY_ROWS, 7))
    arecs[10:15, 0] = F  # out of range: box kept
    boxes = np.zeros(nb, dtype=_lib.BOX_DTYPE)
    boxes["x"], boxes["y"] = rng.uniform(-300, 600, nb), rng.uniform(-300, 600, nb)
    boxes["w"], boxes["h"] = rng.uniform(0, 300, nb), rng.uniform(0, 300, nb)
    gboxes = Guarded.of(torch.from_numpy(boxes.view(np.uint8).copy()), 48)
    gast = Guarded.of(torch.from_numpy(arecs), arecs.size)
    tag = "mono advance"
    st = chk.run(tag, lambda: _lib.check(lib.fear_advance_targets_mono(
        gboxes.ptr(), gtable.ptr(), F, gast.ptr(), nb, 256, stream()), tag), [gtable, gboxes], [],
        owned={gast: (nb, slice(1, 5))}, on_fill=on_fill)[0].cpu().numpy()
    surfaces_ok(tag)
    for i in range(nb):
        if 10 <= i < 15:
            want = arecs[i, 1:5]
        else:
            b = np.array([boxes["x"][i], boxes["y"][i], boxes["w"][i], boxes["h"][i]])
            h, w = SHAPES[arecs[i, 0]][0]
            want = image_ops.clamp_bbox(image_ops.rescale_bbox(b, arecs[i, 5:9], 256), (h, w, 3))
        if not np.array_equal(st[i, 1:5], want):
            chk.fail(f"{tag} target {i}: box differs from the host rescale + clamp")
            break
    gsums = Guarded.out((F, 3), torch.int64, 3)
    tag = "mono frame_sums"
    sums = chk.run(tag, lambda: _lib.check(lib.fear_frame_sums_mono_u8(gtable.ptr(), F, gsums.ptr(), stream()),
                                           tag), [gtable], [gsums], on_fill=on_fill)[0].cpu().numpy().view(np.uint64)
    surfaces_ok(tag)
    for i, s in enumerate(surfaces):
        if not np.array_equal(sums[i], s.rgb.sum(axis=(0, 1), dtype=np.uint64)):
            chk.fail(f"{tag} frame {i}: differs from numpy")


def thermal_codes(clip, T):
    """The demo clip as a thermal core's 16-bit codes: a narrow band 30000 + 8 * luma, plus a fixed pattern."""
    pattern = (np.indices(clip.shape[1:3]).sum(0) % 5).astype(np.uint16)
    return [(30000 + 8 * (f.astype(np.uint32) @ np.array([77, 150, 29]) >> 8) + pattern).astype(np.uint16)
            for f in clip[:T + 1]]


def surface(codes, byte):
    """uint16 codes on the device with 32 more samples of pitch, those samples' bytes set to ``byte``."""
    h, w = codes.shape
    surf = torch.full((h, 2 * (w + 32)), byte, dtype=torch.uint8)
    surf[:, :2 * w] = torch.from_numpy(np.ascontiguousarray(codes).view(np.uint8))
    return fb.MonoFrame(surf.cuda().view(torch.int16).view(torch.uint16)[:, :w], bits=16, agc="minmax")


def group_trackers(chk, res):
    clip = fo.read_video_rgb(os.path.join(GOLDEN, "test.mp4"))
    T = 30
    rows = thermal_codes(clip, T)
    init = golden("video_teacher.npz")["init_bbox"]
    cfg = fb.FEAR_XS_TRACKER_KWARGS
    targets = [[163, 53, 45, 174], [0, 0, 40, 60], [440, 200, 40, 56], [300, 80, 60, 90]]

    def poison_multi(trk, net, fill):
        word, byte = FILLS[fill]
        _lib.check(_lib.load().fear_debug_fill_workspace(net._handle, word, stream()), "fear_debug_fill_workspace")
        b, n = trk._buf, len(trk)
        if b is None:
            return
        b["zf"][n:].view(torch.int32).fill_(as_i32(word))
        b["crops"][n:].fill_(byte)
        b["tcrops"][n:].fill_(byte)
        if b["mono"] is not None:  # rewritten by every call
            b["mono"].fill_(byte)

    def run_multi(eager, poisoned):
        net = make_net(1)
        trk = fb.FEARMultiTracker(net, cuda_id=0, max_targets=8, **(dict(cfg, cuda_graph=False) if eager else cfg))
        outs = []
        for t in range(T + 1):
            fill = "AB"[t % 2]
            frames = [surface(rows[t], FILLS[fill][1] if poisoned else 0) for _ in range(2)]
            if poisoned:
                poison_multi(trk, net, fill)
                chk.calls += 1
            if t == 0:
                trk.add(frames, targets, [0, 1, 1, 0])
            else:
                outs.append(trk.update(frames))
        return outs

    for eager in (False, True):
        want, got = run_multi(eager, False), run_multi(eager, True)
        for t, (a, b) in enumerate(zip(got, want)):
            if not all(np.array_equal(a[k], b[k]) for k in ("ids", "bbox", "score")):
                chk.fail(f"multi-tracker eager={eager} frame {t + 1}: differs from the unpoisoned tracker")
                break
        res[f"multi eager={eager} last boxes"] = want[-1]["bbox"].tolist()

    def run_single(extra, poisoned):
        net = make_net(1)
        trk = fb.FEARTracker(net, cuda_id=0, **dict(cfg, **extra))
        if poisoned:
            trk._device_frame_state()
        out = []
        for t in range(T + 1):
            fill = "AB"[t % 2]
            frame = surface(rows[t], FILLS[fill][1] if poisoned else 0)
            if poisoned:
                poison_single(trk, net, fill)
                chk.calls += 1
            if t == 0:
                trk.initialize(frame, init)
            else:
                trk.update(frame)
            out.append(single_state(trk))
        return out

    for name, extra in (("plain", {}), ("smooth", {"smooth": True})):
        want, got = run_single(extra, False), run_single(extra, True)
        bad = [t for t, (a, b) in enumerate(zip(got, want)) if a != b]
        if bad:
            chk.fail(f"FEARTracker {name}: frame {bad[0]} differs from the unpoisoned run")
        res[f"single {name} last box"] = want[-1][0]


def main():
    torch.manual_seed(0)
    chk, res = Checker(), {}
    group_kernels(chk, np.random.default_rng(29))
    group_trackers(chk, res)
    res.update(chk.report())
    print("POISON_CHECK " + json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
