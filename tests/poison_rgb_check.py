"""The RGB-frame entry points and trackers on poisoned memory, in their own process (as tests/poison_check.py, whose
guarded buffers, fills and checker it reuses).  Prints one JSON line.

    python tests/poison_rgb_check.py

Kernels: RGB frames of four containers (pitched 8-bit BGRA, rgb48le, x2rgb10le words, 12-bit planar RGB) live in guarded
allocations whose guard bands and whose bytes past each row are filled with 0, fill A and fill B in turn.
fear_crop_targets_rgb_u8, fear_advance_targets_rgb and fear_frame_sums_rgb_u8 read a guarded FearFrameRGB table with
decoy entries past F and write guarded crops, state rows and sums.  Every result must be the same under every fill and
equal cv2 / the host rescale / numpy on the RGB frames; no guard band, sample byte, record or state field the call does
not own may change.

Trackers: FEARMultiTracker (graphed and eager) and FEARTracker (plain and smooth) on BGRA and x2rgb10le frames made from
the demo clip, with the net's workspace, the trackers' own buffers and the frames' pitch bytes poisoned before every
call, must give what the same trackers give unpoisoned.
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
from tests.test_gpu_rgb_formats import layout_data  # noqa: E402

# (H, W), layout, bits, pitch bytes past the row (a multiple of the sample size)
SHAPES = [((255, 480), "bgra", 8, 32), ((91, 334), "rgb48le", 16, 0), ((37, 1005), "x2rgb10le", 10, 12),
          ((64, 203), "planar", 12, 6)]
TARGETS = [(0, [163, 53, 45, 174]), (0, [-10, 100, 40, 30]), (0, [450, 200, 60, 90]), (1, [0, 0, 3, 3]),
           (1, [-300, -200, 900, 500]), (2, [990, 20, 30, 30]), (2, [400, 5, 200, 20]), (3, [100, 10, 80, 40]),
           (4, [10, 10, 20, 20])]
N_DECOY_ROWS = 5
RGB_INTS = _lib.RGB_DTYPE.itemsize // 4


class Surface:
    """One RGB frame in a guarded allocation: ``rows`` (rows, pitch) bytes (three planes' rows one after another for a
    planar frame), the bytes past each row poisoned by every fill and checked never to be written."""

    def __init__(self, codes: np.ndarray, layout: str, bits: int, extra: int, rng):
        data = layout_data(codes, layout, bits, rng)
        self.rgb = image_ops.rgb_frame_to_rgb(data, layout, bits)
        self.h, self.w = codes.shape[:2]
        planes = np.ascontiguousarray(data.reshape(-1, self.w) if layout == "planar" else data.reshape(self.h, -1))
        body = planes.view(np.uint8)
        self.need = body.shape[1]
        rows = np.zeros((body.shape[0], self.need + extra), np.uint8)
        rows[:, :self.need] = body
        self.rows, self.layout, self.bits, self.es = rows, layout, bits, data.dtype.itemsize
        self.g = Guarded(rows.size, frame=rows.size, words=False, data=torch.from_numpy(rows.reshape(-1)).cuda())

    def record(self):
        p, pitch, h, w = self.g.ptr(), self.rows.shape[1], self.h, self.w
        if self.layout == "planar":
            return (p, p + h * pitch, p + 2 * h * pitch, pitch, self.es, h, w, self.es, self.bits, 0, 0, 0, 0)
        if self.layout in image_ops.X2RGB10_LAYOUTS:
            return (p, p, p, pitch, 4, h, w, 4, 10, *image_ops.X2RGB10_LAYOUTS[self.layout], 0)
        _, n, idx = image_ops.RGB_PACKED_LAYOUTS[self.layout]
        es = self.es
        return (p + idx[0] * es, p + idx[1] * es, p + idx[2] * es, pitch, n * es, h, w, es, 8 * es, 0, 0, 0, 0)

    def fill(self, fill):
        self.g.fill(fill)
        self.g.raw.view(self.rows.shape)[:, self.need:] = FILLS[fill][1]

    def ok(self, fill):
        body = self.g.raw.view(self.rows.shape)[:, :self.need]
        return self.g.guards_ok(fill) and bool(torch.equal(body, self.g.data.view(self.rows.shape)[:, :self.need]))


def group_kernels(chk, rng):
    from tests.test_gpu_multi_tracker import _cv2_crop

    lib = _lib.load()
    surfaces = [Surface(rng.integers(0, 1 << bits, (h, w, 3)).astype(np.uint8 if bits == 8 else np.uint16), layout,
                        bits, extra, rng) for (h, w), layout, bits, extra in SHAPES]
    F = len(surfaces)
    r0, r2 = surfaces[0].record(), surfaces[2].record()
    decoys = [r0[:7] + (2, 10, 0, 0, 0, 0), r2[:9] + (0, 0, 0, 0)]  # past F: never read
    table = np.array([s.record() for s in surfaces] + decoys, dtype=_lib.RGB_DTYPE)
    gtable = Guarded.of(torch.from_numpy(table.view(np.int32).reshape(-1, RGB_INTS).copy()), RGB_INTS)
    fills = []

    def on_fill(fill):
        for s in surfaces:
            s.fill(fill)
        fills[:] = [fill]

    def surfaces_ok(tag):
        if not all(s.ok(fills[0]) for s in surfaces):
            chk.fail(f"{tag}: an RGB frame or its guard band was written")

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
        tag = f"rgb crop {size} {off}"
        crops, st = chk.run(tag, lambda: _lib.check(lib.fear_crop_targets_rgb_u8(
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
    tag = "rgb advance"
    st = chk.run(tag, lambda: _lib.check(lib.fear_advance_targets_rgb(
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
    tag = "rgb frame_sums"
    sums = chk.run(tag, lambda: _lib.check(lib.fear_frame_sums_rgb_u8(gtable.ptr(), F, gsums.ptr(), stream()),
                                           tag), [gtable], [gsums], on_fill=on_fill)[0].cpu().numpy().view(np.uint64)
    surfaces_ok(tag)
    for i, s in enumerate(surfaces):
        if not np.array_equal(sums[i], s.rgb.sum(axis=(0, 1), dtype=np.uint64)):
            chk.fail(f"{tag} frame {i}: differs from numpy")


def bgra(rgb, byte):
    """An RGB frame as BGRA on the device, alpha and 16 pixels of pitch set to ``byte``."""
    h, w, _ = rgb.shape
    surf = torch.full((h, w + 16, 4), byte, dtype=torch.uint8)
    surf[:, :w, :3] = torch.from_numpy(np.ascontiguousarray(rgb[..., ::-1]))
    return fb.RGBFrame(surf.cuda()[:, :w], "bgra")


def x2rgb10(rgb, byte):
    """An RGB frame as x2rgb10le words on the device (spare bits and 8 words of pitch from ``byte``)."""
    h, w, _ = rgb.shape
    codes = (rgb.astype(np.int64) * 1023 + 127) // 255
    words = image_ops.x2rgb10_pack(codes, "x2rgb10le", np.full((h, w), byte & 3))
    surf = np.full((h, w + 8), np.uint32(byte * 0x01010101), np.uint32)
    surf[:, :w] = words
    return fb.RGBFrame(torch.from_numpy(surf.view(np.int32)).cuda()[:, :w], "x2rgb10le")


def group_trackers(chk, res):
    clip = fo.read_video_rgb(os.path.join(GOLDEN, "test.mp4"))
    T = 30
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
        if b["rgb"] is not None:  # rewritten by every call
            b["rgb"].fill_(byte)

    def run_multi(eager, poisoned):
        net = make_net(1)
        trk = fb.FEARMultiTracker(net, cuda_id=0, max_targets=8, **(dict(cfg, cuda_graph=False) if eager else cfg))
        outs = []
        for t in range(T + 1):
            fill = "AB"[t % 2]
            byte = FILLS[fill][1] if poisoned else 0
            frames = [bgra(clip[t], byte), x2rgb10(clip[t], byte)]
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
            frame = (bgra if t % 3 else x2rgb10)(clip[t], FILLS[fill][1] if poisoned else 0)
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
