"""FEARTracker on device frames with poisoned memory, in its own process (as tests/poison_check.py, whose fills it
reuses).  Prints one JSON line.

    python tests/poison_tracker_device_check.py

Each run tracks the first frames of the demo clip from the reference's initial box, on frames that live inside larger
surfaces: an RGBA surface's RGB view, a region of interest inside a larger canvas, a pitched NV12 surface and a pitched
YUV 4:4:4 surface, with ``smooth`` off and on, graphed and eager.  The clean run fills every byte outside the frames
(alpha, row-pitch gaps, the canvas border) with 0 and poisons nothing.  The poisoned run fills those bytes with 0xA5 /
0x5A (alternating per frame), and before every call fills the net's workspace (fear_debug_fill_workspace) and the
tracker's own device buffers (crops, sums, box records, the per-call inputs) with fill A or B.  Both runs must give
the same boxes and the same tracking_state on every frame.
"""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import feartracker_b200 as fb  # noqa: E402
from feartracker_b200 import _lib  # noqa: E402
from feartracker_b200.tracker import _DEVICE_INPUT_BYTES  # noqa: E402
from oracle import fear_oracle as fo  # noqa: E402
from tests.helpers import GOLDEN, golden  # noqa: E402
from tests.poison_check import FILLS, Checker, as_i32, make_net, stream  # noqa: E402

T = 40


def rgba(f, byte):
    t = torch.full(f.shape[:2] + (4,), byte, dtype=torch.uint8)
    t[..., :3] = torch.from_numpy(f)
    return t.cuda()[..., :3]


def roi(f, byte):
    h, w = f.shape[:2]
    canvas = torch.full((h + 40, w + 64, 3), byte, dtype=torch.uint8)
    canvas[17:17 + h, 29:29 + w] = torch.from_numpy(f)
    return canvas.cuda()[17:17 + h, 29:29 + w]


def nv12(f, byte):
    import cv2

    h, w = f.shape[:2]
    i420 = cv2.cvtColor(f, cv2.COLOR_RGB2YUV_I420).reshape(-1)
    q = h * w // 4
    surf = torch.full((h + h // 2, w + 32), byte, dtype=torch.uint8)
    surf[:h, :w] = torch.from_numpy(i420[:h * w].reshape(h, w))
    uv = np.stack([i420[h * w:h * w + q].reshape(h // 2, w // 2), i420[h * w + q:].reshape(h // 2, w // 2)], -1)
    surf[h:, :w] = torch.from_numpy(uv.reshape(h // 2, w))
    return fb.YUV420Frame.nv12(surf.cuda()[:, :w])


def i444(f, byte):
    h, w = f.shape[:2]
    surf = torch.full((3 * h, w + 48), byte, dtype=torch.uint8)
    for k in range(3):  # any planes will do: both runs read the same ones
        surf[k * h:(k + 1) * h, :w] = torch.from_numpy(np.ascontiguousarray(f[..., k]))
    return fb.YUV444Frame.i444(surf.cuda()[:, :w], matrix="bt709", full_range=True)


KINDS = {"rgba": rgba, "roi": roi, "nv12": nv12, "i444": i444}


def poison(trk, net, fill):
    word, byte = FILLS[fill]
    _lib.check(_lib.load().fear_debug_fill_workspace(net._handle, word, stream()), "fear_debug_fill_workspace")
    st = getattr(trk, "_device_state", None)
    if st is None:
        return
    for key in ("crop", "tcrop", "smooth_boxes"):
        st[key].fill_(byte)
    st["sums"].view(torch.int32).fill_(as_i32(word))
    st["dev_in"][:_DEVICE_INPUT_BYTES].fill_(byte)  # rewritten by every call; the window after it is not
    if st["boxes"] is not None:
        st["boxes"].fill_(byte)


def state(trk):
    s = trk.tracking_state
    return (np.asarray(s.bbox).tolist(), np.asarray(s.mapping).tolist(), np.asarray(s.prev_size).tolist(),
            s.mean_color.tobytes(), [list(map(int, p)) for p in s.paths])


def run(clip, init, kind, extra, poisoned, chk):
    net = make_net(1)
    trk = fb.FEARTracker(net, cuda_id=0, **dict(fb.FEAR_XS_TRACKER_KWARGS, **extra))
    if poisoned:
        trk._device_frame_state()  # allocate the tracker's buffers now, so that initialize finds them poisoned
    out = []
    for t in range(T + 1):
        fill = "AB"[t % 2]
        frame = KINDS[kind](clip[t], FILLS[fill][1] if poisoned else 0)
        if poisoned:
            poison(trk, net, fill)
            chk.calls += 1
        if t == 0:
            trk.initialize(frame, init)
        else:
            trk.update(frame)
        out.append(state(trk))
    return out


def main():
    torch.manual_seed(0)
    chk = Checker()
    clip = fo.read_video_rgb(os.path.join(GOLDEN, "test.mp4"))
    init = golden("video_teacher.npz")["init_bbox"]
    res = {"frames": T}
    for kind in KINDS:
        for name, extra in (("plain", {}), ("smooth", {"smooth": True}), ("eager", {"cuda_graph": False}),
                            ("eager smooth", {"cuda_graph": False, "smooth": True})):
            want = run(clip, init, kind, extra, False, chk)
            got = run(clip, init, kind, extra, True, chk)
            bad = [t for t, (a, b) in enumerate(zip(got, want)) if a != b]
            if bad:
                chk.fail(f"{kind} {name}: frame {bad[0]} differs from the unpoisoned run: {got[bad[0]]} vs "
                         f"{want[bad[0]]}")
            res[f"{kind} {name} last box"] = want[-1][0]
    res.update(chk.report())
    print("POISON_CHECK " + json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
