#!/usr/bin/env python
"""Config 3 (BASELINE.json): streaming single-object tracking over the demo clip (tests/golden/test.mp4,
661 frames 480x256, init box [163,53,45,174]) with FEARTracker on one H100; sequentially dependent frames
(batch 1).  Prints one JSON line: frames/s incl. host crop/resize + H2D + kernels + D2H of the box record,
the split between host pre/post-processing and the device call, and agreement with the reference trajectory.

    python tools/bench_stream.py [--repeat 3] [--host-normalize]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import feartracker_b200 as fb  # noqa: E402
from bench import load_state  # noqa: E402


def read_video(path):
    import cv2

    cap, frames = cv2.VideoCapture(path), []
    while True:
        ok, f = cap.read()
        if not ok:
            break
        frames.append(cv2.cvtColor(f, cv2.COLOR_BGR2RGB))
    return frames


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--host-normalize", action="store_true")
    args = ap.parse_args()
    g = np.load(os.path.join(ROOT, "tests", "golden", "video_teacher.npz"))
    frames = read_video(os.path.join(ROOT, "tests", "golden", "test.mp4"))
    net = fb.FEARNet(**fb.FEAR_XS_MODEL_KWARGS)
    net.load_state_dict(load_state(), strict=True)
    net = net.cuda().eval()
    cfg = dict(fb.FEAR_XS_TRACKER_KWARGS, host_normalize=args.host_normalize)
    best, traj = None, None
    for _ in range(args.repeat):
        trk = fb.FEARTracker(net, cuda_id=0, **cfg)
        trk.initialize(frames[0], g["init_bbox"])
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = [trk.update(f)["bbox"] for f in frames[1:]]
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        if best is None or dt < best:
            best, traj = dt, np.array([list(map(int, b)) for b in out])
    same = int((traj == g["trajectory"]).all(1).sum())
    # device-only time of one track call (events), batch 1
    trk = fb.FEARTracker(net, cuda_id=0, **cfg)
    trk.initialize(frames[0], g["init_bbox"])
    crop = trk._preprocess_image(np.ascontiguousarray(frames[1][:256, :256]))
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(10):
        net.track_boxes(crop, trk._template_features)
    a.record()
    for _ in range(100):
        net.track_boxes(crop, trk._template_features)
    b.record()
    torch.cuda.synchronize()
    dev_ms = a.elapsed_time(b) / 100
    n = len(frames) - 1
    print(json.dumps({
        "metric": "FEAR-XS streaming track loop (config 3), frames/s", "value": n / best, "unit": "frames/s",
        "frames": n, "ms_per_frame": best / n * 1e3, "device_call_ms_batch1": dev_ms,
        "host_share": 1.0 - dev_ms / (best / n * 1e3), "identical_boxes": same, "of": n,
        "input": "uint8 crop upload, normalisation in the stem kernel" if not args.host_normalize else
                 "host-normalised fp32 crop upload", "launches_per_frame": 70,
    }))


if __name__ == "__main__":
    main()
