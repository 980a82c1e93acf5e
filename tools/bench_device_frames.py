#!/usr/bin/env python
"""FEARMultiTracker on 1080p streams, frames given as numpy arrays in host memory or as CUDA tensors already on the
device.  The demo clip (tests/golden/test.mp4, 480x256) is resized to 1920x1080 with cv2.resize; stream s starts at clip
frame 20 * s and cycles through --clip-frames frames kept in memory (host for the numpy arm, device for the CUDA arm).
Each stream holds the jittered golden boxes of bench_multi.py, scaled to 1080p.  For F streams x k targets per stream,
each arm reports:
  host_ms_per_update   wall time of one update() (numpy: pack + upload; both: table upload, graph replay, read-back)
  target_frames_per_s  N / host_ms_per_update
  device_ms_per_step   CUDA events around replays of the captured step
  add_ms               wall time of adding all N targets (initialize: frame sums, template crops and features)
Both arms run in the same process on the same targets, alternated in blocks of --block updates.  One JSON line, with
the card name, power limit and SM clock read by nvidia-smi right after the timed runs.

    python tools/bench_device_frames.py [--streams 1,4,8] [--targets 4,32] [--updates 300] [--block 50]
"""
import argparse
import json
import os
import sys
import time

import cv2
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import feartracker_b200 as fb  # noqa: E402
from bench import load_state  # noqa: E402
from bench_multi import card_info, jittered_boxes  # noqa: E402
from oracle.fear_oracle import read_video_rgb  # noqa: E402

W, H = 1920, 1080
WARMUP = 3  # eager warm-up + capture + one replay
ADD_REPEATS = 5


def make_streams(clip, num_streams, clip_frames):
    """Per stream, a (clip_frames, 1080, 1920, 3) uint8 array of resized clip frames starting at frame 20 * s."""
    out = []
    for s in range(num_streams):
        arr = np.empty((clip_frames, H, W, 3), np.uint8)
        for i in range(clip_frames):
            arr[i] = cv2.resize(clip[(20 * s + i) % len(clip)], (W, H))
        out.append(arr)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", default="1,4,8")
    ap.add_argument("--targets", default="4,32", help="targets per stream")
    ap.add_argument("--updates", type=int, default=300, help="timed updates per arm")
    ap.add_argument("--block", type=int, default=50, help="updates per arm before switching to the other arm")
    ap.add_argument("--clip-frames", type=int, default=40, help="1080p frames per stream kept in memory")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_device_frames.py measures on a CUDA device; none is available")
    clip = read_video_rgb(os.path.join(ROOT, "tests", "golden", "test.mp4"))
    stream_counts = [int(s) for s in args.streams.split(",")]
    host = make_streams(clip, max(stream_counts), args.clip_frames)
    dev = [torch.from_numpy(a).cuda() for a in host]
    torch.cuda.synchronize()
    net = fb.FEARNet(**fb.FEAR_XS_MODEL_KWARGS)
    net.load_state_dict(load_state(), strict=True)
    net = net.cuda().eval()
    cfg = fb.FEAR_XS_TRACKER_KWARGS
    scale = np.array([W / 480, H / 256, W / 480, H / 256])
    T = args.clip_frames

    def frames(arm, F, i):
        src = host if arm == "numpy" else dev
        return [src[s][i % T] for s in range(F)]

    results = []
    for F in stream_counts:
        for k in (int(t) for t in args.targets.split(",")):
            n = F * k
            rects = np.concatenate([np.rint(jittered_boxes(k, seed=s) * scale) for s in range(F)])
            streams = np.repeat(np.arange(F), k)
            arms = {a: fb.FEARMultiTracker(net, cuda_id=0, max_targets=n, **cfg) for a in ("numpy", "cuda")}
            row = {"streams": F, "targets_per_stream": k, "N": n}
            for arm, trk in arms.items():
                trk.initialize(frames(arm, F, 0), rects, streams)  # warm-up
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(ADD_REPEATS):
                    trk.initialize(frames(arm, F, 0), rects, streams)
                row[arm] = {"add_ms": (time.perf_counter() - t0) * 1e3 / ADD_REPEATS}
                for i in range(1, 1 + WARMUP):
                    trk.update(frames(arm, F, i))
            spent = {a: 0.0 for a in arms}
            done = {a: 0 for a in arms}
            pos = {a: 1 + WARMUP for a in arms}
            order = list(arms)
            while min(done.values()) < args.updates:
                for arm in order:
                    m = min(args.block, args.updates - done[arm])
                    batch = [frames(arm, F, pos[arm] + j) for j in range(m)]
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    for fr in batch:
                        arms[arm].update(fr)
                    spent[arm] += time.perf_counter() - t0
                    done[arm] += m
                    pos[arm] += m
                order.reverse()
            for arm, trk in arms.items():
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(50):
                    trk._graph.replay()
                b.record()
                torch.cuda.synchronize()
                host_ms = spent[arm] * 1e3 / done[arm]
                row[arm].update(host_ms_per_update=host_ms, target_frames_per_s=n * 1e3 / host_ms,
                                device_ms_per_step=a.elapsed_time(b) / 50)
            results.append(row)
            del arms
    print(json.dumps({"metric": "FEARMultiTracker on 1920x1080 streams: numpy frames from host memory vs CUDA frames "
                                "already on the device",
                      "card": card_info(torch.cuda.current_device()), "timed_updates_per_arm": args.updates,
                      "results": results}))


if __name__ == "__main__":
    main()
