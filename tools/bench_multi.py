#!/usr/bin/env python
"""Multi-target tracking throughput: FEARMultiTracker on the demo clip (tests/golden/test.mp4, 480x256) with N targets
initialised from a seeded jitter of the golden box [163,53,45,174], one batched step per frame.  Prints one JSON line
with, per N:
  host_ms_per_update   wall time of one update() (frame upload, graph replay, box read-back, synchronisation)
  target_frames_per_s  N / host_ms_per_update
  device_ms_per_step   CUDA events around replays of the captured step (crop + network + decode + advance)
  launches_per_step    kernel launches of one step
  sequential           for N <= 16, the same targets as N FEARTracker(gpu_crop=True) stepped one after another
and the card name, power limit and SM clock read with nvidia-smi right after the timed runs.

    python tools/bench_multi.py [--sizes 1,4,16,64,256] [--frames 600] [--seq-frames 200]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import feartracker_b200 as fb  # noqa: E402
from bench import load_state  # noqa: E402
from oracle.fear_oracle import read_video_rgb  # noqa: E402

GOLDEN_BOX = np.array([163, 53, 45, 174], dtype=np.float64)
WARMUP = 3  # eager warm-up + capture + one replay


def jittered_boxes(n, seed=0):
    rng = np.random.default_rng(seed)
    out = np.tile(GOLDEN_BOX, (n, 1))
    out[1:, :2] += rng.uniform(-40, 40, (n - 1, 2))
    out[1:, 2:] *= rng.uniform(0.7, 1.3, (n - 1, 2))
    return np.rint(out)


def card_info(index):
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        line = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", str(index)],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        return None
    return dict(zip(q.split(","), (c.strip() for c in line.split(",")))) if line else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,4,16,64,256")
    ap.add_argument("--frames", type=int, default=600, help="timed updates per N")
    ap.add_argument("--seq-frames", type=int, default=200, help="timed frames of the sequential comparison")
    args = ap.parse_args()
    frames = read_video_rgb(os.path.join(ROOT, "tests", "golden", "test.mp4"))
    timed = frames[1 + WARMUP:1 + WARMUP + args.frames]
    net = fb.FEARNet(**fb.FEAR_XS_MODEL_KWARGS)
    net.load_state_dict(load_state(), strict=True)
    net = net.cuda().eval()
    cfg = fb.FEAR_XS_TRACKER_KWARGS
    results = []
    for n in (int(s) for s in args.sizes.split(",")):
        rects = jittered_boxes(n)
        trk = fb.FEARMultiTracker(net, cuda_id=0, max_targets=n, **cfg)
        trk.initialize(frames[0], rects)
        for f in frames[1:1 + WARMUP]:
            trk.update(f)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for f in timed:
            trk.update(f)
        host_ms = (time.perf_counter() - t0) * 1e3 / len(timed)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(50):
            trk._graph.replay()
        b.record()
        torch.cuda.synchronize()
        l0 = net.launch_count()  # one eager step: the network's launches (counted by the library) + crop + advance
        trk._step(n, 1, torch.device("cuda", torch.cuda.current_device()))
        torch.cuda.synchronize()
        row = {"N": n, "host_ms_per_update": host_ms, "target_frames_per_s": n * 1e3 / host_ms,
               "device_ms_per_step": a.elapsed_time(b) / 50, "launches_per_step": net.launch_count() - l0 + 2}
        if n <= 16:
            seq = [fb.FEARTracker(net, cuda_id=0, gpu_crop=True, **cfg) for _ in range(n)]
            for t, r in zip(seq, rects):
                t.initialize(frames[0], r)
            for f in frames[1:1 + WARMUP]:
                for t in seq:
                    t.update(f)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for f in timed[:args.seq_frames]:
                for t in seq:
                    t.update(f)
            seq_ms = (time.perf_counter() - t0) * 1e3 / len(timed[:args.seq_frames])
            row["sequential"] = {"host_ms_per_frame": seq_ms, "target_frames_per_s": n * 1e3 / seq_ms}
        results.append(row)
    print(json.dumps({"metric": "FEARMultiTracker target-frames/s on the demo clip (one batched step per frame)",
                      "card": card_info(torch.cuda.current_device()), "timed_updates": len(timed),
                      "results": results}))


if __name__ == "__main__":
    main()
