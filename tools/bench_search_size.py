#!/usr/bin/env python
"""Search crop side S (instance_size; score_size = S / 16) against throughput.  For each S in --sizes:
  track_boxes_fps           FEARNet.track_boxes on B = --batch uint8 (B, S, S, 3) crops: frames per second from CUDA
                            events around --steps calls, after --warmup calls
  launches_per_step         kernel launches of one track_boxes call (fear_launch_count)
  multi_device_ms_per_step  FEARMultiTracker on 1080p uint8 RGB frames in device memory, --streams streams x --targets
                            targets each: CUDA events around --step-repeats replays of the captured step (crop of
                            every target, network, decode, box update)
The sizes are alternated in --rounds rounds over one FEARNet and one tracker per size, so slow drift on the card affects
every size alike; each figure is the median over rounds.  One JSON line, with the card name, power limit and SM clock
read by nvidia-smi after the timed runs.

    python tools/bench_search_size.py [--sizes 128,160,192,224,256] [--batch 256] [--rounds 3]
"""
import argparse
import json
import os
import sys

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

H, W = 1080, 1920


def timed(fn, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="128,160,192,224,256")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--streams", type=int, default=8)
    ap.add_argument("--targets", type=int, default=32)
    ap.add_argument("--step-repeats", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_search_size needs a CUDA device")
    sizes = [int(s) for s in args.sizes.split(",")]
    net = fb.FEARNet(**fb.FEAR_XS_MODEL_KWARGS)
    net.load_state_dict(load_state(), strict=True)
    net = net.cuda().eval()
    n_targets = args.streams * args.targets
    net.reserve(max(args.batch, n_targets))
    g = torch.Generator().manual_seed(0)
    zf = net.get_features(torch.randint(0, 256, (1, 128, 128, 3), generator=g, dtype=torch.uint8).cuda())
    crops = {s: torch.randint(0, 256, (args.batch, s, s, 3), generator=g, dtype=torch.uint8).cuda() for s in sizes}

    clip = read_video_rgb(os.path.join(ROOT, "tests", "golden", "test.mp4"))
    frames = [torch.from_numpy(cv2.resize(clip[(5 * i) % len(clip)], (W, H))).cuda() for i in range(args.streams)]
    boxes = jittered_boxes(args.targets) * (W / clip.shape[2])
    rects = np.concatenate([boxes for _ in range(args.streams)])
    streams = np.repeat(np.arange(args.streams), args.targets)
    trackers = {}
    for s in sizes:
        cfg = dict(fb.FEAR_XS_TRACKER_KWARGS, instance_size=s, score_size=s // 16)
        trk = fb.FEARMultiTracker(net, cuda_id=0, max_targets=n_targets, **cfg)
        trk.add(frames, rects, streams)
        for _ in range(3):  # eager warm-up, capture, one replay
            trk.update(frames)
        trackers[s] = trk

    res = {s: {"fps": [], "multi_ms": []} for s in sizes}
    for _ in range(args.rounds):
        for s in sizes:
            x = crops[s]
            for _ in range(args.warmup):
                net.track_boxes(x, zf)
            n0 = net.launch_count()
            net.track_boxes(x, zf)
            res[s]["launches"] = net.launch_count() - n0
            ms = timed(lambda: net.track_boxes(x, zf), args.steps)
            res[s]["fps"].append(args.batch / ms * 1e3)
            trk = trackers[s]
            trk.update(frames)  # the graph of this tracker is current: replay it
            assert trk._graph is not None, "the multi-tracker step was not captured"
            res[s]["multi_ms"].append(timed(trk._graph.replay, args.step_repeats))
    torch.cuda.synchronize()
    out = {"metric": "search_size", "batch": args.batch, "streams": args.streams, "targets_per_stream": args.targets,
           "frame": f"{W}x{H}", "rounds": args.rounds, "card": card_info(torch.cuda.current_device()),
           "sizes": {str(s): {"score_side": s // 16, "track_boxes_fps": float(np.median(r["fps"])),
                              "launches_per_step": r["launches"],
                              "multi_device_ms_per_step": float(np.median(r["multi_ms"])),
                              "fps_rounds": [round(v, 1) for v in r["fps"]],
                              "multi_ms_rounds": [round(v, 4) for v in r["multi_ms"]]} for s, r in res.items()}}
    line = json.dumps(out)
    print(line, flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
