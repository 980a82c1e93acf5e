#!/usr/bin/env python
"""FEARTracker (one target) on frames in host memory against frames already in GPU memory, at 1920x1080 (the demo clip,
tests/golden/test.mp4, resized with cv2.resize) and at the clip's native 480x256.  Arms, each with smooth off and on:
  numpy_gpu_crop   FEARTracker(gpu_crop=True) fed numpy frames: the frame is uploaded every update, then crop,
                   network and decode replay as one CUDA graph
  cuda_rgb         the same frames as uint8 (H, W, 3) CUDA tensors, read in place by fear_crop_targets_view_u8
  nv12             the same frames as pitched NV12 surfaces on the device (cv2's I420 conversion, 2048-byte pitch at
                   1080p, 512 at 480x256), YUV420Frame.nv12, converted inside fear_crop_targets_ycbcr_u8
Each arm tracks --clip-frames frames kept in memory from the reference's initial box (scaled), one update per frame,
re-initialised (untimed) when they run out; the arms alternate in blocks of --block updates.  Per arm:
  host_ms_per_update   wall time of one update() (each ends in a synchronise)
  frames_per_s         1000 / host_ms_per_update
  device_ms_per_step   CUDA events around --step-repeats replays of the arm's captured graph alone
One JSON line, with the card name, power limit and SM clock read by nvidia-smi right after the timed runs.

    python tools/bench_tracker_device_frames.py [--updates 600] [--block 50] [--clip-frames 120]
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
from bench_multi import card_info  # noqa: E402
from oracle.fear_oracle import read_video_rgb  # noqa: E402

INIT = np.array([163, 53, 45, 174])  # the reference's initial box on frame 0 of the demo clip (480x256)
WARMUP = 3  # eager warm-up + capture + one replay
SIZES = {"1920x1080": (1920, 1080), "480x256": (480, 256)}


def nv12_surface(rgb, pitch):
    h, w = rgb.shape[:2]
    i420 = cv2.cvtColor(rgb, cv2.COLOR_RGB2YUV_I420).reshape(-1)
    q = h * w // 4
    surf = np.zeros((h + h // 2, pitch), np.uint8)
    surf[:h, :w] = i420[:h * w].reshape(h, w)
    surf[h:, :w:2] = i420[h * w:h * w + q].reshape(h // 2, w // 2)
    surf[h:, 1:w:2] = i420[h * w + q:].reshape(h // 2, w // 2)
    return surf


class Arm:
    def __init__(self, net, frames, init, extra):
        self.trk = fb.FEARTracker(net, cuda_id=0, **dict(fb.FEAR_XS_TRACKER_KWARGS, **extra))
        self.frames, self.init, self.t = frames, init, 0
        self.restart()

    def restart(self):
        self.trk.initialize(self.frames[0], self.init)
        self.t = 1

    def update(self):
        if self.t == len(self.frames):
            torch.cuda.synchronize()
            self.restart()
        self.trk.update(self.frames[self.t])
        self.t += 1

    def graph(self):
        st = getattr(self.trk, "_device_state", None) or getattr(self.trk, "_gpu_crop_state", None)
        return st["graph"]


def measure(net, host, init, args):
    w = host.shape[2]
    pitch = 2048 if w > 512 else 512
    cuda = torch.from_numpy(host).cuda()
    surfaces = torch.from_numpy(np.stack([nv12_surface(f, pitch) for f in host])).cuda()
    kinds = {"numpy_gpu_crop": list(host), "cuda_rgb": list(cuda),
             "nv12": [fb.YUV420Frame.nv12(s[:, :w]) for s in surfaces]}
    arms = {}
    for smooth in (False, True):
        for kind, frames in kinds.items():
            name = kind + ("_smooth" if smooth else "")
            arms[name] = Arm(net, frames, init, dict(gpu_crop=True, smooth=True) if smooth else dict(gpu_crop=True))
    for arm in arms.values():
        for _ in range(WARMUP):
            arm.update()
    spent, done, order = {a: 0.0 for a in arms}, {a: 0 for a in arms}, list(arms)
    while min(done.values()) < args.updates:
        for name in order:
            arm, m = arms[name], min(args.block, args.updates - done[name])
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(m):
                arm.update()
            spent[name] += time.perf_counter() - t0
            done[name] += m
        order.reverse()
    results = {}
    for name, arm in arms.items():
        host_ms = spent[name] * 1e3 / done[name]
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        graph = arm.graph()
        a.record()
        for _ in range(args.step_repeats):
            graph.replay()
        b.record()
        torch.cuda.synchronize()
        results[name] = dict(host_ms_per_update=host_ms, frames_per_s=1e3 / host_ms,
                             device_ms_per_step=a.elapsed_time(b) / args.step_repeats)
    return results


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--updates", type=int, default=600, help="timed updates per arm")
    ap.add_argument("--block", type=int, default=50, help="updates per arm before switching to the next arm")
    ap.add_argument("--clip-frames", type=int, default=120, help="clip frames kept in memory per arm")
    ap.add_argument("--step-repeats", type=int, default=200, help="graph replays timed with CUDA events")
    ap.add_argument("--sizes", default=",".join(SIZES))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tracker_device_frames.py measures on a CUDA device; none is available")
    clip = read_video_rgb(os.path.join(ROOT, "tests", "golden", "test.mp4"))[:args.clip_frames]
    net = fb.FEARNet(**fb.FEAR_XS_MODEL_KWARGS)
    net.load_state_dict(load_state(), strict=True)
    net = net.cuda().eval()
    results = {}
    for size in args.sizes.split(","):
        w, h = SIZES[size]
        host = np.stack([f if (w, h) == (480, 256) else cv2.resize(f, (w, h)) for f in clip])
        init = np.rint(INIT * np.array([w / 480, h / 256, w / 480, h / 256])).astype(np.int64)
        results[size] = measure(net, host, init, args)
        torch.cuda.empty_cache()
    print(json.dumps({"metric": "FEARTracker, one target: numpy frames (gpu_crop) vs CUDA RGB tensors vs NV12 surfaces "
                                "on the device, smooth off and on",
                      "card": card_info(torch.cuda.current_device()), "timed_updates_per_arm": args.updates,
                      "results": results}))


if __name__ == "__main__":
    main()
