#!/usr/bin/env python
"""FEARTracker with ``smooth: true`` (scale / ratio penalty, window, size smoothing) on the demo clip
(tests/golden/test.mp4, 480x256), three arms in one process on the same frames:
  host_smooth      FEARTracker(smooth=True): host crop, eager net.track, maps copied back, numpy post-processing
  gpu_crop         FEARTracker(gpu_crop=True): crop, network and plain decode as one graph replay
  gpu_crop_smooth  FEARTracker(gpu_crop=True, smooth=True): crop, network and fear_decode_smooth as one graph replay
Each arm tracks the clip from the reference's initial box, one update per frame, re-initialised (untimed) when the
clip ends; the arms alternate in blocks of --block updates.  Per arm:
  host_ms_per_update     wall time of one update() (each ends in a synchronise)
  frames_per_s           1000 / host_ms_per_update
  device_ms_per_update   CUDA events around --step-repeats update() calls; it includes the device's idle gaps
  device_ms_per_step     gpu_crop arms: CUDA events around --step-repeats replays of the captured graph alone
Then the kernel time of fear_decode_smooth (and of fear_decode, for scale) at B = 1 and 256: CUDA events around
--kernel-launches back-to-back launches.  One JSON line, with the card name, power limit and SM clock read by
nvidia-smi right after the timed runs.

    python tools/bench_smooth.py [--updates 600] [--block 50]
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
sys.path.insert(0, os.path.join(ROOT, "tools"))
import feartracker_b200 as fb  # noqa: E402
from bench import load_state  # noqa: E402
from bench_multi import card_info  # noqa: E402
from feartracker_b200 import _lib  # noqa: E402
from oracle.fear_oracle import read_video_rgb  # noqa: E402

INIT = np.array([163, 53, 45, 174])  # the reference's initial box on frame 0 of the demo clip
WARMUP = 3  # eager warm-up + capture + one replay
ARMS = {"host_smooth": dict(smooth=True), "gpu_crop": dict(gpu_crop=True), "gpu_crop_smooth": dict(gpu_crop=True, smooth=True)}


class Arm:
    def __init__(self, net, clip, extra):
        self.trk = fb.FEARTracker(net, cuda_id=0, **dict(fb.FEAR_XS_TRACKER_KWARGS, **extra))
        self.clip, self.t = clip, 0
        self.restart()

    def restart(self):
        self.trk.initialize(self.clip[0], INIT)
        self.t = 1

    def update(self):
        if self.t == len(self.clip):
            torch.cuda.synchronize()
            self.restart()
        self.trk.update(self.clip[self.t])
        self.t += 1


def time_kernel(entry, args, launches):
    for _ in range(10):
        entry(*args)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(launches):
        entry(*args)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / launches


def kernel_times(launches):
    lib, s = _lib.load(), torch.cuda.current_stream().cuda_stream
    g = torch.Generator().manual_seed(1)
    params = torch.cat([torch.tensor([0.062, 0.38, 0.765], dtype=torch.float64),
                        torch.from_numpy(np.outer(np.hanning(16), np.hanning(16)).reshape(256))]).cuda()
    out = {}
    for B in (1, 256):
        reg = (10 + 60 * torch.rand(B, 4, 16, 16, generator=g)).cuda()
        cls = torch.randn(B, 1, 16, 16, generator=g).cuda()
        prev = (20 + 100 * torch.rand(B, 2, generator=g, dtype=torch.float64)).cuda()
        boxes = torch.empty(B, 48, dtype=torch.uint8, device="cuda")
        smooth = time_kernel(lambda: lib.fear_decode_smooth(reg.data_ptr(), cls.data_ptr(), B, prev.data_ptr(),
                                                            params.data_ptr(), boxes.data_ptr(), s), (), launches)
        plain = time_kernel(lambda: lib.fear_decode(reg.data_ptr(), cls.data_ptr(), B, 1, boxes.data_ptr(), s), (),
                            launches)
        out[f"B{B}"] = dict(decode_smooth_us=smooth, decode_us=plain)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--updates", type=int, default=600, help="timed updates per arm")
    ap.add_argument("--block", type=int, default=50, help="updates per arm before switching to the next arm")
    ap.add_argument("--step-repeats", type=int, default=200, help="updates / graph replays timed with CUDA events")
    ap.add_argument("--kernel-launches", type=int, default=5000, help="launches per kernel timing")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_smooth.py measures on a CUDA device; none is available")
    clip = read_video_rgb(os.path.join(ROOT, "tests", "golden", "test.mp4"))
    net = fb.FEARNet(**fb.FEAR_XS_MODEL_KWARGS)
    net.load_state_dict(load_state(), strict=True)
    net = net.cuda().eval()
    arms = {name: Arm(net, clip, extra) for name, extra in ARMS.items()}
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
        a.record()
        for _ in range(args.step_repeats):
            arm.update()
        b.record()
        torch.cuda.synchronize()
        row = dict(host_ms_per_update=host_ms, frames_per_s=1e3 / host_ms,
                   device_ms_per_update=a.elapsed_time(b) / args.step_repeats)
        graph = getattr(arm.trk, "_gpu_crop_state", {}).get("graph")
        if graph is not None:
            a.record()
            for _ in range(args.step_repeats):
                graph.replay()
            b.record()
            torch.cuda.synchronize()
            row["device_ms_per_step"] = a.elapsed_time(b) / args.step_repeats
        results[name] = row
    kernels = kernel_times(args.kernel_launches)
    print(json.dumps({"metric": "FEARTracker smooth post-processing: host path vs gpu_crop graph, demo clip 480x256",
                      "card": card_info(torch.cuda.current_device()), "timed_updates_per_arm": args.updates,
                      "arms": results, "kernel_us": kernels}))


if __name__ == "__main__":
    main()
