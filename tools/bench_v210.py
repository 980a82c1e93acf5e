#!/usr/bin/env python
"""FEARMultiTracker on 1080p v210 streams (10-bit 4:2:2 as SDI capture cards deliver it) in device memory.  Arms, all
10-bit BT.601 limited range 4:2:2 of the same codes:
  v210         V210Frames: the capture buffers (row pitch 5120 bytes, 128 * ceil(1920 / 48)) read in place, every
               pixel the kernels read unpacked and converted inside the crop and frame-sum kernels (the
               FearFrameYCbCrV210 table)
  unpack_i422  the same buffers unpacked with torch ops every update into three uint16 planes, then
               YUV422Frame(y, u, v, bits=10) (the FearFrameYCbCr table): what a user had to do before V210Frame
  p210         P210 YUV422Frames (uint16 NV16, MSB-aligned, row pitch 4096 bytes) of the same codes: the existing
               10-bit 4:2:2 path, as the yardstick
The demo clip (tests/golden/test.mp4, 480x256) is resized to 1920x1080 with cv2.resize; --clip-frames of its frames
are encoded once by the forward H.273 equations (chroma: the mean over each pixel pair) and kept on the device, and
stream s reads clip frame (3 s + t) mod --clip-frames at update t.  Each stream holds the jittered golden boxes of
bench_multi.py, scaled to 1080p.  For F streams x k targets per stream, each arm reports:
  host_ms_per_update   wall time of one update(), frame construction (and for unpack_i422 the unpack) included
  target_frames_per_s  N / host_ms_per_update
  device_ms_per_step   CUDA events around --step-repeats replays of the captured step
and unpack_i422 also unpack_device_ms_per_update, CUDA events around --step-repeats unpacks of F buffers.  The arms run
in the same process on the same targets, alternated in blocks of --block updates.  One JSON line, with the card name,
power limit and SM clock read by nvidia-smi right after the timed runs.

    python tools/bench_v210.py [--configs 8x4,8x32] [--updates 300] [--block 50]
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
from bench_yuv_subsampling import H, W, encode  # noqa: E402
from feartracker_b200 import image_ops  # noqa: E402
from oracle.fear_oracle import read_video_rgb  # noqa: E402

WARMUP = 3  # eager warm-up + capture + one replay
ARMS = ("v210", "unpack_i422", "p210")
P210_PITCH = 2048  # uint16 samples


def make_surfaces(clip, clip_frames):
    """clip_frames v210 buffers (H, 5120) uint8 and P210 surfaces (2H, 1920) uint16 views of the same codes."""
    v210, p210 = [], []
    for i in range(clip_frames):
        y, u, v = encode(cv2.resize(clip[(7 * i) % len(clip)], (W, H)), 10, (1, 0))
        v210.append(torch.from_numpy(image_ops.v210_pack(y, u, v)).cuda())
        plane = (np.concatenate([y, np.stack([u, v], -1).reshape(-1, W)]) << 6).astype(np.uint16)
        t = torch.zeros((2 * H, P210_PITCH), dtype=torch.int16, device="cuda")
        t[:, :W] = torch.from_numpy(plane.view(np.int16)).cuda()
        p210.append(t.view(torch.uint16)[:, :W])
    return v210, p210


def unpack(t: torch.Tensor):
    """The (y, u, v) uint16 planes of a 1080p v210 buffer with torch ops (image_ops.v210_unpack on the device)."""
    words = t[:, :image_ops.v210_row_bytes(W)].contiguous().view(torch.int32).view(H, -1, 4)
    codes = torch.stack([(words >> s) & 1023 for s in (0, 10, 20)], -1).view(H, -1, 12)
    y = codes[..., 1::2].reshape(H, -1)[:, :W]
    u = codes[..., 0::4].reshape(H, -1)[:, :W // 2]
    v = codes[..., 2::4].reshape(H, -1)[:, :W // 2]
    return tuple(p.to(torch.uint16) for p in (y, u, v))


def frames(surfaces, arm, num_streams, t):
    v210, p210 = surfaces
    idx = [(3 * s + t) % len(v210) for s in range(num_streams)]
    if arm == "v210":
        return [fb.V210Frame(v210[i], W) for i in idx]
    if arm == "unpack_i422":
        return [fb.YUV422Frame(*unpack(v210[i]), bits=10) for i in idx]
    return [fb.YUV422Frame.nv16(p210[i], bits=10) for i in idx]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="8x4,8x32", help="streams x targets per stream")
    ap.add_argument("--updates", type=int, default=300, help="timed updates per arm")
    ap.add_argument("--block", type=int, default=50, help="updates per arm before switching to the next arm")
    ap.add_argument("--clip-frames", type=int, default=12, help="1080p frames kept on the device per layout")
    ap.add_argument("--step-repeats", type=int, default=100, help="graph replays timed with CUDA events per arm")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_v210.py measures on a CUDA device; none is available")
    clip = read_video_rgb(os.path.join(ROOT, "tests", "golden", "test.mp4"))
    surfaces = make_surfaces(clip, args.clip_frames)
    torch.cuda.synchronize()
    net = fb.FEARNet(**fb.FEAR_XS_MODEL_KWARGS)
    net.load_state_dict(load_state(), strict=True)
    net = net.cuda().eval()
    cfg = fb.FEAR_XS_TRACKER_KWARGS
    scale = np.array([W / 480, H / 256, W / 480, H / 256])
    results = []
    for config in args.configs.split(","):
        F, k = (int(v) for v in config.split("x"))
        n = F * k
        rects = np.concatenate([np.rint(jittered_boxes(k, seed=s) * scale) for s in range(F)])
        streams = np.repeat(np.arange(F), k)
        trackers = {a: fb.FEARMultiTracker(net, cuda_id=0, max_targets=n, **cfg) for a in ARMS}
        row = {"streams": F, "targets_per_stream": k, "N": n}
        for arm, trk in trackers.items():
            trk.initialize(frames(surfaces, arm, F, 0), rects, streams)
            for t in range(1, 1 + WARMUP):
                trk.update(frames(surfaces, arm, F, t))
        spent = {a: 0.0 for a in ARMS}
        done = {a: 0 for a in ARMS}
        held = {}
        order = list(ARMS)
        while min(done.values()) < args.updates:
            for arm in order:
                m = min(args.block, args.updates - done[arm])
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for j in range(m):
                    fr = frames(surfaces, arm, F, 1 + WARMUP + done[arm] + j)
                    trackers[arm].update(fr)
                spent[arm] += time.perf_counter() - t0
                held[arm] = fr  # the frames the tracker's table points at, kept alive for the replays below
                done[arm] += m
            order.reverse()
        for arm, trk in trackers.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.step_repeats):
                trk._graph.replay()
            b.record()
            torch.cuda.synchronize()
            host_ms = spent[arm] * 1e3 / done[arm]
            row[arm] = dict(table=trk._graph_key[2], host_ms_per_update=host_ms, target_frames_per_s=n * 1e3 / host_ms,
                            device_ms_per_step=a.elapsed_time(b) / args.step_repeats)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for r in range(args.step_repeats):
            planes = [unpack(surfaces[0][(3 * s + r) % len(surfaces[0])]) for s in range(F)]
        b.record()
        torch.cuda.synchronize()
        row["unpack_i422"]["unpack_device_ms_per_update"] = a.elapsed_time(b) / args.step_repeats
        results.append(row)
        del trackers, held, planes
    print(json.dumps({"metric": "FEARMultiTracker on 1920x1080 v210 streams in device memory: read in place, unpacked "
                                "with torch first, and P210", "card": card_info(torch.cuda.current_device()),
                      "timed_updates_per_arm": args.updates, "results": results}))


if __name__ == "__main__":
    main()
