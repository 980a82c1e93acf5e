#!/usr/bin/env python
"""FEARMultiTracker on 1080p YUV streams in device memory at three chroma subsamplings, each read in place (every pixel
the kernels read is converted inside the crop and frame-sum kernels).  Arms, all 8-bit BT.601 limited range except
P210:
  nv12_420      NV12 YUV420Frames, row pitch 2048 bytes (the FearFrameYUV table)
  yuyv_422      packed YUYV YUV422Frames (a UVC webcam's format), row pitch 4096 bytes (the FearFrameYCbCr table)
  p210_422      10-bit P210 YUV422Frames (uint16, MSB-aligned), row pitch 4096 bytes
  i444_pitched  planar I444 YUV444Frames, row pitch 2048 bytes
The demo clip (tests/golden/test.mp4, 480x256) is resized to 1920x1080 with cv2.resize; --clip-frames of its frames
are encoded once per layout by the forward H.273 equations (chroma: the mean over each chroma sample's pixels) and
kept on the device, and stream s reads clip frame (3 s + t) mod --clip-frames at update t.  Each stream holds the
jittered golden boxes of bench_multi.py, scaled to 1080p.  For F streams x k targets per stream, each arm reports:
  host_ms_per_update   wall time of one update(), frame construction included
  target_frames_per_s  N / host_ms_per_update
  device_ms_per_step   CUDA events around --step-repeats replays of the captured step
The arms run in the same process on the same targets, alternated in blocks of --block updates.  One JSON line, with
the card name, power limit and SM clock read by nvidia-smi right after the timed runs.

    python tools/bench_yuv_subsampling.py [--configs 8x4,8x32] [--updates 300] [--block 50]
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
from feartracker_b200 import image_ops  # noqa: E402
from oracle.fear_oracle import read_video_rgb  # noqa: E402

W, H = 1920, 1080
WARMUP = 3  # eager warm-up + capture + one replay
ARMS = {  # name: (layout, bits, (chroma_shift_x, chroma_shift_y), row pitch in samples)
    "nv12_420": ("nv12", 8, (1, 1), 2048),
    "yuyv_422": ("yuyv", 8, (1, 0), 4096),
    "p210_422": ("nv16", 10, (1, 0), 2048),
    "i444_pitched": ("i444", 8, (0, 0), 2048),
}


def encode(rgb, bits, chroma_shift):
    """BT.601 limited-range code planes (Y (H, W), U and V (H >> sy, W >> sx)) of an RGB frame by the forward H.273
    equations."""
    _, kr, kb = image_ops.YUV_MATRICES["bt601"]
    r, g, b = (rgb[..., c].astype(np.float64) / 255.0 for c in range(3))
    yn = kr * r + (1.0 - kr - kb) * g + kb * b
    pb, pr = (b - yn) / (2.0 * (1.0 - kb)), (r - yn) / (2.0 * (1.0 - kr))
    sx, sy = chroma_shift
    pb, pr = (p.reshape(H >> sy, 1 << sy, W >> sx, 1 << sx).mean(axis=(1, 3)) for p in (pb, pr))
    m = 1 << (bits - 8)
    return [np.clip(np.rint(off * m + scale * m * p), 0, (1 << bits) - 1).astype(np.int64)
            for off, scale, p in ((16, 219, yn), (128, 224, pb), (128, 224, pr))]


def make_surfaces(clip, clip_frames):
    """Per arm, clip_frames device surfaces of (rows, pitch) samples holding the layout in their first columns."""
    out = {}
    for arm, (layout, bits, shifts, pitch) in ARMS.items():
        dtype = np.uint8 if bits == 8 else np.uint16
        shift = 16 - bits if bits > 8 else 0
        surfs = []
        for i in range(clip_frames):
            y, u, v = (p << shift for p in encode(cv2.resize(clip[(7 * i) % len(clip)], (W, H)), bits, shifts))
            if layout in ("nv12", "nv16"):
                plane = np.concatenate([y, np.stack([u, v], -1).reshape(-1, W)])
            elif layout == "yuyv":
                plane = np.empty((H, 2 * W), np.int64)
                plane[:, 0::2], plane[:, 1::4], plane[:, 3::4] = y, u, v
            else:
                plane = np.concatenate([y, u, v])
            plane = plane.astype(dtype)
            t = torch.zeros((plane.shape[0], pitch), dtype=torch.uint8 if bits == 8 else torch.int16, device="cuda")
            t[:, :plane.shape[1]] = torch.from_numpy(plane if bits == 8 else plane.view(np.int16)).cuda()
            surfs.append((t if bits == 8 else t.view(torch.uint16))[:, :plane.shape[1]])
        out[arm] = surfs
    return out


def frames(surfaces, arm, num_streams, t):
    layout, bits, _, _ = ARMS[arm]
    make = {"nv12": fb.YUV420Frame.nv12, "yuyv": fb.YUV422Frame.yuyv, "nv16": fb.YUV422Frame.nv16,
            "i444": fb.YUV444Frame.i444}[layout]
    surfs = surfaces[arm]
    return [make(surfs[(3 * s + t) % len(surfs)], bits=bits) for s in range(num_streams)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="8x4,8x32", help="streams x targets per stream")
    ap.add_argument("--updates", type=int, default=300, help="timed updates per arm")
    ap.add_argument("--block", type=int, default=50, help="updates per arm before switching to the next arm")
    ap.add_argument("--clip-frames", type=int, default=12, help="1080p frames per layout kept on the device")
    ap.add_argument("--step-repeats", type=int, default=100, help="graph replays timed with CUDA events per arm")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_yuv_subsampling.py measures on a CUDA device; none is available")
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
        results.append(row)
        del trackers, held
    print(json.dumps({"metric": "FEARMultiTracker on 1920x1080 YUV streams in device memory at 4:2:0, 4:2:2 and 4:4:4, "
                                "read in place", "card": card_info(torch.cuda.current_device()),
                      "timed_updates_per_arm": args.updates, "results": results}))


if __name__ == "__main__":
    main()
