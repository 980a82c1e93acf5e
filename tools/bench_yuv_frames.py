#!/usr/bin/env python
"""FEARMultiTracker on 1080p NV12 streams already in device memory, as a hardware video decoder leaves them: read in
place as YUV420Frames, or converted to RGB first.  The demo clip (tests/golden/test.mp4, 480x256) is resized to
1920x1080 with cv2.resize and converted with cv2.cvtColor(COLOR_RGB2YUV_I420); stream s starts at clip frame 20 * s and
cycles through --clip-frames frames, each kept on the device as an NV12 surface with a row pitch of 2048 bytes.  Each
stream holds the jittered golden boxes of bench_multi.py, scaled to 1080p.  Arms:
  yuv       the surfaces passed as YUV420Frame.nv12(surface[:, :1920]): each pixel the kernels read is converted inside
            the crop and frame-sum kernels
  convert   every update converts each surface into a freshly allocated (1080, 1920, 3) RGB tensor on the current
            stream (nv12_to_rgb: a torch restatement of the conversion the kernels use, a few unfused elementwise ops),
            then passes the RGB tensors
For F streams x k targets per stream, each arm reports:
  host_ms_per_update   wall time of one update(), frame preparation included (YUV420Frame records / the conversion)
  target_frames_per_s  N / host_ms_per_update
  device_ms_per_step   CUDA events around replays of the captured step (convert: conversion of the F frames + replay)
  add_ms               wall time of adding all N targets (initialize: frame sums, template crops and features)
and rgb_bytes_per_update, the RGB frames the yuv arm does not allocate (F x 1080 x 1920 x 3).  Both arms run in the
same process on the same targets, alternated in blocks of --block updates, and must return identical boxes and scores
on their last update.  One JSON line, with the card name, power limit and SM clock read by nvidia-smi right after the
timed runs.

    python tools/bench_yuv_frames.py [--streams 1,4,8] [--targets 4,32] [--updates 300] [--block 50]
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
PITCH = 2048
WARMUP = 3  # eager warm-up + capture + one replay
ADD_REPEATS = 5
STEP_REPEATS = 50


def make_surfaces(clip, num_streams, clip_frames):
    """Per stream, a (clip_frames, 1620, PITCH) uint8 CUDA tensor of pitched NV12 surfaces of the resized clip."""
    out = []
    for s in range(num_streams):
        surf = torch.zeros((clip_frames, H * 3 // 2, PITCH), dtype=torch.uint8, device="cuda")
        for i in range(clip_frames):
            i420 = cv2.cvtColor(cv2.resize(clip[(20 * s + i) % len(clip)], (W, H)), cv2.COLOR_RGB2YUV_I420)
            u = i420[H:H + H // 4].reshape(H // 2, W // 2)
            v = i420[H + H // 4:].reshape(H // 2, W // 2)
            nv12 = np.concatenate([i420[:H], np.stack([u, v], -1).reshape(H // 2, W)])
            surf[i, :, :W] = torch.from_numpy(nv12).cuda()
        out.append(surf)
    return out


def nv12_to_rgb(t: torch.Tensor) -> torch.Tensor:
    """(3H/2, W) NV12 -> a new (H, W, 3) uint8 RGB tensor, with the integer BT.601 conversion of cv2.cvtColor
    (COLOR_YUV2RGB_NV12) that the kernels use: nearest chroma, 20-bit fixed point, round half up."""
    h = 2 * t.shape[0] // 3
    uv = t[h:]
    y = t[:h].int()
    u = uv[:, 0::2].int().repeat_interleave(2, 0).repeat_interleave(2, 1) - 128
    v = uv[:, 1::2].int().repeat_interleave(2, 0).repeat_interleave(2, 1) - 128
    yy = (y - 16).clamp_min(0) * 1220542 + (1 << 19)
    r = (yy + 1673527 * v) >> 20
    g = (yy - 852492 * v - 409993 * u) >> 20
    b = (yy + 2116026 * u) >> 20
    return torch.stack([r, g, b], -1).clamp(0, 255).to(torch.uint8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", default="1,4,8")
    ap.add_argument("--targets", default="4,32", help="targets per stream")
    ap.add_argument("--updates", type=int, default=300, help="timed updates per arm")
    ap.add_argument("--block", type=int, default=50, help="updates per arm before switching to the other arm")
    ap.add_argument("--clip-frames", type=int, default=40, help="1080p NV12 surfaces per stream kept on the device")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_yuv_frames.py measures on a CUDA device; none is available")
    clip = read_video_rgb(os.path.join(ROOT, "tests", "golden", "test.mp4"))
    stream_counts = [int(s) for s in args.streams.split(",")]
    surfaces = make_surfaces(clip, max(stream_counts), args.clip_frames)
    torch.cuda.synchronize()
    net = fb.FEARNet(**fb.FEAR_XS_MODEL_KWARGS)
    net.load_state_dict(load_state(), strict=True)
    net = net.cuda().eval()
    cfg = fb.FEAR_XS_TRACKER_KWARGS
    scale = np.array([W / 480, H / 256, W / 480, H / 256])
    T = args.clip_frames

    def frames(arm, F, i):
        nv12 = [surfaces[s][i % T, :, :W] for s in range(F)]
        return [fb.YUV420Frame.nv12(t) for t in nv12] if arm == "yuv" else [nv12_to_rgb(t) for t in nv12]

    results = []
    for F in stream_counts:
        for k in (int(t) for t in args.targets.split(",")):
            n = F * k
            rects = np.concatenate([np.rint(jittered_boxes(k, seed=s) * scale) for s in range(F)])
            streams = np.repeat(np.arange(F), k)
            arms = {a: fb.FEARMultiTracker(net, cuda_id=0, max_targets=n, **cfg) for a in ("yuv", "convert")}
            row = {"streams": F, "targets_per_stream": k, "N": n, "rgb_bytes_per_update": F * H * W * 3}
            held, last = {}, {}
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
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    for j in range(m):
                        fr = frames(arm, F, pos[arm] + j)
                        last[arm] = arms[arm].update(fr)
                    spent[arm] += time.perf_counter() - t0
                    held[arm] = fr  # the frames the tracker's table points at, kept alive for the replays below
                    done[arm] += m
                    pos[arm] += m
                order.reverse()
            for arm, trk in arms.items():
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for i in range(STEP_REPEATS):
                    if arm == "convert":
                        frames(arm, F, i)
                    trk._graph.replay()
                b.record()
                torch.cuda.synchronize()
                host_ms = spent[arm] * 1e3 / done[arm]
                row[arm].update(host_ms_per_update=host_ms, target_frames_per_s=n * 1e3 / host_ms,
                                device_ms_per_step=a.elapsed_time(b) / STEP_REPEATS)
            for key in ("ids", "bbox", "score"):
                assert np.array_equal(last["yuv"][key], last["convert"][key]), (F, k, key)
            results.append(row)
            del arms, held
    print(json.dumps({"metric": "FEARMultiTracker on 1920x1080 NV12 streams in device memory: YUV420Frame read in "
                                "place vs converted to an RGB tensor every update",
                      "card": card_info(torch.cuda.current_device()), "timed_updates_per_arm": args.updates,
                      "results": results}))


if __name__ == "__main__":
    main()
