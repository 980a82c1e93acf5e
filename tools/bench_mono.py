#!/usr/bin/env python
"""FEARMultiTracker on 1080p single-channel streams (as mono machine-vision cameras, mono CSI-2 sensors and thermal
cores deliver them) in device memory.  Arms:
  mono8         MonoFrames of 8-bit grey frames (row pitch 2048 bytes) read in place, every tap mapped to grey inside
                the crop and frame-sum kernels (the FearFrameMono table)
  mono12_msb    MonoFrame(bits=12, msb=True) of the same picture at 12 bits, MSB-aligned in uint16 (row pitch 4096
                bytes): the same kernels with the 12-bit mapping
  raw10         MonoFrame.raw10 of the picture at 10 bits packed as MIPI CSI-2 RAW10 / Y10P (row pitch 2432 bytes)
  y16_agc       MonoFrame(bits=16, agc="minmax") of a thermal core's narrow band of 16-bit codes (30000 + 8 * grey):
                fear_frame_range_mono then the same kernels with min-max gain control, 49 launches per step
  torch_agc     the same Y16 frames converted with torch every update (aminmax, the gain as a table of the codes in
                range, a gather, expanded to a contiguous (H, W, 3) uint8 tensor), then CUDA RGB frames (the
                FearFrameView table): what a user had to do before MonoFrame
  resident_rgb  the grey RGB frames of y16_agc converted once and kept on the device: the yardstick, what the step
                costs with no conversion at all
The demo clip (tests/golden/test.mp4, 480x256) is resized to 1920x1080 with cv2.resize and converted with
cv2.COLOR_RGB2GRAY; --clip-frames of its frames are kept on the device per layout, and stream s reads clip frame
(3 s + t) mod --clip-frames at update t.  Each stream holds the jittered golden boxes of bench_multi.py, scaled to
1080p.  For F streams x k targets per stream, each arm reports:
  host_ms_per_update   wall time of one update(), frame construction (and for torch_agc the conversion) included
  target_frames_per_s  N / host_ms_per_update
  device_ms_per_step   CUDA events around --step-repeats replays of the captured step
and torch_agc also convert_device_ms_per_update, CUDA events around --step-repeats conversions of F frames.  The arms
run in the same process on the same targets, alternated in blocks of --block updates.  One JSON line, with the card
name, power limit and SM clock read by nvidia-smi right after the timed runs.

    python tools/bench_mono.py [--configs 8x4,8x32] [--updates 300] [--block 50]
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
ARMS = ("mono8", "mono12_msb", "raw10", "y16_agc", "torch_agc", "resident_rgb")
PITCH8 = 2048
PITCH16 = 2048  # uint16 samples
PITCH10 = 2432  # >= 5 * 1920 / 4 = 2400


def torch_agc(codes: torch.Tensor) -> torch.Tensor:
    """image_ops.mono_to_rgb(codes, 16, "minmax") with torch ops on the device: torch.aminmax of the frame, the grey
    value of each code in [lo, hi] by OpenCV's gain (image_ops.minmax_normalize of those codes, a table of hi - lo + 1
    bytes sent to the device), a gather through that table, then the grey triple made contiguous."""
    lo, hi = (int(v) for v in torch.aminmax(codes.to(torch.int32)))
    lut = torch.from_numpy(image_ops.minmax_normalize(np.arange(lo, hi + 1, dtype=np.uint16)) if hi > lo
                           else np.zeros(1, np.uint8)).to(codes.device)
    g = lut[codes.to(torch.int64) - lo]
    return g[..., None].expand(H, W, 3).contiguous()


def make_surfaces(clip, clip_frames):
    """Per clip frame: the 8-bit grey frame (pitched), its 12-bit MSB and RAW10 containers, the thermal Y16 codes, and
    the grey RGB frame of those codes with gain control."""
    s = {k: [] for k in ("mono8", "mono12_msb", "raw10", "y16", "rgb")}
    for i in range(clip_frames):
        g = cv2.cvtColor(cv2.resize(clip[(7 * i) % len(clip)], (W, H)), cv2.COLOR_RGB2GRAY)
        t = torch.zeros((H, PITCH8), dtype=torch.uint8, device="cuda")
        t[:, :W] = torch.from_numpy(g).cuda()
        s["mono8"].append(t[:, :W])
        c12 = ((g.astype(np.uint16) * 4095 + 127) // 255) << 4
        t = torch.zeros((H, PITCH16), dtype=torch.int16, device="cuda")
        t[:, :W] = torch.from_numpy(c12.view(np.int16)).cuda()
        s["mono12_msb"].append(t.view(torch.uint16)[:, :W])
        s["raw10"].append(torch.from_numpy(image_ops.mipi_pack(g.astype(np.uint16) * 4, 10, PITCH10)).cuda())
        y16 = (30000 + 8 * g.astype(np.uint16)).astype(np.uint16)
        t = torch.zeros((H, PITCH16), dtype=torch.int16, device="cuda")
        t[:, :W] = torch.from_numpy(y16.view(np.int16)).cuda()
        s["y16"].append(t.view(torch.uint16)[:, :W])
        s["rgb"].append(torch.from_numpy(image_ops.mono_to_rgb(y16, 16, "minmax")).cuda())
    return s


def frames(s, arm, num_streams, t):
    idx = [(3 * k + t) % len(s["mono8"]) for k in range(num_streams)]
    if arm == "mono8":
        return [fb.MonoFrame(s["mono8"][i]) for i in idx]
    if arm == "mono12_msb":
        return [fb.MonoFrame(s["mono12_msb"][i], bits=12, msb=True) for i in idx]
    if arm == "raw10":
        return [fb.MonoFrame.raw10(s["raw10"][i][:, :W * 5 // 4], W) for i in idx]
    if arm == "y16_agc":
        return [fb.MonoFrame(s["y16"][i], bits=16, agc="minmax") for i in idx]
    if arm == "torch_agc":
        return [torch_agc(s["y16"][i]) for i in idx]
    return [s["rgb"][i] for i in idx]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="8x4,8x32", help="streams x targets per stream")
    ap.add_argument("--updates", type=int, default=300, help="timed updates per arm")
    ap.add_argument("--block", type=int, default=50, help="updates per arm before switching to the next arm")
    ap.add_argument("--clip-frames", type=int, default=12, help="1080p frames kept on the device per layout")
    ap.add_argument("--step-repeats", type=int, default=100, help="graph replays timed with CUDA events per arm")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mono.py measures on a CUDA device; none is available")
    clip = read_video_rgb(os.path.join(ROOT, "tests", "golden", "test.mp4"))
    surfaces = make_surfaces(clip, args.clip_frames)
    if not torch.equal(torch_agc(surfaces["y16"][0]), surfaces["rgb"][0]):
        raise SystemExit("the torch conversion differs from image_ops.mono_to_rgb")
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
            rgbs = [torch_agc(surfaces["y16"][(3 * s + r) % len(surfaces["y16"])]) for s in range(F)]
        b.record()
        torch.cuda.synchronize()
        row["torch_agc"]["convert_device_ms_per_update"] = a.elapsed_time(b) / args.step_repeats
        results.append(row)
        del trackers, held, rgbs
    print(json.dumps({"metric": "FEARMultiTracker on 1920x1080 mono streams in device memory: read in place (Mono8, "
                                "Mono12 MSB, RAW10, Y16 with min-max AGC), converted with torch first, and resident RGB",
                      "card": card_info(torch.cuda.current_device()), "timed_updates_per_arm": args.updates,
                      "results": results}))


if __name__ == "__main__":
    main()
