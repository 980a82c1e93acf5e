#!/usr/bin/env python
"""FEARMultiTracker on 1080p RGB streams in device memory in the layouts OpenCV, capture cards, screen capture and
16-bit decoders hand over.  Arms:
  resident_rgb   uint8 (H, W, 3) RGB tensors kept on the device (the FearFrameView table): the yardstick, what the step
                 costs with no conversion at all
  bgra           RGBFrame(t, "bgra") of BGRA surfaces (cv2.cudacodec's default, DeckLink's 8-bit BGRA), read in place
                 (the FearFrameRGB table)
  x2rgb10le      RGBFrame(t, "x2rgb10le") of 10-bit RGB in 32-bit words (DRM XRGB2101010)
  rgb48le        RGBFrame(t, "rgb48le") of 16-bit RGB (ProRes 4444, 16-bit PNG / TIFF)
  gbrp16le       RGBFrame.planar(r, g, b, bits=16) of three 16-bit planes (ffmpeg's gbrp16le)
  torch_<layout> the same frames converted to a contiguous uint8 (H, W, 3) RGB tensor with torch every update, then
                 CUDA RGB frames (the FearFrameView table): a channel index + contiguous for bgra; the shift and mask,
                 the float64 map rint(255 * (v * (1 / (2^bits - 1)))) and the cast for the wide layouts -- what a user
                 had to do before RGBFrame (checked equal to image_ops.rgb_frame_to_rgb before timing)
The demo clip (tests/golden/test.mp4, 480x256) is resized to 1920x1080 with cv2.resize; its codes at 10 and 16 bits
are round(v * (2^bits - 1) / 255).  --clip-frames of its frames are kept on the device per layout, and stream s reads
clip frame (3 s + t) mod --clip-frames at update t.  Each stream holds the jittered golden boxes of bench_multi.py,
scaled to 1080p.  For F streams x k targets per stream, each arm reports:
  host_ms_per_update   wall time of one update(), frame construction (and for torch_* the conversion) included
  target_frames_per_s  N / host_ms_per_update
  device_ms_per_step   CUDA events around --step-repeats replays of the captured step
and each torch_* arm also convert_device_ms_per_update, CUDA events around --step-repeats conversions of F frames.  The
arms run in the same process on the same targets, alternated in blocks of --block updates.  One JSON line, with the
card name, power limit and SM clock read by nvidia-smi right after the timed runs.

    python tools/bench_rgb_formats.py [--configs 8x4,8x32] [--updates 300] [--block 50]
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
LAYOUTS = ("bgra", "x2rgb10le", "rgb48le", "gbrp16le")
ARMS = ("resident_rgb",) + LAYOUTS + tuple(f"torch_{k}" for k in LAYOUTS)


def to_u8(v: torch.Tensor, bits: int) -> torch.Tensor:
    """image_ops.raw_to_u8 with torch: rint(255 * (v * (1 / (2^bits - 1)))) in float64, clamped, as uint8."""
    return torch.clamp(torch.round(255.0 * (v.double() * (1.0 / float((1 << bits) - 1)))), 0, 255).to(torch.uint8)


def torch_convert(layout: str, t) -> torch.Tensor:
    """The contiguous uint8 (H, W, 3) RGB tensor of one frame's samples, with torch ops on the device."""
    if layout == "bgra":
        return t[..., [2, 1, 0]].contiguous()
    if layout == "x2rgb10le":
        w = t.to(torch.int64)
        return to_u8(torch.stack([(w >> s) & 1023 for s in (20, 10, 0)], -1), 10)
    if layout == "rgb48le":
        return to_u8(t.to(torch.int32), 16)
    return to_u8(torch.stack([p.to(torch.int32) for p in t], -1), 16)  # gbrp16le: (r, g, b) planes


def make_surfaces(clip, clip_frames):
    """Per clip frame: the RGB frame, and its samples in every layout on the device (BGRA and x2rgb10 words pitched
    to 2048 pixels, rgb48 tight, the gbrp16 planes one (3, H, W) tensor)."""
    s = {k: [] for k in ("rgb",) + LAYOUTS}
    for i in range(clip_frames):
        rgb = cv2.resize(clip[(7 * i) % len(clip)], (W, H))
        s["rgb"].append(torch.from_numpy(rgb).cuda())
        bgra = np.full((H, 2048, 4), 255, np.uint8)
        bgra[:, :W, :3] = rgb[..., ::-1]
        s["bgra"].append(torch.from_numpy(bgra).cuda()[:, :W])
        c10 = (rgb.astype(np.int64) * 1023 + 127) // 255
        words = np.zeros((H, 2048), np.uint32)
        words[:, :W] = image_ops.x2rgb10_pack(c10, "x2rgb10le", np.full((H, W), 3))
        s["x2rgb10le"].append(torch.from_numpy(words.view(np.int32)).cuda()[:, :W])
        c16 = ((rgb.astype(np.int64) * 65535 + 127) // 255).astype(np.uint16)
        s["rgb48le"].append(torch.from_numpy(c16.view(np.int16)).cuda().view(torch.uint16))
        planes = np.ascontiguousarray(np.moveaxis(c16, -1, 0))
        s["gbrp16le"].append(torch.from_numpy(planes.view(np.int16)).cuda().view(torch.uint16))
    return s


def rgb_frame(layout: str, t) -> fb.RGBFrame:
    return fb.RGBFrame.planar(*t, bits=16) if layout == "gbrp16le" else fb.RGBFrame(t, layout)


def reference(layout: str, t) -> np.ndarray:
    """image_ops.rgb_frame_to_rgb of the samples, copied back from the device."""
    if layout == "gbrp16le":
        return image_ops.rgb_frame_to_rgb(t.view(torch.int16).cpu().numpy().view(np.uint16), "planar", 16)
    a = t.cpu().numpy()
    return image_ops.rgb_frame_to_rgb(a.view(np.uint16) if layout == "rgb48le" else a, layout)


def frames(s, arm, num_streams, t):
    idx = [(3 * k + t) % len(s["rgb"]) for k in range(num_streams)]
    if arm == "resident_rgb":
        return [s["rgb"][i] for i in idx]
    if arm.startswith("torch_"):
        layout = arm[len("torch_"):]
        return [torch_convert(layout, s[layout][i]) for i in idx]
    return [rgb_frame(arm, s[arm][i]) for i in idx]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="8x4,8x32", help="streams x targets per stream")
    ap.add_argument("--updates", type=int, default=300, help="timed updates per arm")
    ap.add_argument("--block", type=int, default=50, help="updates per arm before switching to the next arm")
    ap.add_argument("--clip-frames", type=int, default=12, help="1080p frames kept on the device per layout")
    ap.add_argument("--step-repeats", type=int, default=100, help="graph replays timed with CUDA events per arm")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_rgb_formats.py measures on a CUDA device; none is available")
    clip = read_video_rgb(os.path.join(ROOT, "tests", "golden", "test.mp4"))
    surfaces = make_surfaces(clip, args.clip_frames)
    for layout in LAYOUTS:
        if not np.array_equal(torch_convert(layout, surfaces[layout][0]).cpu().numpy(),
                              reference(layout, surfaces[layout][0])):
            raise SystemExit(f"the torch conversion of {layout} differs from image_ops.rgb_frame_to_rgb")
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
        for layout in LAYOUTS:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for r in range(args.step_repeats):
                rgbs = [torch_convert(layout, surfaces[layout][(3 * s + r) % args.clip_frames]) for s in range(F)]
            b.record()
            torch.cuda.synchronize()
            row[f"torch_{layout}"]["convert_device_ms_per_update"] = a.elapsed_time(b) / args.step_repeats
        results.append(row)
        del trackers, held, rgbs
    print(json.dumps({"metric": "FEARMultiTracker on 1920x1080 RGB streams in device memory: read in place (BGRA, "
                                "x2rgb10le, rgb48le, gbrp16le), converted with torch first, and resident RGB",
                      "card": card_info(torch.cuda.current_device()), "timed_updates_per_arm": args.updates,
                      "results": results}))


if __name__ == "__main__":
    main()
