#!/usr/bin/env python
"""FEARMultiTracker on 1080p HDR streams (10-bit BT.2020 P010, as NVDEC decodes HEVC Main10) in device memory.  Arms:
  pq              PQ P010 YUV420Frames (transfer="pq"): read in place, every tap the kernels read tone-mapped to SDR
                  inside the crop and frame-sum kernels (the FearFrameYCbCrHDR table)
  hlg             HLG P010 YUV420Frames (transfer="hlg") of the same clip, likewise
  sdr             the PQ arm's codes read as BT.2020 SDR (no transfer, the FearFrameYUV table): today's path, the
                  yardstick
  torch_tonemap   the PQ arm's surfaces tone-mapped to a (1080, 1920, 3) uint8 RGB tensor with torch ops (float32,
                  the same chain) every update, then tracked as CUDA tensors: what a user had to do before
The demo clip (tests/golden/test.mp4, 480x256) is resized to 1920x1080 with cv2.resize and made HDR the BT.2408 way
(tests/hdr_frames.py: SDR white at 203 cd/m²); --clip-frames frames are kept on the device and stream s reads clip
frame (3 s + t) mod --clip-frames at update t.  Each stream holds the jittered golden boxes of bench_multi.py, scaled to
1080p.  For F streams x k targets per stream, each arm reports:
  host_ms_per_update   wall time of one update(), frame construction (and for torch_tonemap the tone mapping) included
  device_ms_per_step   CUDA events around --step-repeats replays of the captured step
and torch_tonemap also tonemap_device_ms_per_update, CUDA events around --step-repeats tone mappings of F surfaces.
The arms run in the same process on the same targets, alternated in blocks of --block updates.  One JSON line, with
the card name, power limit and SM clock read by nvidia-smi right after the timed runs.

    python tools/bench_hdr.py [--configs 8x4,8x32] [--updates 200] [--block 50]
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
from tests.hdr_frames import hdr_codes  # noqa: E402

H, W = 1080, 1920
PITCH = 2048  # uint16 samples per P010 row
WARMUP = 3  # eager warm-up + capture + one replay
ARMS = ("pq", "hlg", "sdr", "torch_tonemap")


def make_surfaces(clip, clip_frames, transfer):
    out = []
    for i in range(clip_frames):
        y, u, v = hdr_codes(cv2.resize(clip[(7 * i) % len(clip)], (W, H)), transfer, 10, False, "420")
        plane = (np.concatenate([y, np.stack([u, v], -1).reshape(-1, W)]) << 6).astype(np.uint16)
        t = torch.zeros((H * 3 // 2, PITCH), dtype=torch.int16, device="cuda")
        t[:, :W] = torch.from_numpy(plane.view(np.int16)).cuda()
        out.append(t.view(torch.uint16)[:, :W])
    return out


def torch_tonemap_pq(t: torch.Tensor) -> torch.Tensor:
    """A P010 PQ surface -> (H, W, 3) uint8 SDR BT.709 RGB with torch ops in float32 (the chain of
    image_ops.hdr_to_sdr, nearest chroma)."""
    s = (t.view(torch.int16).to(torch.int32) & 0xFFFF) >> 6
    y = s[:H].float()
    uv = s[H:].view(H // 2, W // 2, 2).float().repeat_interleave(2, 0).repeat_interleave(2, 1)
    yn, pb, pr = (y - 64) / 876, (uv[..., 0] - 512) / 896, (uv[..., 1] - 512) / 896
    e = torch.stack([yn + 1.4746 * pr, yn - 0.16455 * pb - 0.57135 * pr, yn + 1.8814 * pb], -1).clamp(0, 1)
    p = e ** (1 / image_ops.PQ_M2)
    fd = 10000 * ((p - image_ops.PQ_C1).clamp_min(0) / (image_ops.PQ_C2 - image_ops.PQ_C3 * p)) ** (1 / image_ops.PQ_M1)
    c = (fd / 1000).clamp_max(1) ** (1 / 2.4)
    yl = 0.2627 * c[..., 0] + 0.6780 * c[..., 1] + 0.0593 * c[..., 2]
    k = image_ops.HDR_CONSTANTS
    yp = torch.log1p(k["rho_hdr_m1"] * yl) / k["ln_rho_hdr"]
    yc = torch.where(yp <= 0.7399, 1.077 * yp, torch.where(yp < 0.9909, -1.1510 * yp * yp + 2.7811 * yp - 0.6302,
                                                          0.5 * yp + 0.5))
    ysdr = (k["rho_sdr"] ** yc - 1) / k["rho_sdr_m1"]
    f = torch.where(yl > 0, ysdr / (1.1 * yl).clamp_min(1e-12), torch.zeros_like(yl))
    cb, cr = f * (c[..., 2] - yl) / 1.8814, f * (c[..., 0] - yl) / 1.4746
    yt = ysdr - (0.1 * cr).clamp_min(0)
    r, b = yt + 1.4746 * cr, yt + 1.8814 * cb
    g = (yt - 0.2627 * r - 0.0593 * b) / 0.6780
    lin = torch.stack([r, g, b], -1).clamp(0, 1) ** 2.4
    m = torch.tensor(image_ops.bt2020_to_bt709_matrix(), dtype=torch.float32, device=t.device)
    out = (lin @ m.T).clamp(0, 1) ** (1 / 2.4)
    return torch.round(out * 255).to(torch.uint8)


def frames(surf, arm, num_streams, t):
    src = surf["hlg"] if arm == "hlg" else surf["pq"]
    idx = [(3 * s + t) % len(src) for s in range(num_streams)]
    if arm == "torch_tonemap":
        return [torch_tonemap_pq(src[i]) for i in idx]
    transfer = None if arm == "sdr" else arm
    return [fb.YUV420Frame.nv12(src[i], matrix="bt2020", bits=10, transfer=transfer) for i in idx]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="8x4,8x32", help="streams x targets per stream")
    ap.add_argument("--updates", type=int, default=200, help="timed updates per arm")
    ap.add_argument("--block", type=int, default=50, help="updates per arm before switching to the next arm")
    ap.add_argument("--clip-frames", type=int, default=12, help="1080p frames kept on the device per transfer")
    ap.add_argument("--step-repeats", type=int, default=50, help="graph replays timed with CUDA events per arm")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_hdr.py measures on a CUDA device; none is available")
    clip = read_video_rgb(os.path.join(ROOT, "tests", "golden", "test.mp4"))
    surf = {tr: make_surfaces(clip, args.clip_frames, tr) for tr in ("pq", "hlg")}
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
            trk.initialize(frames(surf, arm, F, 0), rects, streams)
            for t in range(1, 1 + WARMUP):
                trk.update(frames(surf, arm, F, t))
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
                    fr = frames(surf, arm, F, 1 + WARMUP + done[arm] + j)
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
            row[arm] = dict(table=trk._graph_key[2], host_ms_per_update=host_ms,
                            device_ms_per_step=a.elapsed_time(b) / args.step_repeats)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for r in range(args.step_repeats):
            rgbs = [torch_tonemap_pq(surf["pq"][(3 * s + r) % len(surf["pq"])]) for s in range(F)]
        b.record()
        torch.cuda.synchronize()
        row["torch_tonemap"]["tonemap_device_ms_per_update"] = a.elapsed_time(b) / args.step_repeats
        results.append(row)
        del trackers, held, rgbs
    print(json.dumps({"metric": "FEARMultiTracker on 1920x1080 HDR P010 streams in device memory: PQ and HLG tone-mapped "
                                "in the crop, BT.2020 SDR, and tone-mapped with torch first",
                      "card": card_info(torch.cuda.current_device()), "timed_updates_per_arm": args.updates,
                      "results": results}))


if __name__ == "__main__":
    main()
