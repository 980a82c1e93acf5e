#!/usr/bin/env python
"""FEARMultiTracker on 1080p raw Bayer streams (as machine-vision and CSI-2 cameras deliver them) in device memory.
Arms, all of the same mosaics:
  bayer8          BayerFrames of 8-bit RGGB mosaics (row pitch 2048 bytes) read in place, every tap demosaiced inside
                  the crop and frame-sum kernels (the FearFrameBayer table)
  raw10           BayerFrame.raw10 of the same codes x 4 packed as MIPI CSI-2 RAW10 (row pitch 2432 bytes): the same
                  kernels with the packed fetch and the 10-bit mapping
  torch_demosaic  the 8-bit mosaics demosaiced with torch ops every update into fresh (H, W, 3) uint8 tensors
                  (image_ops.bayer_to_rgb on the device), then CUDA RGB frames (the FearFrameView table): what a user
                  had to do before BayerFrame
  resident_rgb    the same RGB frames demosaiced once and kept on the device: the yardstick, what the step costs with
                  no demosaic at all
The demo clip (tests/golden/test.mp4, 480x256) is resized to 1920x1080 with cv2.resize and sampled through an RGGB
filter; --clip-frames of its frames are kept on the device, and stream s reads clip frame (3 s + t) mod --clip-frames
at update t.  Each stream holds the jittered golden boxes of bench_multi.py, scaled to 1080p.  For F streams x k
targets per stream, each arm reports:
  host_ms_per_update   wall time of one update(), frame construction (and for torch_demosaic the demosaic) included
  target_frames_per_s  N / host_ms_per_update
  device_ms_per_step   CUDA events around --step-repeats replays of the captured step
and torch_demosaic also demosaic_device_ms_per_update, CUDA events around --step-repeats demosaics of F mosaics.  The
arms run in the same process on the same targets, alternated in blocks of --block updates.  One JSON line, with the
card name, power limit and SM clock read by nvidia-smi right after the timed runs.

    python tools/bench_bayer.py [--configs 8x4,8x32] [--updates 300] [--block 50]
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
ARMS = ("bayer8", "raw10", "torch_demosaic", "resident_rgb")
PITCH8 = 2048
PITCH10 = 2432  # >= 5 * 1920 / 4 = 2400


def rggb(rgb: np.ndarray) -> np.ndarray:
    """The 8-bit RGGB mosaic of an RGB frame: R at (even, even), B at (odd, odd), G elsewhere."""
    out = rgb[..., 1].copy()
    out[0::2, 0::2] = rgb[0::2, 0::2, 0]
    out[1::2, 1::2] = rgb[1::2, 1::2, 2]
    return out


class TorchDemosaic:
    """image_ops.bayer_to_rgb of an 8-bit RGGB (H, W) mosaic with torch ops on the device: int32 cross, diagonal,
    horizontal and vertical averages of the interior, selected per site, then the border rows and columns copied in."""

    def __init__(self, dev):
        yy = torch.arange(1, H - 1, device=dev)[:, None]
        xx = torch.arange(1, W - 1, device=dev)[None, :]
        self.r_row, r_col = (yy % 2 == 0).expand(H - 2, W - 2), (xx % 2 == 0).expand(H - 2, W - 2)
        self.rb = self.r_row == r_col
        self.rows = torch.arange(H, device=dev).clamp(1, H - 2) - 1
        self.cols = torch.arange(W, device=dev).clamp(1, W - 2) - 1

    def __call__(self, raw: torch.Tensor) -> torch.Tensor:
        s = raw.to(torch.int32)
        c, n, so, we, e = s[1:-1, 1:-1], s[:-2, 1:-1], s[2:, 1:-1], s[1:-1, :-2], s[1:-1, 2:]
        cross = (n + so + we + e + 2) >> 2
        diag = (s[:-2, :-2] + s[:-2, 2:] + s[2:, :-2] + s[2:, 2:] + 2) >> 2
        hor, ver = (we + e + 1) >> 1, (n + so + 1) >> 1
        rr = self.r_row
        r = torch.where(self.rb, torch.where(rr, c, diag), torch.where(rr, hor, ver))
        g = torch.where(self.rb, cross, c)
        b = torch.where(self.rb, torch.where(rr, diag, c), torch.where(rr, ver, hor))
        inner = torch.stack([r, g, b], -1).to(torch.uint8)
        return inner.index_select(0, self.rows).index_select(1, self.cols)


def make_surfaces(clip, clip_frames):
    """clip_frames 8-bit mosaics (pitched), RAW10 buffers of their codes x 4, and the demosaiced RGB frames."""
    m8, m10, rgb = [], [], []
    for i in range(clip_frames):
        mosaic = rggb(cv2.resize(clip[(7 * i) % len(clip)], (W, H)))
        t = torch.zeros((H, PITCH8), dtype=torch.uint8, device="cuda")
        t[:, :W] = torch.from_numpy(mosaic).cuda()
        m8.append(t[:, :W])
        m10.append(torch.from_numpy(image_ops.mipi_pack(mosaic.astype(np.uint16) * 4, 10, PITCH10)).cuda())
        rgb.append(torch.from_numpy(image_ops.bayer_to_rgb(mosaic, "RGGB", 8)).cuda())
    return m8, m10, rgb


def frames(surfaces, demosaic, arm, num_streams, t):
    m8, m10, rgb = surfaces
    idx = [(3 * s + t) % len(m8) for s in range(num_streams)]
    if arm == "bayer8":
        return [fb.BayerFrame(m8[i]) for i in idx]
    if arm == "raw10":
        return [fb.BayerFrame.raw10(m10[i][:, :W * 5 // 4], W) for i in idx]
    if arm == "torch_demosaic":
        return [demosaic(m8[i]) for i in idx]
    return [rgb[i] for i in idx]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="8x4,8x32", help="streams x targets per stream")
    ap.add_argument("--updates", type=int, default=300, help="timed updates per arm")
    ap.add_argument("--block", type=int, default=50, help="updates per arm before switching to the next arm")
    ap.add_argument("--clip-frames", type=int, default=12, help="1080p frames kept on the device per layout")
    ap.add_argument("--step-repeats", type=int, default=100, help="graph replays timed with CUDA events per arm")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_bayer.py measures on a CUDA device; none is available")
    clip = read_video_rgb(os.path.join(ROOT, "tests", "golden", "test.mp4"))
    surfaces = make_surfaces(clip, args.clip_frames)
    demosaic = TorchDemosaic(torch.device("cuda"))
    if not torch.equal(demosaic(surfaces[0][0]), surfaces[2][0]):
        raise SystemExit("the torch demosaic differs from image_ops.bayer_to_rgb")
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
            trk.initialize(frames(surfaces, demosaic, arm, F, 0), rects, streams)
            for t in range(1, 1 + WARMUP):
                trk.update(frames(surfaces, demosaic, arm, F, t))
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
                    fr = frames(surfaces, demosaic, arm, F, 1 + WARMUP + done[arm] + j)
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
            rgbs = [demosaic(surfaces[0][(3 * s + r) % len(surfaces[0])]) for s in range(F)]
        b.record()
        torch.cuda.synchronize()
        row["torch_demosaic"]["demosaic_device_ms_per_update"] = a.elapsed_time(b) / args.step_repeats
        results.append(row)
        del trackers, held, rgbs
    print(json.dumps({"metric": "FEARMultiTracker on 1920x1080 Bayer streams in device memory: read in place (8-bit, "
                                "RAW10), demosaiced with torch first, and resident RGB", "card":
                      card_info(torch.cuda.current_device()), "timed_updates_per_arm": args.updates,
                      "results": results}))


if __name__ == "__main__":
    main()
