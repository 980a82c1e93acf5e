#!/usr/bin/env python
"""FEARMultiTracker on rotated and mirrored 1080p streams (phone video's display rotation, cameras mounted upside down
or mirrored), oriented inside the crop, against the torch turn it replaces.  Two sources:
  nv12   pitched NV12 decoder surfaces (YUV420Frame.nv12), converted inside the crop
  rgb    resident uint8 (1080, 1920, 3) RGB tensors
and for each the arms:
  plain      the frames as they are (no orientation: the yardstick)
  o0 .. o5   fb.Oriented(frame) with code 0 (no turn, the oriented entry points), 1 (90 degrees clockwise), 2 (180) and
             5 (mirrored, then 90): the kernels map each display pixel to its stored pixel
  torch      what a user had to do before Oriented, for code 1: convert to an RGB tensor with torch (nv12: the integer
             BT.601 conversion of tools/bench_yuv_frames.py), torch.rot90(k=-1) and .contiguous(), then pass the tensor
             (checked equal to image_ops.orient of the frame the tracker sees before timing)
The demo clip (tests/golden/test.mp4, 480x256) is resized to 1920x1080 with cv2.resize; stream s reads clip frame
(3 s + t) mod --clip-frames at update t.  Each stream holds the jittered golden boxes of bench_multi.py, scaled to the
display size.  For F streams x k targets per stream, each arm reports:
  host_ms_per_update   wall time of one update(), frame wrapping (and for torch the turn) included
  device_ms_per_step   CUDA events around --step-repeats replays of the captured step
The arms run in the same process on the same targets, alternated in blocks of --block updates.  Then the crop kernel
alone: CUDA events around --crop-repeats launches of fear_crop_targets_oriented_u8 per code on the NV12 and RGB tables
of the 8 x 32 targets, against the plain crop entry point.  One JSON line, with the card name, power limit and SM clock
read by nvidia-smi right after the timed runs.

    python tools/bench_orientation.py [--configs 8x4,8x32] [--updates 300] [--block 50]
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
from bench_yuv_frames import nv12_to_rgb  # noqa: E402
from feartracker_b200 import _lib, image_ops  # noqa: E402
from feartracker_b200 import multi_tracker as mt  # noqa: E402
from oracle.fear_oracle import read_video_rgb  # noqa: E402

W, H, PITCH = 1920, 1080, 2048
WARMUP = 3  # eager warm-up + capture + one replay
CODES = {"o0": 0, "o1": 1, "o2": 2, "o5": 5}
ARMS = ("plain",) + tuple(CODES) + ("torch",)
TORCH_CODE = 1


def make_surfaces(clip, clip_frames):
    """Per clip frame: the RGB tensor and a pitched NV12 surface of the resized clip, on the device."""
    rgb, nv12 = [], []
    for i in range(clip_frames):
        frame = cv2.resize(clip[(7 * i) % len(clip)], (W, H))
        rgb.append(torch.from_numpy(frame).cuda())
        i420 = cv2.cvtColor(frame, cv2.COLOR_RGB2YUV_I420)
        u, v = i420[H:H + H // 4].reshape(H // 2, W // 2), i420[H + H // 4:].reshape(H // 2, W // 2)
        surf = np.zeros((H * 3 // 2, PITCH), np.uint8)
        surf[:, :W] = np.concatenate([i420[:H], np.stack([u, v], -1).reshape(H // 2, W)])
        nv12.append(torch.from_numpy(surf).cuda()[:, :W])
    return {"rgb": rgb, "nv12": nv12}


def stored(source, t):
    return fb.YUV420Frame.nv12(t) if source == "nv12" else t


def torch_turn(source, t):
    rgb = nv12_to_rgb(t) if source == "nv12" else t
    return torch.rot90(rgb, k=-1, dims=(0, 1)).contiguous()  # 90 degrees clockwise: image_ops.orient code 1


def frames(s, source, arm, num_streams, t):
    idx = [(3 * k + t) % len(s[source]) for k in range(num_streams)]
    if arm == "plain":
        return [stored(source, s[source][i]) for i in idx]
    if arm == "torch":
        return [torch_turn(source, s[source][i]) for i in idx]
    c = CODES[arm]
    return [fb.Oriented(stored(source, s[source][i]), 90 * (c & 3), bool(c & 4)) for i in idx]


def seen(source, t):
    if source == "rgb":
        return t.cpu().numpy()
    h = 2 * t.shape[0] // 3
    a = t.cpu().numpy()
    return image_ops.yuv_to_rgb(a[:h], a[h:, 0::2], a[h:, 1::2])


def crop_kernel_ms(trk, table, num_frames, n, codes, repeats):
    """ms per launch of the oriented crop (codes given) or the table's plain crop (codes None) on the tracker's
    current table and targets, from CUDA events over ``repeats`` launches."""
    lib, b = _lib.load(), trk._buf
    size = int(trk.tracking_config["instance_size"])
    s = torch.cuda.current_stream().cuda_stream
    d_codes = None if codes is None else torch.full((num_frames,), codes, dtype=torch.int32, device="cuda")

    def launch():
        if d_codes is None:
            fn = mt.ENTRY_POINTS[table][1]
            _lib.check(getattr(lib, fn)(b[table].data_ptr(), num_frames, b["state"].data_ptr(), n, 2.0, size,
                                        b["crops"].data_ptr(), s), fn)
        else:
            _lib.check(lib.fear_crop_targets_oriented_u8(_lib.ORIENT_TABLES[table], b[table].data_ptr(),
                                                         d_codes.data_ptr(), num_frames, b["state"].data_ptr(), n, 2.0,
                                                         size, b["crops"].data_ptr(), s), "oriented crop")

    for _ in range(5):
        launch()
    a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(repeats):
        launch()
    e.record()
    torch.cuda.synchronize()
    return a.elapsed_time(e) / repeats


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="8x4,8x32", help="streams x targets per stream")
    ap.add_argument("--updates", type=int, default=300, help="timed updates per arm")
    ap.add_argument("--block", type=int, default=50, help="updates per arm before switching to the next arm")
    ap.add_argument("--clip-frames", type=int, default=12, help="1080p frames kept on the device per source")
    ap.add_argument("--step-repeats", type=int, default=100, help="graph replays timed with CUDA events per arm")
    ap.add_argument("--crop-repeats", type=int, default=200, help="crop launches timed with CUDA events per code")
    ap.add_argument("--sources", default="nv12,rgb")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_orientation.py measures on a CUDA device; none is available")
    clip = read_video_rgb(os.path.join(ROOT, "tests", "golden", "test.mp4"))
    surfaces = make_surfaces(clip, args.clip_frames)
    sources = args.sources.split(",")
    for source in sources:
        t = surfaces[source][0]
        if not np.array_equal(torch_turn(source, t).cpu().numpy(), image_ops.orient(seen(source, t), TORCH_CODE)):
            raise SystemExit(f"the torch turn of {source} differs from image_ops.orient")
    net = fb.FEARNet(**fb.FEAR_XS_MODEL_KWARGS)
    net.load_state_dict(load_state(), strict=True)
    net = net.cuda().eval()
    cfg = fb.FEAR_XS_TRACKER_KWARGS
    results, crop_rows = [], []
    for config in args.configs.split(","):
        F, k = (int(v) for v in config.split("x"))
        n = F * k
        streams = np.repeat(np.arange(F), k)
        for source in sources:
            trackers, rects = {}, {}
            for arm in ARMS:
                turned = arm == "torch" or (arm in CODES and CODES[arm] & 1)
                dw, dh = (H, W) if turned else (W, H)
                rects[arm] = np.concatenate([np.rint(jittered_boxes(k, seed=s) * np.array([dw / 480, dh / 256] * 2))
                                             for s in range(F)])
                trackers[arm] = fb.FEARMultiTracker(net, cuda_id=0, max_targets=n, **cfg)
            row = {"source": source, "streams": F, "targets_per_stream": k, "N": n}
            for arm, trk in trackers.items():
                trk.initialize(frames(surfaces, source, arm, F, 0), rects[arm], streams)
                for t in range(1, 1 + WARMUP):
                    trk.update(frames(surfaces, source, arm, F, t))
            spent, done, held, order = {a: 0.0 for a in ARMS}, {a: 0 for a in ARMS}, {}, list(ARMS)
            while min(done.values()) < args.updates:
                for arm in order:
                    m = min(args.block, args.updates - done[arm])
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    for j in range(m):
                        fr = frames(surfaces, source, arm, F, 1 + WARMUP + done[arm] + j)
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
                row[arm] = dict(table=trk._graph_key[2], oriented=trk._graph_key[5], host_ms_per_update=host_ms,
                                target_frames_per_s=n * 1e3 / host_ms,
                                device_ms_per_step=a.elapsed_time(b) / args.step_repeats)
            if config == args.configs.split(",")[-1]:
                trk = trackers["o1"]
                table = trk._graph_key[2]
                crop = {"source": source, "N": n, "table": table,
                        "plain_ms": crop_kernel_ms(trk, table, F, n, None, args.crop_repeats)}
                for c in range(8):
                    crop[f"code{c}_ms"] = crop_kernel_ms(trk, table, F, n, c, args.crop_repeats)
                crop_rows.append(crop)
            results.append(row)
            del trackers, held
    print(json.dumps({"metric": "FEARMultiTracker on rotated / mirrored 1920x1080 streams: Oriented (codes 0, 1, 2, 5) "
                                "read in place, the torch turn (convert + rot90 + contiguous), and plain frames",
                      "card": card_info(torch.cuda.current_device()), "timed_updates_per_arm": args.updates,
                      "results": results, "crop_kernel": crop_rows}))


if __name__ == "__main__":
    main()
