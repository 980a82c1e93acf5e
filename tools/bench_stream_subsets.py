#!/usr/bin/env python
"""FEARMultiTracker on 1080p streams that do not tick together: half of the streams have a new frame at each update,
the halves alternating.  Arms:
  list_all       list updates with a new frame of every stream (every stream ticks every update): the yardstick
  mapping_half   mapping updates {stream id: frame} of half of the streams, halves alternating: only their targets are
                 stepped (fear_gather_targets -> step on M = N / 2 -> fear_scatter_targets)
  list_repeat    list updates of every stream where the other half gets its previous frame again: what a user had to
                 do before mappings (the repeated frames carry no new information, and move the boxes)
each on NV12 surfaces (YUV420Frame.nv12, the "yuv" table) and on uint8 RGB tensors on the device (the "views" table).
The demo clip (tests/golden/test.mp4, 480x256) is resized to 1920x1080 with cv2.resize; --clip-frames of its frames
are kept on the device in both forms, and stream s reads clip frame (3 s + t) mod --clip-frames at its tick t.  Each
stream holds the jittered golden boxes of bench_multi.py, scaled to 1080p.  For F streams x k targets per stream,
each arm reports:
  host_ms_per_update       wall time of one update()
  device_ms_per_step       CUDA events around --step-repeats replays of the captured step graph
  new_target_frames_per_s  targets stepped on a new frame per update / host_ms_per_update (N for list_all, N / 2 for
                           the other two arms)
The arms run in the same process, alternated in blocks of --block updates.  Then fear_gather_targets +
fear_scatter_targets alone, at M = 32 and M = 256 of 256 target rows: CUDA events around --kernel-repeats launch pairs.
One JSON line, with the card name, power limit and SM clock read by nvidia-smi right after the timed runs.

    python tools/bench_stream_subsets.py [--configs 8x4,8x32] [--updates 300] [--block 50]
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
from feartracker_b200 import _lib  # noqa: E402
from oracle.fear_oracle import read_video_rgb  # noqa: E402

W, H = 1920, 1080
WARMUP = 4  # eager warm-up + capture + replays of both halves
KINDS = ("nv12", "tensor")
ARMS = ("list_all", "mapping_half", "list_repeat")


def make_surfaces(clip, clip_frames):
    """Per clip frame: the RGB tensor and its NV12 surface (cv2's I420 with the chroma interleaved) on the device."""
    s = {"tensor": [], "nv12": []}
    for i in range(clip_frames):
        rgb = cv2.resize(clip[(7 * i) % len(clip)], (W, H))
        s["tensor"].append(torch.from_numpy(rgb).cuda())
        i420 = cv2.cvtColor(rgb, cv2.COLOR_RGB2YUV_I420).reshape(-1)
        q = W * H // 4
        uv = np.stack([i420[W * H:W * H + q], i420[W * H + q:]], -1).reshape(H // 2, W)
        s["nv12"].append(torch.from_numpy(np.concatenate([i420[:W * H].reshape(H, W), uv])).cuda())
    return s


def frame(s, kind, stream, tick):
    t = s[kind][(3 * stream + tick) % len(s[kind])]
    return fb.YUV420Frame.nv12(t) if kind == "nv12" else t


def update_args(s, kind, arm, num_streams, u):
    """The frames of update u: the ticking half is u % 2; a stream's tick counts its own new frames."""
    half = [j for j in range(num_streams) if j % 2 == u % 2]
    if arm == "list_all":
        return [frame(s, kind, j, u) for j in range(num_streams)]
    if arm == "mapping_half":
        return {j: frame(s, kind, j, u // 2) for j in half}
    # list_repeat: the other half gets the frame it had at its own last tick
    return [frame(s, kind, j, u // 2 if j % 2 == u % 2 else (u - 1) // 2) for j in range(num_streams)]


def step_graph(trk, arm):
    if arm == "mapping_half":
        graphs = [e["graph"] for e in trk._subset_graphs.values() if e["graph"] is not None]
        assert len(graphs) == 1, "both halves share one captured subset step"
        return graphs[0]
    return trk._graph


def time_gather_scatter(lib, repeats):
    """ms per fear_gather_targets + fear_scatter_targets pair at M = 32 and M = 256 of 256 rows."""
    n = 256
    targets = torch.zeros((n, _lib.TARGET_INTS), dtype=torch.int32, device="cuda")
    zf = torch.randn((n, 256, 8, 8), device="cuda")
    step_t, step_z = torch.empty_like(targets), torch.empty_like(zf)
    out = {}
    for m in (32, 256):
        rows = torch.from_numpy(np.random.default_rng(m).permutation(n)[:m].astype(np.int32))
        select = torch.stack([rows, torch.arange(m, dtype=torch.int32) % 8], 1).cuda()
        s = torch.cuda.current_stream().cuda_stream

        def pair():
            _lib.check(lib.fear_gather_targets(targets.data_ptr(), n, zf.data_ptr(), select.data_ptr(), m,
                                               step_t.data_ptr(), step_z.data_ptr(), s), "fear_gather_targets")
            _lib.check(lib.fear_scatter_targets(step_t.data_ptr(), select.data_ptr(), m, targets.data_ptr(), n, s),
                       "fear_scatter_targets")

        for _ in range(10):
            pair()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(repeats):
            pair()
        b.record()
        torch.cuda.synchronize()
        ms = a.elapsed_time(b) / repeats
        out[f"M{m}"] = dict(ms_per_gather_scatter=ms, template_bytes_moved=2 * m * 65536,
                            template_GB_per_s=2 * m * 65536 / (ms * 1e-3) / 1e9)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="8x4,8x32", help="streams x targets per stream")
    ap.add_argument("--updates", type=int, default=300, help="timed updates per arm")
    ap.add_argument("--block", type=int, default=50, help="updates per arm before switching to the next arm")
    ap.add_argument("--clip-frames", type=int, default=12, help="1080p frames kept on the device per form")
    ap.add_argument("--step-repeats", type=int, default=100, help="graph replays timed with CUDA events per arm")
    ap.add_argument("--kernel-repeats", type=int, default=2000, help="gather + scatter pairs timed per M")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_stream_subsets.py measures on a CUDA device; none is available")
    clip = read_video_rgb(os.path.join(ROOT, "tests", "golden", "test.mp4"))
    surfaces = make_surfaces(clip, args.clip_frames)
    torch.cuda.synchronize()
    net = fb.FEARNet(**fb.FEAR_XS_MODEL_KWARGS)
    net.load_state_dict(load_state(), strict=True)
    net = net.cuda().eval()
    cfg = fb.FEAR_XS_TRACKER_KWARGS
    scale = np.array([W / 480, H / 256, W / 480, H / 256])
    names = [(k, a) for k in KINDS for a in ARMS]
    results = []
    for config in args.configs.split(","):
        F, k = (int(v) for v in config.split("x"))
        n = F * k
        rects = np.concatenate([np.rint(jittered_boxes(k, seed=s) * scale) for s in range(F)])
        streams = np.repeat(np.arange(F), k)
        trackers = {key: fb.FEARMultiTracker(net, cuda_id=0, max_targets=n, **cfg) for key in names}
        row = {"streams": F, "targets_per_stream": k, "N": n}
        for (kind, arm), trk in trackers.items():
            trk.initialize([frame(surfaces, kind, j, 0) for j in range(F)], rects, streams)
            for u in range(1, 1 + WARMUP):
                trk.update(update_args(surfaces, kind, arm, F, u))
        spent = {key: 0.0 for key in names}
        done = {key: 0 for key in names}
        order = list(names)
        while min(done.values()) < args.updates:
            for key in order:
                m = min(args.block, args.updates - done[key])
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for j in range(m):
                    trackers[key].update(update_args(surfaces, *key, F, 1 + WARMUP + done[key] + j))
                spent[key] += time.perf_counter() - t0
                done[key] += m
            order.reverse()
        for (kind, arm), trk in trackers.items():
            g = step_graph(trk, arm)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.step_repeats):
                g.replay()
            b.record()
            torch.cuda.synchronize()
            host_ms = spent[(kind, arm)] * 1e3 / done[(kind, arm)]
            new = n if arm == "list_all" else n // 2
            row[f"{kind}_{arm}"] = dict(host_ms_per_update=host_ms, device_ms_per_step=a.elapsed_time(b) / args.step_repeats,
                                        new_target_frames_per_s=new * 1e3 / host_ms)
        results.append(row)
        del trackers
    kernels = time_gather_scatter(_lib.load(), args.kernel_repeats)
    print(json.dumps({"metric": "FEARMultiTracker on 1920x1080 streams ticking in alternating halves: list updates of "
                                "every stream, mapping updates of the ticking half, and list updates repeating the other "
                                "half's previous frame", "card": card_info(torch.cuda.current_device()),
                      "timed_updates_per_arm": args.updates, "results": results, "gather_scatter": kernels}))


if __name__ == "__main__":
    main()
