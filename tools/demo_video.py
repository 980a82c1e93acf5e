#!/usr/bin/env python
"""H100 counterpart of the reference's demo_video.py (reference demo_video.py:14-62): track one object through a
video with FEARTracker and write the annotated clip.  hydra / fire / imageio are not needed: the two YAML files the
demo composes (model/fear.yaml, tracker/siam_tracker.yaml) are read directly when a reference config tree is given,
otherwise the same values built into feartracker_b200 are used; video IO goes through cv2.

    python tools/demo_video.py --video tests/golden/test.mp4 --weights FEAR-XS-NoEmbs.ckpt \
        --bbox 163 53 45 174 --out outputs/test.mp4 [--config-dir /path/to/model_training/config]
"""
import argparse
import os
import sys

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import feartracker_b200 as fb  # noqa: E402


def load_configs(config_dir):
    model, tracker = dict(fb.FEAR_XS_MODEL_KWARGS), dict(fb.FEAR_XS_TRACKER_KWARGS)
    if config_dir:
        import yaml

        with open(os.path.join(config_dir, "model", "fear.yaml")) as f:
            model = {k: v for k, v in yaml.safe_load(f).items() if k != "_target_"}
        with open(os.path.join(config_dir, "tracker", "siam_tracker.yaml")) as f:
            tracker = {k: v for k, v in yaml.safe_load(f).items() if k != "_target_"}
        for k, v in tracker.items():  # the only interpolation the demo needs: ${model.stride}
            if isinstance(v, str) and v.startswith("${model."):
                tracker[k] = model[v[len("${model."):-1]]
    return model, tracker


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--video", default=os.path.join(ROOT, "tests", "golden", "test.mp4"))
    ap.add_argument("--weights", default=None, help="Lightning checkpoint (default: the hot-path fixture weights)")
    ap.add_argument("--bbox", type=int, nargs=4, default=[163, 53, 45, 174])
    ap.add_argument("--out", default=os.path.join(ROOT, "outputs", "test.mp4"))
    ap.add_argument("--config-dir", default=None)
    args = ap.parse_args()

    model_cfg, tracker_cfg = load_configs(args.config_dir)
    net = fb.FEARNet(**model_cfg)
    if args.weights:
        fb.load_from_lighting(net, args.weights)
    else:
        from bench import load_state

        net.load_state_dict(load_state(), strict=True)
    tracker = fb.FEARTracker(net.cuda().eval(), cuda_id=0, **tracker_cfg)

    cap = cv2.VideoCapture(args.video)
    fps = cap.get(cv2.CAP_PROP_FPS) or 25.0
    frames = []
    while True:
        ok, f = cap.read()
        if not ok:
            break
        frames.append(cv2.cvtColor(f, cv2.COLOR_BGR2RGB))
    boxes = [np.array(args.bbox)]
    tracker.initialize(frames[0], boxes[0])
    for frame in frames[1:]:
        boxes.append(tracker.update(frame)["bbox"])
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    h, w = frames[0].shape[:2]
    out = cv2.VideoWriter(args.out, cv2.VideoWriter_fourcc(*"mp4v"), fps, (w, h))
    for frame, (x, y, bw, bh) in zip(frames, boxes):
        img = cv2.cvtColor(frame, cv2.COLOR_RGB2BGR).copy()
        cv2.rectangle(img, (int(x), int(y)), (int(x + bw), int(y + bh)), (0, 255, 0), 5)
        out.write(img)
    out.release()
    print(f"tracked {len(frames) - 1} frames -> {args.out}; last box {list(map(int, boxes[-1]))}")


if __name__ == "__main__":
    main()
