"""The oriented crop and advance entry points on poisoned memory, in their own process (as tests/poison_check.py, whose
guarded buffers, fills and checker it reuses).  Prints one JSON line.

    python tests/poison_orientation_check.py

For each frame table, two frames and their records: the table, the orientation codes, the decoded boxes, the FearTarget
rows and the crops live in guarded allocations whose guard bands (and the outputs) are filled with 0, fill A and fill B
in turn.  fear_crop_targets_oriented_u8 then fear_advance_targets_oriented run on every code pair, with a null code
array, and with codes outside [0, 7].  Every result must be the same under every fill and equal the plain view entry
points on image_ops.orient of the frame the table's kernels see; no guard band, input or FearTarget field the calls do
not own may change.
"""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from feartracker_b200 import _lib, image_ops  # noqa: E402
from tests.poison_check import Checker, Guarded, stream  # noqa: E402
from tests.test_gpu_orientation import (TABLE_FRAMES, boxes_for, seen, table_of, targets_for,  # noqa: E402
                                        view_step)

SIZE, OFFSET = 64, 2.0


def group_table(chk, name, rng):
    lib = _lib.load()
    a = rng.integers(0, 256, (37, 53, 3), dtype=np.uint8)
    b = rng.integers(0, 256, (64, 90, 3), dtype=np.uint8)
    frames = TABLE_FRAMES[name](a, b)
    rgbs = [seen(f) for f in frames]
    table = table_of(frames, name)
    if name == "mono":  # the code ranges the crop reads, written once into the table's data
        _lib.check(lib.fear_frame_range_mono(table.data_ptr(), len(frames), None), "fear_frame_range_mono")
        torch.cuda.synchronize()
    gtable = Guarded(table.numel(), words=False, data=table)
    for codes in [(c, (5 * c + 2) % 8) for c in range(8)] + [None, (8, 3), (-1, 9)]:
        known = [0 if codes is None else c for c in codes or (0, 0)]
        shapes = [image_ops.orient(r, c if 0 <= c <= 7 else 0).shape[:2] for r, c in zip(rgbs, known)]
        targets = targets_for(shapes)
        n = targets.shape[0]
        gt = Guarded.of(targets)
        gboxes = Guarded.of(boxes_for(n, 11).view(torch.int32))
        gcrops = Guarded(n * SIZE * SIZE * 3, frame=SIZE * SIZE * 3, words=False)
        gcrops.dtype, gcrops.shape = torch.uint8, (n, SIZE, SIZE, 3)
        inputs = [gtable, gboxes]
        gcodes = None
        if codes is not None:
            gcodes = Guarded.of(torch.tensor(codes, dtype=torch.int32))
            inputs.append(gcodes)
        t = _lib.ORIENT_TABLES[name]

        def call():
            cp = None if gcodes is None else gcodes.ptr()
            _lib.check(lib.fear_crop_targets_oriented_u8(t, gtable.ptr(), cp, 2, gt.ptr(), n, OFFSET, SIZE,
                                                         gcrops.ptr(), stream()), "fear_crop_targets_oriented_u8")
            _lib.check(lib.fear_advance_targets_oriented(gboxes.ptr(), t, gtable.ptr(), cp, 2, gt.ptr(), n, 256,
                                                         stream()), "fear_advance_targets_oriented")

        tag = f"{name} codes {codes}"
        crops, rows = chk.run(tag, call, inputs, [gcrops], owned={gt: (n, slice(1, 9))})
        crops, rows = crops.cpu().numpy(), rows.cpu().numpy()
        if all(0 <= c <= 7 for c in known):
            want = view_step([np.ascontiguousarray(image_ops.orient(r, c)) for r, c in zip(rgbs, known)], targets,
                             gboxes.data.view(torch.uint8), OFFSET, SIZE)
            if not (np.array_equal(crops, want[0]) and np.array_equal(rows, want[1])):
                chk.fail(f"{tag}: differs from the view entry points on the oriented frames")
        else:
            first = targets.cpu().numpy()[:, 0] == 0
            if not (crops[first] == np.array([17, 99, 201], np.uint8)).all():
                chk.fail(f"{tag}: an unreadable code does not give a padding crop")
            if not np.array_equal(rows[first][:, 1:5], targets.cpu().numpy()[first][:, 1:5]):
                chk.fail(f"{tag}: an unreadable code moved its box")


def main():
    torch.manual_seed(0)
    chk, rng = Checker(), np.random.default_rng(31)
    for name in TABLE_FRAMES:
        group_table(chk, name, rng)
    print("POISON_CHECK " + json.dumps(chk.report()), flush=True)


if __name__ == "__main__":
    main()
