"""fear_decode_smooth on poisoned memory, in its own process (as tests/poison_check.py, whose Guarded buffers, fills and
Checker it reuses).  Prints one JSON line.

    python tests/poison_smooth_check.py

Maps, prev_size, params and the FearBox array are views into larger allocations with guard bands; each call runs with
everything filled with 0, then fill A, then fill B, and must give bit-identical records, leave every guard band and
input untouched, and agree with FEARTracker._smooth_postprocess.  B is only ever a launch argument, never poisoned.
"""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import feartracker_b200 as fb  # noqa: E402
from feartracker_b200 import _lib  # noqa: E402
from tests.poison_check import Checker, Guarded, stream  # noqa: E402


def main():
    torch.manual_seed(0)
    chk, lib = Checker(), _lib.load()
    g = torch.Generator().manual_seed(606)
    cfg = dict(fb.FEAR_XS_TRACKER_KWARGS, smooth=True)
    trk = fb.FEARTracker(None, cuda_id=0, **cfg)
    window = np.asarray(trk.window, dtype=np.float64).reshape(256)
    params = torch.from_numpy(np.concatenate([[cfg["penalty_k"], cfg["window_influence"], cfg["lr"]], window]))
    mismatches = 0
    for B in (1, 7, 4096):
        cls = 3.0 * torch.randn(B, 1, 16, 16, generator=g)
        cls[::5] = torch.randint(-4, 5, (len(cls[::5]), 1, 16, 16), generator=g).float() / 2  # ties
        reg = 10.0 + 60.0 * torch.rand(B, 4, 16, 16, generator=g)
        prev = 20.0 + 100.0 * torch.rand(B, 2, generator=g, dtype=torch.float64)
        gr, gc = Guarded.of(reg, 1024), Guarded.of(cls, 256)
        gp, gq = Guarded.of(prev, 2), Guarded.of(params, 259)
        gbox = Guarded.out((B, _lib.BOX_DTYPE.itemsize), torch.uint8, 48)
        rec = chk.run(f"decode_smooth B={B}", lambda: _lib.check(
            lib.fear_decode_smooth(gr.ptr(), gc.ptr(), B, gp.ptr(), gq.ptr(), gbox.ptr(), stream()),
            "fear_decode_smooth"), [gr, gc, gp, gq], [gbox])[0]
        rec = rec.cpu().numpy().view(_lib.BOX_DTYPE).reshape(-1)
        score = cls.cuda().sigmoid().cpu().numpy()
        for i in range(min(B, 64)):
            trk.tracking_state.prev_size = prev[i].numpy()
            box, sc = trk._smooth_postprocess(reg[i].numpy().astype(np.float64), score[i, 0])
            got = np.array([rec["x"][i], rec["y"][i], rec["w"][i], rec["h"][i]])
            if not (np.allclose(got, box, rtol=1e-12, atol=0) and np.float32(rec["score"][i]) == np.float32(sc)
                    and rec["flat"][i] == rec["row"][i] * 16 + rec["col"][i]):
                mismatches += 1
        if mismatches:
            chk.fail(f"decode_smooth B={B}: {mismatches} records differ from _smooth_postprocess")
    res = chk.report()
    res["host_mismatches"] = mismatches
    print("POISON_CHECK " + json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
