"""GPU: the persistent 1x1-conv GEMM (pw_tc_kernel) at every batch where its tile schedule changes.

The kernel runs min(tiles, SMs) CTAs; CTA c walks tiles c, c + G, c + 2G, ... and its producer streams the CTA's whole
chunk sequence through a ring of up to MAX_STAGES stages, across tile boundaries.  For each launch class of the step
the batches below, derived from the device's SM count, give some CTA exactly one tile, two tiles, an odd count >= 3,
enough chunks that every ring stage's parity wraps (within a tile where the class has more chunks than stages, and
across at least two tile boundaries), and the same with T mod G != 0.  Each case runs `tests/pw_schedule_check.py`
on all its batches in one process: backbone, head intermediates, maps and FearBox records of every frame bit-identical
to the frame's B = 1 result on a poisoned workspace, and B = 1 within the fp64-oracle bars.  B = 256 is also run.
"""
import json
import math
import os
import subprocess
import sys

import pytest

from tests import schedule_plan as sp

HERE = os.path.dirname(os.path.abspath(__file__))
MAX_STAGES = 4                  # kPwMaxStages of csrc/kernels_tc.cuh
WRAP_CHUNKS = 3 * MAX_STAGES    # every stage completes phases 0, 1, 0
CASES = ["one", "two", "odd", "wrap", "wrap_partial"]

# launch class: (a layer of the flagship step in that class, output pixels per frame, K, N) at 256 x 256 search crops
PW_CLASSES = {
    "plain_k_tail": ("xif3_0.pwl", 32 * 32, 144, 32),
    "plain": ("xif4_0.pwl", 16 * 16, 192, 64),
    "dw3_map32": ("xif3_3.dw+pwl", 32 * 32, 192, 32),
    "dw5_map32": ("xif3_1.dw+pwl", 32 * 32, 96, 32),
    "dw5_map16": ("xif4_1.dw+pwl", 16 * 16, 192, 64),
    "head_sepconv_nt128": ("cls_encode dw+pw", 16 * 16, 256, 256),
    "neck_nt128": ("neck", 16 * 16, 112, 256),
}


def tiles_and_chunks(pixels, K, N):
    """Tiles per frame and K chunks of one launch (launch_pw / launch_pw_dw: 128-row tiles, pw_tile_n columns)."""
    nt = sp._pw_tile_n(N)
    return pixels // 128 * -(-((N + 15) & ~15) // nt), -(-K // 32)


def pw_schedule_batches(num_sms, tiles_per_frame, chunks):
    """Batches whose tile counts T = B * tiles_per_frame give, on num_sms persistent CTAs, a CTA with: one tile
    (T < G), two tiles, an odd count >= 3, at least max(3, WRAP_CHUNKS / chunks) tiles with T mod G == 0, and one more
    frame (T mod G != 0).  Returns {case name: B}."""
    G, t = num_sms, tiles_per_frame
    assert 0 < t < G, "every case needs more SMs than tiles per frame"
    most = lambda B: -(-B * t // G)  # tiles of the busiest CTA
    one = (G - 1) // t
    two = next(B for B in range(1, G + 1) if most(B) == 2)
    odd = next(B for B in range(two, 4 * G) if most(B) >= 3 and most(B) % 2 == 1)
    need = max(3, -(-WRAP_CHUNKS // chunks))
    step = G // math.gcd(G, t)  # T is a multiple of G exactly when B is a multiple of step
    even = step * max(1, -(-need * G // (step * t)))
    return {"one": one, "two": two, "odd": odd, "wrap": even, "wrap_partial": even + 1}


def case_batches(num_sms, case):
    return sorted({pw_schedule_batches(num_sms, *tiles_and_chunks(*shape))[case] for _, *shape in PW_CLASSES.values()})


def test_batch_picker_cpu():
    names = {ln.name for ln in sp.launches("track_u8", Bz=1)}
    assert {layer for layer, *_ in PW_CLASSES.values()} <= names
    assert pw_schedule_batches(132, 4, 8) == {"one": 32, "two": 34, "odd": 67, "wrap": 99, "wrap_partial": 100}
    for G in (114, 120, 131, 132, 144):
        for layer, *shape in PW_CLASSES.values():
            t, nc = tiles_and_chunks(*shape)
            cases = pw_schedule_batches(G, t, nc)
            most = {k: -(-B * t // G) for k, B in cases.items()}
            assert cases["one"] * t < G and most["one"] == 1, (G, layer)
            assert most["two"] == 2, (G, layer)
            assert most["odd"] >= 3 and most["odd"] % 2 == 1, (G, layer)
            assert cases["wrap"] * t % G == 0 and most["wrap"] >= 3 and most["wrap"] * nc >= WRAP_CHUNKS, (G, layer)
            assert cases["wrap_partial"] * t % G != 0 and most["wrap_partial"] == most["wrap"] + 1, (G, layer)


def _run(batches, out_dir):
    proc = subprocess.run([sys.executable, os.path.join(HERE, "pw_schedule_check.py"), *map(str, batches)],
                          capture_output=True, text=True, timeout=1800)
    with open(os.path.join(out_dir, "pw_schedule_check.log"), "w") as f:
        f.write(proc.stdout + "\n--- stderr ---\n" + proc.stderr)
    lines = [l for l in proc.stdout.splitlines() if l.startswith("PW_SCHEDULE_CHECK ")]
    assert proc.returncode == 0 and lines, f"pw_schedule_check {batches} failed: {proc.stderr[-2000:]}"
    return json.loads(lines[-1][len("PW_SCHEDULE_CHECK "):])


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES + ["b256"])
def test_pw_schedule(case, tmp_path):
    import torch

    G = torch.cuda.get_device_properties(0).multi_processor_count
    batches = [256] if case == "b256" else case_batches(G, case)
    res = _run(batches, str(tmp_path))
    assert res["batches"] == batches and res["runs"] == len(batches)
    assert res["n_failures"] == 0, res["failures"]
