"""GPU: the persistent fused xif2_0 kernel (irf_s2_fused_kernel) at every batch where its tile schedule changes.

The kernel runs min(tiles, SMs) CTAs; CTA c walks tiles c, c + G, c + 2G, ... and its two warpgroups take them in
turn, each refilling its own input-box buffer (one mbarrier per warpgroup).  The batches below are derived from the
device's SM count so that some CTA gets exactly one tile, two tiles, an odd count (the warpgroups end on different
tiles), enough tiles that both mbarriers' parities wrap, and the same with a partial last round.  Each case runs
`tests/tc_check.py irf B` in its own process: bit-identical to the three-kernel path (fuse_irf=0) on the
backbone prefix and on the full features, and within 2e-5 of the fp64 oracle, on search- (256 x 256) and
template-sized (128 x 128) inputs.
"""
import json
import math
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
# xif2_0 maps a 256 x 256 crop's 128 x 128 map to 64 x 64: 8 x 4 output tiles of 8 x 16 pixels
SEARCH_TILES_PER_FRAME = (256 // 4 // 8) * (256 // 4 // 16)
MIN_TILES_FOR_WRAP = 8  # 4 tiles per warpgroup: each of the two box mbarriers completes phases 0, 1, 0, 1


def irf_schedule_batches(num_sms, tiles_per_frame=SEARCH_TILES_PER_FRAME):
    """Batches whose tile counts T = B * tiles_per_frame give, on num_sms persistent CTAs, a CTA with: one tile
    (T < G), two tiles, an odd count >= 3, >= MIN_TILES_FOR_WRAP tiles with T mod G == 0, and one more frame (T mod
    G != 0).  Returns {case name: B}."""
    G, t = num_sms, tiles_per_frame
    assert 0 < t < G, "every case needs more SMs than tiles per frame"
    most = lambda B: -(-B * t // G)  # tiles of the busiest CTA
    one = (G - 1) // t
    two = next(B for B in range(1, G + 1) if most(B) == 2)
    odd = next(B for B in range(two, 4 * G) if most(B) >= 3 and most(B) % 2 == 1)
    step = G // math.gcd(G, t)  # T is a multiple of G exactly when B is a multiple of step
    even = step * max(1, -(-MIN_TILES_FOR_WRAP * G // (step * t)))
    return {"one": one, "two": two, "odd": odd, "wrap": even, "wrap_partial": even + 1}


def test_batch_picker_cpu():
    assert irf_schedule_batches(132) == {"one": 4, "two": 5, "odd": 9, "wrap": 33, "wrap_partial": 34}
    for G in (114, 120, 131, 132, 144):
        for t in (8, 32):
            cases = irf_schedule_batches(G, t)
            most = {k: -(-B * t // G) for k, B in cases.items()}
            assert cases["one"] * t < G and most["one"] == 1
            assert most["two"] == 2
            assert most["odd"] >= 3 and most["odd"] % 2 == 1
            assert cases["wrap"] * t % G == 0 and most["wrap"] >= MIN_TILES_FOR_WRAP
            assert cases["wrap_partial"] * t % G != 0 and most["wrap_partial"] == most["wrap"] + 1


def _run_irf(B, out_dir):
    proc = subprocess.run([sys.executable, os.path.join(HERE, "tc_check.py"), "irf", str(B)], capture_output=True,
                          text=True, timeout=600)
    with open(os.path.join(out_dir, f"tc_check_irf_{B}.log"), "w") as f:
        f.write(proc.stdout + "\n--- stderr ---\n" + proc.stderr)
    lines = [l for l in proc.stdout.splitlines() if l.startswith("TC_CHECK ")]
    assert proc.returncode == 0 and lines, f"tc_check irf {B} failed: {proc.stderr[-2000:]}"
    return json.loads(lines[-1][len("TC_CHECK "):])


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["one", "two", "odd", "wrap", "wrap_partial", "b256"])
def test_fused_irf_schedule(case, tmp_path):
    import torch

    G = torch.cuda.get_device_properties(0).multi_processor_count
    B = 256 if case == "b256" else irf_schedule_batches(G)[case]
    res = _run_irf(B, str(tmp_path))
    for name in ("search", "template"):
        r = res[name]
        assert r["bit_identical"] and r["features_bit_identical"], (B, name, r)
        assert r["vs_oracle"][1] < 2e-5, (B, name, r)
