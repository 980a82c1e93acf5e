"""GPU: search crops of every side S in {16, 32, ..., 256} (score maps of side s = S / 16) through FEARNet, the sized C
entry points, the decode and both trackers, against the fp64 oracle and the host.  Each case runs in its own process
(tests/search_size_check.py) so a device trap in one cannot poison the others."""
import json
import os
import subprocess
import sys

import pytest

from tests.helpers import TOL

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
SIZES = list(range(16, 257, 16))
OUT = None  # log directory of this run (set by _log_dir)


@pytest.fixture(scope="module", autouse=True)
def _log_dir(tmp_path_factory):
    global OUT
    OUT = str(tmp_path_factory.mktemp("search_size_check"))


def _run(*args, timeout=900):
    proc = subprocess.run([sys.executable, os.path.join(HERE, "search_size_check.py"), *map(str, args)],
                          capture_output=True, text=True, timeout=timeout)
    with open(os.path.join(OUT, "search_size_check_" + "_".join(map(str, args)) + ".log"), "w") as f:
        f.write(proc.stdout + "\n--- stderr ---\n" + proc.stderr)
    lines = [l for l in proc.stdout.splitlines() if l.startswith("SEARCH_SIZE_CHECK ")]
    assert proc.returncode == 0 and lines, f"search_size_check {args} failed: {proc.stderr[-3000:]}"
    return json.loads(lines[-1][len("SEARCH_SIZE_CHECK "):])


# The cls map holds logits that cross zero.  Its element-wise error (tests/helpers.py map_errors) divides by
# max(|b|, 1e-3 * ||b||inf), so at a cell near zero it is 1e3 times the inf-norm error there, at most 1e3 * e2.  The
# inf-norm error of the cls map is 0.5-6.4e-6 at every S (3.8e-6 at 256); which cell carries it decides e1.  On this
# file's seeded inputs (the kernels are deterministic) e1 of the cls map stays within TOL except at the four sides
# below, where a near-zero cell carries it.  Measured per S, worst over track / forward / connect_model, B and Bz:
#   S:   16     32     48     64     80     96     112    128    144    160    176    192    208    224    240    256
#   e1:  5e-7   1.3e-6 1.3e-6 1.7e-6 1.6e-6 3.7e-6 5.8e-6 6.5e-6 1.8e-5 4.6e-4 2.4e-3 2.8e-3 2.2e-3 1.3e-3 5.7e-4 7.7e-4
#   e2:  5e-7   1.3e-6 1.3e-6 1.7e-6 1.5e-6 2.4e-6 3.8e-6 4.0e-6 5.0e-6 6.4e-6 4.6e-6 4.4e-6 3.1e-6 3.7e-6 3.3e-6 3.8e-6
# At those four sides the cls map is held to e1 <= 3e-3 and to an inf-norm error of 1e-5 (100x below TOL, so a
# regression of 1e-5 * ||cls||inf at any cell fails); everywhere else, and for the bbox map everywhere, both <= TOL.
CLS_NEAR_ZERO = {176: 3e-3, 192: 3e-3, 208: 3e-3, 224: 3e-3}
CLS_NEAR_ZERO_INF = 1e-5


def _maps_ok(errs, size):
    """[bbox, cls] map errors within TOL (the cls exception above at the sides listed in CLS_NEAR_ZERO)."""
    (b1, b2), (c1, c2) = errs
    if size in CLS_NEAR_ZERO:
        cls_ok = c1 <= CLS_NEAR_ZERO[size] and c2 <= CLS_NEAR_ZERO_INF
    else:
        cls_ok = c1 <= TOL and c2 <= TOL
    return b1 <= TOL and b2 <= TOL and cls_ok


@pytest.mark.parametrize("size", SIZES)
def test_parity_with_the_fp64_oracle(size):
    """B in {1, 3}, Bz in {1, B}: track (float and uint8), track_boxes, forward and connect_model with and without the
    update template, within the map bars of tests/helpers.py (cls: see CLS_NEAR_ZERO); decoded rows / columns equal to
    the oracle decode's, boxes
    within rtol 1e-3 / atol 2e-2; uint8 == float bit for bit."""
    res = _run("parity", size)
    for tag, r in res.items():
        assert r["shape_ok"], tag
        assert _maps_ok(r["track"], size), (tag, r["track"])
        assert r["uint8_bit_identical"] and r["track_boxes_maps_equal"], tag
        assert r["rows_cols_equal"] and r["flat_ok"], tag
        assert r["box_worst"] <= 1.0, (tag, r["box_worst"])
        assert _maps_ok(r["forward"], size) if "forward" in r else True, (tag, r.get("forward"))
        for key in ("connect", "connect_update"):
            bbox_cls, (cls_dw, x_reg) = r[key][:2], r[key][2:]
            assert _maps_ok(bbox_cls, size), (tag, key, r[key])
            # the intermediates keep the bars of test_gpu_parity.py's head test
            assert cls_dw[0] <= 2e-2 and cls_dw[1] < 1e-4, (tag, key, "cls_dw", cls_dw)
            assert x_reg[0] <= 2e-2 and x_reg[1] <= 5e-5, (tag, key, "x_reg", x_reg)


def test_fixed_size_entry_points_are_the_sized_ones_at_256():
    """fear_track / fear_track_u8 / fear_forward / fear_head_update / fear_decode / fear_decode_smooth give the bytes of
    their sized forms at S = 256 in as many launches; sizes outside the contract are FEAR_EINVAL."""
    res = _run("same256")
    refused = res.pop("refused")
    for name, r in res.items():
        assert r["equal"], name
        if "launches" in r:
            assert r["launches"][0] == r["launches"][1], (name, r["launches"])
    assert all(code == -1 for code in refused.values()), refused


def test_chunked_batch_at_192_equals_one_pass():
    res = _run("chunk")
    assert res["chunk_loop_ran"] and res["chunk_invariant"] and res["n"] == 22


@pytest.mark.parametrize("side", list(range(1, 17)))
def test_decode_at_every_score_side(side):
    """fear_decode_sized (both sigmoid modes) and fear_decode_smooth_sized against the host, with ties, NaN and +-inf."""
    res = _run("decode", side)
    assert all(res["plain"]), res["plain"]
    assert res["coder_records"]
    assert all(res["smooth"]), res["smooth"]


@pytest.mark.parametrize("size", [16, 144, 256])
def test_poisoned_workspace(size):
    res = _run("poison", size)
    assert res["n_failures"] == 0, res["failures"]
    assert res["checked_calls"] > 0


@pytest.mark.parametrize("size", [128, 192])
def test_tracker_trajectories(size):
    """FEARTracker on the first 120 updates of the demo clip against the oracle tracker (the criterion of
    test_free_running_video_trajectory), gpu_crop, CUDA-tensor and NV12 frames against numpy frames, smooth off and on.
    """
    res = _run("trackers", size, timeout=1800)
    for tag, r in res.items():
        assert r["oracle_first30"], (tag, r)
        assert r["min_iou"] > 0.8 and r["mean_iou"] > 0.98, (tag, r)
        assert r["gpu_crop_equal"] and r["cuda_equal"] and r["nv12_equal"], (tag, r)


@pytest.mark.parametrize("size", [128, 192])
def test_multi_tracker_matches_single_trackers(size):
    """FEARMultiTracker (three targets in two streams, the step replayed as a CUDA graph) gives each target's
    FEARTracker(gpu_crop=True) boxes and scores exactly."""
    res = _run("multi", size)
    assert res["graph"] and res["boxes_equal"] and res["scores_equal"], res
