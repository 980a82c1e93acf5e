"""GPU: the persistent kernels (dw_tma_kernel, dw3_pw24_fused_kernel) at every batch where their tile schedule changes,
and one chunk whose workspace passes 2^31 floats.

tests/schedule_plan.py models every launch of get_features / fear_track_u8 / fear_head and picks, for the SM count of
this device, the smallest batch that puts each persistent launch into each regime: under one wave, the first full wave,
a CTA with 2, 3, 5 and >= 9 tiles (the first stage refill, the barrier parity wrap), >= 9 tiles with CTAs ending on
different laps, and the busiest CTA with an odd tile count.  tests/schedule_check.py runs each of those batches on a
poisoned workspace and requires every frame to equal its own B = 1 result bit for bit (the B = 1 results are checked
against the fp64 oracle), runs every option variant at its multi-lap batches, and compares the launch count of each
call with the model.  Each case runs in its own process so a device trap cannot poison the others.
"""
import json
import os
import subprocess
import sys

import pytest

from tests import schedule_plan as sp

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
OUT = None  # log directory of this run (set by _log_dir)


@pytest.fixture(scope="module", autouse=True)
def _log_dir(tmp_path_factory):
    global OUT
    OUT = str(tmp_path_factory.mktemp("schedule_check"))


def _run(*args, timeout=1800):
    proc = subprocess.run([sys.executable, os.path.join(HERE, "schedule_check.py"), *map(str, args)],
                          capture_output=True, text=True, timeout=timeout)
    with open(os.path.join(OUT, "schedule_check_" + "_".join(map(str, args)) + ".log"), "w") as f:
        f.write(proc.stdout + "\n--- stderr ---\n" + proc.stderr)
    lines = [l for l in proc.stdout.splitlines() if l.startswith("SCHEDULE_CHECK ")]
    assert proc.returncode == 0 and lines, f"schedule_check {args} failed: {proc.stderr[-3000:]}"
    return json.loads(lines[-1][len("SCHEDULE_CHECK "):])


def _check(res, entry, H=256, W=256, kind="features"):
    want = sp.planned(entry, H, W, sp.all_variants(kind), res["S"])
    assert [int(b) for b in res["batches"]] == list(want), "the checker ran other batches than the planner picks"
    assert res["runs"] >= 2 * len(want)
    bad = {k: v for k, v in res["dispatch"].items() if v[0] != v[1]}
    assert not bad, f"launch counts (got, planner) differ: {bad}"
    assert res["n_failures"] == 0, res["failures"]


@pytest.mark.parametrize("H,W", list(sp.BATCH_CAPS))
def test_feature_schedules(H, W):
    """get_features_u8 at every planned batch of every option set at the search, template and a non-square size (where
    the stride-1 TMA depthwise kernels run by default)."""
    res = _run("features", H, W)
    _check(res, "get_features", H, W)
    assert max(int(b) for b in res["batches"]) <= sp.BATCH_CAPS[(H, W)]


def test_track_schedules():
    """fear_track_u8 with Bz = B at every planned batch (backbone and head launches) of every option set; fear_head's
    launch counts against the model too."""
    res = _run("track")
    _check(res, "track_u8", kind="track")
    bad = {k: v for k, v in res["dispatch_head"].items() if v[0] != v[1]}
    assert not bad, f"fear_head launch counts (got, planner) differ: {bad}"


def test_batch_past_int32_workspace():
    """B = 1372 in one chunk (bufE then holds B x 128 x 128 x 96 > 2^31 floats): get_features_u8 (default and
    fuse_irf=0) and fear_track_u8 with Bz = B, every frame equal to its B = 1 result.  Needs ~18 GB free."""
    res = _run("large")
    if "skipped" in res:
        pytest.skip(res["skipped"])
    assert res["bufE_floats"] > 2 ** 31 and res["runs"] == 3
    assert res["n_failures"] == 0, res["failures"]
