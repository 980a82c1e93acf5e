"""GPU: every kernel entry point on poisoned memory -- workspace, guard bands around every buffer, outputs and the bytes
around strided frames filled with 0, a NaN pattern and a finite pattern in turn -- against itself (bit for bit) and
against the fp64 oracle, cv2 or numpy.  See tests/poison_check.py; each group runs in its own process.

Depthwise instantiations of launch_dw (feartracker_b200/csrc/fear_context.cu) and where the matrix reaches each
("off" = fuse_stem=0 fuse_irf=0 fuse_dwpw=0 together; head ones run in the head group's dw variants, 16 x 16 maps):
  TMA <5,2>                  default, 128 and 256 (xif3_0, xif4_0)
  TMA <5,1>, <3,1>           fuse_dwpw=0, or off with dw=auto | tma, 256 (xif3_1..3 on 32 x 32, xif4_* on 16 x 16;
                             xif2_2, xif2_3)                        <3,1,no relu/bias>: head, default
  roll (3,1)                 fuse_stem=0 or off, 128 and 256 (xif1_0)   (3,1,no relu/bias): head, dw=roll
  roll (3,2)                 off with dw=roll, 128 and 256 (xif2_0 unfused)
  roll (5,1)                 off with dw=roll, 128 and 256 (xif3_1, xif3_2; xif4_* at 256)
  roll (5,2)                 dw=roll, 128 and 256 (xif3_0; xif4_0 at 256)
  strip <5,1,8>              default, 128 (xif4_1..7 on 8 x 8 maps, where the TMA pipeline declines)
  strip <3,1,4>, <3,2,2>     default, 16 and 48 x 240 (unfused stem and xif2_0), and dw=strip
  strip <5,1,4>, <5,2,2>     dw=strip (off for <5,1,4> at 128 and 256)  <3,1,4,no relu/bias>: head, dw=strip
  pixel <3,1>, <3,2>, <5,1>, <5,2>   dw=pixel (off at 128 and 256), and default on the small maps of 16 and 48 x 240
                             <3,1,no relu/bias>: head, dw=pixel
"""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
OUT = None  # log directory of this run (set by _log_dir)
SIZES = [(16, 16), (128, 128), (256, 256), (48, 240)]


@pytest.fixture(scope="module", autouse=True)
def _log_dir(tmp_path_factory):
    global OUT
    OUT = str(tmp_path_factory.mktemp("poison_check"))


def _run(*args, timeout=1200):
    proc = subprocess.run([sys.executable, os.path.join(HERE, "poison_check.py"), *map(str, args)],
                          capture_output=True, text=True, timeout=timeout)
    with open(os.path.join(OUT, "poison_check_" + "_".join(map(str, args)) + ".log"), "w") as f:
        f.write(proc.stdout + "\n--- stderr ---\n" + proc.stderr)
    lines = [l for l in proc.stdout.splitlines() if l.startswith("POISON_CHECK ")]
    assert proc.returncode == 0 and lines, f"poison_check {args} failed: {proc.stderr[-3000:]}"
    return json.loads(lines[-1][len("POISON_CHECK "):])


def _check(res):
    assert res["checked_calls"] > 0
    assert res["n_failures"] == 0, res["failures"]


def test_fill_workspace_entry_point():
    """fear_debug_fill_workspace fills every word, is refused without a handle, is not counted, keeps the generation
    and works inside a CUDA graph capture."""
    res = _run("entry")
    assert res["null_handle"] == -2  # FEAR_ESTATE
    assert res["launches_of_fill"] == 0 and res["generation_unchanged"]
    assert res["all_poison"] and res["graph_fill"]


@pytest.mark.parametrize("H,W", SIZES)
def test_feature_path_on_poisoned_memory(H, W):
    """get_features (float and uint8), backbone and backbone_prefix 0..16 at B = 1, 3 (R = 8) and 5 (R = 2), every
    option variant and every depthwise kernel with all fusions off."""
    _check(_run("features", H, W))


@pytest.mark.parametrize("group", ["head", "track", "decode", "corr", "crops", "loop", "trackers"])
def test_entry_points_on_poisoned_memory(group):
    _check(_run(group))
