"""GPU: the wgmma (tensor-core, 3xTF32) kernels against an fp64 reference, each case in its own
process so a device trap cannot poison the rest of the suite."""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
OUT = None  # log directory of this run (set by _log_dir)


@pytest.fixture(scope="module", autouse=True)
def _log_dir(tmp_path_factory):
    global OUT
    OUT = str(tmp_path_factory.mktemp("tc_check"))


def _run(*args, timeout=180):
    proc = subprocess.run([sys.executable, os.path.join(HERE, "tc_check.py"), *map(str, args)], capture_output=True,
                          text=True, timeout=timeout)
    with open(os.path.join(OUT, "tc_check_" + "_".join(map(str, args)) + ".log"), "w") as f:
        f.write(proc.stdout + "\n--- stderr ---\n" + proc.stderr)
    lines = [l for l in proc.stdout.splitlines() if l.startswith("TC_CHECK ")]
    assert proc.returncode == 0 and lines, f"tc_check {args} failed: {proc.stderr[-2000:]}"
    return json.loads(lines[-1][len("TC_CHECK "):])


@pytest.mark.parametrize("impl", ["wgmma"])
@pytest.mark.parametrize("B,Bz", [(1, 1), (3, 3), (5, 1), (200, 200), (256, 256), (300, 1)])
def test_corr_tcgen05(B, Bz, impl):
    res = _run("corr", B, Bz, impl)
    assert res["ffma"]["max_err_rel"] < 1e-5, res["ffma"]
    tc = res["wgmma"]
    assert tc["x_intact"], "correlation kernel must not touch the x channels"
    assert tc["max_err_rel"] < 1e-5, tc  # 3xTF32 keeps fp32-level accuracy


@pytest.mark.parametrize("pw,corr", [("wgmma", "ffma"), ("wgmma", "wgmma"), ("ffma", "ffma")])
def test_network_with_tensor_core_kernels(pw, corr):
    """Every 1x1 conv (all layer shapes of FEAR-XS) on the wgmma GEMM: block-by-block and final maps."""
    res = _run("net", pw, corr, timeout=400)
    bad = {k: v for k, v in res["blocks"].items() if v[1] > 1e-5}
    assert not bad, bad
    assert res["reg"][0] <= 1e-3 and res["reg"][1] <= 1e-3, res
    assert res["cls"][0] <= 1e-3 and res["cls"][1] <= 1e-3, res
    assert res["argmax_same"]


@pytest.mark.parametrize("B", [2, 19])
def test_fused_irf_block(B):
    """xif2_0 as one wgmma kernel (expanded tensor on-chip): bit-identical to the three-kernel path, <= 2e-5 of the
    fp64 oracle; B = 19 gives several waves of tiles (608 search tiles on 132 SMs)."""
    res = _run("irf", B, timeout=400)
    for name in ("search", "template"):
        r = res[name]
        assert r["vs_oracle"][1] < 2e-5, (name, r)
        assert r["bit_identical"] and r["features_bit_identical"], (name, r)
