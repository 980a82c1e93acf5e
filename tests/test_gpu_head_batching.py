"""GPU: the head (fear_head, fear_head_update), the entry points that wrap it (fear_track, fear_track_u8, fear_forward,
track_boxes_from_host) and fear_decode at every batch, broadcast and chunk layout.

Every frame holds distinct content.  Each distinct (search, template, update) triple is run once unchunked at B = 1
against the fp64 oracle; every frame of every batched, broadcast or chunked call must equal its B = 1 result bit for
bit (the head's kernels are row-local with a fixed reduction order).  At B = 33 and 34 the head GEMMs launch 132 and
136 CTAs: one wave of an H100's 132 SMs and just past it.  Each group runs in its own process (tests/head_check.py).
"""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
OUT = None  # log directory of this run (set by _log_dir)
MAP_INF_TOL = 1e-4  # inf-norm error of a head map (test_gpu_parity.py::test_batch256_parity_and_host_path)
INTERMEDIATE_INF_TOL = 1e-4  # cls_dw / x_reg (test_gpu_parity.py::test_head_intermediates)
ARGMAX_MARGIN = 1e-4  # below this oracle top-2 margin the argmax is a tie at fp32 resolution

# Kernel launches of one fear_head / fear_head_update call: (once per call, per chunk of at most R frames), by
# (template batch, update batch).  Once: the layout transpose of a broadcast template or update template.  Per chunk:
# the transpose of the search features, of a per-frame template and of a per-frame update template, then run_head --
# 4 SepConvs of the encode / correlation stages and 2 x 2 of the towers (one fused wgmma kernel each), 2 prediction
# depthwise + 2 prediction 1x1 kernels, and the correlation: one launch for both branches, two with an update template.
HEAD_LAUNCHES = {
    ("1", None): (1, 14), ("B", None): (0, 15),
    ("1", "1"): (2, 15), ("1", "B"): (1, 16),
    ("B", "1"): (1, 16), ("B", "B"): (0, 17),
}


@pytest.fixture(scope="module", autouse=True)
def _log_dir(tmp_path_factory):
    global OUT
    OUT = str(tmp_path_factory.mktemp("head_check"))


def _run(group, timeout=900):
    proc = subprocess.run([sys.executable, os.path.join(HERE, "head_check.py"), group],
                          capture_output=True, text=True, timeout=timeout)
    lines = [l for l in proc.stdout.splitlines() if l.startswith("HEAD_CHECK ")]
    with open(os.path.join(OUT, f"head_check_{group}.log"), "w") as f:
        f.write(proc.stdout + "\n--- stderr ---\n" + proc.stderr)
    assert proc.returncode == 0 and lines, f"head_check {group} failed: {proc.stderr[-3000:]}"
    res = json.loads(lines[-1][len("HEAD_CHECK "):])
    print(f"head_check {group}: {json.dumps({k: v for k, v in res.items() if k != 'rows'})}")
    return res


def _check_bits(res):
    assert res["bit_comparisons"] > 0
    assert res["n_bit_failures"] == 0, res["bit_failures"]


def _check_oracle(o, intermediates=True):
    assert o["inf"]["reg"] <= MAP_INF_TOL and o["inf"]["cls"] <= MAP_INF_TOL, o
    if intermediates:
        assert o["inf"]["cls_dw"] <= INTERMEDIATE_INF_TOL and o["inf"]["x_reg"] <= INTERMEDIATE_INF_TOL, o
    # allclose form |a - b| <= 1e-3 |b| + 1e-5 ||b||inf, as the ratio of the two sides
    assert o["allclose_ratio"]["reg"] <= 1 and o["allclose_ratio"]["cls"] <= 1, o
    real = [m for m in o["argmax_mismatch"] if m["margin"] >= ARGMAX_MARGIN]
    assert not real, real


def test_head_batch_broadcast_chunk_matrix():
    """fear_head / fear_head_update at B in {1, 2, 3, 7, 33, 34} unchunked and {1, 3, 4, 5, 8, 9, 11} at R = 4, with
    every Bz in {1, B} and Bu in {none, 1, B}: per-frame bit identity with B = 1, broadcast == expanded templates,
    update = NULL == fear_head, a regression map that ignores the update; the B = 1 results against the oracle."""
    res = _run("matrix")
    _check_bits(res)
    assert res["oracle"]["frames"] >= 6 * 34
    _check_oracle(res["oracle"])


def test_track_and_forward_batched_and_chunked():
    """fear_track, fear_track_u8 and fear_forward (boxes only, maps only, both) at B in {1, 3, 9}, unchunked and at
    R = 4: frame i == fear_head(z_i, get_features(x_i)), records == fear_decode of the maps; 3 frames end to end
    against the fp64 oracle."""
    res = _run("track")
    _check_bits(res)
    _check_oracle(res["oracle_end_to_end"], intermediates=False)


def test_track_boxes_from_host_double_buffered():
    """Two unsynchronised track_boxes_from_host calls (chunks 1 and 3, Bz 1 and 7) each equal track_boxes of their own
    inputs: the result of a call stays valid until the call after next."""
    _check_bits(_run("host"))


def test_head_option_variants():
    """fuse_dwpw = 13 (head SepConv fusion off) is bit-identical; pw x corr in {ffma, wgmma} meet the oracle bars."""
    res = _run("options")
    _check_bits(res)
    _check_oracle(res["oracle"])
    assert len(res["variants"]) == 8
    for name, o in res["variants"].items():
        _check_oracle(o, intermediates=False)


def test_head_launch_counts_and_refused_arguments():
    """The launch count of one head call depends on B only through the number of chunks; refused arguments return
    FEAR_EINVAL and launch nothing."""
    res = _run("launches")
    bad = []
    for row in res["rows"]:
        B, R = row["B"], row["R"] or row["B"]
        key = ("1" if row["Bz"] == 1 else "B", None if row["Bu"] is None else ("1" if row["Bu"] == 1 else "B"))
        once, per_chunk = HEAD_LAUNCHES[key]
        if row["launches"] != once + per_chunk * -(-B // R):
            bad.append(row)
    assert not bad, bad
    covered = {(row["R"], row["B"]) for row in res["rows"]}
    assert covered == {(0, b) for b in (1, 2, 3, 7, 33, 34)} | {(4, b) for b in (1, 3, 4, 5, 8, 9, 11)}, covered
    assert len(res["rows"]) == 11 * 6 + 2 * 2  # B = 1 has one Bz and two Bu patterns
    bad = {k: v for k, v in res["refused"].items() if v != {"rc": res["einval"], "launches": 0}}
    assert not bad, bad


def test_decode_edge_cases():
    """fear_decode (apply_sigmoid 1 and 0; B = 1, 7 and 70 000) == torch.argmax of torch.sigmoid on the same device:
    ties in and across warps, at indices 0 and 255, -0.0 vs 0.0, saturation, denormal sigmoids, +-inf, NaN (greater than
    every number, first NaN wins); score bit-identical to CUDA torch.sigmoid and within 2 ulp of CPU torch.sigmoid;
    float64 boxes bit for bit."""
    res = _run("decode")
    for key in ("mismatch", "score_not_bit_identical", "ulp_fail", "box_mismatch"):
        assert not res[key], (key, res[key])
    cases = res["case_results"]
    assert cases["pos_saturation sigmoid=1"][0] == 40 and cases["pos_saturation sigmoid=0"][0] == 200
    assert cases["neg_saturation sigmoid=1"] == [0, 0.0]
    assert cases["denormal sigmoid=1"][0] == 77 and 0 < cases["denormal sigmoid=1"][1] < 1.2e-38
    assert cases["nan_5_larger_later sigmoid=1"][0] == 5 and cases["nan_32_larger_later sigmoid=0"][0] == 32
    assert cases["tie_index_0_and_255 sigmoid=1"][0] == 0 and cases["zero_before_neg_zero sigmoid=0"][0] == 3
