"""GPU: the feature path (get_features, get_features on uint8, feature_extractor, backbone_prefix) at every kind of crop
size the C ABI accepts -- H, W multiples of 16 in [16, 256], square or not -- against the fp64 oracle.

Each fast path of the executor is guarded by a shape predicate and falls back to a more general kernel when it
declines; at 128 x 128 and 256 x 256 nearly every guard accepts.  The sizes below land on both sides of every guard
(fused stem + xif1_0: H % 32 == 0 and W % 64 == 0; fused xif2_0: the same; fused xif2_2 / xif2_3: H, W % 64 == 0;
depthwise fused into the wgmma 1x1 GEMM: square 16 x 16 or 32 x 32 maps; TMA / rolling-window / strip / per-pixel
depthwise by map side), include maps smaller than a TMA box, 1 x 1 final maps and M < 128 GEMMs.  Each (size, batch)
runs in its own process (tests/shape_check.py) so a device trap in one cannot poison the others.
"""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
OUT = None  # log directory of this run (set by _log_dir)
BLOCK_TOL = 2e-5  # inf-norm error per block, as test_gpu_parity.py::test_backbone_block_by_block
FEAT_TOL, FEAT_INF_TOL = 2e-2, 2e-5  # the feature bar of test_gpu_parity.py

# Which fused paths a get_features call takes at each crop size (H, W), derived from the guards above:
#   stem   stem + xif1_0 in one kernel            (1 launch instead of 3)
#   irf    xif2_0 in one wgmma kernel             (1 launch instead of 3)
#   dw24   xif2_2 and xif2_3 as dw3x3 + 24x24     (1 launch per block instead of 2)
#   gemm   stages whose stride-1 blocks run the depthwise inside the 1x1 GEMM (1 launch per block instead of 2):
#          xif3 (3 blocks) on its H/8 x W/8 map, xif4 (7 blocks) on its H/16 x W/16 map; split by map side 16 | 32
#          because the 32 x 32 form has its own option bit
FAST_PATHS = {
    # (H, W):     stem irf dw24 gemm@16        gemm@32
    (16, 16):     (0,   0,  0,  (),            ()),
    (32, 64):     (1,   1,  0,  (),            ()),
    (64, 64):     (1,   1,  1,  (),            ()),
    (48, 48):     (0,   0,  0,  (),            ()),
    (80, 80):     (0,   0,  0,  (),            ()),
    (96, 160):    (0,   0,  0,  (),            ()),
    (128, 256):   (1,   1,  1,  (),            ()),  # xif3 map 16 x 32: not square, the fused GEMM must decline
    (256, 128):   (1,   1,  1,  (),            ()),
    (16, 256):    (0,   0,  0,  (),            ()),
    (256, 16):    (0,   0,  0,  (),            ()),
    (240, 240):   (0,   0,  0,  (),            ()),
    (208, 144):   (0,   0,  0,  (),            ()),
    (128, 128):   (1,   1,  1,  ("xif3",),     ()),
    (256, 256):   (1,   1,  1,  ("xif4",),     ("xif3",)),
}
STAGE_BLOCKS = {"xif3": 3, "xif4": 7}


def expected_fingerprint(shape):
    """Launches added to one get_features call when each fused path is switched off on its own."""
    stem, irf, dw24, gemm16, gemm32 = FAST_PATHS[shape]
    n16, n32 = (sum(STAGE_BLOCKS[s] for s in stages) for stages in (gemm16, gemm32))
    return {"fuse_stem": 2 * stem, "fuse_irf": 2 * irf, "fuse_dwpw_8": 2 * dw24,
            "fuse_dwpw_1": n16 + n32,  # bit 1 off also disables the 32 x 32 form
            "fuse_dwpw_4": n32}


@pytest.fixture(scope="module", autouse=True)
def _log_dir(tmp_path_factory):
    global OUT
    OUT = str(tmp_path_factory.mktemp("shape_check"))


def _run(*args, timeout=600):
    proc = subprocess.run([sys.executable, os.path.join(HERE, "shape_check.py"), *map(str, args)],
                          capture_output=True, text=True, timeout=timeout)
    with open(os.path.join(OUT, "shape_check_" + "_".join(map(str, args)) + ".log"), "w") as f:
        f.write(proc.stdout + "\n--- stderr ---\n" + proc.stderr)
    lines = [l for l in proc.stdout.splitlines() if l.startswith("SHAPE_CHECK ")]
    assert proc.returncode == 0 and lines, f"shape_check {args} failed: {proc.stderr[-3000:]}"
    return json.loads(lines[-1][len("SHAPE_CHECK "):])


def _check_against_oracle(res, blocks_key, feats_key):
    for image, blocks in res[blocks_key].items():
        bad = {k: v for k, v in blocks.items() if not v < BLOCK_TOL}
        assert not bad, (blocks_key, image, bad)
    for image, f in res[feats_key].items():
        assert f["shapes_ok"], (feats_key, image)
        for what in ("feature_extractor", "get_features"):
            e1, e2 = f[what]
            assert e1 <= FEAT_TOL and e2 <= FEAT_INF_TOL, (feats_key, image, what, e1, e2)


def _check_case(res):
    _check_against_oracle(res, "blocks", "features")
    _check_against_oracle(res, "pw_ffma_blocks", "pw_ffma_features")  # CUDA-core 1x1 convs: same bars
    assert res["uint8_bit_identical"], "uint8 HWC crop normalised in the stem != host-normalised float crop"
    bad = {k: v for k, v in res["options"].items() if not v["bit_identical"]}
    assert not bad, bad


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("H,W", list(FAST_PATHS))
def test_feature_path_at_crop_size(H, W, B):
    """Per-block and feature errors vs the fp64 oracle (default kernels and pw=ffma), uint8 == float input, every
    option that promises bit-identical results, and the launch-count fingerprint of the fused paths."""
    res = _run("case", H, W, B)
    _check_case(res)
    assert res["fingerprint"] == expected_fingerprint((H, W)), (res["fingerprint"], FAST_PATHS[(H, W)])


def test_feature_path_chunked_non_square():
    """B = 5 through a 2-frame workspace (chunks 2, 2, 1) at a non-square size whose fused paths all apply: the same
    checks, and the frames equal those of one unchunked pass bit for bit."""
    res = _run("case", 128, 256, 5, 2)
    _check_case(res)
    assert res["chunk_invariant"]


def test_out_of_range_sizes_are_refused():
    """H, W outside {16, 32, ..., 256} fail with FEAR_EINVAL (a RuntimeError from _lib.check) on every entry point that
    takes a crop size -- including the debug prefix, whose workspace holds 256 x 256 frames at most.  Where the output
    tensor is not empty the refusal must come from the size check itself; an empty output (e.g. 8 x 8 features) is a
    null pointer, refused as a bad argument first."""
    res = _run("reject")
    assert res.pop("valid_call_after")
    bad = {k: v for k, v in res.items() if "failed (-1)" not in v["msg"]}
    assert not bad, bad
    size_checked = {k: v for k, v in res.items() if not v["empty_output"]}
    bad = {k: v for k, v in size_checked.items() if "H, W must be multiples of 16 in [16, 256]" not in v["msg"]}
    assert not bad, bad
    # every entry point reaches its size check at some refused size (272 x 272 has no empty outputs)
    assert {k.split(":")[1] for k in size_checked} == {"get_features", "get_features_u8", "feature_extractor",
                                                       "backbone_prefix_0", "backbone_prefix_16"}
