"""CPU: the tile-schedule planner of the persistent kernels (tests/schedule_plan.py).  Its launch lists are compared with
the library's launch counts on the GPU (tests/test_gpu_schedules.py); here: the tile counts per frame, that every
scheduling regime of every persistent launch is reached on both H100 variants within the batch caps, and the mapping
from an output pixel to its tile and CTA."""
import pytest

from tests import schedule_plan as sp

SIZES = list(sp.BATCH_CAPS)
OPTION_SETS = [opts for _, opts in sp.all_variants("track")]  # every option set of the GPU sweep


def persistent(entry, H=256, W=256, opts=None):
    return {ln.name: (ln.kernel, ln.tiles) for ln in sp.launches(entry, H, W, opts) if ln.persistent}


def test_tile_counts_per_frame():
    """Tiles per frame of every persistent launch at the search (256 x 256) and template (128 x 128) sizes."""
    assert persistent("get_features", 256, 256) == {
        "xif2_2 dw+pw": ("dw3_pw24", 16), "xif2_3 dw+pw": ("dw3_pw24", 16),
        "xif3_0.dw": ("dw_tma<5,2>", 80), "xif4_0.dw": ("dw_tma<5,2>", 24)}
    assert persistent("get_features", 128, 128) == {
        "xif2_2 dw+pw": ("dw3_pw24", 4), "xif2_3 dw+pw": ("dw3_pw24", 4),
        "xif3_0.dw": ("dw_tma<5,2>", 20), "xif4_0.dw": ("dw_tma<5,2>", 6)}
    # stride-1 instantiations, only with the depthwise-in-GEMM fusion off
    s1 = {k: v for k, v in persistent("get_features", 256, 256, {"fuse_dwpw": "0"}).items() if "<5,2>" not in v[0]}
    assert s1 == {"xif2_2.dw": ("dw_tma<3,1>", 16), "xif2_3.dw": ("dw_tma<3,1>", 16),
                  "xif3_1.dw": ("dw_tma<5,1>", 12), "xif3_2.dw": ("dw_tma<5,1>", 24), "xif3_3.dw": ("dw_tma<3,1>", 24),
                  "xif4_1.dw": ("dw_tma<5,1>", 6), "xif4_2.dw": ("dw_tma<5,1>", 12), "xif4_3.dw": ("dw_tma<5,1>", 12),
                  "xif4_4.dw": ("dw_tma<5,1>", 12), "xif4_5.dw": ("dw_tma<5,1>", 21), "xif4_6.dw": ("dw_tma<5,1>", 21),
                  "xif4_7.dw": ("dw_tma<5,1>", 11)}
    s1 = {k: v[1] for k, v in persistent("get_features", 128, 128, {"fuse_dwpw": "0"}).items() if k.startswith("xif3_")
          and k != "xif3_0.dw"}
    assert s1 == {"xif3_1.dw": 3, "xif3_2.dw": 6, "xif3_3.dw": 6}
    # mask value 1 cleared: xif3 (32 x 32) and xif4 (16 x 16) at 256 unfused; mask value 4 cleared: xif3 only
    stages34 = {k: v for k, v in persistent("get_features", 256, 256, {"fuse_dwpw": "0"}).items() if k[3] in "34"}
    assert {k: v for k, v in persistent("get_features", 256, 256, {"fuse_dwpw": "14"}).items() if k[3] in "34"} == stages34
    assert not any(k.startswith("xif4_") and k != "xif4_0.dw" for k in persistent("get_features", 256, 256,
                                                                                  {"fuse_dwpw": "11"}))
    # head SepConvs with mask value 2 cleared: 8 tiles (256 channels) and 10 (the 320-channel concat)
    head = persistent("head", opts={"fuse_dwpw": "13"})
    assert {v for v in head.values()} == {("dw_tma<3,1,no bias>", 8), ("dw_tma<3,1,no bias>", 10)}
    assert head["cls_dw.dw"] == head["reg_dw.dw"] == ("dw_tma<3,1,no bias>", 10)
    # the prediction convolutions' depthwise stage is never fused: persistent in every default head
    assert persistent("head") == {"bbox_pred.dw": ("dw_tma<3,1,no bias>", 8), "cls_pred.dw": ("dw_tma<3,1,no bias>", 8)}
    # no TMA where the option or the map size rules it out
    assert not persistent("get_features", 256, 256, {"dw": "pixel"}).keys() - {"xif2_2 dw+pw", "xif2_3 dw+pw"}
    assert not persistent("get_features", 16, 16)


@pytest.mark.parametrize("S", [sp.H100_SXM_SMS, sp.H100_PCIE_SMS])
@pytest.mark.parametrize("H,W", SIZES)
@pytest.mark.parametrize("opts", OPTION_SETS, ids=lambda o: ",".join(f"{k}={v}" for k, v in o.items()) or "default")
def test_every_regime_reached_under_the_cap(H, W, opts, S):
    """Every regime of every persistent launch of get_features (and, at 256 x 256, fear_track_u8) has a batch, and each
    batch really is in the regime it is listed for."""
    cap = sp.BATCH_CAPS[(H, W)]
    entries = [("get_features", {})] + ([("track_u8", {})] if (H, W) == (256, 256) else [])
    for entry, kw in entries:
        p = sp.plan(entry, H, W, opts, S, **kw)
        assert max(p) <= cap, (entry, max(p), cap)
        lns = {ln.name: ln for ln in sp.launches(entry, H, W, opts, **kw) if ln.persistent}
        for name, ln in lns.items():
            reached = {r.split(": ")[1] for B, rs in p.items() for r in rs if r.startswith(name + " [")}
            assert reached == set(sp.REGIME_NAMES), (entry, name, set(sp.REGIME_NAMES) - reached)
        for B, rs in p.items():
            for r in rs:
                name, regime = r.split(" [")[0], r.split(": ")[1]
                t = lns[name].tiles
                assert sp.in_regime(regime, B * t, S, t), (B, r)
                assert B == 1 or not sp.in_regime(regime, (B - 1) * t, S, t), ("not the smallest batch", B, r)


def test_regime_definitions():
    S = 132
    assert sp.in_regime("under_one_wave", 131, S, 1) and not sp.in_regime("under_one_wave", 132, S, 1)
    assert sp.in_regime("first_partial_wave", 160, S, 80) and not sp.in_regime("first_partial_wave", 240, S, 80)
    assert sp.cta_tile_counts(160, S) == (132, 2) and sp.in_regime("cta_2_tiles", 160, S, 80)
    assert not sp.in_regime("cta_3_tiles", 264, S, 8) and sp.in_regime("cta_3_tiles", 272, S, 8)
    assert sp.in_regime("cta_9plus_tiles", 1056 + 8, S, 8) and not sp.in_regime("cta_9plus_tiles", 1056, S, 8)
    assert not sp.in_regime("cta_9plus_uneven", 9 * 132, S, 4) and sp.in_regime("cta_9plus_uneven", 1060, S, 4)
    assert sp.in_regime("busiest_odd", 2 * 132 + 1, S, 1) and not sp.in_regime("busiest_odd", 2 * 132, S, 1)
    assert not sp.in_regime("busiest_odd", 100, S, 1)  # one tile per CTA is not a multi-lap odd count


def test_tile_owner_mapping():
    """Pixel -> tile -> CTA as the kernels walk tiles (tile = blockIdx.x + it * gridDim.x)."""
    ln = [l for l in sp.launches("get_features", 256, 256) if l.name == "xif3_0.dw"][0]  # 32 x 32 out, 8 x 8 tiles
    assert (ln.tiles_x, ln.tiles_y, ln.cblocks, ln.th) == (4, 4, 5, 8)
    o = sp.tile_owner(ln, 14, 132, frame=3, y=17, x=30, cb=2)
    assert o["tile"] == ((3 * 4 + 2) * 4 + 3) * 5 + 2 == 297
    assert (o["grid"], o["cta"], o["iteration"], o["stage"], o["parity"], o["group"]) == (132, 33, 2, 2, 0, 0)
    o = sp.tile_owner(ln, 1, 132, frame=0, y=31, x=31, cb=4)
    assert (o["tile"], o["grid"], o["cta"], o["iteration"]) == (79, 80, 79, 0)


def test_large_batch_crosses_int32():
    B = sp.smallest_batch_past_int32()
    assert B == 1372 and B % 7 == 0
    assert B * sp.K_ACT_E > 2 ** 31 >= (B - 7) * sp.K_ACT_E
    assert 16 << 30 < sp.workspace_bytes(B) < 18 << 30  # the reason the GPU case needs ~18 GB free


def test_launch_model_matches_the_fused_path_fingerprints():
    """The planner's launch counts reproduce the fingerprints tests/test_gpu_shapes.py measures on the GPU."""
    from tests.test_gpu_shapes import FAST_PATHS, expected_fingerprint

    options = {"fuse_stem": ("fuse_stem", "0"), "fuse_irf": ("fuse_irf", "0"), "fuse_dwpw_1": ("fuse_dwpw", "14"),
               "fuse_dwpw_4": ("fuse_dwpw", "11"), "fuse_dwpw_8": ("fuse_dwpw", "7")}  # as tests/shape_check.py
    for (H, W) in FAST_PATHS:
        base = len(sp.launches("get_features", H, W))
        got = {name: len(sp.launches("get_features", H, W, {k: v})) - base for name, (k, v) in options.items()}
        assert got == expected_fingerprint((H, W)), (H, W, got)
