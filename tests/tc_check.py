"""Stand-alone checker for the wgmma kernels (run in its own process: a device-side trap would
poison the CUDA context of the main pytest process).  Prints one JSON object.

    python tests/tc_check.py corr [B] [Bz]
"""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from feartracker_b200 import _lib  # noqa: E402


def _select_corr(lib, impl):
    _lib.check(lib.fear_set_option(None, b"corr", impl.encode()), "fear_set_option")


def corr_case(lib, B, Bz, impl, seed=0):
    g = torch.Generator().manual_seed(seed)
    zt = torch.randn(Bz, 64, 256, generator=g)
    cat = torch.randn(B, 256, 320, generator=g)
    ref = torch.einsum("bpc,bkc->bpk", cat[:, :, :256].double(), (zt if Bz == B else zt.expand(B, 64, 256)).double())
    _select_corr(lib, impl)
    zc, cc = zt.cuda(), cat.cuda()
    _lib.check(lib.fear_corr_nhwc_f32(zc.data_ptr(), Bz, cc.data_ptr(), B, torch.cuda.current_stream().cuda_stream),
               "fear_corr_nhwc_f32")
    torch.cuda.synchronize()
    out = cc.cpu()
    x_intact = bool(torch.equal(out[:, :, :256], cat[:, :, :256]))
    got = out[:, :, 256:].double()
    err = (got - ref).abs()
    scale = ref.abs().max().item()
    # error map per (frame, 32-pixel block, 8-template-cell block) to localise layout mistakes
    blocks = err.reshape(B, 8, 32, 8, 8).amax(dim=(2, 4)) / scale
    return {
        "impl": impl, "B": B, "Bz": Bz, "x_intact": x_intact, "max_err_rel": err.max().item() / scale,
        "mean_err_rel": err.mean().item() / scale, "worst_block": blocks.flatten().argmax().item(),
        "block_err_max_per_frame": blocks.amax(dim=(1, 2)).tolist(),
        "sample_got": got[0, 0, :4].tolist(), "sample_ref": ref[0, 0, :4].tolist(),
        "sample_got_p129": got[0, 129, :4].tolist(), "sample_ref_p129": ref[0, 129, :4].tolist(),
    }


def net_case(pw, corr):
    """Whole network with the selected kernel implementations vs the fp64 oracle: per-block backbone
    errors (localises a bad layer shape), head intermediates and the final maps."""
    import feartracker_b200 as fb
    from oracle import fear_oracle as fo
    from tests.helpers import load_full_state, map_errors

    sd = load_full_state()
    net = fb.FEARNet(**fb.FEAR_XS_MODEL_KWARGS)
    net.load_state_dict(sd, strict=True)
    net = net.cuda().eval()
    net.reserve(4)
    net.set_option("pw", pw)
    net.set_option("corr", corr)
    sd64 = fo.to_dtype({k: v for k, v in sd.items() if v.is_floating_point()}, torch.float64)
    zt, xt, _, _ = fo.synthetic_crops(3)  # 3 frames: template branch M = 192 (M % 128 = 64 tail)
    col = {}
    zf64 = fo.get_features(sd64, zt.double())
    xf64 = fo.get_features(sd64, xt.double(), col)
    names = ["xif0_0"] + [s.name for s in fo.FBNET_C[1:fo.NUM_HOT_BLOCKS] if s.kind == "ir"]
    res = {"pw": pw, "corr": corr, "blocks": {}}
    for n, name in enumerate(names):
        mine = net.backbone_prefix(xt.cuda(), n).cpu().numpy()
        res["blocks"][name] = map_errors(mine, col[name].numpy())
    zf = net.get_features(zt.cuda())
    res["zf"] = map_errors(zf.cpu().numpy(), zf64.numpy())
    hcol = {}
    ref = fo.connector(sd64, zf64, xf64, hcol)
    out = net.track(xt.cuda(), zf)
    for name, want in (("cls_dw", hcol["cls_dw"]), ("reg_dw", hcol["reg_dw"]), ("x_reg", hcol["x_reg"]),
                       ("cls_tower", hcol["cls_tower"])):
        res[name] = map_errors(net.head_tensor(name, 3).cpu().numpy(), want.numpy())
    for key, short in ((fo.TARGET_REGRESSION_LABEL_KEY, "reg"), (fo.TARGET_CLASSIFICATION_KEY, "cls")):
        res[short] = map_errors(out[key].cpu().numpy(), ref[key].numpy())
    res["argmax_same"] = bool((out[fo.TARGET_CLASSIFICATION_KEY].flatten(1).argmax(1).cpu()
                               == ref[fo.TARGET_CLASSIFICATION_KEY].flatten(1).argmax(1)).all())
    return res


def corr_perf(lib, impl, B=256, iters=50):
    """Timing only: the channels-last correlation kernel on B frames, rotating over 4 buffers (> L2)."""
    _select_corr(lib, impl)
    zt = torch.randn(B, 64, 256, device="cuda")
    cats = [torch.randn(B, 256, 320, device="cuda") for _ in range(4)]
    st = torch.cuda.current_stream().cuda_stream
    for c in cats:
        _lib.check(lib.fear_corr_nhwc_f32(zt.data_ptr(), B, c.data_ptr(), B, st), "corr")
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for i in range(iters):
        _lib.check(lib.fear_corr_nhwc_f32(zt.data_ptr(), B, cats[i % 4].data_ptr(), B, st), "corr")
    b.record()
    torch.cuda.synchronize()
    us = a.elapsed_time(b) * 1e3 / iters
    return {"impl": impl, "us": us, "GBps": 393216 * B / us * 1e-3}


def irf_case(B):
    """Fused xif2_0 kernel (expand -> depthwise s2 -> project in one launch) vs the three-kernel path (must be
    bit-identical) and vs the fp64 oracle, on search- and template-sized inputs; B frames so that every persistent
    CTA walks several tiles."""
    import feartracker_b200 as fb
    from oracle import fear_oracle as fo
    from tests.helpers import load_full_state, map_errors, poison_workspace

    sd = load_full_state()
    net = fb.FEARNet(**fb.FEAR_XS_MODEL_KWARGS)
    net.load_state_dict(sd, strict=True)
    net = net.cuda().eval()
    net.reserve(B)
    sd64 = fo.to_dtype({k: v for k, v in sd.items() if v.is_floating_point()}, torch.float64)
    res = {"B": B}
    for name, size in (("search", 256), ("template", 128)):
        g = torch.Generator().manual_seed(B + size)
        x = torch.randn(B, 3, size, size, generator=g)
        net.set_option("fuse_irf", "0")
        ref = net.backbone_prefix(x.cuda(), 2)
        ref_full = net.get_features(x.cuda())
        net.set_option("fuse_irf", "1")
        poison_workspace(net)  # the fused kernel may not pass on values the three-kernel run left in the workspace
        got = net.backbone_prefix(x.cuda(), 2)
        got_full = net.get_features(x.cuda())
        torch.cuda.synchronize()
        diff = (got - ref).abs()
        col = {}
        fo.get_features(sd64, x[:2].double(), col)
        res[name] = {
            "bit_identical": bool(torch.equal(got, ref)), "features_bit_identical": bool(torch.equal(got_full, ref_full)),
            "max_abs_diff": float(diff.max()), "ref_absmax": float(ref.abs().max()),
            "worst_frame": int(diff.flatten(1).amax(1).argmax()),
            "per_frame_max": diff.flatten(1).amax(1).tolist()[:8],
            "vs_oracle": map_errors(got[:2].cpu().numpy(), col["xif2_0"].numpy()),
            "unfused_vs_oracle": map_errors(ref[:2].cpu().numpy(), col["xif2_0"].numpy()),
        }
    return res


def main():
    mode = sys.argv[1]
    lib = _lib.init(0)
    res = {"mode": mode}
    if mode == "corr":
        B = int(sys.argv[2]) if len(sys.argv) > 2 else 3
        Bz = int(sys.argv[3]) if len(sys.argv) > 3 else B
        impl = sys.argv[4] if len(sys.argv) > 4 else "wgmma"
        res["ffma"] = corr_case(lib, B, Bz, "ffma")
        res["wgmma"] = corr_case(lib, B, Bz, impl)
    elif mode == "corrperf":
        res["perf"] = [corr_perf(lib, impl) for impl in sys.argv[2:]]
    elif mode == "net":
        res.update(net_case(sys.argv[2], sys.argv[3]))
    elif mode == "irf":
        res.update(irf_case(int(sys.argv[2]) if len(sys.argv) > 2 else 16))
    print("TC_CHECK " + json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
