"""Stand-alone checker of the feature path at one crop size (run in its own process: a device-side trap would poison
the CUDA context of the main pytest process).  Prints one JSON line.

    python tests/shape_check.py case H W B [CHUNK]   # CHUNK: hold the library at a CHUNK-frame workspace
    python tests/shape_check.py reject                # out-of-range sizes must be refused

Everything is compared with the fp64 oracle (oracle/fear_oracle.py) on two seeded inputs per case: ImageNet-normalised
uniform uint8 crops (also fed as raw uint8 HWC) and standard-normal images.
"""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import feartracker_b200 as fb  # noqa: E402
from oracle import fear_oracle as fo  # noqa: E402
from tests.helpers import load_full_state, map_errors, poison_workspace  # noqa: E402

BLOCK_NAMES = ["xif0_0"] + [s.name for s in fo.FBNET_C[1:fo.NUM_HOT_BLOCKS] if s.kind == "ir"]
DEFAULTS = {"fuse_stem": "1", "fuse_irf": "1", "fuse_dwpw": "15", "dw": "auto", "pw": "auto"}
# Options whose kernels promise the same arithmetic in the same order as the default path: features must not change a bit.
BIT_IDENTICAL_OPTIONS = [("fuse_stem", "0"), ("fuse_irf", "0"), ("fuse_dwpw", "0"),
                         ("dw", "pixel"), ("dw", "strip"), ("dw", "roll"), ("dw", "tma")]
# One fused path off at a time: the launch count of a get_features call changes exactly when that path ran.
FINGERPRINT_OPTIONS = {"fuse_stem": ("fuse_stem", "0"), "fuse_irf": ("fuse_irf", "0"),
                       "fuse_dwpw_1": ("fuse_dwpw", "14"), "fuse_dwpw_4": ("fuse_dwpw", "11"),
                       "fuse_dwpw_8": ("fuse_dwpw", "7")}


def make_net(reserve):
    sd = load_full_state()
    net = fb.FEARNet(**fb.FEAR_XS_MODEL_KWARGS)
    net.load_state_dict(sd, strict=True)
    net = net.cuda().eval()
    net.reserve(reserve)
    sd64 = fo.to_dtype({k: v for k, v in sd.items() if v.is_floating_point()}, torch.float64)
    return net, sd64


def with_option(net, key, value, fn):
    net.set_option(key, value)
    poison_workspace(net)  # the variant may not pass on values an earlier run left in the workspace
    try:
        return fn()
    finally:
        net.set_option(key, DEFAULTS[key])


def oracle_errors(net, images, cols, nb):
    """Per-block inf-norm errors (backbone_prefix on the first nb frames) and the feature-level errors."""
    blocks, feats = {}, {}
    for name, x in images.items():
        xc, col = x.cuda(), cols[name]
        blocks[name] = {blk: map_errors(net.backbone_prefix(xc[:nb], n).cpu().numpy(), col[blk][:nb].numpy())[1]
                        for n, blk in enumerate(BLOCK_NAMES)}
        fe, gf = net.feature_extractor(xc), net.get_features(xc)
        feats[name] = {"feature_extractor": map_errors(fe.cpu().numpy(), col["xif4_7"].numpy()),
                       "get_features": map_errors(gf.cpu().numpy(), col["neck"].numpy()),
                       "shapes_ok": tuple(fe.shape) == tuple(col["xif4_7"].shape)
                       and tuple(gf.shape) == tuple(col["neck"].shape)}
    return blocks, feats


def case(H, W, B, chunk=0):
    net, sd64 = make_net(chunk or B)
    if chunk:
        net.set_option("pw", "auto")  # packs the weights now: the library's workspace holds `chunk` frames
        net._reserved = 10 ** 9  # keep the library at that workspace: forces the chunk loop
    x, u = fo.shape_crops(H, W, B, seed=5)
    g = torch.Generator().manual_seed(H * 1000 + W * 10 + B)
    images = {"crop": x, "randn": torch.randn(B, 3, H, W, generator=g)}
    u8 = u.permute(0, 2, 3, 1).contiguous().cuda()
    cols = {}
    for name, img in images.items():
        cols[name] = {}
        fo.get_features(sd64, img.double(), cols[name])
    nb = min(B, chunk) if chunk else B  # backbone_prefix runs on at most the reserved batch
    res = {"H": H, "W": W, "B": B, "chunk": chunk}
    res["blocks"], res["features"] = oracle_errors(net, images, cols, nb)
    res["pw_ffma_blocks"], res["pw_ffma_features"] = with_option(net, "pw", "ffma",
                                                                 lambda: oracle_errors(net, images, cols, nb))

    def outputs():
        return ([net.get_features(images[n].cuda()) for n in images] + [net.get_features(u8)]
                + [net.feature_extractor(images["crop"].cuda())])

    ref = outputs()
    res["uint8_bit_identical"] = bool(torch.equal(ref[2], ref[0]))
    res["options"] = {}
    for key, value in BIT_IDENTICAL_OPTIONS:
        got = with_option(net, key, value, outputs)
        res["options"][f"{key}={value}"] = {
            "bit_identical": all(torch.equal(a, b) for a, b in zip(got, ref)),
            "max_abs_diff": max(float((a - b).abs().max()) for a, b in zip(got, ref))}
    if chunk:
        net._reserved = 0
        net.reserve(B)  # whole batch in one pass: per-frame results may not depend on the chunking
        res["chunk_invariant"] = all(torch.equal(a, b) for a, b in zip(outputs(), ref))
    else:
        xc = images["crop"].cuda()

        def launches():
            n0 = net.launch_count()
            net.get_features(xc)
            return net.launch_count() - n0

        base = launches()
        res["launches"] = base
        res["fingerprint"] = {name: with_option(net, key, value, launches) - base
                              for name, (key, value) in FINGERPRINT_OPTIONS.items()}
    torch.cuda.synchronize()
    return res


REJECT_SIZES = [(8, 8), (24, 24), (272, 272), (8, 64), (64, 8), (24, 48), (48, 24), (272, 64), (64, 272), (256, 272)]


def reject():
    """Every entry point that takes a crop size refuses sizes outside the contract with FEAR_EINVAL; a valid call
    still works afterwards.  Per call: the error message, and whether the output tensor is empty (H or W below the
    entry point's downsampling factor: a null output pointer, refused before the size check)."""
    net, _ = make_net(2)
    res = {}
    for H, W in REJECT_SIZES:
        x = torch.zeros(2, 3, H, W, device="cuda")
        u8 = torch.zeros(2, H, W, 3, device="cuda", dtype=torch.uint8)
        calls = {"get_features": (16, lambda: net.get_features(x)), "get_features_u8": (16, lambda: net.get_features(u8)),
                 "feature_extractor": (16, lambda: net.feature_extractor(x)),
                 "backbone_prefix_0": (2, lambda: net.backbone_prefix(x, 0)),
                 "backbone_prefix_16": (32, lambda: net.backbone_prefix(x, 16))}
        for entry, (down, fn) in calls.items():
            try:
                fn()
                torch.cuda.synchronize()
                msg = "accepted"
            except RuntimeError as e:
                msg = str(e)
            res[f"{H}x{W}:{entry}"] = {"msg": msg, "empty_output": H // down == 0 or W // down == 0}
    ok = net.get_features(torch.zeros(1, 3, 32, 32, device="cuda"))
    torch.cuda.synchronize()
    res["valid_call_after"] = tuple(ok.shape) == (1, 256, 2, 2) and bool(torch.isfinite(ok).all())
    return res


def main():
    mode = sys.argv[1]
    if mode == "case":
        res = case(*map(int, sys.argv[2:]))
    elif mode == "reject":
        res = reject()
    else:
        raise SystemExit(f"unknown mode {mode!r}")
    print("SHAPE_CHECK " + json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
