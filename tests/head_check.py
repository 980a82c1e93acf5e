"""Stand-alone checker of the head, the entry points that wrap it and the box decode at every batch, broadcast and
chunk layout (run in its own process: a device-side trap would poison the CUDA context of the main pytest process).
Prints one JSON line.

    python tests/head_check.py GROUP      # GROUP: matrix | track | host | options | launches | decode

Every frame of every call holds distinct content, so a chunk that read or wrote at the wrong frame offset shows.  The
head's kernels are row-local with a fixed reduction order, so:
  (a) each distinct (search, template, update) triple is run once unchunked at B = 1 and compared with the fp64 oracle
      (fo.box_tower on the GPU's own fp32 features, cast to float64: the head's error alone, not the backbone's);
  (b) every frame of every batched, broadcast or chunked call must equal its B = 1 result bit for bit.
Handles come from FEARNet.reserve(R) and the C ABI is called directly through _lib with net._handle, so a batch larger
than R is chunked inside the library.
"""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import feartracker_b200 as fb  # noqa: E402
from feartracker_b200 import _lib  # noqa: E402
from oracle import fear_oracle as fo  # noqa: E402
from tests.helpers import TOL, load_full_state, map_errors, poison_workspace  # noqa: E402

R, C = fo.TARGET_REGRESSION_LABEL_KEY, fo.TARGET_CLASSIFICATION_KEY
FEAR_EINVAL = -1
MARGIN = 1e-4  # oracle top-2 logit margin below which the argmax is a tie at fp32 resolution
MATRIX = {0: [1, 2, 3, 7, 33, 34], 4: [1, 3, 4, 5, 8, 9, 11]}  # reservation (0 = unchunked) -> batches
POOL = max(MATRIX[0])


def make_net(reserve):
    """A FEARNet whose library handle holds a `reserve`-frame workspace."""
    net = fb.FEARNet(**fb.FEAR_XS_MODEL_KWARGS)
    net.load_state_dict(load_full_state(), strict=True)
    net = net.cuda().eval()
    net.reserve(reserve)
    net._ensure_handle(torch.device("cuda", torch.cuda.current_device()))
    return net


def sd64():
    return fo.to_dtype({k: v for k, v in load_full_state().items() if v.is_floating_point()}, torch.float64)


def stream():
    return torch.cuda.current_stream().cuda_stream


def ptr(t):
    return t.data_ptr() if t is not None else None


def maps(B):
    return torch.empty((B, 4, 16, 16), device="cuda"), torch.empty((B, 1, 16, 16), device="cuda")


def head(net, z, x, u=None):
    """fear_head (u None) or fear_head_update on the handle: (bbox, cls)."""
    B = x.shape[0]
    bbox, cls = maps(B)
    lib = _lib.load()
    if u is None:
        _lib.check(lib.fear_head(net._handle, z.data_ptr(), z.shape[0], x.data_ptr(), B, bbox.data_ptr(),
                                 cls.data_ptr(), stream()), "fear_head")
    else:
        _lib.check(lib.fear_head_update(net._handle, z.data_ptr(), z.shape[0], u.data_ptr(), u.shape[0], x.data_ptr(),
                                        B, bbox.data_ptr(), cls.data_ptr(), stream()), "fear_head_update")
    return bbox, cls


def feature_pools(net, n, magnitudes=True):
    """Search features of n synthetic search crops and two sets of template features (different seeds); with
    `magnitudes`, a few entries are standard-normal features scaled x0.5 and x4 instead."""
    _, xt, _, _ = fo.synthetic_crops(n)
    zc, _ = fo.shape_crops(128, 128, n, seed=21)
    uc, _ = fo.shape_crops(128, 128, n, seed=22)
    x, z, u = (net.get_features(t.cuda()) for t in (xt, zc, uc))
    if magnitudes:
        g = torch.Generator().manual_seed(77)
        x[1] = 0.5 * torch.randn(256, 16, 16, generator=g).cuda()
        x[4] = 4.0 * torch.randn(256, 16, 16, generator=g).cuda()
        z[3] = 4.0 * torch.randn(256, 8, 8, generator=g).cuda()
        u[2] = 0.5 * torch.randn(256, 8, 8, generator=g).cuda()
    return x, z, u


class BitCheck:
    """Counts bit-for-bit comparisons and records the failing ones."""

    def __init__(self):
        self.count, self.failures = 0, []

    def eq(self, a, b, what):
        self.count += 1
        if not torch.equal(a, b):
            diff = float((a.float() - b.float()).abs().nan_to_num(float("inf")).max()) if a.shape == b.shape else -1
            self.failures.append(f"{what}: max |diff| {diff:.3e}")

    def report(self):
        return {"bit_comparisons": self.count, "bit_failures": self.failures[:40], "n_bit_failures": len(self.failures)}


class HeadRefs:
    """Unchunked B = 1 head results per distinct (x, z, u) triple of pool indices (u None: no update), with the
    cls_dw / x_reg intermediates of the same call."""

    def __init__(self, net, X, Z, U):
        self.net, self.X, self.Z, self.U, self.cache = net, X, Z, U, {}

    def get(self, key):
        if key not in self.cache:
            xi, zi, ui = key
            u = None if ui is None else self.U[ui:ui + 1]
            bbox, cls = head(self.net, self.Z[zi:zi + 1], self.X[xi:xi + 1], u)
            self.cache[key] = (bbox, cls, self.net.head_tensor("cls_dw", 1), self.net.head_tensor("x_reg", 1))
        return self.cache[key]


def oracle_errors(sd, keys, X, Z, U, outputs):
    """Per-frame comparison of head outputs with fp64 BoxTower.forward: outputs[k] = (bbox, cls[, cls_dw, x_reg]) of
    triple keys[k].  Returns the worst inf-norm error per map, the worst allclose ratio
    |a - b| / (TOL |b| + 1e-5 ||b||inf) (<= 1 passes), and the argmax mismatches with their oracle margins."""
    res = {"frames": len(keys), "inf": {}, "allclose_ratio": {}, "argmax_mismatch": []}
    for with_u in (False, True):
        ks = [i for i, k in enumerate(keys) if (k[2] is not None) == with_u]
        if not ks:
            continue
        xi = torch.tensor([keys[i][0] for i in ks])
        zi = torch.tensor([keys[i][1] for i in ks])
        x, z = X[xi.cuda()].cpu().double(), Z[zi.cuda()].cpu().double()
        u = U[torch.tensor([keys[i][2] for i in ks]).cuda()].cpu().double() if with_u else None
        with torch.no_grad():
            want = fo.box_tower(sd, x, z, u)
        for j, i in enumerate(ks):
            got = outputs[i]
            for name, a, b in zip(("reg", "cls", "cls_dw", "x_reg"), got, want):
                a, b = a[0].cpu().numpy().astype(np.float64), b[j].numpy()
                e2 = map_errors(a, b)[1]
                res["inf"][name] = max(res["inf"].get(name, 0.0), e2)
                if name in ("reg", "cls"):
                    ratio = float((np.abs(a - b) / (TOL * np.abs(b) + 1e-5 * np.abs(b).max())).max())
                    res["allclose_ratio"][name] = max(res["allclose_ratio"].get(name, 0.0), ratio)
            top2 = want[1][j].flatten().topk(2).values
            margin = float(top2[0] - top2[1])
            if int(got[1].flatten().argmax()) != int(want[1][j].flatten().argmax()):
                res["argmax_mismatch"].append({"key": list(keys[i]), "margin": margin})
    return res


def check_refs(sd, refs):
    keys = list(refs.cache)
    return oracle_errors(sd, keys, refs.X, refs.Z, refs.U, [refs.cache[k] for k in keys])


# ----------------------------------------------------------------------------------------------------------- groups
def group_matrix():
    """fear_head / fear_head_update over B, Bz in {1, B}, Bu in {none, 1, B}, unchunked and at R = 4."""
    full = make_net(POOL)
    X, Z, U = feature_pools(full, POOL)
    refs, bits = HeadRefs(full, X, Z, U), BitCheck()
    nets = {0: full, 4: make_net(4)}
    for R_, batches in MATRIX.items():
        net = nets[R_]
        for B in batches:
            start = (5 * B + R_) % POOL  # frames at different pool positions for every call
            idx = [(start + k) % POOL for k in range(B)]
            zb = (start + B) % POOL  # the broadcast template (and update template) of this call
            xs = X[idx]
            for bz in sorted({1, B}):
                z = Z[[zb]] if bz == 1 else Z[idx]
                zkey = [zb] * B if bz == 1 else idx
                reg_by_update = []
                for bu in [None] + sorted({1, B}):
                    u = None if bu is None else (U[[zb]] if bu == 1 else U[idx])
                    ukey = [None] * B if bu is None else ([zb] * B if bu == 1 else idx)
                    bbox, cls = head(net, z, xs, u)
                    tag = f"R={R_} B={B} Bz={bz} Bu={bu}"
                    for k in range(B):
                        rb, rc, _, _ = refs.get((idx[k], zkey[k], ukey[k]))
                        bits.eq(bbox[k:k + 1], rb, f"{tag} frame {k} reg")
                        bits.eq(cls[k:k + 1], rc, f"{tag} frame {k} cls")
                    if B > 1 and (bz == 1 or bu == 1):  # broadcast == the template(s) expanded to B rows
                        ze = z.expand(B, -1, -1, -1).contiguous()
                        ue = None if u is None else u.expand(B, -1, -1, -1).contiguous()
                        eb, ec = head(net, ze, xs, ue)
                        bits.eq(eb, bbox, f"{tag} expanded templates reg")
                        bits.eq(ec, cls, f"{tag} expanded templates cls")
                    if bu is None:  # fear_head_update(update = NULL) is fear_head
                        hb, hc = maps(B)
                        _lib.check(_lib.load().fear_head_update(net._handle, z.data_ptr(), z.shape[0], None, 0,
                                                                xs.data_ptr(), B, hb.data_ptr(), hc.data_ptr(),
                                                                stream()), "fear_head_update")
                        bits.eq(hb, bbox, f"{tag} fear_head_update(NULL) reg")
                        bits.eq(hc, cls, f"{tag} fear_head_update(NULL) cls")
                    reg_by_update.append(bbox)
                for k, other in enumerate(reg_by_update[1:]):  # the regression map ignores the update template
                    bits.eq(other, reg_by_update[0], f"R={R_} B={B} Bz={bz} reg with update #{k + 1}")
    torch.cuda.synchronize()
    res = bits.report()
    res["oracle"] = check_refs(sd64(), refs)
    return res


def track_call(net, entry, search, z, B, want_maps=True, want_boxes=True):
    """fear_track / fear_track_u8 / fear_forward through the C ABI; z is template features or (forward) crops."""
    bbox, cls = maps(B) if want_maps else (None, None)
    boxes = torch.empty((B, _lib.BOX_DTYPE.itemsize), device="cuda", dtype=torch.uint8) if want_boxes else None
    lib = _lib.load()
    if entry == "forward":
        rc = lib.fear_forward(net._handle, z.data_ptr(), search.data_ptr(), B, ptr(bbox), ptr(cls), ptr(boxes), stream())
    else:
        fn = lib.fear_track_u8 if entry == "track_u8" else lib.fear_track
        rc = fn(net._handle, search.data_ptr(), z.data_ptr(), z.shape[0], B, ptr(bbox), ptr(cls), ptr(boxes), stream())
    _lib.check(rc, entry)
    return bbox, cls, boxes


def decode(bbox, cls, apply_sigmoid=1):
    B = bbox.shape[0]
    boxes = torch.empty((B, _lib.BOX_DTYPE.itemsize), device="cuda", dtype=torch.uint8)
    _lib.check(_lib.load().fear_decode(bbox.data_ptr(), cls.data_ptr(), B, apply_sigmoid, boxes.data_ptr(), stream()),
               "fear_decode")
    return boxes


def group_track():
    """fear_track / fear_track_u8 / fear_forward at B in {1, 3, 9}, unchunked and at R = 4, against fear_head of
    per-frame features; boxes-only / maps-only / both; 3 frames against the end-to-end fp64 oracle."""
    n = 9
    full, r4 = make_net(n), make_net(4)
    tc, xt, _, xu = fo.synthetic_crops(n)
    xs, ts = xt.cuda(), tc.cuda()
    xu8 = xu.permute(0, 2, 3, 1).contiguous().cuda()
    xf = torch.cat([full.get_features(xs[i:i + 1]) for i in range(n)])
    zf = torch.cat([full.get_features(ts[i:i + 1]) for i in range(n)])
    bits = BitCheck()
    ref = {}  # (search frame, template frame) -> B = 1 fear_head maps

    def want(i, j):
        if (i, j) not in ref:
            ref[(i, j)] = head(full, zf[j:j + 1], xf[i:i + 1])
        return ref[(i, j)]

    for R_, net in ((0, full), (4, r4)):
        for B in (1, 3, 9):
            start = {1: 5, 3: 2, 9: 0}[B]
            idx = [(start + k) % n for k in range(B)]
            zb = (start + B + 1) % n
            # (Bz, template features or crops, template frame of each position); forward computes a per-frame template's
            # features inside the chunk loop
            cases = [(1, "track", zf[[zb]], [zb] * B), (B, "track", zf[idx], idx), (B, "forward", ts[idx], idx)]
            for bz, kind, z, zkey in cases[1:] if B == 1 else cases:
                tag = f"R={R_} B={B} Bz={bz}"
                entries = (("forward", xs[idx]),) if kind == "forward" else (("track", xs[idx]), ("track_u8", xu8[idx]))
                runs = {}
                for entry, search in entries:
                    runs[entry + " both"] = track_call(net, entry, search, z, B)
                    runs[entry + " maps"] = track_call(net, entry, search, z, B, want_boxes=False)
                    runs[entry + " boxes"] = track_call(net, entry, search, z, B, want_maps=False)
                for name, (bbox, cls, boxes) in runs.items():
                    if bbox is not None:
                        for k in range(B):
                            rb, rcl = want(idx[k], zkey[k])
                            bits.eq(bbox[k:k + 1], rb, f"{tag} {name} frame {k} reg")
                            bits.eq(cls[k:k + 1], rcl, f"{tag} {name} frame {k} cls")
                    if boxes is not None:
                        rb = torch.cat([want(idx[k], zkey[k])[0] for k in range(B)])
                        rcl = torch.cat([want(idx[k], zkey[k])[1] for k in range(B)])
                        bits.eq(boxes, decode(rb, rcl), f"{tag} {name} records == fear_decode of the maps")
    torch.cuda.synchronize()
    res = bits.report()
    # end to end: crops -> maps against the fp64 oracle for 3 frames (unchunked, B = 3 per-frame templates)
    sd = sd64()
    with torch.no_grad():
        oracle = fo.track(sd, xt[:3].double(), fo.get_features(sd, tc[:3].double()))
    got = {R: torch.cat([want(i, i)[0] for i in range(3)]).cpu().double(),
           C: torch.cat([want(i, i)[1] for i in range(3)]).cpu().double()}
    e2e = {"inf": {}, "allclose_ratio": {}, "argmax_mismatch": []}
    for key, name in ((R, "reg"), (C, "cls")):
        for k in range(3):
            a, b = got[key][k].numpy(), oracle[key][k].numpy()
            e2e["inf"][name] = max(e2e["inf"].get(name, 0.0), map_errors(a, b)[1])
            ratio = float((np.abs(a - b) / (TOL * np.abs(b) + 1e-5 * np.abs(b).max())).max())
            e2e["allclose_ratio"][name] = max(e2e["allclose_ratio"].get(name, 0.0), ratio)
    for k in range(3):
        top2 = oracle[C][k].flatten().topk(2).values
        if int(got[C][k].flatten().argmax()) != int(oracle[C][k].flatten().argmax()):
            e2e["argmax_mismatch"].append({"key": [k], "margin": float(top2[0] - top2[1])})
    res["oracle_end_to_end"] = e2e
    return res


def group_host():
    """track_boxes_from_host: B = 7, chunks 1 and 3 (slices 2, 2, 3), Bz in {1, 7}; two calls back to back without
    synchronisation must both equal track_boxes of their own inputs."""
    B = 7
    net = make_net(B)
    sets = []
    for seed in (101, 202):
        tc, xt, _, xu = fo.synthetic_crops(B, seed=seed)
        zf = net.get_features(tc.cuda())
        sets.append(dict(xdev=xt.cuda(), xhost=xu.permute(0, 2, 3, 1).contiguous().pin_memory(), z=zf,
                         zhost=zf.cpu().pin_memory()))
    bits = BitCheck()
    for chunks in (1, 3):
        for bz in (1, B):
            out_host = torch.empty((B, _lib.BOX_DTYPE.itemsize), dtype=torch.uint8).pin_memory()
            got = [net.track_boxes_from_host(s["xhost"], s["zhost"][:bz], out_host=out_host if k else None,
                                             chunks=chunks) for k, s in enumerate(sets)]
            torch.cuda.synchronize()
            want = [net.track_boxes(s["xdev"], s["z"][:bz]) for s in sets]
            torch.cuda.synchronize()
            for k in range(2):
                bits.eq(got[k], want[k], f"chunks={chunks} Bz={bz} call {k}")
            bits.eq(out_host, want[1].cpu(), f"chunks={chunks} Bz={bz} out_host")
            if torch.equal(want[0], want[1]):  # else a mixed-up staging set could go unnoticed
                bits.failures.append(f"chunks={chunks} Bz={bz}: the two input sets decode to the same records")
    return bits.report()


def group_options():
    """Head option variants at B = 3 (unchunked) and B = 5 (R = 4), Bz = 1, Bu = B: fuse_dwpw = 13 (head SepConv
    fusion off) is bit-identical to the default; pw x corr in {ffma, wgmma} meet the oracle bars."""
    n = 5
    full = make_net(n)
    X, Z, U = feature_pools(full, n + 1)
    refs, bits = HeadRefs(full, X, Z, U), BitCheck()
    sd = sd64()
    res = {"variants": {}}
    for R_, B, net in ((0, 3, full), (4, 5, make_net(4))):
        idx = list(range(B))
        zb = n
        xs, z, u = X[idx], Z[[zb]], U[idx]
        keys = [(i, zb, i) for i in idx]
        base = head(net, z, xs, u)
        for k in range(B):
            rb, rc, _, _ = refs.get(keys[k])
            bits.eq(base[0][k:k + 1], rb, f"R={R_} B={B} default frame {k} reg")
            bits.eq(base[1][k:k + 1], rc, f"R={R_} B={B} default frame {k} cls")
        net.set_option("fuse_dwpw", "13")
        poison_workspace(net)  # each variant may not pass on values an earlier run left in the workspace
        try:
            got = head(net, z, xs, u)
        finally:
            net.set_option("fuse_dwpw", "15")
        bits.eq(got[0], base[0], f"R={R_} B={B} fuse_dwpw=13 reg")
        bits.eq(got[1], base[1], f"R={R_} B={B} fuse_dwpw=13 cls")
        for pw in ("ffma", "wgmma"):
            for corr in ("ffma", "wgmma"):
                net.set_option("pw", pw)
                net.set_option("corr", corr)
                poison_workspace(net)
                try:
                    bbox, cls = head(net, z, xs, u)
                finally:
                    net.set_option("pw", "auto")
                    net.set_option("corr", "auto")
                outs = [(bbox[k:k + 1], cls[k:k + 1]) for k in range(B)]
                res["variants"][f"R={R_} B={B} pw={pw} corr={corr}"] = oracle_errors(sd, keys, X, Z, U, outs)
    torch.cuda.synchronize()
    res.update(bits.report())
    res["oracle"] = check_refs(sd, refs)
    return res


def group_launches():
    """Kernel launches of one fear_head / fear_head_update call per (R, B, Bz, Bu), and the argument checks."""
    nets = {0: make_net(POOL), 4: make_net(4)}
    X, Z, U = feature_pools(nets[0], POOL, magnitudes=False)
    rows = []
    for R_, batches in MATRIX.items():
        net = nets[R_]
        for B in batches:
            for bz in sorted({1, B}):
                for bu in [None] + sorted({1, B}):
                    z = Z[:bz]
                    u = None if bu is None else U[:bu]
                    n0 = net.launch_count()
                    head(net, z, X[:B], u)
                    rows.append({"R": R_, "B": B, "Bz": bz, "Bu": bu, "launches": net.launch_count() - n0})
    # refused arguments: FEAR_EINVAL before any launch (buffers sized so that even a wrongly accepted call stays in
    # bounds of its inputs)
    net, B = nets[4], 3
    lib = _lib.load()
    bbox, cls = maps(B)
    z4, u4, x = Z[:4], U[:4], X[:B]
    calls = {
        "Bz=0": (z4, 0, None, 0, B, bbox, cls), "Bz=2": (z4, 2, None, 0, B, bbox, cls),
        "Bz=4": (z4, 4, None, 0, B, bbox, cls), "Bz=2 update": (z4, 2, u4, B, B, bbox, cls),
        "Bu=0": (z4, B, u4, 0, B, bbox, cls), "Bu=2": (z4, B, u4, 2, B, bbox, cls), "Bu=4": (z4, 1, u4, 4, B, bbox, cls),
        "bbox=NULL": (z4, B, u4, B, B, None, cls), "cls=NULL": (z4, B, u4, B, B, bbox, None),
        "bbox=cls=NULL": (z4, 1, None, 0, B, None, None), "B=0": (z4, 1, u4, 1, 0, bbox, cls),
        "B=-1": (z4, 1, None, 0, -1, bbox, cls),
    }
    refused = {}
    for name, (z, bz, u, bu, b, bb, cc) in calls.items():
        n0 = net.launch_count()
        rc = lib.fear_head_update(net._handle, z.data_ptr(), bz, ptr(u), bu, x.data_ptr(), b, ptr(bb), ptr(cc), stream())
        refused[name] = {"rc": rc, "launches": net.launch_count() - n0}
    n0 = net.launch_count()
    refused["fear_head Bz=2"] = {"rc": lib.fear_head(net._handle, z4.data_ptr(), 2, x.data_ptr(), B, bbox.data_ptr(),
                                                     cls.data_ptr(), stream()), "launches": net.launch_count() - n0}
    head(net, Z[:1], x, U[:B])  # the handle still works afterwards
    torch.cuda.synchronize()
    return {"rows": rows, "refused": refused, "einval": FEAR_EINVAL}


# ---------------------------------------------------------------------------------------------------------- decode
NAN, INF = float("nan"), float("inf")


def decode_cases():
    """Constructed cls rows (256 logits each): name -> tensor.  Background is standard normal * 0.5 (|x| < 3)."""
    g = torch.Generator().manual_seed(404)
    cases = {}

    def row(background=None, **at):
        r = 0.5 * torch.randn(256, generator=g) if background is None else torch.full((256,), float(background))
        for k, v in at.items():
            r[int(k[1:])] = v
        return r

    cases["tie_in_warp"] = row(i9=5.0, i20=5.0)
    cases["tie_in_warp_high_lane_first"] = row(i52=5.0, i33=5.0)
    cases["tie_across_warps"] = row(i70=5.0, i200=5.0, i130=5.0)
    cases["tie_index_0_and_255"] = row(i0=5.0, i255=5.0)
    cases["tie_index_255_only_max"] = row(i255=5.0)
    cases["all_equal"] = row(0.25)
    cases["neg_zero_before_zero"] = row(-1.0, i3=-0.0, i17=0.0)
    cases["zero_before_neg_zero"] = row(-1.0, i3=0.0, i17=-0.0)
    cases["pos_saturation"] = row(i40=17.0, i200=100.0)
    r = -90.0 - 50.0 * torch.rand(256, generator=g)
    r[0], r[150] = -135.0, -90.0
    cases["neg_saturation"] = r
    cases["denormal"] = row(-100.0, i3=-88.5, i77=-88.0)
    cases["denormal_reversed"] = row(-100.0, i3=-88.0, i77=-88.5)
    cases["pos_inf"] = row(i123=INF, i50=1e30)
    cases["pos_inf_only"] = row(i123=INF)
    cases["neg_inf"] = row(i0=-INF, i1=-INF)
    cases["all_neg_inf"] = row(-INF)
    cases["nan_0_alone"] = row(i0=NAN)
    cases["nan_5_alone"] = row(i5=NAN)
    cases["nan_32_alone"] = row(i32=NAN)
    cases["nan_0_larger_later"] = row(i0=NAN, i100=3.0)
    cases["nan_5_larger_later"] = row(i5=NAN, i100=3.0)
    cases["nan_32_larger_later"] = row(i32=NAN, i100=3.0)
    cases["nan_5_and_32"] = row(i32=NAN, i5=NAN, i100=3.0)
    cases["nan_200_and_inf"] = row(i200=NAN, i7=INF)
    cases["all_nan"] = row(NAN)
    return cases


def expected_decode(reg, cls, apply_sigmoid):
    """torch on the same CUDA device: expected scores, argmax, score at the argmax and float64 boxes (fo.make_grid)."""
    scores = (cls.sigmoid() if apply_sigmoid else cls).reshape(cls.shape[0], 256)
    flat = scores.argmax(1)
    score = scores.gather(1, flat[:, None])[:, 0]
    gx, gy = (g.reshape(256).cuda() for g in fo.make_grid(16, 16, 256))
    r = reg.reshape(reg.shape[0], 4, 256).double()
    pick = [r[:, c].gather(1, flat[:, None])[:, 0] for c in range(4)]
    x1, y1 = gx[flat] - pick[0], gy[flat] - pick[1]
    x2, y2 = gx[flat] + pick[2], gy[flat] + pick[3]
    return flat, score, torch.stack([x1, y1, x2 - x1, y2 - y1], 1)


def group_decode():
    """fear_decode with apply_sigmoid 1 and 0 at B = 1 (every constructed row alone), B = 7 and B = 70 000 (past the
    65 535 limit of a grid's y / z dimension) against torch.argmax / torch.sigmoid on the same device."""
    cases = decode_cases()
    names = list(cases)
    g = torch.Generator().manual_seed(405)
    B_big = 70000
    big = 2.0 * torch.randn(B_big, 256, generator=g)
    big[::3] = torch.randint(-6, 7, (len(big[::3]), 256), generator=g).float() / 4  # many exact ties
    places = [0, 1, 31, 32, 4095, 65534, 65535, 65536, 65537, 69000]
    places += list(range(69999 - (len(names) - len(places)) + 1, 70000))
    for p, name in zip(places, names):
        big[p] = cases[name]
    reg_big = 60.0 * torch.rand(B_big, 4, 256, generator=g)
    # inf in the regression map at the decoded cell: tie_index_0_and_255, pos_saturation (sigmoid), tie_in_warp
    reg_big[places[names.index("tie_index_0_and_255")], 0, 0] = INF
    reg_big[places[names.index("pos_saturation")], 2, 40] = INF
    reg_big[places[names.index("tie_in_warp")], 1, 9] = -INF
    batches = {"B=7": (torch.stack([cases[n] for n in names[:7]]), reg_big[places[:7]]),
               "B=70000": (big, reg_big)}
    for n in names:
        batches[f"B=1 {n}"] = (cases[n][None], reg_big[places[names.index(n)]][None])
    res = {"mismatch": [], "score_not_bit_identical": [], "ulp_fail": [], "box_mismatch": [], "rows": 0,
           "max_ulp_vs_cpu": 0.0, "case_results": {}}
    for label, (cls2d, reg) in batches.items():
        B = cls2d.shape[0]
        cls = cls2d.reshape(B, 1, 16, 16).cuda()
        regd = reg.reshape(B, 4, 16, 16).contiguous().cuda()
        for aps in (1, 0):
            rec = decode(regd, cls, aps).cpu().numpy().view(_lib.BOX_DTYPE).reshape(-1)
            flat, score, box = expected_decode(regd, cls, aps)
            flat, score, box = flat.cpu().numpy(), score.cpu().numpy(), box.cpu().numpy()
            res["rows"] += B
            bad = np.nonzero((rec["flat"] != flat) | (rec["row"] != flat // 16) | (rec["col"] != flat % 16))[0]
            res["mismatch"] += [{"batch": label, "sigmoid": aps, "frame": int(i), "got": int(rec["flat"][i]),
                                 "want": int(flat[i])} for i in bad[:10]]
            same = (rec["score"].view(np.uint32) == score.view(np.uint32)) | (np.isnan(rec["score"]) & np.isnan(score))
            res["score_not_bit_identical"] += [{"batch": label, "sigmoid": aps, "frame": int(i),
                                                "got": float(rec["score"][i]), "want": float(score[i])}
                                               for i in np.nonzero(~same)[0][:10]]
            got_box = np.stack([rec["x"], rec["y"], rec["w"], rec["h"]], 1)
            box_ok = ((got_box == box) | (np.isnan(got_box) & np.isnan(box))).all(1)
            res["box_mismatch"] += [{"batch": label, "sigmoid": aps, "frame": int(i)} for i in np.nonzero(~box_ok)[0][:10]]
            if aps:  # score within 2 ulp of CPU torch.sigmoid, denormal spacing included (not at the expf overflow edge)
                logit = cls2d.gather(1, torch.from_numpy(flat).long()[:, None])[:, 0].numpy()
                cpu = torch.sigmoid(torch.from_numpy(logit)).numpy()
                keep = ~np.isnan(logit) & (np.abs(np.abs(logit) - 88.72) >= 0.05)
                ulps = np.abs(rec["score"].astype(np.float64) - cpu.astype(np.float64)) / np.spacing(np.abs(cpu))
                if keep.any():
                    res["max_ulp_vs_cpu"] = max(res["max_ulp_vs_cpu"], float(np.nan_to_num(ulps[keep], nan=np.inf).max()))
                res["ulp_fail"] += [{"batch": label, "frame": int(i), "got": float(rec["score"][i]),
                                     "cpu": float(cpu[i]), "ulp": float(ulps[i])}
                                    for i in np.nonzero(keep & ~(ulps <= 2))[0][:10]]
            if label.startswith("B=1 "):
                res["case_results"][f"{label[4:]} sigmoid={aps}"] = [int(rec["flat"][0]), float(rec["score"][0])]
                # fo.decode (the reference decode) on the expected scores: same cell, float64 boxes bit for bit
                scores = (cls.sigmoid() if aps else cls).cpu()
                bbox, coords = fo.decode(regd.cpu(), scores, use_sigmoid=False)
                if coords != [(int(rec["row"][0]), int(rec["col"][0]))] or not (
                        (bbox.numpy() == got_box) | (np.isnan(bbox.numpy()) & np.isnan(got_box))).all():
                    res["box_mismatch"].append({"batch": label, "sigmoid": aps, "vs": "fo.decode",
                                                "coords": [list(c) for c in coords]})
    return res


GROUPS = {"matrix": group_matrix, "track": group_track, "host": group_host, "options": group_options,
          "launches": group_launches, "decode": group_decode}


def main():
    torch.manual_seed(0)
    res = GROUPS[sys.argv[1]]()
    print("HEAD_CHECK " + json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
