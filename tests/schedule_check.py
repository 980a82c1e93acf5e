"""Stand-alone checker of the persistent kernels' tile schedules (run in its own process: a device-side trap would poison
the CUDA context of the main pytest process).  Prints one JSON line.

    python tests/schedule_check.py features H W   # get_features_u8 at one crop size
    python tests/schedule_check.py track          # fear_track_u8 (256 x 256 search, template batch Bz = B)
    python tests/schedule_check.py large          # one chunk whose workspace passes 2^31 floats

Inputs: 7 distinct seeded crops (oracle.fear_oracle.shape_crops); frame i of a batch is input i mod 7.  Each input is
first run at B = 1 and checked against the fp64 oracle (block by block through fear_debug_backbone_prefix, features,
maps).  Then, at every batch tests/schedule_plan.py picks for the S SMs of this device -- the smallest batch that puts
each persistent launch into each scheduling regime -- the call runs on a workspace poisoned with POISON_A and again with
POISON_B (outputs pre-filled with the same word), and every frame must equal its B = 1 result bit for bit.  Option
variants run at each of their batches that gives some CTA two or more tiles: the variants that promise the default's
arithmetic must equal the default's B = 1 results; pw=ffma and corr=ffma, which compute differently, their own B = 1
results (checked against the oracle at the same bars).  The launch count of every (size, options) call must equal the
planner's model.  A frame that differs is located: the first backbone block whose output differs at that batch, and
the tile, CTA, iteration, ring stage and consumer group the planner assigns to the first differing pixel.
"""
import contextlib
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import feartracker_b200 as fb  # noqa: E402
from feartracker_b200 import _lib  # noqa: E402
from oracle import fear_oracle as fo  # noqa: E402
from tests import schedule_plan as sp  # noqa: E402
from tests.helpers import POISON_A, POISON_B, TOL, load_full_state, map_errors, poison_workspace  # noqa: E402

N_INPUTS = 7
SEARCH_SEEDS = [701 + i for i in range(N_INPUTS)]
TEMPLATE_SEEDS = [801 + i for i in range(N_INPUTS)]
POISONS = {"A": (POISON_A, 0xA5), "B": (POISON_B, 0x5A)}
BLOCK_TOL, FEAT_TOL, FEAT_INF_TOL, HEAD_INF_TOL, MARGIN = 2e-5, 2e-2, 2e-5, 1e-4, 1e-4  # the bars of the other checks
BLOCK_NAMES = ["xif0_0"] + [b[0] for b in sp.BLOCKS]
MAX_REPORTED = 40


def stream():
    return torch.cuda.current_stream().cuda_stream


def num_sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def make_net(reserve):
    net = fb.FEARNet(**fb.FEAR_XS_MODEL_KWARGS)
    net.load_state_dict(load_full_state(), strict=True)
    net = net.cuda().eval()
    net.reserve(reserve)
    net._ensure_handle(torch.device("cuda", torch.cuda.current_device()))
    return net


def sd64():
    return fo.to_dtype({k: v for k, v in load_full_state().items() if v.is_floating_point()}, torch.float64)


@contextlib.contextmanager
def options(net, opts):
    try:
        for k, v in opts.items():
            net.set_option(k, v)
        yield
    finally:
        for k in opts:
            net.set_option(k, sp.DEFAULTS[k])


def inputs(H, W, seeds):
    xs, us = zip(*(fo.shape_crops(H, W, 1, seed=s) for s in seeds))
    x = torch.cat(xs)
    return x, torch.cat(us).permute(0, 2, 3, 1).contiguous()


class Report:
    def __init__(self):
        self.failures, self.n_failures, self.runs, self.worst = [], 0, 0, {}

    def fail(self, what):
        self.n_failures += 1
        if len(self.failures) < MAX_REPORTED:
            self.failures.append(what)

    def error(self, key, value, bar, what):
        self.worst[key] = max(self.worst.get(key, 0.0), float(value))
        if not value <= bar:
            self.fail(f"{what}: {key} {value:.3e} above {bar:g}")

    def dump(self):
        return {"failures": self.failures, "n_failures": self.n_failures, "runs": self.runs, "worst": self.worst}


# ------------------------------------------------------------------------------------------------------ entry points
def features_u8(net, u, word_byte):
    """fear_get_features_u8 on a workspace and an output filled with the poison word."""
    word, _ = word_byte
    B, H, W, _ = u.shape
    poison_workspace(net, word)
    out = torch.full((B, 256, H // 16, W // 16), word, dtype=torch.int32, device="cuda").view(torch.float32)
    _lib.check(_lib.load().fear_get_features_u8(net._handle, u.data_ptr(), B, H, W, out.data_ptr(), stream()),
               "fear_get_features_u8")
    return [out]


def track_u8(net, u, z, word_byte):
    """fear_track_u8 with maps and FearBox records, template batch z.shape[0], on poisoned workspace and outputs."""
    word, byte = word_byte
    B = u.shape[0]
    poison_workspace(net, word)
    bbox = torch.full((B, 4, 16, 16), word, dtype=torch.int32, device="cuda").view(torch.float32)
    cls = torch.full((B, 1, 16, 16), word, dtype=torch.int32, device="cuda").view(torch.float32)
    boxes = torch.full((B, _lib.BOX_DTYPE.itemsize), byte, dtype=torch.uint8, device="cuda")
    _lib.check(_lib.load().fear_track_u8(net._handle, u.data_ptr(), z.data_ptr(), z.shape[0], B, bbox.data_ptr(),
                                         cls.data_ptr(), boxes.data_ptr(), stream()), "fear_track_u8")
    return [bbox, cls, boxes]


def launches_of(net, fn):
    n0 = net.launch_count()
    fn()
    torch.cuda.synchronize()
    return net.launch_count() - n0


def bad_frames(got, want):
    """Frames where any output differs from the expected one (bitwise: NaN payloads count)."""
    bad = torch.zeros(got[0].shape[0], dtype=torch.bool, device=got[0].device)
    for g, w in zip(got, want):
        g8, w8 = g.contiguous().view(torch.uint8), w.contiguous().view(torch.uint8)
        bad |= (g8 != w8).reshape(g8.shape[0], -1).any(1)
    return bad.nonzero().flatten().tolist()


def locate(net, x1, idx, f, opts, H, W, S):
    """First backbone block whose output for frame f differs between the batch and B = 1, and the tile / CTA the planner
    assigns to its first differing pixel (fear_debug_backbone_prefix: the plain stem, then the same blocks)."""
    xb = x1[idx].cuda()
    B = len(idx)
    plan = sp.launches("backbone_prefix", H, W, opts)
    for n, name in enumerate(BLOCK_NAMES):
        poison_workspace(net, POISON_A)
        pb = net.backbone_prefix(xb, n)[f]
        poison_workspace(net, POISON_A)
        p1 = net.backbone_prefix(xb[f:f + 1], n)[0]
        diff = (pb.view(torch.int32) != p1.view(torch.int32)).nonzero()
        if not len(diff):
            continue
        c, y, x = (int(v) for v in diff[0])
        owners = []
        for ln in plan:
            if ln.persistent and ln.name.split(" ")[0].split(".")[0] == name:
                owners += [dict(sp.tile_owner(ln, B, S, f, y, x, cb), launch=ln.name, kernel=ln.kernel, cb=cb)
                           for cb in range(ln.cblocks)]
        return {"first_bad_block": name, "pixel": [c, y, x], "differing_values": int(len(diff)), "owners": owners[:8]}
    return {"first_bad_block": None, "note": "every backbone block matches: the difference is after the backbone"}


def sweep(rep, net, run, expected, batches, variants, entry, H, W, S, x_float, located):
    """Run `run(idx, poison)` at every batch: the default at every planned batch with both poisons, each variant at its
    multi-lap batches; every frame must equal expected[variant][input]."""
    for vname, opts in variants:
        own = vname if vname in expected else "default"
        mine = [B for B in batches if not opts or sp.multi_lap(entry, B, H, W, opts, S)] or [max(batches)]
        for B in mine:
            idx = [i % N_INPUTS for i in range(B)]
            want = [e[idx] for e in expected[own]]
            for pname, pw in POISONS.items():
                with options(net, opts):
                    got = run(idx, pw)
                    torch.cuda.synchronize()
                    rep.runs += 1
                    bad = bad_frames(got, want)
                    if bad:
                        f = bad[0]
                        where = {"variant": vname, "B": B, "poison": pname, "bad_frames": bad[:16],
                                 "n_bad_frames": len(bad), "frame": f, "input": idx[f]}
                        if x_float is not None and len(located) < 3:  # a few locations say enough
                            located[(vname, B, pname)] = True
                            where.update(locate(net, x_float, idx, f, opts, H, W, S))
                        rep.fail(where)


def dispatch(rep, net, entry, variants, fn, H=256, W=256, **kw):
    """Launch count of one call per option set == the planner's launch list."""
    out = {}
    for vname, opts in variants:
        with options(net, opts):
            got = launches_of(net, fn)
        want = len(sp.launches(entry, H, W, opts, **kw))
        out[vname] = [got, want]
        if got != want:
            rep.fail(f"{entry} {H}x{W} {vname}: {got} launches, the planner models {want}")
    return out


# ---------------------------------------------------------------------------------------------------------- features
def check_features(H, W):
    S, sd, rep = num_sms(), sd64(), Report()
    variants = sp.all_variants("features")
    batches = sp.planned("get_features", H, W, variants, S)
    net = make_net(max(batches))
    x1, u1 = inputs(H, W, SEARCH_SEEDS)
    res = {"mode": "features", "H": H, "W": W, "S": S, "batches": batches}

    # B = 1 against the fp64 oracle, for the default and for pw=ffma (its own arithmetic)
    cols = []
    for i in range(N_INPUTS):
        col = {}
        with torch.no_grad():
            fo.get_features(sd, x1[i:i + 1].double(), col)
        cols.append(col)
    expected = {}
    for vname, opts in [("default", {})] + [(f"{k}={v}", {k: v}) for k, v in sp.OWN_REFERENCE["features"]]:
        outs = []
        with options(net, opts):
            for i in range(N_INPUTS):
                xc, col, tag = x1[i:i + 1].cuda(), cols[i], f"{vname} input {i} B=1"
                for n, blk in enumerate(BLOCK_NAMES):
                    e2 = map_errors(net.backbone_prefix(xc, n).cpu().numpy(), col[blk].numpy())[1]
                    rep.error("block_inf", e2, BLOCK_TOL, f"{tag} {blk}")
                gf, fe = net.get_features(xc), net.feature_extractor(xc)
                for what, got, key in (("get_features", gf, "neck"), ("feature_extractor", fe, "xif4_7")):
                    e1, e2 = map_errors(got.cpu().numpy(), col[key].numpy())
                    rep.error(f"{what}_rel", e1, FEAT_TOL, f"{tag} {what}")
                    rep.error(f"{what}_inf", e2, FEAT_INF_TOL, f"{tag} {what}")
                a, b = (features_u8(net, u1[i:i + 1].cuda(), p)[0] for p in POISONS.values())
                if not (torch.equal(a, b) and torch.equal(a, gf)):
                    rep.fail(f"{tag}: uint8 features differ between poisons or from the float-input features")
                outs.append(a)
        expected[vname] = [torch.cat(outs)]
    res["oracle_worst"] = dict(rep.worst)

    u1c = u1.cuda()
    res["dispatch"] = dispatch(rep, net, "get_features", variants, lambda: features_u8(net, u1c[:1], POISONS["A"]),
                               H, W)
    sweep(rep, net, lambda idx, p: features_u8(net, u1c[idx], p), expected, list(batches), variants,
          "get_features", H, W, S, x1, {})
    res.update(rep.dump())
    return res


# ------------------------------------------------------------------------------------------------------------- track
def track_refs(rep, net, sd, x1, u1, t1, variants, oracle=True):
    """Template features (B = 1 each) and the B = 1 track results of every own-reference variant; maps checked against
    the fp64 oracle (fo.track on the oracle's own template features)."""
    z1 = torch.cat([net.get_features(t1[i:i + 1].cuda()) for i in range(N_INPUTS)])
    wants = []
    if oracle:
        with torch.no_grad():
            wants = [fo.track(sd, x1[i:i + 1].double(), fo.get_features(sd, t1[i:i + 1].double()))
                     for i in range(N_INPUTS)]
    expected = {}
    for vname, opts in variants:
        outs = []
        with options(net, opts):
            for i in range(N_INPUTS):
                a, b = (track_u8(net, u1[i:i + 1].cuda(), z1[i:i + 1], p) for p in POISONS.values())
                if not all(torch.equal(p, q) for p, q in zip(a, b)):
                    rep.fail(f"track {vname} input {i} B=1: results differ between poisons")
                outs.append(a)
                if not oracle:
                    continue
                tag = f"track {vname} input {i} B=1"
                for key, got in ((fo.TARGET_REGRESSION_LABEL_KEY, a[0]), (fo.TARGET_CLASSIFICATION_KEY, a[1])):
                    g, w = got[0].cpu().double().numpy(), wants[i][key][0].numpy()
                    rep.error("map_inf", map_errors(g, w)[1], HEAD_INF_TOL, f"{tag} {key}")
                    if not (np.abs(g - w) <= TOL * np.abs(w) + 1e-5 * np.abs(w).max()).all():
                        rep.fail(f"{tag} {key}: outside the allclose bar")
                wc = wants[i][fo.TARGET_CLASSIFICATION_KEY][0].flatten()
                top2 = wc.topk(2).values
                if float(top2[0] - top2[1]) >= MARGIN and int(a[1][0].flatten().argmax()) != int(wc.argmax()):
                    rep.fail(f"{tag}: argmax differs from the oracle")
        expected[vname] = [torch.cat([o[k] for o in outs]) for k in range(3)]
    return z1, expected


def check_track():
    S, sd, rep = num_sms(), sd64(), Report()
    variants = sp.all_variants("track")
    batches = sp.planned("track_u8", 256, 256, variants, S)
    net = make_net(max(batches))
    x1, u1 = inputs(256, 256, SEARCH_SEEDS)
    t1, _ = inputs(128, 128, TEMPLATE_SEEDS)
    res = {"mode": "track", "S": S, "batches": batches}
    own = [("default", {})] + [(f"{k}={v}", {k: v}) for k, v in sp.OWN_REFERENCE["track"]]
    z1, expected = track_refs(rep, net, sd, x1, u1, t1, own)
    res["oracle_worst"] = dict(rep.worst)

    u1c = u1.cuda()
    res["dispatch"] = dispatch(rep, net, "track_u8", variants, lambda: track_u8(net, u1c[:2], z1[:2], POISONS["A"]))
    xf = net.get_features(x1[:2].cuda())
    res["dispatch_head"] = dispatch(rep, net, "head", variants, lambda: net.connector(z1[:2], xf))
    sweep(rep, net, lambda idx, p: track_u8(net, u1c[idx], z1[idx], p), expected, list(batches), variants,
          "track_u8", 256, 256, S, x1, {})
    res.update(rep.dump())
    return res


# ------------------------------------------------------------------------------------------------------------- large
def check_large():
    """get_features_u8 (default and fuse_irf=0, whose 128 x 128 x 96 expanded tensor of xif2_0 then spans more than
    2^31 floats of bufE) and fear_track_u8 with Bz = B, at the smallest multiple of 7 frames whose workspace holds more
    than 2^31 floats per buffer slot, in one chunk.  The B = 1 results these are compared with are the ones the
    `track` and `features 256 256` modes check against the oracle (same seeds)."""
    S, rep = num_sms(), Report()
    B = sp.smallest_batch_past_int32(N_INPUTS)
    io = B * (3 * 256 * 256 + 4 * 256 * 256 + 4 * 256 * 64 + 4 * 5 * 256 + _lib.BOX_DTYPE.itemsize) * 2
    need = sp.workspace_bytes(B) + io + (1 << 30)
    free, total = torch.cuda.mem_get_info()
    res = {"mode": "large", "S": S, "B": B, "workspace_bytes": sp.workspace_bytes(B), "bufE_floats": B * sp.K_ACT_E,
           "need_bytes": need, "free_bytes": free, "total_bytes": total}
    if free < need:
        res["skipped"] = f"needs ~{need / 2 ** 30:.1f} GiB free for B = {B}, the device has {free / 2 ** 30:.1f} GiB"
        return res
    net = make_net(B)
    x1, u1 = inputs(256, 256, SEARCH_SEEDS)
    t1, _ = inputs(128, 128, TEMPLATE_SEEDS)
    u1c = u1.cuda()
    idx = [i % N_INPUTS for i in range(B)]
    res["regimes"] = {ln.name: {"tiles": B * ln.tiles, "busiest_cta_tiles": sp.cta_tile_counts(B * ln.tiles, S)[1]}
                      for ln in sp.launches("track_u8") if ln.persistent}
    # features
    ref = torch.cat([features_u8(net, u1c[i:i + 1], POISONS["A"])[0] for i in range(N_INPUTS)])
    ub = u1c[idx]
    for vname, opts in (("default", {}), ("fuse_irf=0", {"fuse_irf": "0"})):
        with options(net, opts):
            n0 = net.launch_count()
            got = features_u8(net, ub, POISONS["B"])
            torch.cuda.synchronize()
            rep.runs += 1
            if net.launch_count() - n0 != len(sp.launches("get_features", 256, 256, opts)):
                rep.fail(f"get_features_u8 B={B} {vname}: not one chunk")
        bad = bad_frames(got, [ref[idx]])
        if bad:
            rep.fail({"entry": "get_features_u8", "variant": vname, "B": B, "bad_frames": bad[:16],
                      "n_bad_frames": len(bad)})
        del got
    del ub
    # track, Bz = B
    z1, expected = track_refs(rep, net, None, None, u1, t1, [("default", {})], oracle=False)
    got = track_u8(net, u1c[idx], z1[idx], POISONS["A"])
    torch.cuda.synchronize()
    rep.runs += 1
    bad = bad_frames(got, [e[idx] for e in expected["default"]])
    if bad:
        rep.fail({"entry": "track_u8", "B": B, "bad_frames": bad[:16], "n_bad_frames": len(bad)})
    res.update(rep.dump())
    return res


def main():
    mode = sys.argv[1]
    if mode == "features":
        res = check_features(int(sys.argv[2]), int(sys.argv[3]))
    elif mode == "track":
        res = check_track()
    elif mode == "large":
        res = check_large()
    else:
        raise SystemExit(f"unknown mode {mode!r}")
    print("SCHEDULE_CHECK " + json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
