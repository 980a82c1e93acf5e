"""Stand-alone checker of every kernel entry point on poisoned memory (run in its own process: a device-side trap would
poison the CUDA context of the main pytest process).  Prints one JSON line.

    python tests/poison_check.py GROUP   # GROUP: entry | features H W | head | track | decode | corr | crops | loop |
                                         #        trackers

The other GPU tests all run on memory whose contents favour the kernels: fresh workspace reads as zero (the padding a
convolution wants), a variant run finds the values of the default run in the workspace, and torch.empty outputs often
hold an earlier identical result.  Here every checked call runs three times, with the library workspace
(fear_debug_fill_workspace), every guard band and every output filled first with 0, then with fill A, then with fill B:
  floats  A = 0x7FA5A5A5 (a NaN with a payload no kernel emits)   B = 0x4B800001 (+16 777 218.0, survives a ReLU)
  bytes   A = 0xA5                                                  B = 0x5A
and the three results must be bit-identical, every guard band must still hold its fill, the inputs must be unchanged,
no float output may still hold fill A and records keep every field the entry point does not own.  Every device buffer
handed to the C ABI is a view into a larger allocation with a guard band of max(64 KiB, one frame) on each side.
Nothing a kernel uses as an address, index, stride or size is ever poisoned: rows of a frame table or target array past
the ones a call may read hold valid decoys (a real frame, a real target), so a kernel that reads them gives a wrong
answer instead of a fault.  The zero-fill run is also compared with the fp64 oracle, cv2 or numpy.
"""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import feartracker_b200 as fb  # noqa: E402
from feartracker_b200 import _lib, image_ops  # noqa: E402
from oracle import fear_oracle as fo  # noqa: E402
from tests.helpers import POISON_A, POISON_B, TOL, load_full_state, map_errors  # noqa: E402

FILLS = {"zero": (0, 0), "A": (POISON_A, 0xA5), "B": (POISON_B, 0x5A)}  # name -> (32-bit word, byte)
MIN_GUARD = 64 << 10
FEAT_INF_TOL, HEAD_INF_TOL, CORR_INF_TOL, MARGIN = 2e-5, 1e-4, 1e-5, 1e-4
BIT_IDENTICAL_OPTIONS = [("fuse_stem", "0"), ("fuse_irf", "0"), ("fuse_dwpw", "0"),
                         ("dw", "pixel"), ("dw", "strip"), ("dw", "roll"), ("dw", "tma"), ("pdl", "0")]
DEFAULTS = {"fuse_stem": "1", "fuse_irf": "1", "fuse_dwpw": "15", "dw": "auto", "pw": "auto", "corr": "auto", "pdl": "1"}
# every fusion off at once, with each depthwise kernel: the only way the rolling-window 3x3 stride-2 kernel (xif2_0
# unfused) and, at crop sizes the fused paths tile, the unfused depthwise kernels of every block run
FUSIONS_OFF = [("fuse_stem", "0"), ("fuse_irf", "0"), ("fuse_dwpw", "0")]
DW_IMPLS = ["auto", "pixel", "strip", "roll", "tma"]


def stream():
    return torch.cuda.current_stream().cuda_stream


def as_i32(word):
    return word - (1 << 32) if word >= 1 << 31 else word


class Guarded:
    """A device buffer of `nbytes` at an `align`-byte aligned offset of a larger uint8 allocation, with a guard band of
    at least max(64 KiB, `frame` bytes) on each side.  `words`: float / int32 memory, filled with 32-bit words (else
    with bytes).  `data`: contents of an input (uint8 tensor of nbytes), restored after every fill."""

    def __init__(self, nbytes, frame=0, align=256, words=True, data=None):
        guard = -(-max(MIN_GUARD, frame) // 1024) * 1024
        self.base = torch.empty(guard + align + nbytes + guard + 8, dtype=torch.uint8, device="cuda")
        self.off = guard + (-(self.base.data_ptr() + guard)) % align
        self.n, self.words, self.data = nbytes, words, data
        self.base = self.base[:(self.base.numel() // 4) * 4]

    @classmethod
    def of(cls, t, frame_elems=1, **kw):
        """A guarded copy of tensor t (an input): frame_elems = elements per frame of t."""
        t = t.contiguous()
        raw = t.view(-1).view(torch.uint8) if t.dtype != torch.uint8 else t.view(-1)
        g = cls(raw.numel(), frame=frame_elems * t.element_size(), words=t.dtype != torch.uint8, data=raw.cuda(), **kw)
        g.dtype, g.shape = t.dtype, tuple(t.shape)
        return g

    @classmethod
    def out(cls, shape, dtype, frame_elems=1, **kw):
        n = int(np.prod(shape)) * torch.tensor([], dtype=dtype).element_size()
        g = cls(n, frame=frame_elems * torch.tensor([], dtype=dtype).element_size(), words=dtype != torch.uint8, **kw)
        g.dtype, g.shape = dtype, tuple(shape)
        return g

    @property
    def raw(self):
        return self.base[self.off:self.off + self.n]

    @property
    def t(self):
        return self.raw.view(self.dtype).view(self.shape)

    def ptr(self):
        return self.base.data_ptr() + self.off

    def pattern(self, fill, n):
        word, byte = FILLS[fill]
        if self.words:
            return torch.full((n // 4,), as_i32(word), dtype=torch.int32, device="cuda").view(torch.uint8)
        return torch.full((n,), byte, dtype=torch.uint8, device="cuda")

    def fill(self, fill):
        self.base.copy_(self.pattern(fill, self.base.numel()))
        if self.data is not None:
            self.raw.copy_(self.data)

    def guards_ok(self, fill):
        pat = self.pattern(fill, self.base.numel())
        return bool(torch.equal(self.base[:self.off], pat[:self.off])
                    and torch.equal(self.base[self.off + self.n:], pat[self.off + self.n:]))


class Checker:
    """Runs checked calls and collects failures."""

    def __init__(self):
        self.failures, self.calls = [], 0

    def fail(self, msg):
        self.failures.append(msg)

    def run(self, tag, call, inputs=(), outputs=(), nets=(), owned=None, on_fill=None):
        """call() three times (fills zero, A, B).  inputs: Guarded inputs; outputs: Guarded outputs (fully written);
        owned: {Guarded in/out record buffer: (rows, field slice it writes)}; nets: FEARNets whose workspaces are
        poisoned; on_fill(fill): poisons whatever else the call reads.  Returns the outputs (and owned buffers) of the zero-fill run as clones."""
        owned = owned or {}
        results = {}
        for fill in FILLS:
            for net in nets:
                _lib.check(_lib.load().fear_debug_fill_workspace(net._handle, FILLS[fill][0], stream()),
                           "fear_debug_fill_workspace")
            for g in list(inputs) + list(outputs) + list(owned):
                g.fill(fill)
            if on_fill is not None:
                on_fill(fill)
            call()
            torch.cuda.synchronize()
            self.calls += 1
            for k, g in enumerate(list(inputs) + list(outputs) + list(owned)):
                if not g.guards_ok(fill):
                    bad = torch.nonzero(g.base != g.pattern(fill, g.base.numel()))[:, 0]
                    bad = bad[(bad < g.off) | (bad >= g.off + g.n)]
                    self.fail(f"{tag} fill {fill}: guard band of buffer {k} written at byte offsets "
                              f"{(bad[:4] - g.off).tolist()} relative to the buffer ({g.n} bytes)")
            for k, g in enumerate(inputs):
                if not torch.equal(g.raw, g.data):
                    self.fail(f"{tag} fill {fill}: input {k} changed")
            for k, g in enumerate(outputs):
                if fill == "A" and g.words and g.dtype == torch.float32:
                    left = int((g.t.view(torch.int32) == as_i32(POISON_A)).sum())
                    if left:
                        self.fail(f"{tag}: output {k} has {left} elements never written (still fill A)")
            for k, (g, (rows, fields)) in enumerate(owned.items()):
                got, was = g.t.view(-1, g.shape[-1]), g.data.view(torch.int32).view(-1, g.shape[-1])
                keep = torch.ones(got.shape, dtype=torch.bool, device="cuda")
                keep[:rows, fields] = False
                if not torch.equal(got[keep], was[keep]):
                    self.fail(f"{tag} fill {fill}: record buffer {k} changed outside rows [0, {rows}) fields {fields}")
            results[fill] = [g.t.clone() for g in list(outputs) + list(owned)]
        for fill in ("A", "B"):
            for k, (a, b) in enumerate(zip(results["zero"], results[fill])):
                if not torch.equal(a.view(torch.uint8) if a.dtype != torch.uint8 else a,
                                   b.view(torch.uint8) if b.dtype != torch.uint8 else b):
                    diff = (a.double() - b.double()).abs().nan_to_num(float("inf")).max() if a.is_floating_point() \
                        else (a != b).sum()
                    self.fail(f"{tag}: output {k} differs between fill zero and fill {fill} (max |diff| {float(diff):.3e})")
        return results["zero"]

    def report(self):
        return {"checked_calls": self.calls, "failures": self.failures[:60], "n_failures": len(self.failures)}


def make_net(reserve):
    net = fb.FEARNet(**fb.FEAR_XS_MODEL_KWARGS)
    net.load_state_dict(load_full_state(), strict=True)
    net = net.cuda().eval()
    net.reserve(reserve)
    net._ensure_handle(torch.device("cuda", torch.cuda.current_device()))
    return net


def sd64():
    return fo.to_dtype({k: v for k, v in load_full_state().items() if v.is_floating_point()}, torch.float64)


def set_options(net, opts):
    for k, v in opts:
        net.set_option(k, v)


def reset_options(net):
    for k, v in DEFAULTS.items():
        net.set_option(k, v)


def worst(res, key, value):
    res[key] = max(res.get(key, 0.0), float(value))


# ------------------------------------------------------------------------------------------------------- features
def group_features(H, W):
    """fear_get_features, fear_get_features_u8, fear_backbone and fear_debug_backbone_prefix (n = 0..16) at one crop
    size: B = 1 and 3 on a handle reserved for 8 (slots of frames B..7 hold poison), B = 5 on a handle held at 2 frames
    (chunks reuse slots holding another frame's values); every option variant, each after a fresh poison."""
    lib, chk, sd = _lib.load(), Checker(), sd64()
    res = {"H": H, "W": W, "oracle": {}, "variants": []}
    nets = {8: make_net(8), 2: make_net(2)}
    variants = [("default", [])] + [(f"{k}={v}", [(k, v)]) for k, v in BIT_IDENTICAL_OPTIONS] + [("pw=ffma", [("pw", "ffma")])]
    variants += [("fusions_off dw=" + d, FUSIONS_OFF + [("dw", d)]) for d in DW_IMPLS]
    names = ["xif0_0"] + [s.name for s in fo.FBNET_C[1:fo.NUM_HOT_BLOCKS] if s.kind == "ir"]
    P = (H // 16) * (W // 16)
    for R_, B in ((8, 1), (8, 3), (2, 5)):
        net = nets[R_]
        x, u = fo.shape_crops(H, W, B, seed=31 + B)
        col = {}
        with torch.no_grad():
            fo.get_features(sd, x.double(), col)
        gx = Guarded.of(x, 3 * H * W)
        gu = Guarded.of(u.permute(0, 2, 3, 1).contiguous(), 3 * H * W)
        nb = min(B, R_)  # fear_debug_backbone_prefix runs on at most the reserved batch
        gxp = Guarded.of(x[:nb], 3 * H * W)
        ref = {}
        for vname, opts in variants:
            set_options(net, opts)
            try:
                outs = {}
                for entry, gin in (("get_features", gx), ("get_features_u8", gu), ("backbone", gx)):
                    ch = 112 if entry == "backbone" else 256
                    go = Guarded.out((B, ch, H // 16, W // 16), torch.float32, ch * P)
                    fn = {"get_features": lib.fear_get_features, "get_features_u8": lib.fear_get_features_u8,
                          "backbone": lib.fear_backbone}[entry]
                    outs[entry] = chk.run(f"{H}x{W} R={R_} B={B} {vname} {entry}",
                                          lambda: _lib.check(fn(net._handle, gin.ptr(), B, H, W, go.ptr(), stream()), entry),
                                          inputs=[gin], outputs=[go], nets=[net])[0]
                down, ch = 2, 16
                for n in range(len(names)):
                    if n:
                        spec = [s for s in fo.FBNET_C[1:fo.NUM_HOT_BLOCKS] if s.kind == "ir"][n - 1]
                        down, ch = down * spec.stride, spec.cout
                    go = Guarded.out((nb, ch, H // down, W // down), torch.float32, ch * (H // down) * (W // down))
                    outs[f"prefix{n}"] = chk.run(
                        f"{H}x{W} R={R_} B={B} {vname} backbone_prefix {n}",
                        lambda: _lib.check(lib.fear_debug_backbone_prefix(net._handle, gxp.ptr(), nb, H, W, n, go.ptr(),
                                                                          stream()), "fear_debug_backbone_prefix"),
                        inputs=[gxp], outputs=[go], nets=[net])[0]
            finally:
                reset_options(net)
            tag = f"{H}x{W} R={R_} B={B} {vname}"
            if vname in ("default", "pw=ffma"):  # oracle anchor
                o = res["oracle"].setdefault(vname, {})
                for entry, key in (("get_features", "neck"), ("get_features_u8", "neck"), ("backbone", "xif4_7")):
                    e2 = map_errors(outs[entry].cpu().numpy(), col[key].numpy())[1]
                    worst(o, entry, e2)
                    if not e2 <= FEAT_INF_TOL:
                        chk.fail(f"{tag} {entry}: inf-norm error {e2:.3e} vs the fp64 oracle")
                for n, name in enumerate(names):
                    e2 = map_errors(outs[f"prefix{n}"].cpu().numpy(), col[name][:nb].numpy())[1]
                    worst(o, "backbone_prefix", e2)
                    if not e2 <= FEAT_INF_TOL:
                        chk.fail(f"{tag} backbone_prefix {n} ({name}): inf-norm error {e2:.3e} vs the fp64 oracle")
            if vname == "default":
                ref = outs
            elif vname != "pw=ffma":
                bad = [k for k in outs if not torch.equal(outs[k], ref[k])]
                if bad:
                    chk.fail(f"{tag}: not bit-identical to the default in {bad[:6]}")
            res["variants"].append(tag)
    res.update(chk.report())
    return res


# ----------------------------------------------------------------------------------------------------------- head
def head_call(net, gz, Bz, gu, Bu, gx, B, gb, gc):
    lib = _lib.load()
    if gu is None:
        rc = lib.fear_head(net._handle, gz.ptr(), Bz, gx.ptr(), B, gb.ptr(), gc.ptr(), stream())
    else:
        rc = lib.fear_head_update(net._handle, gz.ptr(), Bz, gu.ptr(), Bu, gx.ptr(), B, gb.ptr(), gc.ptr(), stream())
    _lib.check(rc, "fear_head")


def head_oracle(chk, res, tag, sd, x, z, u, bbox, cls, extra=None):
    """Outputs of one head call vs fp64 BoxTower.forward (on the GPU's features): inf-norm <= 1e-4, the allclose form
    |a - b| <= 1e-3 |b| + 1e-5 ||b||inf, argmax exact where the oracle's top-2 margin is >= 1e-4."""
    B = x.shape[0]
    with torch.no_grad():
        want = fo.box_tower(sd, x.cpu().double(), z.cpu().double().expand(B, -1, -1, -1),
                            None if u is None else u.cpu().double().expand(B, -1, -1, -1))
    got = [bbox, cls] + (list(extra) if extra else [])
    for name, a, b in zip(("reg", "cls", "cls_dw", "x_reg"), got, want):
        a, b = a.cpu().double().numpy(), b.numpy()
        for k in range(B):
            e2 = map_errors(a[k], b[k])[1]
            worst(res, name, e2)
            if not e2 <= HEAD_INF_TOL:
                chk.fail(f"{tag} frame {k} {name}: inf-norm error {e2:.3e} vs the fp64 oracle")
            if name in ("reg", "cls") and not (np.abs(a[k] - b[k]) <= TOL * np.abs(b[k]) + 1e-5 * np.abs(b[k]).max()).all():
                chk.fail(f"{tag} frame {k} {name}: outside the allclose bar")
    for k in range(B):
        top2 = want[1][k].flatten().topk(2).values
        if float(top2[0] - top2[1]) >= MARGIN and int(cls[k].flatten().argmax()) != int(want[1][k].flatten().argmax()):
            chk.fail(f"{tag} frame {k}: argmax differs from the oracle")


HEAD_TENSORS = {"search_features": 256, "cat_cls": 320, "cat_reg": 320, "cls_dw": 256, "reg_dw": 256, "x_reg": 256,
                "cls_tower": 256}


def group_head():
    """fear_head / fear_head_update at B in {1, 3, 34} unchunked and B = 5 at R = 4, Bz in {1, B}, Bu in {none, 1, B};
    corr x pw in {ffma, wgmma}, fuse_dwpw = 13 and each depthwise kernel, each after a poison; every
    fear_debug_head_tensor name."""
    chk, sd, lib = Checker(), sd64(), _lib.load()
    res = {"oracle": {}, "variants": {}}
    full, r4 = make_net(34), make_net(4)
    n = 34
    _, xt, _, _ = fo.synthetic_crops(n)
    zc, _ = fo.shape_crops(128, 128, n, seed=41)
    uc, _ = fo.shape_crops(128, 128, n, seed=42)
    X, Z, U = (full.get_features(t.cuda()) for t in (xt, zc, uc))
    refs = {}  # (R, B, Bz, Bu) -> (bbox, cls)
    for R_, B, net in ((0, 1, full), (0, 3, full), (0, 34, full), (4, 5, r4)):
        idx = [(7 * B + k) % n for k in range(B)]
        for bz in sorted({1, B}):
            for bu in [None] + sorted({1, B}):
                x = X[idx]
                z = Z[idx[-1:]] if bz == 1 else Z[idx]
                u = None if bu is None else (U[idx[:1]] if bu == 1 else U[idx])
                gx, gz = Guarded.of(x, 256 * 256), Guarded.of(z, 256 * 64)
                gu = None if u is None else Guarded.of(u, 256 * 64)
                gb, gc = Guarded.out((B, 4, 16, 16), torch.float32, 1024), Guarded.out((B, 1, 16, 16), torch.float32, 256)
                tag = f"head R={R_} B={B} Bz={bz} Bu={bu}"
                ins = [g for g in (gx, gz, gu) if g is not None]
                bbox, cls = chk.run(tag, lambda: head_call(net, gz, bz, gu, bu, gx, B, gb, gc), ins, [gb, gc], [net])
                refs[(R_, B, bz, bu)] = (bbox, cls)
                if B in (3, 5) or (B == 34 and bz == 1 and bu == B):  # oracle anchors
                    head_oracle(chk, res["oracle"], tag, sd, x, z, u, bbox, cls)
                if (R_, B) == (0, 3) and bz == B and bu == 1:
                    # every debug head tensor of this call, rows of B frames out of a 34-frame workspace
                    run_head = lambda: head_call(net, gz, bz, gu, bu, gx, B, gb, gc)  # noqa: E731
                    got = {}
                    for name, ch in HEAD_TENSORS.items():
                        go = Guarded.out((B, ch, 16, 16), torch.float32, ch * 256)

                        def call(name=name, go=go):
                            run_head()
                            _lib.check(lib.fear_debug_head_tensor(net._handle, name.encode(), B, go.ptr(), stream()),
                                       "fear_debug_head_tensor")
                        got[name] = chk.run(f"{tag} head_tensor {name}", call, ins, [go], [net])[0]
                    if not torch.equal(got["search_features"], x.reshape(B, 256, 16, 16)):
                        chk.fail(f"{tag} head_tensor search_features != the call's search features")
                    with torch.no_grad():
                        want = fo.box_tower(sd, x.cpu().double(), z.cpu().double(), u.cpu().double().expand(B, -1, -1, -1))
                    for name, w in (("cls_dw", want[2]), ("x_reg", want[3])):
                        e2 = map_errors(got[name].cpu().numpy(), w.numpy())[1]
                        worst(res["oracle"], "head_tensor " + name, e2)
                        if not e2 <= HEAD_INF_TOL:
                            chk.fail(f"{tag} head_tensor {name}: inf-norm error {e2:.3e} vs the fp64 oracle")
    # option variants at B = 3 (unchunked) and B = 5 (R = 4), Bz = 1, Bu = B
    variants = [("fuse_dwpw=13", [("fuse_dwpw", "13")])] + [(f"dw={d}", [("dw", d)]) for d in DW_IMPLS[1:]]
    variants += [(f"pw={p} corr={c}", [("pw", p), ("corr", c)]) for p in ("ffma", "wgmma") for c in ("ffma", "wgmma")]
    for R_, B, net in ((0, 3, full), (4, 5, r4)):
        idx = [(7 * B + k) % n for k in range(B)]
        x, z, u = X[idx], Z[idx[-1:]], U[idx]
        gx, gz, gu = Guarded.of(x, 256 * 256), Guarded.of(z, 256 * 64), Guarded.of(u, 256 * 64)
        gb, gc = Guarded.out((B, 4, 16, 16), torch.float32, 1024), Guarded.out((B, 1, 16, 16), torch.float32, 256)
        base = refs[(R_, B, 1, B)]
        for vname, opts in variants:
            set_options(net, opts)
            tag = f"head R={R_} B={B} Bz=1 Bu={B} {vname}"
            try:
                bbox, cls = chk.run(tag, lambda: head_call(net, gz, 1, gu, B, gx, B, gb, gc), [gx, gz, gu], [gb, gc], [net])
            finally:
                reset_options(net)
            if vname.startswith("pw="):
                o = res["variants"].setdefault(vname, {})
                head_oracle(chk, o, tag, sd, x, z, u, bbox, cls)
            elif not (torch.equal(bbox, base[0]) and torch.equal(cls, base[1])):
                chk.fail(f"{tag}: not bit-identical to the default")
    res.update(chk.report())
    return res


# ---------------------------------------------------------------------------------------------------------- track
def group_track():
    """fear_track, fear_track_u8 and fear_forward with boxes only, maps only and both, B = 3 unchunked (R = 8) and
    B = 5 at R = 2; guards around whichever outputs are non-null."""
    chk, sd, lib = Checker(), sd64(), _lib.load()
    res = {"oracle": {}}
    n = 5
    tc, xt, _, xu = fo.synthetic_crops(n, seed=77)
    with torch.no_grad():
        want = fo.track(sd, xt.double(), fo.get_features(sd, tc.double()))
    nets = {8: make_net(8), 2: make_net(2)}
    zf = nets[8].get_features(tc.cuda())
    ref = {}
    for R_, B in ((8, 3), (2, 5)):
        net = nets[R_]
        gxs, gxu = Guarded.of(xt[:B], 3 * 256 * 256), Guarded.of(xu[:B].permute(0, 2, 3, 1).contiguous(), 3 * 256 * 256)
        gt, gz = Guarded.of(tc[:B], 3 * 128 * 128), Guarded.of(zf[:B], 256 * 64)
        gz1 = Guarded.of(zf[:1], 256 * 64)
        for entry in ("track", "track_u8", "forward"):
            for bz in ((B,) if entry == "forward" else (1, B)):
                for want_maps, want_boxes in ((True, True), (True, False), (False, True)):
                    gb = Guarded.out((B, 4, 16, 16), torch.float32, 1024) if want_maps else None
                    gc = Guarded.out((B, 1, 16, 16), torch.float32, 256) if want_maps else None
                    gbox = Guarded.out((B, _lib.BOX_DTYPE.itemsize), torch.uint8, 48) if want_boxes else None
                    outs = [g for g in (gb, gc, gbox) if g is not None]
                    p = [g.ptr() if g is not None else None for g in (gb, gc, gbox)]
                    zz = gz1 if bz == 1 else gz
                    if entry == "forward":
                        ins = [gt, gxs]
                        call = lambda: _lib.check(lib.fear_forward(net._handle, gt.ptr(), gxs.ptr(), B, *p, stream()),  # noqa: E731
                                                  "fear_forward")
                    else:
                        gs = gxu if entry == "track_u8" else gxs
                        fn = lib.fear_track_u8 if entry == "track_u8" else lib.fear_track
                        ins = [gs, zz]
                        call = lambda: _lib.check(fn(net._handle, gs.ptr(), zz.ptr(), bz, B, *p, stream()), entry)  # noqa: E731
                    tag = f"{entry} R={R_} B={B} Bz={bz} maps={want_maps} boxes={want_boxes}"
                    got = chk.run(tag, call, ins, outs, [net])
                    if want_boxes:
                        rec = got[-1]
                        if entry != "forward" and want_maps and not torch.equal(rec, decode_boxes(got[0], got[1])):
                            chk.fail(f"{tag}: records != fear_decode of the maps")
                        key = (entry, bz == 1)  # frames 0..2 and their templates are the same at B = 3 and 5
                        if R_ == 8:
                            ref[key] = rec
                        elif not torch.equal(rec[:3], ref[key]):
                            chk.fail(f"{tag}: chunked records differ from the unchunked ones")
                    if want_maps and bz == B:
                        bbox, cls = got[0], got[1]
                        for k in range(B):
                            for name, a, b in (("reg", bbox[k], want[fo.TARGET_REGRESSION_LABEL_KEY][k]),
                                               ("cls", cls[k], want[fo.TARGET_CLASSIFICATION_KEY][k])):
                                a, b = a.cpu().double().numpy(), b.numpy()
                                e2 = map_errors(a, b)[1]
                                worst(res["oracle"], name, e2)
                                if not (e2 <= HEAD_INF_TOL and (np.abs(a - b) <= TOL * np.abs(b) + 1e-5 * np.abs(b).max()).all()):
                                    chk.fail(f"{tag} frame {k} {name}: inf-norm error {e2:.3e} vs the fp64 oracle")
                            top2 = want[fo.TARGET_CLASSIFICATION_KEY][k].flatten().topk(2).values
                            if float(top2[0] - top2[1]) >= MARGIN and int(cls[k].flatten().argmax()) != \
                                    int(want[fo.TARGET_CLASSIFICATION_KEY][k].flatten().argmax()):
                                chk.fail(f"{tag} frame {k}: argmax differs from the oracle")
    res.update(chk.report())
    return res


def decode_boxes(bbox, cls, aps=1):
    B = bbox.shape[0]
    out = torch.empty((B, _lib.BOX_DTYPE.itemsize), dtype=torch.uint8, device="cuda")
    _lib.check(_lib.load().fear_decode(bbox.data_ptr(), cls.data_ptr(), B, aps, out.data_ptr(), stream()), "fear_decode")
    return out


# --------------------------------------------------------------------------------------------------------- decode
def group_decode():
    """fear_decode at B = 1, 7 and 70 000 with guards around the maps and the FearBox array, against torch."""
    from tests.head_check import expected_decode

    chk, lib = Checker(), _lib.load()
    g = torch.Generator().manual_seed(505)
    for B in (1, 7, 70000):
        cls = 2.0 * torch.randn(B, 1, 16, 16, generator=g)
        cls[::3] = torch.randint(-6, 7, (len(cls[::3]), 1, 16, 16), generator=g).float() / 4  # ties
        reg = 60.0 * torch.rand(B, 4, 16, 16, generator=g)
        gr, gc = Guarded.of(reg, 1024), Guarded.of(cls, 256)
        for aps in (1, 0):
            gbox = Guarded.out((B, _lib.BOX_DTYPE.itemsize), torch.uint8, 48)
            rec = chk.run(f"decode B={B} sigmoid={aps}", lambda: _lib.check(
                lib.fear_decode(gr.ptr(), gc.ptr(), B, aps, gbox.ptr(), stream()), "fear_decode"), [gr, gc], [gbox])[0]
            rec = rec.cpu().numpy().view(_lib.BOX_DTYPE).reshape(-1)
            flat, score, box = (t.cpu().numpy() for t in expected_decode(reg.cuda(), cls.cuda(), aps))
            got_box = np.stack([rec["x"], rec["y"], rec["w"], rec["h"]], 1)
            if not (np.array_equal(rec["flat"], flat) and np.array_equal(rec["row"], flat // 16)
                    and np.array_equal(rec["col"], flat % 16) and np.array_equal(got_box, box)
                    and np.array_equal(rec["score"].view(np.uint32), score.view(np.uint32))):
                chk.fail(f"decode B={B} sigmoid={aps}: records differ from torch")
    return chk.report()


# ----------------------------------------------------------------------------------------------------------- corr
def group_corr():
    """fear_corr_concat_f32, fear_corr_concat_ws_f32 (the caller's workspace guarded and poisoned) and fear_corr_nhwc_f32
    (in place: channels [0, 256) unchanged, [256, 320) poisoned first and fully written) at B in {1, 3, 5}, Bz in {1, B}."""
    chk, lib = Checker(), _lib.init(0)  # the wgmma forms need the library's per-device state
    res = {"oracle": {}}
    for B in (1, 3, 5):
        for bz in sorted({1, B}):
            g = torch.Generator().manual_seed(10 * B + bz)
            z = torch.randn(bz, 256, 64, generator=g)
            x = torch.randn(B, 256, 16, 16, generator=g)
            want = fo.pixelwise_correlation(z.double(), x.double())
            gz, gx = Guarded.of(z, 256 * 64), Guarded.of(x, 256 * 256)
            go = Guarded.out((B, 320, 16, 16), torch.float32, 320 * 256)
            need = lib.fear_corr_concat_workspace_bytes(B, bz)
            gws = Guarded(need, frame=320 * 256 * 4, align=1024)
            gws.dtype, gws.shape = torch.float32, (need // 4,)
            tag = f"corr B={B} Bz={bz}"
            out = chk.run(tag + " concat", lambda: _lib.check(
                lib.fear_corr_concat_f32(gz.ptr(), bz, gx.ptr(), B, go.ptr(), stream()), "fear_corr_concat_f32"),
                [gz, gx], [go])[0]
            # the caller's workspace is scratch: poisoned (as an output) but not required to be fully written
            out_ws = chk.run(tag + " concat_ws", lambda: _lib.check(
                lib.fear_corr_concat_ws_f32(gz.ptr(), bz, gx.ptr(), B, go.ptr(), gws.ptr(), need, stream()),
                "fear_corr_concat_ws_f32"), [gz, gx], [go], on_fill=gws.fill)[0]
            if not gws.guards_ok("B"):
                chk.fail(f"{tag} concat_ws: caller workspace guard written")
            # channels-last core in place: cat[b, p, :256] = x, cat[b, p, 256:] poisoned with the fill of the run
            zt = z.permute(0, 2, 1).contiguous()  # [k][c]
            cat0 = torch.empty(B, 256, 320)
            cat0[:, :, :256] = x.reshape(B, 256, 256).permute(0, 2, 1)
            gzt, gcat = Guarded.of(zt, 64 * 256), Guarded.of(cat0, 256 * 320)
            runs = []
            for fill in FILLS:
                gzt.fill(fill)
                gcat.fill(fill)
                gcat.t.view(torch.int32)[:, :, 256:] = as_i32(FILLS[fill][0])
                _lib.check(lib.fear_corr_nhwc_f32(gzt.ptr(), bz, gcat.ptr(), B, stream()), "fear_corr_nhwc_f32")
                torch.cuda.synchronize()
                chk.calls += 1
                cat = gcat.t.clone()
                runs.append(cat)
                if not (gzt.guards_ok(fill) and gcat.guards_ok(fill) and torch.equal(gzt.raw, gzt.data)):
                    chk.fail(f"{tag} nhwc fill {fill}: a guard band or the template changed")
                if not torch.equal(cat[:, :, :256].cpu(), cat0[:, :, :256]):
                    chk.fail(f"{tag} nhwc fill {fill}: channels [0, 256) changed")
                if fill == "A" and bool((cat.view(torch.int32)[:, :, 256:] == as_i32(POISON_A)).any()):
                    chk.fail(f"{tag} nhwc: correlation channels left unwritten")
            if not all(torch.equal(r.view(torch.int32), runs[0].view(torch.int32)) for r in runs[1:]):
                chk.fail(f"{tag} nhwc: result depends on the fill")
            for what, a in (("concat", out), ("concat_ws", out_ws),
                            ("nhwc", runs[0].permute(0, 2, 1).reshape(B, 320, 16, 16))):
                a = a.cpu()
                if not torch.equal(a[:, :256], x):
                    chk.fail(f"{tag} {what}: channels [0, 256) are not x")
                e2 = map_errors(a[:, 256:].numpy(), want[:, 256:].numpy())[1]
                worst(res["oracle"], what, e2)
                if not e2 < CORR_INF_TOL:
                    chk.fail(f"{tag} {what}: inf-norm error {e2:.3e} vs the fp64 oracle")
    res.update(chk.report())
    return res


# ---------------------------------------------------------------------------------------------------------- crops
def group_crops():
    """fear_crop_resize_u8 with the frame in a guarded allocation (guards above, below and after the last pixel) on the
    windows of test_device_crop_resize_is_bit_identical_to_cv2, against cv2."""
    chk, lib = Checker(), _lib.load()
    rng = np.random.default_rng(9)
    frame = rng.integers(0, 256, (256, 480, 3), dtype=np.uint8)
    mean = np.mean(frame, axis=(0, 1))
    gf = Guarded(frame.size, frame=frame.size, words=False, data=torch.from_numpy(frame).reshape(-1).cuda())
    for box in ([163, 53, 45, 174], [0, 0, 30, 40], [450, 230, 30, 26], [-5, -7, 50, 60], [10, 200, 400, 56],
                [177, 64, 128, 128]):
        box = image_ops.clamp_bbox(box, frame.shape)
        for size, off in ((256, 2), (128, 0.2), (256, 0.5)):
            want = image_ops.extended_crop(frame, box, size, off, mean)[0]
            params, _, _ = image_ops.crop_params(box, size, off, mean)
            gp = Guarded.of(torch.from_numpy(params), params.size)
            go = Guarded(size * size * 3, frame=size * size * 3, words=False)
            go.dtype, go.shape = torch.uint8, (size, size, 3)
            got = chk.run(f"crop_resize {list(box)} {size} {off}", lambda: _lib.check(
                lib.fear_crop_resize_u8(gf.ptr(), 256, 480, gp.ptr(), go.ptr(), size, stream()), "fear_crop_resize_u8"),
                [gf, gp], [go])[0]
            if not np.array_equal(got.cpu().numpy(), want):
                chk.fail(f"crop_resize {list(box)} {size} {off}: differs from cv2")
    return chk.report()


# ----------------------------------------------------------------------------------------------------------- loop
LOOP_SHAPES = [(256, 480), (181, 97), (90, 333)]
LOOP_TARGETS = [
    (0, [163, 53, 45, 174]), (0, [-10, 100, 40, 30]), (0, [450, 20, 60, 40]), (0, [200, -15, 30, 50]),
    (0, [100, 240, 50, 40]), (0, [0, 0, 3, 3]), (0, [477, 253, 3, 3]), (0, [-50, 30, 600, 100]),
    (2, [-300, -200, 900, 500]), (2, [330, 87, 3, 3]), (2, [5, 40, 320, 20]),
] + [(1, [48 - s // 2, 90 - s // 2, s, s]) for s in (1, 2, 3, 5, 9, 17, 33, 64, 120, 200)]
N_DECOY_ROWS = 3  # target rows >= N and frame table entries >= F: valid records that a call may not read


class FrameSet:
    """LOOP_SHAPES frames (RGB truth `rgb`) laid out for one frame source in guarded allocations; `fill` poisons every
    byte outside the frames' pixels (guards, alignment gaps, alpha bytes, row pitch, the region around a region of
    interest).  `gtable` holds the F records and N_DECOY_ROWS decoys past them (other frames of the set)."""

    def __init__(self, source, rng):
        self.source, self.F = source, len(LOOP_SHAPES)
        self.parts = []  # (Guarded, writer(raw)) pairs: writer puts the pixels back after a fill
        recs = []
        if source == "packed":
            frames = [rng.integers(0, 256, s + (3,), dtype=np.uint8) for s in LOOP_SHAPES]
            self.rgb = frames
            offs, off = [], 0
            for f in frames:  # 16-byte aligned with a 13-byte gap: the gaps hold poison
                offs.append(off)
                off += -(-(f.size + 13) // 16) * 16
            g = Guarded(off, frame=max(f.size for f in frames), words=False)
            data = torch.from_numpy(np.concatenate([np.pad(f.reshape(-1), (0, -(-(f.size + 13) // 16) * 16 - f.size))
                                                    for f in frames])).cuda()
            mask = torch.zeros(off, dtype=torch.bool, device="cuda")
            for f, o in zip(frames, offs):
                mask[o:o + f.size] = True
            self.parts.append((g, lambda raw, data=data, mask=mask: raw.copy_(torch.where(mask, data, raw))))
            self.base_ptr = g.ptr()
            recs = [(o, h, w) for o, (h, w) in zip(offs, LOOP_SHAPES)]
            self.dtype = _lib.FRAME_DTYPE
        elif source == "views":
            frames = [rng.integers(0, 256, s + (3,), dtype=np.uint8) for s in LOOP_SHAPES]
            self.rgb = frames
            self.dtype = _lib.VIEW_DTYPE
            for (h, w), f, kind in zip(LOOP_SHAPES, frames, ("rgba", "pitch", "roi")):
                if kind == "rgba":
                    rs, ps, y0, x0, rows = 4 * w, 4, 0, 0, h
                elif kind == "pitch":
                    rs, ps, y0, x0, rows = 3 * w + 37, 3, 0, 0, h
                else:  # region of interest of a larger frame
                    rs, ps, y0, x0, rows = 3 * (w + 11), 3, 5, 7, h + 9
                g = Guarded(rows * rs, frame=rows * rs, words=False)
                idx = torch.from_numpy(((np.arange(h)[:, None, None] + y0) * rs + (np.arange(w)[None, :, None] + x0) * ps
                                        + np.arange(3)[None, None, :]).reshape(-1)).cuda()
                px = torch.from_numpy(f.reshape(-1)).cuda()
                self.parts.append((g, lambda raw, idx=idx, px=px: raw.index_put_((idx,), px)))
                recs.append((g.ptr() + y0 * rs + x0 * ps, rs, ps, 1, h, w))
        else:  # YUV 4:2:0: NV12 with a row pitch (8-bit) or P010 with a pitch and a BT.709 matrix (source "yuv")
            self.dtype = _lib.YUV420_DTYPE if source == "yuv420" else _lib.YUV_DTYPE
            self.rgb = []
            for k, (h, w) in enumerate(LOOP_SHAPES):
                h, w = h + h % 2, w + w % 2  # 4:2:0 needs even sides
                bits = 8 if source == "yuv420" or k == 1 else 10
                es = 1 if bits == 8 else 2
                pitch = w * es + 64
                yv = rng.integers(0, 1 << bits, (h, w)).astype(np.uint16)
                uv = rng.integers(0, 1 << bits, (h // 2, w // 2, 2)).astype(np.uint16)
                shift = 16 - bits if bits > 8 else 0
                matrix = "bt601" if source == "yuv420" else ("bt709", "bt601", "bt2020")[k]
                full = source == "yuv" and k == 2
                self.rgb.append(image_ops.yuv420_to_rgb(yv << shift, uv[..., 0] << shift, uv[..., 1] << shift, matrix,
                                                        full, bits, shift))
                g = Guarded(pitch * (h + h // 2), frame=pitch * h, words=False)
                surf = np.full((h + h // 2, pitch), 0, np.uint8)
                if es == 1:
                    surf[:h, :w] = yv
                    surf[h:, :w] = uv.reshape(h // 2, w).astype(np.uint8)
                else:
                    surf[:h, :2 * w] = (yv << shift).astype("<u2").view(np.uint8)
                    surf[h:, :2 * w] = (uv.reshape(h // 2, w) << shift).astype("<u2").view(np.uint8)
                mask = np.zeros_like(surf, dtype=bool)
                mask[:, :w * es] = True
                data, m = torch.from_numpy(surf.reshape(-1)).cuda(), torch.from_numpy(mask.reshape(-1)).cuda()
                self.parts.append((g, lambda raw, data=data, m=m: raw.copy_(torch.where(m, data, raw))))
                base = g.ptr()
                rec = (base, base + h * pitch, base + h * pitch + es, pitch, es, pitch, 2 * es, h, w)
                if source == "yuv":
                    rec += (image_ops.YUV_MATRICES[matrix][0], int(full), bits, shift)
                recs.append(rec)
        self.shapes = [r.shape[:2] for r in self.rgb]
        decoys = [recs[(i + 1) % self.F] for i in range(N_DECOY_ROWS)]  # entries >= F: other real frames
        table = np.array(recs + decoys, dtype=self.dtype).view(np.uint8)
        self.gtable = Guarded.of(torch.from_numpy(table.copy()), self.dtype.itemsize)

    def fill(self, fill):
        for g, writer in self.parts:
            g.fill(fill)
            writer(g.raw)

    def guards_ok(self, fill):
        return all(g.guards_ok(fill) for g, _ in self.parts)

    def frame_bytes_ok(self, snapshot):
        return all(torch.equal(g.base, s) for (g, _), s in zip(self.parts, snapshot))

    def snapshot(self):
        return [g.base.clone() for g, _ in self.parts]

    def crop(self, lib, gtable, gstate, N, off, size, gcrops):
        t, s = gtable.ptr(), gstate.ptr()
        if self.source == "packed":
            rc = lib.fear_crop_targets_u8(self.base_ptr, t, self.F, s, N, off, size, gcrops.ptr(), stream())
        else:
            fn = {"views": lib.fear_crop_targets_view_u8, "yuv420": lib.fear_crop_targets_yuv420_u8,
                  "yuv": lib.fear_crop_targets_yuv_u8}[self.source]
            rc = fn(t, self.F, s, N, off, size, gcrops.ptr(), stream())
        _lib.check(rc, "crop_targets " + self.source)

    def advance(self, lib, gboxes, gstate, N):
        fn = {"packed": lib.fear_advance_targets, "views": lib.fear_advance_targets_view,
              "yuv420": lib.fear_advance_targets_yuv420, "yuv": lib.fear_advance_targets_yuv}[self.source]
        _lib.check(fn(gboxes.ptr(), self.gtable.ptr(), self.F, gstate.ptr(), N, 256, stream()), "advance " + self.source)

    def sums(self, lib, gsums):
        fn = {"views": lib.fear_frame_sums_u8, "yuv420": lib.fear_frame_sums_yuv420_u8,
              "yuv": lib.fear_frame_sums_yuv_u8}[self.source]
        _lib.check(fn(self.gtable.ptr(), self.F, gsums.ptr(), stream()), "frame_sums " + self.source)


def group_loop():
    """fear_crop_targets*, fear_advance_targets* and fear_frame_sums* for packed FearFrame, FearFrameView,
    FearFrameYUV420 and FearFrameYUV frames in guarded, poisoned allocations, with decoy table entries and target rows."""
    from tests.test_gpu_multi_tracker import _cv2_crop

    chk, lib = Checker(), _lib.load()
    rng = np.random.default_rng(23)
    for source in ("packed", "views", "yuv420", "yuv"):
        fs = FrameSet(source, rng)
        means = [np.mean(f, axis=(0, 1)) for f in fs.rgb]
        targets = [(f, box) for f, box in LOOP_TARGETS]
        N = len(targets)
        recs = np.zeros((N + N_DECOY_ROWS, _lib.TARGET_INTS), dtype=np.int32)
        for i, (f, box) in enumerate(targets + [(k % fs.F, [20 + k, 30, 40, 50]) for k in range(N_DECOY_ROWS)]):
            recs[i, 0], recs[i, 1:5] = f, box
            recs[i, 9:12] = np.clip(np.rint(means[f]), 0, 255)
            recs[i, 12:16] = [1000 + i, -7, 12345, i]  # reserved fields: kept
        recs[N - 1, 0] = fs.F + 1  # frame index outside [0, F) (a decoy entry sits at F): padding crop, box kept
        gstate = Guarded.of(torch.from_numpy(recs), recs.size)
        snap = []

        def on_fill(fill, fs=fs):
            fs.fill(fill)
            snap[:] = [fill, fs.snapshot()]
        for size, off in ((256, 2.0), (128, 0.2)):
            gcrops = Guarded.out((N, size, size, 3), torch.uint8, size * size * 3)
            tag = f"{source} crop {size} {off}"
            crops, state = chk.run(tag, lambda: fs.crop(lib, fs.gtable, gstate, N, off, size, gcrops), [fs.gtable],
                                   [gcrops], owned={gstate: (N, slice(5, 9))}, on_fill=on_fill)
            if not fs.guards_ok(snap[0]) or not fs.frame_bytes_ok(snap[1]):
                chk.fail(f"{tag}: a frame buffer was written")
            got, ctx = crops.cpu().numpy(), state.cpu().numpy()[:, 5:9]
            for i, (f, box) in enumerate(targets[:-1]):
                if not np.array_equal(ctx[i], image_ops.context_box(box, off)):
                    chk.fail(f"{tag} target {i}: context box")
                if not np.array_equal(got[i], _cv2_crop(fs.rgb[f], box, size, off, means[f])):
                    chk.fail(f"{tag} target {i} frame {f} {box}: crop differs from cv2")
            if not (got[N - 1] == recs[N - 1, 9:12].astype(np.uint8)).all():
                chk.fail(f"{tag}: out-of-range target is not a padding-colour crop")
        # advance: random boxes against the host rescale + clamp
        nb = 2000
        arecs = np.zeros((nb + N_DECOY_ROWS, _lib.TARGET_INTS), dtype=np.int32)
        arecs[:, 0] = rng.integers(0, fs.F, nb + N_DECOY_ROWS)
        arecs[:, 1:5] = rng.integers(0, 50, (nb + N_DECOY_ROWS, 4))
        arecs[:, 5:7] = rng.integers(-600, 700, (nb + N_DECOY_ROWS, 2))
        arecs[:, 7:9] = rng.integers(1, 2000, (nb + N_DECOY_ROWS, 2))
        arecs[:, 9:16] = rng.integers(-99, 999, (nb + N_DECOY_ROWS, 7))
        arecs[10:15, 0] = fs.F + 1  # out of range: box kept (not at the end, where a short grid would hide)
        boxes = np.zeros(nb, dtype=_lib.BOX_DTYPE)
        boxes["x"], boxes["y"] = rng.uniform(-300, 600, nb), rng.uniform(-300, 600, nb)
        boxes["w"], boxes["h"] = rng.uniform(0, 300, nb), rng.uniform(0, 300, nb)
        gboxes = Guarded.of(torch.from_numpy(boxes.view(np.uint8).copy()), 48)
        gast = Guarded.of(torch.from_numpy(arecs), arecs.size)
        tag = f"{source} advance"
        state = chk.run(tag, lambda: fs.advance(lib, gboxes, gast, nb), [fs.gtable, gboxes], [],
                        owned={gast: (nb, slice(1, 5))}, on_fill=on_fill)[0].cpu().numpy()
        for i in range(nb):
            if 10 <= i < 15:
                want = arecs[i, 1:5]
            else:
                b = np.array([boxes["x"][i], boxes["y"][i], boxes["w"][i], boxes["h"][i]])
                h, w = fs.shapes[arecs[i, 0]]
                want = image_ops.clamp_bbox(image_ops.rescale_bbox(b, arecs[i, 5:9], 256), (h, w, 3))
            if not np.array_equal(state[i, 1:5], want):
                chk.fail(f"{tag} target {i}: box differs from the host rescale + clamp")
                break
        if source != "packed":
            gsums = Guarded.out((fs.F, 3), torch.int64, 3)
            sums = chk.run(f"{source} frame_sums", lambda: fs.sums(lib, gsums), [fs.gtable], [gsums],
                           on_fill=on_fill)[0].cpu().numpy().view(np.uint64)
            for i, f in enumerate(fs.rgb):
                if not np.array_equal(sums[i], f.sum(axis=(0, 1), dtype=np.uint64)):
                    chk.fail(f"{source} frame_sums frame {i}: differs from numpy")
    return chk.report()


# ------------------------------------------------------------------------------------------------------- trackers
def group_trackers():
    """FEARMultiTracker on the demo clip (the 8 CLIP_TARGETS plus a second, cropped stream whose packed frames leave
    alignment gaps) in three runs -- graph, eager, YUV frames -- with the net's workspace, zf / crop rows >= n and the
    packed frame buffer's gaps poisoned and state rows >= n filled with decoys before every update and add; one remove
    and one late add.  Every id, box and score must equal an unpoisoned tracker's.  Then FEARTracker(gpu_crop=True) with
    the workspace poisoned between updates must give the golden trajectory."""
    import cv2

    from feartracker_b200.multi_tracker import YUV420Frame
    from tests.helpers import GOLDEN, golden
    from tests.test_gpu_multi_tracker import CLIP_TARGETS

    cfg = fb.FEAR_XS_TRACKER_KWARGS
    clip = fo.read_video_rgb(os.path.join(GOLDEN, "test.mp4"))
    T = 60
    window = np.ascontiguousarray(clip[:T + 1, 30:200, 50:350])  # 170 x 300 x 3: not a multiple of 16 bytes
    late = [[300, 80, 60, 90], [20, 20, 40, 40]]
    chk = Checker()
    res = {"frames": T}

    def nv12(frame):
        h, w = frame.shape[:2]
        i420 = cv2.cvtColor(frame, cv2.COLOR_RGB2YUV_I420).reshape(-1)
        q = h * w // 4
        surf = torch.full((h + h // 2, w + 32), 0xA5, dtype=torch.uint8)  # pitch bytes hold poison
        surf[:h, :w] = torch.from_numpy(i420[:h * w].reshape(h, w))
        uv = np.stack([i420[h * w:h * w + q].reshape(h // 2, w // 2), i420[h * w + q:].reshape(h // 2, w // 2)], -1)
        surf[h:, :w] = torch.from_numpy(uv.reshape(h // 2, w))
        return YUV420Frame.nv12(surf.cuda()[:, :w])

    def frames_at(t, kind):
        fr = [window[t], clip[t]]
        return [nv12(f) for f in fr] if kind == "yuv" else fr

    def poison(trk, net, fill):
        word, byte = FILLS[fill]
        _lib.check(_lib.load().fear_debug_fill_workspace(net._handle, word, stream()), "fear_debug_fill_workspace")
        b, n = trk._buf, len(trk)
        if b is None:
            return
        b["zf"][n:].view(torch.int32).fill_(as_i32(word))
        b["crops"][n:].fill_(byte)
        b["tcrops"][n:].fill_(byte)
        decoy = torch.tensor([0, 100, 100, 50, 50, 0, 0, 0, 0, 1, 2, 3, 0, 0, 0, 0], dtype=torch.int32)
        b["state"][n:] = decoy.cuda()
        if b["frames_pin"] is not None:  # the packed numpy frames' alignment gaps and tail
            pin, offs = b["frames_pin"].numpy(), b["offsets"]
            ends = [o + f.size for o, f in zip(offs, (window[0], clip[0]))]
            for e, nxt in zip(ends, offs[1:] + [pin.size]):
                pin[e:nxt] = byte
            b["frames"][b["nbytes"]:].fill_(byte)

    def run(kind, eager, poisoned):
        net = make_net(1)
        c = dict(cfg, cuda_graph=False) if eager else cfg
        trk = fb.FEARMultiTracker(net, cuda_id=0, max_targets=12, **c)
        outs = []
        fills = ["A", "B"]

        def step(t, fn):
            placed = poisoned and trk._buf is not None  # the first add allocates the tracker's buffers
            if poisoned:
                poison(trk, net, fills[t % 2])
                chk.calls += 1
            out = fn()
            if placed:
                n = len(trk)
                torch.cuda.synchronize()
                if not bool((trk._buf["state"][n:, 1:5] == torch.tensor([100, 100, 50, 50], device="cuda")).all()):
                    chk.fail(f"{kind} eager={eager} step {t}: a decoy state row past n was written")
            return out

        step(0, lambda: trk.add(frames_at(0, kind), CLIP_TARGETS + [[40, 30, 50, 60]], [1] * 8 + [0]))
        for t in range(1, T + 1):
            if t == 25:
                trk.remove([2, 6])
            if t == 30:
                step(t, lambda: trk.add(frames_at(t, kind), late, [1, 0]))
            outs.append(step(t, lambda: trk.update(frames_at(t, kind))))
        return outs

    for kind, eager in (("numpy", False), ("numpy", True), ("yuv", False)):
        want = run(kind, eager, False)
        got = run(kind, eager, True)
        for t, (a, b) in enumerate(zip(got, want)):
            if not (np.array_equal(a["ids"], b["ids"]) and np.array_equal(a["bbox"], b["bbox"])
                    and np.array_equal(a["score"], b["score"])):
                chk.fail(f"multi-tracker {kind} eager={eager} frame {t + 1}: differs from the unpoisoned tracker")
                break
        res[f"{kind} eager={eager} targets"] = int(len(got[-1]["ids"]))
    # FEARTracker(gpu_crop=True): the workspace poisoned between updates
    g = golden("video_teacher.npz")
    net = make_net(1)
    trk = fb.FEARTracker(net, cuda_id=0, gpu_crop=True, **cfg)
    trk.initialize(clip[0], g["init_bbox"])
    traj = []
    for t, f in enumerate(clip[1:]):
        _lib.check(_lib.load().fear_debug_fill_workspace(net._handle, FILLS["AB"[t % 2]][0], stream()),
                   "fear_debug_fill_workspace")
        traj.append(list(map(int, trk.update(f)["bbox"])))
        chk.calls += 1
    same = (np.array(traj) == g["trajectory"]).all(1)
    if not same.all():
        chk.fail(f"FEARTracker(gpu_crop) on a poisoned workspace leaves the golden trajectory at frame "
                 f"{int(np.argmin(same)) + 1}")
    res["gpu_crop_frames"] = len(traj)
    res.update(chk.report())
    return res


# ------------------------------------------------------------------------------------------------------- the entry
def group_entry():
    """fear_debug_fill_workspace itself: refused without a handle, counted nowhere, generation unchanged, fills every
    word of the workspace (seen through fear_debug_head_tensor rows a call did not write)."""
    lib, res = _lib.load(), {}
    res["null_handle"] = lib.fear_debug_fill_workspace(None, 0, None)
    net = make_net(2)
    n0, g0 = net.launch_count(), net.generation()
    _lib.check(lib.fear_debug_fill_workspace(net._handle, POISON_A, stream()), "fear_debug_fill_workspace")
    out = torch.empty(2, 320, 16, 16, device="cuda")
    _lib.check(lib.fear_debug_head_tensor(net._handle, b"cat_reg", 2, out.data_ptr(), stream()), "head_tensor")
    n1 = net.launch_count()
    torch.cuda.synchronize()
    res["launches_of_fill"] = n1 - n0 - 1  # the head-tensor copy is one counted launch
    res["generation_unchanged"] = net.generation() == g0
    res["all_poison"] = bool((out.view(torch.int32) == as_i32(POISON_A)).all())
    # captured into a CUDA graph and replayed
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            _lib.check(lib.fear_debug_fill_workspace(net._handle, POISON_B, torch.cuda.current_stream().cuda_stream),
                       "fear_debug_fill_workspace")
    torch.cuda.current_stream().wait_stream(s)
    g.replay()
    out2 = torch.empty(2, 256, 16, 16, device="cuda")
    _lib.check(lib.fear_debug_head_tensor(net._handle, b"cls_tower", 2, out2.data_ptr(), stream()), "head_tensor")
    torch.cuda.synchronize()
    res["graph_fill"] = bool((out2.view(torch.int32) == as_i32(POISON_B)).all())
    return res


GROUPS = {"features": group_features, "head": group_head, "track": group_track, "decode": group_decode,
          "corr": group_corr, "crops": group_crops, "loop": group_loop, "trackers": group_trackers,
          "entry": group_entry}


def main():
    torch.manual_seed(0)
    args = sys.argv[2:]
    if sys.argv[1] == "features":
        args = [int(a) for a in args]
    res = GROUPS[sys.argv[1]](*args)
    print("POISON_CHECK " + json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
