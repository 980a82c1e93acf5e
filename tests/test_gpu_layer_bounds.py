"""Every stage of the hot path, in isolation, against the element-wise fp64 error model of tests/layer_bounds.py.

Each stage's input is the library's own fp32 output of the previous stage (fear_debug_backbone_prefix,
fear_debug_head_tensor); the stage runs once more in float64 from the folded weights the library was packed with, and
every output element must lie within (a) the worst-case bound, and the stage's RMS error within (b) the model's RMS
bound.  Weight sets: the checkpoint, a wide-scale set and a set with tf32-exact GEMM weights, all packed through
fear_pack_weights.  Observed / bound ratios of every stage go to layer_bounds.json in the test's tmp directory and to
stdout."""
import ctypes
import hashlib
import json
import os

import numpy as np
import pytest
import torch

from feartracker_b200 import _lib
from tests import layer_bounds as lb
from tests.helpers import load_full_state

pytestmark = pytest.mark.gpu

# fear_track_u8 at 256 x 256: the busiest CTA of xif3_0's depthwise launch (dw_tma<5,2>) gets 9 tiles at B = 14 on 132
# SMs (tests/schedule_plan.py, regime cta_9plus_tiles)
B_SCHED = 14
VARIANTS = {"default": {}, "pw=ffma": {"pw": "ffma"}, "corr=ffma": {"corr": "ffma"}, "fuse_irf=0": {"fuse_irf": "0"}}
REPORT = {}


class Handle:
    """One fear_pack_weights handle on a given blob."""

    def __init__(self, blob, offsets, opts, reserve):
        self.lib = _lib.init(0)
        self.h = ctypes.c_void_p()
        _lib.check(self.lib.fear_pack_weights(blob.ctypes.data_as(ctypes.c_void_p),
                                              offsets.ctypes.data_as(ctypes.POINTER(ctypes.c_uint64)),
                                              len(offsets) - 1, ctypes.byref(self.h)), "fear_pack_weights")
        for k, v in opts.items():
            _lib.check(self.lib.fear_set_option(self.h, k.encode(), v.encode()), "fear_set_option")
        _lib.check(self.lib.fear_reserve(self.h, reserve), "fear_reserve")
        self.st = torch.cuda.current_stream().cuda_stream

    def free(self):
        self.lib.fear_free(self.h)

    def prefix(self, img, n):
        B, _, H, W = img.shape
        s = lb.BLOCKS[n - 1] if n else None
        c = s.cout if n else 16
        down = 2 * int(np.prod([b.stride for b in lb.BLOCKS[:n]]))
        out = torch.empty((B, c, H // down, W // down), device="cuda")
        _lib.check(self.lib.fear_debug_backbone_prefix(self.h, img.data_ptr(), B, H, W, n, out.data_ptr(), self.st),
                   "fear_debug_backbone_prefix")
        return out

    def features_u8(self, u8):
        B, H, W, _ = u8.shape
        out = torch.empty((B, 256, H // 16, W // 16), device="cuda")
        _lib.check(self.lib.fear_get_features_u8(self.h, u8.data_ptr(), B, H, W, out.data_ptr(), self.st),
                   "fear_get_features_u8")
        return out

    def track_u8(self, u8, zf):
        B = u8.shape[0]
        bbox, cls = torch.empty((B, 4, 16, 16), device="cuda"), torch.empty((B, 1, 16, 16), device="cuda")
        _lib.check(self.lib.fear_track_u8(self.h, u8.data_ptr(), zf.data_ptr(), zf.shape[0], B, bbox.data_ptr(),
                                          cls.data_ptr(), None, self.st), "fear_track_u8")
        return bbox, cls

    def head(self, zf, xf, zu=None):
        B = xf.shape[0]
        bbox, cls = torch.empty((B, 4, 16, 16), device="cuda"), torch.empty((B, 1, 16, 16), device="cuda")
        _lib.check(self.lib.fear_head_update(self.h, zf.data_ptr(), zf.shape[0], zu.data_ptr() if zu is not None else None,
                                             zu.shape[0] if zu is not None else 0, xf.data_ptr(), B, bbox.data_ptr(),
                                             cls.data_ptr(), self.st), "fear_head_update")
        return bbox, cls

    def head_tensor(self, name, B):
        out = torch.empty((B, 320 if name.startswith("cat_") else 256, 16, 16), device="cuda")
        _lib.check(self.lib.fear_debug_head_tensor(self.h, name.encode(), B, out.data_ptr(), self.st),
                   "fear_debug_head_tensor")
        return out


class Rep(dict):
    """Per-stage results of one case (weight set / options / entry point / batch), named for failure messages."""

    def __init__(self, case):
        super().__init__()
        self.case = case


class Checker:
    """Runs the fp64 stage of each frame and accumulates the (a) / (b) ratios per stage.  The oracle is cached on the
    stage, the arithmetic the options select for it (pw, corr) and the stage's input bytes: a frame whose input is
    bit-identical to one seen before under the same arithmetic reuses its oracle."""

    def __init__(self, W):
        self.W, self.cache, self.arith = W, {}, ("auto", "auto")

    def check(self, rep, stage, got, fn, *inputs, log_of_exp=False):
        a, b2 = 0.0, 0.0
        for f in range(got.shape[0]):
            xs = [t[f:f + 1].detach().cpu() if t.shape[0] > 1 else t.detach().cpu() for t in inputs]
            key = (stage, self.arith, hashlib.sha1(b"".join(x.numpy().tobytes() for x in xs)).hexdigest())
            if key not in self.cache:
                self.cache[key] = fn(*[lb.exact(x) for x in xs])
            r = lb.compare(got[f:f + 1], self.cache[key], log_of_exp=log_of_exp)
            assert r["nonfinite"] == 0, \
                f"{rep.case}: stage {stage}: frame {f}: {r['nonfinite']} output elements are not finite" + \
                (" (bbox <= 0 or inf)" if log_of_exp else "")
            a, b2 = max(a, r["a"]), b2 + r["b"] ** 2
        old = rep.get(stage)
        n = got.shape[0]
        if old:
            a, b2, n = max(a, old["a"]), b2 + old["b"] ** 2 * old["frames"], n + old["frames"]
        rep[stage] = {"a": a, "b": float(np.sqrt(b2 / n)), "frames": n}


def _crops(H, W, n=None):
    c = lb.input_crops(H, W)
    names = list(c)
    if n is not None:
        names = [names[i % len(names)] for i in range(n)]
    return names, np.stack([c[k] for k in names])


def _backbone(h, chk, rep, u8, pw):
    img = lb.normalize_u8(u8).cuda()
    P = [h.prefix(img, n) for n in range(len(lb.BLOCKS) + 1)]
    chk.check(rep, "stem", P[0], lambda x: lb.stem(chk.W, x), img)
    for n, s in enumerate(lb.BLOCKS):
        chk.check(rep, s.name, P[n + 1], lambda x, n=n: lb.block(chk.W, n, x, pw), P[n])
    feat = h.features_u8(torch.from_numpy(u8).cuda())
    chk.check(rep, "neck", feat, lambda x: lb.neck(chk.W, x, pw), P[-1])
    return feat


def _head_stages(h, chk, rep, B, zf, zu, bbox, cls, pw, corr, tag):
    T = {n: h.head_tensor(n, B) for n in ("search_features", "cat_cls", "cat_reg", "cls_dw", "reg_dw", "x_reg",
                                          "cls_tower")}
    W = chk.W
    for br, z in (("cls", zu if zu is not None else zf), ("reg", zf)):
        cat = T["cat_" + br]
        chk.check(rep, f"{tag}{br}_encode", cat[:, :256], lambda x, br=br: lb.sepconv(W, br + "_encode", x, pw),
                  T["search_features"])
        chk.check(rep, f"{tag}{br}_corr", cat[:, 256:], lambda zz, x: lb.correlation(zz, x, corr), z, cat[:, :256])
        chk.check(rep, f"{tag}{br}_dw", T[br + "_dw"], lambda x, br=br: lb.sepconv(W, br + "_dw", x, pw), cat)
    chk.check(rep, f"{tag}cls_tower", T["cls_tower"], lambda x: lb.tower(W, "cls_tower", x, pw), T["cls_dw"])
    chk.check(rep, f"{tag}bbox_tower", T["x_reg"], lambda x: lb.tower(W, "bbox_tower", x, pw), T["reg_dw"])
    chk.check(rep, f"{tag}cls", cls, lambda x: lb.pred(W, "cls_pred", x), T["cls_tower"])
    chk.check(rep, f"{tag}bbox", bbox, lambda x: lb.pred(W, "bbox_pred", x), T["x_reg"], log_of_exp=True)
    return T


def _corr_entry_points(chk, rep, zf, x):
    """fear_corr_nhwc_f32 / fear_corr_concat_ws_f32 (wgmma) and fear_corr_concat_f32 (CUDA cores) on the head's own
    encode output and template features."""
    lib = _lib.init(0)
    st = torch.cuda.current_stream().cuda_stream
    B, Bz = x.shape[0], zf.shape[0]
    z = zf.reshape(Bz, 256, 64).contiguous()
    xc = x.contiguous()
    out = torch.empty(B, 320, 16, 16, device="cuda")
    _lib.check(lib.fear_corr_concat_f32(z.data_ptr(), Bz, xc.data_ptr(), B, out.data_ptr(), st), "fear_corr_concat_f32")
    chk.check(rep, "corr_concat_f32", out[:, 256:], lambda zz, xx: lb.correlation(zz, xx, "ffma"), zf, x)
    need = lib.fear_corr_concat_workspace_bytes(B, Bz)
    ws = torch.empty(need // 4 + 256, device="cuda")
    off = (-ws.data_ptr()) % 1024
    out2 = torch.empty_like(out)
    _lib.check(lib.fear_corr_concat_ws_f32(z.data_ptr(), Bz, xc.data_ptr(), B, out2.data_ptr(), ws.data_ptr() + off,
                                           need, st), "fear_corr_concat_ws_f32")
    chk.check(rep, "corr_concat_ws_f32", out2[:, 256:], lambda zz, xx: lb.correlation(zz, xx), zf, x)
    zt = z.transpose(1, 2).contiguous()  # [Bz][64][256]
    cat = torch.zeros(B, 256, 320, device="cuda")
    cat[:, :, :256] = x.reshape(B, 256, 256).transpose(1, 2)
    _lib.check(lib.fear_corr_nhwc_f32(zt.data_ptr(), Bz, cat.data_ptr(), B, st), "fear_corr_nhwc_f32")
    s = cat[:, :, 256:].transpose(1, 2).reshape(B, 64, 16, 16)
    chk.check(rep, "corr_nhwc_f32", s, lambda zz, xx: lb.correlation(zz, xx), zf, x)


@pytest.fixture(scope="module")
def sets():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    table = _lib.weight_table()
    sd = {k: v for k, v in load_full_state().items() if v.is_floating_point()}
    return {k: (v, lb.unpack(*v, table)) for k, v in lb.weight_sets(sd, table).items()}


@pytest.fixture(scope="module", autouse=True)
def _dump(tmp_path_factory):
    yield
    path = os.path.join(str(tmp_path_factory.mktemp("layer_bounds")), "layer_bounds.json")
    with open(path, "w") as f:
        json.dump(REPORT, f, indent=1)
    worst = {case: {k: max(v[k] for v in st.values()) for k in ("a", "b")} for case, st in REPORT.items()}
    print("\nLAYER_BOUNDS " + json.dumps({"worst": worst, "stages": REPORT}))


_CHECKERS = {}


def _rep(reports, case):
    return reports.setdefault(case, Rep(case))


@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("wset", ["checkpoint", "wide", "tf32_exact"])
def test_every_stage_within_error_model(sets, wset, variant):
    (blob, off), W = sets[wset]
    chk = _CHECKERS.setdefault(wset, Checker(W))
    opts = VARIANTS[variant]
    pw, corr = opts.get("pw", "auto"), opts.get("corr", "auto")
    chk.arith = (pw, corr)
    h = Handle(blob, off, opts, B_SCHED)
    reports = {}
    try:
        # batches: every search crop alone (B = 1), and for the default options the scheduled batch
        names, crops = _crops(256, 256)
        tnames, tcrops = _crops(128, 128, len(names))
        batches = [[i] for i in range(len(names))]
        if variant == "default":
            batches.append([i % len(names) for i in range(B_SCHED)])
        for idx in batches:
            B = len(idx)
            rep = _rep(reports, f"{wset}/{variant}/track_u8 B={B}")
            u8 = crops[idx]
            zfe = h.features_u8(torch.from_numpy(tcrops[idx]).cuda())
            if variant != "corr=ffma":
                _backbone(h, chk, rep, u8, pw)
            bbox, cls = h.track_u8(torch.from_numpy(u8).cuda(), zfe)
            T = _head_stages(h, chk, rep, B, zfe, None, bbox, cls, pw, corr, "")
            xf = T["search_features"]
            rep = _rep(reports, f"{wset}/{variant}/head B={B}")
            bbox, cls = h.head(zfe, xf)
            _head_stages(h, chk, rep, B, zfe, None, bbox, cls, pw, corr, "")
            rep = _rep(reports, f"{wset}/{variant}/head_update B=Bu={B}")
            zu = torch.roll(zfe, 1, 0) if B > 1 else h.features_u8(torch.from_numpy(tcrops[[1]]).cuda())
            bbox, cls = h.head(zfe, xf, zu)
            _head_stages(h, chk, rep, B, zfe, zu, bbox, cls, pw, corr, "")
            if variant == "default" and B == 1:
                _corr_entry_points(chk, _rep(reports, f"{wset}/corr entry points"), zfe, T["cat_cls"][:, :256])
        if variant in ("default", "pw=ffma"):
            for H, Wd in ((128, 128), (128, 256)):
                _, c = _crops(H, Wd)
                for i in range(len(c)):
                    _backbone(h, chk, _rep(reports, f"{wset}/{variant}/features_u8 {H}x{Wd} B=1"), c[i:i + 1], pw)
    finally:
        torch.cuda.synchronize()
        h.free()
    REPORT.update(reports)
    bad = [f"{case}: stage {st}: (a) {r['a']:.3g}, (b) {r['b']:.3g}" for case, rep in reports.items()
           for st, r in rep.items() if not (r["a"] <= 1 and r["b"] <= 1)]
    assert not bad, "observed / bound > 1:\n" + "\n".join(bad)
