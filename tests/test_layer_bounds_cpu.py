"""CPU checks of the element-wise error model of tests/layer_bounds.py: it holds for an fp32 emulation of the
3xTF32 and CUDA-core arithmetic, it rejects emulated precision mutants, and the weight blobs the GPU test packs
round-trip through the library's weight order."""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from feartracker_b200 import _lib
from oracle import fear_oracle as fo
from tests import layer_bounds as lb
from tests.helpers import load_full_state

XIF4_5 = 13  # index of xif4_5 in lb.BLOCKS


@pytest.fixture(scope="module")
def table():
    return _lib.weight_table()


@pytest.fixture(scope="module")
def sets(table):
    return lb.weight_sets({k: v for k, v in load_full_state().items() if v.is_floating_point()}, table)


# ------------------------------------------------------------------------------------------------ emulation
def _trunc_tf32(a):
    return (np.ascontiguousarray(a, dtype=np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def _to_f32_rz(s):
    """float64 -> float32 rounded toward zero."""
    f = s.astype(np.float32)
    over = np.abs(f.astype(np.float64)) > np.abs(s)
    f[over] = np.nextafter(f[over], np.float32(0))
    return f


def gemm_3xtf32(x, w, b, res=None, relu=False, w_lo_round="rna", drop_last_corr=False, w_split="rna"):
    """Emulation of pw_tc_kernel on (M, K) fp32 activations and (N, K) fp32 weights: load_a_frags' truncation split,
    fear_pack_weights' rna split (or a truncated w_lo), tf32 truncation of x_lo by the tensor core, exact products,
    one truncating fp32 accumulation per k = 8 step (main and correction accumulators), then the epilogue.
    drop_last_corr skips both correction products of the last 32-channel chunk.  w_split="trunc" splits the second
    operand as corr_tc_kernel splits the templates (hi truncated, lo exact and truncated by the tensor core)."""
    xh = _trunc_tf32(x)
    xl = _trunc_tf32((x - xh).astype(np.float32))
    if w_split == "trunc":
        wh = _trunc_tf32(w)
        wl = _trunc_tf32((w - wh).astype(np.float32))
    else:
        wh = lb._round_tf32(w)
        r = (w - wh).astype(np.float32)
        wl = lb._round_tf32(r) if w_lo_round == "rna" else _trunc_tf32(r)
    M, K = x.shape
    main = np.zeros((M, w.shape[0]), np.float32)
    corr = np.zeros_like(main)
    last_chunk = 32 * ((K - 1) // 32)
    for k0 in range(0, K, 8):
        sl = slice(k0, min(k0 + 8, K))
        x8h, x8l = xh[:, sl].astype(np.float64), xl[:, sl].astype(np.float64)
        w8h, w8l = wh[:, sl].astype(np.float64), wl[:, sl].astype(np.float64)
        main = _to_f32_rz(main.astype(np.float64) + x8h @ w8h.T)
        if drop_last_corr and k0 >= last_chunk:
            continue
        corr = _to_f32_rz(corr.astype(np.float64) + x8h @ w8l.T)
        corr = _to_f32_rz(corr.astype(np.float64) + x8l @ w8h.T)
    o = main + corr
    bb = np.broadcast_to(b.astype(np.float32), o.shape)
    if res is not None:
        bb = bb + res
    o = o + bb
    return np.maximum(o, 0) if relu else o


def _nhwc(t):
    return t.permute(0, 2, 3, 1).reshape(-1, t.shape[1]).numpy()


def _nchw(a, like):
    B, _, H, W = like.shape
    return torch.from_numpy(np.ascontiguousarray(a)).view(B, H, W, -1).permute(0, 3, 1, 2)


def emulate_block(W32, n, x32, **kw):
    """Block n in fp32: the 1x1 convs through gemm_3xtf32 (or torch fp32 for the CUDA-core 16x16 / 24x24 ones), the
    depthwise conv in torch fp32.  kw go to the pwl GEMM."""
    s = lb.BLOCKS[n]
    h = x32
    tc = lambda a, b: (a, b) not in ((16, 16), (24, 24))  # noqa: E731
    if s.expand != 1:
        w, b = W32[s.name + ".pw.w"], W32[s.name + ".pw.b"]
        h = (_nchw(gemm_3xtf32(_nhwc(h), w[:, :, 0, 0].numpy(), b.numpy(), relu=True), h) if tc(s.cin, s.mid)
             else torch.relu(F.conv2d(h, w, b)))
    h = torch.relu(F.conv2d(h, W32[s.name + ".dw.w"], W32[s.name + ".dw.b"], s.stride, s.k // 2, 1, s.mid))
    w, b = W32[s.name + ".pwl.w"], W32[s.name + ".pwl.b"]
    if not tc(s.mid, s.cout):
        y = F.conv2d(h, w, b)
        return y + x32 if s.residual else y
    res = _nhwc(x32) if s.residual else None
    return _nchw(gemm_3xtf32(_nhwc(h), w[:, :, 0, 0].numpy(), b.numpy(), res=res, **kw), h)


@pytest.fixture(scope="module")
def chain(sets, table):
    """fp64 chain of the checkpoint on synthetic_crops(2): the input of every block, cast to fp32."""
    W64 = lb.unpack(*sets["checkpoint"], table)
    W32 = {k: v.float() for k, v in W64.items()}
    _, xt, _, _ = fo.synthetic_crops(2)
    x = lb.stem(W64, lb.exact(xt)).y
    ins = []
    for n in range(len(lb.BLOCKS)):
        ins.append(x.float())
        x = lb.block(W64, n, lb.exact(x.float())).y
    return W64, W32, xt, ins


def emulate_pw(x32, w, b, relu=False):
    """A 1x1 conv on the tensor cores (NCHW fp32 in and out)."""
    return _nchw(gemm_3xtf32(_nhwc(x32), w[:, :, 0, 0].numpy(), b.numpy(), relu=relu), x32)


def emulate_sepconv(W32, prefix, x32):
    """Head SepConv: depthwise 3x3 on CUDA cores (torch fp32), then the 1x1 conv on the tensor cores + ReLU."""
    d = F.conv2d(x32, W32[prefix + ".dw.w"], None, 1, 1, 1, x32.shape[1])
    return emulate_pw(d, W32[prefix + ".pw.w"], W32[prefix + ".pw.b"], relu=True)


def emulate_corr(z32, x32):
    """corr_tc_kernel per frame: (256 search cells x 256 ch) against (64 template cells x 256 ch), both operands split
    by truncation, main + corr as the only epilogue add."""
    out = []
    for b in range(x32.shape[0]):
        X = x32[b].reshape(256, 256).T.contiguous().numpy()
        Z = z32[b].reshape(256, 64).T.contiguous().numpy()
        out.append(gemm_3xtf32(X, Z, np.zeros(64, np.float32), w_split="trunc").T.reshape(64, 16, 16))
    return torch.from_numpy(np.ascontiguousarray(np.stack(out)))


def emulate_pred(W32, name, x32, exp=False):
    """Depthwise 3x3 (torch fp32), then pred_pw_kernel's order: per lane 8 products (1 multiply, 7 fma), a 5-level
    butterfly of fp32 adds over 32 lanes, + bias, expf for bbox."""
    d = F.conv2d(x32, W32[name + ".dw.w"], None, 1, 1, 1, 256)
    B = d.shape[0]
    v = d.permute(0, 2, 3, 1).reshape(-1, 256).numpy().astype(np.float64)
    w = W32[name + ".pw.w"][:, :, 0, 0].numpy().astype(np.float64)
    lane = np.arange(32)
    chans = [4 * lane + i for i in range(4)] + [128 + 4 * lane + i for i in range(4)]  # each (32,)
    outs = []
    for o in range(w.shape[0]):
        s = (v[:, chans[0]] * w[o, chans[0]]).astype(np.float32)
        for c in chans[1:]:
            s = (v[:, c] * w[o, c] + s.astype(np.float64)).astype(np.float32)  # fma: exact product, one rounding
        for dd in (16, 8, 4, 2, 1):
            s = (s + s[:, lane ^ dd]).astype(np.float32)
        outs.append((s[:, 0] + np.float32(W32[name + ".pw.b"][o].item())).astype(np.float32))
    y = torch.from_numpy(np.stack(outs, 1)).view(B, 16, 16, -1).permute(0, 3, 1, 2)
    return torch.exp(y) if exp else y


# ------------------------------------------------------------------------------------------------ tests
def test_weight_blobs_round_trip_library_order(sets, table):
    """Each blob holds exactly the library's tensors in fear_weight_name order with fear_weight_numel elements, and the
    fp64 tensors the oracle unpacks are the blob's values."""
    assert [n for n, _ in table] == [_lib.load().fear_weight_name(i).decode() for i in range(len(table))]
    for name, (blob, off) in sets.items():
        assert blob.dtype == np.float32 and off.dtype == np.uint64 and len(off) == len(table) + 1
        assert int(off[-1]) == blob.size == sum(n for _, n in table), name
        assert np.isfinite(blob).all(), name
        W = lb.unpack(blob, off, table)
        for i, (tname, numel) in enumerate(table):
            seg = blob[int(off[i]):int(off[i + 1])]
            assert seg.size == numel
            if tname in W:
                np.testing.assert_array_equal(W[tname].reshape(-1).numpy(), seg.astype(np.float64))
    ck, _ = sets["checkpoint"]
    from feartracker_b200 import weights

    sd = {k: v for k, v in load_full_state().items() if v.is_floating_point()}
    np.testing.assert_array_equal(ck, weights.pack(sd, table)[0])
    # tf32-exact set: every GEMM weight has w_lo = 0; the other two have non-zero lo parts nearly everywhere
    for name, (blob, off) in sets.items():
        gem = np.concatenate([blob[int(off[i]):int(off[i + 1])] for i, (t, _) in enumerate(table) if lb.is_gemm_weight(t)])
        lo_zero = float(np.mean(lb._round_tf32(gem) == gem))
        if name == "tf32_exact":
            assert lo_zero == 1.0
        else:
            assert lo_zero < 0.01, (name, lo_zero)
    # wide set: every GEMM layer has output channels ~10^4 below its largest
    W = lb.unpack(*sets["wide"], table)
    for t, _ in table:
        if lb.is_gemm_weight(t):
            w = W[t].reshape(W[t].shape[0], -1).abs().amax(1)
            assert float(w.max() / w.min()) > 1e3, t


def test_model_holds_for_fp32_emulation(chain):
    """Every backbone block emulated in fp32 (3xTF32 GEMMs bit-modelled in numpy, CUDA-core convs in torch fp32) from
    the fp32 block input: every element within (a), the RMS within (b); likewise the stem."""
    W64, W32, xt, ins = chain
    report = {"stem": lb.compare(F.relu(F.conv2d(xt, W32["stem.w"], W32["stem.b"], 2, 1)), lb.stem(W64, lb.exact(xt)))}
    for n, x32 in enumerate(ins):
        report[lb.BLOCKS[n].name] = lb.compare(emulate_block(W32, n, x32), lb.block(W64, n, lb.exact(x32)))
    bad = {k: v for k, v in report.items() if not (v["a"] <= 1 and v["b"] <= 1)}
    assert not bad, bad


def test_model_holds_for_fp32_emulation_of_neck_and_head(chain, table, sets):
    """The neck and every head stage emulated in fp32 with the arithmetic the model assigns to it (3xTF32 GEMM and
    correlation bit-modelled in numpy, CUDA-core depthwise and FFMA correlation in torch fp32, pred_pw_kernel's order,
    expf) from the fp32 stage input: every element within (a), the RMS within (b)."""
    W64, W32, _, ins = chain
    zt, _, _, _ = fo.synthetic_crops(2)
    x = lb.block(W64, len(lb.BLOCKS) - 1, lb.exact(ins[-1])).y.float()
    z = lb.stem(W64, lb.exact(zt)).y
    for n in range(len(lb.BLOCKS)):
        z = lb.block(W64, n, lb.exact(z.float())).y
    zf = lb.neck(W64, lb.exact(z.float())).y.float()
    report = {"neck": lb.compare(emulate_pw(x, W32["neck.w"], W32["neck.b"]), lb.neck(W64, lb.exact(x)))}
    xf = lb.neck(W64, lb.exact(x)).y.float()
    for br in ("cls", "reg"):
        enc = lb.sepconv(W64, br + "_encode", lb.exact(xf)).y.float()
        report[br + "_encode"] = lb.compare(emulate_sepconv(W32, br + "_encode", xf), lb.sepconv(W64, br + "_encode", lb.exact(xf)))
        want = lb.correlation(lb.exact(zf), lb.exact(enc))
        report[br + "_corr"] = lb.compare(emulate_corr(zf, enc), want)
        zz, ee = zf.reshape(2, 256, 64), enc.reshape(2, 256, 256)
        report[br + "_corr_ffma"] = lb.compare(torch.bmm(zz.transpose(1, 2), ee).view(2, 64, 16, 16),
                                               lb.correlation(lb.exact(zf), lb.exact(enc), "ffma"))
        cat = torch.cat([enc, want.y.float()], 1)
        report[br + "_dw"] = lb.compare(emulate_sepconv(W32, br + "_dw", cat), lb.sepconv(W64, br + "_dw", lb.exact(cat)))
        dw = lb.sepconv(W64, br + "_dw", lb.exact(cat)).y.float()
        tw = "cls_tower" if br == "cls" else "bbox_tower"
        mid = emulate_sepconv(W32, tw + ".0", dw)
        report[tw] = lb.compare(emulate_sepconv(W32, tw + ".1", mid), lb.tower(W64, tw, lb.exact(dw)))
        t = lb.tower(W64, tw, lb.exact(dw)).y.float()
        pn = "cls_pred" if br == "cls" else "bbox_pred"
        report[pn] = lb.compare(emulate_pred(W32, pn, t, exp=pn == "bbox_pred"), lb.pred(W64, pn, lb.exact(t)),
                                log_of_exp=pn == "bbox_pred")
    bad = {k: v for k, v in report.items() if not (v["a"] <= 1 and v["b"] <= 1 and v["nonfinite"] == 0)}
    assert not bad, (bad, report)


@pytest.mark.parametrize("scaled", [False, True])
def test_model_holds_for_coherent_correlation(scaled):
    """The correlation with non-negative operands, whose truncation errors all keep one sign and add up coherently,
    optionally with per-channel scales in 2^[-8, 8]: the emulated corr_tc_kernel stays within (a) and (b)."""
    g = torch.Generator().manual_seed(5 + scaled)
    z = torch.rand(2, 256, 8, 8, generator=g)
    x = torch.rand(2, 256, 16, 16, generator=g)
    if scaled:
        z = z * 2.0 ** (torch.rand(1, 256, 1, 1, generator=g) * 16 - 8)
        x = x * 2.0 ** (torch.rand(1, 256, 1, 1, generator=g) * 16 - 8)
    r = lb.compare(emulate_corr(z, x), lb.correlation(lb.exact(z), lb.exact(x)))
    assert r["a"] <= 1 and r["b"] <= 1, r


def test_emulated_mutants_fail_the_rms_check(chain, tmp_path):
    """(1) xif4_5.pwl without the 3xTF32 correction of its last 32-channel chunk fails (b) by a wide margin (the suite's
    inf-norm bar of 2e-5, recorded as inf_norm, sees it by less).  (2) w_lo truncated instead of rna-rounded is only
    recorded: a truncated lo part errs by < 2^-21 |w| against <= 2^-22 |w| for rna, the same size as the truncation
    error of the activation split (< 2^-21 |x|) that the model must admit for a correct kernel, so no bound that
    admits a correct kernel can reject it."""
    W64, W32, _, ins = chain
    x32 = ins[XIF4_5]
    want = lb.block(W64, XIF4_5, lb.exact(x32))
    report = {}
    for name, kw in (("correct", {}), ("no_corr_last_chunk", {"drop_last_corr": True}),
                     ("w_lo_truncated", {"w_lo_round": "trunc"})):
        got = emulate_block(W32, XIF4_5, x32, **kw)
        r = lb.compare(got, want)
        r["inf_norm"] = lb.legacy_inf_norm(got, want.y)
        report[name] = r
    m = report["no_corr_last_chunk"]
    assert report["correct"]["b"] <= 1 and report["correct"]["a"] <= 1, report
    assert m["b"] > 3, report  # fails the RMS check
    assert m["b"] / report["correct"]["b"] > 15, report  # far above what the correct kernel reaches
    with open(os.path.join(str(tmp_path), "mutant_margins.json"), "w") as f:
        json.dump(report, f, indent=1)
    print(json.dumps(report))
