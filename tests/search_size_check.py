"""Stand-alone checker of the search-size entry points (run in its own process: a device-side trap would poison the
CUDA context of the main pytest process).  Prints one JSON line.

    python tests/search_size_check.py parity S     # track / track_boxes / forward / connect_model vs the fp64 oracle
    python tests/search_size_check.py same256      # the fixed-size entry points run the sized ones at S = 256
    python tests/search_size_check.py chunk        # S = 192 through a 2-frame workspace == one unchunked pass
    python tests/search_size_check.py decode s     # fear_decode_sized / fear_decode_smooth_sized vs the host
    python tests/search_size_check.py poison S     # every sized entry point on a poisoned workspace, guarded buffers
    python tests/search_size_check.py trackers S   # FEARTracker on tests/golden/test.mp4, every frame path
    python tests/search_size_check.py multi S      # FEARMultiTracker vs one FEARTracker(gpu_crop) per target
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
from tests.helpers import GOLDEN, load_full_state, map_errors  # noqa: E402

R, C = fo.TARGET_REGRESSION_LABEL_KEY, fo.TARGET_CLASSIFICATION_KEY


def cfg_for(size, **kw):
    return dict(fb.FEAR_XS_TRACKER_KWARGS, instance_size=size, score_size=size // 16, **kw)


def make_net(reserve):
    net = fb.FEARNet(**fb.FEAR_XS_MODEL_KWARGS)
    net.load_state_dict(load_full_state(), strict=True)
    net = net.cuda().eval()
    net.reserve(reserve)
    return net


def sd64():
    return fo.to_dtype({k: v for k, v in load_full_state().items() if v.is_floating_point()}, torch.float64)


def stream():
    return torch.cuda.current_stream().cuda_stream


def records(boxes):
    return boxes.cpu().numpy().view(_lib.BOX_DTYPE).reshape(-1)


def maps_err(got, want):
    return [map_errors(got[k].cpu().numpy(), want[k].numpy()) for k in (R, C)]


def boxes_vs_oracle(rec, maps64, size):
    """rows / columns equal to the oracle decode of the fp64 maps; the boxes' largest violation of rtol 1e-3 /
    atol 2e-2 (<= 1 passes)."""
    bbox, coords = fo.decode(maps64[R], maps64[C], config=cfg_for(size))
    rc_ok = [(int(r), int(c)) for r, c in zip(rec["row"], rec["col"])] == [(int(r), int(c)) for r, c in coords]
    got = np.stack([rec["x"], rec["y"], rec["w"], rec["h"]], 1)
    want = bbox.numpy()
    worst = float((np.abs(got - want) / (2e-2 + 1e-3 * np.abs(want))).max())
    flat_ok = bool((rec["flat"] == rec["row"] * (size // 16) + rec["col"]).all())
    return {"rows_cols_equal": rc_ok, "flat_ok": flat_ok, "box_worst": worst}


def parity(size):
    sd = sd64()
    net = make_net(3)
    res = {}
    for B in (1, 3):
        zt, _ = fo.shape_crops(128, 128, B, seed=size + B)
        ut, _ = fo.shape_crops(128, 128, B, seed=size + B + 500)
        x, u = fo.shape_crops(size, size, B, seed=size * 7 + B)
        u8 = u.permute(0, 2, 3, 1).contiguous().cuda()
        zf = net.get_features(zt.cuda())
        uf = net.get_features(ut.cuda())
        zf64 = fo.get_features(sd, zt.double())
        xf = net.get_features(x.cuda())
        for Bz in sorted({1, B}):
            tag = f"B{B}_Bz{Bz}"
            want = fo.track(sd, x.double(), zf64[:Bz])
            got = net.track(x.cuda(), zf[:Bz])
            got_u8 = net.track(u8, zf[:Bz])
            boxes, maps_b = net.track_boxes(x.cuda(), zf[:Bz], with_maps=True)
            boxes_u8 = net.track_boxes(u8, zf[:Bz])
            r = {"shape_ok": tuple(got[R].shape) == (B, 4, size // 16, size // 16)
                 and tuple(got[C].shape) == (B, 1, size // 16, size // 16),
                 "track": maps_err(got, want),
                 "uint8_bit_identical": all(torch.equal(got[k], got_u8[k]) for k in (R, C))
                 and records(boxes).tobytes() == records(boxes_u8).tobytes(),
                 "track_boxes_maps_equal": all(torch.equal(got[k], maps_b[k]) for k in (R, C))}
            r.update(boxes_vs_oracle(records(boxes), want, size))
            # the head alone on the library's own search features, with and without the dynamic template
            xf64 = xf.double().cpu()
            for name, upd in (("connect", None), ("connect_update", uf[:Bz])):
                bb, cc, cls_dw, x_reg = net.connect_model(xf, zf[:Bz], upd)
                wb, wc, wdw, wreg = fo.box_tower(sd, xf64, zf.double().cpu()[:Bz],
                                                 None if upd is None else uf.double().cpu()[:Bz])
                r[name] = [map_errors(a.cpu().numpy(), b.numpy()) for a, b in
                           ((bb, wb), (cc, wc), (cls_dw, wdw), (x_reg, wreg))]
            if Bz == B:
                fwd = net((zt.cuda(), x.cuda()))
                r["forward"] = maps_err(fwd, fo.forward(sd, zt.double(), x.double()))
            res[tag] = r
    torch.cuda.synchronize()
    return res


def same256():
    """The fixed-size entry points (fear_track, fear_track_u8, fear_forward, fear_head_update, fear_decode,
    fear_decode_smooth) and the sized ones FEARNet calls, at S = 256: the same maps and box bytes in the same number of
    launches, i.e. one code path; and FEAR_EINVAL for sizes outside the contract.  Identity with the kernels as they
    were before the sized entry points is bench.py --dump-outputs' comparison at S = 256, not this one's."""
    net = make_net(3)
    lib = _lib.load()
    zt, _ = fo.shape_crops(128, 128, 3, seed=1)
    x, u = fo.shape_crops(256, 256, 3, seed=2)
    zt, x, u8 = zt.cuda(), x.cuda(), u.permute(0, 2, 3, 1).contiguous().cuda()
    zf = net.get_features(zt)
    h = net._handle

    def outs():
        return (torch.empty(3, 4, 16, 16, device="cuda"), torch.empty(3, 1, 16, 16, device="cuda"),
                torch.empty(3, 48, dtype=torch.uint8, device="cuda"))

    res = {}
    for name, call_old, call_new in (
        ("track", lambda b, c, o: lib.fear_track(h, x.data_ptr(), zf.data_ptr(), 3, 3, b, c, o, stream()),
         lambda b, c, o: lib.fear_track_sized(h, x.data_ptr(), 256, zf.data_ptr(), 3, 3, b, c, o, stream())),
        ("track_u8", lambda b, c, o: lib.fear_track_u8(h, u8.data_ptr(), zf.data_ptr(), 1, 3, b, c, o, stream()),
         lambda b, c, o: lib.fear_track_sized_u8(h, u8.data_ptr(), 256, zf.data_ptr(), 1, 3, b, c, o, stream())),
        ("forward", lambda b, c, o: lib.fear_forward(h, zt.data_ptr(), x.data_ptr(), 3, b, c, o, stream()),
         lambda b, c, o: lib.fear_forward_sized(h, zt.data_ptr(), x.data_ptr(), 256, 3, b, c, o, stream())),
    ):
        a, b = outs(), outs()
        n0 = net.launch_count()
        _lib.check(call_old(*(t.data_ptr() for t in a)), name)
        n1 = net.launch_count()
        _lib.check(call_new(*(t.data_ptr() for t in b)), name + "_sized")
        n2 = net.launch_count()
        res[name] = {"equal": all(torch.equal(p, q) for p, q in zip(a, b)), "launches": [n1 - n0, n2 - n1]}
    xf = net.get_features(x)
    a, b = outs(), outs()
    _lib.check(lib.fear_head_update(h, zf.data_ptr(), 3, zf.data_ptr(), 1, xf.data_ptr(), 3, a[0].data_ptr(),
                                    a[1].data_ptr(), stream()), "fear_head_update")
    _lib.check(lib.fear_head_sized(h, zf.data_ptr(), 3, zf.data_ptr(), 1, xf.data_ptr(), 3, 16, b[0].data_ptr(),
                                   b[1].data_ptr(), stream()), "fear_head_sized")
    res["head"] = {"equal": torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])}
    _lib.check(lib.fear_decode(a[0].data_ptr(), a[1].data_ptr(), 3, 1, a[2].data_ptr(), stream()), "fear_decode")
    _lib.check(lib.fear_decode_sized(a[0].data_ptr(), a[1].data_ptr(), 3, 16, 1, b[2].data_ptr(), stream()),
               "fear_decode_sized")
    res["decode"] = {"equal": torch.equal(a[2], b[2])}
    prev = torch.tensor([[40.0, 60.0]] * 3, dtype=torch.float64, device="cuda")
    win = np.outer(np.hanning(16), np.hanning(16)).reshape(-1)
    params = torch.from_numpy(np.concatenate([[0.062, 0.38, 0.765], win])).cuda()
    _lib.check(lib.fear_decode_smooth(a[0].data_ptr(), a[1].data_ptr(), 3, prev.data_ptr(), params.data_ptr(),
                                      a[2].data_ptr(), stream()), "fear_decode_smooth")
    _lib.check(lib.fear_decode_smooth_sized(a[0].data_ptr(), a[1].data_ptr(), 3, 16, prev.data_ptr(),
                                            params.data_ptr(), b[2].data_ptr(), stream()), "fear_decode_smooth_sized")
    res["decode_smooth"] = {"equal": torch.equal(a[2], b[2])}
    # a size outside the contract is FEAR_EINVAL on every sized entry point
    refused = {}
    for S in (0, 8, 24, 255, 272):
        refused[f"track_{S}"] = lib.fear_track_sized(h, x.data_ptr(), S, zf.data_ptr(), 3, 3, a[0].data_ptr(),
                                                     a[1].data_ptr(), None, stream())
        refused[f"track_u8_{S}"] = lib.fear_track_sized_u8(h, u8.data_ptr(), S, zf.data_ptr(), 3, 3, a[0].data_ptr(),
                                                           a[1].data_ptr(), None, stream())
        refused[f"forward_{S}"] = lib.fear_forward_sized(h, zt.data_ptr(), x.data_ptr(), S, 3, a[0].data_ptr(),
                                                         a[1].data_ptr(), None, stream())
    for s in (0, 17):
        refused[f"head_{s}"] = lib.fear_head_sized(h, zf.data_ptr(), 3, None, 0, xf.data_ptr(), 3, s, a[0].data_ptr(),
                                                   a[1].data_ptr(), stream())
    res["refused"] = refused
    torch.cuda.synchronize()
    return res


def chunk():
    """B = 5 at S = 192 through the C entry points on a 2-frame workspace (chunks 2, 2, 1), then the same calls after
    fear_reserve(5) (one pass): every map and box record must be the same bit for bit."""
    B, size, side = 5, 192, 12
    zt, _ = fo.shape_crops(128, 128, B, seed=3)
    x, u = fo.shape_crops(size, size, B, seed=4)
    zt, x, u8 = zt.cuda(), x.cuda(), u.permute(0, 2, 3, 1).contiguous().cuda()
    net = make_net(2)
    h, lib = net._ensure_handle(torch.device("cuda", torch.cuda.current_device()))  # the library holds 2 frames

    def outputs():
        zf = torch.empty(B, 256, 8, 8, device="cuda")
        _lib.check(lib.fear_get_features(h, zt.data_ptr(), B, 128, 128, zf.data_ptr(), stream()), "fear_get_features")
        xf = torch.empty(B, 256, side, side, device="cuda")
        _lib.check(lib.fear_get_features(h, x.data_ptr(), B, size, size, xf.data_ptr(), stream()), "fear_get_features")
        zu = zf.flip(0).contiguous()  # dynamic templates of the cls branch
        out = [zf, xf, zu]

        def maps(boxes=True):
            m = (torch.empty(B, 4, side, side, device="cuda"), torch.empty(B, 1, side, side, device="cuda"))
            m += (torch.empty(B, 48, dtype=torch.uint8, device="cuda"),) if boxes else ()
            out.extend(m)
            return [t.data_ptr() for t in m]

        for Bz in (1, B):
            _lib.check(lib.fear_track_sized(h, x.data_ptr(), size, zf.data_ptr(), Bz, B, *maps(), stream()), "track")
            _lib.check(lib.fear_track_sized_u8(h, u8.data_ptr(), size, zf.data_ptr(), Bz, B, *maps(), stream()), "u8")
            b, c = maps(boxes=False)
            _lib.check(lib.fear_head_sized(h, zf.data_ptr(), Bz, zu.data_ptr(), Bz, xf.data_ptr(), B, side, b, c,
                                           stream()), "head")
        _lib.check(lib.fear_forward_sized(h, zt.data_ptr(), x.data_ptr(), size, B, *maps(), stream()), "forward")
        torch.cuda.synchronize()
        return [t.clone() for t in out]

    chunked = outputs()
    n0 = net.launch_count()
    outputs()
    launches_chunked = net.launch_count() - n0
    net.reserve(B)  # whole batch in one pass
    whole = outputs()
    n0 = net.launch_count()
    outputs()
    launches_whole = net.launch_count() - n0
    return {"chunk_invariant": all(torch.equal(a, b) for a, b in zip(chunked, whole)), "n": len(whole),
            "chunk_loop_ran": launches_chunked > launches_whole}


def decode(side):
    """Decode on s x s maps with ties, NaN and +-inf cells against the host: fo.decode (FEARBoxCoder.decode of the
    reference) for fear_decode_sized, FEARTracker._smooth_postprocess for fear_decode_smooth_sized."""
    size, P = 16 * side, side * side
    g = torch.Generator().manual_seed(side)
    B = 12
    reg = torch.rand(B, 4, side, side, generator=g) * 40 + 1
    cls = torch.randn(B, 1, side, side, generator=g)
    flat = cls.view(B, -1)
    flat[1] = 0.5  # all tied: the first cell wins
    if P > 1:
        flat[2, P // 2:] = 3.0  # a tie between later cells
        flat[3, -1] = float("nan")  # NaN is greater than every number
        flat[4, P // 3] = float("inf")
        flat[5, :] = float("-inf")  # every cell -inf: cell 0
        flat[6, 1::2] = float("nan")  # the first NaN wins
        flat[7, 0] = float("-inf")
    cfg = cfg_for(size, smooth=True)
    coder = fb.FEARBoxCoder(cfg)
    host = fb.FEARTracker(None, cuda_id=0, **cfg)
    res = {"plain": [], "smooth": []}
    regc, clsc = reg.cuda().contiguous(), cls.cuda().contiguous()
    for use_sigmoid in (1, 0):
        boxes = torch.full((B, 48), 0xA5, dtype=torch.uint8, device="cuda")
        _lib.check(_lib.load().fear_decode_sized(regc.data_ptr(), clsc.data_ptr(), B, side, use_sigmoid, boxes.data_ptr(),
                                                 stream()), "fear_decode_sized")
        rec = records(boxes)
        # the kernel's float32 sigmoid equals torch's on the device bit for bit (DESIGN 4.7): the host decodes those scores
        scores = cls.cuda().sigmoid().cpu() if use_sigmoid else cls
        for i in range(B):
            bbox, coords = fo.decode(reg[i:i + 1], scores[i:i + 1], use_sigmoid=False, config=cfg)
            r, c = coords[0]
            want = bbox.numpy()[0]
            got = np.array([rec["x"][i], rec["y"][i], rec["w"][i], rec["h"][i]])
            s_want = np.float32(scores.view(B, -1)[i, r * side + c])
            res["plain"].append(bool((rec["row"][i], rec["col"][i]) == (r, c) and rec["flat"][i] == r * side + c
                                     and np.array_equal(got, want)
                                     and np.float32(rec["score"][i]).tobytes() == s_want.tobytes()))
        if use_sigmoid:
            res["coder_records"] = coder.decode_records(reg.cuda(), cls.cuda()).tobytes() == rec.tobytes()
    window = np.asarray(host.window, dtype=np.float64).reshape(P)
    params = torch.from_numpy(np.concatenate([[cfg["penalty_k"], cfg["window_influence"], cfg["lr"]], window])).cuda()
    prev = np.stack([np.linspace(20, 90, B), np.linspace(70, 15, B)], 1)
    boxes = torch.full((B, 48), 0xA5, dtype=torch.uint8, device="cuda")
    prevc = torch.from_numpy(prev).cuda()
    _lib.check(_lib.load().fear_decode_smooth_sized(regc.data_ptr(), clsc.data_ptr(), B, side, prevc.data_ptr(),
                                                    params.data_ptr(), boxes.data_ptr(), stream()),
               "fear_decode_smooth_sized")
    rec = records(boxes)
    for i in range(B):
        host.tracking_state.prev_size = prev[i]
        with np.errstate(all="ignore"):
            box, score = host._postprocess({R: regc[i:i + 1], C: clsc[i:i + 1]})
        got = np.array([rec["x"][i], rec["y"][i], rec["w"][i], rec["h"][i]])
        res["smooth"].append(bool(np.allclose(got, box, rtol=1e-12, atol=1e-12, equal_nan=True)
                                  and np.float32(rec["score"][i]).tobytes() == np.float32(score).tobytes()))
    torch.cuda.synchronize()
    return res


def poison(size):
    """Every sized entry point at S on a poisoned workspace with guarded inputs and outputs (tests/poison_check.py's
    Checker): three fills give the same outputs, no guard band is written, no input changes."""
    from tests.poison_check import Checker, Guarded

    side, B = size // 16, 3
    net = make_net(B)
    net._ensure_handle(torch.device("cuda", torch.cuda.current_device()))
    lib, h = _lib.load(), net._handle
    zt, _ = fo.shape_crops(128, 128, B, seed=9)
    x, u = fo.shape_crops(size, size, B, seed=10)
    zf = net.get_features(zt.cuda()).cpu()
    xf = net.get_features(x.cuda()).cpu()
    P = side * side
    gx = Guarded.of(x, 3 * size * size)
    gu = Guarded.of(u.permute(0, 2, 3, 1).contiguous(), 3 * size * size)
    gt = Guarded.of(zt, 3 * 128 * 128)
    gz = Guarded.of(zf, 256 * 64)
    gxf = Guarded.of(xf, 256 * P)
    bb, cc = Guarded.out((B, 4, side, side), torch.float32, 4 * P), Guarded.out((B, 1, side, side), torch.float32, P)
    bx = Guarded.out((B, 48), torch.uint8, 48)
    prev = Guarded.of(torch.tensor([[30.0, 50.0]] * B, dtype=torch.float64), 2)
    win = np.outer(np.hanning(side), np.hanning(side)).reshape(-1)
    params = Guarded.of(torch.from_numpy(np.concatenate([[0.062, 0.38, 0.765], win])), 3 + P)
    chk = Checker()
    outs = (bb, cc, bx)
    for Bz in (1, B):
        chk.run(f"track_sized Bz={Bz}", lambda: _lib.check(lib.fear_track_sized(
            h, gx.ptr(), size, gz.ptr(), Bz, B, bb.ptr(), cc.ptr(), bx.ptr(), stream()), "t"), [gx, gz], outs, [net])
        chk.run(f"track_sized_u8 Bz={Bz}", lambda: _lib.check(lib.fear_track_sized_u8(
            h, gu.ptr(), size, gz.ptr(), Bz, B, bb.ptr(), cc.ptr(), bx.ptr(), stream()), "t"), [gu, gz], outs, [net])
        for upd in (0, 1):
            chk.run(f"head_sized Bz={Bz} update={upd}", lambda: _lib.check(lib.fear_head_sized(
                h, gz.ptr(), Bz, gz.ptr() if upd else None, 1 if upd else 0, gxf.ptr(), B, side, bb.ptr(), cc.ptr(),
                stream()), "h"), [gz, gxf], (bb, cc), [net])
    chk.run("forward_sized", lambda: _lib.check(lib.fear_forward_sized(
        h, gt.ptr(), gx.ptr(), size, B, bb.ptr(), cc.ptr(), bx.ptr(), stream()), "f"), [gt, gx], outs, [net])
    maps = [Guarded.of(t, 1) for t in (bb.t.cpu(), cc.t.cpu())]
    for sig in (0, 1):
        chk.run(f"decode_sized sigmoid={sig}", lambda: _lib.check(lib.fear_decode_sized(
            maps[0].ptr(), maps[1].ptr(), B, side, sig, bx.ptr(), stream()), "d"), maps, [bx])
    chk.run("decode_smooth_sized", lambda: _lib.check(lib.fear_decode_smooth_sized(
        maps[0].ptr(), maps[1].ptr(), B, side, prev.ptr(), params.ptr(), bx.ptr(), stream()), "s"),
        maps + [prev, params], [bx])
    return chk.report()


def nv12_of(rgb):
    """(NV12 surface (3H/2, W) uint8, the RGB frame cv2 converts it to)."""
    import cv2

    i420 = cv2.cvtColor(rgb, cv2.COLOR_RGB2YUV_I420)
    h, w = rgb.shape[:2]
    u, v = i420[h:h + h // 4].reshape(h // 2, w // 2), i420[h + h // 4:].reshape(h // 2, w // 2)
    nv12 = np.concatenate([i420[:h], np.stack([u, v], 2).reshape(h // 2, w)], 0)
    return nv12, cv2.cvtColor(nv12, cv2.COLOR_YUV2RGB_NV12)


def iou(a, b):
    x1, y1 = np.maximum(a[:, 0], b[:, 0]), np.maximum(a[:, 1], b[:, 1])
    x2, y2 = np.minimum(a[:, 0] + a[:, 2], b[:, 0] + b[:, 2]), np.minimum(a[:, 1] + a[:, 3], b[:, 1] + b[:, 3])
    inter = np.clip(x2 - x1, 0, None) * np.clip(y2 - y1, 0, None)
    return inter / (a[:, 2] * a[:, 3] + b[:, 2] * b[:, 3] - inter)


def run_tracker(trk, frames, init, feed=lambda f: f):
    trk.initialize(feed(frames[0]), init)
    return np.array([list(map(int, trk.update(feed(f))["bbox"])) for f in frames[1:]], dtype=np.int64)


def trackers(size):
    """FEARTracker vs the oracle tracker, gpu_crop vs host crop, CUDA-tensor and NV12 frames vs numpy frames, smooth off
    and on."""
    clip = fo.read_video_rgb(os.path.join(GOLDEN, "test.mp4"))[:121]  # the fp64 oracle tracker costs ~1 s a frame
    init = np.load(os.path.join(GOLDEN, "video_teacher.npz"))["init_bbox"]
    net = make_net(8)
    sd = sd64()
    nv12 = [nv12_of(f) for f in clip[:41]]
    res = {}
    for smooth in (False, True):
        cfg = cfg_for(size, smooth=smooth)
        oracle = fo.OracleTracker(sd, cfg)
        oracle.initialize(clip[0], init)
        want = np.array([list(map(int, oracle.update(f)["bbox"])) for f in clip[1:]], dtype=np.int64)
        host = run_tracker(fb.FEARTracker(net, cuda_id=0, **cfg), clip, init)
        same = (host == want).all(1)
        ious = iou(host.astype(np.float64), want.astype(np.float64))
        gpu_crop = run_tracker(fb.FEARTracker(net, cuda_id=0, **dict(cfg, gpu_crop=True)), clip, init)
        cuda = run_tracker(fb.FEARTracker(net, cuda_id=0, **cfg), clip, init, lambda f: torch.from_numpy(f).cuda())
        yuv = run_tracker(fb.FEARTracker(net, cuda_id=0, **cfg), [n for n, _ in nv12], init,
                          lambda f: fb.YUV420Frame.nv12(torch.from_numpy(f).cuda()))
        yuv_rgb = run_tracker(fb.FEARTracker(net, cuda_id=0, **cfg), [r for _, r in nv12], init)
        res[f"smooth={smooth}"] = {
            "frames": int(len(host)), "identical": int(same.sum()), "oracle_first30": bool(same[:30].all()),
            "min_iou": float(ious.min()), "mean_iou": float(ious.mean()),
            "gpu_crop_equal": bool(np.array_equal(gpu_crop, host)), "cuda_equal": bool(np.array_equal(cuda, host)),
            "nv12_equal": bool(np.array_equal(yuv, yuv_rgb))}
    torch.cuda.synchronize()
    return res


def multi_case(net, size, frames):
    """Targets in two streams (the clip and its mirror image), the step replayed as a CUDA graph, against one
    FEARTracker(gpu_crop=True) per target."""
    cfg = cfg_for(size)
    rects = [[200, 120, 60, 80], [420, 200, 90, 70], [100, 300, 50, 50]]
    streams = [0, 1, 0]
    clips = [frames[:21], frames[:21, :, ::-1].copy()]
    multi = fb.FEARMultiTracker(net, cuda_id=0, max_targets=8, **cfg)
    multi.add([c[0] for c in clips], rects, streams)
    singles, records_of = [], []
    for r, s in zip(rects, streams):
        t = fb.FEARTracker(net, cuda_id=0, **dict(cfg, gpu_crop=True))
        t.initialize(clips[s][0], r)
        singles.append(t)
        # the score of an update is in the box record of its step; update() returns only the box
        last = {}
        step = t._track_record_gpu_crop

        def capture(*a, step=step, last=last):
            last["rec"] = step(*a)
            return last["rec"]
        t._track_record_gpu_crop = capture
        records_of.append(last)
    boxes_equal = scores_equal = True
    for i in range(1, 21):
        out = multi.update([c[i] for c in clips])
        for k, (t, s) in enumerate(zip(singles, streams)):
            want = t.update(clips[s][i])["bbox"]
            boxes_equal &= bool(np.array_equal(np.asarray(out["bbox"][k], dtype=np.int64),
                                               np.asarray(want, dtype=np.int64)))
            got, rec = np.float32(out["score"][k]), np.float32(records_of[k]["rec"]["score"])
            scores_equal &= got.tobytes() == rec.tobytes()
    return {"boxes_equal": boxes_equal, "scores_equal": scores_equal, "graph": multi._graph is not None}


def multi(size):
    clip = fo.read_video_rgb(os.path.join(GOLDEN, "test.mp4"))
    return multi_case(make_net(8), size, clip)


def main():
    mode = sys.argv[1]
    args = list(map(int, sys.argv[2:]))
    res = {"parity": parity, "same256": same256, "chunk": chunk, "decode": decode, "poison": poison,
           "trackers": trackers, "multi": multi}[mode](*args)
    print("SEARCH_SIZE_CHECK " + json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
