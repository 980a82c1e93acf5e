"""Generate ``tests/golden/*`` from the REAL reference source and pin the restatement to it.

Run in the build container only (needs ``/root/reference``):  ``python -m oracle.make_golden``

What it does
1. imports the reference's unmodified ``FEARNet`` / ``FEARTracker`` through ``ref_shims`` and
   strict-loads the shipped checkpoint;
2. asserts ``oracle.fear_oracle`` reproduces the reference bit-for-bit in fp32 AND fp64
   (maps, features, decode, full video trajectory);
3. writes the fixtures the tests on the GPU box compare against (that box has no reference):
     fear_xs_hotpath_state.npz   hot-path subset of the checkpoint (raw, unfolded, fp32)
     maps_seed0.npz              C1: torch.manual_seed(0) randn pair -> maps (fp32 ref + fp64 ref)
     synthetic_b4.npz            C2-style uint8-derived crops (seed 20260924), 4 frames, fp64 maps
     video_teacher.npz           C3: reference trajectory (660 int boxes) + 9 teacher-forced frames
     block_stats.json            per-block activation statistics of the reference (fp32, seed0)
     test.mp4                    the demo clip (data asset, MIT) so config 3 can run on the GPU box
"""
import hashlib
import json
import os
import shutil

import numpy as np
import torch

from oracle import fear_oracle as fo
from oracle import ref_shims

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
R, C = fo.TARGET_REGRESSION_LABEL_KEY, fo.TARGET_CLASSIFICATION_KEY
TEACHER_FRAMES = [1, 2, 3, 11, 51, 120, 200, 400, 660]


def _eq(a: torch.Tensor, b: torch.Tensor, what: str) -> None:
    assert a.shape == b.shape and a.dtype == b.dtype, (what, a.shape, b.shape, a.dtype, b.dtype)
    assert torch.equal(a, b), f"restatement differs from reference: {what} max|d|={(a - b).abs().max().item():.3e}"


def main() -> None:
    os.makedirs(OUT, exist_ok=True)
    torch.set_num_threads(os.cpu_count())
    net = ref_shims.build_reference_net()
    sd32 = fo.load_lightning_state(ref_shims.REF_CKPT)
    assert len(sd32) == 520
    sd64 = fo.to_dtype(sd32, torch.float64)

    # ---- fixture 0: hot-path weights ----------------------------------------------------
    keys = fo.hot_path_keys(sd32)
    np.savez_compressed(os.path.join(OUT, "fear_xs_hotpath_state.npz"), **{k: sd32[k].numpy() for k in keys})
    all_keys = {k: [list(v.shape), str(v.dtype).replace("torch.", "")] for k, v in sd32.items()}
    with open(os.path.join(OUT, "state_dict_keys.json"), "w") as f:
        json.dump(all_keys, f, indent=0, sort_keys=True)
    # the reference's own outputs and checkpoint bytes, for tests/test_oracle_cpu.py::test_restatement_equals_reference_source
    h = hashlib.sha256()
    for k in sorted(keys):
        h.update(k.encode())
        h.update(sd32[k].contiguous().numpy().tobytes())
    with open(os.path.join(OUT, "reference_state_sha256.json"), "w") as f:
        json.dump({"tensors": len(keys), "sha256": h.hexdigest()}, f)
    zt7, xt7, _, _ = fo.synthetic_crops(2, seed=7)
    with torch.no_grad():
        ref7 = net((zt7, xt7))
    np.savez_compressed(os.path.join(OUT, "reference_forward_seed7.npz"), reg=ref7[R].numpy(), cls=ref7[C].numpy())

    # ---- fixture 1 (C1): seed-0 randn pair ----------------------------------------------
    torch.manual_seed(0)
    z = torch.randn(1, 3, 128, 128)
    x = torch.randn(1, 3, 256, 256)
    with torch.no_grad():
        ref32 = net((z, x))
        ref_zf = net.get_features(z)
        ref_trk = net.track(x, ref_zf)
    _eq(ref32[R], ref_trk[R], "forward vs track (reg)")
    mine = fo.forward(sd32, z, x)
    _eq(ref32[R], mine[R], "seed0 reg fp32")
    _eq(ref32[C], mine[C], "seed0 cls fp32")
    with torch.no_grad():
        _eq(ref_zf, fo.get_features(sd32, z), "seed0 template features fp32")

    # per-block statistics of the REFERENCE (hooks on its own modules)
    stats = {}
    hooks = []
    stages = net.encoder.model.backbone.stages
    for name, mod in list(stages.named_children())[: fo.NUM_HOT_BLOCKS]:
        hooks.append(mod.register_forward_hook(
            lambda m, i, o, name=name: stats.__setitem__(name, [float(o.mean()), float(o.std()), float(o.abs().max())])))
    hooks.append(net.neck.register_forward_hook(
        lambda m, i, o: stats.__setitem__("neck", [float(o.mean()), float(o.std()), float(o.abs().max())])))
    with torch.no_grad():
        net.get_features(x)
    for h in hooks:
        h.remove()
    col = {}
    with torch.no_grad():
        fo.get_features(sd32, x, col)
    for k, v in stats.items():
        mine_stat = [float(col[k].mean()), float(col[k].std()), float(col[k].abs().max())]
        assert mine_stat == v, (k, mine_stat, v)
    with open(os.path.join(OUT, "block_stats.json"), "w") as f:
        json.dump(stats, f, indent=1)

    net64 = ref_shims.build_reference_net().double()
    with torch.no_grad():
        ref64 = net64((z.double(), x.double()))
        ref_zf64 = net64.get_features(z.double())
    mine64 = fo.forward(sd64, z.double(), x.double())
    _eq(ref64[R], mine64[R], "seed0 reg fp64")
    _eq(ref64[C], mine64[C], "seed0 cls fp64")
    bbox, coords = fo.decode(ref32[R], ref32[C])
    ref_coder_box = None
    ref_shims.install()
    from model_training.dataset.box_coder import FEARBoxCoder  # reference source

    coder = FEARBoxCoder(ref_shims.REF_TRACKER_KWARGS)
    dec = coder.decode(regression_map=ref32[R], classification_map=ref32[C], use_sigmoid=True)
    _eq(dec.bbox, bbox, "decode bbox")
    assert dec.pred_coords == coords, (dec.pred_coords, coords)
    np.savez_compressed(
        os.path.join(OUT, "maps_seed0.npz"),
        reg32=ref32[R].numpy(), cls32=ref32[C].numpy(), reg64=ref64[R].numpy(), cls64=ref64[C].numpy(),
        zf32=ref_zf.numpy(), zf64=ref_zf64.numpy(), bbox=dec.bbox.numpy(), coords=np.array(coords),
    )
    print("C1 seed0: argmax", coords, "bbox", dec.bbox.numpy())

    # ---- fixture 2 (C2-style): synthetic uint8-derived crops, 4 frames, fp64 maps ---------
    zt, xt, zu, xu = fo.synthetic_crops(4)
    with torch.no_grad():
        r64 = net64((zt.double(), xt.double()))
        zf64 = net64.get_features(zt.double())
        r64_bz1 = net64.track(xt.double(), zf64[:1])  # template batch-1 broadcast
    m64 = fo.forward(sd64, zt.double(), xt.double())
    _eq(r64[R], m64[R], "synthetic reg fp64")
    _eq(r64[C], m64[C], "synthetic cls fp64")
    _eq(r64_bz1[R], fo.track(sd64, xt.double(), zf64[:1])[R], "synthetic Bz=1 reg fp64")
    with torch.no_grad():
        r32 = net((zt, xt))
    m32 = fo.forward(sd32, zt, xt)
    _eq(r32[R], m32[R], "synthetic reg fp32")
    dec = coder.decode(regression_map=r64[R], classification_map=r64[C], use_sigmoid=True)
    cls_flat = r64[C].flatten(1)
    top2 = cls_flat.topk(2, dim=1).values
    np.savez_compressed(
        os.path.join(OUT, "synthetic_b4.npz"),
        reg64=r64[R].numpy(), cls64=r64[C].numpy(), zf64=zf64.numpy(),
        reg64_bz1=r64_bz1[R].numpy(), cls64_bz1=r64_bz1[C].numpy(),
        bbox=dec.bbox.numpy(), coords=np.array(dec.pred_coords), margin=(top2[:, 0] - top2[:, 1]).numpy(),
        seed=np.array(20260924),
    )
    print("C2 synthetic: argmax", cls_flat.argmax(1).tolist(), "reg mean", float(r64[R].mean()))

    # ---- fixture 3 (C3): video trajectory + teacher-forced frames --------------------------
    frames = fo.read_video_rgb(ref_shims.REF_VIDEO)
    ref_trk = ref_shims.build_reference_tracker(net)
    mine_trk = fo.OracleTracker(sd32)
    init = np.array(ref_shims.REF_INIT_BBOX)
    ref_trk.initialize(frames[0], init)
    mine_trk.initialize(frames[0], init)
    _eq(ref_trk._template_features, mine_trk.template_features, "template features (video)")
    traj = []
    teacher = {}
    for i in range(1, len(frames)):
        rb = ref_trk.update(frames[i])["bbox"]
        mb = mine_trk.update(frames[i])["bbox"]
        assert list(rb) == list(mb), (i, rb, mb)
        traj.append(list(map(int, rb)))
        if i in TEACHER_FRAMES:
            crop = mine_trk.last_search_crop
            o64 = fo.track(sd64, fo.preprocess_image(crop).double(), ref_trk._template_features.double())
            teacher[i] = (crop.copy(), o64[R].numpy(), o64[C].numpy(), np.array(traj[-1]))
    traj = np.array(traj, dtype=np.int64)
    sha = hashlib.sha1(traj.tobytes()).hexdigest()
    print("C3 video:", len(frames), "frames; sha1(traj) =", sha, "; boxes:",
          {i: traj[i - 1].tolist() for i in TEACHER_FRAMES})
    np.savez_compressed(
        os.path.join(OUT, "video_teacher.npz"),
        trajectory=traj, sha1=np.array(sha), init_bbox=init, template_crop=mine_trk.template_crop,
        template_features=ref_trk._template_features.detach().numpy(), frames=np.array(TEACHER_FRAMES),
        search_crops=np.stack([teacher[i][0] for i in TEACHER_FRAMES]),
        reg64=np.concatenate([teacher[i][1] for i in TEACHER_FRAMES]),
        cls64=np.concatenate([teacher[i][2] for i in TEACHER_FRAMES]),
        boxes=np.stack([teacher[i][3] for i in TEACHER_FRAMES]),
    )
    shutil.copyfile(ref_shims.REF_VIDEO, os.path.join(OUT, "test.mp4"))
    print("golden fixtures written to", OUT)


if __name__ == "__main__":
    main()
