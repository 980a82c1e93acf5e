"""Stand-alone checker of the persistent 1x1-conv GEMM (pw_tc_kernel) at given batches; run in its own process (a
device-side trap would poison the CUDA context of the main pytest process).  Prints one JSON line.

    python tests/pw_schedule_check.py B [B ...]

Inputs: the 7 seeded crops of tests/schedule_check.py; frame i of a batch is input i mod 7.  Each input is first run at
B = 1: the backbone (fear_debug_backbone_prefix, all blocks) against the fp64 oracle at the block bar, fear_track_u8's
maps against the oracle at the track bars, and the head intermediates of that call (fear_debug_head_tensor) kept.
Then, at every batch, the same calls run on a workspace poisoned with POISON_A (outputs pre-filled with it), and every
frame of the backbone output, of the head intermediates and of the maps and FearBox records must equal its B = 1 result
bit for bit.
"""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import fear_oracle as fo  # noqa: E402
from tests import schedule_check as sc  # noqa: E402
from tests.helpers import POISON_A, map_errors, poison_workspace  # noqa: E402

HEAD_TENSORS = ["search_features", "cat_cls", "cat_reg", "cls_dw", "reg_dw", "x_reg", "cls_tower"]
LAST_BLOCK = len(sc.BLOCK_NAMES) - 1


def backbone(net, x):
    poison_workspace(net, POISON_A)
    return net.backbone_prefix(x, LAST_BLOCK)


def track(net, u, z):
    out = sc.track_u8(net, u, z, sc.POISONS["A"])
    return out, [net.head_tensor(name, u.shape[0]) for name in HEAD_TENSORS]


def main():
    batches = [int(b) for b in sys.argv[1:]]
    rep = sc.Report()
    net = sc.make_net(max(batches))
    sd = sc.sd64()
    x1, u1 = sc.inputs(256, 256, sc.SEARCH_SEEDS)
    t1, _ = sc.inputs(128, 128, sc.TEMPLATE_SEEDS)
    u1c, x1c = u1.cuda(), x1.cuda()

    # B = 1 references
    z1, expected = sc.track_refs(rep, net, sd, x1, u1, t1, [("default", {})])
    bb1, heads1 = [], []
    for i in range(sc.N_INPUTS):
        col = {}
        with torch.no_grad():
            fo.get_features(sd, x1[i:i + 1].double(), col)
        b = backbone(net, x1c[i:i + 1])
        rep.error("block_inf", map_errors(b.cpu().numpy(), col[sc.BLOCK_NAMES[-1]].numpy())[1], sc.BLOCK_TOL,
                  f"input {i} B=1 backbone")
        bb1.append(b)
        heads1.append(track(net, u1c[i:i + 1], z1[i:i + 1])[1])
    bb1 = torch.cat(bb1)
    heads1 = [torch.cat([h[k] for h in heads1]) for k in range(len(HEAD_TENSORS))]
    res = {"S": sc.num_sms(), "batches": batches, "oracle_worst": dict(rep.worst)}

    for B in batches:
        idx = [i % sc.N_INPUTS for i in range(B)]
        got_track, got_heads = track(net, u1c[idx], z1[idx])
        got_bb = backbone(net, x1c[idx])
        torch.cuda.synchronize()
        rep.runs += 1
        for what, got, want in (("track", got_track, [e[idx] for e in expected["default"]]),
                                ("head_tensors", got_heads, [h[idx] for h in heads1]),
                                ("backbone", [got_bb], [bb1[idx]])):
            bad = sc.bad_frames(got, want)
            if bad:
                rep.fail({"B": B, "what": what, "bad_frames": bad[:16], "n_bad_frames": len(bad)})
    res.update(rep.dump())
    print("PW_SCHEDULE_CHECK " + json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
