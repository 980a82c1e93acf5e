"""Per-launch time of one flagship step (net.track_boxes, 256 x 256 search crops) against the H100's floors.

    python tools/profile_gemm.py [--batch 256] [--steps 5] [--warmup 3] [--out DIR]

Runs warmed-up track_boxes steps under torch.profiler (CUDA activities) and writes DIR/profile_gemm.md and
DIR/profile_gemm.json: one row per kernel launch in issue order, named after the layer it belongs to (the launch
list of tests/schedule_plan.py, which mirrors run_backbone / run_blocks / run_head of fear_context.cu), with its
CUDA time (median over the profiled steps), the FLOPs and bytes the layer needs (computed from its shapes here),
and its floor: the larger of FLOPs at the data-sheet rate (dense TF32 for the 3xTF32 wgmma GEMMs, FP32 for
CUDA-core work) and bytes at the data-sheet HBM bandwidth. The GPU's name, power limit and SM clocks are read in
the same run. Run it in a process of its own: tracing slows the host.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import schedule_plan as sp  # noqa: E402

TF32_FLOPS, FP32_FLOPS, HBM_BPS = 495e12, 67e12, 3.35e12  # H100 SXM data sheet, dense, 700 W
F = 4  # bytes per fp32


def _block_maps():
    """Block name -> (spec, input map side) for a 256 x 256 search crop (the stem halves it to 128)."""
    out, h = {}, 128
    for name, cin, cout, k, stride, e in sp.BLOCKS:
        out[name] = ((cin, cout, k, stride, e), h)
        h //= stride
    return out


def layer_cost(name: str, B: int):
    """(kind, GEMM M x K x N or None, tensor-core FLOPs, CUDA-core FLOPs, HBM bytes) of one launch of the step."""
    blocks = _block_maps()
    gemm = lambda M, K, N: 2 * M * K * N * 3  # noqa: E731  (3xTF32: three tf32 products per multiply-add)
    dwf = lambda M, k, C: 2 * M * k * k * C  # noqa: E731
    base = name.split(".")[0].split(" ")[0]
    if name == "stage template":
        n = B * sp.TMPL_PIX * sp.FEAT_C
        return "layout", None, 0, 0, 2 * n * F
    if name == "stem+xif1_0":
        M = B * 128 * 128
        return "stem", None, 0, M * (2 * 27 * 16 + dwf(1, 3, 16) + 2 * 16 * 16), B * 256 * 256 * 3 * F + M * 16 * F
    if base in blocks:
        (cin, cout, k, stride, e), h = blocks[base]
        mid, ho = cin * e, h // stride
        Mi, Mo = B * h * h, B * ho * ho
        res = stride == 1 and cin == cout
        if name.endswith(" fused"):  # xif2_0 in one kernel
            return "irf_s2", (Mo, mid, cout), gemm(Mi, cin, mid) + gemm(Mo, mid, cout), dwf(Mo, k, mid), \
                (Mi * cin + Mo * cout) * F
        if name.endswith(" dw+pw"):  # expand-1 blocks on CUDA cores
            return "dw3_pw24", None, 0, dwf(Mo, k, cin) + 2 * Mo * cin * cout, (Mi * cin + Mo * cout) * F
        if name.endswith(".pw"):
            return "pw", (Mi, cin, mid), gemm(Mi, cin, mid), 0, (Mi * cin + Mi * mid) * F
        if name.endswith(".dw"):
            return "dw", None, 0, dwf(Mo, k, mid), (Mi * mid + Mo * mid) * F
        if name.endswith(".pwl"):
            return "pw", (Mo, mid, cout), gemm(Mo, mid, cout), 0, (Mo * mid + Mo * cout * (2 if res else 1)) * F
        if name.endswith(".dw+pwl"):
            return "pw_dw", (Mo, mid, cout), gemm(Mo, mid, cout), dwf(Mo, k, mid), \
                (Mi * mid + Mo * cout * (2 if res else 1)) * F
    M = B * sp.SCORE * sp.SCORE
    if name == "neck":
        return "pw", (M, sp.BACKBONE_C, sp.FEAT_C), gemm(M, sp.BACKBONE_C, sp.FEAT_C), 0, \
            M * (sp.BACKBONE_C + sp.FEAT_C) * F
    if name.endswith(" dw+pw"):  # head SepConv: depthwise 3x3 + 1x1 -> 256
        cin = sp.CAT_C if "_dw " in name else sp.FEAT_C
        return "pw_dw", (M, cin, sp.FEAT_C), gemm(M, cin, sp.FEAT_C), dwf(M, 3, cin), M * (cin + sp.FEAT_C) * F
    if name == "corr":  # both branches in one launch
        Mc = 2 * B * sp.SCORE * sp.SCORE
        return "corr", (Mc, sp.FEAT_C, sp.TMPL_PIX), gemm(Mc, sp.FEAT_C, sp.TMPL_PIX), 0, \
            2 * B * (sp.TMPL_PIX * sp.FEAT_C + sp.SCORE ** 2 * (sp.FEAT_C + sp.TMPL_PIX)) * F
    if name.endswith("_pred.dw"):
        return "dw", None, 0, dwf(M, 3, sp.FEAT_C), 2 * M * sp.FEAT_C * F
    if name.endswith("_pred.pw"):
        n = 4 if name.startswith("bbox") else 1
        return "pred", None, 0, 2 * M * sp.FEAT_C * n, M * (sp.FEAT_C + n) * F
    if name == "decode":
        return "decode", None, 0, 0, 5 * M * F + B * 48
    return "other", None, 0, 0, 0


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired) as e:
        return {"error": str(e)}
    return dict(zip(q.split(","), [v.strip() for v in out.split(",")]))


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=5, help="profiled steps; each launch's time is the median")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "profile_gemm"))
    ap.add_argument("--label", default="", help="free text stored with the table (e.g. the build it measures)")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    import feartracker_b200 as fb
    from bench import load_state, synthetic_batch

    if not torch.cuda.is_available():
        sys.exit("profile_gemm needs a CUDA device")
    dev = torch.device("cuda:0")
    net = fb.FEARNet(**fb.FEAR_XS_MODEL_KWARGS)
    net.load_state_dict(load_state(), strict=True)
    net = net.to(dev).eval()
    zt, xt = synthetic_batch(args.batch, 0)
    z_dev, x_dev = net.get_features(zt.to(dev)), xt.to(dev)
    with torch.no_grad():
        for _ in range(args.warmup):
            net.track_boxes(x_dev, z_dev)
        torch.cuda.synchronize()
        n_launch = net.launch_count()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.steps):
                net.track_boxes(x_dev, z_dev)
            torch.cuda.synchronize()
    info = gpu_info()

    kern = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
            and not e.name.startswith(("Memcpy", "Memset", "[memory]"))]
    kern.sort(key=lambda e: e.time_range.start)
    names = [ln.name for ln in sp.launches("track_u8", Bz=args.batch)]
    if len(kern) != args.steps * len(names):
        sys.exit(f"{len(kern)} kernels in {args.steps} steps, expected {len(names)} per step "
                 f"(fear_launch_count {n_launch}): the launch model does not match this build")
    per = len(names)
    rows = []
    for i, name in enumerate(names):
        us = statistics.median(kern[s * per + i].time_range.elapsed_us() for s in range(args.steps))
        kind, mkn, tc_fl, cc_fl, nbytes = layer_cost(name, args.batch)
        t_flop = (tc_fl / TF32_FLOPS + cc_fl / FP32_FLOPS) * 1e6
        t_hbm = nbytes / HBM_BPS * 1e6
        floor = max(t_flop, t_hbm)
        rows.append({"launch": i, "layer": name, "kernel": kern[i].name.split("(")[0][:60], "kind": kind,
                     "mkn": mkn, "us": us, "flops": tc_fl + cc_fl, "bytes": nbytes, "flop_floor_us": t_flop,
                     "hbm_floor_us": t_hbm, "bound": "compute" if t_flop >= t_hbm else "hbm",
                     "of_floor": floor / us if us > 0 else 0.0})

    os.makedirs(args.out, exist_ok=True)
    total = sum(r["us"] for r in rows)
    gemm_us = sum(r["us"] for r in rows if r["kind"] in ("pw", "pw_dw"))
    floor_gemm = sum(max(r["flop_floor_us"], r["hbm_floor_us"]) for r in rows if r["kind"] in ("pw", "pw_dw"))
    summary = {"label": args.label, "gpu": info, "batch": args.batch, "profiled_steps": args.steps,
               "launches_per_step": per, "kernel_us_per_step": total, "pw_tc_kernel_us_per_step": gemm_us,
               "pw_tc_kernel_floor_us": floor_gemm, "rows": rows}
    with open(os.path.join(args.out, "profile_gemm.json"), "w") as f:
        json.dump(summary, f, indent=1)
    lines = [f"# track_boxes step, B = {args.batch}: {args.label}", "",
             f"GPU {info.get('name')}, power limit {info.get('power.limit')}, SM clock {info.get('clocks.sm')} "
             f"(max {info.get('clocks.max.sm')}); median of {args.steps} profiled steps.", "",
             f"Kernel time per step {total:.0f} us over {per} launches; pw_tc_kernel launches {gemm_us:.0f} us "
             f"(floor {floor_gemm:.0f} us).", "",
             "| # | layer | kernel | M x K x N | us | GFLOP | MB | TF32/FP32 floor us | HBM floor us | bound | of floor |",
             "|---|---|---|---|---|---|---|---|---|---|---|"]
    for r in rows:
        mkn = " x ".join(str(v) for v in r["mkn"]) if r["mkn"] else ""
        lines.append(f"| {r['launch']} | {r['layer']} | {r['kernel']} | {mkn} | {r['us']:.1f} | {r['flops'] / 1e9:.1f} | "
                     f"{r['bytes'] / 1e6:.1f} | {r['flop_floor_us']:.1f} | {r['hbm_floor_us']:.1f} | {r['bound']} | "
                     f"{r['of_floor']:.2f} |")
    with open(os.path.join(args.out, "profile_gemm.md"), "w") as f:
        f.write("\n".join(lines) + "\n")
    print("\n".join(lines))


if __name__ == "__main__":
    main()
