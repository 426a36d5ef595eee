"""Cost of distillation from unlabeled samples (FPDTrainStep(kd_unlabeled_thre=...), KD.UNLABELED).

Kernels, at the two FPD shapes (hg_fpd: 4 stacks, B 32, 64x64, J 16; hrnet_fpd: 1 stack, B 24, 64x48, J 17), each
captured once in a CUDA graph of --launches calls and timed with CUDA events over --repeats replays, variants
alternating: fpd_kd_weights, and for a JointsMSELoss and a JointsKLDLoss (T = 1) kd term the fused loss through the
existing entry point against the kd-weighted one (fpd_loss_kdw_fused). Steps: hg_fpd and hrnet_fpd FPDTrainStep (bench.py's
student, teacher and batch, half the samples unlabeled) with the mode off and on (thre 0.2), alternating over
--step-repeats windows of --step-iters replays. Prints one JSON object: median and (min, max) per variant, the card's
name, power limit and SM clocks, and the HBM lower bound of the weight pass (one read of the teacher's last heat-map at
3.35 TB/s; a bound, not a measurement).

    python tools/bench_unlabeled_kd.py [--launches 200] [--repeats 9] [--step-iters 10] [--step-repeats 7]
                                      [--first off|on] [--no-kernels] [--out FILE]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
SHAPES = {"hg_fpd": (4, 32, 16, 64, 64), "hrnet_fpd": (1, 24, 17, 64, 48)}     # stacks, B, J, h, w
HBM_BYTES_PER_S = 3.35e12
THRE = 0.2


def nvsmi(fields):
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=" + fields, "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def summary(ts):
    return {"median": round(statistics.median(ts), 3), "min": round(min(ts), 3), "max": round(max(ts), 3)}


def time_graphs(fns, launches, repeats):
    """us per call of each fn: one graph of `launches` calls per fn, replays alternating between the fns."""
    graphs = {}
    for name, fn in fns.items():
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for _ in range(launches):
                fn()
        g.replay()
        graphs[name] = g
    torch.cuda.synchronize()
    times = {k: [] for k in graphs}
    for _ in range(repeats):
        for name, g in graphs.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            g.replay()
            e1.record()
            e1.synchronize()
            times[name].append(e0.elapsed_time(e1) * 1e3 / launches)
    return {k: summary(v) for k, v in times.items()}


def kernels(args, dev):
    from fpd_b200 import ops
    out = {}
    for name, (S, B, J, h, w) in SHAPES.items():
        g = torch.Generator(device=dev).manual_seed(1)
        target = torch.rand(B, J, h, w, generator=g, device=dev)
        teacher = 0.3 * torch.randn(B, h, w, J, generator=g, device=dev)
        outs = [0.3 * torch.randn(B, h, w, J, generator=g, device=dev) for _ in range(S)]
        tw = (torch.rand(B, J, generator=g, device=dev) > 0.2).float()
        tw[::2] = 0.0
        kdw = ops.kd_weights(teacher, tw, THRE)
        grads = [torch.empty_like(o) for o in outs]
        losses = torch.empty(3, device=dev)
        kdw_buf = torch.empty_like(kdw)
        fns = {"kd_weights": lambda: ops.kd_weights(teacher, tw, THRE, out=kdw_buf)}
        for crit, kw in (("mse", {}), ("kl", {"kd_temperature": 1.0})):
            fns["loss_%s_existing" % crit] = (lambda kw=kw: ops.fpd_loss(outs, target, teacher, tw, 0.5, grads_out=grads,
                                                                        losses_out=losses, **kw))
            fns["loss_%s_kd_weighted" % crit] = (lambda kw=kw: ops.fpd_loss(outs, target, teacher, tw, 0.5,
                                                                           grads_out=grads, losses_out=losses,
                                                                           kd_weight=kdw, **kw))
        res = time_graphs(fns, args.launches, args.repeats)
        nbytes = B * h * w * J * 4
        res["kd_weights_lower_bound"] = {"bytes_read": nbytes, "us_at_3.35TBps": round(nbytes / HBM_BYTES_PER_S * 1e6, 2)}
        out[name] = res
    return out


def steps(args, dev):
    from bench import CONFIGS, build_models, synthetic_batch
    from fpd_b200.train_step import FPDTrainStep
    out = {}
    for name in ("hg_fpd", "hrnet_fpd"):
        c = CONFIGS[name]
        x, target, tw = (t.to(dev) for t in synthetic_batch(c["batch"], 1000, c["H"], c["W"], c["J"]))
        target[::2] = 0.0
        tw[::2] = 0.0
        runs = {}
        order = (("off", None), ("on", THRE)) if args.first == "off" else (("on", THRE), ("off", None))
        for key, thre in order:
            student, teacher = build_models(name, dev)
            runs[key] = FPDTrainStep(student, teacher, alpha=0.5, kd_unlabeled_thre=thre)
            for _ in range(3):
                runs[key].step(x, target, tw)
        torch.cuda.synchronize()
        times = {k: [] for k in runs}
        for _ in range(args.step_repeats):
            for key, st in runs.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.step_iters):
                    st.step(x, target, tw)
                e1.record()
                e1.synchronize()
                times[key].append(e0.elapsed_time(e1) / args.step_iters)
        out[name] = {"ms_per_step_" + k: summary(v) for k, v in times.items()}
        out[name]["launches_per_step"] = {k: st.launches_per_step for k, st in runs.items()}
        del runs
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=9)
    ap.add_argument("--step-iters", type=int, default=10)
    ap.add_argument("--step-repeats", type=int, default=7)
    ap.add_argument("--first", choices=["off", "on"], default="off",
                    help="which of the two steps is built (and captured) first: run both ways to see the order's effect")
    ap.add_argument("--no-kernels", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_unlabeled_kd: needs a CUDA device")
    import fpd_b200  # noqa: F401
    dev = torch.device("cuda")
    result = {"card": torch.cuda.get_device_name(0), "power_limit_and_max_sm_clock": nvsmi("power.limit,clocks.max.sm")}
    if not args.no_kernels:
        result["kernels_us"] = kernels(args, dev)
    result["steps_built_first"] = args.first
    result["steps"] = steps(args, dev)
    result["sm_clock_and_power_after"] = nvsmi("clocks.sm,power.draw")
    text = json.dumps(result, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
