"""Cost of feature distillation (FPDTrainStep(feature_weight=..., feature_adapter=...), KD.FEATURE_WEIGHT).

Kernel: fpd_feature_mse at the head-feature shapes of the two FPD configurations (hg_fpd: B 32, 64x64, 256 channels,
teacher in fp32 and in fp16; hrnet_fpd: B 24, 64x48, 48 channels), captured once in a CUDA graph of --launches calls and
timed with CUDA events over --repeats replays, variants alternating; next to it the HBM lower bound of its one pass (read
A(s) and t, write the gradient, at 3.35 TB/s: a bound, not a measurement). Steps: hg_fpd and hrnet_fpd FPDTrainStep
(bench.py's student, teacher and batch) with the term off and on (weight 1.0), alternating over --step-repeats windows of
--step-iters replays. Prints one JSON object: median and (min, max) per variant, the card's name, power limit and SM
clocks.

    python tools/bench_feature_kd.py [--launches 200] [--repeats 9] [--step-iters 10] [--step-repeats 7]
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
SHAPES = {"hg_fpd": (32, 64, 64, 256), "hrnet_fpd": (24, 64, 48, 48)}     # B, h, w, teacher channels
HBM_BYTES_PER_S = 3.35e12
WEIGHT = 1.0


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
    for name, (B, h, w, C) in SHAPES.items():
        g = torch.Generator(device=dev).manual_seed(1)
        t = torch.relu(torch.randn(B, h, w, C, generator=g, device=dev))
        s = t + 0.3 * torch.randn(B, h, w, C, generator=g, device=dev)
        t16 = t.half()
        grad, loss, losses = torch.empty_like(s), torch.empty(1, device=dev), torch.zeros(3, device=dev)
        fns = {"teacher_fp32": lambda: ops.feature_mse(s, t, WEIGHT, grad_out=grad, loss_out=loss, losses=losses)}
        if name == "hg_fpd":
            fns["teacher_fp16"] = lambda: ops.feature_mse(s, t16, WEIGHT, grad_out=grad, loss_out=loss, losses=losses)
        res = time_graphs(fns, args.launches, args.repeats)
        n = s.numel()
        for key in fns:
            nbytes = n * (4 + (2 if key == "teacher_fp16" else 4) + 4)
            bound = nbytes / HBM_BYTES_PER_S * 1e6
            res[key]["bytes"] = nbytes
            res[key]["hbm_bound_us_at_3.35TBps"] = round(bound, 2)
            res[key]["share_of_hbm_bound"] = round(bound / res[key]["median"], 3)
        out[name] = res
    return out


def steps(args, dev):
    from bench import CONFIGS, build_models, synthetic_batch
    from fpd_b200.train_step import FeatureAdapter, FPDTrainStep
    out = {}
    for name in ("hg_fpd", "hrnet_fpd"):
        c = CONFIGS[name]
        x, target, tw = (t.to(dev) for t in synthetic_batch(c["batch"], 1000, c["H"], c["W"], c["J"]))
        runs = {}
        order = ("off", "on") if args.first == "off" else ("on", "off")
        for key in order:
            student, teacher = build_models(name, dev)
            kw = {}
            if key == "on":
                kw = dict(feature_weight=WEIGHT, feature_adapter=FeatureAdapter(student, teacher).to(dev))
            runs[key] = FPDTrainStep(student, teacher, alpha=0.5, **kw)
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
        off, on = statistics.median(times["off"]), statistics.median(times["on"])
        out[name]["added_ms_median"] = round(on - off, 3)
        out[name]["added_share"] = round((on - off) / off, 4)
        out[name]["launches_per_step"] = {k: st.launches_per_step for k, st in runs.items()}
        out[name]["feature_loss_on"] = float(runs["on"].feature_loss)
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
        raise SystemExit("bench_feature_kd: needs a CUDA device")
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
