"""Cost of distilling from a teacher at its own input size (FPDTrainStep.step(..., teacher_x=), a 384x288 teacher for a
256x192 student).

Kernel: fpd_heatmap_resample at [24, 96, 72, 17] -> [24, 64, 48, 17] (the hrnet_fpd teacher's map onto the student's
grid), captured once in a CUDA graph of --launches calls and timed with CUDA events over --repeats replays, with the HBM
lower bound of one read of the input and one write of the output at 3.35 TB/s (a bound, not a measurement).
Steps: bench.py's hrnet_fpd workload (HRNet-w32 student at 256x192, HRNet-w48 teacher, B = 24, FPDTrainStep with its
graph) with the teacher reading the student's 256x192 batch or its own 384x288 crop, each with the teacher's inference
precision "fp32" and "fp16": four captured steps, alternating over --step-repeats windows of --step-iters replays.
Prints one JSON object: median and (min, max) per variant, the card's name, power limit and SM clocks.

    python tools/bench_teacher_size.py [--launches 200] [--repeats 9] [--step-iters 10] [--step-repeats 5] [--out FILE]
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
HBM_BYTES_PER_S = 3.35e12
RESAMPLE = ((24, 96, 72, 17), (64, 48))


def nvsmi(fields):
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=" + fields, "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def summary(ts):
    return {"median": round(statistics.median(ts), 3), "min": round(min(ts), 3), "max": round(max(ts), 3)}


def kernel(args, dev):
    from fpd_b200 import ops
    shape, out_hw = RESAMPLE
    hm = torch.randn(shape, device=dev)
    out = torch.empty((shape[0],) + out_hw + (shape[3],), device=dev)
    for _ in range(3):
        ops.resample_heatmaps(hm, out_hw, out=out)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(args.launches):
            ops.resample_heatmaps(hm, out_hw, out=out)
    g.replay()
    torch.cuda.synchronize()
    ts = []
    for _ in range(args.repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.replay()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3 / args.launches)
    nbytes = (hm.numel() + out.numel()) * 4
    return {"shape": "%s -> %s" % (list(shape), [shape[0], *out_hw, shape[3]]), "us_per_call": summary(ts),
            "hbm_lower_bound_us": round(nbytes / HBM_BYTES_PER_S * 1e6, 2)}


def steps(args, dev):
    from bench import CONFIGS, build_models, synthetic_batch
    from fpd_b200.engine import set_inference_precision
    from fpd_b200.train_step import FPDTrainStep
    c = CONFIGS["hrnet_fpd"]
    x, target, tw = (t.to(dev) for t in synthetic_batch(c["batch"], 1000, c["H"], c["W"], c["J"]))
    tx = torch.randn(c["batch"], 3, c["H"] * 3 // 2, c["W"] * 3 // 2, generator=torch.Generator().manual_seed(7)).to(dev)
    runs = {}
    for prec in ("fp32", "fp16"):
        for size, t_in in (("teacher_256x192", None), ("teacher_384x288", tx)):
            student, teacher = build_models("hrnet_fpd", dev)
            set_inference_precision(teacher, prec)
            st = FPDTrainStep(student, teacher, alpha=0.5)
            for _ in range(3):
                st.step(x, target, tw, teacher_x=t_in)
            runs["%s_%s" % (size, prec)] = (st, t_in)
    torch.cuda.synchronize()
    times = {k: [] for k in runs}
    for _ in range(args.step_repeats):
        for key, (st, t_in) in runs.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.step_iters):
                st.step(x, target, tw, teacher_x=t_in)
            e1.record()
            e1.synchronize()
            times[key].append(e0.elapsed_time(e1) / args.step_iters)
    out = {"ms_per_step_" + k: summary(v) for k, v in times.items()}
    out["launches_per_step"] = {k: st.launches_per_step for k, (st, _) in runs.items()}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=9)
    ap.add_argument("--step-iters", type=int, default=10)
    ap.add_argument("--step-repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_teacher_size: needs a CUDA device")
    import fpd_b200  # noqa: F401
    dev = torch.device("cuda")
    result = {"card": torch.cuda.get_device_name(0), "power_limit_and_max_sm_clock": nvsmi("power.limit,clocks.max.sm")}
    result["resample_kernel"] = kernel(args, dev)
    result["hrnet_fpd_steps"] = steps(args, dev)
    result["sm_clock_and_power_after"] = nvsmi("clocks.sm,power.draw")
    text = json.dumps(result, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
