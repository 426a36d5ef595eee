"""Fused FPD loss time: fpd_loss_fused (both terms JointsMSELoss, one pass over the heat-maps) against
fpd_loss_ohkm_fused (both terms JointsOHKMMSELoss, topk 8: sums, selection, gradient pass) at the two FPD bench
shapes, value + gradient. --kl adds fpd_loss_kl_fused (both terms JointsKLDLoss, T = 1: maxima and exp-sums, merge,
gradient pass), and the time of one hg_fpd FPDTrainStep (bench.py's student, teacher and batch) with a JointsKLDLoss
kd term against JointsMSELoss, the two steps alternating over --step-repeats windows of --step-iters replays. Each variant is captured once in a CUDA graph of --launches calls and timed with CUDA events
over --repeats replays, the two variants alternating. Prints one JSON object with the card's name, power limit and the
SM clock read after the timed windows.

    python tools/bench_loss.py [--launches 200] [--repeats 7] [--kl] [--step-iters 20] [--step-repeats 5] [--out FILE]

Bytes per call are what the kernels must move at least: every stack read once (MSE) or twice (OHKM), the target and
the teacher read, every gradient written; KL reads every stack twice, like OHKM.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
# name, stacks, batch, joints, heat-map (h, w), teacher
SHAPES = [("hg_fpd", 4, 32, 16, (64, 64), True), ("hrnet_fpd", 1, 24, 17, (64, 48), True)]


def nvsmi(fields):
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=" + fields, "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def time_steps(args, dev):
    """ms per hg_fpd FPDTrainStep (graph replay + fused Adam) with kd_temperature=1 against the MSE kd term."""
    from bench import CONFIGS, build_models, synthetic_batch
    from fpd_b200.train_step import FPDTrainStep
    c = CONFIGS["hg_fpd"]
    x, target, tw = (t.to(dev) for t in synthetic_batch(c["batch"], 1000, c["H"], c["W"], c["J"]))
    steps = {}
    for key, kw in (("mse", {}), ("kl_kd_T1", {"kd_temperature": 1.0})):
        student, teacher = build_models("hg_fpd", dev)
        steps[key] = FPDTrainStep(student, teacher, alpha=0.5, **kw)
        for _ in range(3):
            steps[key].step(x, target, tw)
    torch.cuda.synchronize()
    times = {k: [] for k in steps}
    for _ in range(args.step_repeats):
        for key, st in steps.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.step_iters):
                st.step(x, target, tw)
            e1.record()
            e1.synchronize()
            times[key].append(e0.elapsed_time(e1) / args.step_iters)
    out = {"iters_per_window": args.step_iters, "windows": args.step_repeats}
    for key, ts in times.items():
        ts = sorted(ts)
        out[key] = {"ms_median": round(ts[len(ts) // 2], 3), "ms_min": round(ts[0], 3), "ms_max": round(ts[-1], 3)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--kl", action="store_true")
    ap.add_argument("--step-iters", type=int, default=20)
    ap.add_argument("--step-repeats", type=int, default=5)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_loss.py needs a CUDA device")
    import fpd_b200  # noqa: F401
    from fpd_b200 import ops
    dev = torch.device("cuda", 0)
    result = {"card": torch.cuda.get_device_name(0), "power_limit_and_max_sm_clock": nvsmi("power.limit,clocks.max.sm"),
              "launches_per_window": args.launches, "repeats": args.repeats, "shapes": []}
    for name, S, B, J, (h, w), has_teacher in SHAPES:
        g = torch.Generator(device=dev).manual_seed(1)
        tgt = torch.rand(B, J, h, w, generator=g, device=dev)
        outs = [torch.rand(B, h, w, J, generator=g, device=dev) for _ in range(S)]
        teacher = torch.rand(B, h, w, J, generator=g, device=dev) if has_teacher else None
        tw = (torch.rand(B, J, generator=g, device=dev) > 0.1).float()
        grads = [torch.empty_like(o) for o in outs]
        losses = torch.empty(3, device=dev)
        variants = {"mse": dict(), "ohkm_topk8": dict(pose_topk=8, kd_topk=8)}
        if args.kl:
            variants["kl_T1"] = dict(pose_temperature=1.0, kd_temperature=1.0)
        graphs = {}
        for key, kw in variants.items():
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(3):
                    ops.fpd_loss(outs, tgt, teacher, tw, 0.5, grads_out=grads, losses_out=losses, **kw)
            torch.cuda.current_stream().wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                for _ in range(args.launches):
                    ops.fpd_loss(outs, tgt, teacher, tw, 0.5, grads_out=grads, losses_out=losses, **kw)
            graph.replay()
            graphs[key] = graph
        torch.cuda.synchronize()
        times = {k: [] for k in variants}
        for _ in range(args.repeats):
            for key, graph in graphs.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                graph.replay()
                e1.record()
                e1.synchronize()
                times[key].append(e0.elapsed_time(e1) * 1000.0 / args.launches)
        fmap = B * h * w * J * 4
        moved = {"mse": (S + 2 + S) * fmap if has_teacher else (S + 1 + S) * fmap,
                 "ohkm_topk8": (2 * S + 2 * (2 if has_teacher else 1) + S) * fmap}
        moved["kl_T1"] = moved["ohkm_topk8"]
        entry = {"shape": name, "S": S, "B": B, "J": J, "hw": [h, w], "teacher": has_teacher}
        for key, ts in times.items():
            ts = sorted(ts)
            entry[key] = {"us_median": round(ts[len(ts) // 2], 2), "us_min": round(ts[0], 2), "us_max": round(ts[-1], 2),
                          "min_bytes": moved[key],
                          "GBps_at_median": round(moved[key] / (ts[len(ts) // 2] * 1e-6) / 1e9, 1)}
        entry["ohkm_over_mse"] = round(entry["ohkm_topk8"]["us_median"] / entry["mse"]["us_median"], 3)
        if args.kl:
            entry["kl_over_mse"] = round(entry["kl_T1"]["us_median"] / entry["mse"]["us_median"], 3)
            entry["kl_over_ohkm"] = round(entry["kl_T1"]["us_median"] / entry["ohkm_topk8"]["us_median"], 3)
        result["shapes"].append(entry)
    if args.kl:
        result["hg_fpd_step"] = time_steps(args, dev)
    result["sm_clock_and_power_after"] = nvsmi("clocks.sm,power.draw")
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
