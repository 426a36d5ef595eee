"""Inference precisions "fp32" (3xFP16 / 3xTF32, the default), "fp16" (single-pass FP16) and "fp16_act" (single-pass
FP16 with fp16 activation storage; engine.set_inference_precision) on the benchmark workloads, alternating window by
window:

  hg_infer      hourglass s4 f128 flip-test inference (FlipTestInference graph), batch 128
  hrnet_infer   HRNet-w32 flip test, 256x192, batch 24
  diag_teacher  the hg_fpd teacher's forward alone (s8 f256, no flip), batch 32
  hg_fpd        FPDTrainStep, student s4 f128 + teacher s8 f256 in the given precision, batch 32
  hrnet_fpd     FPDTrainStep, student w32 + teacher w48, batch 24

Prints ms per call, median (min-max) over the windows, the speed-up of each reduced precision over "fp32", and, for the
inference workloads, the arg-max agreement of each with "fp32" on the timed batch, with the card's name, power limit
and SM clock.

    python tools/bench_infer_precision.py [--windows 7] [--steps 10] [--only hg_infer,...] [--modes fp32,fp16,fp16_act]
"""
import argparse
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                           "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout.strip()


def workload(name, dev):
    """-> (network whose precision is switched, run(): one call, outputs(): (idx, maxval) or None)."""
    from bench import CONFIGS, MPII_FLIP_PAIRS, build_models, synthetic_batch
    from fpd_b200.infer_step import FlipTestInference
    from fpd_b200.train_step import FPDTrainStep
    cfg_name = {"hg_infer": "hg_infer", "hrnet_infer": "hrnet_fpd", "diag_teacher": "diag_teacher", "hg_fpd": "hg_fpd",
                "hrnet_fpd": "hrnet_fpd"}[name]
    c = CONFIGS[cfg_name]
    student, teacher = build_models(cfg_name, dev)
    x, target, tw = (t.to(dev) for t in synthetic_batch(c["batch"], 1000, c["H"], c["W"], c["J"]))
    if name in ("hg_fpd", "hrnet_fpd"):
        step = FPDTrainStep(student, teacher, alpha=0.5, lr=c["lr"])
        return teacher, lambda: step.step(x, target, tw), None
    pairs = MPII_FLIP_PAIRS if c["J"] == 16 else [(1, 2), (3, 4), (5, 6), (7, 8), (9, 10), (11, 12), (13, 14), (15, 16)]
    inf = FlipTestInference(student, pairs, shift_heatmap=True, flip_test=c.get("flip", True), want_avg=False)
    res = {}

    def run():
        res["r"] = inf(x)
    return student, run, lambda: (res["r"]["idx"].clone(), res["r"]["maxval"].clone())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--only", default="hg_infer,hrnet_infer,diag_teacher,hg_fpd,hrnet_fpd")
    ap.add_argument("--modes", default="fp32,fp16,fp16_act")
    args = ap.parse_args()
    modes = args.modes.split(",")
    import fpd_b200  # noqa: F401
    from fpd_b200.engine import set_inference_precision
    assert torch.cuda.is_available(), "bench_infer_precision needs a CUDA device"
    dev = torch.device("cuda", 0)
    print("device: %s (name, power limit, SM clock, max SM clock)" % card())
    for name in args.only.split(","):
        net, run, outputs = workload(name, dev)
        times = {m: [] for m in modes}
        outs = {}
        for prec in modes:                  # warm-up: capture each precision's graph once
            set_inference_precision(net, prec)
            for _ in range(3):
                run()
            torch.cuda.synchronize()
            if outputs is not None:
                outs[prec] = outputs()
        for _ in range(args.windows):
            for prec in modes:
                set_inference_precision(net, prec)
                run()                         # the switch re-captures: keep that out of the window
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.steps):
                    run()
                e1.record()
                torch.cuda.synchronize()
                times[prec].append(e0.elapsed_time(e1) / args.steps)
        med = {m: sorted(times[m])[len(times[m]) // 2] for m in modes}
        line = name
        for prec in modes:
            t = sorted(times[prec])
            line += "  %s %.2f ms (%.2f-%.2f)" % (prec, med[prec], t[0], t[-1])
        for prec in modes[1:]:
            line += "  %s speed-up %.2fx" % (prec, med[modes[0]] / med[prec])
        if outputs is not None:
            i32, m32 = outs[modes[0]]
            for prec in modes[1:]:
                i16, m16 = outs[prec]
                line += "  %s arg-max identical %.2f %% of (b, j), max |dmaxval| %.2e" % (
                    prec, 100 * (i32 == i16).float().mean().item(), (m32 - m16).abs().max().item())
        print(line, flush=True)
        set_inference_precision(net, "fp32")
        del net, run, outputs
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
