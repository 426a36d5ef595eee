"""Training precision "fp32" (3xFP16 / 3xTF32, the default) against "fp16" (single-pass FP16 forward and data-gradient
convolutions, single-pass TF32 weight gradients: engine.set_training_precision) on bench.py's training workloads, the
two alternating window by window. Each step is FPDTrainStep with its CUDA graph, in the configuration bench.py runs:

  hg_fpd      student hourglass s4 f128 + frozen teacher s8 f256, 256x256, batch 32
  hrnet_fpd   student HRNet-w32 + frozen teacher w48, 256x192, batch 24
  res50_mse   pose_resnet-50, plain MSE, 256x256, batch 32
  hg_mse_s1   hourglass s1 f64, plain MSE, 256x256, batch 2

The workloads with a teacher run twice: teacher at inference precision "fp32", then at "fp16" (the combination a user
turns on with both switches). Prints ms per step, median (min-max) over the windows, with the card's name, power limit
and SM clock read in the same run.

    python tools/bench_train_precision.py [--windows 7] [--steps 10] [--only hg_fpd,...]
"""
import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--only", default="hg_fpd,hrnet_fpd,res50_mse,hg_mse_s1")
    args = ap.parse_args()
    import fpd_b200  # noqa: F401
    from bench import CONFIGS, build_models, synthetic_batch
    from bench_infer_precision import card
    from fpd_b200.engine import set_inference_precision, set_training_precision
    from fpd_b200.train_step import FPDTrainStep
    assert torch.cuda.is_available(), "bench_train_precision needs a CUDA device"
    dev = torch.device("cuda", 0)
    print("device: %s (name, power limit, SM clock, max SM clock)" % card())
    for name in args.only.split(","):
        c = CONFIGS[name]
        student, teacher = build_models(name, dev)
        x, target, tw = (t.to(dev) for t in synthetic_batch(c["batch"], 1000, c["H"], c["W"], c["J"]))
        step = FPDTrainStep(student, teacher, alpha=0.5 if teacher is not None else 0.0, lr=c["lr"])
        for t_prec in (("fp32", "fp16") if teacher is not None else ("fp32",)):
            if teacher is not None:
                set_inference_precision(teacher, t_prec)
            times = {"fp32": [], "fp16": []}
            for prec in ("fp32", "fp16"):       # warm-up: capture each precision's graph once
                set_training_precision(student, prec)
                for _ in range(3):
                    step.step(x, target, tw)
                torch.cuda.synchronize()
            for _ in range(args.windows):
                for prec in ("fp32", "fp16"):
                    set_training_precision(student, prec)
                    step.step(x, target, tw)          # the switch captures again: keep that out of the window
                    torch.cuda.synchronize()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(args.steps):
                        step.step(x, target, tw)
                    e1.record()
                    torch.cuda.synchronize()
                    times[prec].append(e0.elapsed_time(e1) / args.steps)
            line = "%-10s teacher %-4s" % (name, t_prec if teacher is not None else "-")
            med = {}
            for prec in ("fp32", "fp16"):
                t = sorted(times[prec])
                med[prec] = t[len(t) // 2]
                line += "  student %s %.2f ms (%.2f-%.2f)" % (prec, med[prec], t[0], t[-1])
            line += "  speed-up %.3fx" % (med["fp32"] / med["fp16"])
            print(line, flush=True)
        set_training_precision(student, "fp32")
        del student, teacher, step
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
