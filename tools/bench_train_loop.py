"""train() / fpd_train() per-step time: the eager fused route against the graph route (one FPDTrainStep replay per batch,
the caller's torch.optim.Adam stepping on the gradient views, losses and PCK counts copied to pinned host memory, the host
waiting only at the end of the epoch), plus the peak device memory with the training graph and validate()'s graph both
alive. Synthetic batches already on the device, the same seeded batch for both routes. Prints one JSON object with the
card's name, power limit and the SM clock read after each timed window.

    python tools/bench_train_loop.py [--steps 20] [--repeats 3] [--only hg_fpd,hrnet_fpd,res50_mse] [--out FILE]

ms per step = (time of an epoch of 3 + N batches - time of an epoch of 3 batches) / N, each window ending in a device
synchronise, so the per-call set-up (and the graph capture, which the first warm-up call pays) cancels. The two routes
alternate within each repeat.
"""
import argparse
import json
import os
import subprocess
import sys
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
NS = types.SimpleNamespace
MPII_FLIP = [[0, 5], [1, 4], [2, 3], [10, 15], [11, 14], [12, 13]]
COCO_FLIP = [[1, 2], [3, 4], [5, 6], [7, 8], [9, 10], [11, 12], [13, 14], [15, 16]]
WORKLOADS = ["hg_fpd", "hrnet_fpd", "res50_mse"]          # bench.py's configurations of the same names


def nvsmi(fields):
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=" + fields, "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


class _ValSet:
    def __init__(self, n, pairs):
        self.n, self.flip_pairs = n, pairs

    def __len__(self):
        return self.n

    def evaluate(self, cfg, preds, output_dir, all_boxes, image_path, filenames, imgnums):
        return {"Mean": 0.0}, 0.0


def batches(n, B, H, W, J):
    from bench import synthetic_batch
    x, t, w = synthetic_batch(B, 1, H, W, J)
    x, t, w = x.cuda(), t.cuda(), w.cuda()
    rng = np.random.RandomState(0)
    meta = {"center": torch.from_numpy(rng.uniform(100, 500, (B, 2))), "scale": torch.from_numpy(rng.uniform(0.5, 3, (B, 2))),
            "score": torch.ones(B, dtype=torch.float64), "image": ["img"] * B}
    return [(x, t, w, meta)] * n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--only", default=",".join(WORKLOADS))
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import bench
    import fpd_b200  # noqa: F401
    from fpd_b200.lib.core import function as F
    from fpd_b200.lib.core.loss import JointsMSELoss
    import logging
    logging.getLogger(F.__name__).setLevel(logging.WARNING)
    out = {"card": torch.cuda.get_device_name(0), "power_limit_and_max_sm_clock": nvsmi("power.limit,clocks.max.sm"),
           "steps": args.steps, "repeats": args.repeats, "workloads": []}
    for name in [n for n in args.only.split(",") if n]:
        c = bench.CONFIGS[name]
        B, H, W, J = c["batch"], c["H"], c["W"], c["J"]
        student, teacher = bench.build_models(name, torch.device("cuda", 0))
        opt = torch.optim.Adam(student.parameters(), lr=c["lr"])
        cfg = NS(MODEL=NS(NUM_JOINTS=J, NAME=name), KD=NS(ALPHA=0.5), PRINT_FREQ=10 ** 6, DEBUG=NS(DEBUG=False),
                 TEST=NS(FLIP_TEST=True, SHIFT_HEATMAP=True, POST_PROCESS=True))
        crit = JointsMSELoss(True)
        short, long_ = batches(3, B, H, W, J), batches(3 + args.steps, B, H, W, J)

        def epoch(loader, graph):
            F._TRAIN_GRAPH = graph
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            if teacher is not None:
                F.fpd_train(cfg, loader, student, teacher, crit, crit, opt, 0, "/tmp", "/tmp", None)
            else:
                F.train(cfg, loader, student, crit, opt, 0, "/tmp", "/tmp", None)
            torch.cuda.synchronize()
            return time.perf_counter() - t0

        for graph in (False, True):                      # warm-up: module loads, workspaces, the one capture
            epoch(short, graph)
        ms = {"eager": [], "graph": []}
        clocks = []
        for _ in range(args.repeats):
            for graph in (False, True):
                t_short = epoch(short, graph)
                t_long = epoch(long_, graph)
                clocks.append(nvsmi("clocks.sm,power.draw"))
                ms["graph" if graph else "eager"].append((t_long - t_short) / args.steps * 1e3)
        # peak memory of a graph-route epoch followed by validate() (which captures its own graph) while the training
        # graph stays cached, as tools/fpd_train.py runs them
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        epoch(short, True)
        flip = MPII_FLIP if J == 16 else COCO_FLIP
        F.validate(cfg, short, _ValSet(3 * B, flip), student, crit, "/tmp", "/tmp", None)
        torch.cuda.synchronize()
        F._TRAIN_GRAPH = True
        row = {"workload": c["workload"], "loop": "fpd_train" if teacher is not None else "train",
               "sm_clock_and_power_after_window": clocks,
               "peak_allocated_GiB_train_and_validate_graphs": torch.cuda.max_memory_allocated() / 2 ** 30,
               "peak_reserved_GiB_train_and_validate_graphs": torch.cuda.max_memory_reserved() / 2 ** 30}
        for k, v in ms.items():
            row[k + "_ms_per_step"] = {"median": float(np.median(v)), "min": float(min(v)), "max": float(max(v))}
        row["speedup_median"] = row["eager_ms_per_step"]["median"] / row["graph_ms_per_step"]["median"]
        out["workloads"].append(row)
        F._train_step_cache.clear()
        del student, teacher, opt
        torch.cuda.empty_cache()
        print(json.dumps(row), flush=True)
    s = json.dumps(out, indent=1)
    print(s)
    if args.out:
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
