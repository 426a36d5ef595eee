"""validate() per-batch time: the eager fused route against the graph route (one FlipTestInference replay per batch,
results copied to pinned host memory, the host waiting only on PRINT_FREQ batches and at the end). Flip test, shift and
post-process on, synthetic batches already on the device, a trivial evaluate(). Prints one JSON object with the card's
name, power limit and the SM clock read after each timed window.

    python tools/bench_validate.py [--batches 40] [--repeats 5] [--out FILE]

ms per batch = (time of validate over 5 + N batches - time over 5 batches) / N, so the per-call set-up (and the graph
capture) cancels. The two routes alternate within each repeat.
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
# name, batch, input (H, W), joints, flip pairs
WORKLOADS = [("hourglass s4 f128 256x256", 32, (256, 256), 16, MPII_FLIP),
             ("hrnet w32 256x192", 24, (256, 192), 17, COCO_FLIP)]


def nvsmi(fields):
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=" + fields, "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def build(name, J):
    import bench
    if name.startswith("hourglass"):
        from fpd_b200.lib.models import hourglass as H
        return H.get_pose_net(bench.cfg(128, 4, J), False)
    from fpd_b200.lib.models import pose_hrnet as H
    return H.get_pose_net(bench.hrnet_cfg(32, J), False)


class _ValSet:
    def __init__(self, n, pairs):
        self.n, self.flip_pairs = n, pairs

    def __len__(self):
        return self.n

    def evaluate(self, cfg, preds, output_dir, all_boxes, image_path, filenames, imgnums):
        return {"Mean": 0.0}, 0.0


def loader(n, B, hw, J):
    from bench import synthetic_batch
    rng = np.random.RandomState(0)
    x, t, w = synthetic_batch(B, 1, hw[0], hw[1], J)
    x, t, w = x.cuda(), t.cuda(), w.cuda()
    meta = {"center": torch.from_numpy(rng.uniform(100, 500, (B, 2))), "scale": torch.from_numpy(rng.uniform(0.5, 3, (B, 2))),
            "score": torch.ones(B, dtype=torch.float64), "image": ["img"] * B}
    return [(x, t, w, meta)] * n


def time_validate(F, cfg, net, crit, batches, graph, pairs):
    F._VALIDATE_GRAPH = graph
    ds = _ValSet(len(batches) * batches[0][0].shape[0], pairs)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    F.validate(cfg, batches, ds, net, crit, "/tmp", "/tmp", None)
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=40)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import fpd_b200  # noqa: F401
    from fpd_b200.lib.core import function as F
    from fpd_b200.lib.core.loss import JointsMSELoss
    import logging
    logging.getLogger(F.__name__).setLevel(logging.WARNING)
    out = {"card": torch.cuda.get_device_name(0), "power_limit_and_max_sm_clock": nvsmi("power.limit,clocks.max.sm"),
           "batches": args.batches, "repeats": args.repeats, "workloads": []}
    for name, B, hw, J, pairs in WORKLOADS:
        torch.manual_seed(0)
        net = build(name, J).cuda()
        cfg = NS(MODEL=NS(NUM_JOINTS=J, NAME=name), PRINT_FREQ=100, DEBUG=NS(DEBUG=False),
                 TEST=NS(FLIP_TEST=True, SHIFT_HEATMAP=True, POST_PROCESS=True))
        crit = JointsMSELoss(True)
        short, long_ = loader(5, B, hw, J), loader(5 + args.batches, B, hw, J)
        for graph in (False, True):                       # warm-up: module loads, weight caches, first capture
            time_validate(F, cfg, net, crit, short, graph, pairs)
        ms = {"eager": [], "graph": []}
        clocks = []
        for _ in range(args.repeats):
            for graph in (False, True):
                t_short = time_validate(F, cfg, net, crit, short, graph, pairs)
                t_long = time_validate(F, cfg, net, crit, long_, graph, pairs)
                clocks.append(nvsmi("clocks.sm,power.draw"))
                ms["graph" if graph else "eager"].append((t_long - t_short) / args.batches * 1e3)
        F._VALIDATE_GRAPH = True
        row = {"workload": name, "batch": B, "input_hw": list(hw), "joints": J, "sm_clock_and_power_after_window": clocks}
        for k, v in ms.items():
            row[k + "_ms_per_batch"] = {"median": float(np.median(v)), "min": float(min(v)), "max": float(max(v))}
        row["speedup_median"] = row["eager_ms_per_batch"]["median"] / row["graph_ms_per_batch"]["median"]
        out["workloads"].append(row)
        del net
        torch.cuda.empty_cache()
    s = json.dumps(out, indent=1)
    print(s)
    if args.out:
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
