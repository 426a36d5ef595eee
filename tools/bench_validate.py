"""validate() per-batch time: the eager fused route against the graph route (one FlipTestInference replay per batch,
results copied to pinned host memory, the host waiting only on PRINT_FREQ batches and at the end). Flip test, shift and
post-process on, synthetic batches already on the device, a trivial evaluate(). Prints one JSON object with the card's
name, power limit and the SM clock read after each timed window.

    python tools/bench_validate.py [--batches 40] [--repeats 5] [--dark] [--out FILE]

ms per batch = (time of validate over 5 + N batches - time over 5 batches) / N, so the per-call set-up (and the graph
capture) cancels. The two routes alternate within each repeat. --dark compares two graph routes instead: DARK's decode
(TEST.DARK, blur kernel 11) against the default quarter-pixel decode; it also times the two decode calls alone with CUDA
events on the workload's merged maps (ops.final_preds_dark against ops.final_preds), since their difference is what
DARK adds to a batch and is far below the spread of the per-batch times.
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
    """Seconds for one validate() over `batches`, synchronised at both ends."""
    F._VALIDATE_GRAPH = graph
    ds = _ValSet(len(batches) * batches[0][0].shape[0], pairs)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    F.validate(cfg, batches, ds, net, crit, "/tmp", "/tmp", None)
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def time_decodes(B, J, h, w, repeats, launches=500):
    """Device ms per call of ops.final_preds (quarter-pixel nudge) and ops.final_preds_dark on one batch of merged
    maps, CUDA events around `launches` back-to-back calls, the two alternating `repeats` times."""
    from fpd_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(0)
    avg = torch.rand((B, h, w, J), device="cuda", generator=g)
    _, idx, mv = ops.flip_merge_argmax(avg, want_avg=False)
    inv = torch.tensor([[4.0, 0.0, 1.0, 0.0, 4.0, 2.0]] * B, dtype=torch.float64, device="cuda")
    out = torch.empty((B, J, 3), device="cuda")
    calls = {"quarter": lambda: ops.final_preds(avg, idx, mv, inv, True, out=out),
             "dark": lambda: ops.final_preds_dark(avg, idx, mv, inv, 11, out=out)}
    ms = {k: [] for k in calls}
    for f in calls.values():
        for _ in range(20):
            f()
    for _ in range(repeats):
        for k, f in calls.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(launches):
                f()
            e1.record()
            e1.synchronize()
            ms[k].append(e0.elapsed_time(e1) / launches)
    return {k + "_decode_ms": {"median": float(np.median(v)), "min": float(min(v)), "max": float(max(v))}
            for k, v in ms.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=40)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--dark", action="store_true", help="time DARK's decode against the quarter-pixel one (graph route)")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import fpd_b200  # noqa: F401
    from fpd_b200.lib.core import function as F
    from fpd_b200.lib.core.loss import JointsMSELoss
    import logging
    logging.getLogger(F.__name__).setLevel(logging.WARNING)
    out = {"card": torch.cuda.get_device_name(0), "power_limit_and_max_sm_clock": nvsmi("power.limit,clocks.max.sm"),
           "batches": args.batches, "repeats": args.repeats, "workloads": []}
    # (name, graph route, TEST.DARK)
    routes = [("quarter", True, False), ("dark", True, True)] if args.dark else [("eager", False, False),
                                                                                ("graph", True, False)]
    out["routes"] = [r[0] for r in routes]
    for name, B, hw, J, pairs in WORKLOADS:
        torch.manual_seed(0)
        net = build(name, J).cuda()
        cfgs = {r: NS(MODEL=NS(NUM_JOINTS=J, NAME=name), PRINT_FREQ=100, DEBUG=NS(DEBUG=False),
                      TEST=NS(FLIP_TEST=True, SHIFT_HEATMAP=True, POST_PROCESS=True, DARK=dark, BLUR_KERNEL=11))
                for r, _, dark in routes}
        crit = JointsMSELoss(True)
        short, long_ = loader(5, B, hw, J), loader(5 + args.batches, B, hw, J)
        for r, graph, _ in routes:                        # warm-up: module loads, weight caches, first capture
            time_validate(F, cfgs[r], net, crit, short, graph, pairs)
        ms = {r: [] for r, _, _ in routes}
        clocks = []
        for _ in range(args.repeats):
            for r, graph, _ in routes:
                t_short = time_validate(F, cfgs[r], net, crit, short, graph, pairs)
                t_long = time_validate(F, cfgs[r], net, crit, long_, graph, pairs)
                clocks.append(nvsmi("clocks.sm,power.draw"))
                ms[r].append((t_long - t_short) / args.batches * 1e3)
        F._VALIDATE_GRAPH = True
        row = {"workload": name, "batch": B, "input_hw": list(hw), "joints": J, "sm_clock_and_power_after_window": clocks}
        for k, v in ms.items():
            row[k + "_ms_per_batch"] = {"median": float(np.median(v)), "min": float(min(v)), "max": float(max(v))}
        if args.dark:
            row["dark_extra_pct_median"] = 100.0 * (row["dark_ms_per_batch"]["median"] /
                                                    row["quarter_ms_per_batch"]["median"] - 1.0)
            row.update(time_decodes(B, J, hw[0] // 4, hw[1] // 4, args.repeats))
            row["dark_decode_extra_pct_of_quarter_batch"] = 100.0 * (
                row["dark_decode_ms"]["median"] - row["quarter_decode_ms"]["median"]) / row["quarter_ms_per_batch"]["median"]
        else:
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
