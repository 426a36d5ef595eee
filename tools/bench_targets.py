"""Device time of the heat-map target kernels at the two training shapes: fpd_gaussian_targets (the reference's rounded
targets), fpd_gaussian_targets_udp (UDP) and fpd_gaussian_targets_unbiased (DARK). Prints one JSON object with the
card's name, power limit and the SM clock read after the timed windows.

    python tools/bench_targets.py [--repeats 15] [--launches 200] [--out FILE]

Each window is one CUDA graph of `launches` back-to-back calls of one kernel on preallocated buffers, timed with CUDA
events around its replay, so the time is the device's and not the Python dispatch's. The kernels alternate window by
window; each reports the median (min-max) µs per call over `repeats` windows.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
# name, batch, joints, input (w, h), heat-map (w, h)
SHAPES = [("hourglass / MPII", 32, 16, (256, 256), (64, 64)), ("HRNet / COCO", 24, 17, (192, 256), (48, 64))]


def nvsmi(fields):
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=" + fields, "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def calls(B, J, img, hm, sigma=2):
    """One zero-argument launcher per kernel, on the same joints and output buffers."""
    from fpd_b200 import ops
    N = ops.N
    rng = np.random.RandomState(0)
    j = np.zeros((B, J, 3), np.float32)
    j[..., 0] = rng.uniform(-0.1, 1.1, (B, J)) * img[0]        # a few joints outside the crop, as after augmentation
    j[..., 1] = rng.uniform(-0.1, 1.1, (B, J)) * img[1]
    joints = torch.from_numpy(j).cuda()
    vis = torch.from_numpy((rng.rand(B, J, 3) > 0.15).astype(np.float32)).cuda()
    target = torch.empty((B, J, hm[1], hm[0]), device="cuda")
    tw = torch.empty((B, J, 1), device="cuda")
    table = ops.gaussian_table(sigma, "cuda")
    lib = N.lib()
    p = lambda t: t.data_ptr()                                                  # noqa: E731

    def run(rc, name):
        if rc != 0:
            raise RuntimeError("%s: %s" % (name, N.last_error()))
    common = (B, J, hm[1], hm[0], img[0], img[1], sigma)
    return {
        "default": lambda s: run(lib.fpd_gaussian_targets(p(joints), p(vis), None, p(table), p(target), p(tw), *common,
                                                          s), "gaussian_targets"),
        "udp": lambda s: run(lib.fpd_gaussian_targets_udp(p(joints), p(vis), None, p(target), p(tw), *common, s),
                             "gaussian_targets_udp"),
        "unbiased": lambda s: run(lib.fpd_gaussian_targets_unbiased(p(joints), p(vis), None, p(target), p(tw), *common,
                                                                    s), "gaussian_targets_unbiased"),
    }


def time_shape(B, J, img, hm, repeats, launches):
    fns = calls(B, J, img, hm)
    graphs = {}
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for f in fns.values():                                      # warm-up: module load
            for _ in range(10):
                f(side.cuda_stream)
    torch.cuda.current_stream().wait_stream(side)
    for k, f in fns.items():
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            s = torch.cuda.current_stream().cuda_stream
            for _ in range(launches):
                f(s)
        g.replay()
        graphs[k] = g
    torch.cuda.synchronize()
    us = {k: [] for k in fns}
    for _ in range(repeats):
        for k, g in graphs.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            g.replay()
            e1.record()
            e1.synchronize()
            us[k].append(e0.elapsed_time(e1) * 1e3 / launches)
    return {k: {"median": float(np.median(v)), "min": float(min(v)), "max": float(max(v))} for k, v in us.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=15)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_targets.py needs a CUDA device")
    import fpd_b200  # noqa: F401
    out = {"card": torch.cuda.get_device_name(0), "power_limit_and_max_sm_clock": nvsmi("power.limit,clocks.max.sm"),
           "repeats": args.repeats, "launches_per_window": args.launches, "shapes": []}
    for name, B, J, img, hm in SHAPES:
        row = {"shape": name, "batch": B, "joints": J, "input_wh": list(img), "heatmap_wh": list(hm)}
        row["us_per_call"] = time_shape(B, J, img, hm, args.repeats, args.launches)
        row["sm_clock_and_power_after"] = nvsmi("clocks.sm,power.draw")
        row["udp_over_default_median"] = row["us_per_call"]["udp"]["median"] / row["us_per_call"]["default"]["median"]
        out["shapes"].append(row)
    s = json.dumps(out, indent=1)
    print(s)
    if args.out:
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
