"""Kernel time of the weight gradients of one hg_fpd step (student s4 f128, batch 32): the tap-row kernel
(wgrad_halo_kernel) against the per-tap kernel (wgrad_wgmma_kernel), switched with ops.set_wgrad_halo in one process.

The shapes, their launch counts and whether the call applies the BN affine + ReLU to x are recorded from one eager
training step. Each shape then runs from a CUDA graph of `--per` launches (weight-gradient kernel + reduce) over two
rotating input sets, with an L2 flush before every timed window; the two kernels' windows alternate. Prints µs per
launch (median and range over the windows), the launch-weighted per-step total, and the share of the 3-pass TF32
bound (3 x algorithmic FLOPs at 495 TFLOP/s, the H100 SXM data sheet), with the card's name, power limit and SM clock.

    python tools/bench_wgrad.py [--windows 7] [--per 8]
"""
import argparse
import collections
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

TF32_FLOPS = 495e12   # H100 SXM data sheet, dense


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    return q


def step_shapes():
    """{(B, H, W, Cin, Cout, k, bn_relu): launches} of one eager hg_fpd step."""
    from fpd_b200 import ops
    from fpd_b200.lib.models import hourglass as H
    from fpd_b200.train_step import FPDTrainStep
    from bench import cfg, synthetic_batch
    counts = collections.Counter()
    orig = ops.conv2d_wgrad_tc_fused

    def rec(x, dy, k, **kw):
        counts[tuple(x.shape) + (dy.shape[-1], k, kw.get("scale") is not None)] += 1
        return orig(x, dy, k, **kw)
    torch.manual_seed(0)
    student = H.get_pose_net(cfg(128, 4), True).cuda()
    teacher = H.get_pose_net(cfg(256, 8), False).cuda()
    step = FPDTrainStep(student, teacher, use_graph=False)
    x, t, w = (v.cuda() for v in synthetic_batch(32, 0))
    step.step(x, t, w)
    torch.cuda.synchronize()
    ops.conv2d_wgrad_tc_fused = rec
    try:
        step.step(x, t, w)
        torch.cuda.synchronize()
    finally:
        ops.conv2d_wgrad_tc_fused = orig
    del step, student, teacher
    torch.cuda.empty_cache()
    return counts


def setup(shape, g):
    from fpd_b200 import ops
    B, H, W, Cin, Cout, k, bn = shape
    xs = [torch.randn(B, H, W, Cin, device="cuda", generator=g) for _ in range(2)]
    dys = [torch.randn(B, H, W, Cout, device="cuda", generator=g) * 1e-3 for _ in range(2)]
    outs = [torch.empty(Cout, Cin, k, k, device="cuda") for _ in range(2)]
    kw = {}
    if bn:
        kw = dict(mean=torch.randn(Cin, device="cuda", generator=g), scale=torch.rand(Cin, device="cuda", generator=g),
                  shift=torch.randn(Cin, device="cuda", generator=g), relu=True)

    def launch(i):
        ops.conv2d_wgrad_tc_fused(xs[i % 2], dys[i % 2], k, out=outs[i % 2], **kw)
    return launch


def capture(launch, per):
    for i in range(2):
        launch(i)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        with torch.cuda.graph(graph, stream=side):
            for i in range(per):
                launch(i)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    return graph


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--per", type=int, default=8)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_wgrad measures on the GPU"
    import fpd_b200  # noqa: F401
    from fpd_b200 import ops
    print("device: %s (name, power limit, SM clock, max SM clock)" % card())
    prev = ops.set_wgrad_halo(True)
    shapes = step_shapes()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(0)
    print("%-34s %6s %10s %18s %10s %18s %8s %8s %8s" % (
        "shape (B,H,W,Cin->Cout,k,pre)", "x/step", "row us", "row range", "tap us", "tap range", "speedup",
        "row %TF", "tap %TF"))
    tot = {True: 0.0, False: 0.0}
    try:
        for shape, n in sorted(shapes.items(), key=lambda kv: -kv[0][0] * kv[0][1] * kv[0][2] * kv[0][3] * kv[0][4]
                               * kv[0][5] ** 2 * kv[1]):
            B, H, W, Cin, Cout, k, bn = shape
            if not ops.conv2d_wgrad_tc_supported(Cin, Cout, k):
                continue
            launch = setup(shape, g)
            graphs = {}
            for on in (True, False):
                ops.set_wgrad_halo(on)
                graphs[on] = capture(launch, args.per)
            times = {True: [], False: []}
            for _ in range(args.windows):
                for on in (True, False):
                    flush.zero_()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    graphs[on].replay()
                    e1.record()
                    torch.cuda.synchronize()
                    times[on].append(1000.0 * e0.elapsed_time(e1) / args.per)
            med = {kk: sorted(v)[len(v) // 2] for kk, v in times.items()}
            for on in (True, False):
                tot[on] += n * med[on]
            bound_us = 3 * 2.0 * B * H * W * Cin * Cout * k * k / TF32_FLOPS * 1e6
            print("%-34s %6d %10.1f %18s %10.1f %18s %7.2fx %7.1f%% %7.1f%%" % (
                "%d,%d,%d,%d->%d,%dx%d,%s" % (B, H, W, Cin, Cout, k, k, "bn" if bn else "-"), n, med[True],
                "%.1f-%.1f" % (min(times[True]), max(times[True])), med[False],
                "%.1f-%.1f" % (min(times[False]), max(times[False])), med[False] / med[True],
                100.0 * bound_us / med[True], 100.0 * bound_us / med[False]), flush=True)
            del graphs, launch
            torch.cuda.empty_cache()
    finally:
        ops.set_wgrad_halo(prev)
    print("weight gradients of one hg_fpd step (kernel + reduce): tap-row %.2f ms, per-tap %.2f ms" % (
        tot[True] / 1000.0, tot[False] / 1000.0))
    print("device: %s (name, power limit, SM clock, max SM clock)" % card())


if __name__ == "__main__":
    main()
