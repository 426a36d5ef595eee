"""Kernel time of the 3x3 3xFP16 convolutions of one hg_fpd step (student s4 f128 + teacher s8 f256, batch 32), forward
and data gradient, on whichever kernel the build selects for them (conv_halo_kernel where its halo fits).

The shapes, their launch counts and the call's form (BN affine + ReLU on the input, bias, residual, epilogue statistics;
data gradient = power-of-two input scale and ReLU mask) are recorded from one eager training step. Each form then runs
from a CUDA graph of `--per` launches over two rotating input / output sets, with an L2 flush before every timed window.
Prints µs per launch (median and range over the windows), the launch-weighted per-step total, and the share of the
fp16 tensor-core peak in executed MMAs (3 passes x the algorithmic FLOPs at 989 TFLOP/s, the H100 SXM data sheet's
dense figure), with the card's name, power limit and SM clock.

With --single-pass, each forward form also runs on ops.conv2d_tc_f16x1 (single-pass FP16, no epilogue statistics),
the two alternating window by window, and the single-pass share of the fp16 peak counts 1 x the algorithmic FLOPs.
With --train, the single-pass calls are the training precision "fp16" ones: the statistics forms keep their epilogue
statistics and the data gradients run too, with their power-of-two input scale.
With --half-io, each forward form (without statistics) runs on the single-pass kernel with fp32 activations against the
same kernel with fp16 activations (ops.conv2d_tc_f16x1_io: fp16 x, residual and y, inference precision "fp16_act"),
and the share of the HBM bound (3.35 TB/s) is that of the fp16 form's least bytes (2 per activation read or written).

    python tools/bench_conv3x3.py [--windows 7] [--per 8] [--single-pass [--train] | --half-io]
"""
import argparse
import collections
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

F16_FLOPS = 989e12   # H100 SXM data sheet, dense fp16
HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    return q


def form_of(kw):
    if kw.get("in_scale") is not None:
        return "dgrad" + (" mask" if kw.get("relu_mask") is not None else "")
    parts = []
    if kw.get("scale") is not None:
        parts.append("bn")
    if kw.get("bias") is not None:
        parts.append("bias")
    if kw.get("residual") is not None:
        parts.append("res")
    if kw.get("relu_mask") is not None:
        parts.append("mask")
    if kw.get("stats_part") is not None:
        parts.append("stats")
    return "+".join(parts) or "plain"


def step_shapes():
    """{(B, H, W, Cin, Cout, form): launches} of the 3x3 3xFP16 calls of one eager hg_fpd step."""
    from fpd_b200 import ops
    from fpd_b200.lib.models import hourglass as H
    from fpd_b200.train_step import FPDTrainStep
    from bench import cfg, synthetic_batch
    counts = collections.Counter()
    orig = ops.conv2d_tc_h

    def rec(x, w_hi, w_lo, k, **kw):
        if k == 3 and w_hi.dtype == torch.float16 and w_lo is not None:
            counts[tuple(x.shape) + (w_hi.shape[1], form_of(kw))] += 1
        return orig(x, w_hi, w_lo, k, **kw)
    torch.manual_seed(0)
    student = H.get_pose_net(cfg(128, 4), True).cuda()
    teacher = H.get_pose_net(cfg(256, 8), False).cuda()
    step = FPDTrainStep(student, teacher, use_graph=False)
    x, t, w = (v.cuda() for v in synthetic_batch(32, 0))
    step.step(x, t, w)
    torch.cuda.synchronize()
    ops.conv2d_tc_h = rec
    try:
        step.step(x, t, w)
        torch.cuda.synchronize()
    finally:
        ops.conv2d_tc_h = orig
    del step, student, teacher
    torch.cuda.empty_cache()
    return counts


def setup(shape, g, single=False, train=False):
    from fpd_b200 import ops
    B, H, W, Cin, Cout, form = shape
    xs = [torch.randn(B, H, W, Cin, device="cuda", generator=g) * (1e-3 if form.startswith("dgrad") else 1.0)
          for _ in range(2)]
    ys = [torch.empty(B, H, W, Cout, device="cuda") for _ in range(2)]
    w = torch.randn(Cout, Cin, 3, 3, device="cuda", generator=g) * (1.0 / (9 * Cin) ** 0.5)
    w_hi, w_lo = ops.weight_prep_f16(w)   # a data gradient's flipped weights have this [tap][Cout][Cin] layout too
    kw = {}
    if form.startswith("dgrad"):
        kw["in_scale"] = torch.tensor([1024.0, 1.0 / 1024.0], device="cuda")
    if "bn" in form:
        kw.update(mean=torch.randn(Cin, device="cuda", generator=g), scale=torch.rand(Cin, device="cuda", generator=g),
                  shift=torch.randn(Cin, device="cuda", generator=g), relu=True)
    if "bias" in form:
        kw["bias"] = torch.randn(Cout, device="cuda", generator=g)
    if "stats" in form:
        nblk = int(ops.N.lib().fpd_conv2d_tc_h_stats_blocks(B, H, W, Cin, Cout, 3, 1))
        kw["stats_part"] = torch.empty((nblk, Cout, 2), dtype=torch.float64, device="cuda")
        kw["stats_pivot"] = torch.zeros(Cout, device="cuda")
    res = [torch.randn(B, H, W, Cout, device="cuda", generator=g) for _ in range(2)] if "res" in form else None
    mask = [torch.randn(B, H, W, Cout, device="cuda", generator=g) for _ in range(2)] if "mask" in form else None

    def launch(i):
        ops.conv2d_tc_h(xs[i % 2], w_hi, w_lo, 3, residual=res[i % 2] if res else None,
                        relu_mask=mask[i % 2] if mask else None, out=ys[i % 2], **kw)
    if not single:
        return launch
    w1, _ = ops.weight_prep_f16(w, split=False)
    kw1 = {k: v for k, v in kw.items() if not k.startswith("stats")}
    if train and "stats" in form:
        nblk = ops.conv2d_tc_f16x1_train_plan(B, H, W, Cin, Cout, 3, stats=True)[1]
        kw1["stats_part"] = torch.empty((nblk, Cout, 2), dtype=torch.float64, device="cuda")
        kw1["stats_pivot"] = kw["stats_pivot"]

    def launch1(i):
        ops.conv2d_tc_f16x1(xs[i % 2], w1, 3, residual=res[i % 2] if res else None,
                            relu_mask=mask[i % 2] if mask else None, out=ys[i % 2], **kw1)
    return launch, launch1


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
    ap.add_argument("--single-pass", action="store_true")
    ap.add_argument("--train", action="store_true")
    ap.add_argument("--half-io", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_conv3x3 measures on the GPU"
    import fpd_b200  # noqa: F401
    print("device: %s (name, power limit, SM clock, max SM clock)" % card())
    shapes = step_shapes()
    if args.single_pass:
        return single_pass(shapes, args)
    if args.half_io:
        return half_io(shapes, args)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(0)
    print("%-40s %6s %10s %18s %8s" % ("shape (B,H,W,Cin->Cout form)", "x/step", "us", "range", "%F16"))
    tot = 0.0
    for shape, n in sorted(shapes.items(), key=lambda kv: -kv[0][0] * kv[0][1] * kv[0][2] * kv[0][3] * kv[0][4] * kv[1]):
        B, H, W, Cin, Cout, form = shape
        launch = setup(shape, g)
        graph = capture(launch, args.per)
        times = []
        for _ in range(args.windows):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            graph.replay()
            e1.record()
            torch.cuda.synchronize()
            times.append(1000.0 * e0.elapsed_time(e1) / args.per)
        med = sorted(times)[len(times) // 2]
        tot += n * med
        bound_us = 3 * 2.0 * B * H * W * Cin * Cout * 9 / F16_FLOPS * 1e6
        print("%-40s %6d %10.1f %18s %7.1f%%" % (
            "%d,%d,%d,%d->%d %s" % (B, H, W, Cin, Cout, form), n, med, "%.1f-%.1f" % (min(times), max(times)),
            100.0 * bound_us / med), flush=True)
        del graph, launch
        torch.cuda.empty_cache()
    print("3x3 3xFP16 convolutions of one hg_fpd step: %.2f ms" % (tot / 1000.0))
    print("device: %s (name, power limit, SM clock, max SM clock)" % card())


def window(graph, per, flush):
    flush.zero_()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    graph.replay()
    e1.record()
    torch.cuda.synchronize()
    return 1000.0 * e0.elapsed_time(e1) / per


def single_pass(shapes, args):
    """The step's forward forms on the 3-pass kernel against the single-pass one, windows alternating."""
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(0)
    print("%-40s %6s %10s %14s %10s %14s %8s %8s" % ("shape (B,H,W,Cin->Cout form)", "x/step", "3-pass us", "range",
                                                     "1-pass us", "range", "speedup", "%F16 1x"))
    tot3 = tot1 = 0.0
    for shape, n in sorted(shapes.items(), key=lambda kv: -kv[0][0] * kv[0][1] * kv[0][2] * kv[0][3] * kv[0][4] * kv[1]):
        B, H, W, Cin, Cout, form = shape
        if form.startswith("dgrad") and not args.train:
            continue
        launches = setup(shape, g, single=True, train=args.train)
        graphs = [capture(fn, args.per) for fn in launches]
        times = [[], []]
        for _ in range(args.windows):
            for i, gr in enumerate(graphs):
                times[i].append(window(gr, args.per, flush))
        med = [sorted(t)[len(t) // 2] for t in times]
        tot3 += n * med[0]
        tot1 += n * med[1]
        bound_us = 2.0 * B * H * W * Cin * Cout * 9 / F16_FLOPS * 1e6
        print("%-40s %6d %10.1f %14s %10.1f %14s %7.2fx %7.1f%%" % (
            "%d,%d,%d,%d->%d %s" % (B, H, W, Cin, Cout, form), n, med[0], "%.1f-%.1f" % (min(times[0]), max(times[0])),
            med[1], "%.1f-%.1f" % (min(times[1]), max(times[1])), med[0] / med[1], 100.0 * bound_us / med[1]),
            flush=True)
        del graphs, launches
        torch.cuda.empty_cache()
    print("3x3 %s convolutions of one hg_fpd step: 3-pass %.2f ms, single-pass %.2f ms" % (
        "forward and data-gradient" if args.train else "forward", tot3 / 1000.0, tot1 / 1000.0))
    print("device: %s (name, power limit, SM clock, max SM clock)" % card())


def half_io(shapes, args):
    """The step's forward forms (statistics dropped: eval forwards carry none) on the single-pass kernel with fp32
    activations against fp16 activations, windows alternating."""
    from fpd_b200 import ops
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(0)
    print("%-40s %6s %10s %14s %10s %14s %8s %9s %7s" % ("shape (B,H,W,Cin->Cout form)", "x/step", "f32-io us", "range",
                                                         "f16-io us", "range", "speedup", "least MB", "HBM %"))
    forms = collections.Counter()
    for (B, H, W, Cin, Cout, form), n in shapes.items():
        if not form.startswith("dgrad"):
            forms[(B, H, W, Cin, Cout, "+".join(f for f in form.split("+") if f not in ("stats", "mask")) or "plain")] += n
    tot32 = tot16 = 0.0
    for shape, n in sorted(forms.items(), key=lambda kv: -kv[0][0] * kv[0][1] * kv[0][2] * kv[0][3] * kv[0][4] * kv[1]):
        B, H, W, Cin, Cout, form = shape
        launch32 = setup(shape, g, single=True)[1]
        xs = [torch.randn(B, H, W, Cin, device="cuda", generator=g).half() for _ in range(2)]
        ys = [torch.empty(B, H, W, Cout, device="cuda", dtype=torch.float16) for _ in range(2)]
        res = [torch.randn(B, H, W, Cout, device="cuda", generator=g).half() for _ in range(2)] if "res" in form else None
        w1, _ = ops.weight_prep_f16(torch.randn(Cout, Cin, 3, 3, device="cuda", generator=g) * 0.05, split=False)
        kw = {}
        if "bn" in form:
            kw.update(mean=torch.randn(Cin, device="cuda", generator=g), scale=torch.rand(Cin, device="cuda", generator=g),
                      shift=torch.randn(Cin, device="cuda", generator=g), relu=True)
        if "bias" in form:
            kw["bias"] = torch.randn(Cout, device="cuda", generator=g)

        def launch16(i):
            ops.conv2d_tc_f16x1_io(xs[i % 2], w1, 3, residual=res[i % 2] if res else None, out=ys[i % 2],
                                   out_dtype=torch.float16, **kw)
        graphs = [capture(launch32, args.per), capture(launch16, args.per)]
        times = [[], []]
        for _ in range(args.windows):
            for i, gr in enumerate(graphs):
                times[i].append(window(gr, args.per, flush))
        med = [sorted(t)[len(t) // 2] for t in times]
        tot32 += n * med[0]
        tot16 += n * med[1]
        nbytes = 2 * B * H * W * (Cin + Cout * (2 if res else 1))
        print("%-40s %6d %10.1f %14s %10.1f %14s %7.2fx %9.1f %6.0f%%" % (
            "%d,%d,%d,%d->%d %s" % (B, H, W, Cin, Cout, form), n, med[0], "%.1f-%.1f" % (min(times[0]), max(times[0])),
            med[1], "%.1f-%.1f" % (min(times[1]), max(times[1])), med[0] / med[1], nbytes / 1e6,
            100.0 * nbytes / HBM_BYTES_PER_S * 1e6 / med[1]), flush=True)
        del graphs
        torch.cuda.empty_cache()
    print("3x3 forward convolutions of one hg_fpd step, single pass: fp32 activations %.2f ms, fp16 activations %.2f ms"
          % (tot32 / 1000.0, tot16 / 1000.0))
    print("device: %s (name, power limit, SM clock, max SM clock)" % card())


if __name__ == "__main__":
    main()
