"""Kernel time of the 1x1 3xFP16 convolutions of one hg_fpd step (batch 32, 64x64): the weight-resident kernel
(pw_conv_wgmma_kernel) against the staged kernel (conv_wgmma_kernel), switched with ops.set_conv1x1 in one process.

Each kernel runs from a CUDA graph of `--per` launches over two rotating input / output sets (each set alone is larger
than the 50 MB L2), with an L2 flush before every timed window; the two kernels' windows alternate. Prints µs per launch
(median and range over the windows), the least HBM bytes of one launch (input, output, and residual where the call has
one: weights are read from L2) and the achieved share of 3.35 TB/s, with the card's name, power limit and SM clock.

With --single-pass, the forward forms instead run on the 3-pass weight-resident kernel against the single-pass one
(ops.conv2d_tc_f16x1, pw_conv_f16x1_kernel); the HBM share is then the single-pass kernel's. --train adds the data
gradients, single-pass with their power-of-two input scale as the training precision "fp16" runs them.
With --half-io, the forward forms run on the single-pass kernel with fp16 activations (ops.conv2d_tc_f16x1_io: fp16 x,
residual and y, inference precision "fp16_act") against the same kernel with fp32 activations; the least bytes and the
HBM share are then those of the fp16 form (2 bytes per activation).

    python tools/bench_conv1x1.py [--windows 7] [--per 8] [--single-pass [--train] | --half-io]
"""
import argparse
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet

# (Cin, Cout, form, launches per hg_fpd step): "fwd" = BN affine + ReLU + bias, "fwd_res" adds the residual,
# "bias" / "bias_res" = no input transform, "dgrad" = data gradient with in_scale
SHAPES = [
    (128, 256, "fwd_res", 18), (256, 256, "bias", 8), (256, 256, "bias_res", 7), (256, 128, "fwd", 17),
    (128, 64, "fwd", 9), (128, 64, "dgrad", 11), (64, 128, "fwd_res", 10), (64, 128, "dgrad", 9),
    (128, 128, "dgrad", 7), (128, 128, "bias", 4), (128, 128, "bias_res", 3),
    (256, 16, "bias", 8), (16, 256, "bias_res", 7), (128, 16, "bias", 4), (16, 128, "bias_res", 3),
    (16, 128, "dgrad", 4), (128, 16, "dgrad", 3),
]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    return q


def setup(B, H, W, Cin, Cout, form, g, single=False, half=False):
    from fpd_b200 import ops
    dt = torch.float16 if half else torch.float32
    xs = [torch.randn(B, H, W, Cin, device="cuda", generator=g).to(dt) for _ in range(2)]
    ys = [torch.empty(B, H, W, Cout, device="cuda", dtype=dt) for _ in range(2)]
    w = torch.randn(Cout, Cin, 1, 1, device="cuda", generator=g) * (1.0 / Cin ** 0.5)
    w_hi, w_lo = ops.weight_prep_f16(w)
    kw = {}
    if form.startswith("fwd"):
        kw = dict(mean=torch.randn(Cin, device="cuda", generator=g), scale=torch.rand(Cin, device="cuda", generator=g),
                  shift=torch.randn(Cin, device="cuda", generator=g), relu=True)
    if form != "dgrad":
        kw["bias"] = torch.randn(Cout, device="cuda", generator=g)
    else:
        kw["in_scale"] = torch.tensor([256.0, 1.0 / 256.0], device="cuda")
    res = [torch.randn(B, H, W, Cout, device="cuda", generator=g).to(dt) for _ in range(2)] if form.endswith("res") else None
    nbytes = (2 if half else 4) * B * H * W * (Cin + Cout * (2 if res else 1))

    def launch(i):
        if half:
            ops.conv2d_tc_f16x1_io(xs[i % 2], w1, 1, residual=res[i % 2] if res else None, out=ys[i % 2],
                                   out_dtype=torch.float16, **kw)
        elif single:
            ops.conv2d_tc_f16x1(xs[i % 2], w1, 1, residual=res[i % 2] if res else None, out=ys[i % 2], **kw)
        else:
            ops.conv2d_tc_h(xs[i % 2], w_hi, w_lo, 1, residual=res[i % 2] if res else None, out=ys[i % 2], **kw)
    w1 = ops.weight_prep_f16(w, split=False)[0] if (single or half) else None
    return launch, nbytes


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
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--hw", type=int, default=64)
    ap.add_argument("--single-pass", action="store_true")
    ap.add_argument("--train", action="store_true")
    ap.add_argument("--half-io", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_conv1x1 measures on the GPU"
    import fpd_b200  # noqa: F401
    from fpd_b200 import ops
    print("device: %s (name, power limit, SM clock, max SM clock)" % card())
    B, H, W = args.batch, args.hw, args.hw
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(0)
    names = ("f16-io", "f32-io") if args.half_io else ("1-pass", "3-pass") if args.single_pass else ("pw", "staged")
    print("%-22s %6s %10s %22s %10s %22s %8s %9s %7s" % (
        "shape (Cin->Cout form)", "x/step", names[0] + " us", names[0] + " range", names[1] + " us",
        names[1] + " range", "speedup", "least MB", "HBM %"))
    prev = ops.set_conv1x1(True)
    tot_pw = tot_st = 0.0
    try:
        for (Cin, Cout, form, n) in SHAPES:
            if (args.single_pass or args.half_io) and form == "dgrad" and not args.train:
                continue
            if args.half_io:       # True: fp16 activations, False: fp32 activations, both single pass
                launch, nbytes = setup(B, H, W, Cin, Cout, form, g, half=True)
                graphs = {True: capture(launch, args.per),
                          False: capture(setup(B, H, W, Cin, Cout, form, g, single=True)[0], args.per)}
            else:
                launch, nbytes = setup(B, H, W, Cin, Cout, form, g)
            if not args.half_io:
                graphs = {}
                for on in (True, False):
                    ops.set_conv1x1(on)
                    graphs[on] = capture(launch, args.per)
            if args.single_pass:   # True: single pass, False: the 3-pass weight-resident kernel
                ops.set_conv1x1(True)
                graphs = {False: graphs[True], True: capture(setup(B, H, W, Cin, Cout, form, g, single=True)[0],
                                                             args.per)}
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
            med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
            tot_pw += n * med[True]
            tot_st += n * med[False]
            least_us = nbytes / HBM_BYTES_PER_S * 1e6
            print("%-22s %6d %10.1f %22s %10.1f %22s %7.2fx %9.1f %6.0f%%" % (
                "%d->%d %s" % (Cin, Cout, form), n, med[True], "%.1f-%.1f" % (min(times[True]), max(times[True])),
                med[False], "%.1f-%.1f" % (min(times[False]), max(times[False])), med[False] / med[True], nbytes / 1e6,
                100.0 * least_us / med[True]), flush=True)
            del graphs, launch
            torch.cuda.empty_cache()
    finally:
        ops.set_conv1x1(prev)
    print("these shapes, one step at %dx%d: %s %.2f ms, %s %.2f ms" % (H, W, names[0], tot_pw / 1000.0, names[1],
                                                                       tot_st / 1000.0))
    print("device: %s (name, power limit, SM clock, max SM clock)" % card())


if __name__ == "__main__":
    main()
