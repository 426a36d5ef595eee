"""Per-shape breakdown of the tensor-core convolution kernels inside one eager FPD step (hg_fpd shapes: student s4 f128,
teacher s8 f256, B=32).

Every ops.conv2d_tc_h / ops.conv2d_tc_fused call (forward and data-gradient convolutions: conv_wgmma_kernel or
conv_halo_kernel) and every ops.conv2d_wgrad_tc_fused call (wgrad_halo_kernel or wgrad_wgmma_kernel) is recorded on
the host with its shape; the i-th kernel of each family in the CUPTI trace is matched to the i-th call, and time is
aggregated per (kernel, shape). Each weight gradient is followed by one wgrad_reduce_kernel, reported beside the family.
The side streams (teacher overlap, hourglass branch fork, weight-gradient stream) are switched off so that each family
runs on one stream in call order; the kernels and their shapes are the same as in the overlapped step.

    python tools/profile_convs.py [--training-precision fp16]      # writes profile_out/profile_convs[_fp16].txt

--training-precision fp16 profiles the student at engine.set_training_precision("fp16"): its forward and data-gradient
convolutions then run on ops.conv2d_tc_f16x1 (conv_halo_f16x1_kernel, pw_conv_f16x1_kernel, or conv_wgmma_kernel
single-pass) and its weight gradients single-pass; the "wgrad" share of the step decides whether a faster weight
gradient is worth having.
"""
import argparse
import collections
import os
import re
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FAMILIES = {"conv": ("conv_wgmma_kernel", "conv_halo_kernel", "conv_halo_f16x1_kernel", "pw_conv_f16x1_kernel"),
            "wgrad": ("wgrad_halo_kernel", "wgrad_wgmma_kernel")}


def kernel_label(name):
    """'void fpd::(anonymous namespace)::conv_halo_kernel<128>(...)' -> 'conv_halo_kernel<128>'"""
    m = re.search(r"(\w+_kernel<[^>]*>)", name)
    return m.group(1) if m else name[:60]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--training-precision", default="fp32", choices=("fp32", "fp16"))
    args = ap.parse_args()
    for k in ("FPD_OVERLAP_TEACHER", "FPD_FORK_UP1", "FPD_WGRAD_STREAM"):
        os.environ[k] = "0"
    import fpd_b200  # noqa: F401
    from fpd_b200 import ops
    from fpd_b200.lib.models import hourglass as H
    from fpd_b200.train_step import FPDTrainStep
    from bench import cfg, synthetic_batch
    calls = collections.defaultdict(list)
    orig_h, orig_fused, orig_wgrad = ops.conv2d_tc_h, ops.conv2d_tc_fused, ops.conv2d_wgrad_tc_fused
    orig_f16x1 = ops.conv2d_tc_f16x1

    def conv_h(x, w_hi, w_lo, k, **kw):
        tag = "dgrad" if kw.get("in_scale") is not None or kw.get("relu_mask") is not None else "fwd"
        calls["conv"].append((tuple(x.shape), w_hi.shape[1], k, str(w_hi.dtype).replace("torch.", ""), tag))
        return orig_h(x, w_hi, w_lo, k, **kw)

    def conv_fused(x, w_hi, w_lo, k, **kw):
        calls["conv"].append((tuple(x.shape), w_hi.shape[1], k, "tf32", "fused"))
        return orig_fused(x, w_hi, w_lo, k, **kw)

    def conv_f16x1(x, w, k, **kw):
        tag = "dgrad" if kw.get("in_scale") is not None else "fwd"
        calls["conv"].append((tuple(x.shape), w.shape[1], k, "f16x1", tag))
        return orig_f16x1(x, w, k, **kw)

    def wgrad(x, dy, k, **kw):
        calls["wgrad"].append((tuple(x.shape), dy.shape[-1], k, "tf32x%d" % kw.get("passes", 3), "wgrad"))
        return orig_wgrad(x, dy, k, **kw)
    ops.conv2d_tc_h, ops.conv2d_tc_fused, ops.conv2d_wgrad_tc_fused = conv_h, conv_fused, wgrad
    ops.conv2d_tc_f16x1 = conv_f16x1
    from fpd_b200.engine import set_training_precision
    torch.manual_seed(0)
    student = H.get_pose_net(cfg(128, 4), True).cuda()
    teacher = H.get_pose_net(cfg(256, 8), False).cuda()
    set_training_precision(student, args.training_precision)
    step = FPDTrainStep(student, teacher, use_graph=False)
    x, t, w = (v.cuda() for v in synthetic_batch(32, 0))
    for _ in range(2):
        step.step(x, t, w)
    torch.cuda.synchronize()
    calls.clear()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step.step(x, t, w)
        torch.cuda.synchronize()
    evs = sorted([e for e in prof.events() if e.device_type is not None and "cuda" in str(e.device_type).lower()],
                 key=lambda e: e.time_range.start)
    step_us = sum(e.time_range.end - e.time_range.start for e in evs)
    out = ["one eager FPD step (side streams off), student training precision %s, device %s: kernel time %.2f ms" % (
        args.training_precision, torch.cuda.get_device_name(0), step_us / 1000.0)]
    for fam, shapes in calls.items():
        ks = [e for e in evs if any(n in e.name for n in FAMILIES[fam])]
        assert len(ks) == len(shapes), (fam, len(ks), len(shapes))
        agg = collections.defaultdict(lambda: [0, 0.0])
        for e, s in zip(ks, shapes):
            agg[(kernel_label(e.name),) + s][0] += 1
            agg[(kernel_label(e.name),) + s][1] += e.time_range.end - e.time_range.start
        tot = sum(v[1] for v in agg.values())
        out.append("%s: %d launches, %.2f ms (%.1f%% of the step's kernel time)" % (
            fam, len(ks), tot / 1000.0, 100.0 * tot / step_us))
        by_kernel = collections.defaultdict(float)
        for s, v in agg.items():
            by_kernel[s[0]] += v[1]
        for kname, us in sorted(by_kernel.items(), key=lambda kv: -kv[1]):
            out.append("  %-28s %8.2f ms" % (kname, us / 1000.0))
        if fam == "wgrad":
            red = [e for e in evs if "wgrad_reduce_kernel" in e.name]
            red_us = sum(e.time_range.end - e.time_range.start for e in red)
            out.append("  %-28s %8.2f ms (%d launches); wgrad family with the reduce: %.2f ms" % (
                "wgrad_reduce_kernel", red_us / 1000.0, len(red), (tot + red_us) / 1000.0))
        for s, v in sorted(agg.items(), key=lambda kv: -kv[1][1])[:30]:
            kname, (B, Hh, Ww, Cin), Cout, k, prec, tag = s
            gf = 2.0 * B * Hh * Ww * Cin * Cout * k * k / 1e9
            out.append("  %8.1f us %5.1f%% x%-3d avg %7.1f us  %-24s %-5s %-7s in[%d,%d,%d,%d] Cout=%d k=%d  "
                       "%.2f GF/launch -> %.0f TF/s alg" % (
                           v[1], 100 * v[1] / tot, v[0], v[1] / v[0], kname, tag, prec, B, Hh, Ww, Cin, Cout, k, gf,
                           gf / (v[1] / v[0]) * 1e3))
    text = "\n".join(out)
    path = os.path.join(ROOT, "profile_out", "profile_convs%s.txt" % (
        "" if args.training_precision == "fp32" else "_" + args.training_precision))
    os.makedirs(os.path.dirname(path), exist_ok=True)
    open(path, "w").write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
