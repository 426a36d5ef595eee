"""Per-shape breakdown of the tensor-core conv / wgrad kernels inside one eager FPD step: records every call's shape on the
host, matches the i-th kernel of each type in a CUPTI trace to the i-th call, aggregates by (kernel, shape)."""
import collections
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import fpd_b200  # noqa: F401
    from fpd_b200 import ops
    from fpd_b200.lib.models import hourglass as H
    from fpd_b200.train_step import FPDTrainStep
    from bench import cfg, synthetic_batch
    os.environ["FPD_OVERLAP_TEACHER"] = "0"
    calls = collections.defaultdict(list)
    orig_conv, orig_wgrad = ops.conv2d_tc_fused, ops.conv2d_wgrad_tc_fused

    def conv(x, w_hi, w_lo, k, **kw):
        calls["conv_tc_ts_kernel"].append((tuple(x.shape), w_hi.shape[1], k))
        return orig_conv(x, w_hi, w_lo, k, **kw)

    def wgrad(x, dy, k, **kw):
        calls["wgrad_tc_fused_kernel"].append((tuple(x.shape), dy.shape[-1], k))
        return orig_wgrad(x, dy, k, **kw)
    ops.conv2d_tc_fused, ops.conv2d_wgrad_tc_fused = conv, wgrad
    torch.manual_seed(0)
    student = H.get_pose_net(cfg(128, 4), True).cuda()
    teacher = H.get_pose_net(cfg(256, 8), False).cuda()
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
    out = []
    for kname, shapes in calls.items():
        ks = [e for e in evs if kname in e.name]
        assert len(ks) == len(shapes), (kname, len(ks), len(shapes))
        agg = collections.defaultdict(lambda: [0, 0.0])
        for e, s in zip(ks, shapes):
            dur = e.time_range.end - e.time_range.start
            agg[s][0] += 1
            agg[s][1] += dur
        tot = sum(v[1] for v in agg.values())
        out.append("%s: %d launches, %.2f ms" % (kname, len(ks), tot / 1000.0))
        for s, v in sorted(agg.items(), key=lambda kv: -kv[1][1])[:22]:
            (B, Hh, Ww, Cin), Cout, k = s
            gf = 2.0 * B * Hh * Ww * Cin * Cout * k * k / 1e9
            out.append("  %8.1f us %5.1f%% x%-3d avg %7.1f us  in[%d,%d,%d,%d] Cout=%d k=%d  %.1f GF/launch -> %.0f TF/s alg" % (
                v[1], 100 * v[1] / tot, v[0], v[1] / v[0], B, Hh, Ww, Cin, Cout, k, gf, gf / (v[1] / v[0]) * 1e-3 * 1e3))
    text = "\n".join(out)
    path = os.path.join(ROOT, "profile_out", "profile_convs.txt")
    os.makedirs(os.path.dirname(path), exist_ok=True)
    open(path, "w").write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
