"""Kernel-level breakdown of one eager FPD training step (BASELINE configs[1] shapes).

    python tools/profile_step.py                 # torch.profiler (CUPTI) table, warm caches
    ncu --metrics gpu__time_duration.sum --clock-control none --profile-from-start off --csv \
        --log-file profile_out/launches.csv python tools/profile_step.py --ncu      # per-launch kernel durations
"""
import argparse
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
NS = types.SimpleNamespace


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ncu", action="store_true")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--out", default=os.path.join(ROOT, "profile_out", "profile_step.txt"))
    args = ap.parse_args()
    import fpd_b200  # noqa: F401
    from fpd_b200.lib.models import hourglass as H
    from fpd_b200.train_step import FPDTrainStep
    sys.path.insert(0, ROOT)
    from bench import cfg, synthetic_batch
    torch.manual_seed(0)
    student = H.get_pose_net(cfg(128, 4), True).cuda()
    teacher = H.get_pose_net(cfg(256, 8), False).cuda()
    step = FPDTrainStep(student, teacher, use_graph=False)
    x, t, w = (v.cuda() for v in synthetic_batch(args.batch, 0))
    for _ in range(2):
        step.step(x, t, w)
    torch.cuda.synchronize()
    if args.ncu:
        torch.cuda.profiler.start()
        step.step(x, t, w)
        torch.cuda.synchronize()
        torch.cuda.profiler.stop()
        return
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
        step.step(x, t, w)
        torch.cuda.synchronize()
    rows = []
    for e in prof.key_averages():
        dt = getattr(e, "device_time_total", None)
        if dt is None:
            dt = getattr(e, "cuda_time_total", 0)
        if dt and e.device_type is not None and "cuda" in str(e.device_type).lower():
            rows.append((dt, e.count, e.key))
    if not rows:  # fall back: every event with device time
        for e in prof.key_averages():
            dt = getattr(e, "device_time_total", 0) or getattr(e, "cuda_time_total", 0)
            if dt:
                rows.append((dt, e.count, e.key))
    rows.sort(reverse=True)
    total = sum(r[0] for r in rows)
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as fh:
        fh.write("one eager FPD step, B=%d: total device time %.3f ms over %d kernel types\n" % (
            args.batch, total / 1000.0, len(rows)))
        for dt, cnt, key in rows[:40]:
            fh.write("%9.3f ms %6.2f%% x%-5d %s\n" % (dt / 1000.0, 100.0 * dt / total, cnt, key[:110]))
    print(open(args.out).read())


if __name__ == "__main__":
    main()
