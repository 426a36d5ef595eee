"""Timeline of ONE graph-replayed FPD training step (the bench configuration): which streams are busy when, how many
SMs the resident kernels can cover, and where the step's wall time goes.

    python tools/timeline_step.py [--batch 32] [--tag r2a]

Writes profile_out/timeline_<tag>.csv.gz (name, stream, start_us, dur_us, grid) and profile_out/timeline_<tag>.txt:
  * span of the step, per-stream busy time,
  * "SM cover": integral over time of min(132, sum of grid sizes of the kernels running) / (132 x span) -- an upper
    bound on how much of the chip the launched grids could occupy (persistent kernels: grid <= 132),
  * time split by how many SMs the running kernels cover (<25 %, 25-50 %, 50-100 %, full),
  * per kernel family: launches, summed duration, duration-weighted mean grid.
CUPTI timestamps under a profiler: use the SHARES, not the absolute step time (bench.py is the step time)."""
import argparse
import collections
import gzip
import json
import os
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def short(name):
    n = name.replace("fpd::(anonymous namespace)::", "").replace("void ", "")
    for cut in ("(", "<"):
        if cut == "<" and ("channel_reduce" in n or "conv_tc_h" in n):
            continue
        i = n.find(cut)
        if i > 0:
            n = n[:i]
    return n[:60]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--tag", default="r2")
    ap.add_argument("--eager", action="store_true")
    ap.add_argument("--config", default="hg_fpd")
    args = ap.parse_args()
    import fpd_b200  # noqa: F401
    from fpd_b200.train_step import FPDTrainStep
    import bench
    from bench import synthetic_batch
    c = bench.CONFIGS[args.config]
    student, teacher = bench.build_models(args.config, torch.device("cuda"))
    step = FPDTrainStep(student, teacher, lr=c["lr"], use_graph=not args.eager)
    if args.batch <= 0:
        args.batch = c["batch"]
    x, t, w = (v.cuda() for v in synthetic_batch(args.batch, 0, c["H"], c["W"], c["J"]))
    for _ in range(4):
        step.step(x, t, w)
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step.step(x, t, w)
        torch.cuda.synchronize()
    tmp = tempfile.mktemp(suffix=".json")
    prof.export_chrome_trace(tmp)
    with open(tmp) as fh:
        trace = json.load(fh)
    os.remove(tmp)
    ev = []
    for e in trace["traceEvents"]:
        if e.get("cat") == "kernel" and e.get("ph") == "X":
            a = e.get("args", {})
            g = a.get("grid", [1, 1, 1])
            grid = int(g[0]) * int(g[1]) * int(g[2])
            ev.append((float(e["ts"]), float(e["dur"]), int(a.get("stream", 0)), grid, e["name"]))
    ev.sort()
    t0 = ev[0][0]
    t1 = max(s + d for s, d, _, _, _ in ev)
    span = t1 - t0
    out_dir = os.path.join(ROOT, "profile_out")
    os.makedirs(out_dir, exist_ok=True)
    with gzip.open(os.path.join(out_dir, "timeline_%s.csv.gz" % args.tag), "wt") as fh:
        fh.write("name,stream,start_us,dur_us,grid\n")
        for s, d, st, g, n in ev:
            fh.write("%s,%d,%.3f,%.3f,%d\n" % (short(n), st, s - t0, d, g))
    # sweep
    pts = []
    for s, d, st, g, n in ev:
        pts.append((s, g, 1))
        pts.append((s + d, -g, -1))
    pts.sort()
    cover = 0.0
    buckets = collections.OrderedDict((k, 0.0) for k in ("idle", "<25%", "25-50%", "50-100%", "full"))
    conc = collections.Counter()
    cur_g = cur_n = 0
    last = t0
    for tt, dg, dn in pts:
        dt = tt - last
        if dt > 0:
            c = min(132, cur_g)
            cover += dt * c
            k = "idle" if cur_n == 0 else "<25%" if c < 33 else "25-50%" if c < 66 else "50-100%" if c < 132 else "full"
            buckets[k] += dt
            conc[min(cur_n, 6)] += dt
        cur_g += dg
        cur_n += dn
        last = tt
    streams = collections.defaultdict(float)
    fam = collections.defaultdict(lambda: [0, 0.0, 0.0, 0])
    for s, d, st, g, n in ev:
        streams[st] += d
        f = fam[short(n)]
        f[0] += 1
        f[1] += d
        f[2] += d * min(g, 132)
        f[3] += 1 if g < 132 else 0
    lines = []
    lines.append("config %s" % args.config)
    lines.append("one %s FPD step, B=%d: %d kernels, span %.3f ms, summed kernel time %.3f ms" % (
        "eager" if args.eager else "graph-replayed", args.batch, len(ev), span / 1e3, sum(e[1] for e in ev) / 1e3))
    lines.append("SM cover (time-integral of min(132, sum of running grids)) = %.3f of 132 x span" % (cover / (132 * span)))
    lines.append("time by SM cover of the running kernels: " + ", ".join("%s %.2f ms" % (k, v / 1e3) for k, v in buckets.items()))
    lines.append("time by number of concurrently running kernels: " + ", ".join(
        "%s%d: %.2f ms" % (">=" if k == 6 else "", k, v / 1e3) for k, v in sorted(conc.items())))
    lines.append("per stream busy ms: " + ", ".join("s%d %.2f" % (k, v / 1e3) for k, v in sorted(streams.items(), key=lambda kv: -kv[1])))
    lines.append("%-58s %6s %9s %9s %7s" % ("kernel", "n", "sum ms", "mean grid", "n<132"))
    for k, f in sorted(fam.items(), key=lambda kv: -kv[1][1]):
        lines.append("%-58s %6d %9.3f %9.1f %7d" % (k, f[0], f[1] / 1e3, f[2] / max(f[1], 1e-9), f[3]))
    txt = "\n".join(lines)
    with open(os.path.join(out_dir, "timeline_%s.txt" % args.tag), "w") as fh:
        fh.write(txt + "\n")
    print(txt)


if __name__ == "__main__":
    main()
