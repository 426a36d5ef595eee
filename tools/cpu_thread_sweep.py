"""Thread-count sweep of the CPU legs (the reference's own modules, oracle/_ref) on the GPU host, so that
`cpu_baseline` / `--impl reference` use the thread count the reference actually runs fastest with on that machine.

    python tools/cpu_thread_sweep.py > cpu_thread_sweep.txt
"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CODE = r'''
import sys, time, json
sys.path.insert(0, %r)
import bench
ips, n, threads, kind = bench.time_cpu(%r, %d, steps=%d, warmup=1, max_seconds=%f)
print(json.dumps({"config": %r, "batch": %d, "threads": threads, "images_per_s": round(ips, 3), "steps": n, "kind": kind}))
'''


THREADS = (4, 8, 16, 24, 32, 64)


def main():
    ncpu = len(os.sched_getaffinity(0))
    print("# host: %d schedulable CPUs; %s" % (ncpu, open("/proc/cpuinfo").read().split("model name")[1].split("\n")[0].strip(": \t")))
    global THREADS
    if len(sys.argv) > 1 and sys.argv[1] == "small":      # second pass: small batches around the best thread counts
        THREADS = (8, 16, 24)
        plan = [("hg_fpd", 2, 3, 30.0), ("hg_fpd", 4, 3, 30.0), ("hrnet_fpd", 2, 3, 30.0), ("hrnet_fpd", 4, 3, 30.0),
                ("hg_infer", 4, 3, 20.0), ("hg_infer", 8, 3, 20.0)]
    else:
        plan = [("hg_fpd", 8, 2, 40.0), ("hg_fpd", 32, 1, 60.0), ("hg_mse_s1", 2, 10, 15.0), ("hg_infer", 16, 2, 30.0),
                ("hrnet_fpd", 8, 2, 40.0)]
    for name, B, steps, mx in plan:
        for t in THREADS:
            if t > ncpu:
                continue
            if B == 32 and t not in (8, 16, 32):
                continue
            env = dict(os.environ, FPD_CPU_THREADS=str(t), OMP_NUM_THREADS=str(t))
            r = subprocess.run([sys.executable, "-c", CODE % (ROOT, name, B, steps, mx, name, B)], env=env,
                               capture_output=True, text=True, timeout=600)
            print(r.stdout.strip() or ("ERR " + r.stderr.strip()[-300:]), flush=True)


if __name__ == "__main__":
    main()
