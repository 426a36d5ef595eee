"""Build libfpd_b200.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU).

Usage: python build.py [--force]. Used by __graft_entry__.build(). Objects are cached under
csrc/_build/ keyed on source mtime; the .so and the objects are build products (git-ignored).
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libfpd_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC",
         "--expt-relaxed-constexpr", "-Xptxas", "-v"]
SOURCES = ["conv_wgmma.cu", "conv_simt.cu", "elementwise.cu", "loss.cu", "decode.cu", "nms.cu", "adam.cu", "augment.cu"]


def _newer(a, b):
    return (not os.path.exists(b)) or os.path.getmtime(a) > os.path.getmtime(b)


def build(force=False, verbose=False):
    bdir = os.path.join(CSRC, "_build")
    os.makedirs(bdir, exist_ok=True)
    headers = [os.path.join(CSRC, h) for h in ("common.cuh", "wgmma.cuh")] + [
        os.path.join(HERE, "..", "include", "fpd_b200.h")]
    hdr_m = max(os.path.getmtime(h) for h in headers)
    jobs = []
    objs = []
    for s in SOURCES:
        src = os.path.join(CSRC, s)
        obj = os.path.join(bdir, s.replace(".cu", ".o"))
        objs.append(obj)
        if force or _newer(src, obj) or hdr_m > os.path.getmtime(obj):
            jobs.append((src, obj))

    def compile_one(job):
        src, obj = job
        r = subprocess.run([NVCC, *FLAGS, "-c", src, "-o", obj], capture_output=True, text=True)
        return src, r

    with ThreadPoolExecutor(max_workers=8) as ex:
        for src, r in ex.map(compile_one, jobs):
            log = os.path.join(bdir, os.path.basename(src) + ".log")
            with open(log, "w") as f:
                f.write(r.stdout + r.stderr)
            if r.returncode != 0:
                sys.stderr.write(r.stdout + r.stderr)
                raise RuntimeError("nvcc failed for %s" % src)
            if verbose:
                sys.stderr.write(r.stderr)
    if jobs or not os.path.exists(OUT):
        r = subprocess.run([NVCC, "-shared", "-o", OUT, *objs, "-lcudart"], capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("link failed")
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
