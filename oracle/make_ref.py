"""Recipe for oracle/_ref/: the reference's OWN hot-path Python modules, made available to the GPU box.

The reference is pure Python on this path (no C / C++ to compile), and /root/reference does not exist on the GPU box, so
the "compile the reference where it lies" step of a C reference becomes: copy the handful of hot-path source files,
unmodified, into oracle/_ref/lib/ -- a git-ignored, gpurun-shipped directory (like a built .so). They are used ONLY as
the checker / CPU baseline: `bench.py --impl reference` and `bench.py`'s cpu_baseline leg time these very modules on the
host cores (cpu_baseline.kind = "reference"), and tests/ may compare against them. Nothing under
fast-human-pose-estimation.pytorch_b200/ imports them. Run by __graft_entry__.build() when /root/reference is present:

    python oracle/make_ref.py [/root/reference]
"""
import hashlib
import json
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
DST = os.path.join(HERE, "_ref")
FILES = [
    "lib/models/hourglass.py",      # Bottleneck / Hourglass / HourglassNet / get_pose_net
    "lib/models/pose_hrnet.py",     # HRNet (a5-a7)
    "lib/models/pose_resnet.py",    # ResNet + deconv head (f4)
    "lib/core/loss.py",             # JointsMSELoss (a8)
    "lib/core/inference.py",        # get_max_preds / get_final_preds (a11, f1)
    "lib/core/evaluate.py",         # accuracy (f1)
    "lib/utils/transforms.py",      # flip_back, transform_preds (a12)
    "lib/nms/nms.py",               # numpy nms / oks_nms (a13, f3)
    "experiments/fpd_coco/hrnet/w32_256x192_adam_lr1e-3.yaml",
    "experiments/fpd_coco/hrnet/w48_256x192_adam_lr1e-3.yaml",
]


def make(ref_root="/root/reference"):
    if not os.path.isdir(ref_root):
        return None
    manifest = {}
    for rel in FILES:
        src = os.path.join(ref_root, rel)
        dst = os.path.join(DST, rel)
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        shutil.copyfile(src, dst)
        with open(src, "rb") as fh:
            manifest[rel] = hashlib.sha256(fh.read()).hexdigest()
    with open(os.path.join(DST, "MANIFEST.json"), "w") as fh:
        json.dump({"source": ref_root, "sha256": manifest}, fh, indent=1, sort_keys=True)
    return DST


if __name__ == "__main__":
    print(make(sys.argv[1] if len(sys.argv) > 1 else "/root/reference"))
