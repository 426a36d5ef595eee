"""Input-crop benchmark: the device crop (csrc/augment.cu) on batches drawn by RawJointsDataset from 640x480 sources
with the reference's default augmentation (SCALE_FACTOR 0.25, ROT_FACTOR 30, flip, half body), and the host work per
sample against the reference's per-sample path. Prints one JSON object (with the card's name and power limit).

    python tools/bench_augment.py [--iters 300] [--host-samples 200] [--out FILE]

Needs cv2 (the crop matrices) and a CUDA device. Source images are synthetic PNGs in a temporary directory; decoding is
excluded from every host timing.
"""
import argparse
import json
import os
import random
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12       # H100 SXM data sheet
WORKLOADS = [(32, (256, 256), (64, 64)), (128, (256, 256), (64, 64)), (24, (192, 256), (48, 64))]   # B, (w, h), heat-map
COCO_FLIP = [[1, 2], [3, 4], [5, 6], [7, 8], [9, 10], [11, 12], [13, 14], [15, 16]]
MEAN, STD = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return {"name": name, "power_limit_and_max_sm_clock": q}


def dataset(image_paths, size, heatmap, n, rng):
    from oracle.augment_oracle import StandInDataset
    cfg = {"is_train": True, "color_rgb": True, "image_size": list(size), "heatmap_size": list(heatmap), "sigma": 2,
           "scale_factor": 0.25, "rotation_factor": 30, "flip": True, "num_joints_half_body": 8, "prob_half_body": 0.3,
           "num_joints": 17, "flip_pairs": COCO_FLIP, "upper_body_ids": list(range(11)), "mean": MEAN, "std": STD}
    aspect = size[0] / size[1]
    db = []
    for i in range(n):
        bw = rng.uniform(60, 400)
        c = np.array([rng.uniform(100, 540), rng.uniform(80, 400)], np.float32)
        joints = np.zeros((17, 3))
        joints[:, 0] = c[0] + rng.uniform(-0.5, 0.5, 17) * bw
        joints[:, 1] = c[1] + rng.uniform(-0.5, 0.5, 17) * bw / aspect
        vis = np.zeros((17, 3))
        vis[:, :2] = (rng.rand(17) > 0.2)[:, None]
        db.append({"image": image_paths[i % len(image_paths)], "filename": "", "imgnum": 0, "center": c,
                   "scale": np.array([bw / 200, bw / aspect / 200], np.float32) * 1.25, "joints_3d": joints * vis,
                   "joints_3d_vis": vis})
    return StandInDataset(cfg, db)


class _Cached:
    """RawJointsDataset with the decode replaced by a lookup, so that host timings exclude imread."""

    def __init__(self, raw, images):
        self.raw, self.images = raw, images
        raw.read_image = lambda f: self.images[f]


def host_reference(ds, images, idx):
    """The reference's per-sample work after the draws: warpAffine, ToTensor + Normalize, generate_target."""
    import cv2
    from fpd_b200.augment import crop_matrix
    from oracle.decode_oracle import generate_target
    rec = ds.db[idx]
    img = images[rec["image"]]
    if idx % 2:
        img = img[:, ::-1, :]                                # half of the training samples are mirrored
    trans = crop_matrix(rec["center"], rec["scale"], 15.0, ds.image_size)
    t0 = time.perf_counter()
    crop = cv2.warpAffine(img, trans, (int(ds.image_size[0]), int(ds.image_size[1])), flags=cv2.INTER_LINEAR)
    x = ds.transform(crop)
    joints = rec["joints_3d"].copy()
    for j in range(ds.num_joints):
        if rec["joints_3d_vis"][j, 0] > 0:
            joints[j, :2] = np.dot(trans, np.array([joints[j, 0], joints[j, 1], 1.]))[:2]
    target, tw = generate_target(joints, rec["joints_3d_vis"], ds.image_size, ds.heatmap_size, ds.sigma)
    torch.from_numpy(target), torch.from_numpy(tw)
    return time.perf_counter() - t0, x


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=300)
    ap.add_argument("--host-samples", type=int, default=200)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import cv2
    import fpd_b200  # noqa: F401
    from fpd_b200 import augment as A
    from fpd_b200 import ops
    assert torch.cuda.is_available(), "bench_augment needs a CUDA device"
    rng = np.random.RandomState(0)
    tmp = tempfile.mkdtemp()
    images = {}
    for k in range(4):
        yy, xx = np.mgrid[0:480, 0:640]
        img = (128 + 100 * np.sin(xx * rng.uniform(0.01, 0.1) + k)[..., None] * np.cos(yy * 0.03)[..., None]
               + rng.randint(0, 40, (480, 640, 3))).clip(0, 255).astype(np.uint8)
        p = os.path.join(tmp, "src%d.png" % k)
        cv2.imwrite(p, img)
        images[p] = cv2.imread(p, cv2.IMREAD_COLOR | cv2.IMREAD_IGNORE_ORIENTATION)
    result = {"card": card(), "source": "640x480", "workloads": []}
    for B, size, heatmap in WORKLOADS:
        ds = dataset(list(images), size, heatmap, max(B, args.host_samples), rng)
        raw = A.RawJointsDataset(ds)
        _Cached(raw, images)
        np.random.seed(1)
        random.seed(1)
        batch = A.raw_collate([raw[i] for i in range(B)])
        batch = {k: (v.pin_memory() if torch.is_tensor(v) else v) for k, v in batch.items()}
        loader = A.DeviceCropLoader([batch], heatmap, 2)
        dev = loader.to_device(batch)
        out = torch.empty((B, 3, size[1], size[0]), device="cuda")
        norm = batch["norm"].numpy()

        def launch():
            ops.crop_affine_normalize(dev["pixels"], dev["desc"], dev["inv"], size, norm[:3], norm[3:],
                                      desc_host=batch["desc"], inv_host=batch["inv"], out=out)
        for _ in range(20):
            launch()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.iters):
            launch()
        e1.record()
        torch.cuda.synchronize()
        call_us = e0.elapsed_time(e1) * 1e3 / args.iters
        # device time of the kernel alone (the loop above also contains the host-side argument checks)
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.iters):
                launch()
            torch.cuda.synchronize()
        ks = [e for e in prof.key_averages() if "crop_affine_normalize" in e.key]
        kernel_us = sum(e.device_time_total for e in ks) / max(1, sum(e.count for e in ks))
        region_bytes = int(batch["pixels"].numel())
        out_bytes = out.numel() * 4
        moved = region_bytes + out_bytes + B * (7 + 6) * 8
        J, hw = 17, heatmap[0] * heatmap[1]
        h2d_new = (region_bytes + B * ((7 + 6) * 8 + 2 * J * 3 * 4)) / B
        h2d_ref = 3 * size[0] * size[1] * 4 + J * hw * 4 + J * 4
        # host time per sample: the worker's __getitem__ (decode excluded) against the reference's per-sample path
        np.random.seed(2)
        random.seed(2)
        n = args.host_samples
        t0 = time.perf_counter()
        for i in range(n):
            raw[i]
        new_ms = (time.perf_counter() - t0) * 1e3 / n
        ref_ms = sum(host_reference(ds, images, i)[0] for i in range(n)) * 1e3 / n
        result["workloads"].append({
            "batch": B, "out_hw": [size[1], size[0]], "kernel_us": round(kernel_us, 2), "call_us": round(call_us, 2),
            "bytes_moved": moved, "region_bytes": region_bytes, "out_bytes": out_bytes,
            "achieved_GBps": round(moved / (kernel_us * 1e-6) / 1e9, 1),
            "hbm_share": round(moved / (kernel_us * 1e-6) / HBM_BYTES_PER_S, 4),
            "h2d_bytes_per_sample": {"new": int(h2d_new), "reference": h2d_ref},
            "host_ms_per_sample": {"new_getitem": round(new_ms, 3), "reference_warp_totensor_target": round(ref_ms, 3)},
        })
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
