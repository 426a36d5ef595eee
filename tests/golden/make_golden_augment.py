"""Generate tests/golden/augment.npz by running the REAL reference's JointsDataset.__getitem__ (/root/reference,
read-only) on seeded synthetic inputs. Run in the build container only:

    python tests/golden/make_golden_augment.py

The vectors pin the input crop: oracle/augment_oracle.py and csrc/augment.cu (tests/test_augment_cpu.py,
tests/test_augment_gpu.py).
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import NS, OUT, REF, load  # noqa: E402

COCO_FLIP = [[1, 2], [3, 4], [5, 6], [7, 8], [9, 10], [11, 12], [13, 14], [15, 16]]     # lib/dataset/coco.py:93-96
MPII_FLIP = [[0, 5], [1, 4], [2, 3], [10, 15], [11, 14], [12, 13]]                      # lib/dataset/mpii.py:31-35
AUGMENT_SETS = [   # tag, train, COLOR_RGB, IMAGE_SIZE (w, h), HEATMAP_SIZE, joints ("coco" / "mpii"), samples, seed, boxes
    ("train_bgr", True, False, (48, 64), (12, 16), "coco", 14, 11, "random"),
    ("train_rgb", True, True, (48, 64), (12, 16), "mpii", 10, 12, "random"),
    ("eval_edges_bgr", False, False, (48, 64), (12, 16), "coco", 10, 13, "edges"),
    ("eval_rgb", False, True, (48, 64), (12, 16), "mpii", 4, 14, "random"),
    ("train_256x192", True, True, (192, 256), (48, 64), "coco", 1, 15, "random"),
    ("train_256x256", True, False, (256, 256), (64, 64), "mpii", 1, 16, "random"),
    ("eval_256x256", False, True, (256, 256), (64, 64), "mpii", 1, 17, "random"),
]
# (h, w), pattern; (41, 37) is smaller than the crop. "smooth": sinusoids with sharp edges, every tap weight matters;
# "blocks": overlapping flat rectangles, whose crops compress well enough to keep the larger outputs in the file
AUGMENT_IMAGES = [((120, 160), "blocks"), ((97, 131), "blocks"), ((75, 53), "smooth"), ((41, 37), "smooth"),
                  ((150, 201), "blocks"), ((64, 64), "smooth"), ((173, 229), "blocks")]
BLOCK_IMAGES = [k for k, (_, kind) in enumerate(AUGMENT_IMAGES) if kind == "blocks"]


def main():
    """augment.npz: the reference's real JointsDataset.__getitem__ (lib/dataset/JointsDataset.py:113-198) on a subclass
    with a synthetic db over PNG images (lossless: the stored arrays are what imread returns), np.random / random seeded
    per set, cv2.warpAffine wrapped to record every forward matrix and uint8 crop. Covers train mode (flip, scale,
    rotation, half body) and eval mode, COLOR_RGB on and off, crops clipped at each border, entirely outside the image and
    enlarged, odd source sizes (one smaller than the crop), 64x48 outputs and a few at 256x192 / 256x256."""
    import json
    import random
    import tempfile
    import cv2
    import torchvision.transforms as T
    sys.path.insert(0, os.path.join(REF, "lib"))
    JD = load("ref_joints_dataset_aug", "lib/dataset/JointsDataset.py").JointsDataset
    rng = np.random.RandomState(21)
    save = {"cv2_version": np.array(cv2.__version__)}
    mean, std = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]     # tools/fpd_train.py:182-184
    save["mean"], save["std"] = np.array(mean), np.array(std)
    tmp = tempfile.mkdtemp()
    paths = []
    for k, ((h, w), pattern) in enumerate(AUGMENT_IMAGES):
        yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
        img = np.zeros((h, w, 3), np.float64)
        if pattern == "smooth":
            for c in range(3):
                f = rng.uniform(0.05, 0.4, 2)
                img[..., c] = 128 + 90 * np.sin(f[0] * xx + rng.uniform(0, 6)) * np.cos(f[1] * yy + rng.uniform(0, 6))
            img[(xx // 7 + yy // 5) % 4 == 0] += 40
        else:
            img[:] = rng.randint(0, 256, 3)
            for _ in range(30):
                x0, y0 = rng.randint(0, w), rng.randint(0, h)
                img[y0:y0 + rng.randint(3, h // 2), x0:x0 + rng.randint(3, w // 2)] = rng.randint(0, 256, 3)
        img = np.clip(img, 0, 255).astype(np.uint8)
        p = os.path.join(tmp, "img%d.png" % k)
        cv2.imwrite(p, img)
        back = cv2.imread(p, cv2.IMREAD_COLOR | cv2.IMREAD_IGNORE_ORIENTATION)
        assert np.array_equal(back, img)
        save["img/%d" % k] = back
        paths.append(p)

    rec = []
    warp = cv2.warpAffine

    def spy(src, M, dsize, **kw):
        out = warp(src, M, dsize, **kw)
        rec.append((M.copy(), out.copy(), src.strides[1] < 0))
        return out
    for tag, train, rgb, isz, hsz, kind, n, seed, boxes in AUGMENT_SETS:
        J = 17 if kind == "coco" else 16
        cfg = {"is_train": train, "color_rgb": rgb, "image_size": list(isz), "heatmap_size": list(hsz), "sigma": 2,
               "scale_factor": 0.35, "rotation_factor": 45, "flip": True, "num_joints_half_body": 8,
               "prob_half_body": 0.5, "num_joints": J, "flip_pairs": COCO_FLIP if kind == "coco" else MPII_FLIP,
               "upper_body_ids": list(range(11)) if kind == "coco" else [7, 8, 9, 10, 11, 12, 13, 14, 15],
               "mean": mean, "std": std}
        ref_cfg = NS(OUTPUT_DIR=tmp, DATASET=NS(DATA_FORMAT="png", SCALE_FACTOR=cfg["scale_factor"],
                                                ROT_FACTOR=cfg["rotation_factor"], FLIP=True, NUM_JOINTS_HALF_BODY=8,
                                                PROB_HALF_BODY=cfg["prob_half_body"], COLOR_RGB=rgb),
                     MODEL=NS(TARGET_TYPE="gaussian", IMAGE_SIZE=list(isz), HEATMAP_SIZE=list(hsz), SIGMA=2),
                     LOSS=NS(USE_DIFFERENT_JOINTS_WEIGHT=False))
        fdt = np.float32 if kind == "coco" else np.float64      # coco.py:228-238 / mpii.py:68-69
        aspect = isz[0] / isz[1]
        db = []
        for i in range(n):
            if boxes == "edges":
                k = [0, 1, 4, 6, 2, 3, 5, 0, 1, 4][i]
            elif isz == (48, 64):
                k = rng.randint(len(AUGMENT_IMAGES))
            else:
                k = BLOCK_IMAGES[rng.randint(len(BLOCK_IMAGES))]
            ih, iw = AUGMENT_IMAGES[k][0]
            bw = rng.uniform(0.3, 1.2) * min(iw, ih)
            c = np.array([rng.uniform(0.2, 0.8) * iw, rng.uniform(0.2, 0.8) * ih])
            if boxes == "edges":   # clipped at the left, right, top, bottom border; outside; enlarged; larger than the image
                c, bw = [(np.array([2.0, ih / 2]), 0.6 * ih), (np.array([iw - 3.0, ih / 2]), 0.6 * ih),
                         (np.array([iw / 2, 1.5]), 0.5 * iw), (np.array([iw / 2, ih - 0.5]), 0.5 * iw),
                         (np.array([-400.0, -300.0]), 30.0), (np.array([iw * 0.4, ih * 0.6]), 9.0),
                         (np.array([iw * 0.5, ih * 0.5]), 2.5 * max(iw, ih)), (np.array([iw * 0.7, ih * 0.3]), 14.0),
                         (np.array([0.0, 0.0]), 40.0), (np.array([iw + 5.0, ih + 4.0]), 40.0)][i]
            s = np.array([bw / 200.0, bw / aspect / 200.0], fdt) * 1.25
            joints = np.zeros((J, 3), np.float64)
            joints[:, 0] = c[0] + rng.uniform(-0.5, 0.5, J) * bw
            joints[:, 1] = c[1] + rng.uniform(-0.5, 0.5, J) * bw / aspect
            vis = np.zeros((J, 3), np.float64)
            vis[:, 0] = vis[:, 1] = (rng.rand(J) > (0.15 if i % 3 else 0.6)).astype(np.float64)
            joints *= vis
            db.append({"image": paths[k], "filename": "", "imgnum": 0, "center": np.array(c, fdt), "scale": s,
                       "joints_3d": joints, "joints_3d_vis": vis, "k": k})

        class Synthetic(JD):
            def __init__(self):
                super().__init__(ref_cfg, tmp, "synthetic", train,
                                 T.Compose([T.ToTensor(), T.Normalize(mean=mean, std=std)]))
                self.num_joints = J
                self.flip_pairs = cfg["flip_pairs"]
                self.upper_body_ids = tuple(cfg["upper_body_ids"])
                self.aspect_ratio = aspect
                self.db = [{kk: v for kk, v in d.items() if kk != "k"} for d in db]
        ds = Synthetic()
        np.random.seed(seed)
        random.seed(seed)
        rec.clear()
        cv2.warpAffine = spy
        try:
            items = [ds[i] for i in range(n)]
        finally:
            cv2.warpAffine = warp
        assert len(rec) == n
        p = tag + "/"
        save[p + "cfg"] = np.array(json.dumps(cfg))
        save[p + "seed"] = np.int64(seed)
        save[p + "db_image"] = np.array([d["k"] for d in db], np.int64)
        save[p + "db_center"] = np.stack([d["center"] for d in db])
        save[p + "db_scale"] = np.stack([d["scale"] for d in db])
        save[p + "db_joints"] = np.stack([d["joints_3d"] for d in db])
        save[p + "db_joints_vis"] = np.stack([d["joints_3d_vis"] for d in db])
        save[p + "trans"] = np.stack([m for m, _, _ in rec])
        save[p + "inv"] = np.stack([cv2.invertAffineTransform(m) for m, _, _ in rec])
        save[p + "crop"] = np.stack([o for _, o, _ in rec])
        save[p + "flipped"] = np.array([f for _, _, f in rec])
        save[p + "target"] = np.stack([it[1].numpy() for it in items])
        save[p + "target_weight"] = np.stack([it[2].numpy() for it in items])
        for key in ("joints", "joints_vis", "center", "scale", "rotation", "score"):
            save[p + "meta_" + key] = np.stack([np.asarray(it[3][key], np.float64) for it in items])
        if isz == (48, 64):   # the float input of a few samples
            save[p + "input_idx"] = np.arange(1)
            save[p + "input"] = np.stack([items[0][0].numpy()])
    save["sets"] = np.array([s[0] for s in AUGMENT_SETS])
    out = os.path.join(OUT, "augment.npz")
    np.savez_compressed(out, **save)
    print("augment.npz", os.path.getsize(out))

if __name__ == "__main__":
    main()
