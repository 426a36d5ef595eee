"""Generate tests/golden/unlabeled.npz by running the REAL reference's JointsDataset.__getitem__ (/root/reference,
read-only) on training records without keypoints (joints_3d_vis all zero: unlabeled person boxes) mixed with labeled
ones. Run in the build container only:

    python tests/golden/make_golden_unlabeled.py

The file has augment.npz's layout (tests/_augment_cases.py reads both), plus <set>/db_score. It pins
fpd_b200.augment.RawJointsDataset on such records: no half-body draw for a zero-visibility record, the same draws
otherwise, the same matrices and joints (tests/test_unlabeled_kd_cpu.py).
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import NS, OUT, REF, load  # noqa: E402
from make_golden_augment import COCO_FLIP, MPII_FLIP  # noqa: E402

SETS = [   # tag, COLOR_RGB, joints, samples, seed
    ("unlabeled_coco_bgr", False, "coco", 10, 31),
    ("unlabeled_mpii_rgb", True, "mpii", 8, 32),
]
IMAGES = [(97, 131), (75, 53)]
IMAGE_SIZE, HEATMAP_SIZE = (48, 64), (12, 16)


def main():
    """Every other record is unlabeled (zero joints and visibility, a detection score); the labeled records have most
    joints visible, so the half-body draw runs for them and the draw sequence interleaves both kinds."""
    import json
    import random
    import tempfile
    import cv2
    import torchvision.transforms as T
    sys.path.insert(0, os.path.join(REF, "lib"))
    JD = load("ref_joints_dataset_unlabeled", "lib/dataset/JointsDataset.py").JointsDataset
    rng = np.random.RandomState(41)
    save = {"cv2_version": np.array(cv2.__version__)}
    mean, std = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
    save["mean"], save["std"] = np.array(mean), np.array(std)
    tmp = tempfile.mkdtemp()
    paths = []
    for k, (h, w) in enumerate(IMAGES):
        img = np.zeros((h, w, 3), np.uint8)
        img[:] = rng.randint(0, 256, 3)
        for _ in range(20):
            x0, y0 = rng.randint(0, w), rng.randint(0, h)
            img[y0:y0 + rng.randint(3, h // 2), x0:x0 + rng.randint(3, w // 2)] = rng.randint(0, 256, 3)
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
    for tag, rgb, kind, n, seed in SETS:
        J = 17 if kind == "coco" else 16
        cfg = {"is_train": True, "color_rgb": rgb, "image_size": list(IMAGE_SIZE), "heatmap_size": list(HEATMAP_SIZE),
               "sigma": 2, "scale_factor": 0.35, "rotation_factor": 45, "flip": True, "num_joints_half_body": 8,
               "prob_half_body": 0.5, "num_joints": J, "flip_pairs": COCO_FLIP if kind == "coco" else MPII_FLIP,
               "upper_body_ids": list(range(11)) if kind == "coco" else [7, 8, 9, 10, 11, 12, 13, 14, 15],
               "mean": mean, "std": std}
        ref_cfg = NS(OUTPUT_DIR=tmp, DATASET=NS(DATA_FORMAT="png", SCALE_FACTOR=cfg["scale_factor"],
                                                ROT_FACTOR=cfg["rotation_factor"], FLIP=True, NUM_JOINTS_HALF_BODY=8,
                                                PROB_HALF_BODY=cfg["prob_half_body"], COLOR_RGB=rgb),
                     MODEL=NS(TARGET_TYPE="gaussian", IMAGE_SIZE=list(IMAGE_SIZE), HEATMAP_SIZE=list(HEATMAP_SIZE),
                              SIGMA=2),
                     LOSS=NS(USE_DIFFERENT_JOINTS_WEIGHT=False))
        fdt = np.float32 if kind == "coco" else np.float64
        aspect = IMAGE_SIZE[0] / IMAGE_SIZE[1]
        db = []
        for i in range(n):
            k = rng.randint(len(IMAGES))
            ih, iw = IMAGES[k]
            bw = rng.uniform(0.3, 1.2) * min(iw, ih)
            c = np.array([rng.uniform(0.2, 0.8) * iw, rng.uniform(0.2, 0.8) * ih])
            s = np.array([bw / 200.0, bw / aspect / 200.0], fdt) * 1.25
            joints = np.zeros((J, 3), np.float64)
            vis = np.zeros((J, 3), np.float64)
            score = 1.0
            if i % 2:
                joints[:, 0] = c[0] + rng.uniform(-0.5, 0.5, J) * bw
                joints[:, 1] = c[1] + rng.uniform(-0.5, 0.5, J) * bw / aspect
                vis[:, 0] = vis[:, 1] = (rng.rand(J) > 0.1).astype(np.float64)
                joints *= vis
            else:
                score = float(rng.uniform(0.3, 1.0))
            db.append({"image": paths[k], "filename": "", "imgnum": 0, "center": np.array(c, fdt), "scale": s,
                       "score": score, "joints_3d": joints, "joints_3d_vis": vis, "k": k})

        class Synthetic(JD):
            def __init__(self):
                super().__init__(ref_cfg, tmp, "synthetic", True,
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
        save[p + "db_score"] = np.array([d["score"] for d in db], np.float64)
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
    save["sets"] = np.array([s[0] for s in SETS])
    out = os.path.join(OUT, "unlabeled.npz")
    np.savez_compressed(out, **save)
    print("unlabeled.npz", os.path.getsize(out))


if __name__ == "__main__":
    main()
