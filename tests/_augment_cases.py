"""Shared readers of tests/golden/augment.npz, which tests/golden/make_golden_augment.py makes from the reference's
JointsDataset."""
import json
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "augment.npz")


def golden():
    return np.load(GOLDEN)


def sets(g):
    return [str(s) for s in g["sets"]]


def cfg(g, tag):
    return json.loads(str(g[tag + "/cfg"]))


def out_size(g, tag):
    return tuple(cfg(g, tag)["image_size"])


def source(g, tag, i):
    """The image the reference warped for sample i: mirrored when it was flipped, RGB when COLOR_RGB is set."""
    img = g["img/%d" % int(g[tag + "/db_image"][i])]
    if g[tag + "/flipped"][i]:
        img = img[:, ::-1]
    if cfg(g, tag)["color_rgb"]:
        img = img[..., ::-1]
    return np.ascontiguousarray(img)


def samples(g):
    """(tag, index) of every golden sample."""
    return [(t, i) for t in sets(g) for i in range(len(g[t + "/crop"]))]


def db(g, tag, image_paths):
    """The set's db records (image k at image_paths[k])."""
    out = []
    for i, k in enumerate(g[tag + "/db_image"]):
        out.append({"image": image_paths[int(k)], "filename": "", "imgnum": 0,
                    "center": g[tag + "/db_center"][i].copy(), "scale": g[tag + "/db_scale"][i].copy(),
                    "joints_3d": g[tag + "/db_joints"][i].copy(), "joints_3d_vis": g[tag + "/db_joints_vis"][i].copy()})
    return out


def write_images(g, directory):
    """The golden source images as PNG files (lossless); returns their paths by index."""
    import cv2
    paths = []
    k = 0
    while "img/%d" % k in g.files:
        p = os.path.join(str(directory), "img%d.png" % k)
        assert cv2.imwrite(p, g["img/%d" % k])
        paths.append(p)
        k += 1
    return paths


def stand_in(g, tag, image_paths):
    from oracle.augment_oracle import StandInDataset
    return StandInDataset(cfg(g, tag), db(g, tag, image_paths))


def seed(g, tag):
    import random
    s = int(g[tag + "/seed"])
    np.random.seed(s)
    random.seed(s)
