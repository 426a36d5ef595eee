"""The input crop's specification (oracle/augment_oracle.py) and host side (fpd_b200.augment) against the reference's
JointsDataset.__getitem__, recorded in tests/golden/augment.npz."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import fpd_b200  # noqa: E402,F401
from fpd_b200 import augment as A  # noqa: E402
from oracle import augment_oracle as O  # noqa: E402
import _augment_cases as C  # noqa: E402

G = C.golden()


def _clipped(img, inv, size):
    x0, y0, x1, y1 = A.source_window(inv, size, img.shape[1], img.shape[0])
    return img[y0:y1, x0:x1], (x0, y0)


def test_golden_covers_the_cases():
    n_flip = sum(int(G[t + "/flipped"].sum()) for t in C.sets(G))
    assert n_flip >= 5
    assert any(np.any(G[t + "/meta_rotation"] != 0) for t in C.sets(G))
    assert not G["eval_edges_bgr/crop"][4].any()      # the crop entirely outside its image
    sizes = {C.out_size(G, t) for t in C.sets(G)}
    assert {(48, 64), (192, 256), (256, 256)} <= sizes


@pytest.mark.parametrize("tag", C.sets(G))
def test_oracle_reproduces_golden_crops(tag):
    size = C.out_size(G, tag)
    for i in range(len(G[tag + "/crop"])):
        img = C.source(G, tag, i)
        got = O.warp_region(img, (0, 0), G[tag + "/inv"][i], size)
        np.testing.assert_array_equal(got, G[tag + "/crop"][i], err_msg="%s[%d]" % (tag, i))
        region, origin = _clipped(img, G[tag + "/inv"][i], size)
        np.testing.assert_array_equal(O.warp_region(region, origin, G[tag + "/inv"][i], size), G[tag + "/crop"][i])


def test_oracle_normalize_matches_golden_input():
    mean, std = G["mean"].astype(np.float32), G["std"].astype(np.float32)
    n = 0
    for tag in C.sets(G):
        if tag + "/input" not in G.files:
            continue
        for j, i in enumerate(G[tag + "/input_idx"]):
            got = O.normalize(G[tag + "/crop"][i], mean, std)
            assert got.dtype == np.float32
            np.testing.assert_array_equal(got, G[tag + "/input"][j])
            n += 1
    assert n >= 4


def test_clipped_region_equals_full_image_on_random_matrices():
    rng = np.random.RandomState(3)
    img = rng.randint(0, 256, (83, 117, 3)).astype(np.uint8)
    for _ in range(60):
        size = (int(rng.choice([16, 24, 48])), int(rng.choice([16, 32, 64])))
        a = rng.uniform(-2.5, 2.5, (2, 2))
        if abs(np.linalg.det(a)) < 0.05:
            continue
        b = rng.uniform(-60, 160, 2)
        inv = np.concatenate([a, b[:, None]], 1)
        full = O.warp_region(img, (0, 0), inv, size)
        region, origin = _clipped(img, inv, size)
        np.testing.assert_array_equal(O.warp_region(region, origin, inv, size), full)


def test_restated_inverse_equals_cv2():
    for tag in C.sets(G):
        for m, inv in zip(G[tag + "/trans"], G[tag + "/inv"]):
            np.testing.assert_array_equal(A.invert_affine(m), inv)


def test_float32_joints_give_the_reference_heatmap_centres():
    """The device targets take float32 joints; the reference rounds mu = int(x / stride + 0.5) in float64."""
    for tag in C.sets(G):
        c = C.cfg(G, tag)
        stride = np.array(c["image_size"], np.float64) / np.array(c["heatmap_size"], np.float64)
        j64 = G[tag + "/meta_joints"][..., :2]
        j32 = j64.astype(np.float32).astype(np.float64)
        np.testing.assert_array_equal((j64 / stride + 0.5).astype(np.int64), (j32 / stride + 0.5).astype(np.int64))


def _items(tag, paths):
    ds = A.RawJointsDataset(C.stand_in(G, tag, paths))
    C.seed(G, tag)
    return ds, [ds[i] for i in range(len(ds))]


@pytest.mark.parametrize("tag", C.sets(G))
def test_raw_dataset_reproduces_reference_draws(tag, tmp_path):
    pytest.importorskip("cv2")
    paths = C.write_images(G, tmp_path)
    ds, items = _items(tag, paths)
    np.testing.assert_array_equal(ds.mean, np.float32(G["mean"]))
    size = C.out_size(G, tag)
    for i, it in enumerate(items):
        meta = it["meta"]
        for key in ("center", "scale", "rotation", "score", "joints", "joints_vis"):
            np.testing.assert_array_equal(np.asarray(meta[key], np.float64), G[tag + "/meta_" + key][i],
                                          err_msg="%s[%d] %s" % (tag, i, key))
        np.testing.assert_array_equal(it["inv"], G[tag + "/inv"][i])
        np.testing.assert_array_equal(
            A.crop_matrix(meta["center"], meta["scale"], meta["rotation"], np.array(size)), G[tag + "/trans"][i])
        region, origin = _clipped(C.source(G, tag, i), it["inv"], size)
        np.testing.assert_array_equal(it["region"], region)
        assert it["region"].flags.c_contiguous and it["region"].dtype == np.uint8
        np.testing.assert_array_equal(it["desc"][1:3], origin)
        np.testing.assert_array_equal(O.warp_region(it["region"], it["desc"][1:3], it["inv"], size), G[tag + "/crop"][i])


def test_raw_dataset_refuses_other_transforms():
    ds = C.stand_in(G, "eval_rgb", ["x"] * 8)
    ds.transform = None
    with pytest.raises(ValueError):
        A.RawJointsDataset(ds)


def test_raw_collate_round_trips(tmp_path):
    pytest.importorskip("cv2")
    paths = C.write_images(G, tmp_path)
    _, items = _items("eval_edges_bgr", paths)
    batch = A.raw_collate(items)
    assert batch["pixels"].dtype == torch.uint8 and batch["pixels"].dim() == 1
    assert batch["desc"].shape == (len(items), 7) and batch["inv"].shape == (len(items), 6)
    assert batch["pixels"].numel() == sum(it["region"].size for it in items)
    for i, it in enumerate(items):
        off, rx, ry, rw, rh, iw, ih = batch["desc"][i].tolist()
        got = batch["pixels"][off:off + rw * rh * 3].numpy().reshape(rh, rw, 3)
        np.testing.assert_array_equal(got, it["region"])
        assert [rx, ry, iw, ih] == [it["desc"][1], it["desc"][2], it["desc"][5], it["desc"][6]]
        np.testing.assert_array_equal(batch["inv"][i].numpy().reshape(2, 3), it["inv"])
        np.testing.assert_array_equal(batch["joints"][i].numpy(), it["joints"].astype(np.float32))
        np.testing.assert_array_equal(batch["joints_vis"][i].numpy(), it["joints_vis"].astype(np.float32))
    assert batch["out_size"].tolist() == [48, 64]
    np.testing.assert_array_equal(batch["norm"].numpy(), np.concatenate([G["mean"], G["std"]]).astype(np.float32))
    assert batch["meta"]["center"].shape == (len(items), 2) and len(batch["meta"]["image"]) == len(items)
    assert not batch["desc"][4, 3:5].any()     # the crop outside its image reads nothing
