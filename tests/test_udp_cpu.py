"""UDP (unbiased data processing, Huang et al., CVPR 2020) without a GPU: the crop matrix (augment.udp_crop_matrix)
against a closed-form fp64 model, its flip symmetry, the decode matrices (inverse_affines(..., udp=True)),
RawJointsDataset(udp=True) on a small synthetic dataset, an fp64 model of the targets (fpd_gaussian_targets_udp)
checked against itself, and the host-side checks of the new entry point. tests/test_udp_gpu.py holds the kernel to this
model."""
import ctypes
import os
import sys
import types

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

NS = types.SimpleNamespace


# ----------------------------------------------------------------------------------------------- fp64 models
def model_crop(center, scale, rot, size):
    """The UDP crop as a product of 3x3 matrices: translate the centre to 0, rotate by -rot (the reference's
    get_affine_transform turns the source box by +rot), scale by (size - 1) / (scale * 200), translate to the centre of
    the output's pixel-centre span."""
    c = np.asarray(center, np.float64)
    box = np.asarray(scale, np.float64) * 200.0
    t = np.deg2rad(rot)
    to0 = np.array([[1, 0, -c[0]], [0, 1, -c[1]], [0, 0, 1]], np.float64)
    turn = np.array([[np.cos(t), np.sin(t), 0], [-np.sin(t), np.cos(t), 0], [0, 0, 1]])
    scl = np.diag([(size[0] - 1) / box[0], (size[1] - 1) / box[1], 1.0])
    out = np.array([[1, 0, (size[0] - 1) / 2], [0, 1, (size[1] - 1) / 2], [0, 0, 1]], np.float64)
    return (out @ scl @ turn @ to0)[:2]


def apply(m, pts):
    pts = np.asarray(pts, np.float64).reshape(-1, 2)
    return pts @ m[:, :2].T + m[:, 2]


def udp_targets(joints, joints_vis, heatmap_size, image_size, sigma, joints_weight=None):
    """joints, joints_vis [N,J,3] -> (target [N,J,H,W], weight [N,J,1]) in float64: stride (image - 1) / (map - 1),
    centre mu = joint / stride unrounded, generate_target's window and visibility around int(mu + 0.5), the Gaussian
    on mu inside the window."""
    W, H = heatmap_size
    sx, sy = (image_size[0] - 1.0) / (W - 1), (image_size[1] - 1.0) / (H - 1)
    n, J = joints.shape[:2]
    tmp = 3 * sigma
    target = np.zeros((n, J, H, W))
    weight = np.zeros((n, J, 1))
    ys, xs = np.mgrid[0:H, 0:W].astype(np.float64)
    for i in range(n):
        for j in range(J):
            mx, my = np.float64(joints[i, j, 0]) / sx, np.float64(joints[i, j, 1]) / sy
            cx, cy = int(mx + 0.5), int(my + 0.5)
            v = np.float64(joints_vis[i, j, 0])
            if cx - tmp >= W or cy - tmp >= H or cx + tmp + 1 < 0 or cy + tmp + 1 < 0:
                v = 0.0
            elif v > 0.5:
                win = (np.abs(xs - cx) <= tmp) & (np.abs(ys - cy) <= tmp)
                g = np.exp(-((xs - mx) ** 2 + (ys - my) ** 2) / (2.0 * sigma * sigma))
                target[i, j] = np.where(win, g, 0.0)
            weight[i, j, 0] = v * (1.0 if joints_weight is None else joints_weight[j])
    return target, weight


def default_targets(joints, heatmap_size, image_size, sigma):
    """generate_target's map for visible joints: stride image / map, the Gaussian on the rounded centre."""
    W, H = heatmap_size
    n, J = joints.shape[:2]
    ys, xs = np.mgrid[0:H, 0:W]
    out = np.zeros((n, J, H, W))
    for i in range(n):
        for j in range(J):
            cx = int(joints[i, j, 0] / (image_size[0] / W) + 0.5)
            cy = int(joints[i, j, 1] / (image_size[1] / H) + 0.5)
            g = np.exp(-((xs - cx) ** 2 + (ys - cy) ** 2) / (2.0 * sigma * sigma))
            out[i, j] = np.where((np.abs(xs - cx) <= 3 * sigma) & (np.abs(ys - cy) <= 3 * sigma), g, 0.0)
    return out


def flip_joints(joints, image_w):
    """Mirrored crop coordinates x -> image_w - 1 - x (no joint-pair swap: a pure geometric mirror)."""
    f = joints.copy()
    f[..., 0] = (image_w - 1) - f[..., 0]
    return f


def flip_case(rng, n, J, image_size, heatmap_size):
    """Joints inside the crop, multiples of 1/256 px so that their float32 mirror is exact, none at a rounding tie of
    the window centre (where int(mu + 0.5) and its mirror round to different pixels)."""
    W = heatmap_size[0]
    sx = (image_size[0] - 1.0) / (W - 1)
    j = np.zeros((n, J, 3), np.float32)
    j[..., 0] = np.round(rng.uniform(0, image_size[0] - 1, (n, J)) * 256) / 256
    j[..., 1] = np.round(rng.uniform(0, image_size[1] - 1, (n, J)) * 256) / 256
    frac = (j[..., 0].astype(np.float64) / sx + 0.5) % 1.0
    j[..., 0] = np.where(np.minimum(frac, 1 - frac) < 1e-6, j[..., 0] + 1.0 / 64, j[..., 0])
    return j


# ----------------------------------------------------------------------------------------------- crop matrix
SIZES = [(192, 256), (256, 256), (288, 384), (48, 64)]


def _cases(seed=0, n=40):
    rng = np.random.RandomState(seed)
    for k in range(n):
        size = SIZES[k % len(SIZES)]
        c = rng.uniform(-50, 900, 2)
        s = rng.uniform(0.3, 4.0) * np.array([1.0, size[1] / size[0]])
        rot = 0.0 if k % 4 == 0 else rng.uniform(-80, 80)
        yield c, s, rot, size


def test_crop_matrix_matches_closed_form():
    from fpd_b200.augment import udp_crop_matrix
    for c, s, rot, size in _cases():
        m = udp_crop_matrix(c, s, rot, size)
        assert m.dtype == np.float64 and m.shape == (2, 3)
        np.testing.assert_allclose(m, model_crop(c, s, rot, size), rtol=0, atol=1e-12)
        np.testing.assert_allclose(apply(m, c), [[(size[0] - 1) / 2, (size[1] - 1) / 2]], rtol=0, atol=1e-12)


def test_crop_matrix_maps_box_edges_to_first_and_last_pixel_centres():
    from fpd_b200.augment import udp_crop_matrix
    for c, s, _, size in _cases(1):
        m = udp_crop_matrix(c, s, 0.0, size)
        half = s * 100.0
        edges = [c - half, c + half, [c[0] - half[0], c[1] + half[1]]]
        np.testing.assert_allclose(apply(m, edges), [[0, 0], [size[0] - 1, size[1] - 1], [0, size[1] - 1]],
                                   rtol=0, atol=1e-9)
    # a scalar scale stands for both axes, as in crop_matrix
    np.testing.assert_array_equal(udp_crop_matrix([10.0, 20.0], 1.5, 7.0, (48, 64)),
                                  udp_crop_matrix([10.0, 20.0], [1.5, 1.5], 7.0, (48, 64)))


def test_crop_matrix_rotates_like_the_reference():
    """The same rot turns the crop the same way as crop_matrix (cv2's solve of the reference's float32 points)."""
    pytest.importorskip("cv2")
    from fpd_b200.augment import crop_matrix, udp_crop_matrix
    for c, s, rot, size in _cases(2):
        s = np.array([s[0], s[0]])
        ref = crop_matrix(c, s, rot, np.array(size))
        udp = udp_crop_matrix(c, s, rot, size)
        # rows scaled to unit length: the rotations alone (UDP scales the two axes slightly differently)
        ref_rot = ref[:, :2] / np.linalg.norm(ref[:, :2], axis=1, keepdims=True)
        udp_rot = udp[:, :2] / np.linalg.norm(udp[:, :2], axis=1, keepdims=True)
        np.testing.assert_allclose(udp_rot, ref_rot, rtol=0, atol=1e-5)
        if rot != 0:
            assert abs(udp_rot[0, 1]) > 1e-3


def test_flip_symmetry_is_exact():
    """Mirroring the image (x -> width - 1 - x, the centre with it) and cropping gives the mirror x -> W - 1 - x of the
    unmirrored crop: exactly, in fp64, for dyadic inputs, and to 1e-12 for any. A rotated crop mirrors into the crop
    rotated the other way."""
    from fpd_b200.augment import udp_crop_matrix
    width = 640
    rng = np.random.RandomState(3)
    for size, box in (((192, 256), 256.0), ((256, 256), 512.0), ((48, 64), 64.0)):
        c = np.array([300.5, 211.25])
        s = np.array([box, box * size[1] / size[0]]) / 200.0
        pts = np.round(rng.uniform(-100, 700, (64, 2)) * 16) / 16
        a = apply(udp_crop_matrix(c, s, 0.0, size), pts)
        fc = np.array([width - 1 - c[0], c[1]])
        fp = np.stack([width - 1 - pts[:, 0], pts[:, 1]], 1)
        b = apply(udp_crop_matrix(fc, s, 0.0, size), fp)
        np.testing.assert_array_equal(b[:, 0], (size[0] - 1) - a[:, 0])
        np.testing.assert_array_equal(b[:, 1], a[:, 1])
    for c, s, rot, size in _cases(4):
        pts = rng.uniform(-100, 1000, (16, 2))
        a = apply(udp_crop_matrix(c, s, rot, size), pts)
        fc = np.array([width - 1 - c[0], c[1]])
        fp = np.stack([width - 1 - pts[:, 0], pts[:, 1]], 1)
        b = apply(udp_crop_matrix(fc, s, -rot, size), fp)
        np.testing.assert_allclose(b[:, 0], (size[0] - 1) - a[:, 0], rtol=0, atol=1e-12)
        np.testing.assert_allclose(b[:, 1], a[:, 1], rtol=0, atol=1e-12)


def test_decode_matrices_invert_crop_and_stride():
    """inverse_affines(udp=True) after the UDP crop and the heat-map stride (image - 1) / (map - 1) is the identity."""
    from fpd_b200.augment import udp_crop_matrix
    from fpd_b200.lib.core.inference import inverse_affines
    rng = np.random.RandomState(5)
    for size, hm in (((192, 256), (48, 64)), ((256, 256), (64, 64)), ((288, 384), (72, 96))):
        B = 8
        c = rng.uniform(0, 800, (B, 2))
        s = rng.uniform(0.3, 4.0, (B, 2))
        inv = inverse_affines(c, s, hm, udp=True)
        assert inv.shape == (B, 6) and inv.dtype == np.float64
        stride = (np.array(size, np.float64) - 1) / (np.array(hm, np.float64) - 1)
        for b in range(B):
            pts = rng.uniform(-200, 1000, (20, 2))
            in_hm = apply(udp_crop_matrix(c[b], s[b], 0.0, size), pts) / stride
            np.testing.assert_allclose(apply(inv[b].reshape(2, 3), in_hm), pts, rtol=0, atol=1e-9)
    # the default matrices are untouched by the new argument
    np.testing.assert_array_equal(inverse_affines(c, s, (48, 64)), inverse_affines(c, s, (48, 64), udp=False))


def test_get_final_preds_maps_through_udp_matrices(monkeypatch):
    """The eager decode: the same heat-map coordinates, mapped by the UDP matrices when TEST.UDP is set."""
    import torch
    from fpd_b200.lib.core import inference as I
    B, J, h, w = 3, 4, 16, 12
    rng = np.random.RandomState(6)
    idx = rng.randint(0, h * w, (B, J))
    mv = rng.uniform(0.1, 1, (B, J)).astype(np.float32)
    monkeypatch.setattr(I, "_device_argmax", lambda hm: (torch.from_numpy(idx), torch.from_numpy(mv)))
    c, s = rng.uniform(100, 400, (B, 2)), rng.uniform(0.5, 2, (B, 2))
    hm = torch.zeros(B, J, h, w)
    cfg = NS(TEST=NS(POST_PROCESS=False, UDP=True))
    preds, maxvals = I.get_final_preds(cfg, hm, c, s)
    coords, _ = I.preds_from_argmax(idx, mv, w)
    for b in range(B):
        want = c[b] - s[b] * 100 + coords[b].astype(np.float64) * s[b] * 200 / np.array([w - 1, h - 1])
        np.testing.assert_allclose(preds[b], want, rtol=0, atol=1e-4)
    np.testing.assert_array_equal(maxvals[..., 0], mv)
    plain, _ = I.get_final_preds(NS(TEST=NS(POST_PROCESS=False)), hm, c, s)
    assert not np.allclose(plain, preds)


# ----------------------------------------------------------------------------------------------- RawJointsDataset
def _synthetic(tmp_path, is_train, flip, n=6, size=(48, 64)):
    import cv2
    from oracle.augment_oracle import StandInDataset
    rng = np.random.RandomState(7 + int(is_train) + 2 * int(flip))
    paths = []
    for k in range(2):
        img = rng.randint(0, 256, (90 + 30 * k, 120 + 17 * k, 3)).astype(np.uint8)
        paths.append(os.path.join(str(tmp_path), "s%d.png" % k))
        assert cv2.imwrite(paths[-1], img)
    J = 16
    db = []
    for i in range(n):
        joints = np.zeros((J, 3))
        joints[:, 0] = rng.uniform(0, 120, J)
        joints[:, 1] = rng.uniform(0, 90, J)
        vis = np.zeros((J, 3))
        vis[:, :2] = (rng.rand(J) > 0.2)[:, None]
        db.append({"image": paths[i % 2], "filename": "", "imgnum": i,
                   "center": np.array([rng.uniform(30, 90), rng.uniform(20, 70)]),
                   "scale": np.array([rng.uniform(0.2, 0.6), 0.0]), "joints_3d": joints, "joints_3d_vis": vis})
        db[-1]["scale"][1] = db[-1]["scale"][0] * size[1] / size[0]
    cfg = dict(is_train=is_train, color_rgb=True, image_size=list(size), heatmap_size=[size[0] // 4, size[1] // 4],
               sigma=2, scale_factor=0.35, rotation_factor=45, flip=flip, num_joints_half_body=8, prob_half_body=0.0,
               num_joints=J, flip_pairs=[[0, 5], [1, 4], [2, 3], [10, 15], [11, 14], [12, 13]],
               upper_body_ids=list(range(7, 16)), mean=[0.485, 0.456, 0.406], std=[0.229, 0.224, 0.225])
    return StandInDataset(cfg, db)


@pytest.mark.parametrize("is_train,flip", [(False, False), (True, False), (True, True)])
def test_raw_dataset_udp_items(tmp_path, is_train, flip):
    pytest.importorskip("cv2")
    import cv2
    from fpd_b200 import augment as A
    from oracle import augment_oracle as O
    base = _synthetic(tmp_path, is_train, flip)
    ds = A.RawJointsDataset(base, udp=True)
    assert not A.RawJointsDataset(base).udp
    np.random.seed(0)
    import random
    random.seed(0)
    size = ds.image_size
    flipped_any = rotated_any = False
    for i in range(len(ds)):
        it = ds[i]
        meta, rec = it["meta"], base.db[i]
        img = cv2.imread(rec["image"], cv2.IMREAD_COLOR)
        flipped = bool(meta["center"][0] != rec["center"][0])
        flipped_any |= flipped
        rotated_any |= meta["rotation"] != 0
        if flipped:
            assert meta["center"][0] == img.shape[1] - rec["center"][0] - 1
        trans = A.udp_crop_matrix(meta["center"], meta["scale"], meta["rotation"], size)
        np.testing.assert_array_equal(it["inv"], A.invert_affine(trans))
        # the joints went through the item's own matrix (mirrored first, pairs swapped, when flipped)
        src, src_vis = rec["joints_3d"].copy(), rec["joints_3d_vis"].copy()
        if flipped:
            src, src_vis = A._flip_joints(src, src_vis, img.shape[1], base.flip_pairs)
        vis = src_vis[:, 0] > 0
        np.testing.assert_array_equal(it["joints_vis"], src_vis)
        np.testing.assert_allclose(it["joints"][vis, :2], apply(trans, src[vis, :2]), rtol=0, atol=1e-9)
        np.testing.assert_array_equal(it["joints"][~vis, :2], src[~vis, :2])
        # the region holds every pixel the crop reads, and the crop equals cv2.warpAffine with the UDP matrix
        mirrored = img[:, ::-1] if flipped else img
        mirrored = np.ascontiguousarray(mirrored[..., ::-1])                    # COLOR_RGB
        full = O.warp_region(mirrored, (0, 0), it["inv"], size)
        np.testing.assert_array_equal(O.warp_region(it["region"], it["desc"][1:3], it["inv"], size), full)
        np.testing.assert_array_equal(full, cv2.warpAffine(mirrored, trans, (int(size[0]), int(size[1])),
                                                           flags=cv2.INTER_LINEAR))
    assert flipped_any == flip and rotated_any == is_train


# ----------------------------------------------------------------------------------------------- the target model
def test_model_targets_window_and_visibility():
    W, H, img = 48, 64, (192, 256)
    sx, sy = (img[0] - 1) / (W - 1), (img[1] - 1) / (H - 1)
    # window centre int(mu + 0.5), truncated toward zero: -7.4 -> -6, window -12..0, in; -8.6 -> -8, out; 53.4 -> 53,
    # in; 53.55 -> 54, out. -8.4 -> -7: the window ends at x = -1, yet generate_target's rule (br < 0) keeps weight 1
    mus = [(-7.4, 20.0), (-8.6, 20.0), (10.0, 10.0), (53.4, 8.0), (53.55, 8.0), (10.0, -8.6), (10.0, 69.4),
           (-8.4, 20.0)]
    joints = np.array([[[mx * sx, my * sy, 0] for mx, my in mus]])
    vis = np.ones((1, len(mus), 3))
    vis[0, 2] = 0
    t, w = udp_targets(joints, vis, (W, H), img, 2)
    assert w[0, :, 0].tolist() == [1, 0, 0, 1, 0, 0, 1, 1]
    assert [bool(t[0, k].any()) for k in range(len(mus))] == [True, False, False, True, False, False, True, False]
    # an interior joint: 13 x 13 support around the rounded centre, the peak value exp(-d^2 / 8) at the nearest pixel
    j = np.array([[[20.3 * sx, 30.8 * sy, 0]]])
    t, _ = udp_targets(j, np.ones((1, 1, 3)), (W, H), img, 2)
    ys, xs = np.nonzero(t[0, 0])
    assert (xs.min(), xs.max(), ys.min(), ys.max()) == (14, 26, 25, 37)
    assert np.isclose(t[0, 0].max(), np.exp(-(0.3 ** 2 + 0.2 ** 2) / 8))


@pytest.mark.parametrize("image_size,heatmap_size", [((256, 256), (64, 64)), ((192, 256), (48, 64))])
def test_model_flip_consistency(image_size, heatmap_size):
    """The UDP target of the mirrored joints is the mirror of the target; the default target is off by a pixel."""
    rng = np.random.RandomState(8)
    j = flip_case(rng, 2, 17, image_size, heatmap_size)
    vis = np.ones_like(j)
    t, _ = udp_targets(j, vis, heatmap_size, image_size, 2)
    tf, _ = udp_targets(flip_joints(j, image_size[0]), vis, heatmap_size, image_size, 2)
    assert np.abs(tf - t[..., ::-1]).max() < 1e-12
    d = default_targets(j, heatmap_size, image_size, 2)
    df = default_targets(flip_joints(j, image_size[0]), heatmap_size, image_size, 2)
    assert np.abs(df - d[..., ::-1]).max() > 0.1


def _model_round_trip(decode, margin, n=200):
    rng = np.random.RandomState(9)
    W, H = 48, 64
    mu = np.stack([rng.uniform(margin, W - 1 - margin, n), rng.uniform(margin, H - 1 - margin, n)], 1)
    j = np.concatenate([mu, np.zeros((n, 1))], 1)[None]
    t, _ = udp_targets(j, np.ones_like(j), (W, H), (W, H), 2)
    return max(np.abs(np.array(decode(t[0, k])) - mu[k]).max() for k in range(n))


def test_model_round_trip():
    """The UDP target's arg-max is the pixel nearest the joint, so the quarter-pixel nudge lands within 0.25 px. DARK's
    decode recovers the joint to 0.01 px from 4 px inside the border on, although the target stops at 3 sigma."""
    import test_dark_cpu as D
    assert _model_round_trip(D.quarter_decode, 2) <= 0.25 + 1e-12
    assert _model_round_trip(D.dark_decode, 4) < 0.01


# ----------------------------------------------------------------------------------------------- entry point, options
def test_ctypes_entry_exists():
    import fpd_b200  # noqa: F401
    from fpd_b200 import _native as N
    assert N.lib().fpd_gaussian_targets_udp.argtypes == N._SIGNATURES["fpd_gaussian_targets_udp"][1]


@pytest.mark.parametrize("null_at, sizes, message", [
    (0, (1, 17, 64, 48, 192, 256, 2), "gaussian_targets_udp: null pointer"),
    (4, (1, 17, 64, 48, 192, 256, 2), "gaussian_targets_udp: null pointer"),
    (None, (1, 17, 64, 48, 192, 256, 0), "gaussian_targets_udp: bad sizes"),
    (None, (1, 17, 1, 48, 192, 256, 2), "gaussian_targets_udp: bad sizes"),
    (None, (1, 17, 64, 48, 1, 256, 2), "gaussian_targets_udp: bad sizes"),
    (None, (-1, 17, 64, 48, 192, 256, 2), "gaussian_targets_udp: bad sizes"),
])
def test_gaussian_targets_udp_host_checks(null_at, sizes, message):
    import fpd_b200  # noqa: F401
    from fpd_b200 import _native as N
    ptrs = [ctypes.c_void_p(16)] * 5
    ptrs[2] = None                  # joints_weight is optional
    if null_at is not None:
        ptrs[null_at] = None
    assert N.lib().fpd_gaussian_targets_udp(*ptrs, *sizes, None) == -1
    assert N.last_error() == message


def test_options_default_off_and_exclusive():
    import fpd_b200  # noqa: F401
    from fpd_b200.augment import DeviceCropLoader
    from fpd_b200.lib.core.inference import use_udp
    from fpd_b200.targets import TargetGenerator
    assert not use_udp(NS(TEST=NS(POST_PROCESS=True)))
    assert use_udp(NS(TEST=NS(POST_PROCESS=True, UDP=True)))
    assert use_udp(NS(TEST=NS(POST_PROCESS=False, UDP=True)))      # the matrices apply to the raw arg-max as well
    with pytest.raises(ValueError, match="two different target encodings"):
        TargetGenerator((192, 256), (48, 64), 2, unbiased=True, udp=True)
    with pytest.raises(ValueError, match="two different target encodings"):
        DeviceCropLoader([], (48, 64), 2, unbiased=True, udp=True)
    g = TargetGenerator((192, 256), (48, 64), 2, device="cpu")
    assert not g.udp and not g.unbiased
