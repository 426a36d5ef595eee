"""UDP on the device: fpd_gaussian_targets_udp against the fp64 model of tests/test_udp_cpu.py, the crop kernel on UDP
matrices against cv2.warpAffine + ToTensor + Normalize, flip consistency, the round trip through targets and both
decodes, validate() with TEST.UDP (graph route equal to the eager route, bit for bit), and a UDP training batch through
FPDTrainStep."""
import os
import sys
import types

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
NS = types.SimpleNamespace
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
import test_udp_cpu as M  # noqa: E402

SHAPES = [((48, 64), (192, 256), 2), ((64, 64), (256, 256), 2), ((72, 96), (288, 384), 3)]


def _target_joints(rng, n, J, hm_size, img_size, sigma):
    """Random joints (some far outside), joints 0-4 px from each border of the map, windows just inside and just outside
    it, in image units; some joints invisible."""
    W, H = hm_size
    sx, sy = (img_size[0] - 1.0) / (W - 1), (img_size[1] - 1.0) / (H - 1)
    mu = np.stack([rng.uniform(-12, W + 12, (n, J)), rng.uniform(-12, H + 12, (n, J))], -1)
    t = 3 * sigma
    edge = []
    for d in (0.0, 0.3, 1.0, 1.7, 2.5, 3.0, 3.6, 4.0):
        edge += [(d, H / 2 + d), (W - 1 - d, H / 2 - d), (W / 2 + d, d), (W / 2 - d, H - 1 - d)]
    # window centre int(mu + 0.5), truncated toward zero: the last centre generate_target's rule keeps, and the first it
    # drops, on each side
    edge += [(-t - 2.4, 10.2), (-t - 2.6, 10.2), (W - 1 + t + 0.4, 10.2), (W - 1 + t + 0.55, 10.2),
             (10.2, -t - 2.4), (10.2, -t - 2.6), (10.2, H - 1 + t + 0.4), (10.2, H - 1 + t + 0.55)]
    edge = np.array(edge)
    for k in range(0, len(edge), J):
        part = edge[k:k + J]
        mu[k // J, :len(part)] = part
    j = np.zeros((n, J, 3), np.float32)
    j[..., 0] = mu[..., 0] * sx
    j[..., 1] = mu[..., 1] * sy
    vis = (rng.rand(n, J, 3) > 0.15).astype(np.float32)
    vis[:(len(edge) + J - 1) // J] = 1
    return j, vis, len(edge)


@pytest.mark.parametrize("hm_size,img_size,sigma", SHAPES)
@pytest.mark.parametrize("use_w", [False, True])
def test_targets_match_fp64_model(hm_size, img_size, sigma, use_w):
    import fpd_b200  # noqa: F401
    from fpd_b200 import ops
    rng = np.random.RandomState(sigma + hm_size[0] + int(use_w))
    n, J = 8, 17
    joints, vis, n_edge = _target_joints(rng, n, J, hm_size, img_size, sigma)
    jw = rng.uniform(0.5, 1.5, J).astype(np.float32) if use_w else None
    jd, vd = torch.from_numpy(joints).cuda(), torch.from_numpy(vis).cuda()
    jwd = None if jw is None else torch.from_numpy(jw)
    t, w = ops.gaussian_targets_udp(jd, vd, hm_size, img_size, sigma, jwd)
    rt, rw = M.udp_targets(joints, vis, hm_size, img_size, sigma, jw)
    err = np.abs(t.cpu().numpy() - rt).max()
    assert err < 1e-6, err
    assert np.array_equal(w.cpu().numpy(), rw.astype(np.float32))
    flat = rw[..., 0].reshape(-1)
    assert (flat[n_edge - 8:n_edge] > 0).tolist() == [True, False] * 4      # the windows just in and just out
    assert (rw == 0).any() and (rw > 0).any() and (vis[..., 0] == 0).any()
    # deterministic: a second run and a graph replay give the same bits
    t2, w2 = ops.gaussian_targets_udp(jd, vd, hm_size, img_size, sigma, jwd)
    assert torch.equal(t, t2) and torch.equal(w, w2)
    jw_dev = None if jwd is None else jwd.cuda()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.gaussian_targets_udp(jd, vd, hm_size, img_size, sigma, jw_dev)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        tg, wg = ops.gaussian_targets_udp(jd, vd, hm_size, img_size, sigma, jw_dev)
    tg.fill_(7.0)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(tg, t) and torch.equal(wg, w)


def test_crop_on_udp_matrices_equals_cv2_warp_to_tensor_normalize():
    import cv2
    from torchvision import transforms as T
    from fpd_b200 import augment as A
    from fpd_b200 import ops
    mean, std = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
    norm = T.Compose([T.ToTensor(), T.Normalize(mean, std)])
    rng = np.random.RandomState(12)
    items, want = [], []
    for k in range(16):
        size = M.SIZES[k % 3]
        h, w = int(rng.randint(60, 500)), int(rng.randint(60, 500))
        img = rng.randint(0, 256, (h, w, 3)).astype(np.uint8)
        c = np.array([rng.uniform(-0.2, 1.2) * w, rng.uniform(-0.2, 1.2) * h])
        s = rng.uniform(0.2, 3.0) * np.array([1.0, size[1] / size[0]])
        rot = 0.0 if k % 4 == 0 else rng.uniform(-60, 60)
        trans = A.udp_crop_matrix(c, s, rot, size)
        inv = A.invert_affine(trans)
        x0, y0, x1, y1 = A.source_window(inv, size, w, h)
        region = np.ascontiguousarray(img[y0:y1, x0:x1])
        desc = np.array([0, x0, y0, region.shape[1], region.shape[0], w, h], np.int64)
        z = np.zeros((1, 3))
        items.append({"region": region, "desc": desc, "inv": inv, "joints": z, "joints_vis": z, "out_size": size,
                      "mean": np.float32(mean), "std": np.float32(std), "meta": {"i": k}})
        want.append(norm(cv2.warpAffine(img, trans, size, flags=cv2.INTER_LINEAR)))
    by_size = {}
    for it, wt in zip(items, want):
        by_size.setdefault(it["out_size"], []).append((it, wt))
    for size, group in by_size.items():
        batch = A.raw_collate([it for it, _ in group])
        dev = {key: batch[key].cuda() for key in ("pixels", "desc", "inv")}
        out = ops.crop_affine_normalize(dev["pixels"], dev["desc"], dev["inv"], size, np.float32(mean), np.float32(std),
                                        desc_host=batch["desc"], inv_host=batch["inv"]).cpu()
        for i, (_, wt) in enumerate(group):
            assert torch.equal(out[i], wt), (size, i)


@pytest.mark.parametrize("img_size,hm_size", [((256, 256), (64, 64)), ((192, 256), (48, 64))])
def test_flip_consistency(img_size, hm_size):
    """The UDP target of the mirrored joints (x -> image_w - 1 - x) is the mirror of the target. The default target is
    not: its stride image / map puts the mirrored centre up to a pixel away, the bias UDP removes."""
    from fpd_b200 import ops
    rng = np.random.RandomState(13)
    j = M.flip_case(rng, 8, 17, img_size, hm_size)
    vis = torch.ones(8, 17, 3, device="cuda")
    jd, jf = torch.from_numpy(j).cuda(), torch.from_numpy(M.flip_joints(j, img_size[0])).cuda()
    t, _ = ops.gaussian_targets_udp(jd, vis, hm_size, img_size, 2)
    tf, _ = ops.gaussian_targets_udp(jf, vis, hm_size, img_size, 2)
    udp_err = (tf - t.flip(3)).abs().max().item()
    d, _ = ops.gaussian_targets(jd, vis, hm_size, img_size, 2)
    df, _ = ops.gaussian_targets(jf, vis, hm_size, img_size, 2)
    default_err = (df - d.flip(3)).abs().max().item()
    print("flip consistency: UDP %.3g, default %.3g" % (udp_err, default_err))
    assert udp_err < 1e-7
    assert default_err > 0.1


def _round_trip_case(rng, B, J, img_size, hm_size, margin):
    """Image-space joints whose heat-map position is at least `margin` px inside the map, the crop-space joints the UDP
    crop (rot 0) makes of them, and the per-sample centres, scales and heat-map units."""
    from fpd_b200.augment import udp_crop_matrix
    W, H = hm_size
    c = rng.uniform(150, 450, (B, 2))
    s = rng.uniform(0.8, 2.5, (B, 1)) * np.array([[1.0, img_size[1] / img_size[0]]])
    mu = np.stack([rng.uniform(margin, W - 1 - margin, (B, J)), rng.uniform(margin, H - 1 - margin, (B, J))], -1)
    stride = (np.array(img_size, np.float64) - 1) / (np.array(hm_size, np.float64) - 1)
    crop = np.zeros((B, J, 3), np.float32)
    img_pts = np.zeros((B, J, 2))
    for b in range(B):
        m = udp_crop_matrix(c[b], s[b], 0.0, img_size)
        q = mu[b] * stride
        crop[b, :, :2] = q
        img_pts[b] = (q - m[:, 2]) @ np.linalg.inv(m[:, :2]).T
    unit = s * 200.0 / (np.array(hm_size, np.float64) - 1)          # image px per heat-map px, per axis
    return crop, img_pts, c, s, unit


def test_round_trip_through_targets_and_decodes():
    from fpd_b200.lib.core.inference import get_final_preds
    from fpd_b200.targets import TargetGenerator
    rng = np.random.RandomState(14)
    B, J = 16, 17
    img_size, hm_size = (192, 256), (48, 64)
    crop, img_pts, c, s, unit = _round_trip_case(rng, B, J, img_size, hm_size, 4.0)
    target, tw = TargetGenerator(img_size, hm_size, 2, udp=True)(crop, np.ones_like(crop))
    assert torch.all(tw == 1)
    errs = {}
    for name, dark in (("dark", True), ("quarter", False)):
        cfg = NS(TEST=NS(POST_PROCESS=True, DARK=dark, UDP=True))
        preds, _ = get_final_preds(cfg, target, c, s)
        errs[name] = (np.abs(preds - img_pts) / unit[:, None, :]).max()
    cfg = NS(TEST=NS(POST_PROCESS=True, DARK=True))
    preds, _ = get_final_preds(cfg, target, c, s)
    errs["dark, default matrices"] = (np.abs(preds - img_pts) / unit[:, None, :]).max()
    print("round trip, max error in heat-map px: " + ", ".join("%s %.4g" % kv for kv in errs.items()))
    assert errs["dark"] < 1e-2
    assert errs["quarter"] <= 0.25 + 1e-4
    assert errs["dark, default matrices"] > 0.1


# ----------------------------------------------------------------------------------------------- validate()
FLIP_PAIRS = [[0, 5], [1, 4], [2, 3], [10, 15], [11, 14], [12, 13]]


@pytest.fixture(scope="module")
def hourglass():
    import fpd_b200  # noqa: F401
    from fpd_b200.lib.models import hourglass as H
    torch.manual_seed(11)
    net = H.get_pose_net(NS(MODEL=NS(EXTRA=NS(NUM_FEATURES=64, NUM_STACKS=2, NUM_BLOCKS=1), NUM_JOINTS=16)), True)
    for mod in net.modules():
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.running_mean.normal_(0, 0.1)
            mod.running_var.uniform_(0.5, 1.5)
    return net.cuda()


def _batch(B, seed):
    from bench import synthetic_batch
    x, t, w = synthetic_batch(B, seed, 128, 128, 16)
    rng = np.random.RandomState(seed)
    meta = {"center": torch.from_numpy(rng.uniform(100, 500, (B, 2))),
            "scale": torch.from_numpy(rng.uniform(0.5, 3, (B, 2))),
            "score": torch.from_numpy(rng.uniform(0.5, 1, B)), "image": ["img%d_%d" % (seed, b) for b in range(B)]}
    return x, t, w, meta


class _ValSet:
    def __init__(self, n):
        self.n, self.flip_pairs, self.seen = n, FLIP_PAIRS, None

    def __len__(self):
        return self.n

    def evaluate(self, cfg, preds, output_dir, all_boxes, image_path, filenames, imgnums):
        self.seen = preds.copy()
        return {"Mean": float(preds[..., :2].mean())}, float(preds[..., :2].mean())


class _Writer:
    def __init__(self):
        self.scalars = []

    def add_scalar(self, tag, v, step):
        self.scalars.append((tag, v, step))

    def add_scalars(self, tag, d, step):
        pass


@pytest.mark.parametrize("flip", [True, False])
def test_validate_udp_graph_route_equals_eager_route(hourglass, flip, monkeypatch):
    from fpd_b200.lib.core import function as F
    from fpd_b200.lib.core.loss import JointsMSELoss
    loader = [_batch(3, 30), _batch(3, 31), _batch(2, 32)]
    seen = {}
    for udp, dark in ((True, False), (True, True), (False, False)):
        for graph in (True, False):
            monkeypatch.setattr(F, "_VALIDATE_GRAPH", graph)
            # UDP configs turn SHIFT_HEATMAP off: the flipped map already lines up
            cfg = NS(MODEL=NS(NUM_JOINTS=16, NAME="hourglass"), PRINT_FREQ=2, DEBUG=NS(DEBUG=False),
                     TEST=NS(FLIP_TEST=flip, SHIFT_HEATMAP=not udp, POST_PROCESS=True, DARK=dark, UDP=udp))
            ds = _ValSet(8)
            wd = {"writer": _Writer(), "valid_global_steps": 0}
            perf = F.validate(cfg, loader, ds, hourglass, JointsMSELoss(True), "/tmp", "/tmp", wd)
            seen[udp, dark, graph] = (perf, ds.seen, wd["writer"].scalars)
        (pg, sg, wg), (pe, se, we) = seen[udp, dark, True], seen[udp, dark, False]
        assert np.array_equal(sg, se) and pg == pe
        assert wg == we and {t for t, _, _ in wg} == {"valid_loss", "valid_acc"}
    assert not np.array_equal(seen[True, False, True][1], seen[False, False, True][1])
    assert not np.array_equal(seen[True, False, True][1], seen[True, True, True][1])
    if not flip:
        # without the flip test SHIFT_HEATMAP plays no part, so both configs decode the same heat-map coordinates: the
        # UDP predictions are the default ones taken back to the map and mapped by UDP's matrices
        from fpd_b200.lib.core.inference import inverse_affines
        base = seen[False, False, True][1][..., :2].astype(np.float64)
        c = np.concatenate([m["center"].numpy() for _, _, _, m in loader])
        s = np.concatenate([m["scale"].numpy() for _, _, _, m in loader])
        d = inverse_affines(c, s, [32, 32]).reshape(-1, 2, 3)
        u = inverse_affines(c, s, [32, 32], udp=True).reshape(-1, 2, 3)
        hm = np.stack([np.linalg.solve(d[b, :, :2], (base[b] - d[b, :, 2]).T).T for b in range(len(d))])
        want = np.einsum("bij,bkj->bki", u[:, :, :2], hm) + u[:, None, :, 2]
        np.testing.assert_allclose(seen[True, False, True][1][..., :2], want, rtol=0, atol=2e-3)


# ----------------------------------------------------------------------------------------------- training
def test_device_crop_loader_udp_batch_through_fpd_train_step(tmp_path):
    pytest.importorskip("cv2")
    from fpd_b200 import augment as A
    from fpd_b200 import ops
    from fpd_b200.lib.models import hourglass as H
    from fpd_b200.train_step import FPDTrainStep
    base = M._synthetic(tmp_path, True, True, n=4, size=(64, 64))
    np.random.seed(1)
    import random
    random.seed(1)
    loader = torch.utils.data.DataLoader(A.RawJointsDataset(base, udp=True), batch_size=4, shuffle=False,
                                         num_workers=0, collate_fn=A.raw_collate, pin_memory=True)
    dl = A.DeviceCropLoader(loader, base.heatmap_size, base.sigma, udp=True)
    batch = next(iter(dl.loader))
    x, target, tw, meta = dl.process(batch)
    want_t, want_w = ops.gaussian_targets_udp(batch["joints"].cuda(), batch["joints_vis"].cuda(), (16, 16), (64, 64), 2)
    assert torch.equal(target, want_t) and torch.equal(tw, want_w)
    assert x.shape == (4, 3, 64, 64) and target.shape == (4, 16, 16, 16) and bool((tw > 0).any())

    def net(feat, stacks):
        return H.get_pose_net(NS(MODEL=NS(EXTRA=NS(NUM_FEATURES=feat, NUM_STACKS=stacks, NUM_BLOCKS=1),
                                          NUM_JOINTS=16)), True)
    torch.manual_seed(3)
    init_s, init_t = net(64, 2).state_dict(), net(64, 1).state_dict()
    res = []
    for use_graph in (False, True):
        s, t = net(64, 2), net(64, 1)
        s.load_state_dict(init_s)
        t.load_state_dict(init_t)
        step = FPDTrainStep(s.cuda(), t.cuda(), alpha=0.5, lr=1e-3, use_graph=use_graph)
        losses = step.step(x, target, tw).clone()
        torch.cuda.synchronize()
        res.append((losses.cpu(), step.flat.flat.clone()))
    (le, fe), (lg, fg) = res
    assert torch.isfinite(le).all() and float(le[0]) > 0
    assert torch.equal(le, lg) and torch.equal(fe, fg)
