"""DARK on the device: fpd_final_preds_dark and fpd_gaussian_targets_unbiased against the fp64 model of
tests/test_dark_cpu.py, the edge cases where the Taylor step must not move the arg-max, the round trip through both
kernels, and the opt-in through FlipTestInference and validate() (graph route equal to the eager route, bit for bit)."""
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
import test_dark_cpu as M  # noqa: E402


def _identity_inv(B):
    return torch.tensor([[1.0, 0.0, 0.0, 0.0, 1.0, 0.0]] * B, dtype=torch.float64, device="cuda")


def _noisy_peaks(rng, B, J, h, w):
    """Gaussians of random amplitude and width at random sub-pixel centres (some near the borders) plus noise."""
    ys, xs = np.mgrid[0:h, 0:w].astype(np.float64)
    hm = np.empty((B, J, h, w), np.float32)
    for b in range(B):
        for j in range(J):
            cx, cy = rng.uniform(-1, w), rng.uniform(-1, h)
            s = rng.uniform(1.5, 3.0)
            g = rng.uniform(0.3, 1.0) * np.exp(-((xs - cx) ** 2 + (ys - cy) ** 2) / (2 * s * s))
            hm[b, j] = g + rng.uniform(-0.01, 0.03, (h, w))
    return hm


def _decode(hm_nchw, inv, k=11):
    from fpd_b200 import ops
    nhwc = ops.nchw_to_nhwc(hm_nchw)
    _, idx, mv = ops.flip_merge_argmax(nhwc, want_avg=False)
    return ops.final_preds_dark(nhwc, idx, mv, inv, k), ops.final_preds(nhwc, idx, mv, inv, False), mv


@pytest.mark.parametrize("h,w", [(64, 64), (64, 48), (96, 72)])
@pytest.mark.parametrize("J", [16, 17])
@pytest.mark.parametrize("k", [11, 3, 15])
def test_decode_matches_fp64_model(h, w, J, k):
    import fpd_b200  # noqa: F401
    rng = np.random.RandomState(h * 100 + w + J + k)
    B = 32 if k == 11 else 4
    hm = _noisy_peaks(rng, B, J, h, w)
    preds, _, mv = _decode(torch.from_numpy(hm).cuda(), _identity_inv(B), k)
    preds = preds.cpu().numpy()
    assert np.array_equal(preds[..., 2].view(np.int32), mv.cpu().numpy().view(np.int32))
    ref = np.array([[M.dark_decode(hm[b, j].astype(np.float64), k) for j in range(J)] for b in range(B)])
    err = np.abs(preds[..., :2] - ref)
    assert err.max() < 1e-4, (err.max(), np.unravel_index(err.argmax(), err.shape))
    moved = np.abs(ref - np.round(ref)).max(-1) > 1e-3
    assert moved.mean() > 0.5            # most peaks are interior: the step is exercised, not skipped


def _edge_maps(h, w):
    """Maps on which DARK must leave the arg-max where it is."""
    ys, xs = np.mgrid[0:h, 0:w].astype(np.float64)
    maps = []
    for cx, cy in [(0, h // 2), (1, h // 2), (w - 2, h // 2), (w - 1, h // 2),
                   (w // 2, 0), (w // 2, 1), (w // 2, h - 2), (w // 2, h - 1), (1, h - 1)]:
        maps.append(np.exp(-((xs - cx - 0.3) ** 2 + (ys - cy + 0.2) ** 2) / 8.0))   # arg-max within 2 px of a border
    maps.append(np.full((h, w), 0.5))                                                # constant: det = 0
    maps.append(np.zeros((h, w)))                                                    # all zero
    neg = -np.ones((h, w))
    neg[h // 2, w // 2] = 1.0                                                        # blur < 0 everywhere: every log clamps
    maps.append(neg)
    maps.append(-0.5 - np.random.RandomState(0).rand(h, w))                          # all negative
    tie = np.zeros((h, w))
    tie[1, w // 2] = tie[h // 2, w // 3] = 1.0                                       # tie: the first maximum is at y = 1
    maps.append(tie)
    return np.stack(maps)[None].astype(np.float32)


@pytest.mark.parametrize("h,w", [(64, 48), (96, 72)])
def test_decode_edge_cases_equal_the_raw_argmax(h, w):
    import fpd_b200  # noqa: F401
    from fpd_b200.lib.core.inference import inverse_affines
    hm = np.repeat(_edge_maps(h, w), 2, axis=0)
    B = hm.shape[0]
    assert M.blur(hm[0, 11].astype(np.float64), 11).max() < 0
    inv = torch.from_numpy(inverse_affines(np.array([[200.0, 150.0], [320.5, 99.25]]), np.array([[1.1, 1.5], [2.3, 3.0]]),
                                           [w, h])).cuda()
    for k in (3, 11, 15):
        dark, raw, _ = _decode(torch.from_numpy(hm).cuda(), inv, k)
        assert torch.equal(dark.view(torch.int32), raw.view(torch.int32)), k


def _target_joints(n, J, rng, img_w, img_h, stride):
    """Random joints plus joints just inside and just outside each border of the 3 sigma (sigma = 2) window."""
    j = np.zeros((n, J, 3), np.float32)
    j[..., 0] = rng.uniform(-40, img_w + 40, (n, J))
    j[..., 1] = rng.uniform(-40, img_h + 40, (n, J))
    W, H = img_w / stride, img_h / stride
    edge = [(-7.0 - 0.01, 10), (-7.0 + 0.1, 10), (W + 6 - 0.1, 10), (W + 6, 10),
            (10, -7.0 - 0.01), (10, -7.0 + 0.1), (10, H + 6 - 0.1), (10, H + 6)]
    for i, (x, y) in enumerate(edge):
        j[0, i, :2] = (x * stride, y * stride)
    vis = (rng.rand(n, J, 3) > 0.2).astype(np.float32)
    vis[0, :len(edge)] = 1
    return j, vis


@pytest.mark.parametrize("hm_size,img_size,sigma", [((48, 64), (192, 256), 2), ((72, 96), (288, 384), 2),
                                                    ((64, 64), (256, 256), 3)])
@pytest.mark.parametrize("use_w", [False, True])
def test_targets_match_fp64_model(hm_size, img_size, sigma, use_w):
    import fpd_b200  # noqa: F401
    from fpd_b200 import ops
    rng = np.random.RandomState(sigma + hm_size[0] + int(use_w))
    n, J = 6, 17
    joints, vis = _target_joints(n, J, rng, img_size[0], img_size[1], img_size[0] // hm_size[0])
    jw = rng.uniform(0.5, 1.5, J).astype(np.float32) if use_w else None
    t, w = ops.gaussian_targets_unbiased(torch.from_numpy(joints).cuda(), torch.from_numpy(vis).cuda(), hm_size, img_size,
                                         sigma, None if jw is None else torch.from_numpy(jw))
    rt, rw = M.unbiased_targets(joints, vis, hm_size, img_size, sigma, jw)
    assert np.abs(t.cpu().numpy() - rt).max() < 1e-6
    assert np.array_equal(w.cpu().numpy(), rw.astype(np.float32))
    if sigma == 2:
        assert (rw[0, :8, 0] > 0).tolist() == [False, True, True, False, False, True, True, False]
    assert (rw == 0).any() and (rw > 0).any()


def test_round_trip_on_the_device():
    import fpd_b200  # noqa: F401
    from fpd_b200.targets import TargetGenerator
    rng = np.random.RandomState(5)
    B, J = 8, 17
    m = 4 * M.border_margin(2)
    joints = np.zeros((B, J, 3), np.float32)
    joints[..., 0] = rng.uniform(m, 188 - m, (B, J))    # the last heat-map column, 47, is image x = 188
    joints[..., 1] = rng.uniform(m, 252 - m, (B, J))
    gen = TargetGenerator((192, 256), (48, 64), 2, unbiased=True)
    target, tw = gen(joints, np.ones_like(joints))
    assert torch.all(tw == 1)
    preds, raw, _ = _decode(target, _identity_inv(B))
    want = joints[..., :2].astype(np.float64) / 4
    assert np.abs(preds.cpu().numpy()[..., :2] - want).max() < 0.02
    assert np.abs(raw.cpu().numpy()[..., :2] - want).max() > 0.3     # the arg-max alone misses
    # the default generator still stamps the rounded Gaussian
    t0, _ = TargetGenerator((192, 256), (48, 64), 2)(joints, np.ones_like(joints))
    assert not torch.equal(t0, target)


# ----------------------------------------------------------------------------------------------- FlipTestInference, validate()
FLIP_PAIRS = [[0, 5], [1, 4], [2, 3], [10, 15], [11, 14], [12, 13]]


def _hourglass():
    from fpd_b200.lib.models import hourglass as H
    cfg = NS(MODEL=NS(EXTRA=NS(NUM_FEATURES=64, NUM_STACKS=2, NUM_BLOCKS=1), NUM_JOINTS=16, NAME="hourglass"))
    return H.get_pose_net(cfg, True), (128, 128), 16


def _hrnet():
    from fpd_b200.lib.models import pose_hrnet as H
    from bench import _wrap

    def stage(nmod, chans):
        return dict(NUM_MODULES=nmod, NUM_BRANCHES=len(chans), BLOCK='BASIC', NUM_BLOCKS=[1] * len(chans),
                    NUM_CHANNELS=chans, FUSE_METHOD='SUM')
    cfg = _wrap(dict(MODEL=dict(NUM_JOINTS=17, INIT_WEIGHTS=False, PRETRAINED='', EXTRA=dict(
        PRETRAINED_LAYERS=['*'], FINAL_CONV_KERNEL=1, STAGE2=stage(1, [8, 16]), STAGE3=stage(2, [8, 16, 32]),
        STAGE4=stage(1, [8, 16, 32, 64])))))
    return H.get_pose_net(cfg, is_train=False), (128, 96), 17


NETS = {"hourglass": _hourglass, "hrnet": _hrnet}


@pytest.fixture(scope="module")
def nets():
    import fpd_b200  # noqa: F401
    out = {}
    for kind, make in NETS.items():
        torch.manual_seed(11)
        net, hw, J = make()
        for mod in net.modules():
            if isinstance(mod, torch.nn.BatchNorm2d):
                mod.running_mean.normal_(0, 0.1)
                mod.running_var.uniform_(0.5, 1.5)
        out[kind] = (net.cuda(), hw, J)
    return out


def _batch(B, seed, hw, J):
    from bench import synthetic_batch
    x, t, w = synthetic_batch(B, seed, hw[0], hw[1], J)
    rng = np.random.RandomState(seed)
    meta = {"center": torch.from_numpy(rng.uniform(100, 500, (B, 2))), "scale": torch.from_numpy(rng.uniform(0.5, 3, (B, 2))),
            "score": torch.from_numpy(rng.uniform(0.5, 1, B)), "image": ["img%d_%d" % (seed, b) for b in range(B)]}
    return x, t, w, meta


def test_flip_test_inference_dark_graph_equals_eager(nets):
    from fpd_b200 import ops
    from fpd_b200.infer_step import FlipTestInference
    from fpd_b200.lib.core.inference import inverse_affines
    net, hw, J = nets["hourglass"]
    runs = {g: FlipTestInference(net, FLIP_PAIRS, use_graph=g, decode=True) for g in (True, False)}
    graphs = []
    for B, seed, k, pp in ((3, 1, 11, "dark"), (3, 2, 11, "dark"), (3, 3, 7, "dark"), (3, 4, 7, True), (3, 5, 11, "dark")):
        x, t, w, meta = _batch(B, seed, hw, J)
        inv = inverse_affines(meta["center"].numpy(), meta["scale"].numpy(), [t.shape[3], t.shape[2]])
        res = {g: r(x, inv=inv, target=t, target_weight=w, post_process=pp, blur_kernel=k) for g, r in runs.items()}
        got, ref = res[True], res[False]
        for key in ("preds", "loss3", "pck", "avg_nhwc"):
            assert torch.equal(got[key], ref[key]), key
        if pp == "dark":
            again = ops.final_preds_dark(got["avg_nhwc"], got["idx"], got["maxval"], torch.from_numpy(inv).cuda(), k)
            assert torch.equal(got["preds"], again)
            nudged = ops.final_preds(got["avg_nhwc"], got["idx"], got["maxval"], torch.from_numpy(inv).cuda(), True)
            assert not torch.equal(got["preds"], nudged)
        graphs.append(runs[True].graph)
    # same key replays; a new blur_kernel or post_process captures again
    assert graphs[1] is graphs[0]
    assert graphs[2] is not graphs[1] and graphs[3] is not graphs[2] and graphs[4] is not graphs[3]


class _ValSet:
    def __init__(self, n, J):
        self.n = n
        self.flip_pairs = [p for p in FLIP_PAIRS if max(p) < J]
        self.seen = None

    def __len__(self):
        return self.n

    def evaluate(self, cfg, preds, output_dir, all_boxes, image_path, filenames, imgnums):
        self.seen = preds.copy()
        return {"Mean": float(preds[..., :2].mean())}, float(preds[..., :2].mean())


@pytest.mark.parametrize("kind", list(NETS))
@pytest.mark.parametrize("flip", [True, False])
def test_validate_dark_graph_route_equals_eager_route(nets, kind, flip, monkeypatch):
    from fpd_b200.lib.core import function as F
    from fpd_b200.lib.core.loss import JointsMSELoss
    net, hw, J = nets[kind]
    loader = [_batch(3, 20, hw, J), _batch(3, 21, hw, J), _batch(2, 22, hw, J)]
    seen = {}
    for dark, k in ((True, 11), (True, 5), (False, 11)):
        for graph in (True, False):
            monkeypatch.setattr(F, "_VALIDATE_GRAPH", graph)
            cfg = NS(MODEL=NS(NUM_JOINTS=J, NAME=kind), PRINT_FREQ=2, DEBUG=NS(DEBUG=False),
                     TEST=NS(FLIP_TEST=flip, SHIFT_HEATMAP=True, POST_PROCESS=True, DARK=dark, BLUR_KERNEL=k))
            ds = _ValSet(8, J)
            F.validate(cfg, loader, ds, net, JointsMSELoss(True), "/tmp", "/tmp", None)
            seen[dark, k, graph] = ds.seen
        assert np.array_equal(seen[dark, k, True], seen[dark, k, False])
    assert not np.array_equal(seen[True, 11, True], seen[False, 11, True])
    assert not np.array_equal(seen[True, 11, True], seen[True, 5, True])
    assert np.array_equal(seen[True, 11, True][..., 2], seen[False, 11, True][..., 2])
