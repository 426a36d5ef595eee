"""Distilling from a teacher at its own input size, on the host: the teacher's crop in RawJointsDataset (same random
draws, the reference's matrices bit for bit, one region that serves both crops), raw_collate's teacher keys, every
refusal, and an fp64 restatement of fpd_heatmap_resample with the geometry it has to get right (no GPU needed)."""
import os
import random
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import fpd_b200  # noqa: E402,F401
from fpd_b200 import augment as A  # noqa: E402
import _augment_cases as C  # noqa: E402

G = C.golden()


def teacher_size(size):
    """A larger input of the same aspect: 1.5x (the shipped 256x192 -> 384x288 pair) where that is integral, else 2x."""
    w, h = size
    return (w * 3 // 2, h * 3 // 2) if w % 2 == 0 and h % 2 == 0 else (2 * w, 2 * h)


def resample_heatmaps(hm, out_hw, udp=False):
    """fpd_heatmap_resample in numpy: the position is the fp32 product of the output index and the fp32 ratio, as the
    kernel computes it; the bilinear interpolation is fp64. hm [B,Hi,Wi,C] -> [B,Ho,Wo,C] float64."""
    hm = np.asarray(hm, np.float64)
    B, Hi, Wi, C = hm.shape
    Ho, Wo = out_hw

    def axis(n_in, n_out):
        if udp:
            ratio = np.float32((n_in - 1) / (n_out - 1)) if n_out > 1 else np.float32(0)
        else:
            ratio = np.float32(n_in / n_out)
        pos = np.clip(np.arange(n_out, dtype=np.float32) * ratio, np.float32(0), np.float32(n_in - 1))
        i0 = pos.astype(np.int64)
        return i0, np.minimum(i0 + 1, n_in - 1), (pos - i0.astype(np.float32)).astype(np.float64)
    y0, y1, fy = axis(Hi, Ho)
    x0, x1, fx = axis(Wi, Wo)
    fx, fy = fx[None, None, :, None], fy[None, :, None, None]
    top = (1 - fx) * hm[:, y0][:, :, x0] + fx * hm[:, y0][:, :, x1]
    bot = (1 - fx) * hm[:, y1][:, :, x0] + fx * hm[:, y1][:, :, x1]
    return (1 - fy) * top + fy * bot


# ------------------------------------------------------------------------------------------------ the dataset
def _items(tag, paths, **kw):
    """Every item of the set and the np.random / random states after each one."""
    ds = A.RawJointsDataset(C.stand_in(G, tag, paths), **kw)
    C.seed(G, tag)
    items, states = [], []
    for i in range(len(ds)):
        items.append(ds[i])
        states.append((np.random.get_state()[1].copy(), np.random.get_state()[2], random.getstate()))
    return ds, items, states


@pytest.mark.parametrize("udp", [False, True])
@pytest.mark.parametrize("tag", C.sets(G))
def test_teacher_crop_draws_matrices_and_region(tag, udp, tmp_path):
    cv2 = pytest.importorskip("cv2")
    from oracle import augment_oracle as O
    paths = C.write_images(G, tmp_path)
    size = C.out_size(G, tag)
    tsize = teacher_size(size)
    _, plain, st_plain = _items(tag, paths, udp=udp)
    ds, items, st = _items(tag, paths, udp=udp, teacher_image_size=tsize)
    assert ds.teacher_image_size == tsize
    matrix = A.udp_crop_matrix if udp else A.crop_matrix
    for i, (a, b) in enumerate(zip(plain, items)):
        # the same draws, in the same order
        assert np.array_equal(st_plain[i][0], st[i][0]) and st_plain[i][1:] == st[i][1:], i
        np.testing.assert_array_equal(a['inv'], b['inv'])
        np.testing.assert_array_equal(a['joints'], b['joints'])
        m = b['meta']
        want = A.invert_affine(matrix(m['center'], m['scale'], m['rotation'], tsize))
        assert np.array_equal(b['teacher_inv'], want), i
        assert b['teacher_out_size'] == tsize and b['teacher_udp'] == udp and 'teacher_inv' not in a
        # the region holds both crops' windows, and the student's window is what it was
        _, x0, y0, w, h, iw, ih = b['desc']
        for inv, sz in ((b['inv'], size), (b['teacher_inv'], tsize)):
            wx0, wy0, wx1, wy1 = A.source_window(inv, sz, iw, ih)
            if wx1 > wx0 and wy1 > wy0:
                assert x0 <= wx0 and y0 <= wy0 and wx1 <= x0 + w and wy1 <= y0 + h, (i, (wx0, wy0, wx1, wy1))
        _, px0, py0, pw, ph, _, _ = a['desc']
        assert px0 >= x0 and py0 >= y0 and px0 + pw <= x0 + w and py0 + ph <= y0 + h
        # both crops through the grown region (the kernel's fixed-point model) against cv2 on the whole source image
        src = C.source(G, tag, i)
        for inv, sz in ((b['inv'], size), (b['teacher_inv'], tsize)):
            fwd = matrix(m['center'], m['scale'], m['rotation'], sz)
            ref = cv2.warpAffine(src, fwd, (int(sz[0]), int(sz[1])), flags=cv2.INTER_LINEAR)
            assert np.array_equal(O.warp_region(b['region'], (x0, y0), inv, sz), ref), (i, sz)


def test_collate_carries_the_teacher_crop(tmp_path):
    pytest.importorskip("cv2")
    paths = C.write_images(G, tmp_path)
    tag = C.sets(G)[0]
    tsize = teacher_size(C.out_size(G, tag))
    _, items, _ = _items(tag, paths, teacher_image_size=tsize)
    batch = A.raw_collate(items)
    assert batch['teacher_inv'].dtype == torch.float64 and tuple(batch['teacher_inv'].shape) == (len(items), 6)
    np.testing.assert_array_equal(batch['teacher_inv'].numpy(), np.stack([it['teacher_inv'].reshape(6) for it in items]))
    assert batch['teacher_out_size'].tolist() == list(tsize) and batch['teacher_udp'] is False
    assert 'teacher_inv' not in A.raw_collate([dict(it, **{}) for it in _items(tag, paths)[1]])
    mixed = [items[0], {k: v for k, v in items[1].items() if not k.startswith('teacher_')}]
    with pytest.raises(ValueError, match="teacher crop"):
        A.raw_collate(mixed)


# ------------------------------------------------------------------------------------------------ refusals
def test_dataset_refuses_another_aspect_ratio(tmp_path):
    ds = C.stand_in(G, C.sets(G)[0], [str(tmp_path / "none.png")] * 64)
    w, h = (int(v) for v in ds.image_size)
    with pytest.raises(ValueError, match="aspect ratio"):
        A.RawJointsDataset(ds, teacher_image_size=(w * 3 // 2, h * 3 // 2 + 1))
    with pytest.raises(ValueError, match="aspect ratio"):
        A.RawJointsDataset(ds, teacher_image_size=(h, w))
    with pytest.raises(ValueError, match="positive"):
        A.RawJointsDataset(ds, teacher_image_size=(0, 0))
    assert A.RawJointsDataset(ds, teacher_image_size=(2 * w, 2 * h)).teacher_image_size == (2 * w, 2 * h)


def _hg(feat, stacks):
    import types
    from fpd_b200.lib.models import hourglass as H
    NS = types.SimpleNamespace
    return H.get_pose_net(NS(MODEL=NS(EXTRA=NS(NUM_FEATURES=feat, NUM_STACKS=stacks, NUM_BLOCKS=1), NUM_JOINTS=16)),
                          False)


def test_train_step_refuses_bad_teacher_inputs(monkeypatch):
    """Each refusal comes before any device work (the streams are stood in for)."""
    from fpd_b200.train_step import FeatureAdapter, FPDTrainStep
    monkeypatch.setattr(torch.cuda, "Stream", lambda *a, **k: None)
    s, t = _hg(64, 1), _hg(128, 1)
    x, target, tw = torch.zeros(2, 3, 64, 64), torch.zeros(2, 16, 16, 16), torch.ones(2, 16, 1)
    tx = torch.zeros(2, 3, 96, 96)
    with pytest.raises(ValueError, match="needs a teacher"):
        FPDTrainStep(s, None).step(x, target, tw, teacher_x=tx)
    with pytest.raises(ValueError, match="batch"):
        FPDTrainStep(s, t).step(x, target, tw, teacher_x=tx[:1])
    with pytest.raises(ValueError, match="batch"):
        FPDTrainStep(s, t).step(x, target, tw, teacher_x=tx[0])
    with pytest.raises(ValueError, match="feature distillation"):
        FPDTrainStep(s, t, feature_weight=0.1, feature_adapter=FeatureAdapter(s, t)).step(x, target, tw, teacher_x=tx)
    monkeypatch.setenv("FPD_PIPELINE_TEACHER", "1")
    step = FPDTrainStep(s, t)
    assert step.pipeline
    with pytest.raises(ValueError, match="FPD_PIPELINE_TEACHER"):
        step.step(x, target, tw, teacher_x=tx)


def test_fpd_train_refuses_feature_kd_with_a_teacher_input(monkeypatch):
    import types
    from fpd_b200.lib.core import function as F
    from fpd_b200.lib.core.loss import JointsMSELoss
    from fpd_b200.train_step import FeatureAdapter
    NS = types.SimpleNamespace
    s, t = _hg(64, 1), _hg(128, 1)
    a = FeatureAdapter(s, t)
    opt = torch.optim.Adam(list(s.parameters()) + list(a.parameters()))
    monkeypatch.setattr(torch.Tensor, "cuda", lambda self, *args, **k: self)
    meta = {"teacher_input": torch.zeros(2, 3, 96, 96), "teacher_udp": False}
    loader = [(torch.zeros(2, 3, 64, 64), torch.zeros(2, 16, 16, 16), torch.ones(2, 16, 1), meta)]
    cfg = NS(KD=NS(ALPHA=0.5, FEATURE_WEIGHT=0.1), PRINT_FREQ=1, DEBUG=NS(DEBUG=False))
    with pytest.raises(ValueError, match="teacher input of its own size"):
        F.fpd_train(cfg, loader, s, t, JointsMSELoss(True), JointsMSELoss(True), opt, 0, "/tmp", "/tmp", None,
                    feature_adapter=a)


def test_teacher_input_reaches_each_fused_route(monkeypatch):
    """fpd_train hands meta['teacher_input'] and meta['teacher_udp'] to the graph route's step and to the eager route."""
    import types
    from fpd_b200 import train_step
    from fpd_b200.lib.core import function as F
    from fpd_b200.lib.core.loss import JointsMSELoss
    NS = types.SimpleNamespace
    s, t = _hg(64, 1), _hg(64, 1)
    opt = torch.optim.Adam(s.parameters())
    monkeypatch.setattr(torch.Tensor, "cuda", lambda self, *args, **k: self)
    tx = torch.zeros(2, 3, 96, 96)
    loader = [(torch.zeros(2, 3, 64, 64), torch.zeros(2, 16, 16, 16), torch.ones(2, 16, 1),
               {"teacher_input": tx, "teacher_udp": True})]
    cfg = NS(KD=NS(ALPHA=0.5), PRINT_FREQ=100, DEBUG=NS(DEBUG=False))
    seen = []

    def rec_fused(model, tmodel, input, target, target_weight, alpha, use_tw, graph=None, **kw):
        seen.append(("fused", graph is not None, kw.get("teacher_input") is tx, kw.get("teacher_udp")))
        return torch.zeros(3), torch.zeros(2, 16, 16, 16)
    monkeypatch.setattr(F, "_fused_step", rec_fused)
    monkeypatch.setattr(F, "_device_accuracy", lambda out, target: (0.0, 0, None))
    monkeypatch.setattr(F, "_TRAIN_GRAPH", False)
    F.fpd_train(cfg, loader, s, t, JointsMSELoss(True), JointsMSELoss(True), opt, 0, "/tmp", "/tmp", None)
    assert seen == [("fused", False, True, True)]

    class RecStep:
        def __init__(self, *a, **k):
            seen.append(("FPDTrainStep", k.get("teacher_input_udp")))
            self.params, self.grad_views, self.teacher_input_udp = [], [], k.get("teacher_input_udp", False)
            self.counts = torch.zeros(16, 2, dtype=torch.int32)
    monkeypatch.setattr(train_step, "FPDTrainStep", RecStep)
    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self, *a, **k: self)
    orig_empty = torch.empty
    monkeypatch.setattr(torch, "empty", lambda *a, pin_memory=False, **k: orig_empty(*a, **k))
    monkeypatch.setattr(torch.cuda, "Event", lambda *a, **k: NS(record=lambda *a: None, synchronize=lambda: None))
    monkeypatch.setattr(F, "_TRAIN_GRAPH", True)
    F._train_step_cache.clear()
    seen.clear()
    F.fpd_train(cfg, loader, s, t, JointsMSELoss(True), JointsMSELoss(True), opt, 0, "/tmp", "/tmp", None)
    F._train_step_cache.clear()
    assert seen[0] == ("FPDTrainStep", True)
    assert seen[1] == ("fused", True, True, True)


# ------------------------------------------------------------------------------------------------ the resample geometry
def _gaussian(H, W, mu, sigma):
    ys, xs = np.mgrid[0:H, 0:W].astype(np.float64)
    return np.exp(-((xs - mu[0]) ** 2 + (ys - mu[1]) ** 2) / (2 * sigma ** 2))


@pytest.mark.parametrize("udp", [False, True])
def test_teacher_gaussian_lands_on_the_student_joint(udp):
    """A sigma-3 Gaussian at teacher pixel 1.5 mu (96x72) peaks within 0.5 px of mu on the 64x48 grid, in both crop
    conventions."""
    rng = np.random.RandomState(0)
    for _ in range(20):
        mu = np.array([rng.uniform(4, 44), rng.uniform(4, 60)])
        hm = _gaussian(96, 72, 1.5 * mu, 3.0)[None, :, :, None]
        out = resample_heatmaps(hm, (64, 48), udp)[0, :, :, 0]
        v, u = np.unravel_index(np.argmax(out), out.shape)
        # the sub-pixel peak by a parabola through the arg-max's neighbours
        du = 0.5 * (out[v, u - 1] - out[v, u + 1]) / (out[v, u - 1] - 2 * out[v, u] + out[v, u + 1])
        dv = 0.5 * (out[v - 1, u] - out[v + 1, u]) / (out[v - 1, u] - 2 * out[v, u] + out[v + 1, u])
        assert abs(u + du - mu[0]) <= 0.5 and abs(v + dv - mu[1]) <= 0.5, (mu, u + du, v + dv)


def test_restatement_copies_equal_sizes_and_clamps_edges():
    rng = np.random.RandomState(1)
    hm = rng.rand(2, 12, 9, 5).astype(np.float32)
    for udp in (False, True):
        np.testing.assert_array_equal(resample_heatmaps(hm, (12, 9), udp), hm)
    up = resample_heatmaps(hm, (16, 12), False)       # ratio 0.75: the last row / column fall past the map and clamp
    np.testing.assert_array_equal(up[:, 15, 11], hm[:, 11, 8])
    np.testing.assert_array_equal(up[:, 0, 0], hm[:, 0, 0])
    h64 = hm.astype(np.float64)
    np.testing.assert_allclose(up[:, 1, 0], 0.25 * h64[:, 0, 0] + 0.75 * h64[:, 1, 0], rtol=1e-12)


def test_wrapper_refuses_bad_arguments_before_the_device():
    from fpd_b200 import ops
    cpu = torch.zeros(1, 4, 4, 3)
    with pytest.raises(ValueError, match="CUDA"):
        ops.resample_heatmaps(cpu, (2, 2))
