"""Distillation from unlabeled person boxes on the H100: fpd_kd_weights against a numpy evaluation of the rule, the
kd-weighted fused loss against the fp64 model for every criteria mix, bit-identity with the existing entry points and
with the mode off, the three fpd_train routes, and a synthetic mixed dataset end to end."""
import os
import random
import sys
import types

import numpy as np
import pytest
import torch

NS = types.SimpleNamespace
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import _kld_model as K  # noqa: E402

pytestmark = pytest.mark.gpu

THRE = 0.2
KINDS = {"mse": ("mse",), "ohkm": ("ohkm", 8), "kl": ("kl", 1.0)}
PAIRS = [(p, k) for p in KINDS for k in KINDS]
SHAPES = {"hg_fpd": (32, 16, 64, 64), "hrnet_fpd": (24, 17, 64, 48)}     # B, J, h, w


def _nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def _nchw(t):
    return t.permute(0, 3, 1, 2).contiguous()


def _rule(teacher_nhwc, tw, thre):
    """The weights in numpy: unlabeled (all J weights exactly 0) -> [max > thre], a NaN map -> 0; else tw."""
    B, h, w, J = teacher_nhwc.shape
    t = teacher_nhwc.cpu().numpy().reshape(B, h * w, J)
    tw = tw.cpu().numpy().reshape(B, J)
    with np.errstate(invalid="ignore"):
        conf = np.where(np.isnan(t).any(1), 0.0, t.max(1) > np.float32(thre)).astype(np.float32)
    return np.where((tw == 0).all(1, keepdims=True), conf, tw)


# ------------------------------------------------------------------------------------------------ fpd_kd_weights
@pytest.mark.parametrize("hw", [(64, 48), (64, 64)])
@pytest.mark.parametrize("J", [16, 17, 64])
@pytest.mark.parametrize("B", [1, 3, 32])
def test_kd_weights_equal_the_numpy_rule(B, J, hw):
    from fpd_b200 import ops
    h, w = hw
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + J * 10 + h * w)
    teacher = 0.15 * torch.randn(B, h, w, J, generator=g, device="cuda")
    tw = (torch.rand(B, J, generator=g, device="cuda") > 0.3).float()
    tw[::2] = 0.0                                     # even samples unlabeled; B = 1: the only sample
    if B > 1:
        tw[1, :3] = 0.0                               # a labeled sample with some zero weights keeps them
        tw[1, 3] = 1.0
    above = float(np.nextafter(np.float32(THRE), np.float32(np.inf)))
    planted = {0: (THRE, 0.0), 1: (above, 1.0), 2: (float("nan"), 0.0), 3: (None, 0.0)}
    for j, (v, _) in planted.items():
        teacher[0, :, :, j] = -1.0 - torch.rand(h, w, generator=g, device="cuda")    # all negative
        if v is not None:
            teacher[0, (7 * j) % h, (5 * j + 3) % w, j] = v
    if B > 1:
        teacher[1, 0, 0, 3] = float("nan")            # a NaN map of a labeled sample: its weight stays
    got = ops.kd_weights(teacher, tw.unsqueeze(2), THRE)
    assert got.shape == (B, J) and got.dtype == torch.float32
    want = _rule(teacher, tw, THRE)
    np.testing.assert_array_equal(got.cpu().numpy(), want)
    assert [float(got[0, j]) for j in planted] == [r for _, r in planted.values()]
    if B > 1:
        assert torch.equal(got[1], tw[1])
    unl = (tw == 0).all(1)
    assert ((got[unl] == 0) | (got[unl] == 1)).all() and (got[unl] == 1).any() and (got[unl] == 0).any()
    # thre below every value: every finite map of an unlabeled sample is accepted
    low = ops.kd_weights(teacher, tw, -10.0)
    np.testing.assert_array_equal(low.cpu().numpy(), _rule(teacher, tw, -10.0))


def test_kd_weights_are_graph_capturable_and_repeat():
    from fpd_b200 import ops
    B, J, h, w = SHAPES["hg_fpd"]
    g = torch.Generator(device="cuda").manual_seed(4)
    teacher = 0.2 * torch.randn(B, h, w, J, generator=g, device="cuda")
    tw = torch.zeros(B, J, device="cuda")
    tw[B // 2:] = 1.0
    out = torch.empty(B, J, device="cuda")
    ops.kd_weights(teacher, tw, THRE, out=out)
    torch.cuda.synchronize()
    first = out.clone()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.kd_weights(teacher, tw, THRE, out=out)
    out.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, first)
    np.testing.assert_array_equal(first.cpu().numpy(), _rule(teacher, tw, THRE))


# ------------------------------------------------------------------------------------------------ kd-weighted loss
def _tols(pose, kd):
    return 1e-5 if "kl" in (pose, kd) else 1e-6       # the existing fused-loss tests' bounds for these criteria


def _draw(gen, B, J, h, w, S):
    target = torch.rand(B, J, h, w, generator=gen, device="cuda")
    teacher = target + 0.3 * torch.randn(B, J, h, w, generator=gen, device="cuda")
    outs = [target + 0.3 * torch.randn(B, J, h, w, generator=gen, device="cuda") for _ in range(S)]
    tw = (torch.rand(B, J, 1, generator=gen, device="cuda") > 0.2).float()
    tw[::2] = 0.0
    kdw = (torch.rand(B, J, 1, generator=gen, device="cuda") > 0.4).float()
    kdw[1::4] = tw[1::4]
    return outs, target, teacher, tw, kdw


def _fp64(outs, target, teacher, tw, kdw, alpha, pose, kd):
    p_sum = k_sum = 0.0
    grads = []
    for o in outs:
        vp, gp = K.criterion(o, target, tw, pose)
        vk, gk = K.criterion(o, teacher, kdw, kd)
        p_sum, k_sum = p_sum + vp, k_sum + vk
        grads.append((1 - alpha) * gp + alpha * gk)
    return p_sum, k_sum, (1 - alpha) * p_sum + alpha * k_sum, grads


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("S", [1, 4, 8])
@pytest.mark.parametrize("pose,kd", PAIRS)
def test_kd_weighted_loss_matches_fp64(pose, kd, S, shape):
    from fpd_b200 import ops
    B, J, h, w = SHAPES[shape]
    gen = torch.Generator(device="cuda").manual_seed(S * 31 + len(pose) * 7 + len(kd) + J)
    outs, target, teacher, tw, kdw = _draw(gen, B, J, h, w, S)
    alpha = 0.3
    losses, grads = ops.fpd_loss([_nhwc(o) for o in outs], target, _nhwc(teacher), tw, alpha, kd_weight=kdw,
                                 **K.fpd_kwargs(KINDS[pose], KINDS[kd]))
    ref = _fp64(outs, target, teacher, tw, kdw, alpha, KINDS[pose], KINDS[kd])
    tol = _tols(pose, kd)
    for got, want in zip(losses.cpu().tolist(), ref[:3]):
        assert abs(got - float(want)) <= tol * abs(float(want)), (got, float(want))
    for g, r in zip(grads, ref[3]):
        err = (_nchw(g).double() - r.double()).abs().max().item()
        assert err <= tol * r.abs().max().item(), (err, r.abs().max().item())


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("pose,kd", PAIRS)
def test_kd_weight_equal_to_target_weight_gives_the_existing_bits(pose, kd, shape):
    from fpd_b200 import ops
    B, J, h, w = SHAPES[shape]
    gen = torch.Generator(device="cuda").manual_seed(len(pose) * 7 + len(kd) + J)
    outs, target, teacher, tw, _ = _draw(gen, B, J, h, w, 4)
    tw = torch.rand(B, J, 1, generator=gen, device="cuda") * (tw + 0.5)     # fractional, some zero
    tw[::3] = 0.0
    outs, teacher = [_nhwc(o) for o in outs], _nhwc(teacher)
    kw = K.fpd_kwargs(KINDS[pose], KINDS[kd])
    for alpha in (0.5, 0.3):
        l0, g0 = ops.fpd_loss(outs, target, teacher, tw, alpha, **kw)
        l0, g0 = l0.clone(), [g.clone() for g in g0]
        l1, g1 = ops.fpd_loss(outs, target, teacher, tw, alpha, kd_weight=tw.clone(), **kw)
        assert torch.equal(l0, l1)
        assert all(torch.equal(a, b) for a, b in zip(g0, g1))


@pytest.mark.parametrize("kd", ["mse", "kl"])
def test_unlabeled_kd_gradient_is_nonzero_exactly_on_accepted_joints(kd):
    from fpd_b200 import ops
    B, J, h, w = SHAPES["hrnet_fpd"]
    gen = torch.Generator(device="cuda").manual_seed(9)
    outs, target, _, tw, _ = _draw(gen, B, J, h, w, 2)
    # per-map maxima spread over about [0, 0.7], around thre
    teacher = 0.1 * torch.randn(B, h, w, J, generator=gen, device="cuda") * 2 * torch.rand(B, 1, 1, J, generator=gen,
                                                                                          device="cuda")
    target[::2] = 0.0
    kdw = ops.kd_weights(teacher, tw, THRE)
    _, grads = ops.fpd_loss([_nhwc(o) for o in outs], target, teacher, tw, 0.5, kd_weight=kdw,
                            **K.fpd_kwargs(KINDS["mse"], KINDS[kd]))
    unl = (tw.reshape(B, J) == 0).all(1)
    acc = kdw[unl] == 1
    assert acc.any() and (~acc).any()
    for g in grads:
        nz = (g[unl] != 0).any(dim=1).any(dim=1)     # [n_unlabeled, J]
        assert torch.equal(nz, acc)


# ------------------------------------------------------------------------------------------------ training
def _cfg(f, s, kd=None, debug=False):
    return NS(MODEL=NS(EXTRA=NS(NUM_FEATURES=f, NUM_STACKS=s, NUM_BLOCKS=1), NUM_JOINTS=16, NAME="hourglass"),
              KD=NS(ALPHA=0.5, **(kd or {})), PRINT_FREQ=1,
              TEST=NS(FLIP_TEST=True, SHIFT_HEATMAP=True, POST_PROCESS=True), DEBUG=NS(DEBUG=debug))


def _net(f, s, sd=None):
    from fpd_b200.lib.models import hourglass as H
    net = H.get_pose_net(_cfg(f, s), True)
    if sd is not None:
        net.load_state_dict(sd)
    return net.cuda()


def _inits(seed):
    torch.manual_seed(seed)
    return ({k: v.clone() for k, v in _net(64, 2).state_dict().items()},
            {k: v.clone() for k, v in _net(64, 1).state_dict().items()})


def _batch(B, seed, unlabeled):
    """bench.synthetic_batch at 128x128 with every labeled sample's weights nonzero and the `unlabeled` samples
    without targets and weights."""
    from bench import synthetic_batch
    x, t, w = synthetic_batch(B, seed, 128, 128)
    w[:, 0] = 1.0
    for b in unlabeled:
        t[b] = 0.0
        w[b] = 0.0
    return x.cuda(), t.cuda(), w.cuda()


def _train_steps(init_s, init_t, batch, thre, steps=2):
    from fpd_b200.train_step import FPDTrainStep
    s, t = _net(64, 2, init_s), _net(64, 1, init_t)
    step = FPDTrainStep(s, t, alpha=0.5, lr=1e-3, kd_unlabeled_thre=thre)
    losses = [step.step(*batch).clone() for _ in range(steps)]
    torch.cuda.synchronize()
    return step.flat.flat.clone(), step.exp_avg.clone(), step.exp_avg_sq.clone(), torch.stack(losses)


@pytest.mark.parametrize("case", ["no_unlabeled_sample", "thre_above_every_teacher_maximum"])
def test_train_step_with_the_mode_on_equals_off(case):
    init_s, init_t = _inits(11)
    if case == "no_unlabeled_sample":
        batch, thre = _batch(4, 12, []), THRE
    else:
        batch, thre = _batch(4, 12, [1, 3]), 1e30
    off = _train_steps(init_s, init_t, batch, None)
    on = _train_steps(init_s, init_t, batch, thre)
    for a, b in zip(off, on):
        assert torch.equal(a, b)
    if case != "no_unlabeled_sample":
        # a reachable threshold changes the update
        assert not torch.equal(_train_steps(init_s, init_t, batch, -1e30)[0], off[0])


class _Writer:
    def __init__(self):
        self.scalars = []

    def add_scalar(self, tag, v, step):
        self.scalars.append((tag, float(v), step))


class _Hide(torch.nn.Module):
    """Hides the engine attributes: function.py takes the generic (reference-like) route."""

    def __init__(self, net):
        super().__init__()
        self.net = net

    def forward(self, x):
        return self.net(x.cuda())


def _meta(B, i):
    return {"center": torch.tensor([[64.0, 64.0]] * B), "scale": torch.tensor([[0.64, 0.64]] * B),
            "score": torch.ones(B), "image": ["img%d_%d" % (i, b) for b in range(B)]}


def _split_thre(init_t, loader):
    """A threshold between two middle maxima of the unlabeled samples' teacher maps: some joints on each side."""
    t = _net(64, 1, init_t).eval()
    m = []
    with torch.no_grad():
        for x, _, w, _ in loader:
            hm = t.forward_nhwc(x.cuda().float().contiguous(), training=False)[-1]
            unl = (w.reshape(w.shape[0], -1) == 0).all(1)
            m.append(hm[unl].amax(dim=(1, 2)).flatten())
    m = torch.cat(m).sort().values.cpu().numpy()
    i = len(m) // 2
    while m[i - 1] == m[i]:
        i += 1
    return float((m[i - 1] + m[i]) / 2)


def _fpd_epoch(F, cfg, loader, init_s, init_t, generic=False):
    from fpd_b200.lib.core.loss import JointsMSELoss
    s, t = _net(64, 2, init_s), _net(64, 1, init_t)
    opt = torch.optim.Adam(s.parameters(), lr=1e-3)
    wd = {"writer": _Writer(), "train_global_steps": 0}
    F.fpd_train(cfg, loader, _Hide(s) if generic else s, t, JointsMSELoss(True), JointsMSELoss(True), opt, 0, "/tmp",
                "/tmp", wd)
    torch.cuda.synchronize()
    sd = {k: v.clone() for k, v in s.state_dict().items()}
    ost = [(k, v.clone() if torch.is_tensor(v) else v) for st in opt.state.values() for k, v in sorted(st.items())]
    return sd, ost, wd["writer"].scalars


def test_fpd_train_routes_agree_on_a_half_unlabeled_batch(monkeypatch):
    from fpd_b200.lib.core import function as F
    init_s, init_t = _inits(13)
    loader = []
    for i in range(3):
        x, t, w = _batch(4, 20 + i, [1, 3])
        loader.append((x.cpu(), t.cpu(), w.cpu(), _meta(4, i)))
    cfg = _cfg(64, 2, {"UNLABELED": True, "UNLABELED_THRE": _split_thre(init_t, loader)})
    runs = []
    for graph in (True, False):
        monkeypatch.setattr(F, "_TRAIN_GRAPH", graph)
        F._train_step_cache.clear()
        runs.append(_fpd_epoch(F, cfg, loader, init_s, init_t))
    F._train_step_cache.clear()
    (sd_g, os_g, sc_g), (sd_e, os_e, sc_e) = runs
    assert all(torch.equal(sd_g[k], sd_e[k]) for k in sd_g)
    assert all(a[0] == b[0] and (torch.equal(a[1], b[1]) if torch.is_tensor(a[1]) else a[1] == b[1])
               for a, b in zip(os_g, os_e))
    assert sc_g == sc_e
    sd_x, _, sc_x = _fpd_epoch(F, cfg, loader, init_s, init_t, generic=True)
    assert len(sc_x) == len(sc_e)
    for (tf, vf, _), (tg, vg, _) in zip(sc_e, sc_x):
        assert tf == tg and abs(vf - vg) <= 1e-4 * max(1.0, abs(vg)), (tf, vf, vg)
    worst = max(((sd_e[k].double() - sd_x[k].double()).abs().max() / sd_x[k].double().abs().max().clamp_min(1e-12))
                .item() for k in sd_e if sd_e[k].is_floating_point())
    assert worst < 1e-4, worst
    # the mode changes what the unlabeled samples contribute
    off = _fpd_epoch(F, _cfg(64, 2), loader, init_s, init_t)
    assert not all(torch.equal(off[0][k], sd_e[k]) for k in sd_e)


# ------------------------------------------------------------------------------------------------ end to end
MPII_FLIP = [[0, 5], [1, 4], [2, 3], [10, 15], [11, 14], [12, 13]]


def _mixed_dataset(tmp_path, n=8):
    """A stand-in MPII training set over synthetic images: odd records labeled, even records unlabeled boxes."""
    import cv2
    from oracle.augment_oracle import StandInDataset
    rng = np.random.RandomState(5)
    paths = []
    for k in range(2):
        img = rng.randint(0, 256, (180, 200, 3)).astype(np.uint8)
        p = str(tmp_path / ("img%d.png" % k))
        assert cv2.imwrite(p, img)
        paths.append(p)
    db = []
    for i in range(n):
        c = np.array([rng.uniform(70, 130), rng.uniform(70, 110)])
        joints, vis = np.zeros((16, 3)), np.zeros((16, 3))
        if i % 2:
            joints[:, :2] = c + rng.uniform(-40, 40, (16, 2))
            vis[:, :2] = 1.0
        db.append({"image": paths[i % 2], "filename": "", "imgnum": 0, "center": c, "scale": np.array([0.8, 0.8]),
                   "joints_3d": joints, "joints_3d_vis": vis})
    cfg = {"is_train": True, "color_rgb": True, "image_size": [128, 128], "heatmap_size": [32, 32], "sigma": 2,
           "scale_factor": 0.25, "rotation_factor": 30, "flip": True, "num_joints_half_body": 8,
           "prob_half_body": 0.3, "num_joints": 16, "flip_pairs": MPII_FLIP,
           "upper_body_ids": [7, 8, 9, 10, 11, 12, 13, 14, 15], "mean": [0.485, 0.456, 0.406],
           "std": [0.229, 0.224, 0.225]}
    return StandInDataset(cfg, db)


def _device_loader(base):
    from fpd_b200.augment import DeviceCropLoader, RawJointsDataset, raw_collate
    loader = torch.utils.data.DataLoader(RawJointsDataset(base), batch_size=4, shuffle=False, collate_fn=raw_collate)
    return DeviceCropLoader(loader, (32, 32), 2)


def _seed(s):
    np.random.seed(s)
    random.seed(s)


def test_end_to_end_mixed_dataset(tmp_path, monkeypatch):
    pytest.importorskip("cv2")
    from fpd_b200 import ops
    from fpd_b200.lib.core import function as F
    from fpd_b200.lib.core.evaluate import pck_from_counts
    from fpd_b200.train_step import FPDTrainStep
    base = _mixed_dataset(tmp_path)
    init_s, init_t = _inits(17)
    _seed(3)
    batches = list(_device_loader(base))
    for _, target, tw, _ in batches:
        unl = (tw.reshape(4, -1) == 0).all(1)
        assert unl.tolist() == [True, False, True, False] and not target[unl].any()
    # PCK counts of a mixed batch are those of its labeled samples alone
    s, t = _net(64, 2, init_s), _net(64, 1, init_t)
    step = FPDTrainStep(s, t, alpha=0.5, use_graph=False, accuracy=True, kd_unlabeled_thre=THRE)
    x, target, tw, _ = batches[0]
    step.step(x, target, tw)
    lab = torch.tensor([1, 3], device="cuda")
    _, idx, mx = ops.flip_merge_argmax(step.last_outs[-1][lab].contiguous(), want_avg=False)
    alone, _ = ops.pck_counts(idx, mx, target[lab].contiguous())
    assert torch.equal(step.counts, alone)
    # one epoch of fpd_train on both fused routes, the loader's draws seeded alike
    cfg = _cfg(64, 2, {"UNLABELED": True, "UNLABELED_THRE": THRE})
    runs = []
    for graph in (True, False):
        monkeypatch.setattr(F, "_TRAIN_GRAPH", graph)
        F._train_step_cache.clear()
        _seed(3)
        runs.append(_fpd_epoch(F, cfg, _device_loader(base), init_s, init_t))
    F._train_step_cache.clear()
    (sd_g, _, sc_g), (sd_e, _, sc_e) = runs
    assert all(torch.equal(sd_g[k], sd_e[k]) for k in sd_g)
    assert sc_g == sc_e and all(np.isfinite(v) for _, v, _ in sc_g)
    _, avg, cnt = pck_from_counts(alone.cpu().numpy())
    assert cnt > 0
