"""Distilling from a teacher at its own input size, on the H100: fpd_heatmap_resample against its fp64 restatement, the
teacher's crop through DeviceCropLoader against cv2, FPDTrainStep with a 384x288 teacher against the oracle, unlabeled
weights from the teacher's own map, the graph / eager / generic routes, and an fp16 teacher."""
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

import _augment_cases as C  # noqa: E402
import _parity as P  # noqa: E402
from test_teacher_size_cpu import resample_heatmaps, teacher_size  # noqa: E402

pytestmark = pytest.mark.gpu

G = C.golden()
TOL = 1e-3      # a network forward against the oracle's, as the existing FPD step tests


@pytest.fixture(scope="module", autouse=True)
def _fp32_reference_mode():
    tf = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf


def _nchw(t):
    return t.permute(0, 3, 1, 2).contiguous()


# ------------------------------------------------------------------------------------------------ the kernel
@pytest.mark.parametrize("sizes", [((96, 72), (64, 48)), ((128, 96), (64, 48)), ((48, 36), (64, 48))])
@pytest.mark.parametrize("udp", [False, True])
@pytest.mark.parametrize("C_", [16, 17])
@pytest.mark.parametrize("B", [1, 5])
def test_kernel_matches_fp64_restatement(sizes, udp, C_, B):
    from fpd_b200 import ops
    (Hi, Wi), (Ho, Wo) = sizes
    g = torch.Generator(device="cuda").manual_seed(Hi + C_ + B + udp)
    hm = torch.randn(B, Hi, Wi, C_, generator=g, device="cuda")
    out = ops.resample_heatmaps(hm, (Ho, Wo), udp=udp)
    ref = resample_heatmaps(hm.cpu().numpy(), (Ho, Wo), udp)
    got = out.cpu().numpy().astype(np.float64)
    assert out.shape == (B, Ho, Wo, C_)
    assert np.abs(got - ref).max() <= 1e-6 * np.abs(ref).max()
    # repeats and a graph replay give the same bits
    assert torch.equal(ops.resample_heatmaps(hm, (Ho, Wo), udp=udp), out)
    dst = torch.empty_like(out)
    ops.resample_heatmaps(hm, (Ho, Wo), udp=udp, out=dst)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.resample_heatmaps(hm, (Ho, Wo), udp=udp, out=dst)
    dst.fill_(float("nan"))
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(dst, out)


@pytest.mark.parametrize("udp", [False, True])
def test_equal_sizes_copy_exactly(udp):
    from fpd_b200 import ops
    hm = torch.randn(3, 64, 48, 17, device="cuda")
    hm[0, 5, 6, 2] = float("inf")          # a neighbour that is not finite leaves the copy exact
    hm[1, 7, 7, 3] = float("nan")
    out = ops.resample_heatmaps(hm, (64, 48), udp=udp)
    assert torch.equal(out.nan_to_num(0.0), hm.nan_to_num(0.0)) and torch.isnan(out[1, 7, 7, 3])


# ------------------------------------------------------------------------------------------------ the crops
@pytest.mark.parametrize("tag", C.sets(G))
def test_device_loader_teacher_crop_matches_cv2(tag, tmp_path):
    cv2 = pytest.importorskip("cv2")
    from fpd_b200 import augment as A
    from oracle import augment_oracle as O
    paths = C.write_images(G, tmp_path)
    size = C.out_size(G, tag)
    tsize = teacher_size(size)
    mean, std = G["mean"].astype(np.float32), G["std"].astype(np.float32)

    def load(**kw):
        ds = C.stand_in(G, tag, paths)
        raw = A.RawJointsDataset(ds, **kw)
        loader = torch.utils.data.DataLoader(raw, batch_size=len(raw), shuffle=False, num_workers=0,
                                             collate_fn=A.raw_collate, pin_memory=True)
        C.seed(G, tag)
        return list(A.DeviceCropLoader(loader, ds.heatmap_size, ds.sigma))
    (inp0, t0, w0, _), = load()
    (inp, tg, tw, meta), = load(teacher_image_size=tsize)
    assert torch.equal(inp, inp0) and torch.equal(tg, t0) and torch.equal(tw, w0)     # the student's batch is unchanged
    tin = meta["teacher_input"]
    assert tin.is_cuda and tuple(tin.shape) == (inp.shape[0], 3, tsize[1], tsize[0]) and meta["teacher_udp"] is False
    for i in range(inp.shape[0]):
        fwd = A.crop_matrix(meta["center"][i].numpy(), meta["scale"][i].numpy(), float(meta["rotation"][i]), tsize)
        ref = cv2.warpAffine(C.source(G, tag, i), fwd, tsize, flags=cv2.INTER_LINEAR)
        assert torch.equal(tin[i].cpu(), torch.from_numpy(O.normalize(ref, mean, std))), i


# ------------------------------------------------------------------------------------------------ networks
class _Cfg(dict):
    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            raise AttributeError(k)


def _wrap(d):
    return _Cfg({k: _wrap(v) for k, v in d.items()}) if isinstance(d, dict) else d


def _hrnet(w):
    from fpd_b200.lib.models import pose_hrnet as H

    def stage(nmod, chans):
        return dict(NUM_MODULES=nmod, NUM_BRANCHES=len(chans), BLOCK='BASIC', NUM_BLOCKS=[1] * len(chans),
                    NUM_CHANNELS=chans, FUSE_METHOD='SUM')
    st = (stage(1, [w, 2 * w]), stage(1, [w, 2 * w, 4 * w]), stage(1, [w, 2 * w, 4 * w, 8 * w]))
    return H.get_pose_net(_wrap(dict(MODEL=dict(NUM_JOINTS=17, INIT_WEIGHTS=False, PRETRAINED='', EXTRA=dict(
        PRETRAINED_LAYERS=['*'], FINAL_CONV_KERNEL=1, STAGE2=st[0], STAGE3=st[1], STAGE4=st[2])))),
        is_train=False).cuda()


def _resnet50():
    from bench import resnet_cfg
    from fpd_b200.lib.models import pose_resnet as R
    from oracle import resnet_oracle as RO
    net = R.get_pose_net(resnet_cfg(50, 17), False)
    net.load_state_dict(RO.synthetic_state({k: v.shape for k, v in net.state_dict().items()}, seed=3))
    return net.cuda()


def _hg(f, s, sd=None):
    from fpd_b200.lib.models import hourglass as H
    net = H.get_pose_net(NS(MODEL=NS(EXTRA=NS(NUM_FEATURES=f, NUM_STACKS=s, NUM_BLOCKS=1), NUM_JOINTS=16)), True)
    if sd is not None:
        net.load_state_dict(sd)
    return net.cuda()


def _batch(B, seed, H, W, J, scale=1.5):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, 3, H, W, generator=g, device="cuda")
    tx = torch.randn(B, 3, int(H * scale), int(W * scale), generator=g, device="cuda")
    target = torch.rand(B, J, H // 4, W // 4, generator=g, device="cuda")
    tw = (torch.rand(B, J, 1, generator=g, device="cuda") > 0.2).float()
    return x, tx, target, tw


# ------------------------------------------------------------------------------------------------ step against the oracle
def _oracle_step(s_sd, t_rs, x, target, tw, alpha, dtype):
    from oracle import hourglass_oracle as O
    from oracle import hrnet_oracle as HO
    sd = P.cast_sd(s_sd, dtype)
    params = P.with_grad(sd)
    outs = [HO.hrnet(HO.annotate_strides(sd), x.to(dtype), training=True)]
    total, pose, kd = O.fpd_loss(outs, target.to(dtype), tw.to(dtype), t_rs.to(dtype), alpha)
    total.backward()
    return [float(v.detach()) for v in (pose, kd, total)], {k: p.grad.detach() for k, p in params.items()}


@pytest.mark.parametrize("teacher_kind", ["hrnet_w48", "pose_resnet50"])
def test_step_with_a_384x288_teacher_matches_the_oracle(teacher_kind):
    from fpd_b200.train_step import FPDTrainStep
    from oracle import hrnet_oracle as HO
    from oracle import resnet_oracle as RO
    torch.manual_seed(5)
    student = _hrnet(32)
    if teacher_kind == "hrnet_w48":
        teacher = _hrnet(48)
        for m in teacher.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                m.running_mean.normal_(0, 0.1)
                m.running_var.uniform_(0.5, 1.5)

        def t_oracle(sd, x):
            return HO.hrnet(HO.annotate_strides(sd), x, training=False)
    else:
        teacher = _resnet50()

        def t_oracle(sd, x):
            return RO.resnet(sd, x, training=False)
    s_sd = {k: v.detach().clone() for k, v in student.state_dict().items()}
    t_sd = {k: v.detach().clone() for k, v in teacher.state_dict().items()}
    x, tx, target, tw = _batch(2, 7, 256, 192, 17)
    alpha = 0.5
    step = FPDTrainStep(student, teacher, alpha=alpha, fused_adam=False)
    losses = [float(v) for v in step.step(x, target, tw, teacher_x=tx).cpu()]
    got = {k: g.clone() for (k, _), g in zip(student.named_parameters(), step.grad_views)}
    native = step._t_keep.outs[-1].data
    assert tuple(native.shape) == (2, 96, 72, 17) and tuple(step.last_teacher.shape) == (2, 64, 48, 17)
    # the teacher's forward on its own crop against the fp32 oracle's
    with torch.no_grad():
        ref_t = t_oracle(P.cast_sd(t_sd, torch.float32), tx)
    assert P.rel_max(_nchw(native), ref_t) < TOL
    # the resample against its fp64 restatement, and the loss on the map it produced
    t_rs = resample_heatmaps(native.cpu().numpy(), (64, 48))
    assert np.abs(step.last_teacher.cpu().numpy() - t_rs).max() <= 1e-6 * np.abs(t_rs).max()
    t_rs = torch.from_numpy(t_rs).cuda().permute(0, 3, 1, 2)
    l32, g32 = _oracle_step(s_sd, t_rs, x, target, tw, alpha, torch.float32)
    l64, g64 = _oracle_step(s_sd, t_rs, x, target, tw, alpha, torch.float64)
    for v, r, r32 in zip(losses, l64, l32):
        # 1e-5 relative, or no further from fp64 than the oracle's own fp32 evaluation gets
        assert abs(v - r) <= max(1e-5 * abs(r), 2 * abs(r32 - r)), (v, r, r32)
    gmax = max(float(v.abs().max()) for v in g64.values())
    zero = {k for k in got if k.endswith(".bias") and k != "final_layer.bias" and float(g64[k].abs().max()) <= 1e-12 * gmax}
    for k in zero:
        assert float(got[k].abs().max()) <= 1e-5 * gmax, k
    P.assert_grads_as_good_as_fp32({k: v for k, v in got.items() if k not in zero},
                                   {k: v for k, v in g32.items() if k not in zero},
                                   {k: v for k, v in g64.items() if k not in zero}, "teacher size %s" % teacher_kind)


# ------------------------------------------------------------------------------------------------ unlabeled weights
def test_kd_weights_read_the_teachers_own_map(monkeypatch):
    from fpd_b200 import ops, train_step
    thre = 0.2
    # a one-pixel peak at teacher pixel (1, 1): no student pixel samples it at more than a quarter of its height
    native = torch.zeros(1, 96, 72, 17, device="cuda")
    native[0, 1, 1, :] = 0.5
    tw = torch.zeros(1, 17, device="cuda")
    rs = ops.resample_heatmaps(native, (64, 48))
    assert float(rs.max()) <= thre < float(native.max())
    assert torch.equal(ops.kd_weights(native, tw, thre), torch.ones(1, 17, device="cuda"))
    assert torch.equal(ops.kd_weights(rs, tw, thre), torch.zeros(1, 17, device="cuda"))
    # the step hands kd_weights the teacher's own map, not the resampled one
    seen = []
    orig = ops.kd_weights

    def rec(t, *a, **k):
        seen.append((tuple(t.shape), t.data_ptr()))
        return orig(t, *a, **k)
    monkeypatch.setattr(ops, "kd_weights", rec)
    torch.manual_seed(2)
    step = train_step.FPDTrainStep(_hg(64, 1), _hg(64, 1), alpha=0.5, use_graph=False, kd_unlabeled_thre=thre)
    x, tx, target, tw4 = _batch(2, 3, 128, 128, 16)
    tw4[0] = 0.0
    step.step(x, target, tw4, teacher_x=tx)
    assert seen == [((2, 48, 48, 16), step._t_keep.outs[-1].data.data_ptr())]


# ------------------------------------------------------------------------------------------------ routes
def _inits(seed):
    torch.manual_seed(seed)
    return ({k: v.clone() for k, v in _hg(64, 2).state_dict().items()},
            {k: v.clone() for k, v in _hg(64, 1).state_dict().items()})


def test_graph_and_eager_steps_are_bit_identical():
    from fpd_b200.train_step import FPDTrainStep
    init_s, init_t = _inits(4)
    batches = [_batch(3, 10 + i, 128, 128, 16) for i in range(2)]
    runs = []
    for use_graph in (True, False):
        s = _hg(64, 2, init_s)
        step = FPDTrainStep(s, _hg(64, 1, init_t), alpha=0.5, lr=1e-3, use_graph=use_graph, kd_unlabeled_thre=0.1)
        ls = [step.step(x, t, w, teacher_x=tx).clone() for x, tx, t, w in batches]
        torch.cuda.synchronize()
        runs.append((torch.stack(ls), step.flat.flat.clone(), step.exp_avg.clone(), step.exp_avg_sq.clone(),
                     [b.clone() for b in s.buffers()]))
    (lg, fg, ag, qg, bg), (le, fe, ae, qe, be) = runs
    assert torch.equal(lg, le) and torch.equal(fg, fe) and torch.equal(ag, ae) and torch.equal(qg, qe)
    assert all(torch.equal(a, b) for a, b in zip(bg, be))
    # the teacher's own input changes the step
    s = _hg(64, 2, init_s)
    plain = FPDTrainStep(s, _hg(64, 1, init_t), alpha=0.5, lr=1e-3, kd_unlabeled_thre=0.1)
    x, _, t, w = batches[0]
    assert not torch.equal(plain.step(x, t, w).clone(), lg[0])


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


def _dataset(tmp_path, n=6):
    """A stand-in MPII training set over synthetic images, 128x128 crops."""
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
        joints[:, :2] = c + rng.uniform(-40, 40, (16, 2))
        vis[:, :2] = 1.0
        db.append({"image": paths[i % 2], "filename": "", "imgnum": 0, "center": c, "scale": np.array([0.8, 0.8]),
                   "joints_3d": joints, "joints_3d_vis": vis})
    flip = [[0, 5], [1, 4], [2, 3], [10, 15], [11, 14], [12, 13]]
    cfg = {"is_train": True, "color_rgb": True, "image_size": [128, 128], "heatmap_size": [32, 32], "sigma": 2,
           "scale_factor": 0.25, "rotation_factor": 30, "flip": True, "num_joints_half_body": 8,
           "prob_half_body": 0.3, "num_joints": 16, "flip_pairs": flip, "upper_body_ids": [7, 8, 9, 10, 11, 12, 13, 14, 15],
           "mean": [0.485, 0.456, 0.406], "std": [0.229, 0.224, 0.225]}
    return StandInDataset(cfg, db)


def _fpd_epoch(F, cfg, base, init_s, init_t, generic=False):
    from fpd_b200.augment import DeviceCropLoader, RawJointsDataset, raw_collate
    from fpd_b200.lib.core.loss import JointsMSELoss
    np.random.seed(3)
    random.seed(3)
    loader = torch.utils.data.DataLoader(RawJointsDataset(base, teacher_image_size=(192, 192)), batch_size=4,
                                         shuffle=False, collate_fn=raw_collate)      # a short last batch of 2
    loader = DeviceCropLoader(loader, (32, 32), 2)
    s, t = _hg(64, 2, init_s), _hg(64, 1, init_t)
    opt = torch.optim.Adam(s.parameters(), lr=1e-3)
    wd = {"writer": _Writer(), "train_global_steps": 0}
    F.fpd_train(cfg, loader, _Hide(s) if generic else s, t, JointsMSELoss(True), JointsMSELoss(True), opt, 0, "/tmp",
                "/tmp", wd)
    torch.cuda.synchronize()
    sd = {k: v.clone() for k, v in s.state_dict().items()}
    ost = [(k, v.clone() if torch.is_tensor(v) else v) for st in opt.state.values() for k, v in sorted(st.items())]
    return sd, ost, wd["writer"].scalars


def test_fpd_train_routes_agree_with_a_teacher_crop(tmp_path, monkeypatch):
    pytest.importorskip("cv2")
    from fpd_b200.lib.core import function as F
    base = _dataset(tmp_path)
    init_s, init_t = _inits(13)
    cfg = NS(KD=NS(ALPHA=0.5), PRINT_FREQ=1, DEBUG=NS(DEBUG=False))
    runs = []
    for graph in (True, False):
        monkeypatch.setattr(F, "_TRAIN_GRAPH", graph)
        F._train_step_cache.clear()
        runs.append(_fpd_epoch(F, cfg, base, init_s, init_t))
    F._train_step_cache.clear()
    (sd_g, os_g, sc_g), (sd_e, os_e, sc_e) = runs
    assert all(torch.equal(sd_g[k], sd_e[k]) for k in sd_g)
    assert all(a[0] == b[0] and (torch.equal(a[1], b[1]) if torch.is_tensor(a[1]) else a[1] == b[1])
               for a, b in zip(os_g, os_e))
    assert sc_g == sc_e and len(sc_g) > 0
    sd_x, _, sc_x = _fpd_epoch(F, cfg, base, init_s, init_t, generic=True)
    assert len(sc_x) == len(sc_e)
    for (tf, vf, _), (tg, vg, _) in zip(sc_e, sc_x):
        assert tf == tg and abs(vf - vg) <= 1e-4 * max(1.0, abs(vg)), (tf, vf, vg)
    worst = max(((sd_e[k].double() - sd_x[k].double()).abs().max() / sd_x[k].double().abs().max().clamp_min(1e-12))
                .item() for k in sd_e if sd_e[k].is_floating_point())
    assert worst < 1e-4, worst


# ------------------------------------------------------------------------------------------------ teacher precision
def test_fp16_teacher_with_its_own_input():
    from fpd_b200.engine import set_inference_precision
    from fpd_b200.train_step import FPDTrainStep
    init_s, init_t = _inits(6)
    x, tx, t, w = _batch(2, 21, 128, 128, 16)
    res = {}
    for prec in ("fp32", "fp16"):
        teacher = _hg(64, 1, init_t)
        set_inference_precision(teacher, prec)
        step = FPDTrainStep(_hg(64, 2, init_s), teacher, alpha=0.5, fused_adam=False)
        res[prec] = (step.step(x, t, w, teacher_x=tx).clone(), step.last_teacher.clone())
        torch.cuda.synchronize()
    (l32, t32), (l16, t16) = res["fp32"], res["fp16"]
    assert torch.isfinite(l16).all() and t16.dtype == torch.float32
    assert P.rel_max(t16, t32) <= 1e-2               # the fp16 inference tests' bound on a network output
    assert P.rel_max(l16, l32) <= 1e-2
