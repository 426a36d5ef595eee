"""JointsOHKMMSELoss on the device: the module form and the fused FPD form against the reference's golden values and
gradients and against the fp64 oracle at training shapes, graph replay, the training loops' fused route against the
generic autograd route, validate()'s graph route against its eager route, and argument checks."""
import ctypes
import os
import sys
import types

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
NS = types.SimpleNamespace
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


@pytest.fixture(scope="module")
def z():
    d = np.load(os.path.join(ROOT, "tests", "golden", "ohkm.npz"), allow_pickle=False)
    return {k: d[k] for k in d.files}


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a.astype(np.float32))).cuda()


def _nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def _nchw(t):
    return t.permute(0, 3, 1, 2).contiguous()


def _grad_close(got, ref, tol=1e-6):
    got = got.detach().double().cpu()
    ref = torch.as_tensor(ref).double().cpu()
    assert torch.equal(got != 0, ref != 0), "selected joints differ"
    err = (got - ref).abs().max().item()
    assert err <= tol * ref.abs().max().item(), (err, ref.abs().max().item())


def _rel(a, b):
    return abs(float(a) - float(b)) / abs(float(b))


def _tags(z, prefix):
    return sorted({k.split("/")[0] for k in z if k.startswith(prefix)})


def _ohkm_fused_raw(outs, target, teacher, tw, alpha, pk, kk, grads=True):
    """fpd_loss_ohkm_fused itself (ops.fpd_loss takes the MSE entry point when both topk are 0)."""
    import fpd_b200  # noqa: F401
    from fpd_b200 import _native as N
    from fpd_b200 import ops
    S = len(outs)
    B, h, w, J = outs[0].shape
    losses = torch.empty(3, device="cuda")
    gl = [torch.empty_like(o) for o in outs] if grads else None
    arr = (ctypes.c_void_p * S)(*[o.data_ptr() for o in outs])
    garr = (ctypes.c_void_p * S)(*[g.data_ptr() for g in gl]) if grads else None
    ws = torch.empty(N.lib().fpd_loss_ohkm_workspace_bytes(S, B, J, h, w), dtype=torch.uint8, device="cuda")
    rc = N.lib().fpd_loss_ohkm_fused(arr, S, ops._p(target), ops._p(teacher), ops._p(tw), float(alpha), garr, 1.0,
                                     ops._p(losses), B, J, h, w, pk, kk, ops._p(ws), ws.numel(), ops._stream())
    return rc, losses, gl


# ------------------------------------------------------------------------------------------------ golden vectors
def test_module_matches_reference_golden(z):
    import fpd_b200  # noqa: F401
    from fpd_b200.lib.core.loss import JointsOHKMMSELoss
    for t in _tags(z, "m"):
        use_tw = bool(z[t + "/use_target_weight"])
        out = _cuda(z[t + "/out"]).requires_grad_(True)
        crit = JointsOHKMMSELoss(use_tw, topk=int(z[t + "/topk"]))
        loss = crit(out, _cuda(z[t + "/target"]), _cuda(z[t + "/target_weight"]))
        assert loss.dim() == 0
        loss.backward()
        assert _rel(loss.item(), z[t + "/loss"]) <= 1e-6, (t, loss.item(), float(z[t + "/loss"]))
        _grad_close(out.grad, z[t + "/grad"])


def _fpd_case(z, t):
    B = z[t + "/target"].shape[0]
    J = z[t + "/target"].shape[1]
    outs = [_nhwc(_cuda(o)) for o in z[t + "/outs"]]
    tw = _cuda(z[t + "/target_weight"]).reshape(B, J) if z[t + "/use_target_weight"] else torch.ones(B, J, device="cuda")
    return (outs, _cuda(z[t + "/target"]), _nhwc(_cuda(z[t + "/teacher"])), tw.contiguous(), float(z[t + "/alpha"]),
            int(z[t + "/pose_topk"]), int(z[t + "/kd_topk"]))


def _per_stack_modules(outs, target, teacher, tw, alpha, pk, kk):
    """The FPD combination from the module form, stack by stack and term by term, on the device."""
    from fpd_b200 import ops

    def crit(o, ref, k):
        if k:
            return ops.joints_ohkm_mse(o, ref, tw, k)
        return ops.joints_mse(o, ref, tw)
    pose = kd = 0.0
    grads = []
    t_nchw = _nchw(teacher)
    for o in outs:
        on = _nchw(o)
        (lp, gp), (lk, gk) = crit(on, target, pk), crit(on, t_nchw, kk)
        pose += lp[0].double().item()
        kd += lk[0].double().item()
        grads.append(_nhwc((1 - alpha) * gp.double() + alpha * gk.double()))
    return pose, kd, (1 - alpha) * pose + alpha * kd, grads


def test_fused_form_matches_reference_golden_and_module_form(z):
    import fpd_b200  # noqa: F401
    from fpd_b200 import ops
    tags = _tags(z, "f")
    assert len(tags) == 4
    for t in tags:
        outs, target, teacher, tw, alpha, pk, kk = _fpd_case(z, t)
        runs = [ops.fpd_loss(outs, target, teacher, tw, alpha, pose_topk=pk, kd_topk=kk)]
        rc, l_raw, g_raw = _ohkm_fused_raw(outs, target, teacher, tw, alpha, pk, kk)
        assert rc == 0
        runs.append((l_raw, g_raw))
        mod = _per_stack_modules(outs, target, teacher, tw, alpha, pk, kk)
        for losses, grads in runs:
            for got, ref, m in zip(losses.cpu().tolist(), z[t + "/losses"], mod[:3]):
                assert _rel(got, ref) <= 1e-6, (t, got, float(ref))
                assert _rel(got, m) <= 1e-6, (t, got, m)
            for g, ref, m in zip(grads, z[t + "/grads"], mod[3]):
                _grad_close(_nchw(g), ref)
                _grad_close(g, m)


# ------------------------------------------------------------------------------------------------ training shapes
def _draw(gen, B, J, h, w, S):
    """Heat-map-like maps: targets in [0, 1), stacks = target + noise whose size varies per (b, j) -> spread-out
    per-joint losses."""
    tgt = torch.rand(B, J, h, w, generator=gen, device="cuda")
    amp = lambda: 0.05 + torch.rand(B, J, 1, 1, generator=gen, device="cuda")  # noqa: E731
    outs = [tgt + amp() * torch.randn(B, J, h, w, generator=gen, device="cuda") for _ in range(S)]
    teacher = tgt + amp() * torch.randn(B, J, h, w, generator=gen, device="cuda")
    tw = (torch.rand(B, J, 1, generator=gen, device="cuda") > 0.15).float()
    return outs, tgt, teacher, tw


def _guarded(seed, B, J, h, w, S, topk):
    """_draw, with every sample whose selection boundary is within 1e-4 relative (oracle.ohkm_oracle.boundary_ok, per
    stack and term) drawn again."""
    from oracle import ohkm_oracle as O
    gen = torch.Generator(device="cuda").manual_seed(seed)
    outs, tgt, teacher, tw = _draw(gen, B, J, h, w, S)
    for _ in range(20):
        bad = set()
        for o in outs:
            for ref in (tgt, teacher):
                l = O.per_joint(o, ref, tw)[0].cpu()
                bad |= {b for b in range(B) if not O.boundary_ok(l[b], topk)}
        if not bad:
            return outs, tgt, teacher, tw
        o2, t2, te2, tw2 = _draw(gen, B, J, h, w, S)
        for b in bad:
            for o, n in zip(outs, o2):
                o[b] = n[b]
            tgt[b], teacher[b], tw[b] = t2[b], te2[b], tw2[b]
    raise AssertionError("tie guard did not converge")


@pytest.mark.parametrize("B,J,h,w,S", [(32, 16, 64, 64, 4), (24, 17, 64, 48, 1)])
def test_training_shapes_match_fp64_oracle(B, J, h, w, S):
    import fpd_b200  # noqa: F401
    from fpd_b200 import ops
    from oracle import ohkm_oracle as O
    topk, alpha = 8, 0.5
    outs, tgt, teacher, tw = _guarded(B * 100 + J, B, J, h, w, S, topk)
    twf = tw.reshape(B, J).contiguous()
    for pk, kk in ((topk, topk), (topk, 0), (0, topk)):
        losses, grads = ops.fpd_loss([_nhwc(o) for o in outs], tgt, _nhwc(teacher), twf, alpha, pose_topk=pk, kd_topk=kk)
        pose, kd, total, rgrads = O.fpd(outs, tgt, teacher, tw, alpha, pk, kk)
        for got, ref in zip(losses.cpu().tolist(), (pose, kd, total)):
            assert _rel(got, ref.item()) <= 1e-5, (pk, kk, got, ref.item())
        for g, r in zip(grads, rgrads):
            _grad_close(_nchw(g), r)
    # the module form on the last stack, with and without weights
    for weights in (tw, None):
        loss3, grad = ops.joints_ohkm_mse(outs[-1], tgt, weights, topk)
        v, rg = O.criterion(outs[-1], tgt, weights, topk)
        assert _rel(loss3[0].item(), v.item()) <= 1e-5
        assert loss3[1].item() == 0.0 and loss3[2].item() == loss3[0].item()
        _grad_close(grad, rg)


def test_batch_of_one_and_selection_ties():
    import fpd_b200  # noqa: F401
    from fpd_b200 import ops
    from oracle import ohkm_oracle as O
    gen = torch.Generator(device="cuda").manual_seed(3)
    o = torch.rand(1, 16, 8, 8, generator=gen, device="cuda")
    g = torch.rand(1, 16, 8, 8, generator=gen, device="cuda")
    loss3, grad = ops.joints_ohkm_mse(o, g, None, 5)
    v, rg = O.criterion(o, g, None, 5)
    assert _rel(loss3[0].item(), v.item()) <= 1e-6
    _grad_close(grad, rg)
    # exact ties: joints 2..9 have identical maps -> the lowest indices are selected
    g[:, 2:10] = g[:, 2:3].clone()
    o = g.clone()
    o[:, 2:10] += 0.5
    o[:, 12] += 0.25
    _, grad = ops.joints_ohkm_mse(o, g, None, 4)
    sel = (grad.abs().amax(dim=(2, 3)) > 0)[0].cpu().tolist()
    assert sel == [j in (2, 3, 4, 5) for j in range(16)]


# ------------------------------------------------------------------------------------------------ graph capture
def test_graph_replay_is_bit_identical_to_eager():
    import fpd_b200  # noqa: F401
    from fpd_b200 import ops
    B, J, h, w, S = 8, 16, 64, 64, 3
    gen = torch.Generator(device="cuda").manual_seed(9)
    sets = [_draw(gen, B, J, h, w, S) for _ in range(3)]

    def prep(s):
        outs, tgt, teacher, tw = s
        return [_nhwc(o) for o in outs], tgt.contiguous(), _nhwc(teacher), tw.reshape(B, J).contiguous()
    st_outs, st_tgt, st_teacher, st_tw = prep(sets[0])
    st_grads = [torch.empty_like(o) for o in st_outs]
    st_losses = torch.empty(3, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ops.fpd_loss(st_outs, st_tgt, st_teacher, st_tw, 0.4, grads_out=st_grads, losses_out=st_losses, pose_topk=8,
                     kd_topk=8)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.fpd_loss(st_outs, st_tgt, st_teacher, st_tw, 0.4, grads_out=st_grads, losses_out=st_losses, pose_topk=8,
                     kd_topk=8)
    for s in sets[1:]:
        outs, tgt, teacher, tw = prep(s)
        ref_l, ref_g = ops.fpd_loss(outs, tgt, teacher, tw, 0.4, pose_topk=8, kd_topk=8)
        for d, src in zip(st_outs + [st_tgt, st_teacher, st_tw], outs + [tgt, teacher, tw]):
            d.copy_(src)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(st_losses, ref_l)
        assert all(torch.equal(a, b) for a, b in zip(st_grads, ref_g))
    # and eager calls repeat themselves bit for bit
    again_l, again_g = ops.fpd_loss(outs, tgt, teacher, tw, 0.4, pose_topk=8, kd_topk=8)
    assert torch.equal(again_l, ref_l) and all(torch.equal(a, b) for a, b in zip(again_g, ref_g))


# ------------------------------------------------------------------------------------------------ training loops
def _cfg(f, s):
    return NS(MODEL=NS(EXTRA=NS(NUM_FEATURES=f, NUM_STACKS=s, NUM_BLOCKS=1), NUM_JOINTS=16, NAME="hourglass"),
              KD=NS(ALPHA=0.5), PRINT_FREQ=1,
              TEST=NS(FLIP_TEST=True, SHIFT_HEATMAP=True, POST_PROCESS=True), DEBUG=NS(DEBUG=False))


def _net(f, s, sd=None):
    from fpd_b200.lib.models import hourglass as H
    net = H.get_pose_net(_cfg(f, s), True)
    if sd is not None:
        net.load_state_dict(sd)
    return net.cuda()


class _Hide(torch.nn.Module):
    """Wrapper that hides the engine attributes -> function.py takes the generic (reference-like) route."""

    def __init__(self, net):
        super().__init__()
        self.net = net

    def forward(self, x):
        return self.net(x.cuda())


def _loader(n, B=2, hw=128):
    from bench import synthetic_batch
    out = []
    for i in range(n):
        x, t, w = synthetic_batch(B, 70 + i, hw, hw)
        meta = {"center": torch.tensor([[64.0, 64.0]] * B), "scale": torch.tensor([[0.64, 0.64]] * B),
                "score": torch.ones(B), "image": ["img%d_%d" % (i, b) for b in range(B)]}
        out.append((x, t, w, meta))
    return out


class _Writer:
    def __init__(self):
        self.scalars = []

    def add_scalar(self, tag, v, step):
        self.scalars.append((tag, float(v), step))

    def add_scalars(self, tag, d, step):
        pass


def _compare_routes(results):
    (sd_f, sc_f), (sd_g, sc_g) = results
    assert len(sc_f) == len(sc_g)
    for (tf, vf, _), (tg, vg, _) in zip(sc_f, sc_g):
        assert tf == tg and abs(vf - vg) <= 1e-4 * max(1.0, abs(vg)), (tf, vf, vg)
    worst = max(((sd_f[k].double() - sd_g[k].double()).abs().max() / sd_g[k].double().abs().max().clamp_min(1e-12)).item()
                for k in sd_f if sd_f[k].is_floating_point())
    assert worst < 1e-4, worst


@pytest.mark.parametrize("pose,kd", [("ohkm", "ohkm"), ("ohkm", "mse"), ("mse", "ohkm")])
def test_fpd_train_fused_route_equals_generic_route(pose, kd, monkeypatch):
    """KD.ALPHA = 0.5: the fused gradient then has the generic route's bits (csrc/loss.cu rounds each term on its own),
    which matters here because Adam turns round-off in the gradients of conv biases ahead of a train-mode BatchNorm
    (zero up to round-off) into whole learning-rate steps."""
    import fpd_b200  # noqa: F401
    from fpd_b200.lib.core import function as F
    from fpd_b200.lib.core.loss import JointsMSELoss, JointsOHKMMSELoss

    def crit(kind):
        return JointsOHKMMSELoss(True, topk=6) if kind == "ohkm" else JointsMSELoss(True)
    torch.manual_seed(5)
    init_s = {k: v.clone() for k, v in _net(64, 2).state_dict().items()}
    init_t = {k: v.clone() for k, v in _net(64, 1).state_dict().items()}
    cfg = _cfg(64, 2)
    loader = _loader(2)
    results = []
    calls = []
    orig = F._fused_step
    monkeypatch.setattr(F, "_fused_step", lambda *a, **k: calls.append(k) or orig(*a, **k))
    for generic in (False, True):
        s, t = _net(64, 2, init_s), _net(64, 1, init_t)
        opt = torch.optim.Adam(s.parameters(), lr=1e-3)
        wd = {"writer": _Writer(), "train_global_steps": 0}
        F.fpd_train(cfg, loader, _Hide(s) if generic else s, t, crit(pose), crit(kd), opt, 0, "/tmp", "/tmp", wd)
        torch.cuda.synchronize()
        results.append(({k: v.clone() for k, v in s.state_dict().items()}, wd["writer"].scalars))
    assert calls == [{"pose_topk": 6 if pose == "ohkm" else 0, "kd_topk": 6 if kd == "ohkm" else 0}] * 2
    _compare_routes(results)


def test_train_fused_route_equals_generic_route(monkeypatch):
    import fpd_b200  # noqa: F401
    from fpd_b200.lib.core import function as F
    from fpd_b200.lib.core.loss import JointsOHKMMSELoss
    torch.manual_seed(6)
    init_s = {k: v.clone() for k, v in _net(64, 2).state_dict().items()}
    cfg = _cfg(64, 2)
    loader = _loader(2)
    calls = []
    orig = F._fused_step
    monkeypatch.setattr(F, "_fused_step", lambda *a, **k: calls.append(k) or orig(*a, **k))
    results = []
    for generic in (False, True):
        s = _net(64, 2, init_s)
        opt = torch.optim.Adam(s.parameters(), lr=1e-3)
        wd = {"writer": _Writer(), "train_global_steps": 0}
        F.train(cfg, loader, _Hide(s) if generic else s, JointsOHKMMSELoss(True, topk=4), opt, 0, "/tmp", "/tmp", wd)
        torch.cuda.synchronize()
        results.append(({k: v.clone() for k, v in s.state_dict().items()}, wd["writer"].scalars))
    assert calls == [{"pose_topk": 4}] * 2
    _compare_routes(results)


class _TinyNet(torch.nn.Module):
    """Carries the attributes of an fpd_b200 network (so the loops consider the fused route) but is a plain conv."""

    def __init__(self, J):
        super().__init__()
        self.conv = torch.nn.Conv2d(3, J, 3, padding=1)

    def engine(self):
        raise AssertionError("the fused route must not be taken")

    def forward_nhwc(self, x, training=False):
        raise AssertionError("the fused route must not be taken")

    def forward(self, x):
        return self.conv(x.cuda())


def test_loops_route_odd_heatmaps_to_generic_path():
    import fpd_b200  # noqa: F401
    from fpd_b200 import ops
    from fpd_b200.lib.core import function as F
    from fpd_b200.lib.core.loss import JointsOHKMMSELoss
    J, hw = 16, 30                                 # h*w = 900, not a multiple of 64
    assert not F._loss_shape_ok(None, J, hw, hw)
    gen = torch.Generator().manual_seed(1)
    loader = [(torch.randn(2, 3, hw, hw, generator=gen), torch.rand(2, J, hw, hw, generator=gen),
               (torch.rand(2, J, 1, generator=gen) > 0.2).float(), {}) for _ in range(2)]
    cfg = _cfg(64, 1)
    torch.manual_seed(0)
    net, tnet = _TinyNet(J).cuda(), _TinyNet(J).cuda()
    opt = torch.optim.Adam(net.parameters(), lr=1e-3)
    wd = {"writer": _Writer(), "train_global_steps": 0}
    F.fpd_train(cfg, loader, net, tnet, JointsOHKMMSELoss(True, 8), JointsOHKMMSELoss(True, 8), opt, 0, "/tmp", "/tmp", wd)
    F.train(cfg, loader, net, JointsOHKMMSELoss(True, 8), opt, 0, "/tmp", "/tmp", wd)
    assert wd["train_global_steps"] == 4
    assert all(np.isfinite(v) for _, v, _ in wd["writer"].scalars)
    # the fused kernel itself refuses the shape
    o = torch.rand(2, hw, hw, J, device="cuda")
    with pytest.raises(RuntimeError, match="multiple of 64"):
        ops.fpd_loss([o], torch.rand(2, J, hw, hw, device="cuda"), o, torch.ones(2, J, device="cuda"), 0.5, pose_topk=8)


# ------------------------------------------------------------------------------------------------ validate
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


def _batch(B, seed, hw, J):
    from bench import synthetic_batch
    x, t, w = synthetic_batch(B, seed, hw[0], hw[1], J)
    rng = np.random.RandomState(seed)
    meta = {"center": torch.from_numpy(rng.uniform(100, 500, (B, 2))), "scale": torch.from_numpy(rng.uniform(0.5, 3, (B, 2))),
            "score": torch.from_numpy(rng.uniform(0.5, 1, B)), "image": ["img%d_%d" % (seed, b) for b in range(B)]}
    return x, t, w, meta


class _ValSet:
    def __init__(self, n, J):
        self.n = n
        self.flip_pairs = [p for p in FLIP_PAIRS if max(p) < J]
        self.seen = None

    def __len__(self):
        return self.n

    def evaluate(self, cfg, preds, output_dir, all_boxes, image_path, filenames, imgnums):
        self.seen = (preds.copy(), all_boxes.copy(), list(image_path))
        return {"Mean": float(preds[..., :2].mean())}, float(preds[..., :2].mean())


@pytest.mark.parametrize("kind", ["hourglass", "hrnet"])
def test_validate_graph_route_equals_eager_route_with_ohkm(kind, monkeypatch):
    import fpd_b200  # noqa: F401
    from fpd_b200.lib.core import function as F
    from fpd_b200.lib.core.loss import JointsMSELoss, JointsOHKMMSELoss
    torch.manual_seed(11)
    net, hw, J = {"hourglass": _hourglass, "hrnet": _hrnet}[kind]()
    for m in net.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.running_mean.normal_(0, 0.1)
            m.running_var.uniform_(0.5, 1.5)
    net = net.cuda()
    loader = [_batch(3, 20, hw, J), _batch(3, 21, hw, J), _batch(2, 22, hw, J)]      # last batch partial
    cfg = NS(MODEL=NS(NUM_JOINTS=J, NAME=kind), PRINT_FREQ=2, DEBUG=NS(DEBUG=False),
             TEST=NS(FLIP_TEST=True, SHIFT_HEATMAP=True, POST_PROCESS=True))
    runs = []
    calls = []
    orig = F._GraphValidation.run
    monkeypatch.setattr(F._GraphValidation, "run", lambda self, *a: calls.append(self.topk) or orig(self, *a))
    for graph, crit in ((True, JointsOHKMMSELoss(True, topk=8)), (False, JointsOHKMMSELoss(True, topk=8)),
                        (True, JointsMSELoss(True))):
        monkeypatch.setattr(F, "_VALIDATE_GRAPH", graph)
        calls.clear()
        ds = _ValSet(8, J)
        wd = {"writer": _Writer(), "valid_global_steps": 0}
        perf = F.validate(cfg, loader, ds, net, crit, "/tmp", "/tmp", wd)
        assert calls == ([crit.topk if hasattr(crit, "topk") else 0] * 3 if graph else [])
        runs.append((perf, ds.seen, wd["writer"].scalars))
    (pg, sg, wg), (pe, se, we), (_, _, wm) = runs
    assert np.array_equal(sg[0], se[0]) and np.array_equal(sg[1], se[1]) and sg[2] == se[2]
    assert pg == pe
    assert wg == we and {t for t, _, _ in wg} == {"valid_loss", "valid_acc"}
    # the loss really is the OHKM one (the MSE graph gives another value, the same accuracy)
    lg = [v for t, v, _ in wg if t == "valid_loss"]
    lm = [v for t, v, _ in wm if t == "valid_loss"]
    assert lg != lm and [v for t, v, _ in wg if t == "valid_acc"] == [v for t, v, _ in wm if t == "valid_acc"]


# ------------------------------------------------------------------------------------------------ bad arguments
def test_bad_arguments_raise():
    import fpd_b200  # noqa: F401
    from fpd_b200 import _native as N
    from fpd_b200 import ops
    from fpd_b200.lib.core.loss import JointsOHKMMSELoss
    o = torch.rand(2, 16, 8, 8, device="cuda")
    tw = torch.ones(2, 16, 1, device="cuda")
    for k in (0, 17, -1):
        with pytest.raises(ValueError):
            JointsOHKMMSELoss(True, topk=k)(o, o, tw)
        with pytest.raises(ValueError):
            ops.joints_ohkm_mse(o, o, tw, k)
    with pytest.raises(RuntimeError):                                           # CPU tensors
        JointsOHKMMSELoss(True)(o.cpu(), o.cpu(), tw.cpu())
    with pytest.raises(ValueError):
        ops.joints_ohkm_mse(o.cpu(), o.cpu(), None, 8)
    o65 = torch.rand(1, 65, 8, 8, device="cuda")
    with pytest.raises(RuntimeError, match="J=65"):
        JointsOHKMMSELoss(False, topk=8)(o65, o65, None)
    # the fused form
    outs = [torch.rand(2, 8, 8, 16, device="cuda")]
    tgt, tw2 = torch.rand(2, 16, 8, 8, device="cuda"), torch.ones(2, 16, device="cuda")
    for pk, kk in ((17, 0), (-1, 8), (8, 17)):
        with pytest.raises(ValueError):
            ops.fpd_loss(outs, tgt, outs[0], tw2, 0.5, pose_topk=pk, kd_topk=kk)
    o65 = [torch.rand(1, 8, 8, 65, device="cuda")]
    with pytest.raises(RuntimeError, match="J=65"):
        ops.fpd_loss(o65, torch.rand(1, 65, 8, 8, device="cuda"), None, torch.ones(1, 65, device="cuda"), 0.5, pose_topk=8)
    with pytest.raises(ValueError):
        ops.fpd_loss([x.cpu() for x in outs], tgt.cpu(), None, tw2.cpu(), 0.5, pose_topk=8)
    # the C entry points check their arguments on the host
    assert _ohkm_fused_raw(outs, tgt, outs[0], tw2, 0.5, 0, 17)[0] != 0          # topk > J
    assert _ohkm_fused_raw(outs, tgt, None, tw2, 0.5, 8, 8)[0] != 0              # kd_topk without a teacher
    assert _ohkm_fused_raw(outs, tgt, outs[0], None, 0.5, 8, 8)[0] != 0          # no target weight
    ws = torch.empty(1 << 16, dtype=torch.uint8, device="cuda")
    loss3 = torch.empty(3, device="cuda")
    lib, p, st = N.lib(), ops._p, ops._stream()
    assert lib.fpd_joints_ohkm(p(o), p(o), None, 8, p(loss3), None, 0, 16, 64, p(ws), ws.numel(), st) != 0   # N = 0
    assert lib.fpd_joints_ohkm(p(o), p(o), None, 0, p(loss3), None, 2, 16, 64, p(ws), ws.numel(), st) != 0   # topk 0
    assert lib.fpd_joints_ohkm(None, p(o), None, 8, p(loss3), None, 2, 16, 64, p(ws), ws.numel(), st) != 0   # NULL
    assert lib.fpd_joints_ohkm(p(o), p(o), None, 8, p(loss3), None, 2, 16, 64, p(ws), 16, None) != 0          # workspace
    assert "workspace" in N.last_error()
    assert lib.fpd_joints_ohkm_workspace_bytes(2, 16) <= ws.numel()
    assert lib.fpd_joints_ohkm(p(o), p(o), None, 8, p(loss3), None, 2, 16, 64, p(ws), ws.numel(), st) == 0
