"""JointsKLDLoss on the device: the module form and the fused FPD form against the fp64 model (tests/_kld_model.py) at
training shapes and temperatures, overflow, exact zeros, NaN propagation, poisoned gradient buffers, graph replay, the
training loops' fused and graph routes against the generic autograd route, validate()'s graph route against its eager
route, and an FPDTrainStep at training precision "fp16"."""
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
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import _kld_model as K  # noqa: E402

LOSS_TOL = 1e-5          # relative, on the loss values
GRAD_TOL = 1e-5          # worst gradient error over the largest gradient magnitude
_observed = {"loss": 0.0, "grad": 0.0}


def _nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def _nchw(t):
    return t.permute(0, 3, 1, 2).contiguous()


def _rel(a, b):
    return abs(float(a) - float(b)) / max(abs(float(b)), 1e-300)


def _check_loss(got, ref):
    e = _rel(got, ref)
    _observed["loss"] = max(_observed["loss"], e)
    assert e <= LOSS_TOL, (float(got), float(ref), e)


def _check_grad(got, ref):
    ref = ref.double()
    err = (got.double() - ref).abs().max().item()
    scale = ref.abs().max().item()
    if scale == 0.0:
        assert err == 0.0
        return
    _observed["grad"] = max(_observed["grad"], err / scale)
    assert err <= GRAD_TOL * scale, (err, scale)


def _weights(gen, kind, B, J):
    if kind == "binary":
        return (torch.rand(B, J, 1, generator=gen, device="cuda") > 0.2).float()
    if kind == "fractional":
        return torch.rand(B, J, 1, generator=gen, device="cuda")
    w = (torch.rand(B, J, 1, generator=gen, device="cuda") > 0.5).float()      # "zero": half the joints, sample 0
    w[0] = 0.0
    return w


def _maps(gen, B, J, h, w, S, amp=1.0):
    """Reference maps and students around them, with a spread of per-map differences."""
    tgt = amp * torch.randn(B, J, h, w, generator=gen, device="cuda")
    spread = lambda: amp * (0.1 + torch.rand(B, J, 1, 1, generator=gen, device="cuda"))  # noqa: E731
    outs = [tgt + spread() * torch.randn(B, J, h, w, generator=gen, device="cuda") for _ in range(S)]
    teacher = tgt + spread() * torch.randn(B, J, h, w, generator=gen, device="cuda")
    return outs, tgt, teacher


# B, J, (h, w), S, pose T, kd T, weights, use_target_weight
CASES = [
    (1, 1, (64, 64), 1, 1.0, 0.25, "binary", True),
    (24, 17, (64, 48), 1, 0.25, 1.0, "fractional", True),
    (32, 16, (64, 64), 4, 1.0, 1.0, "binary", True),
    (32, 16, (64, 64), 4, 4.0, 0.05, "zero", True),
    (24, 64, (96, 72), 8, 0.05, 4.0, "fractional", False),
    (1, 64, (64, 48), 8, 4.0, 0.25, "binary", True),
    (32, 17, (96, 72), 1, 0.05, 0.05, "zero", False),
    (24, 1, (96, 72), 4, 0.25, 4.0, "fractional", True),
]


@pytest.mark.parametrize("B,J,hw,S,tp,tk,wkind,use_tw", CASES)
def test_module_and_fused_forms_match_fp64_model(B, J, hw, S, tp, tk, wkind, use_tw):
    import fpd_b200  # noqa: F401
    from fpd_b200 import ops
    h, w = hw
    gen = torch.Generator(device="cuda").manual_seed(B * 1000 + J * 10 + S)
    outs, tgt, teacher = _maps(gen, B, J, h, w, S)
    tw = _weights(gen, wkind, B, J)
    wt = tw if use_tw else None
    # the module form, per stack and against the teacher
    for o, ref, T in ((outs[0], tgt, tp), (outs[-1], teacher, tk)):
        loss3, grad = ops.joints_kld(o, ref, wt, T)
        v, rg = K.kld(o, ref, wt, T)
        _check_loss(loss3[0].item(), v.item())
        assert loss3[1].item() == 0.0 and loss3[2].item() == loss3[0].item()
        _check_grad(grad, rg)
    # the fused form; use_target_weight False runs with ones, as the training loops do
    twf = (tw if use_tw else torch.ones_like(tw)).reshape(B, J).contiguous()
    alpha = 0.3
    losses, grads = ops.fpd_loss([_nhwc(o) for o in outs], tgt, _nhwc(teacher), twf, alpha, pose_temperature=tp,
                                 kd_temperature=tk)
    pose, kd, total, rgrads = K.fpd(outs, tgt, teacher, wt, alpha, ("kl", tp), ("kl", tk))
    for got, ref in zip(losses.cpu().tolist(), (pose, kd, total)):
        _check_loss(got, ref.item())
    for g, r in zip(grads, rgrads):
        _check_grad(_nchw(g), r)


@pytest.mark.parametrize("pose,kd", [(("mse",), ("kl", 0.25)), (("ohkm", 8), ("kl", 1.0)), (("kl", 4.0), ("mse",)),
                                     (("kl", 1.0), ("ohkm", 4))])
def test_fused_form_mixed_kinds_match_fp64_model(pose, kd):
    import fpd_b200  # noqa: F401
    from fpd_b200 import ops
    B, J, h, w, S = 4, 16, 64, 64, 2
    gen = torch.Generator(device="cuda").manual_seed(77)
    outs, tgt, teacher = _maps(gen, B, J, h, w, S, amp=0.5)
    tw = _weights(gen, "binary", B, J)
    losses, grads = ops.fpd_loss([_nhwc(o) for o in outs], tgt, _nhwc(teacher), tw.reshape(B, J).contiguous(), 0.5,
                                 **K.fpd_kwargs(pose, kd))
    rp, rk, rt, rgrads = K.fpd(outs, tgt, teacher, tw, 0.5, pose, kd)
    for got, ref in zip(losses.cpu().tolist(), (rp, rk, rt)):
        _check_loss(got, ref.item())
    for g, r in zip(grads, rgrads):
        _check_grad(_nchw(g), r)


def test_module_form_takes_any_heatmap_size():
    import fpd_b200  # noqa: F401
    from fpd_b200 import ops
    gen = torch.Generator(device="cuda").manual_seed(4)
    for (B, J, h, w) in ((3, 5, 7, 9), (2, 17, 30, 30), (1, 3, 1, 1), (2, 4, 63, 47)):
        o, r = torch.randn(B, J, h, w, generator=gen, device="cuda"), torch.randn(B, J, h, w, generator=gen, device="cuda")
        tw = torch.rand(B, J, 1, generator=gen, device="cuda")
        loss3, grad = ops.joints_kld(o, r, tw, 0.5)
        v, rg = K.kld(o, r, tw, 0.5)
        if v.item() == 0.0:                    # 1x1 maps: every softmax is 1; the loss is round-off of (r - o) / T
            assert abs(loss3[0].item()) <= 1e-6 and grad.abs().max().item() == 0.0
            continue
        _check_loss(loss3[0].item(), v.item())
        _check_grad(grad, rg)


def test_overflow_large_maps_at_small_temperature():
    import fpd_b200  # noqa: F401
    from fpd_b200 import ops
    B, J, h, w, T = 8, 16, 64, 48, 0.05
    gen = torch.Generator(device="cuda").manual_seed(5)
    o = 100 * torch.rand(B, J, h, w, generator=gen, device="cuda") - 50
    r = 100 * torch.rand(B, J, h, w, generator=gen, device="cuda") - 50
    o[:, :, 0, 0], r[:, :, 1, 1] = 50.0, -50.0
    tw = torch.ones(B, J, 1, device="cuda")
    loss3, grad = ops.joints_kld(o, r, tw, T)
    v, rg = K.kld(o, r, tw, T)
    assert torch.isfinite(loss3).all() and torch.isfinite(grad).all()
    _check_loss(loss3[0].item(), v.item())
    _check_grad(grad, rg)
    losses, grads = ops.fpd_loss([_nhwc(o)], r, _nhwc(r.flip(3).contiguous()), tw.reshape(B, J), 0.5,
                                 pose_temperature=T, kd_temperature=T)
    rp, rk, rt, rgrads = K.fpd([o], r, r.flip(3), tw, 0.5, ("kl", T), ("kl", T))
    assert torch.isfinite(losses).all() and torch.isfinite(grads[0]).all()
    for got, ref in zip(losses.cpu().tolist(), (rp, rk, rt)):
        _check_loss(got, ref.item())
    _check_grad(_nchw(grads[0]), rgrads[0])


def test_student_equal_to_reference_gives_exact_zeros():
    import fpd_b200  # noqa: F401
    from fpd_b200 import ops
    B, J, h, w = 4, 17, 64, 48
    gen = torch.Generator(device="cuda").manual_seed(6)
    r = 3 * torch.randn(B, J, h, w, generator=gen, device="cuda")
    tw = torch.rand(B, J, 1, generator=gen, device="cuda")
    for T in (0.05, 1.0, 4.0):
        loss3, grad = ops.joints_kld(r.clone(), r, tw, T)
        assert loss3.abs().max().item() == 0.0 and grad.abs().max().item() == 0.0
        # the fused kd term: every stack equal to the teacher (alpha = 1: the pose term has no gradient share)
        t = _nhwc(r)
        outs = [t.clone() for _ in range(3)]
        g0 = torch.randn(B, J, h, w, generator=gen, device="cuda")
        losses, grads = ops.fpd_loss(outs, g0, t, tw.reshape(B, J), 1.0, pose_temperature=T, kd_temperature=T)
        assert losses[1].item() == 0.0 and losses[2].item() == 0.0 and losses[0].item() > 0
        assert all(g.abs().max().item() == 0.0 for g in grads)
        # and both terms equal: target, teacher and stacks all the same maps
        losses, grads = ops.fpd_loss(outs, r, t, tw.reshape(B, J), 0.5, pose_temperature=T, kd_temperature=2 * T)
        assert losses.abs().max().item() == 0.0 and all(g.abs().max().item() == 0.0 for g in grads)


def test_nan_in_a_student_map_makes_the_loss_nan():
    import fpd_b200  # noqa: F401
    from fpd_b200 import ops
    B, J, h, w = 2, 16, 64, 64
    gen = torch.Generator(device="cuda").manual_seed(8)
    o, r = torch.randn(B, J, h, w, generator=gen, device="cuda"), torch.randn(B, J, h, w, generator=gen, device="cuda")
    o[1, 3, 10, 20] = float("nan")
    tw = torch.ones(B, J, 1, device="cuda")
    assert torch.isnan(ops.joints_kld(o, r, tw, 1.0)[0][0]).item()
    losses, _ = ops.fpd_loss([_nhwc(o)], r, _nhwc(r), tw.reshape(B, J), 0.5, kd_temperature=1.0)
    assert torch.isnan(losses[1]).item() and torch.isnan(losses[2]).item()
    losses, _ = ops.fpd_loss([_nhwc(o)], r, _nhwc(r), tw.reshape(B, J), 0.5, pose_temperature=1.0, kd_topk=4)
    assert torch.isnan(losses[0]).item() and torch.isnan(losses[2]).item()


def test_every_gradient_element_is_written():
    """Gradient buffers poisoned with NaN before the call come back finite and equal to a fresh call's."""
    import fpd_b200  # noqa: F401
    from fpd_b200 import _native as N
    from fpd_b200 import ops
    B, J, h, w, S = 3, 17, 64, 48, 8
    gen = torch.Generator(device="cuda").manual_seed(10)
    outs, tgt, teacher = _maps(gen, B, J, h, w, S)
    tw = _weights(gen, "zero", B, J).reshape(B, J).contiguous()
    on, tn = [_nhwc(o) for o in outs], _nhwc(teacher)
    for kw in (dict(pose_temperature=1.0, kd_temperature=0.25), dict(pose_topk=4, kd_temperature=1.0),
               dict(kd_temperature=4.0)):
        poisoned = [torch.full_like(o, float("nan")) for o in on]
        ref_l, ref_g = ops.fpd_loss(on, tgt, tn, tw, 0.5, **kw)
        losses, grads = ops.fpd_loss(on, tgt, tn, tw, 0.5, grads_out=poisoned, **kw)
        assert all(torch.isfinite(g).all() for g in grads)
        assert all(torch.equal(a, b) for a, b in zip(grads, ref_g)) and torch.equal(losses, ref_l)
    # the module form through its C entry point
    o, r = outs[0], tgt
    grad = torch.full_like(o, float("nan"))
    loss3 = torch.empty(3, device="cuda")
    ws = torch.empty(N.lib().fpd_joints_kld_workspace_bytes(B, J, h * w), dtype=torch.uint8, device="cuda")
    p = ops._p
    assert N.lib().fpd_joints_kld(p(o), p(r), p(tw), 0.5, p(loss3), p(grad), B, J, h * w, p(ws), ws.numel(),
                                  ops._stream()) == 0
    assert torch.isfinite(grad).all() and torch.equal(grad, ops.joints_kld(o, r, tw, 0.5)[1])


def test_runs_and_graph_replays_are_bit_identical():
    import fpd_b200  # noqa: F401
    from fpd_b200 import ops
    B, J, h, w, S = 8, 16, 64, 64, 3
    gen = torch.Generator(device="cuda").manual_seed(9)
    sets = []
    for _ in range(3):
        outs, tgt, teacher = _maps(gen, B, J, h, w, S)
        sets.append(([_nhwc(o) for o in outs], tgt, _nhwc(teacher), _weights(gen, "fractional", B, J).reshape(B, J)))
    kw = dict(pose_topk=5, kd_temperature=0.5)
    st_outs, st_tgt, st_teacher, st_tw = [[t.clone() for t in sets[0][0]]] + [t.clone() for t in sets[0][1:]]
    st_grads = [torch.empty_like(o) for o in st_outs]
    st_losses = torch.empty(3, device="cuda")
    st_nchw = _nchw(st_outs[0])

    def body():
        ops.fpd_loss(st_outs, st_tgt, st_teacher, st_tw, 0.4, grads_out=st_grads, losses_out=st_losses, **kw)
        return ops.joints_kld(st_nchw, st_tgt, st_tw, 0.25)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        body()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        m_loss, m_grad = body()
    for outs, tgt, teacher, tw in sets[1:]:
        ref_l, ref_g = ops.fpd_loss(outs, tgt, teacher, tw, 0.4, **kw)
        ref_ml, ref_mg = ops.joints_kld(_nchw(outs[0]), tgt, tw, 0.25)
        for d, src in zip(st_outs + [st_tgt, st_teacher, st_tw, st_nchw], outs + [tgt, teacher, tw, _nchw(outs[0])]):
            d.copy_(src)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(st_losses, ref_l) and all(torch.equal(a, b) for a, b in zip(st_grads, ref_g))
        assert torch.equal(m_loss, ref_ml) and torch.equal(m_grad, ref_mg)
        again_l, again_g = ops.fpd_loss(outs, tgt, teacher, tw, 0.4, **kw)
        assert torch.equal(again_l, ref_l) and all(torch.equal(a, b) for a, b in zip(again_g, ref_g))


def test_fused_kd_term_has_the_module_forms_bits():
    """h*w % 64 == 0: the fused form runs the module form's statistics chunk by chunk, so each term's gradient is the
    module form's, scaled by a power of two at alpha = 0.5."""
    import fpd_b200  # noqa: F401
    from fpd_b200 import ops
    B, J, h, w = 4, 16, 64, 48
    gen = torch.Generator(device="cuda").manual_seed(12)
    outs, tgt, teacher = _maps(gen, B, J, h, w, 2)
    tw = _weights(gen, "binary", B, J)
    _, grads = ops.fpd_loss([_nhwc(o) for o in outs], tgt, _nhwc(teacher), tw.reshape(B, J), 0.5,
                            pose_temperature=0.5, kd_temperature=2.0)
    for o, g in zip(outs, grads):
        gp = ops.joints_kld(o, tgt, tw, 0.5)[1]
        gk = ops.joints_kld(o, teacher, tw, 2.0)[1]
        assert torch.equal(_nchw(g), 0.5 * gp + 0.5 * gk)


# ------------------------------------------------------------------------------------------------ training loops
def _cfg(f, s, debug=False):
    return NS(MODEL=NS(EXTRA=NS(NUM_FEATURES=f, NUM_STACKS=s, NUM_BLOCKS=1), NUM_JOINTS=16, NAME="hourglass"),
              KD=NS(ALPHA=0.5), PRINT_FREQ=1,
              TEST=NS(FLIP_TEST=True, SHIFT_HEATMAP=True, POST_PROCESS=True), DEBUG=NS(DEBUG=debug))


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


def _crit(kind):
    from fpd_b200.lib.core.loss import JointsKLDLoss, JointsMSELoss, JointsOHKMMSELoss
    return {"mse": lambda: JointsMSELoss(True), "ohkm": lambda: JointsOHKMMSELoss(True, topk=6),
            "kl": lambda: JointsKLDLoss(True, temperature=0.5)}[kind]()


@pytest.mark.parametrize("pose,kd", [("mse", "kl"), ("ohkm", "kl"), ("kl", "kl")])
def test_fpd_train_fused_route_equals_generic_route(pose, kd, monkeypatch):
    """KD.ALPHA = 0.5: the fused gradient then has the generic route's bits (the module form's statistics are the fused
    form's), which matters because Adam turns round-off in the gradients of conv biases ahead of a train-mode BatchNorm
    into whole learning-rate steps."""
    import fpd_b200  # noqa: F401
    from fpd_b200.lib.core import function as F
    torch.manual_seed(5)
    init_s = {k: v.clone() for k, v in _net(64, 2).state_dict().items()}
    init_t = {k: v.clone() for k, v in _net(64, 1).state_dict().items()}
    cfg = _cfg(64, 2)
    loader = _loader(2)
    results, calls = [], []
    orig = F._fused_step
    monkeypatch.setattr(F, "_fused_step", lambda *a, **k: calls.append(k) or orig(*a, **k))
    for generic in (False, True):
        s, t = _net(64, 2, init_s), _net(64, 1, init_t)
        opt = torch.optim.Adam(s.parameters(), lr=1e-3)
        wd = {"writer": _Writer(), "train_global_steps": 0}
        F.fpd_train(cfg, loader, _Hide(s) if generic else s, t, _crit(pose), _crit(kd), opt, 0, "/tmp", "/tmp", wd)
        torch.cuda.synchronize()
        results.append(({k: v.clone() for k, v in s.state_dict().items()}, wd["writer"].scalars))
    want = {"mse": {"pose_topk": 0}, "ohkm": {"pose_topk": 6}, "kl": {"pose_temperature": 0.5}}[pose]
    assert calls == [{**want, "kd_temperature": 0.5}] * 2
    _compare_routes(results)


def test_train_fused_route_equals_generic_route(monkeypatch):
    import fpd_b200  # noqa: F401
    from fpd_b200.lib.core import function as F
    torch.manual_seed(6)
    init_s = {k: v.clone() for k, v in _net(64, 2).state_dict().items()}
    cfg = _cfg(64, 2)
    loader = _loader(2)
    calls, results = [], []
    orig = F._fused_step
    monkeypatch.setattr(F, "_fused_step", lambda *a, **k: calls.append(k) or orig(*a, **k))
    for generic in (False, True):
        s = _net(64, 2, init_s)
        opt = torch.optim.Adam(s.parameters(), lr=1e-3)
        wd = {"writer": _Writer(), "train_global_steps": 0}
        F.train(cfg, loader, _Hide(s) if generic else s, _crit("kl"), opt, 0, "/tmp", "/tmp", wd)
        torch.cuda.synchronize()
        results.append(({k: v.clone() for k, v in s.state_dict().items()}, wd["writer"].scalars))
    assert calls == [{"pose_temperature": 0.5}] * 2
    _compare_routes(results)


def _opt_state(opt):
    return [(k, v.clone() if torch.is_tensor(v) else v) for st in opt.state.values() for k, v in sorted(st.items())]


@pytest.mark.parametrize("pose,kd", [("mse", "kl"), ("kl", "ohkm"), ("kl", "kl")])
def test_fpd_train_graph_route_equals_eager_fused_route(pose, kd, monkeypatch):
    import fpd_b200  # noqa: F401
    from fpd_b200.lib.core import function as F
    torch.manual_seed(7)
    init_s = {k: v.clone() for k, v in _net(64, 2).state_dict().items()}
    init_t = {k: v.clone() for k, v in _net(64, 1).state_dict().items()}
    loader = _loader(3) + _loader(1, B=1)            # a short last batch takes the eager route in both runs
    runs = []
    for graph in (True, False):
        monkeypatch.setattr(F, "_TRAIN_GRAPH", graph)
        F._train_step_cache.clear()
        s, t = _net(64, 2, init_s), _net(64, 1, init_t)
        opt = torch.optim.Adam(s.parameters(), lr=1e-3)
        wd = {"writer": _Writer(), "train_global_steps": 0}
        F.fpd_train(_cfg(64, 2), loader, s, t, _crit(pose), _crit(kd), opt, 0, "/tmp", "/tmp", wd)
        torch.cuda.synchronize()
        runs.append(({k: v.clone() for k, v in s.state_dict().items()}, _opt_state(opt), wd["writer"].scalars))
    F._train_step_cache.clear()
    (sd_g, os_g, sc_g), (sd_e, os_e, sc_e) = runs
    assert sd_g.keys() == sd_e.keys() and all(torch.equal(sd_g[k], sd_e[k]) for k in sd_g)
    assert len(os_g) == len(os_e) and all(a[0] == b[0] and (torch.equal(a[1], b[1]) if torch.is_tensor(a[1])
                                                            else a[1] == b[1]) for a, b in zip(os_g, os_e))
    assert sc_g == sc_e


# ------------------------------------------------------------------------------------------------ validate
FLIP_PAIRS = [[0, 5], [1, 4], [2, 3], [10, 15], [11, 14], [12, 13]]


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


def test_validate_graph_route_equals_eager_route_with_kld(monkeypatch):
    import fpd_b200  # noqa: F401
    from fpd_b200.lib.core import function as F
    from fpd_b200.lib.core.loss import JointsKLDLoss, JointsMSELoss
    from fpd_b200.lib.models import hourglass as H
    torch.manual_seed(11)
    net = H.get_pose_net(NS(MODEL=NS(EXTRA=NS(NUM_FEATURES=64, NUM_STACKS=2, NUM_BLOCKS=1), NUM_JOINTS=16,
                                     NAME="hourglass")), True)
    for m in net.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.running_mean.normal_(0, 0.1)
            m.running_var.uniform_(0.5, 1.5)
    net = net.cuda()
    hw, J = (128, 128), 16
    loader = [_batch(3, 20, hw, J), _batch(3, 21, hw, J), _batch(2, 22, hw, J)]      # last batch partial
    cfg = NS(MODEL=NS(NUM_JOINTS=J, NAME="hourglass"), PRINT_FREQ=2, DEBUG=NS(DEBUG=False),
             TEST=NS(FLIP_TEST=True, SHIFT_HEATMAP=True, POST_PROCESS=True))
    runs, calls = [], []
    orig = F._GraphValidation.run
    monkeypatch.setattr(F._GraphValidation, "run", lambda self, *a: calls.append(self.temperature) or orig(self, *a))
    for graph, crit in ((True, JointsKLDLoss(True, 0.5)), (False, JointsKLDLoss(True, 0.5)), (True, JointsMSELoss(True))):
        monkeypatch.setattr(F, "_VALIDATE_GRAPH", graph)
        calls.clear()
        ds = _ValSet(8, J)
        wd = {"writer": _Writer(), "valid_global_steps": 0}
        perf = F.validate(cfg, loader, ds, net, crit, "/tmp", "/tmp", wd)
        assert calls == ([getattr(crit, "temperature", 0.0)] * 3 if graph else [])
        runs.append((perf, ds.seen, wd["writer"].scalars))
    (pg, sg, wg), (pe, se, we), (_, _, wm) = runs
    assert np.array_equal(sg[0], se[0]) and np.array_equal(sg[1], se[1]) and sg[2] == se[2]
    assert pg == pe and wg == we
    # the loss really is the KL one (the MSE graph gives another value, the same accuracy)
    lg = [v for t, v, _ in wg if t == "valid_loss"]
    lm = [v for t, v, _ in wm if t == "valid_loss"]
    assert lg != lm and [v for t, v, _ in wg if t == "valid_acc"] == [v for t, v, _ in wm if t == "valid_acc"]


# ------------------------------------------------------------------------------------------------ fp16 training step
def test_train_step_fp16_with_kld_kd_term_graph_equals_eager():
    import fpd_b200  # noqa: F401
    from bench import synthetic_batch
    from fpd_b200.engine import set_training_precision
    from fpd_b200.train_step import FPDTrainStep
    torch.manual_seed(13)
    init_s = {k: v.clone() for k, v in _net(64, 2).state_dict().items()}
    init_t = {k: v.clone() for k, v in _net(64, 1).state_dict().items()}
    batches = [synthetic_batch(4, 90 + i, 128, 128) for i in range(3)]
    runs = []
    for use_graph in (True, False):
        s, t = _net(64, 2, init_s), _net(64, 1, init_t)
        set_training_precision(s, "fp16")
        step = FPDTrainStep(s, t, alpha=0.5, use_graph=use_graph, pose_topk=4, kd_temperature=1.0)
        losses = [step.step(x.cuda(), tg.cuda(), w.cuda()).clone() for x, tg, w in batches]
        torch.cuda.synchronize()
        runs.append((torch.stack(losses), [p.detach().clone() for p in s.parameters()]))
    (lg, pg), (le, pe) = runs
    assert torch.isfinite(lg).all() and (lg[:, 1] > 0).all()
    assert torch.equal(lg, le) and all(torch.equal(a, b) for a, b in zip(pg, pe))


def test_report_observed_error_bounds():
    """Runs last in this file: prints the worst errors the checks above saw."""
    print("\nJointsKLDLoss vs fp64: worst loss rel. error %.3e, worst gradient error / max |gradient| %.3e"
          % (_observed["loss"], _observed["grad"]))
