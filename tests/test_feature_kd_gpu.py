"""Feature distillation on the H100: fpd_feature_mse against fp64 (fp32 and fp16 teachers, repeats, graph replays, NaN),
FPDTrainStep's student and adapter gradients against an fp64 autograd evaluation of the oracle networks for hourglass and
HRNet pairs, the off switch, the graph and eager fpd_train routes, an "fp16_act" teacher, a training run and
checkpoints."""
import copy
import os
import sys
import types

import pytest
import torch
import torch.nn.functional as Fn

NS = types.SimpleNamespace
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import _parity as P  # noqa: E402

pytestmark = pytest.mark.gpu

TOL = 1e-3


@pytest.fixture(scope="module", autouse=True)
def _fp32_reference_mode():
    tf = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf


# ------------------------------------------------------------------------------------------------ the kernel
SHAPES = [(32, 64, 64, 256), (24, 64, 48, 48), (3, 64, 48, 32), (1, 8, 8, 16)]


def _draw(shape, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    t = torch.relu(torch.randn(shape, generator=g, device="cuda"))
    s = t + 0.5 * torch.randn(shape, generator=g, device="cuda")
    return s, t


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("f16", [False, True])
def test_kernel_matches_fp64(shape, f16):
    from fpd_b200 import ops
    s, t = _draw(shape, sum(shape) + f16)
    if f16:
        t = t.half()
    tf = t.float()
    w = 0.37
    losses = torch.tensor([1.0, 2.0, 3.0], device="cuda")
    loss, grad = ops.feature_mse(s, t, w, losses=losses)
    torch.cuda.synchronize()
    d = s.double() - tf.double()
    n = s.numel()
    ref_l = float((d * d).sum() / n)
    ref_g = (2.0 * w / n) * d
    assert abs(float(loss) - ref_l) <= 1e-6 * ref_l, (float(loss), ref_l)
    assert float((grad.double() - ref_g).abs().max()) <= 1e-6 * float(ref_g.abs().max())
    assert float(losses[0]) == 1.0 and float(losses[1]) == 2.0
    assert abs(float(losses[2]) - (3.0 + w * ref_l)) <= 1e-6 * (3.0 + w * ref_l)
    if f16:
        # the fp16 teacher gives the bits of the same teacher widened to fp32
        loss32, grad32 = ops.feature_mse(s, tf, w)
        assert torch.equal(loss32, loss) and torch.equal(grad32, grad)
    # repeats and a graph replay
    l2, g2 = ops.feature_mse(s, t, w)
    assert torch.equal(l2, loss) and torch.equal(g2, grad)
    lo, go = torch.empty(1, device="cuda"), torch.empty_like(s)
    ops.feature_mse(s, t, w, grad_out=go, loss_out=lo)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.feature_mse(s, t, w, grad_out=go, loss_out=lo)
    lo.zero_()
    go.fill_(float("nan"))
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(lo, loss) and torch.equal(go, grad)


@pytest.mark.parametrize("shape", [(32, 64, 64, 256), (1, 8, 8, 16)])
def test_nan_in_student_gives_nan_loss(shape):
    from fpd_b200 import ops
    s, t = _draw(shape, 5)
    s.view(-1)[s.numel() // 3] = float("nan")
    for tt in (t, t.half()):
        loss, _ = ops.feature_mse(s, tt, 1.0)
        assert torch.isnan(loss).all()


def test_unaligned_and_odd_sizes_take_the_scalar_path():
    from fpd_b200 import ops
    base_s, base_t = _draw((1, 5, 7, 3), 9)
    s, t = base_s.reshape(-1)[1:].contiguous(), base_t.reshape(-1)[1:]     # t: offset by one element, n = 104
    loss, grad = ops.feature_mse(s, t, 0.5)
    d = s.double() - t.double()
    assert abs(float(loss) - float((d * d).mean())) <= 1e-6 * float((d * d).mean())
    assert float((grad.double() - d / d.numel()).abs().max()) <= 1e-6 * float((d / d.numel()).abs().max())


# ------------------------------------------------------------------------------------------------ networks
def _hg_cfg(f, s):
    return NS(MODEL=NS(EXTRA=NS(NUM_FEATURES=f, NUM_STACKS=s, NUM_BLOCKS=1), NUM_JOINTS=16, NAME="hourglass"),
              KD=NS(ALPHA=0.5), PRINT_FREQ=1, TEST=NS(FLIP_TEST=True, SHIFT_HEATMAP=True, POST_PROCESS=True),
              DEBUG=NS(DEBUG=False))


def _hg(f, s, sd=None):
    from fpd_b200.lib.models import hourglass as H
    net = H.get_pose_net(_hg_cfg(f, s), True)
    if sd is not None:
        net.load_state_dict(sd)
    return net.cuda()


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


def _randomise_running_stats(net):
    for m in net.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.running_mean.normal_(0, 0.1)
            m.running_var.uniform_(0.5, 1.5)


def _batch(B, seed, H, W, J):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, 3, H, W, generator=g, device="cuda")
    target = torch.rand(B, J, H // 4, W // 4, generator=g, device="cuda")
    tw = (torch.rand(B, J, 1, generator=g, device="cuda") > 0.2).float()
    return x, target, tw


# ------------------------------------------------------------------------------------------------ step against fp64
def _tapped(kind, sd, x, training, nstack, dtype):
    """The oracle network's outputs and its head feature (the input of its last head conv) in `dtype`."""
    from oracle import hourglass_oracle as O
    from oracle import hrnet_oracle as HO
    head = "score.%d" % (nstack - 1) if kind == "hg" else "final_layer"
    mod = O if kind == "hg" else HO
    taken = {}
    orig = mod._conv

    def tap(sd_, name, xin, *a, **k):
        if name == head:
            taken[name] = xin
        return orig(sd_, name, xin, *a, **k)
    mod._conv = tap
    try:
        if kind == "hg":
            outs = O.hourglass_net(sd, x.to(dtype), nstack, training=training)
        else:
            outs = [HO.hrnet(HO.annotate_strides(sd), x.to(dtype), training=training)]
    finally:
        mod._conv = orig
    return outs, taken[head]


def _oracle_step(kind, s_sd, t_heat, t_feat, a_sd, x, target, tw, alpha, w, dtype, stacks):
    """The FPD loss plus w * mean((A(s) - t)^2) by autograd in `dtype`, s the student oracle's head feature (the input of
    its last head conv). The teacher's last heat-map t_heat and head feature t_feat (NCHW) are the ones the step used, so
    that the student's gradients are compared on the same targets: -> (losses (total, pose, kd, feat), {name: grad})."""
    from oracle import hourglass_oracle as O
    sd = P.cast_sd(s_sd, dtype)
    params = P.with_grad(sd)
    outs, s_feat = _tapped(kind, sd, x, True, stacks[0], dtype)
    a = {k: v.detach().clone().to(dtype).requires_grad_(True) for k, v in a_sd.items()}
    total, pose, kd = O.fpd_loss(outs, target.to(dtype), tw.to(dtype), t_heat.to(dtype), alpha)
    af = Fn.conv2d(s_feat, a["conv.weight"], a["conv.bias"])
    feat = ((af - t_feat.to(dtype)) ** 2).mean()
    (total + w * feat).backward()
    grads = {k: p.grad.detach() for k, p in params.items()}
    grads.update({"adapter." + k: p.grad.detach() for k, p in a.items()})
    return (float((total + w * feat).detach()), float(pose.detach()), float(kd.detach()), float(feat.detach())), grads


@pytest.mark.parametrize("kind", ["hg", "hrnet"])
def test_step_gradients_match_fp64(kind):
    from fpd_b200.train_step import FeatureAdapter, FPDTrainStep
    torch.manual_seed(31)
    if kind == "hg":
        student, teacher, stacks, (H, W), J = _hg(64, 2), _hg(128, 1), (2, 1), (128, 128), 16
    else:
        student, teacher, stacks, (H, W), J = _hrnet(32), _hrnet(48), (1, 1), (128, 96), 17     # the shipped pair
    _randomise_running_stats(teacher)
    adapter = FeatureAdapter(student, teacher).cuda()
    torch.nn.init.normal_(adapter.conv.weight, std=0.05)       # a trained-like adapter: a gradient that reaches s
    torch.nn.init.normal_(adapter.conv.bias, std=0.05)
    s_sd = {k: v.detach().clone() for k, v in student.state_dict().items()}
    t_sd = {k: v.detach().clone() for k, v in teacher.state_dict().items()}
    a_sd = {k: v.detach().clone() for k, v in adapter.state_dict().items()}
    x, target, tw = _batch(2, 7, H, W, J)
    alpha, w = 0.5, 0.8
    step = FPDTrainStep(student, teacher, alpha=alpha, fused_adam=False, feature_weight=w, feature_adapter=adapter)
    losses = step.step(x, target, tw).clone()
    feat = float(step.feature_loss)
    torch.cuda.synchronize()
    names = [k for k, _ in student.named_parameters()] + ["adapter.conv.weight", "adapter.conv.bias"]
    got = {k: g.clone() for k, g in zip(names, step.grad_views)}
    t_heat = step.last_teacher.permute(0, 3, 1, 2).contiguous()
    t_feat = step._t_keep.head_feature.data.permute(0, 3, 1, 2).contiguous()
    # the teacher's forward against the oracle's, like the existing FPD step tests
    with torch.no_grad():
        ref_heat, ref_feat = _tapped(kind, P.cast_sd(t_sd, torch.float64), x, False, stacks[1], torch.float64)
    assert P.rel_max(t_heat, ref_heat[-1]) < TOL and P.rel_max(t_feat, ref_feat) < TOL
    l32, g32 = _oracle_step(kind, s_sd, t_heat, t_feat, a_sd, x, target, tw, alpha, w, torch.float32, stacks)
    l64, g64 = _oracle_step(kind, s_sd, t_heat, t_feat, a_sd, x, target, tw, alpha, w, torch.float64, stacks)
    pose, kd, total = [float(v) for v in losses.cpu()]
    for v, r in ((total, l64[0]), (pose, l64[1]), (kd, l64[2]), (feat, l64[3])):
        assert abs(v - r) <= TOL * abs(r), (v, r)
    assert l64[3] > 0.05 * abs(l64[0])           # the feature term is a visible share of the total
    # a conv bias in front of a train-mode BatchNorm has an exactly zero gradient: any two fp32 evaluations leave only
    # cancellation noise there (the per-tensor ratio of two noises says nothing), so those are held to an absolute bound
    gmax = max(float(v.abs().max()) for v in g64.values())
    zero = {k for k in got if k.endswith(".bias") and not k.startswith("adapter.") and k != "final_layer.bias"
            and not k.startswith("score") and float(g64[k].abs().max()) <= 1e-12 * gmax}
    for k in zero:
        assert float(got[k].abs().max()) <= 1e-5 * gmax, (k, float(got[k].abs().max()), gmax)
    P.assert_grads_as_good_as_fp32({k: v for k, v in got.items() if k not in zero},
                                   {k: v for k, v in g32.items() if k not in zero},
                                   {k: v for k, v in g64.items() if k not in zero}, "feature kd step %s" % kind)
    for k in ("adapter.conv.weight", "adapter.conv.bias"):
        assert P.rel_max(got[k], g64[k]) < TOL, (k, P.rel_max(got[k], g64[k]))


# ------------------------------------------------------------------------------------------------ off means unchanged
def _run_steps(s_sd, t_sd, batches, use_graph=True, **kw):
    from fpd_b200.train_step import FPDTrainStep
    s, t = _hg(64, 2, s_sd), _hg(64, 1, t_sd)
    step = FPDTrainStep(s, t, alpha=0.5, lr=1e-3, use_graph=use_graph, **kw)
    ls = [step.step(*b).clone() for b in batches]
    torch.cuda.synchronize()
    return step, s, ls


def test_weight_zero_is_todays_step():
    torch.manual_seed(3)
    s_sd = {k: v.clone() for k, v in _hg(64, 2).state_dict().items()}
    t_sd = {k: v.clone() for k, v in _hg(64, 1).state_dict().items()}
    batches = [_batch(4, 40 + i, 128, 128, 16) for i in range(3)]
    a, sa, la = _run_steps(s_sd, t_sd, batches)
    b, sb, lb = _run_steps(s_sd, t_sd, batches, feature_weight=0.0)
    assert b.adapter is None and b.feature_loss is None and a.flat.numel == b.flat.numel
    assert a.launches_per_step == b.launches_per_step
    assert torch.equal(a.flat.flat, b.flat.flat) and torch.equal(a.exp_avg, b.exp_avg)
    assert torch.equal(a.exp_avg_sq, b.exp_avg_sq)
    assert all(torch.equal(x, y) for x, y in zip(sa.buffers(), sb.buffers()))
    assert all(torch.equal(x, y) for x, y in zip(la, lb))


# ------------------------------------------------------------------------------------------------ fpd_train routes
class _Writer:
    def __init__(self):
        self.scalars = []

    def add_scalar(self, tag, v, step):
        self.scalars.append((tag, float(v), step))


def _meta(B, i):
    return {"center": torch.tensor([[64.0, 64.0]] * B), "scale": torch.tensor([[0.64, 0.64]] * B),
            "score": torch.ones(B), "image": ["img%d_%d" % (i, b) for b in range(B)]}


def _fpd_epoch(F, cfg, loader, init_s, init_t, init_a):
    from fpd_b200.lib.core.loss import JointsMSELoss
    from fpd_b200.train_step import FeatureAdapter
    s, t = _hg(64, 2, init_s), _hg(128, 1, init_t)
    a = FeatureAdapter(s, t).cuda()
    a.load_state_dict(init_a)
    opt = torch.optim.Adam(s.parameters(), lr=1e-3)
    opt.add_param_group({"params": a.parameters()})
    wd = {"writer": _Writer(), "train_global_steps": 0}
    F.fpd_train(cfg, loader, s, t, JointsMSELoss(True), JointsMSELoss(True), opt, 0, "/tmp", "/tmp", wd,
                feature_adapter=a)
    torch.cuda.synchronize()
    sd = {k: v.clone() for k, v in s.state_dict().items()}
    sd.update({"adapter." + k: v.clone() for k, v in a.state_dict().items()})
    ost = [(k, v.clone() if torch.is_tensor(v) else v) for st in opt.state.values() for k, v in sorted(st.items())]
    return sd, ost, wd["writer"].scalars


def test_fpd_train_routes_agree(monkeypatch):
    from fpd_b200.lib.core import function as F
    from fpd_b200.train_step import FeatureAdapter
    torch.manual_seed(17)
    s0, t0 = _hg(64, 2), _hg(128, 1)
    init_s = {k: v.clone() for k, v in s0.state_dict().items()}
    init_t = {k: v.clone() for k, v in t0.state_dict().items()}
    init_a = {k: v.clone() for k, v in FeatureAdapter(s0, t0).state_dict().items()}
    loader = []
    for i, B in enumerate((4, 4, 3)):                 # a short last batch
        x, tg, w = _batch(B, 60 + i, 128, 128, 16)
        loader.append((x.cpu(), tg.cpu(), w.cpu(), _meta(B, i)))
    cfg = _hg_cfg(64, 2)
    cfg.KD.FEATURE_WEIGHT = 0.5
    runs = []
    for graph in (True, False):
        monkeypatch.setattr(F, "_TRAIN_GRAPH", graph)
        F._train_step_cache.clear()
        runs.append(_fpd_epoch(F, cfg, loader, init_s, init_t, init_a))
    F._train_step_cache.clear()
    (sd_g, os_g, sc_g), (sd_e, os_e, sc_e) = runs
    assert all(torch.equal(sd_g[k], sd_e[k]) for k in sd_g)
    assert not torch.equal(sd_g["adapter.conv.weight"], init_a["conv.weight"].cuda())   # the adapter trained
    assert len(os_g) == len(os_e) and all(
        a[0] == b[0] and (torch.equal(a[1], b[1]) if torch.is_tensor(a[1]) else a[1] == b[1]) for a, b in zip(os_g, os_e))
    assert sc_g == sc_e
    feats = [v for tag, v, _ in sc_g if tag == "train_feat_loss"]
    assert len(feats) == 3 and all(v > 0 for v in feats)


# ------------------------------------------------------------------------------------------------ fp16 teacher
def test_fp16_act_teacher_feature_is_read_as_stored(monkeypatch):
    from fpd_b200 import engine, ops
    from fpd_b200.train_step import FeatureAdapter, FPDTrainStep
    torch.manual_seed(23)
    s_sd = {k: v.clone() for k, v in _hg(64, 2).state_dict().items()}
    t_net = _hg(128, 1)
    _randomise_running_stats(t_net)
    t_sd = {k: v.clone() for k, v in t_net.state_dict().items()}
    a_sd = {k: v.clone() for k, v in FeatureAdapter(_hg(64, 2), t_net).state_dict().items()}
    batch = _batch(4, 81, 128, 128, 16)
    widened = []
    real_h2f = ops.half_to_float

    def counting_h2f(x, out=None):
        widened.append(tuple(x.shape))
        return real_h2f(x, out=out)
    monkeypatch.setattr(ops, "half_to_float", counting_h2f)

    def run(weight, widen_first, use_graph=False):
        s, t = _hg(64, 2, s_sd), _hg(128, 1, t_sd)
        engine.set_inference_precision(t, "fp16_act")
        a = FeatureAdapter(s, t).cuda()
        a.load_state_dict(a_sd)
        step = FPDTrainStep(s, t, alpha=0.5, fused_adam=False, use_graph=use_graph, feature_weight=weight,
                            feature_adapter=a if weight else None)
        if widen_first:
            orig = step._feature_term

            def widened_term(s_eng, ctx, t_ctx, losses):
                t_ctx.head_feature.data = real_h2f(t_ctx.head_feature.data)
                return orig(s_eng, ctx, t_ctx, losses)
            step._feature_term = widened_term
        widened.clear()
        losses = step.step(*batch).clone()
        torch.cuda.synchronize()
        n = len(widened)
        return step, losses, [g.clone() for g in step.grad_views], n

    off, _, _, n_off = run(0.0, False)
    on, l_on, g_on, n_on = run(0.7, False)
    assert on._t_keep.head_feature.data.dtype == torch.float16
    assert n_on == n_off                      # the feature term launches no widening
    ref, l_ref, g_ref, _ = run(0.7, True)
    assert torch.equal(l_on, l_ref) and torch.equal(on.feature_loss, ref.feature_loss)
    assert all(torch.equal(a, b) for a, b in zip(g_on, g_ref))
    gr, l_gr, g_gr, _ = run(0.7, False, use_graph=True)           # the graph replays the same kernels
    assert torch.equal(l_gr, l_on) and all(torch.equal(a, b) for a, b in zip(g_gr, g_on))


# ------------------------------------------------------------------------------------------------ it trains
def test_feature_term_alone_trains():
    from fpd_b200.train_step import FeatureAdapter, FPDTrainStep
    torch.manual_seed(5)
    s = _hg(64, 1)
    t = copy.deepcopy(s)
    _randomise_running_stats(t)
    a = FeatureAdapter(s, t).cuda()
    x, target, _ = _batch(4, 99, 128, 128, 16)
    tw = torch.zeros(4, 16, 1, device="cuda")             # no heat-map term: the feature term does all the work
    step = FPDTrainStep(s, t, alpha=0.5, lr=5e-3, feature_weight=1.0, feature_adapter=a)
    curve = []
    for _ in range(30):
        losses = step.step(x, target, tw)
        curve.append(float(step.feature_loss))
        assert float(losses[0]) == 0.0 and float(losses[1]) == 0.0
        assert float(losses[2]) == pytest.approx(curve[-1], rel=1e-6)
    print("feature loss over 30 steps:", ["%.4g" % v for v in curve])
    assert min(curve[1:]) < 0.5 * curve[0], curve


# ------------------------------------------------------------------------------------------------ checkpoints
def test_checkpoint_round_trip_with_the_adapter():
    from fpd_b200.train_step import FeatureAdapter, FPDTrainStep
    torch.manual_seed(11)
    s_sd = {k: v.clone() for k, v in _hg(64, 2).state_dict().items()}
    t_sd = {k: v.clone() for k, v in _hg(128, 1).state_dict().items()}
    a_sd = {k: v.clone() for k, v in FeatureAdapter(_hg(64, 2), _hg(128, 1)).state_dict().items()}
    batches = [_batch(4, 120 + i, 128, 128, 16) for i in range(4)]

    def make(sd_s, sd_a):
        s, t = _hg(64, 2, sd_s), _hg(128, 1, t_sd)
        a = FeatureAdapter(s, t).cuda()
        a.load_state_dict(sd_a)
        return s, a, FPDTrainStep(s, t, alpha=0.5, lr=1e-3, feature_weight=0.5, feature_adapter=a)

    s, a, step = make(s_sd, a_sd)
    for b in batches[:2]:
        step.step(*b)
    torch.cuda.synchronize()
    ck = {"student": {k: v.clone() for k, v in s.state_dict().items()},
          "adapter": {k: v.clone() for k, v in a.state_dict().items()}, "opt": step.state_dict()}
    n_student = sum((p.numel() + 3) // 4 * 4 for p in s.parameters())
    assert ck["opt"]["numel"] == n_student + (64 * 128 + 3) // 4 * 4 + 128
    for b in batches[2:]:
        step.step(*b)
    torch.cuda.synchronize()
    s2, a2, step2 = make(ck["student"], ck["adapter"])
    step2.load_state_dict(ck["opt"])
    for b in batches[2:]:
        step2.step(*b)
    torch.cuda.synchronize()
    assert torch.equal(step.flat.flat, step2.flat.flat)
    assert torch.equal(step.exp_avg, step2.exp_avg) and torch.equal(step.exp_avg_sq, step2.exp_avg_sq)
    assert all(torch.equal(x, y) for x, y in zip(s.buffers(), s2.buffers()))
    assert torch.equal(a.conv.weight, a2.conv.weight) and torch.equal(a.conv.bias, a2.conv.bias)
    assert torch.equal(step.feature_loss, step2.feature_loss)
    # a step without the adapter refuses this state
    s3 = _hg(64, 2, ck["student"])
    with pytest.raises(ValueError, match="flat parameters"):
        FPDTrainStep(s3, _hg(128, 1, t_sd), alpha=0.5).load_state_dict(ck["opt"])
