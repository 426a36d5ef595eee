"""Single-pass FP16 training (engine.set_training_precision, ops.conv2d_tc_f16x1 with epilogue statistics and in_scale)
on the H100: the kernels against fp64 convolutions of the fp16-rounded operands, their statistics against fp64 sums of
their own output, determinism and graph replay, kernel selection, whole networks in train mode against the fp64 oracle,
an over-fit run against the fp32 one, the graph and eager routes of train / fpd_train, and switching the setting.

Every bound here was fixed before the first run on the GPU; DESIGN.md ("Single-pass FP16 training") records the
values observed."""
import os
import sys

import pytest
import torch
import torch.nn.functional as TF

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

import _parity as P  # noqa: E402
from test_infer_f16_gpu import SHAPES, _hourglass, _operands, _randomise_bn, kernel_names, nchw, relerr  # noqa: E402,E501
from test_train_graph_gpu import F as F  # noqa: E402,F401  (the fixture)
from test_train_graph_gpu import _assert_same, _call, _cfg, _hrnet, _inits, _loader, _state  # noqa: E402
from test_train_graph_gpu import _hourglass as _small_hourglass  # noqa: E402


@pytest.fixture(scope="module", autouse=True)
def _fp32_reference_mode():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield


def ops():
    import fpd_b200  # noqa: F401
    from fpd_b200 import ops as o
    return o


# ------------------------------------------------------------------------------------------------ kernels
STAT_SHAPES = [
    (32, 64, 64, 128, 128, 3),     # hg_fpd student 3x3 at 64x64: halo with statistics, four stages
    (4, 128, 128, 32, 32, 3),      # stem resolution
    (3, 13, 17, 64, 256, 3),       # two slices
    (24, 64, 48, 256, 32, 3),      # HRNet transition
    (4, 32, 32, 512, 256, 1),      # 1x1 resident with statistics
    (2, 16, 16, 640, 256, 1),      # 1x1 staged with statistics (the scratch does not fit beside the weights)
]


def _stats_ref(y, pivot):
    """fp64 sums of (y - pivot) as the epilogue forms it (the difference in fp32), and sums of magnitudes that bound
    the rounding of any fp64 summation order."""
    d = (y.reshape(-1, y.shape[-1]) - pivot).double()
    return torch.stack([d.sum(0), (d * d).sum(0)], 1), torch.stack([d.abs().sum(0), (d * d).sum(0)], 1)


@pytest.mark.parametrize("shape", SHAPES + STAT_SHAPES)
def test_forward_with_statistics_against_fp64(shape):
    B, H, W, Cin, Cout, k = shape
    o = ops()
    x, mean, scale, shift, w, bias, res, _ = _operands(shape, 21)
    w1, _ = o.weight_prep_f16(w, split=False)
    kind, nblk = o.conv2d_tc_f16x1_train_plan(B, H, W, Cin, Cout, k, stats=True)
    kw = dict(mean=mean, scale=scale, shift=shift, relu=True, bias=bias, residual=res)
    pivot = torch.randn(Cout, device="cuda") * 0.1
    if Cout > 256:
        assert (kind, nblk) == (None, 0)
        return
    part = torch.full((nblk, Cout, 2), float("nan"), dtype=torch.float64, device="cuda")
    y = o.conv2d_tc_f16x1(x, w1, k, stats_part=part, stats_pivot=pivot, **kw)
    a32 = ((x - mean).double() * scale.double() + shift.double()).float().clamp_min(0.0)
    a16 = a32.clamp(-65504.0, 65504.0).half().double()
    w16 = w1.double().view(k, k, Cout, Cin).permute(2, 3, 0, 1) / 256.0
    ref = TF.conv2d(nchw(a16), w16, bias.double(), padding=k // 2) + nchw(res).double()
    torch.cuda.synchronize()
    assert relerr(nchw(y), ref) <= 1e-4, "%s: %.3e" % (shape, relerr(nchw(y), ref))
    # the same outputs as a call without statistics where both run on the same kernel (a 1x1 call whose statistics
    # scratch does not fit beside the resident weights moves to the staged kernel, which sums each K step apart), and
    # sums that are the fp64 sums of the call's own outputs
    if kind == o.conv2d_tc_f16x1_kernel(B, H, W, Cin, Cout, k):
        assert torch.equal(y, o.conv2d_tc_f16x1(x, w1, k, **kw))
    want, mag = _stats_ref(y, pivot)
    assert torch.isfinite(part).all()
    err = ((part.sum(0) - want).abs() / mag.clamp_min(1e-300)).max().item()
    assert err <= 1e-12, "%s: statistics %.3e" % (shape, err)


def _dy(shape, kind, seed):
    B, H, W, Cin, Cout, k = shape
    g = torch.Generator(device="cuda").manual_seed(seed)
    dy = torch.randn(B, H, W, Cin, device="cuda", generator=g)
    if kind == "top":       # max |dY| S lands at 2^15 - 2^4: the top of [2^14, 2^15), no overflow
        dy = dy / dy.abs().max() * (32752.0 * 2.0 ** -30)
    elif kind == "wide":    # twelve decades of magnitude
        dy = dy * torch.pow(10.0, -12.0 * torch.rand(B, H, W, Cin, device="cuda", generator=g))
    else:
        dy = dy * 1e-4
    return dy


@pytest.mark.parametrize("kind", ["plain", "top", "wide"])
@pytest.mark.parametrize("shape", [(2, 19, 48, 128, 64, 3), (2, 16, 16, 256, 128, 3), (2, 19, 48, 128, 256, 1),
                                   (1, 8, 8, 1024, 64, 1), (2, 9, 11, 16, 48, 3)])
def test_data_gradient_with_in_scale_against_fp64(shape, kind):
    """dX of a convolution with weights w [Cin' = Cout_here][...]: the data-gradient weights of weight_prep_f16 and
    the operand scale of channel_sum(want_amax=True), against fp64 on fp16(dY S) / S."""
    B, H, W, Cin, Cout, k = shape          # Cin: channels of dY, Cout: channels of dX
    o = ops()
    dy = _dy(shape, kind, 31)
    g = torch.Generator(device="cuda").manual_seed(32)
    w = torch.randn(Cin, Cout, k, k, device="cuda", generator=g) * (1.0 / (Cin * k * k) ** 0.5)
    wd, _ = o.weight_prep_f16(w, for_dgrad=True, split=False)
    _, s = o.channel_sum(dy, want_amax=True)
    dx = o.conv2d_tc_f16x1(dy, wd, k, in_scale=s)
    S = s[0].item()
    assert S == 2.0 ** round(torch.log2(torch.tensor(S)).item())
    scaled = dy.double() * S
    assert 2.0 ** 14 <= scaled.abs().max().item() < 2.0 ** 15
    q = scaled.half().double() / S
    assert torch.isfinite(q).all()
    wd16 = wd.double().view(k, k, Cout, Cin).permute(2, 3, 0, 1) / 256.0
    ref = TF.conv2d(nchw(q), wd16, padding=k // 2)
    exact = TF.conv_transpose2d(nchw(dy).double(), w.double(), padding=k // 2)
    torch.cuda.synchronize()
    assert torch.isfinite(dx).all()
    assert relerr(nchw(dx), ref) <= 1e-4, "%s %s: %.3e" % (shape, kind, relerr(nchw(dx), ref))
    assert relerr(nchw(dx), exact) <= 2e-3, "%s %s: %.3e vs unrounded" % (shape, kind, relerr(nchw(dx), exact))


@pytest.mark.parametrize("shape", [(4, 37, 64, 128, 128, 3), (2, 19, 48, 256, 256, 1), (2, 16, 16, 640, 256, 1)])
def test_training_calls_deterministic_and_graph_replay(shape):
    B, H, W, Cin, Cout, k = shape
    o = ops()
    x, mean, scale, shift, w, bias, res, _ = _operands(shape, 23)
    w1, _ = o.weight_prep_f16(w, split=False)
    nblk = o.conv2d_tc_f16x1_train_plan(B, H, W, Cin, Cout, k, stats=True)[1]
    _, s = o.channel_sum(x * 1e-3, want_amax=True)
    pivot = torch.zeros(Cout, device="cuda")

    def run(y, part):
        o.conv2d_tc_f16x1(x, w1, k, mean=mean, scale=scale, shift=shift, relu=True, bias=bias, residual=res, out=y[0],
                          stats_part=part, stats_pivot=pivot)
        o.conv2d_tc_f16x1(x, w1, k, residual=res, out=y[1], in_scale=s)
    ref = (torch.empty(B, H, W, Cout, device="cuda"), torch.empty(B, H, W, Cout, device="cuda"))
    ref_part = torch.empty((nblk, Cout, 2), dtype=torch.float64, device="cuda")
    run(ref, ref_part)
    out = (torch.empty_like(ref[0]), torch.empty_like(ref[1]))
    part = torch.empty_like(ref_part)
    for _ in range(2):
        run(out, part)
        assert torch.equal(out[0], ref[0]) and torch.equal(out[1], ref[1]) and torch.equal(part, ref_part)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        run(out, part)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        run(out, part)
    for t in out + (part,):
        t.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out[0], ref[0]) and torch.equal(out[1], ref[1]) and torch.equal(part, ref_part)


# (B, H, W, Cin, Cout, k), planner choice with statistics, the kernel that must run
SELECTION = [
    ((8, 64, 64, 128, 128, 3), "halo", "::conv_halo_f16x1_kernel<"),
    ((4, 16, 12, 256, 256, 3), "halo", "::conv_halo_f16x1_kernel<"),
    ((8, 32, 32, 256, 128, 1), "1x1", "::pw_conv_f16x1_kernel<"),
    ((2, 16, 16, 640, 256, 1), "staged", "::conv_wgmma_kernel<true"),
]


def _selection_main():
    """Per SELECTION entry: the planner's choice and the kernel names of one statistics call and one in_scale call."""
    import json
    o = ops()
    g = torch.Generator(device="cuda").manual_seed(405)
    out = []
    for (B, H, W, Cin, Cout, k), _, _ in SELECTION:
        x = torch.randn(B, H, W, Cin, device="cuda", generator=g)
        w1, _ = o.weight_prep_f16(torch.randn(Cout, Cin, k, k, device="cuda", generator=g) * 0.05, split=False)
        kind, nblk = o.conv2d_tc_f16x1_train_plan(B, H, W, Cin, Cout, k, stats=True)
        part = torch.empty((nblk, Cout, 2), dtype=torch.float64, device="cuda")
        _, s = o.channel_sum(x, want_amax=True)
        runs = [lambda: o.conv2d_tc_f16x1(x, w1, k, stats_part=part),          # noqa: E731
                lambda: o.conv2d_tc_f16x1(x, w1, k, in_scale=s)]                # noqa: E731
        names = []
        for run in runs:
            run()
            names.append([n for n in kernel_names(run) if "_kernel" in n])
        out.append([kind, names])
    print(json.dumps(out))


def test_selection_by_kernel_name():
    """Traced in a fresh process, as tests/test_infer_f16_gpu.py does."""
    import json
    import subprocess
    code = "import sys; sys.path[:0] = [%r, %r]; import test_train_f16_gpu as t; t._selection_main()" % (HERE, ROOT)
    res = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-2000:]
    got = json.loads(res.stdout.strip().splitlines()[-1])
    for (args, kind, name), (planned, names) in zip(SELECTION, got):
        assert planned == kind, (args, planned)
        assert len(names[0]) > 0 and all(name in n for n in names[0]), (args, names[0])
        assert len(names[1]) > 0 and all("f16x1" in n or "conv_wgmma_kernel<true" in n for n in names[1]), (args, names)


# ------------------------------------------------------------------------------------------------ networks
def _network(kind, training):
    import fpd_b200  # noqa: F401
    from bench import hrnet_cfg, resnet_cfg
    from oracle import hourglass_oracle as O
    from oracle import hrnet_oracle as HO
    from oracle import resnet_oracle as RO
    torch.manual_seed(0)
    if kind == "hourglass":
        net = _hourglass() if training else _randomise_bn(_hourglass())
        return (net.cuda().train(training), (2, 3, 256, 256), 16,
                lambda sd, x: O.hourglass_net(sd, x, 4, training=training))
    if kind == "hrnet_w32":
        from fpd_b200.lib.models import pose_hrnet as H
        net = H.get_pose_net(hrnet_cfg(32), False)
        net = net if training else _randomise_bn(net)
        return (net.cuda().train(training), (2, 3, 256, 192), 17,
                lambda sd, x: [HO.hrnet(HO.annotate_strides(sd), x, training=training)])
    from fpd_b200.lib.models import pose_resnet as R
    net = R.get_pose_net(resnet_cfg(50), False)
    net.load_state_dict(RO.synthetic_state({k: v.shape for k, v in net.state_dict().items()}, seed=7), strict=True)
    return net.cuda().train(training), (2, 3, 256, 256), 16, lambda sd, x: [RO.resnet(sd, x, training=training)]


@pytest.mark.parametrize("training", [False, True])
@pytest.mark.parametrize("kind", ["hourglass", "hrnet_w32", "resnet50"])
def test_network_fp16_tape_against_fp64_oracle(kind, training):
    """One tape-recording forward and its backward at training precision "fp16" against the fp64 oracle.
    Eval mode (fixed BatchNorm statistics) is the well-conditioned check of the whole fp16 forward / data-gradient /
    single-pass weight-gradient chain. Train mode at these sizes amplifies round-off so much that the fp32 oracle's own
    gradients sit 1.5e-2 .. 3e-2 (relative L2) from fp64 (tests/_parity.py); fp16 operands, 2^13 times coarser, push
    its gradients O(1) away from the exact ones, so there the bounds only catch gross errors (a missing operand scale
    is off by 2^14 and more), and test_overfit_one_batch_fp16_follows_fp32 checks what training does with them."""
    from fpd_b200 import ops as o
    from fpd_b200.engine import set_training_precision
    from oracle import hourglass_oracle as O
    net, xshape, J, oracle = _network(kind, training)
    g = torch.Generator(device="cuda").manual_seed(4)
    x = torch.randn(*xshape, device="cuda", generator=g)
    h, w = xshape[2] // 4, xshape[3] // 4
    target = torch.rand(xshape[0], J, h, w, device="cuda", generator=g)
    tw = (torch.rand(xshape[0], J, 1, device="cuda", generator=g) > 0.2).float()
    sd0 = {k: v.detach().clone() for k, v in net.state_dict().items()}
    assert set_training_precision(net, "fp16") == "fp32"
    eng = net.engine()
    ctx = eng.forward(x, training, record_tape=True)
    outs = [v.data.clone() for v in ctx.outs]
    _, grads = o.fpd_loss([v.data for v in ctx.outs], target, None, tw, 0.0)
    pg = eng.backward(ctx, grads)
    ours = {k: pg[p] for k, p in net.named_parameters()}
    set_training_precision(net, "fp32")
    res = {}
    for dtype in (torch.float32, torch.float64):
        sd = P.cast_sd(sd0, dtype)
        params = P.with_grad(sd)
        ref_outs = oracle(sd, x.to(dtype))
        loss, _, _ = O.fpd_loss(ref_outs, target.to(dtype), tw.to(dtype))
        loss.backward()
        res[dtype] = ([t.detach() for t in ref_outs], {k: p.grad.detach() for k, p in params.items()})
    assert all(torch.isfinite(t).all() for t in outs) and all(torch.isfinite(v).all() for v in ours.values())
    herr = [relerr(nchw(a), b) for a, b in zip(outs, res[torch.float64][0])]
    rep = P.grad_report(ours, res[torch.float32][1], res[torch.float64][1], "fp16 training %s" % kind)
    per_tensor = sorted(r[1] for r in rep["rows"])
    print("%s fp16 %s mode: heat-map max-relative %s; gradient relative L2 %.3e (fp32 oracle %.3e), per-tensor "
          "error median %.3e q90 %.3e, median ratio to the fp32 oracle's %.1f" % (
              kind, "train" if training else "eval", ["%.2e" % e for e in herr], rep["l2_ours"], rep["l2_fp32"],
              per_tensor[len(per_tensor) // 2], rep["q90_ours"], rep["median_ratio"]))
    if training:
        assert max(herr) <= 0.25, herr
        assert rep["l2_ours"] <= 1.5, rep["l2_ours"]
        assert per_tensor[len(per_tensor) // 2] <= 1.5
    else:
        assert max(herr) <= 1e-2, herr
        assert rep["l2_ours"] <= 2e-2, rep["l2_ours"]
        assert per_tensor[len(per_tensor) // 2] <= 2e-2
        assert rep["median_ratio"] <= 2.0 ** 13            # fp16's unit round-off over fp32's


# ------------------------------------------------------------------------------------------------ training
def test_overfit_one_batch_fp16_follows_fp32():
    from bench import synthetic_batch
    from fpd_b200.engine import set_training_precision
    from fpd_b200.train_step import FPDTrainStep
    x, target, _ = (t.cuda() for t in synthetic_batch(4, 78, 128, 128))
    tw = torch.ones(4, 16, 1, device="cuda")
    torch.manual_seed(6)
    init = {k: v.clone() for k, v in _small_hourglass(64, 2).state_dict().items()}
    steps = 600
    res = {}
    for prec in ("fp32", "fp16"):
        net = _small_hourglass(64, 2)
        net.load_state_dict(init)
        net = net.cuda()
        set_training_precision(net, prec)
        step = FPDTrainStep(net, None, lr=1e-3)
        losses = []
        for i in range(steps):
            losses.append(step.step(x, target, tw)[2].clone())
        torch.cuda.synchronize()
        heat = step.last_outs[-1].clone()                 # NHWC heat-maps of the last step's forward
        res[prec] = ([v.item() for v in losses], heat)
    l32, l16 = res["fp32"][0], res["fp16"][0]
    h32, h16 = res["fp32"][1], res["fp16"][1]
    B, h, w, J = h32.shape
    i32 = h32.permute(0, 3, 1, 2).reshape(B * J, -1).argmax(1)
    i16 = h16.permute(0, 3, 1, 2).reshape(B * J, -1).argmax(1)
    near = (((i32 % w - i16 % w).abs() <= 1) & ((i32 // w - i16 // w).abs() <= 1)).float().mean().item()
    print("over-fit %d steps: loss %.4e -> fp32 %.4e, fp16 %.4e; arg-max within one pixel on %.1f %% of the joints" % (
        steps, l32[0], l32[-1], l16[-1], 100 * near))
    assert all(v == v and abs(v) < float("inf") for v in l16)
    assert l16[-1] <= 0.5 * l16[0]
    assert l16[-1] <= 2.0 * l32[-1]
    assert near >= 0.75


def _fpd_run_at(F, graph, prec, init_s, init_t, loader, crits):
    from fpd_b200.engine import set_training_precision
    s, t = _small_hourglass(64, 2), _small_hourglass(64, 1)
    s.load_state_dict(init_s)
    t.load_state_dict(init_t)
    s, t = s.cuda(), t.cuda()
    set_training_precision(s, prec)
    opt = torch.optim.Adam(list(s.parameters()), lr=1e-3)
    rec = _call(F, graph, F.fpd_train, _cfg(1), loader, s, t, crits[0], crits[1], opt, 0, "/tmp", "/tmp", "wd")
    return _state(s, opt), rec


def test_fpd_train_graph_route_equals_eager_route_in_fp16(F):
    from fpd_b200.lib.core.loss import JointsMSELoss
    init_s, init_t = _inits(7)
    loader = _loader(3, short=1)
    crits = (JointsMSELoss(True), JointsMSELoss(True))
    st_e, rec_e = _fpd_run_at(F, False, "fp16", init_s, init_t, loader, crits)
    st_g, rec_g = _fpd_run_at(F, True, "fp16", init_s, init_t, loader, crits)
    assert F._rec[2]["graph"] == 3
    _assert_same(st_g, st_e)
    assert rec_g == rec_e
    st_32, _ = _fpd_run_at(F, True, "fp32", init_s, init_t, loader, crits)
    assert not torch.equal(st_32[0]["conv1.weight"], st_g[0]["conv1.weight"])     # fp16 really ran


def test_train_graph_route_equals_eager_route_in_fp16_hrnet(F):
    from fpd_b200.engine import set_training_precision
    from fpd_b200.lib.core.loss import JointsMSELoss
    torch.manual_seed(8)
    init = {k: v.clone() for k, v in _hrnet().state_dict().items()}
    loader = _loader(3, hw=(128, 96), J=17, short=1)
    runs = []
    for graph in (False, True):
        net = _hrnet()
        net.load_state_dict(init)
        net = net.cuda()
        set_training_precision(net, "fp16")
        opt = torch.optim.Adam(net.parameters(), lr=1e-3)
        rec = _call(F, graph, F.train, _cfg(2, 17), loader, net, JointsMSELoss(True), opt, 0, "/tmp", "/tmp", "wd")
        runs.append((_state(net, opt), rec))
    assert F._rec[2]["graph"] == 3
    _assert_same(runs[1][0], runs[0][0])
    assert runs[1][1] == runs[0][1]


def test_switching_captures_again_and_back_is_bit_identical():
    """A cached FPDTrainStep captures again after each switch; a step after switching back equals the step of a network
    that never switched (gradients, losses, running statistics)."""
    from bench import synthetic_batch
    from fpd_b200.engine import set_training_precision
    from fpd_b200.train_step import FPDTrainStep
    x, target, tw = (t.cuda() for t in synthetic_batch(2, 79, 128, 128))
    torch.manual_seed(9)
    init = {k: v.clone() for k, v in _small_hourglass(64, 2).state_dict().items()}

    def make():
        net = _small_hourglass(64, 2)
        net.load_state_dict(init)
        net = net.cuda()
        return net, FPDTrainStep(net, None, fused_adam=False)

    def result(net, step, losses):
        torch.cuda.synchronize()
        return (losses.clone(), step.flat.grad.clone(), [b.clone() for b in net.buffers()])
    net_a, step_a = make()
    ref = result(net_a, step_a, step_a.step(x, target, tw))

    net_b, step_b = make()
    captures = []
    cap = step_b._capture
    step_b._capture = lambda *a: captures.append(1) or cap(*a)
    set_training_precision(net_b, "fp16")
    r16 = result(net_b, step_b, step_b.step(x, target, tw))
    net_b.load_state_dict(init)                     # in place: back to the initial running statistics
    assert set_training_precision(net_b, "fp32") == "fp16"
    r32 = result(net_b, step_b, step_b.step(x, target, tw))
    step_b.step(x, target, tw)                      # no switch: the graph is replayed
    assert len(captures) == 2
    assert not torch.equal(r16[1], ref[1])
    assert torch.equal(r32[0], ref[0]) and torch.equal(r32[1], ref[1])
    assert all(torch.equal(a, b) for a, b in zip(r32[2], ref[2]))
