"""Single-pass FP16 inference (ops.conv2d_tc_f16x1, engine.set_inference_precision) on the H100: the kernels against fp64
convolutions of the fp16-rounded operands, kernel selection, determinism and graph replay, whole networks against the
oracle, key points on trained-like heat-maps, and the graphs that run a network in this mode (validation flip test,
FPD training step with an fp16 teacher)."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


@pytest.fixture(scope="module", autouse=True)
def _fp32_reference_mode():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield


def ops():
    import fpd_b200  # noqa: F401
    from fpd_b200 import ops as o
    return o


def relerr(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30)).item()


def nchw(x):
    return x.permute(0, 3, 1, 2).contiguous()


def kernel_names(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type is not None and "cuda" in str(e.device_type).lower()]


# B, H, W, Cin, Cout, k: ragged last tiles, tiles across images, 1-4 output slices, every planner choice
SHAPES = [
    (3, 5, 7, 16, 48, 3),        # halo, Cin below one channel block
    (2, 13, 64, 48, 96, 3),      # halo, partial channel block
    (1, 37, 64, 128, 128, 3),    # halo, the teacher's shape with a ragged last tile
    (1, 24, 128, 128, 64, 3),    # halo at W = 128 with two channel blocks
    (2, 8, 6, 384, 384, 3),      # halo, HRNet-w48's 384-channel branch: three slices
    (2, 9, 11, 256, 512, 3),     # halo, four slices
    (1, 6, 6, 2048, 64, 3),      # staged: the halo does not fit
    (2, 19, 48, 64, 128, 1),     # 1x1 resident
    (3, 7, 9, 256, 256, 1),      # 1x1 resident, two slices
    (1, 33, 40, 384, 64, 1),
    (2, 16, 16, 640, 128, 1),    # 1x1 resident at Cin = 640
    (1, 8, 8, 1024, 256, 1),     # staged
    (2, 11, 13, 16, 48, 1),
]


def _operands(shape, seed):
    B, H, W, Cin, Cout, k = shape
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, H, W, Cin, device="cuda", generator=g) * 2 + 0.5
    mean = torch.randn(Cin, device="cuda", generator=g)
    scale = torch.rand(Cin, device="cuda", generator=g) + 0.5
    shift = torch.randn(Cin, device="cuda", generator=g) * 0.5 + 0.75
    w = torch.randn(Cout, Cin, k, k, device="cuda", generator=g) * (1.0 / (Cin * k * k) ** 0.5)
    bias = torch.randn(Cout, device="cuda", generator=g)
    res = torch.randn(B, H, W, Cout, device="cuda", generator=g)
    mask = torch.randn(B, H, W, Cout, device="cuda", generator=g)
    return x, mean, scale, shift, w, bias, res, mask


@pytest.mark.parametrize("shape", SHAPES)
def test_kernel_against_fp64_of_rounded_operands(shape):
    B, H, W, Cin, Cout, k = shape
    o = ops()
    x, mean, scale, shift, w, bias, res, mask = _operands(shape, 11)
    w1, lo = o.weight_prep_f16(w, split=False)
    assert lo is None
    y = o.conv2d_tc_f16x1(x, w1, k, mean=mean, scale=scale, shift=shift, relu=True, bias=bias, residual=res,
                          relu_mask=mask)
    # the kernel's operand: fmaf(x - mean, scale, shift) in fp32, ReLU, saturated, rounded to fp16 (RN)
    a32 = ((x - mean).double() * scale.double() + shift.double()).float().clamp_min(0.0)
    a16 = a32.clamp(-65504.0, 65504.0).half().double()
    w16 = w1.double().view(k, k, Cout, Cin).permute(2, 3, 0, 1) / 256.0
    keep = (nchw(mask) > 0).double()
    ref = (F.conv2d(nchw(a16), w16, bias.double(), padding=k // 2) + nchw(res).double()) * keep
    exact = (F.conv2d(nchw(a32).double(), w.double(), bias.double(), padding=k // 2) + nchw(res).double()) * keep
    torch.cuda.synchronize()
    assert relerr(nchw(y), ref) <= 1e-4, "%s: %.3e vs rounded operands" % (shape, relerr(nchw(y), ref))
    assert relerr(nchw(y), exact) <= 2e-3, "%s: %.3e vs unrounded operands" % (shape, relerr(nchw(y), exact))


def test_kernel_without_prologue_or_epilogue():
    """Raw input (no affine, no ReLU: negative operands), no bias / residual / mask, output scale."""
    o = ops()
    for shape in ((2, 9, 10, 64, 64, 3), (2, 9, 10, 128, 64, 1)):
        x, _, _, _, w, _, _, _ = _operands(shape, 12)
        k = shape[-1]
        w1, _ = o.weight_prep_f16(w, split=False)
        y = o.conv2d_tc_f16x1(x, w1, k, out_scale=0.5)
        w16 = w1.double().view(k, k, shape[4], shape[3]).permute(2, 3, 0, 1) / 256.0
        ref = 0.5 * F.conv2d(nchw(x.half().double()), w16, padding=k // 2)
        assert relerr(nchw(y), ref) <= 1e-4, shape


# (B, H, W, Cin, Cout, k), planner choice, the kernel that must run
SELECTION = [
    ((2, 64, 64, 128, 128, 3), "halo", "::conv_halo_f16x1_kernel<"),
    ((1, 32, 128, 128, 128, 3), "halo", "::conv_halo_f16x1_kernel<"),
    ((4, 8, 6, 384, 384, 3), "halo", "::conv_halo_f16x1_kernel<"),
    ((2, 64, 64, 256, 256, 1), "1x1", "::pw_conv_f16x1_kernel<"),
    ((2, 16, 16, 640, 128, 1), "1x1", "::pw_conv_f16x1_kernel<"),
    ((1, 8, 8, 1024, 256, 1), "staged", "::conv_wgmma_kernel<true"),
    ((1, 8, 8, 2048, 64, 3), "staged", "::conv_wgmma_kernel<true"),
]


def _selection_main():
    """Prints, per SELECTION entry, the planner's choice and the names of the kernels one call launched (JSON)."""
    import json
    o = ops()
    g = torch.Generator(device="cuda").manual_seed(404)
    out = []
    for (B, H, W, Cin, Cout, k), _, _ in SELECTION:
        x = torch.randn(B, H, W, Cin, device="cuda", generator=g)
        w1, _ = o.weight_prep_f16(torch.randn(Cout, Cin, k, k, device="cuda", generator=g) * 0.05, split=False)
        run = lambda: o.conv2d_tc_f16x1(x, w1, k)   # noqa: E731
        run()                                       # first launch outside the trace
        out.append([o.conv2d_tc_f16x1_kernel(B, H, W, Cin, Cout, k),
                    [n for n in kernel_names(run) if "_kernel" in n]])
    print(json.dumps(out))


def test_selection_by_kernel_name():
    """The planner's choice, and the profiler's name of the kernel each call ran. Traced in a fresh process, as
    tests/test_wgrad_gpu.py does: late in a long test session the profiler can return no kernel events at all."""
    import json
    import subprocess
    here = os.path.dirname(os.path.abspath(__file__))
    code = "import sys; sys.path[:0] = [%r, %r]; import test_infer_f16_gpu as t; t._selection_main()" % (here, ROOT)
    res = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-2000:]
    got = json.loads(res.stdout.strip().splitlines()[-1])
    for (args, kind, name), (planned, names) in zip(SELECTION, got):
        assert planned == kind, (args, planned)
        assert len(names) > 0 and all(name in n for n in names), (args, names)


@pytest.mark.parametrize("shape", [(2, 37, 64, 128, 128, 3), (2, 19, 48, 256, 256, 1), (1, 8, 8, 1024, 256, 1)])
def test_deterministic_and_graph_replay(shape):
    o = ops()
    x, mean, scale, shift, w, bias, res, _ = _operands(shape, 13)
    w1, _ = o.weight_prep_f16(w, split=False)
    kw = dict(mean=mean, scale=scale, shift=shift, relu=True, bias=bias, residual=res)
    y0 = o.conv2d_tc_f16x1(x, w1, shape[-1], **kw)
    for _ in range(3):
        assert torch.equal(o.conv2d_tc_f16x1(x, w1, shape[-1], **kw), y0)
    out = torch.empty_like(y0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        o.conv2d_tc_f16x1(x, w1, shape[-1], out=out, **kw)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        o.conv2d_tc_f16x1(x, w1, shape[-1], out=out, **kw)
    out.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, y0)


# ------------------------------------------------------------------------------------------------ networks
def _randomise_bn(net):
    for m in net.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.running_mean.normal_(0, 0.1)
            m.running_var.uniform_(0.5, 1.5)
    return net


def _last(out):
    return out[-1] if isinstance(out, (list, tuple)) else out


def _hourglass(f=128, s=4):
    from bench import cfg
    from fpd_b200.lib.models import hourglass as H
    return H.get_pose_net(cfg(f, s), False)


def _network(kind):
    import fpd_b200  # noqa: F401
    from bench import hrnet_cfg, resnet_cfg
    from oracle import hourglass_oracle as O
    from oracle import hrnet_oracle as HO
    from oracle import resnet_oracle as RO
    torch.manual_seed(0)
    if kind == "hourglass":
        net = _randomise_bn(_hourglass()).cuda().eval()
        return net, (2, 3, 256, 256), lambda sd, x: O.hourglass_net(sd, x, 4, training=False)
    if kind == "hrnet_w32":
        from fpd_b200.lib.models import pose_hrnet as H
        net = _randomise_bn(H.get_pose_net(hrnet_cfg(32), False)).cuda().eval()
        return net, (2, 3, 256, 192), lambda sd, x: [HO.hrnet(HO.annotate_strides(sd), x, training=False)]
    from fpd_b200.lib.models import pose_resnet as R
    net = R.get_pose_net(resnet_cfg(50), False)
    net.load_state_dict(RO.synthetic_state({k: v.shape for k, v in net.state_dict().items()}, seed=7), strict=True)
    return net.cuda().eval(), (2, 3, 256, 256), lambda sd, x: [RO.resnet(sd, x, training=False)]


@pytest.mark.parametrize("kind", ["hourglass", "hrnet_w32", "resnet50"])
def test_network_fp16_against_oracle_and_fp32_unchanged(kind):
    from fpd_b200.engine import set_inference_precision
    net, xshape, oracle = _network(kind)
    x = torch.randn(*xshape, device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))
    sd = {k: v.detach().clone() for k, v in net.state_dict().items()}
    with torch.no_grad():
        ref = oracle(sd, x)
        base = [t.clone() for t in net.forward_nhwc(x, training=False)]
        base_net = _last(net(x)).clone()
    tape32 = _last(net(x)).detach().clone()      # grad enabled: a tape-recording eval forward (autograd bridge)
    assert set_inference_precision(net, "fp16") == "fp32"
    with torch.no_grad():
        got = net.forward_nhwc(x, training=False)
        got_net = _last(net(x))
    assert len(got) == len(ref)
    errs = [relerr(nchw(g), r) for g, r in zip(got, ref)]
    print("%s fp16 max-relative error per stack vs the oracle: %s" % (kind, ["%.2e" % e for e in errs]))
    assert all(e <= 1e-2 for e in errs), errs
    assert relerr(got_net, ref[-1]) <= 1e-2
    assert torch.equal(_last(net(x)).detach(), tape32)                # tape-recording forwards stay at fp32 grade
    assert set_inference_precision(net, "fp32") == "fp16"
    with torch.no_grad():
        again = net.forward_nhwc(x, training=False)
        assert torch.equal(_last(net(x)), base_net)
    assert all(torch.equal(a, b) for a, b in zip(again, base))


def _flipped_targets(target, pairs):
    """Target of the mirrored image such that flip_back + shift-by-one lands on `target` again."""
    t = target.clone()
    t[:, :, :, :-1] = target[:, :, :, 1:]
    perm = list(range(t.shape[1]))
    for a, b in pairs:
        perm[a], perm[b] = b, a
    return t.flip(3)[:, perm].contiguous()


def _flip_perm():
    from oracle import decode_oracle as D
    return D.MPII_FLIP_PAIRS


def test_trained_like_heatmaps_keypoints_fp16_vs_fp32():
    """Over-fit one batch (as test_argmax_bit_exact_on_trained_like_heatmaps does), then compare the flip-test key
    points of the two precisions."""
    import fpd_b200  # noqa: F401
    from bench import synthetic_batch
    from fpd_b200.engine import set_inference_precision
    from fpd_b200.infer_step import FlipTestInference
    from fpd_b200.train_step import FPDTrainStep
    pairs = _flip_perm()
    torch.manual_seed(5)
    net = _hourglass().cuda()
    x, target, _ = (t.cuda() for t in synthetic_batch(4, 77))
    tw = torch.ones(4, 16, 1, device="cuda")
    xb = torch.cat([x, x.flip(3)]).contiguous()
    tb = torch.cat([target, _flipped_targets(target, pairs)]).contiguous()
    wb = torch.cat([tw, tw]).contiguous()
    step = FPDTrainStep(net, None, lr=1e-3, use_graph=True)
    steps = int(os.environ.get("FPD_OVERFIT_STEPS", "1200"))
    for i in range(steps):
        if i == steps * 2 // 3:
            step.lr = 2.5e-4
        step.step(xb, tb, wb)
    torch.cuda.synchronize()
    net.eval()
    inf = FlipTestInference(net, pairs, shift_heatmap=True)
    r32 = inf(x)
    idx32, max32 = r32["idx"].clone(), r32["maxval"].clone()
    set_inference_precision(net, "fp16")
    r16 = inf(x)
    idx16, max16 = r16["idx"].clone(), r16["maxval"].clone()
    torch.cuda.synchronize()
    assert (max32 > 0.25).float().mean() > 0.9, "over-fit did not produce peaky heat-maps"
    same = (idx16 == idx32).float().mean().item()
    w = 64
    dx = (idx16 % w - idx32 % w).abs().max().item()
    dy = (idx16 // w - idx32 // w).abs().max().item()
    print("trained-like key points: %.1f %% identical, max |dx| %d, |dy| %d, max |dmaxval| %.2e" % (
        100 * same, dx, dy, (max16 - max32).abs().max().item()))
    assert same >= 0.99
    assert dx <= 1 and dy <= 1


def test_flip_test_graph_recaptures_and_equals_eager_in_fp16():
    import fpd_b200  # noqa: F401
    from fpd_b200.engine import set_inference_precision
    from fpd_b200.infer_step import FlipTestInference
    torch.manual_seed(1)
    net = _randomise_bn(_hourglass(64, 2)).cuda().eval()
    g = torch.Generator(device="cuda").manual_seed(9)
    x = torch.randn(4, 3, 256, 256, device="cuda", generator=g)
    target = torch.rand(4, 16, 64, 64, device="cuda", generator=g)
    tw = torch.ones(4, 16, 1, device="cuda")
    inv = np.tile(np.array([[4.0, 0.0, 0.0, 0.0, 4.0, 0.0]]), (4, 1))
    kw = dict(inv=inv, target=target, target_weight=tw)
    graph = FlipTestInference(net, _flip_perm(), decode=True)
    eager = FlipTestInference(net, _flip_perm(), decode=True, use_graph=False)
    r32 = {k: v.clone() for k, v in graph(x, **kw).items() if torch.is_tensor(v)}
    set_inference_precision(net, "fp16")
    r16 = {k: v.clone() for k, v in graph(x, **kw).items() if torch.is_tensor(v)}
    e16 = eager(x, **kw)
    torch.cuda.synchronize()
    assert not torch.equal(r16["avg_nhwc"], r32["avg_nhwc"])      # the graph captured again in the new precision
    for k in ("idx", "maxval", "avg_nhwc", "preds", "loss3", "pck"):
        assert torch.equal(r16[k], e16[k]), k


def test_fpd_train_step_with_fp16_teacher():
    """The teacher heat-map the step uses is the teacher's fp16 forward; graph and eager routes agree bit for bit."""
    import fpd_b200  # noqa: F401
    from bench import synthetic_batch
    from fpd_b200.engine import set_inference_precision
    from fpd_b200.train_step import FPDTrainStep
    x, target, tw = (t.cuda() for t in synthetic_batch(2, 5))
    results = {}
    for graph in (True, False):
        torch.manual_seed(2)
        student = _hourglass(64, 2).cuda()
        teacher = _randomise_bn(_hourglass(128, 1)).cuda()
        set_inference_precision(teacher, "fp16")
        step = FPDTrainStep(student, teacher, use_graph=graph)
        for _ in range(2):
            losses = step.step(x, target, tw)
        torch.cuda.synchronize()
        with torch.no_grad():
            t_ref = teacher.forward_nhwc(x, training=False)[-1]
        assert torch.equal(step.last_teacher, t_ref)
        results[graph] = (losses.clone(), step.flat.flat.clone())
    assert torch.equal(results[True][0], results[False][0])
    assert torch.equal(results[True][1], results[False][1])
