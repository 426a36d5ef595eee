"""FP16 activation storage (inference precision "fp16_act") on the H100: every half-I/O kernel form bit for bit against
the fp32-activation kernel it derives from, saturation and NaN, determinism and graph replay, whole networks against the
oracle, key points on trained-like heat-maps, the validation graph, the FPD step with an "fp16_act" teacher, and the
activation memory of an eval forward."""
import importlib.util
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
_spec = importlib.util.spec_from_file_location("_infer_f16_gpu", os.path.join(HERE, "test_infer_f16_gpu.py"))
F16 = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(F16)

H16, F32 = torch.float16, torch.float32


@pytest.fixture(scope="module", autouse=True)
def _fp32_reference_mode():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield


def ops():
    import fpd_b200  # noqa: F401
    from fpd_b200 import ops as o
    return o


def rnd16(t):
    """fp16_rn of t saturated to +-65504: the rounding every fp16 store makes."""
    return t.clamp(-65504.0, 65504.0).half()


# ------------------------------------------------------------------------------------------- convolution kernels
IO_SHAPES = [s for s in F16.SHAPES if s[3] not in (1024, 2048)]      # the 11 shapes on the halo and 1x1 kernels
STAGED_SHAPES = [s for s in F16.SHAPES if s[3] in (1024, 2048)]
COMBOS = [(F32, H16), (H16, H16), (H16, F32), (F32, F32)]            # (input, output): stem, body, head, fp32


def test_shape_lists_cover_the_planner():
    o = ops()
    assert len(IO_SHAPES) == 11 and len(STAGED_SHAPES) == 2
    assert all(o.conv2d_tc_f16x1_kernel(*s) in ("halo", "1x1") for s in IO_SHAPES)
    assert all(o.conv2d_tc_f16x1_kernel(*s) == "staged" for s in STAGED_SHAPES)


@pytest.mark.parametrize("combo", COMBOS, ids=["f32in_f16out", "f16in_f16out", "f16in_f32out", "f32in_f32out"])
@pytest.mark.parametrize("shape", IO_SHAPES)
def test_io_forms_bit_exact_against_fp32_kernel(shape, combo):
    """conv2d_tc_f16x1_io == conv2d_tc_f16x1 on the widened input and residual, rounded like the store, bit for bit:
    with and without BN + ReLU, bias and residual."""
    B, H, W, Cin, Cout, k = shape
    tin, tout = combo
    o = ops()
    x, mean, scale, shift, w, bias, res, _ = F16._operands(shape, 21)
    w1, _ = o.weight_prep_f16(w, split=False)
    xi = x.to(tin)
    ri = res.to(tout)
    for kw in (dict(mean=mean, scale=scale, shift=shift, relu=True, bias=bias, residual=ri),
               dict(scale=scale, shift=shift, relu=True),
               dict(bias=bias),
               dict(residual=ri),
               dict()):
        y = o.conv2d_tc_f16x1_io(xi, w1, k, out_dtype=tout, **kw)
        assert y.dtype == tout and y.shape == (B, H, W, Cout)
        kw32 = dict(kw)
        if "residual" in kw32:
            kw32["residual"] = ri.float()
        ref = o.conv2d_tc_f16x1(xi.float(), w1, k, **kw32)
        if tout == H16:
            ref = rnd16(ref)
        assert torch.equal(y, ref), (shape, combo, sorted(kw))


def test_io_forms_refuse_the_staged_shapes():
    o = ops()
    for shape in STAGED_SHAPES:
        x, _, _, _, w, _, _, _ = F16._operands(shape, 22)
        w1, _ = o.weight_prep_f16(w, split=False)
        with pytest.raises(RuntimeError, match="staged"):
            o.conv2d_tc_f16x1_io(x.half(), w1, shape[-1])
    with pytest.raises(ValueError):                                      # residual of another type than y
        x, _, _, _, w, _, res, _ = F16._operands(IO_SHAPES[0], 23)
        o.conv2d_tc_f16x1_io(x.half(), o.weight_prep_f16(w, split=False)[0], 3, residual=res, out_dtype=H16)


@pytest.mark.parametrize("shape", [(2, 37, 64, 128, 128, 3), (2, 19, 48, 256, 256, 1)])
def test_conv_saturates_and_propagates_nan(shape):
    o = ops()
    k = shape[-1]
    x, _, _, _, w, bias, res, _ = F16._operands(shape, 24)
    w1, _ = o.weight_prep_f16(w, split=False)
    r = res.half()
    r[0, 0, 0, :4] = float("nan")
    big = torch.full_like(bias, 1e6)
    big[1::2] = -1e6
    y = o.conv2d_tc_f16x1_io(x.half(), w1, k, bias=big, residual=r, out_dtype=H16)
    yf = y.float()
    assert not torch.isinf(yf).any()
    assert torch.isnan(yf[0, 0, 0, :4]).all()
    assert torch.isnan(yf).sum().item() == 4
    finite = yf[~torch.isnan(yf)].view(-1)
    assert (finite.abs() == 65504.0).all()                               # every output is past the fp16 range
    assert torch.equal(torch.isnan(y), torch.isnan(rnd16(o.conv2d_tc_f16x1(x.half().float(), w1, k, bias=big,
                                                                          residual=r.float()))))


@pytest.mark.parametrize("shape", [(2, 37, 64, 128, 128, 3), (2, 19, 48, 256, 256, 1)])
def test_io_forms_deterministic_and_graph_replay(shape):
    o = ops()
    x, mean, scale, shift, w, bias, res, _ = F16._operands(shape, 25)
    w1, _ = o.weight_prep_f16(w, split=False)
    xh, rh = x.half(), res.half()
    kw = dict(mean=mean, scale=scale, shift=shift, relu=True, bias=bias, residual=rh, out_dtype=H16)
    y0 = o.conv2d_tc_f16x1_io(xh, w1, shape[-1], **kw)
    assert torch.equal(o.conv2d_tc_f16x1_io(xh, w1, shape[-1], **kw), y0)
    out = torch.empty_like(y0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        o.conv2d_tc_f16x1_io(xh, w1, shape[-1], out=out, **kw)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        o.conv2d_tc_f16x1_io(xh, w1, shape[-1], out=out, **kw)
    out.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, y0)


# ------------------------------------------------------------------------------------------- elementwise kernels
def _glue_cases(seed):
    """-> [(name, fp16 call, fp32 call on the widened inputs)] for every fp16 form of the eval glue."""
    o = ops()
    g = torch.Generator(device="cuda").manual_seed(seed)
    C = 48
    x = (torch.randn(2, 16, 24, C, device="cuda", generator=g) * 3).half()
    r = (torch.randn(2, 16, 24, C, device="cuda", generator=g) * 3).half()
    mean = torch.randn(C, device="cuda", generator=g)
    scale = torch.rand(C, device="cuda", generator=g) + 0.5
    shift = torch.randn(C, device="cuda", generator=g)
    low = [(torch.randn(2, 16 >> s, 24 >> s, C, device="cuda", generator=g) * 2).half() for s in range(4)]
    cases = []
    for relu in (False, True):
        for m in (None, mean):
            cases.append(("affine_act relu=%d mean=%d" % (relu, m is not None),
                          lambda relu=relu, m=m: o.affine_act_f16(x, scale, shift, relu, mean=m),
                          lambda relu=relu, m=m: o.affine_act(x.float(), scale, shift, relu, mean=m)))
            cases.append(("affine_add_act relu=%d mean=%d" % (relu, m is not None),
                          lambda relu=relu, m=m: o.affine_add_act_f16(x, r, scale, shift, relu, mean=m),
                          lambda relu=relu, m=m: o.affine_add_act(x.float(), r.float(), scale, shift, relu, mean=m)))
    cases.append(("affine_act identity", lambda: o.affine_act_f16(x), lambda: o.affine_act(x.float())))
    for shifts in ((0, 1), (0, 1, 2, 3), (2, 0, 1), (1, 0)):
        for relu in (True, False):
            terms = [low[s] for s in shifts]
            cases.append(("fuse_sum %s relu=%d" % (shifts, relu),
                          lambda terms=terms, shifts=shifts, relu=relu: o.fuse_sum_f16(terms, list(shifts), relu),
                          lambda terms=terms, shifts=shifts, relu=relu: o.fuse_sum([t.float() for t in terms],
                                                                                   list(shifts), relu)))
    cases.append(("maxpool2x2", lambda: o.maxpool2x2_f16(x), lambda: o.maxpool2x2(x.float())))
    cases.append(("upsample2x_add", lambda: o.upsample2x_add_f16(x, low[1]),
                  lambda: o.upsample2x_add(x.float(), low[1].float())))
    cases.append(("subsample2", lambda: o.subsample2_f16(x), lambda: o.subsample2(x.float())))
    return cases


def test_glue_forms_bit_exact_against_fp32_kernels():
    for name, f16, f32 in _glue_cases(31):
        y = f16()
        assert y.dtype == H16, name
        assert torch.equal(y, rnd16(f32())), name
    o = ops()
    x = (torch.randn(3, 5, 7, 12, device="cuda") * 100).half()
    assert torch.equal(o.half_to_float(x), x.float())


def test_glue_saturates_and_propagates_nan():
    o = ops()
    C = 16
    x = torch.randn(2, 4, 6, C, device="cuda").half()
    x[0, 0, 0, :4] = float("nan")
    scale = torch.full((C,), 1e6, device="cuda")
    scale[::2] = -1e6
    shift = torch.zeros(C, device="cuda")
    y = o.affine_act_f16(x, scale, shift, False).float()
    assert not torch.isinf(y).any() and torch.isnan(y[0, 0, 0, :4]).all()
    big = y[~torch.isnan(y)]
    assert (big.abs() == 65504.0).sum() > 0.9 * big.numel()
    s = o.fuse_sum_f16([torch.full_like(x, 60000.0), torch.full_like(x, 60000.0)], [0, 0], relu=False).float()
    assert torch.equal(s, torch.full_like(s, 65504.0))
    a = o.upsample2x_add_f16(x, torch.full((2, 2, 3, C), -60000.0, device="cuda").half()).float()
    assert not torch.isinf(a).any() and torch.isnan(a[0, 0, 0, :4]).all()
    assert torch.isnan(o.subsample2_f16(x).float()[0, 0, 0, :4]).all()
    assert torch.isnan(o.affine_add_act_f16(x, x, relu=False).float()[0, 0, 0, :4]).all()
    assert torch.isnan(o.half_to_float(x)[0, 0, 0, :4]).all()


def test_glue_deterministic_and_graph_replay():
    cases = _glue_cases(32)
    first = [f16().clone() for _, f16, _ in cases]
    assert all(torch.equal(f16(), y) for (_, f16, _), y in zip(cases, first))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _, f16, _ in cases:
            f16()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = [f16() for _, f16, _ in cases]
    for t in outs:
        t.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(outs, first))


# ------------------------------------------------------------------------------------------- networks
@pytest.mark.parametrize("kind", ["hourglass", "hrnet_w32"])
def test_network_fp16_act_against_oracle(kind):
    from fpd_b200.engine import set_inference_precision
    net, xshape, oracle = F16._network(kind)
    x = torch.randn(*xshape, device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))
    sd = {k: v.detach().clone() for k, v in net.state_dict().items()}
    with torch.no_grad():
        ref = oracle(sd, x)
        base = [t.clone() for t in net.forward_nhwc(x, training=False)]
    tape32 = F16._last(net(x)).detach().clone()
    errs = {}
    for prec in ("fp16", "fp16_act"):
        set_inference_precision(net, prec)
        with torch.no_grad():
            got = net.forward_nhwc(x, training=False)
            got_net = F16._last(net(x))
        assert len(got) == len(ref) and all(g.dtype == F32 for g in got) and got_net.dtype == F32
        errs[prec] = [F16.relerr(F16.nchw(g), r) for g, r in zip(got, ref)]
        assert F16.relerr(got_net, ref[-1]) <= 1e-2
    print("%s max-relative error per output vs the oracle: fp16 %s, fp16_act %s" % (
        kind, ["%.2e" % e for e in errs["fp16"]], ["%.2e" % e for e in errs["fp16_act"]]))
    assert all(e <= 1e-2 for e in errs["fp16_act"]), errs
    assert torch.equal(F16._last(net(x)).detach(), tape32)            # tape-recording forwards stay at fp32 grade
    assert set_inference_precision(net, "fp32") == "fp16_act"
    with torch.no_grad():
        again = net.forward_nhwc(x, training=False)
    assert all(torch.equal(a, b) for a, b in zip(again, base))


def test_network_fp16_act_deterministic():
    from fpd_b200.engine import set_inference_precision
    net, xshape, _ = F16._network("hrnet_w32")
    x = torch.randn(*xshape, device="cuda", generator=torch.Generator(device="cuda").manual_seed(4))
    set_inference_precision(net, "fp16_act")
    with torch.no_grad():
        a = net.forward_nhwc(x, training=False)[-1].clone()
        b = net.forward_nhwc(x, training=False)[-1]
    assert torch.equal(a, b)


def test_trained_like_heatmaps_keypoints_fp16_act_vs_fp32():
    """Over-fit one batch as the "fp16" test does, then compare the flip-test key points: every joint within one pixel."""
    import fpd_b200  # noqa: F401
    from bench import synthetic_batch
    from fpd_b200.engine import set_inference_precision
    from fpd_b200.infer_step import FlipTestInference
    from fpd_b200.train_step import FPDTrainStep
    pairs = F16._flip_perm()
    torch.manual_seed(5)
    net = F16._hourglass().cuda()
    x, target, _ = (t.cuda() for t in synthetic_batch(4, 77))
    tw = torch.ones(4, 16, 1, device="cuda")
    xb = torch.cat([x, x.flip(3)]).contiguous()
    tb = torch.cat([target, F16._flipped_targets(target, pairs)]).contiguous()
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
    set_inference_precision(net, "fp16_act")
    r16 = inf(x)
    idx16, max16 = r16["idx"].clone(), r16["maxval"].clone()
    torch.cuda.synchronize()
    assert (max32 > 0.25).float().mean() > 0.9, "over-fit did not produce peaky heat-maps"
    w = 64
    dx = (idx16 % w - idx32 % w).abs()
    dy = (idx16 // w - idx32 // w).abs()
    print("trained-like key points at fp16_act: %.1f %% identical, max |dx| %d, |dy| %d, max |dmaxval| %.2e" % (
        100 * (idx16 == idx32).float().mean().item(), dx.max().item(), dy.max().item(),
        (max16 - max32).abs().max().item()))
    assert dx.max().item() <= 1 and dy.max().item() <= 1


def test_validate_graph_equals_eager_at_fp16_act():
    import fpd_b200  # noqa: F401
    from fpd_b200.engine import set_inference_precision
    from fpd_b200.infer_step import FlipTestInference
    torch.manual_seed(1)
    net = F16._randomise_bn(F16._hourglass(64, 2)).cuda().eval()
    g = torch.Generator(device="cuda").manual_seed(9)
    x = torch.randn(4, 3, 256, 256, device="cuda", generator=g)
    target = torch.rand(4, 16, 64, 64, device="cuda", generator=g)
    tw = torch.ones(4, 16, 1, device="cuda")
    inv = np.tile(np.array([[4.0, 0.0, 0.0, 0.0, 4.0, 0.0]]), (4, 1))
    kw = dict(inv=inv, target=target, target_weight=tw)
    graph = FlipTestInference(net, F16._flip_perm(), decode=True)
    eager = FlipTestInference(net, F16._flip_perm(), decode=True, use_graph=False)
    set_inference_precision(net, "fp16")
    r16 = {k: v.clone() for k, v in graph(x, **kw).items() if torch.is_tensor(v)}
    set_inference_precision(net, "fp16_act")
    ra = {k: v.clone() for k, v in graph(x, **kw).items() if torch.is_tensor(v)}
    ea = eager(x, **kw)
    torch.cuda.synchronize()
    assert not torch.equal(ra["avg_nhwc"], r16["avg_nhwc"])        # the graph captured again in the new precision
    for k in ("idx", "maxval", "avg_nhwc", "preds", "loss3", "pck"):
        assert torch.equal(ra[k], ea[k]), k


def _fpd_pair(kind):
    torch.manual_seed(2)
    if kind == "hourglass":
        return F16._hourglass(64, 2).cuda(), F16._randomise_bn(F16._hourglass(128, 1)).cuda(), 16, (256, 256)
    from bench import hrnet_cfg
    from fpd_b200.lib.models import pose_hrnet as H
    student = H.get_pose_net(hrnet_cfg(32), False).cuda()
    teacher = F16._randomise_bn(H.get_pose_net(hrnet_cfg(48), False)).cuda()
    return student, teacher, 17, (256, 192)


def _fpd_run(kind, graph, precs, warm=None):
    """FPD steps of a fresh (student, teacher) pair; precs[i]: the teacher's inference precision set before step i (and,
    for i = 0, before the step object is made); warm: a precision the teacher runs one eval forward at first.
    -> (losses, flat parameters, teacher heat-maps of each step)."""
    import fpd_b200  # noqa: F401
    from fpd_b200.engine import set_inference_precision
    from fpd_b200.train_step import FPDTrainStep
    student, teacher, J, (h, w) = _fpd_pair(kind)
    g = torch.Generator(device="cuda").manual_seed(6)
    x = torch.randn(2, 3, h, w, device="cuda", generator=g)
    target = torch.rand(2, J, h // 4, w // 4, device="cuda", generator=g)
    tw = torch.ones(2, J, 1, device="cuda")
    if warm is not None:
        set_inference_precision(teacher, warm)
        with torch.no_grad():
            teacher.forward_nhwc(x, training=False)
    set_inference_precision(teacher, precs[0])
    step = FPDTrainStep(student, teacher, use_graph=graph)
    losses, teach = [], []
    for p in precs:
        set_inference_precision(teacher, p)
        losses.append(step.step(x, target, tw).clone())
        teach.append(step.last_teacher.clone())
    torch.cuda.synchronize()
    with torch.no_grad():
        t_ref = teacher.forward_nhwc(x, training=False)[-1]
    assert torch.equal(step.last_teacher, t_ref)
    return torch.stack(losses), step.flat.flat.clone(), torch.stack(teach)


@pytest.mark.parametrize("kind", ["hourglass", "hrnet"])
def test_fpd_step_with_fp16_act_teacher(kind):
    """Graph capture and replay: two identical runs are bit-identical, and equal the eager route; switching the teacher
    back to "fp32" gives what never switching gives."""
    a = _fpd_run(kind, True, ["fp16_act", "fp16_act"])
    b = _fpd_run(kind, True, ["fp16_act", "fp16_act"])
    e = _fpd_run(kind, False, ["fp16_act", "fp16_act"])
    assert all(torch.equal(u, v) for u, v in zip(a, b))
    assert all(torch.equal(u, v) for u, v in zip(a, e))
    never = _fpd_run(kind, True, ["fp32", "fp32"])
    assert not torch.equal(a[2][0], never[2][0])
    # back to "fp32" after a captured "fp16_act" step: the graph captures again and the teacher is the fp32 one
    back = _fpd_run(kind, True, ["fp16_act", "fp32"])
    assert torch.equal(back[2][1], never[2][1])
    # a teacher that ran at "fp16_act" before the step was made, then switched back: every result equals never switching
    first = _fpd_run(kind, True, ["fp32", "fp32"], warm="fp16_act")
    assert all(torch.equal(u, v) for u, v in zip(first, never))


def test_eval_forward_peak_memory_lower_than_fp16():
    from fpd_b200.engine import set_inference_precision
    net = F16._randomise_bn(F16._hourglass()).cuda().eval()
    x = torch.randn(32, 3, 256, 256, device="cuda")
    peaks = {}
    for prec in ("fp16", "fp16_act", "fp16", "fp16_act"):     # second round: weights cached, allocator warm
        set_inference_precision(net, prec)
        with torch.no_grad():
            net.forward_nhwc(x, training=False)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            out = net.forward_nhwc(x, training=False)
            torch.cuda.synchronize()
            peaks[prec] = torch.cuda.max_memory_allocated() - base
            del out
    print("hourglass s4 f128, B = 32, one eval forward: peak allocated above the resident state: fp16 %.1f MiB, "
          "fp16_act %.1f MiB" % (peaks["fp16"] / 2 ** 20, peaks["fp16_act"] / 2 ** 20))
    assert peaks["fp16_act"] < peaks["fp16"]
