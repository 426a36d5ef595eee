"""Each network at the sizes the reference's fpd_coco experiments ship, against the oracle on the device.

The other network tests run the hourglass only with 16 joints on square inputs, HRNet at 256x192 and below, and
pose_resnet at 256x256 / 256x192. The shipped COCO configurations take routes those never reach
(tests/test_shipped_sizes_cpu.py records them without a GPU):
  * hourglass f256, 17 joints, 256x192: the 256 -> 17 score and 17 -> 256 score_ convolutions on the CUDA cores, the
    residual stream between stacks in fp32 (under "fp16_act": the mixed fp16 / fp32 route from the second stack on), and
    3x3 convolutions at 4x3 in the innermost level; with 8 stacks, the loss kernels' per-stack arrays at their limit
    (kMaxStacks = 8);
  * HRNet-w32 / -w48 at 384x288: branch 3 at 12x9 (odd width), the fuse step's 8x upsampling of 12x9 to 96x72, the
    stem's conv2 at 192x144, and (w48) CUDA-core weight gradients at 96x72;
  * pose_resnet-50 / 101 / 152 at 384x288: layer4 (2048 channels) at 12x9 and the deconvolution head from 12x9;
  * the hourglass at 384x288, which no hourglass can run (12x9 max-pools to 6x4): refused before any launch.

The gradient checks run one tape-recording forward and its backward through ops.fpd_loss, as
tests/test_hrnet_grad_gpu.py does: eval mode (fixed, randomised BatchNorm statistics) per tensor against fp64, train
mode by the fp64-referenced criterion of tests/_parity.py. pose_resnet-101 / -152 run in train mode only: with synthetic
running statistics their residual stream overflows the 3xFP16 operand range in eval mode (tests/test_resnet_gpu.py).
The ResNet oracles run fp64 on the host cores; everything else runs on the device.
"""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)
import _parity as P   # noqa: E402

pytestmark = pytest.mark.gpu
TOL = 1e-3
COCO_FLIP_PAIRS = [[1, 2], [3, 4], [5, 6], [7, 8], [9, 10], [11, 12], [13, 14], [15, 16]]   # lib/dataset/coco.py
J = 17

# name: (family, size, input height, input width); size = (features, stacks), HRNet width or ResNet depth
CONFIGS = {
    "hg_f256_s4": ("hourglass", (256, 4), 256, 192),
    "hg_f256_s8": ("hourglass", (256, 8), 256, 192),
    "hrnet_w32": ("hrnet", 32, 384, 288),
    "hrnet_w48": ("hrnet", 48, 384, 288),
    "resnet50": ("resnet", 50, 384, 288),
    "resnet101": ("resnet", 101, 384, 288),
    "resnet152": ("resnet", 152, 384, 288),
}


@pytest.fixture(scope="module", autouse=True)
def _fp32_reference_mode():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    det = torch.backends.cudnn.deterministic
    torch.backends.cudnn.deterministic = True
    yield
    torch.backends.cudnn.deterministic = det
    _REF.clear()


def _randomise_bn(net):
    """Running statistics and affine parameters away from their defaults (an eval-mode BatchNorm at mean 0, variance 1,
    weight 1, bias 0 is the identity)."""
    for m in net.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.running_mean.normal_(0, 0.1)
            m.running_var.uniform_(0.5, 1.5)
            m.weight.data.uniform_(0.5, 1.5)
            m.bias.data.normal_(0, 0.1)
    return net


def _build(name, seed, training):
    """-> (the network on the device in train or eval mode, oracle(sd, x, training) -> list of NCHW heat-maps, the
    device the fp64 oracle runs on)."""
    import fpd_b200  # noqa: F401
    from bench import cfg, hrnet_cfg, resnet_cfg
    from oracle import resnet_oracle as RO
    family, size, _, _ = CONFIGS[name]
    torch.manual_seed(seed)
    if family == "hourglass":
        from fpd_b200.lib.models import hourglass as HG
        net = HG.get_pose_net(cfg(size[0], size[1], J), False)
    elif family == "hrnet":
        from fpd_b200.lib.models import pose_hrnet as HR
        net = HR.get_pose_net(hrnet_cfg(size, j=J), False)
    else:
        from fpd_b200.lib.models import pose_resnet as R
        net = R.get_pose_net(resnet_cfg(size, j=J), False)
        net.load_state_dict(RO.synthetic_state({k: v.shape for k, v in net.state_dict().items()}, seed=seed))
    if family != "resnet" and not training:
        _randomise_bn(net)
    return (net.cuda().train(training),) + _oracle_fn(name)


def _oracle_fn(name):
    """-> (oracle(sd, x, training) -> list of NCHW heat-maps, the device the fp64 oracle runs on)."""
    from oracle import hourglass_oracle as O
    from oracle import hrnet_oracle as HO
    from oracle import resnet_oracle as RO
    family, size, _, _ = CONFIGS[name]
    if family == "hourglass":
        return (lambda sd, x, tr: O.hourglass_net(sd, x, size[1], training=tr)), "cuda"
    if family == "hrnet":
        return (lambda sd, x, tr: [HO.hrnet(HO.annotate_strides(sd), x, training=tr)]), "cuda"
    # fp64 on the host cores: the device's fp64 convolutions take minutes at these sizes
    return (lambda sd, x, tr: [RO.resnet(sd, x, training=tr)]), "cpu"


def _last(out):
    return out[-1] if isinstance(out, (list, tuple)) else out


def _inputs(name, B, seed):
    """N(0,1) image, uniform target and 0/1 joint weights, drawn on the host."""
    _, _, H, W = CONFIGS[name]
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 3, H, W, generator=g)
    target = torch.rand(B, J, H // 4, W // 4, generator=g)
    tw = (torch.rand(B, J, 1, generator=g) > 0.2).float()
    return x.cuda(), target.cuda(), tw.cuda()


def _engine(net, x, target, tw, training):
    """-> ([NCHW heat-map per output], loss, {name: gradient}) of the engine's tape-recording forward and backward."""
    from fpd_b200 import ops
    eng = net.engine()
    ctx = eng.forward(x, training, record_tape=True)
    outs = [ops.nhwc_to_nchw(v.data) for v in ctx.outs]
    losses, grads = ops.fpd_loss([v.data for v in ctx.outs], target, None, tw, 0.0)
    pg = eng.backward(ctx, grads)
    torch.cuda.synchronize()
    return outs, float(losses[2]), {k: pg[p] for k, p in net.named_parameters()}


def _oracle(oracle, sd0, x, target, tw, training, dtype, device, backward=True):
    """-> ([heat-maps], loss, {name: gradient} or None) of the oracle in `dtype` on `device`, by autograd."""
    from oracle import hourglass_oracle as O
    sd = P.cast_sd(sd0, dtype, device=device)
    params = P.with_grad(sd) if backward else {}
    with torch.set_grad_enabled(backward):
        outs = oracle(sd, x.to(device, dtype), training)
        loss, _, _ = O.fpd_loss(outs, target.to(device, dtype), tw.to(device, dtype))
    if backward:
        loss.backward()
    return [o.detach() for o in outs], loss.item(), ({k: p.grad.detach() for k, p in params.items()} if backward else None)


_REF = {}
_KEEP = {("hg_f256_s4", False), ("hrnet_w32", False)}      # the fp16 checks reuse these


def _reference(name, training):
    """The network, its inputs and the oracle's fp32 and fp64 evaluations (shared by the fp32 and fp16 checks)."""
    key = (name, training)
    if key not in _REF:
        seed = 17 + 2 * list(CONFIGS).index(name) + int(training)
        net, oracle, dev64 = _build(name, seed, training)
        x, target, tw = _inputs(name, 2, 100 + seed)
        sd0 = {k: v.detach().clone() for k, v in net.state_dict().items()}
        backward = name != "hg_f256_s8" or training
        r32 = _oracle(oracle, sd0, x, target, tw, training, torch.float32, "cuda", backward)
        r64 = _oracle(oracle, sd0, x, target, tw, training, torch.float64, dev64, backward)
        for k in [k for k in _REF if k not in _KEEP]:      # the fp64 gradients of w48 alone are 0.5 GB
            del _REF[k]
        _REF[key] = (net, sd0, (x, target, tw), r32, r64)
    return _REF[key]


def _per_tensor(grads, g64):
    """-> [(relative L2 error, max-relative error, name)] of every tensor against fp64, worst L2 first."""
    errs = []
    for k, ref in g64.items():
        ref = ref.double().cpu()
        o = grads[k].reshape(ref.shape).double().cpu()
        errs.append((((o - ref).norm() / ref.norm().clamp_min(1e-300)).item(), P.rel_max(o, ref), k))
    return sorted(errs, reverse=True)


# ------------------------------------------------------------------------------------------------ fp32 against fp64
@pytest.mark.parametrize("name", ["hg_f256_s4", "hg_f256_s8", "hrnet_w32", "hrnet_w48", "resnet50"])
def test_eval_mode_against_fp64(name):
    """Fixed BatchNorm statistics: every heat-map, and (except the 8-stack hourglass, forward only) every parameter
    gradient per tensor: relative L2 within 2e-3, max-relative within 2e-2, the whole gradient within 3x the fp32
    oracle's error."""
    net, sd0, (x, target, tw), (o32, _, g32), (o64, l64, g64) = _reference(name, False)
    net.load_state_dict(sd0)
    outs, loss, ours = _engine(net, x, target, tw, training=False)
    e_out = max(P.rel_max(a, b) for a, b in zip(outs, o64))
    e_out32 = max(P.rel_max(a, b) for a, b in zip(o32, o64))
    msg = "%s eval %s B=2: heat-map max-rel vs fp64 ours %.2e fp32 oracle %.2e; loss rel %.2e" % (
        name, "x".join(map(str, CONFIGS[name][2:])), e_out, e_out32, abs(loss - l64) / abs(l64))
    assert len(outs) == len(o64)
    assert e_out < TOL, msg
    assert abs(loss - l64) < TOL * abs(l64), msg
    if g64 is None:
        print(msg)
        return
    rep = P.grad_report(ours, g32, g64, "%s eval" % name)
    errs, errs32 = _per_tensor(ours, g64), _per_tensor(g32, g64)
    worst_max = max(errs, key=lambda e: e[1])
    print("%s; gradient rel L2 ours %.3e fp32 oracle %.3e; worst tensor rel L2 ours %.2e (%s) fp32 oracle %.2e; worst "
          "max-rel ours %.2e (%s) fp32 oracle %.2e" % (msg, rep["l2_ours"], rep["l2_fp32"], errs[0][0], errs[0][2],
                                                       errs32[0][0], worst_max[1], worst_max[2], max(e[1] for e in errs32)))
    # One ReLU input within round-off of zero that falls the other way moves ONE entry of a tensor at a low resolution
    # (the innermost hourglass level is 4x3: 24 positions per channel) by a large share of it, and nothing else much.
    # At most one tensor may exceed the per-tensor bounds, and only by a single entry; the whole-gradient bound below
    # still holds for it. A wrong kernel moves many entries of many tensors.
    over = [e for e in errs if e[0] >= 2e-3 or e[1] >= 2e-2]
    assert len(over) <= 1, over[:8]
    for _, _, k in over:
        ref, o = g64[k].double().cpu().reshape(-1), ours[k].double().cpu().reshape(-1)
        d = (o - ref).abs()
        rest = torch.ones_like(d, dtype=torch.bool)
        rest[d.argmax()] = False
        e_rest = ((o - ref)[rest].norm() / ref.norm()).item(), (d[rest].max() / ref.abs().max()).item()
        print("%s: one entry off (%.2e of the tensor's maximum), the other %d within rel L2 %.2e, max-rel %.2e" % (
            k, (d.max() / ref.abs().max()).item(), d.numel() - 1, *e_rest))
        assert e_rest[0] < 2e-3 and e_rest[1] < 2e-2, (k, e_rest)
    assert rep["l2_ours"] <= 3 * rep["l2_fp32"] + 1e-5, (rep["l2_ours"], rep["l2_fp32"])


@pytest.mark.parametrize("name", list(CONFIGS))
def test_train_mode_as_good_as_fp32(name):
    """Batch statistics at B = 2: the statistical fp64-referenced criterion (tests/_parity.py)."""
    net, sd0, (x, target, tw), (o32, _, g32), (o64, l64, g64) = _reference(name, True)
    net.load_state_dict(sd0)
    outs, loss, ours = _engine(net, x, target, tw, training=True)
    e_vs32 = max(P.rel_max(a, b) for a, b in zip(outs, o32))
    e_out = max(P.rel_max(a, b) for a, b in zip(outs, o64))
    e_out32 = max(P.rel_max(a.cpu(), b) for a, b in zip(o32, o64))
    rep = P.assert_grads_as_good_as_fp32(ours, g32, g64, "%s train" % name)
    print("%s train: heat-map max-rel vs fp32 oracle %.2e, vs fp64 ours %.2e fp32 oracle %.2e; loss rel %.2e; gradient "
          "rel L2 ours %.3e fp32 oracle %.3e; per-tensor ratio median %.2f q90 %.2f worst %.2f" % (
              name, e_vs32, e_out, e_out32, abs(loss - l64) / abs(l64), rep["l2_ours"], rep["l2_fp32"],
              rep["median_ratio"], rep["q90_ratio"], rep["worst_ratio"]))
    assert e_vs32 < TOL or e_out < 3 * e_out32, (e_vs32, e_out, e_out32)
    assert abs(loss - l64) < TOL * abs(l64), (loss, l64)


# ------------------------------------------------------------------------------------------------ precisions
@pytest.mark.parametrize("name", ["hg_f256_s4", "hrnet_w32"])
def test_inference_precisions_against_oracle(name):
    """"fp16" and "fp16_act" eval forwards against the fp32 oracle, every output within 1e-2 max-relative. At 17 joints
    the hourglass's "fp16_act" forward switches to fp32 activations at the first score_ convolution (CUDA cores) and
    carries the fp32 residual stream through the later stacks. Tape-recording forwards stay at fp32 grade, and "fp32"
    gives back its own result bit for bit."""
    from fpd_b200.engine import set_inference_precision
    net, sd0, (x, _, _), (o32, _, _), _ = _reference(name, False)
    net.load_state_dict(sd0)
    net.eval()
    with torch.no_grad():
        base = [t.clone() for t in net.forward_nhwc(x, training=False)]
    tape32 = _last(net(x)).detach().clone()
    errs = {}
    try:
        for prec in ("fp16", "fp16_act"):
            set_inference_precision(net, prec)
            with torch.no_grad():
                got = net.forward_nhwc(x, training=False)
                got_net = _last(net(x))
            assert len(got) == len(o32) and all(g.dtype == torch.float32 for g in got)
            errs[prec] = [P.rel_max(g.permute(0, 3, 1, 2), r) for g, r in zip(got, o32)]
            assert P.rel_max(got_net, o32[-1]) <= 1e-2
        print("%s max-relative error per output vs the fp32 oracle: fp16 %s, fp16_act %s" % (
            name, ["%.2e" % e for e in errs["fp16"]], ["%.2e" % e for e in errs["fp16_act"]]))
        assert all(e <= 1e-2 for e in errs["fp16"] + errs["fp16_act"]), errs
        assert torch.equal(_last(net(x)).detach(), tape32)
    finally:
        set_inference_precision(net, "fp32")
    with torch.no_grad():
        again = net.forward_nhwc(x, training=False)
    assert all(torch.equal(a, b) for a, b in zip(again, base))


@pytest.mark.parametrize("name", ["hg_f256_s4", "hrnet_w32"])
def test_fp16_training_tape_eval_mode_against_fp64(name):
    """One tape-recording forward and backward at training precision "fp16", fixed BatchNorm statistics, against fp64:
    the bounds of test_train_f16_gpu.py::test_network_fp16_tape_against_fp64_oracle."""
    from fpd_b200.engine import set_training_precision
    net, sd0, (x, target, tw), (_, _, g32), (o64, _, g64) = _reference(name, False)
    net.load_state_dict(sd0)
    assert set_training_precision(net, "fp16") == "fp32"
    try:
        outs, _, ours = _engine(net, x, target, tw, training=False)
    finally:
        set_training_precision(net, "fp32")
    assert all(torch.isfinite(t).all() for t in outs) and all(torch.isfinite(v).all() for v in ours.values())
    herr = [P.rel_max(a, b) for a, b in zip(outs, o64)]
    rep = P.grad_report(ours, g32, g64, "fp16 training %s" % name)
    per_tensor = sorted(r[1] for r in rep["rows"])
    print("%s fp16 tape, eval mode: heat-map max-relative %s; gradient relative L2 %.3e (fp32 oracle %.3e), per-tensor "
          "error median %.3e q90 %.3e, median ratio to the fp32 oracle's %.1f" % (
              name, ["%.2e" % e for e in herr], rep["l2_ours"], rep["l2_fp32"], per_tensor[len(per_tensor) // 2],
              rep["q90_ours"], rep["median_ratio"]))
    assert max(herr) <= 1e-2, herr
    assert rep["l2_ours"] <= 2e-2, rep["l2_ours"]
    assert per_tensor[len(per_tensor) // 2] <= 2e-2
    assert rep["median_ratio"] <= 2.0 ** 13


# ------------------------------------------------------------------------------------------------ trained-like maps
def _flipped_targets(target, pairs):
    """Target of the mirrored image such that flip_back + shift-by-one lands on `target` again."""
    t = target.clone()
    t[:, :, :, :-1] = target[:, :, :, 1:]
    perm = list(range(t.shape[1]))
    for a, b in pairs:
        perm[a], perm[b] = b, a
    return t.flip(3)[:, perm].contiguous()


@pytest.fixture(scope="module")
def trained():
    """{name: (network over-fitted on one batch and its flip, the batch)}: heat-maps with one clear peak per joint, as a
    trained network's, made lazily (as test_infer_f16_gpu.py's key-point test does)."""
    made = {}

    def get(name):
        if name not in made:
            from bench import synthetic_batch
            from fpd_b200.train_step import FPDTrainStep
            net, _, _ = _build(name, 5, True)
            _, _, H, W = CONFIGS[name]
            B = 4 if CONFIGS[name][0] == "hourglass" else 2       # HRNet: fewer images to fit, peaks as clear
            x, target, _ = (t.cuda() for t in synthetic_batch(B, 77, H, W, J))
            tw = torch.ones(B, J, 1, device="cuda")
            xb = torch.cat([x, x.flip(3)]).contiguous()
            tb = torch.cat([target, _flipped_targets(target, COCO_FLIP_PAIRS)]).contiguous()
            wb = torch.cat([tw, tw]).contiguous()
            step = FPDTrainStep(net, None, lr=1e-3, use_graph=True)
            steps = int(os.environ.get("FPD_OVERFIT_STEPS", "1200"))
            if CONFIGS[name][0] == "hrnet":
                steps = steps * 5 // 2            # HRNet's peaks sharpen more slowly
            for i in range(steps):
                if i == steps * 2 // 3:
                    step.lr = 2.5e-4
                step.step(xb, tb, wb)
            torch.cuda.synchronize()
            del step
            net.eval()
            made[name] = (net, x, target)
        return made[name]
    yield get
    made.clear()


@pytest.mark.parametrize("name", ["hg_f256_s4", "hrnet_w32"])
def test_trained_like_keypoints_fp16_act_vs_fp16(trained, name):
    """The flip-test arg-max key points of "fp16_act" and "fp16" on trained-like heat-maps: the rule of the fp16 key-point
    test (99 % identical, every joint within one heat-map pixel)."""
    from fpd_b200.engine import set_inference_precision
    from fpd_b200.infer_step import FlipTestInference
    net, x, _ = trained(name)
    inf = FlipTestInference(net, COCO_FLIP_PAIRS, shift_heatmap=True)
    res = {}
    try:
        for prec in ("fp32", "fp16", "fp16_act"):
            set_inference_precision(net, prec)
            r = inf(x)
            res[prec] = (r["idx"].clone(), r["maxval"].clone())
    finally:
        set_inference_precision(net, "fp32")
    torch.cuda.synchronize()
    assert (res["fp32"][1] > 0.25).float().mean() > 0.9, "over-fit did not produce peaky heat-maps"
    w = CONFIGS[name][3] // 4
    (i16, m16), (ia, ma) = res["fp16"], res["fp16_act"]
    same = (ia == i16).float().mean().item()
    dx = (ia % w - i16 % w).abs().max().item()
    dy = (ia // w - i16 // w).abs().max().item()
    print("%s trained-like key points, fp16_act vs fp16: %.1f %% identical, max |dx| %d, |dy| %d, max |dmaxval| %.2e" % (
        name, 100 * same, dx, dy, (ma - m16).abs().max().item()))
    assert same >= 0.99
    assert dx <= 1 and dy <= 1


@pytest.mark.parametrize("name", ["hg_f256_s4", "hrnet_w32"])
def test_validation_graph_eager_and_oracle(trained, name):
    """FlipTestInference(decode=True) with the COCO flip pairs: the graph and the eager route bit for bit; the arg-max
    bit for bit against the oracle's flip test on trained-like heat-maps and the key points get_final_preds decodes
    from the oracle's merged maps equal, except where the oracle's own quarter-pixel nudge is within round-off of a tie."""
    from fpd_b200.infer_step import FlipTestInference
    from fpd_b200.lib.core.inference import get_final_preds, inverse_affines
    from oracle import decode_oracle as D
    import types
    net, x, target = trained(name)
    B, _, h, w = target.shape
    rng = np.random.RandomState(3)
    c, s = rng.uniform(100, 500, (B, 2)).astype(np.float32), rng.uniform(0.5, 3, (B, 2)).astype(np.float32)
    kw = dict(inv=inverse_affines(c, s, [w, h]), target=target, target_weight=torch.ones(B, J, 1, device="cuda"),
              post_process=True)
    graph = FlipTestInference(net, COCO_FLIP_PAIRS, decode=True)
    eager = FlipTestInference(net, COCO_FLIP_PAIRS, decode=True, use_graph=False)
    rg = {k: v.clone() for k, v in graph(x, **kw).items() if torch.is_tensor(v)}
    re_ = eager(x, **kw)
    torch.cuda.synchronize()
    for k in ("idx", "maxval", "avg_nhwc", "preds", "loss3", "pck"):
        assert torch.equal(rg[k], re_[k]), k
    # the oracle's flip test (function.py:218-240) and get_final_preds on its merged maps
    oracle, _ = _oracle_fn(name)
    sd = {k: v.detach().clone() for k, v in net.state_dict().items()}
    with torch.no_grad():
        a = oracle(sd, x, False)[-1].cpu().numpy()
        b = oracle(sd, x.flip(3).contiguous(), False)[-1].cpu().numpy()
    merged = D.flip_test_merge(a, b, COCO_FLIP_PAIRS, True)
    ref_idx = merged.reshape(B, J, -1).argmax(2)
    assert (merged.reshape(B, J, -1).max(2) > 0.25).mean() > 0.9
    assert np.array_equal(rg["idx"].cpu().numpy(), ref_idx), "arg-max differs for %d of %d joints" % (
        int((rg["idx"].cpu().numpy() != ref_idx).sum()), B * J)
    ref_p, ref_m = get_final_preds(types.SimpleNamespace(TEST=types.SimpleNamespace(POST_PROCESS=True)), merged, c, s)
    got = rg["preds"].cpu().numpy()
    # the merged maps agree to round-off, e; where the oracle's |hm[x+1] - hm[x-1]| (or along y) at the peak is within
    # 2e, the quarter-pixel nudge may go either way
    avg = rg["avg_nhwc"].permute(0, 3, 1, 2).cpu().numpy()
    e = np.abs(avg - merged).max()
    assert e <= TOL * np.abs(merged).max(), e
    tie = np.zeros((B, J), bool)
    for bb in range(B):
        for j in range(J):
            py, px = divmod(int(ref_idx[bb, j]), w)
            m = merged[bb, j]
            if 1 < px < w - 1:
                tie[bb, j] |= abs(m[py, px + 1] - m[py, px - 1]) <= 2 * e
            if 1 < py < h - 1:
                tie[bb, j] |= abs(m[py + 1, px] - m[py - 1, px]) <= 2 * e
    assert tie.mean() < 0.25, tie.sum()
    assert np.array_equal(got[..., :2][~tie], ref_p[~tie]), np.abs(got[..., :2] - ref_p).max()
    assert np.abs(got[..., 2] - ref_m[..., 0]).max() <= TOL * np.abs(ref_m).max()
    print("%s validation: graph == eager; key points equal to the oracle's at %d of %d joints (%d near-ties exempt)" % (
        name, int((~tie).sum()), B * J, int(tie.sum())))


# ------------------------------------------------------------------------------------------------ losses at 8 stacks
def _loss_reference(outs, target, teacher, tw, alpha, pose_topk, kd_topk):
    """fp64 closed form of the FPD loss (lib/core/function.py:127-134) with JointsMSELoss or JointsOHKMMSELoss(topk) per
    term (oracle/ohkm_oracle.py): (pose, kd, total, [d total / d out_s])."""
    from oracle import ohkm_oracle as OH
    if teacher is None:
        pose, grads = 0.0, []
        for o in outs:
            v, g = OH.criterion(o, target, tw, pose_topk)
            pose = pose + v
            grads.append(g)
        return pose, 0.0, pose, grads
    return OH.fpd(outs, target, teacher, tw, alpha, pose_topk, kd_topk)


@pytest.mark.parametrize("topk", [0, 8])
@pytest.mark.parametrize("teacher", [True, False])
@pytest.mark.parametrize("h,w", [(64, 48), (96, 72)])
def test_fpd_loss_eight_stacks_against_fp64(h, w, teacher, topk):
    """S = 8 (hg8), kMaxStacks of fpd_loss_fused and fpd_loss_ohkm_fused: the three losses within 1e-6 and every stack's
    gradient within 1e-5 max-relative of the fp64 closed form; gradient buffers poisoned with NaN first."""
    import fpd_b200  # noqa: F401
    from fpd_b200 import ops
    from oracle import ohkm_oracle as OH
    S, B, alpha = 8, 2, 0.5
    g = torch.Generator(device="cuda").manual_seed(h + w + 2 * teacher + topk)
    outs = [torch.randn(B, J, h, w, device="cuda", generator=g) for _ in range(S)]
    target = torch.rand(B, J, h, w, device="cuda", generator=g)
    t = torch.randn(B, J, h, w, device="cuda", generator=g) if teacher else None
    tw = (torch.rand(B, J, 1, device="cuda", generator=g) > 0.2).float() * (1 + torch.rand(B, J, 1, device="cuda",
                                                                                            generator=g))
    kd_topk = topk if teacher else 0
    if topk:       # the fp32 kernel and the fp64 reference must rank the same joints
        for s in range(S):
            for ref in ([target] + ([t] if teacher else [])):
                l = OH.per_joint(outs[s], ref, tw)[0]
                assert all(OH.boundary_ok(l[b].cpu(), topk) for b in range(B))
    pose, kd, total, grads_ref = _loss_reference(outs, target, t, tw, alpha, topk, kd_topk)
    nhwc = [o.permute(0, 2, 3, 1).contiguous() for o in outs]
    grads = [torch.full_like(o, float("nan")) for o in nhwc]
    losses = torch.full((3,), float("nan"), device="cuda")
    ops.fpd_loss(nhwc, target, t.permute(0, 2, 3, 1).contiguous() if teacher else None, tw, alpha, grads_out=grads,
                 losses_out=losses, pose_topk=topk, kd_topk=kd_topk)
    torch.cuda.synchronize()
    got = [float(v) for v in losses.cpu()]
    ref = [float(pose), float(kd), float(total)]
    e_loss = [abs(a - b) / abs(b) if b else abs(a) for a, b in zip(got, ref)]
    e_grad = [P.rel_max(gm.permute(0, 3, 1, 2), gr) for gm, gr in zip(grads, grads_ref)]
    print("fpd_loss S=8 %dx%d teacher=%s topk=%d: loss rel %s, gradient max-rel per stack %s" % (
        h, w, teacher, topk, ["%.1e" % e for e in e_loss], ["%.1e" % e for e in e_grad]))
    assert all(torch.isfinite(gm).all() for gm in grads), [bool(torch.isfinite(gm).all()) for gm in grads]
    assert max(e_loss) <= 1e-6, e_loss
    assert max(e_grad) <= 1e-5, e_grad


# ------------------------------------------------------------------------------------------------ the FPD step
def test_fpd_step_hg8_student_hg4_teacher():
    """fpd_coco/hourglass: an 8-stack 17-joint student, a frozen 4-stack teacher, 256x192. The captured graph's step
    equals the eager step bit for bit, and the student's heat-maps and the three losses match the fp32 oracle."""
    import fpd_b200  # noqa: F401
    from bench import cfg, synthetic_batch
    from fpd_b200 import ops
    from fpd_b200.lib.models import hourglass as HG
    from fpd_b200.train_step import FPDTrainStep
    from oracle import hourglass_oracle as O
    B = 4
    torch.manual_seed(0)
    student = HG.get_pose_net(cfg(256, 8, J), True)
    teacher = HG.get_pose_net(cfg(256, 4, J), False)
    s_sd0 = {k: v.detach().clone() for k, v in student.state_dict().items()}
    t_sd0 = {k: v.detach().clone() for k, v in teacher.state_dict().items()}
    x, target, tw = (t.cuda() for t in synthetic_batch(B, 1001, 256, 192, J))
    runs = {}
    for graph in (False, True):
        s = HG.get_pose_net(cfg(256, 8, J), True)
        s.load_state_dict(s_sd0)
        t = HG.get_pose_net(cfg(256, 4, J), False)
        t.load_state_dict(t_sd0)
        s.cuda()
        t.cuda()
        step = FPDTrainStep(s, t, alpha=0.5, lr=2.5e-4, use_graph=graph)
        losses = step.step(x, target, tw).clone()
        torch.cuda.synchronize()
        assert (step.graph is not None) == graph
        runs[graph] = (losses, [ops.nhwc_to_nchw(o) for o in step.last_outs],
                       torch.cat([p.detach().reshape(-1) for p in s.parameters()]),
                       {k: v.clone() for k, v in s.state_dict().items() if "running" in k})
        del step, s, t
    (l_e, o_e, w_e, r_e), (l_g, o_g, w_g, r_g) = runs[False], runs[True]
    assert torch.equal(l_e, l_g)
    assert all(torch.equal(a, b) for a, b in zip(o_e, o_g))
    assert torch.equal(w_e, w_g)
    assert all(torch.equal(r_e[k], r_g[k]) for k in r_e)
    # the reference algorithm (function.py:119-147) in fp32
    sd = {k: v.cuda() for k, v in s_sd0.items()}
    with torch.no_grad():
        outs = O.hourglass_net(sd, x, 8, training=True)
        tout = O.hourglass_net({k: v.cuda() for k, v in t_sd0.items()}, x, 4, training=False)[-1]
        total, pose, kd = O.fpd_loss(outs, target, tw, tout, 0.5)
    e_out = [P.rel_max(a, b) for a, b in zip(o_g, outs)]
    pose_g, kd_g, total_g = [float(v) for v in l_g.cpu()]
    e_loss = [abs(a - float(b)) / abs(float(b)) for a, b in ((pose_g, pose), (kd_g, kd), (total_g, total))]
    print("fpd step hg8 + hg4 teacher 256x192 B=%d: graph == eager; heat-map max-rel per stack %s; losses rel %s" % (
        B, ["%.1e" % e for e in e_out], ["%.1e" % e for e in e_loss]))
    assert len(o_g) == 8 and max(e_out) < TOL, e_out
    assert max(e_loss) < TOL, e_loss


# ------------------------------------------------------------------------------------------------ refusal
def test_hourglass_384x288_refused_on_the_device():
    """No hourglass runs 384x288 (12x9 max-pools to 6x4). net(x) and FlipTestInference raise before anything is
    launched or captured; the same model and the same FlipTestInference object then run 256x192 as fresh ones do."""
    import fpd_b200  # noqa: F401
    from bench import cfg
    from fpd_b200 import _native as N
    from fpd_b200.infer_step import FlipTestInference
    from fpd_b200.lib.models import hourglass as HG
    torch.manual_seed(2)
    net = _randomise_bn(HG.get_pose_net(cfg(64, 2, J), True)).cuda()
    g = torch.Generator(device="cuda").manual_seed(6)
    big = torch.randn(2, 3, 384, 288, device="cuda", generator=g)
    x = torch.randn(2, 3, 256, 192, device="cuda", generator=g)
    torch.cuda.synchronize()
    n0 = N.lib().fpd_launch_count()
    for training in (True, False):
        net.train(training)
        with pytest.raises(RuntimeError, match="384x288 input reaches hourglass level 1 at 12x9"):
            net(big)
    net.eval()
    inf = FlipTestInference(net, COCO_FLIP_PAIRS, use_graph=True)
    with pytest.raises(RuntimeError, match="384x288"):
        inf(big)
    assert N.lib().fpd_launch_count() == n0
    assert not net.engine()._branch_streams and inf.graph is None and not torch.cuda.is_current_stream_capturing()
    r = {k: v.clone() for k, v in inf(x).items() if torch.is_tensor(v)}
    fresh = FlipTestInference(net, COCO_FLIP_PAIRS, use_graph=True)(x)
    torch.cuda.synchronize()
    for k in ("idx", "maxval", "avg_nhwc"):
        assert torch.equal(r[k], fresh[k]), k
