"""HRNet-w32 / -w48 gradients at 256x192 against the fp64 oracle, and the `hrnet_fpd` training step that bench.py measures.

The golden HRNet (tests/golden/hrnet_small.npz: branches of 8..64 channels at 128x96) never reaches the backward routes
of the real widths. tests/test_hrnet_routes_cpu.py checks that one step at 2x3x256x192 still takes them:
  * chunked tensor-core weight gradients (ops.conv2d_wgrad_tc_chunked): w32's 256-channel 3x3s at 8x6 in Cin-128
    chunks, w48's 384-channel 3x3s in 128x128 chunks and its 192- / 96-channel 3x3s in 64- / 32-wide chunks;
  * CUDA-core weight gradients (w48): every branch-0 3x3 (48 -> 48 at 64x48, stride 1), and the stride-2 chains out of
    branch 0, which run forward at stride 1 and hand the compact dY to the weight gradient (Engine._conv_at);
  * w48's 384-channel convolutions on the staged 3-pass kernel, three 128-column output slices, forward and data
    gradient;
  * dY's operand scale from the BatchNorm-backward pass (HRNet's convolutions have no bias) at these channel counts.

Every check compares with the oracle (oracle/hrnet_oracle.py) run by autograd in fp32 and fp64 on the same device:
  * eval mode, fixed BatchNorm statistics: a well-conditioned problem, so every parameter gradient is bounded per tensor;
  * train mode: the fp64-referenced statistical criterion of tests/_parity.py. At B = 2 the fp32 oracle's own gradient
    is ~1.5e-2 (relative L2) from fp64, so a per-tensor bound would measure round-off, not the kernels;
  * the hrnet_fpd step (w32 student, frozen w48 teacher, FPDTrainStep with its CUDA graph) at the bench batch,
    FPD_PARITY_HR_B (default 24): heat-maps, losses, running statistics, gradients and the Adam update.
"""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import _parity as P   # noqa: E402

pytestmark = pytest.mark.gpu
TOL = 1e-3
B_HR = int(os.environ.get("FPD_PARITY_HR_B", "24"))


@pytest.fixture(scope="module", autouse=True)
def _fp32_reference_mode():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    det = torch.backends.cudnn.deterministic
    torch.backends.cudnn.deterministic = True
    yield
    torch.backends.cudnn.deterministic = det


def _hrnet(width, seed):
    import fpd_b200  # noqa: F401
    from bench import hrnet_cfg
    from fpd_b200.lib.models import pose_hrnet as H
    torch.manual_seed(seed)
    return H.get_pose_net(hrnet_cfg(width), False)


def _randomise_bn(net):
    """Running statistics and affine parameters away from their defaults (as test_hourglass_gpu's eval-mode backward):
    with mean 0, variance 1, weight 1 and bias 0 an eval-mode BatchNorm is the identity."""
    for m in net.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.running_mean.normal_(0, 0.1)
            m.running_var.uniform_(0.5, 1.5)
            m.weight.data.uniform_(0.5, 1.5)
            m.bias.data.normal_(0, 0.1)
    return net


def _inputs(B, seed, device):
    """N(0,1) image, uniform target and 0/1 joint weights, drawn on the host (the same values on any device)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 3, 256, 192, generator=g)
    target = torch.rand(B, 17, 64, 48, generator=g)
    tw = (torch.rand(B, 17, 1, generator=g) > 0.2).float()
    return x.to(device), target.to(device), tw.to(device)


def _oracle(sd0, x, target, tw, training, dtype):
    """-> (heat-map, loss, {name: gradient}) of the oracle in `dtype`, by autograd."""
    from oracle import hourglass_oracle as O
    from oracle import hrnet_oracle as HO
    sd = HO.annotate_strides(P.cast_sd(sd0, dtype))
    params = P.with_grad(sd)
    out = HO.hrnet(sd, x.to(dtype), training=training)
    loss, _, _ = O.fpd_loss([out], target.to(dtype), tw.to(dtype))
    loss.backward()
    return out.detach(), loss.item(), {k: p.grad.detach() for k, p in params.items()}


def _engine(net, x, target, tw, training):
    """-> (heat-map NCHW, loss, {name: gradient}) of the engine's tape-recording forward and its backward."""
    from fpd_b200 import ops
    eng = net.engine()
    ctx = eng.forward(x, training, record_tape=True)
    out = ops.nhwc_to_nchw(ctx.outs[0].data)
    losses, grads = ops.fpd_loss([v.data for v in ctx.outs], target, None, tw, 0.0)
    pg = eng.backward(ctx, grads)
    torch.cuda.synchronize()
    return out, float(losses[2]), {k: pg[p] for k, p in net.named_parameters()}


def _per_tensor(grads, g64):
    """-> [(relative L2 error, max-relative error, name)] of every tensor against fp64, worst L2 first."""
    errs = []
    for k, ref in g64.items():
        ref = ref.double().cpu()
        o = grads[k].reshape(ref.shape).double().cpu()
        errs.append((((o - ref).norm() / ref.norm().clamp_min(1e-300)).item(), P.rel_max(o, ref), k))
    return sorted(errs, reverse=True)


@pytest.mark.parametrize("width", [32, 48])
def test_eval_mode_backward_per_tensor_against_fp64(width):
    """Fixed BatchNorm statistics: every data- and weight-gradient kernel on the tape, per parameter tensor, against
    fp64. Relative L2 per tensor (a kernel that is off shows there) and max-relative per tensor (looser: one ReLU input
    within round-off of zero that falls the other way moves single entries of the low-resolution branches)."""
    net = _randomise_bn(_hrnet(width, seed=width)).cuda().eval()
    x, target, tw = _inputs(2, 100 + width, "cuda")
    sd0 = {k: v.detach().clone() for k, v in net.state_dict().items()}
    out, loss, ours = _engine(net, x, target, tw, training=False)
    o32, _, g32 = _oracle(sd0, x, target, tw, False, torch.float32)
    o64, l64, g64 = _oracle(sd0, x, target, tw, False, torch.float64)
    rep = P.grad_report(ours, g32, g64, "hrnet w%d eval 256x192 B=2" % width)
    errs = _per_tensor(ours, g64)
    errs32 = _per_tensor(g32, g64)
    worst_max = max(errs, key=lambda e: e[1])
    print("hrnet w%d eval: heat-map max-rel vs fp64 ours %.2e fp32 oracle %.2e; loss rel %.2e; gradient rel L2 ours "
          "%.3e fp32 oracle %.3e; worst tensor rel L2 ours %.2e (%s) fp32 oracle %.2e; worst max-rel ours %.2e (%s) fp32 "
          "oracle %.2e; per-tensor ratio median %.2f worst %.2f" % (
              width, P.rel_max(out, o64), P.rel_max(o32, o64), abs(loss - l64) / abs(l64), rep["l2_ours"], rep["l2_fp32"],
              errs[0][0], errs[0][2], errs32[0][0], worst_max[1], worst_max[2], max(e[1] for e in errs32),
              rep["median_ratio"], rep["worst_ratio"]))
    assert P.rel_max(out, o64) < TOL, "heat-map: %.3e" % P.rel_max(out, o64)
    assert abs(loss - l64) < TOL * abs(l64), (loss, l64)
    assert errs[0][0] < 2e-3, errs[:8]
    assert worst_max[1] < 2e-2, sorted(errs, key=lambda e: -e[1])[:8]
    assert rep["l2_ours"] <= 3 * rep["l2_fp32"] + 1e-5, (rep["l2_ours"], rep["l2_fp32"])


@pytest.mark.parametrize("width", [32, 48])
def test_train_mode_backward_as_good_as_fp32(width):
    """Batch statistics at B = 2: the statistical fp64-referenced criterion (tests/_parity.py), not a per-tensor bound."""
    net = _hrnet(width, seed=width).cuda().train()
    x, target, tw = _inputs(2, 200 + width, "cuda")
    sd0 = {k: v.detach().clone() for k, v in net.state_dict().items()}
    out, loss, ours = _engine(net, x, target, tw, training=True)
    o32, _, g32 = _oracle(sd0, x, target, tw, True, torch.float32)
    o64, l64, g64 = _oracle(sd0, x, target, tw, True, torch.float64)
    e_out, e_out32 = P.rel_max(out, o64), P.rel_max(o32, o64)
    rep = P.assert_grads_as_good_as_fp32(ours, g32, g64, "hrnet w%d train 256x192 B=2" % width)
    print("hrnet w%d train: heat-map max-rel vs fp64 ours %.2e fp32 oracle %.2e (ours vs fp32 %.2e); loss rel %.2e; "
          "gradient rel L2 ours %.3e fp32 oracle %.3e; per-tensor ratio median %.2f q90 %.2f worst %.2f" % (
              width, e_out, e_out32, P.rel_max(out, o32), abs(loss - l64) / abs(l64), rep["l2_ours"], rep["l2_fp32"],
              rep["median_ratio"], rep["q90_ratio"], rep["worst_ratio"]))
    # the forward: within the parity bar of the fp32 oracle, or as close to fp64 as 3x the fp32 oracle gets
    assert P.rel_max(out, o32) < TOL or e_out < 3 * e_out32, (P.rel_max(out, o32), e_out, e_out32)
    assert abs(loss - l64) < TOL * abs(l64), (loss, l64)


def _oracle_fpd(s_sd, t_sd, x, target, tw, dtype, alpha=0.5):
    """function.py:119-147 (fpd_train) on the HRNet oracle in `dtype`: student heat-map, teacher heat-map,
    (total, pose, kd), {name: gradient}, the student's state after the forward (running statistics updated), and its
    parameters."""
    from oracle import hourglass_oracle as O
    from oracle import hrnet_oracle as HO
    sd = HO.annotate_strides(P.cast_sd(s_sd, dtype))
    params = P.with_grad(sd)
    xx = x.to(dtype)
    out = HO.hrnet(sd, xx, training=True)
    with torch.no_grad():
        tout = HO.hrnet(HO.annotate_strides(P.cast_sd(t_sd, dtype)), xx, training=False)
    total, pose, kd = O.fpd_loss([out], target.to(dtype), tw.to(dtype), tout, alpha)
    total.backward()
    grads = {k: p.grad.detach() for k, p in params.items()}
    return out.detach(), tout, (total.item(), pose.item(), kd.item()), grads, sd, params


def test_hrnet_fpd_bench_step_matches_oracle():
    """bench.py's hrnet_fpd: the models build_models makes, FPDTrainStep with its CUDA graph, one captured step."""
    import fpd_b200  # noqa: F401
    from bench import CONFIGS, build_models, synthetic_batch
    from fpd_b200 import ops
    from fpd_b200.train_step import FPDTrainStep
    c = CONFIGS["hrnet_fpd"]
    assert (c["student"], c["teacher"], c["H"], c["W"], c["J"]) == (32, 48, 256, 192, 17)
    lr = c["lr"]
    # ---- exactly what bench.run_b200 builds
    student, teacher = build_models("hrnet_fpd", torch.device("cuda"))
    s_sd0 = {k: v.detach().clone() for k, v in student.state_dict().items()}
    t_sd0 = {k: v.detach().clone() for k, v in teacher.state_dict().items()}
    step = FPDTrainStep(student, teacher, alpha=0.5, lr=lr, use_graph=True)
    assert step.use_graph and step.overlap_teacher and step._wstream is not None and not step.pipeline
    x, target, tw = (t.cuda() for t in synthetic_batch(B_HR, 1000, c["H"], c["W"], c["J"]))
    losses = step.step(x, target, tw).clone()          # capture + ONE replayed update
    torch.cuda.synchronize()
    assert step.graph is not None
    names = [k for k, _ in student.named_parameters()]
    got_out = ops.nhwc_to_nchw(step.last_outs[0])
    got_teacher = ops.nhwc_to_nchw(step.last_teacher)
    got_grads = {k: g.clone() for k, g in zip(names, step.flat.grad_views)}
    got_w = {k: p.detach().clone() for k, p in student.named_parameters()}
    got_sd = {k: v.detach().clone() for k, v in student.state_dict().items()}
    del step
    torch.cuda.empty_cache()

    # ---- the reference algorithm in fp32 (the parity bar) and fp64 (the yardstick for the gradients)
    o32, t32, l32, g32, sd32, p32 = _oracle_fpd(s_sd0, t_sd0, x, target, tw, torch.float32)
    e_out, e_teacher = P.rel_max(got_out, o32), P.rel_max(got_teacher, t32)
    pose, kd, total = [float(v) for v in losses.cpu()]
    e_loss = [abs(a - b) / abs(b) for a, b in ((total, l32[0]), (pose, l32[1]), (kd, l32[2]))]
    assert e_out < TOL, "student heat-map: %.3e" % e_out
    assert e_teacher < TOL, "teacher heat-map: %.3e" % e_teacher
    assert max(e_loss) < TOL, e_loss
    # a fuse-layer BN (last unit of a down path), a branch-3 BN, an up-path BN of the last module and the stem's bn1
    for k in ("bn1.running_mean", "bn1.running_var", "stage3.3.fuse_layers.2.0.1.1.running_mean",
              "stage3.3.fuse_layers.2.0.1.1.running_var", "stage4.2.branches.3.3.bn2.running_mean",
              "stage4.2.branches.3.3.bn2.running_var", "stage4.2.fuse_layers.0.3.1.running_var"):
        assert P.rel_max(got_sd[k], sd32[k]) < TOL, (k, P.rel_max(got_sd[k], sd32[k]))
    assert all(int(v) == 1 for k, v in got_sd.items() if k.endswith("num_batches_tracked"))
    # torch.optim.Adam on the oracle's autograd gradients. The first step moves each weight by lr * g / (|g| + eps), at
    # most lr: where round-off decides the sign of g the two updates differ by up to 2 lr, so the weights are bounded
    # by that, and the updates themselves are compared fp64-referenced below
    opt = torch.optim.Adam(list(p32.values()), lr=lr)
    w_before = {k: v.detach().clone() for k, v in p32.items()}
    opt.step()
    flat_got = torch.cat([got_w[k].reshape(-1) for k in names])
    flat_ref = torch.cat([p32[k].detach().reshape(-1) for k in names])
    assert (flat_got - flat_ref).abs().max().item() <= 2 * lr * (1 + 1e-3)
    del o32, t32, sd32
    torch.cuda.empty_cache()
    o64, t64, l64, g64, _, p64 = _oracle_fpd(s_sd0, t_sd0, x, target, tw, torch.float64)
    rep = P.assert_grads_as_good_as_fp32(got_grads, g32, g64, "bench-config hrnet w32+w48 B=%d" % B_HR)
    # the updates, fp64-referenced like the gradients: the update is a monotone function of each gradient entry, so its
    # error follows the gradient's and gets the gradient's bound
    opt64 = torch.optim.Adam(list(p64.values()), lr=lr)
    w64_before = {k: v.detach().clone() for k, v in p64.items()}
    opt64.step()
    d_got = torch.cat([(got_w[k].double() - s_sd0[k].double()).reshape(-1) for k in names]).cpu()
    d_32 = torch.cat([(p32[k].detach().double() - w_before[k].double()).reshape(-1) for k in names]).cpu()
    d_64 = torch.cat([(p64[k].detach() - w64_before[k]).reshape(-1) for k in names]).cpu()
    e_got = ((d_got - d_64).norm() / d_64.norm()).item()
    e_32 = ((d_32 - d_64).norm() / d_64.norm()).item()
    print("hrnet_fpd step B=%d: heat-map max-rel vs fp32 oracle student %.2e teacher %.2e (vs fp64 %.2e / %.2e); loss "
          "rel total %.2e pose %.2e kd %.2e (total vs fp64 %.2e); gradient rel L2 ours %.3e fp32 oracle %.3e, per-tensor "
          "ratio median %.2f worst %.2f; Adam update rel L2 ours %.3e fp32 oracle %.3e" % (
              B_HR, e_out, e_teacher, P.rel_max(got_out, o64), P.rel_max(got_teacher, t64), e_loss[0], e_loss[1],
              e_loss[2], abs(total - l64[0]) / abs(l64[0]), rep["l2_ours"], rep["l2_fp32"], rep["median_ratio"],
              rep["worst_ratio"], e_got, e_32))
    assert e_got <= P.K_L2 * e_32 + 1e-4, (e_got, e_32)
    assert abs(total - l64[0]) < TOL * abs(l64[0])
