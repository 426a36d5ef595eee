"""GPU parity of the drop-in hourglass (engine + libfpd_b200 kernels) against (a) the golden vectors produced
by the real reference and (b) the oracle restatement run in fp32 on the same inputs. Tolerance: the north-star
bar, max|delta| / max|ref| <= 1e-3 on every output tensor and loss scalar (3xTF32 mode)."""
import os
import types

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
NS = types.SimpleNamespace
TOL = 1e-3


def _load(name):
    z = np.load(os.path.join(GOLD, name), allow_pickle=False)
    return {k: z[k] for k in z.files}


def _sd(gold, prefix="sd/"):
    return {k[len(prefix):]: torch.from_numpy(v.copy()) for k, v in gold.items() if k.startswith(prefix)}


def _rel(a, b):
    a = torch.as_tensor(a).double().cpu()
    b = torch.as_tensor(b).double().cpu()
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()


def _cfg(f, s, j=16):
    return NS(MODEL=NS(EXTRA=NS(NUM_FEATURES=f, NUM_STACKS=s, NUM_BLOCKS=1), NUM_JOINTS=j))


def _net(f, s, sd=None):
    import fpd_b200  # noqa: F401
    from fpd_b200.lib.models import hourglass as H
    net = H.get_pose_net(_cfg(f, s), is_train=True)
    if sd is not None:
        net.load_state_dict(sd, strict=True)
    return net.cuda()


@pytest.fixture(scope="module", autouse=True)
def _fp32_reference_mode():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield


def test_train_forward_backward_matches_reference_golden():
    from fpd_b200.lib.core.loss import JointsMSELoss
    g = _load("hg_s2f64_train.npz")
    net = _net(64, 2, _sd(g))
    net.train()
    x = torch.from_numpy(g["x"]).cuda()
    outs = net(x)
    assert isinstance(outs, list) and len(outs) == 2
    for i, o in enumerate(outs):
        assert tuple(o.shape) == g["out%d" % i].shape
        assert _rel(o.detach(), g["out%d" % i]) < TOL, "stack %d" % i
    crit = JointsMSELoss(use_target_weight=True)
    target = torch.from_numpy(g["target"]).cuda()
    tw = torch.from_numpy(g["target_weight"]).cuda()
    loss = crit(outs[0], target, tw)
    for o in outs[1:]:
        loss += crit(o, target, tw)
    assert abs(loss.item() - float(g["loss"])) < TOL * abs(float(g["loss"]))
    loss.backward()
    # Train-mode gradients of this network are ill-conditioned at the default init: the reference's own fp32
    # gradients differ from an fp64 evaluation by up to 5e-2 per tensor (tools/diag_grad.py), so the
    # whole-gradient relative L2 error is the meaningful check here; exact backward arithmetic is pinned per op in
    # test_ops_gpu.py and at network level in eval mode below.
    num = den = 0.0
    for k, p in net.named_parameters():
        assert p.grad is not None, k
        ref = torch.from_numpy(g["grad/" + k]).double()
        num += float((p.grad.double().cpu() - ref).pow(2).sum())
        den += float(ref.pow(2).sum())
    assert (num / den) ** 0.5 < 5e-2, (num / den) ** 0.5
    sd1 = net.state_dict()
    assert _rel(sd1["bn1.running_mean"], g["after/bn1.running_mean"]) < 1e-4
    assert _rel(sd1["bn1.running_var"], g["after/bn1.running_var"]) < 1e-4
    assert _rel(sd1["fc.1.1.running_var"], g["after/fc.1.1.running_var"]) < 1e-3
    assert int(sd1["bn1.num_batches_tracked"]) == int(g["after/bn1.num_batches_tracked"])


def test_fpd_step_matches_reference_golden():
    from fpd_b200 import ops
    g, f = _load("hg_s2f64_train.npz"), _load("hg_fpd.npz")
    net = _net(64, 2, _sd(g))
    tnet = _net(64, 1, _sd(f, "tsd/"))
    net.train()
    tnet.eval()
    x = torch.from_numpy(g["x"]).cuda()
    with torch.no_grad():
        t_nhwc = tnet.forward_nhwc(x)[-1]
        tout = tnet(x)[-1]
    assert _rel(tout, f["teacher_out"]) < TOL
    assert _rel(ops.nhwc_to_nchw(t_nhwc), f["teacher_out"]) < TOL
    # fused FPD loss on the engine's NHWC heat-maps + explicit backward
    eng = net.engine()
    ctx = eng.forward(x, True, record_tape=True)
    losses, grads = ops.fpd_loss([v.data for v in ctx.outs], torch.from_numpy(g["target"]).cuda(), t_nhwc,
                                 torch.from_numpy(g["target_weight"]).cuda(), float(f["alpha"]))
    pose, kd, total = [float(v) for v in losses.cpu()]
    assert abs(pose - float(f["pose"])) < TOL * abs(float(f["pose"]))
    assert abs(kd - float(f["kd"])) < TOL * abs(float(f["kd"]))
    assert abs(total - float(f["loss"])) < TOL * abs(float(f["loss"]))
    pg = eng.backward(ctx, grads)
    named = dict(net.named_parameters())
    norms = dict(zip(f["grad_names"].tolist(), f["grad_norms"].tolist()))
    tot_ref = sum(v * v for v in norms.values()) ** 0.5
    tot = sum(pg[p].double().norm().item() ** 2 for p in named.values()) ** 0.5
    assert abs(tot - tot_ref) < 5e-2 * tot_ref, (tot, tot_ref)   # see the conditioning note in the test above
    num = den = 0.0
    for k in [k[5:] for k in f if k.startswith("grad/")]:
        ref = torch.from_numpy(f["grad/" + k]).double()
        num += float((pg[named[k]].reshape(named[k].shape).double().cpu() - ref).pow(2).sum())
        den += float(ref.pow(2).sum())
    assert (num / den) ** 0.5 < 5e-2


def test_eval_mode_backward_matches_oracle():
    """Well-conditioned backward check (fixed BN statistics): every parameter gradient of the engine's tape against the
    oracle's autograd in fp32 on the same device, max|delta|/max|ref| per tensor."""
    from fpd_b200 import ops
    from oracle import hourglass_oracle as O
    torch.manual_seed(2)
    net = _net(64, 2)
    for m in net.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.running_mean.normal_(0, 0.1)
            m.running_var.uniform_(0.5, 1.5)
            m.weight.data.uniform_(0.5, 1.5)
            m.bias.data.normal_(0, 0.1)
    net.eval()
    B = 2
    x = torch.randn(B, 3, 128, 128, device="cuda")
    target = torch.rand(B, 16, 32, 32, device="cuda")
    tw = torch.rand(B, 16, 1, device="cuda")
    sd = {k: v.detach().clone() for k, v in net.state_dict().items()}
    params = {k: v.requires_grad_(True) for k, v in sd.items() if v.is_floating_point() and "running" not in k}
    sd.update(params)
    outs = O.hourglass_net(sd, x, num_stacks=2, training=False)
    loss, _, _ = O.fpd_loss(outs, target, tw)
    loss.backward()
    eng = net.engine()
    ctx = eng.forward(x, False, record_tape=True)
    losses, grads = ops.fpd_loss([v.data for v in ctx.outs], target, None, tw.reshape(B, -1), 0.0)
    assert abs(losses[2].item() - loss.item()) < 1e-4 * abs(loss.item())
    pg = eng.backward(ctx, grads)
    worst, name = 0.0, None
    for k, p in net.named_parameters():
        e = _rel(pg[p].reshape(p.shape), params[k].grad)
        if e > worst:
            worst, name = e, k
    assert worst < 2e-3, (worst, name)


@pytest.mark.parametrize("f,s,B,hw,training", [(128, 4, 2, 256, True), (256, 2, 1, 256, False), (64, 1, 2, 256, True)])
def test_forward_matches_oracle_at_baseline_shapes(f, s, B, hw, training):
    """BASELINE configs' channel widths / resolutions (student f=128 s=4, teacher-width f=256, cfg-1 f=64 s=1)
    against the oracle run with torch fp32 (TF32 off) on the same device and weights."""
    from oracle import hourglass_oracle as O
    torch.manual_seed(0)
    net = _net(f, s)
    net.train(training)
    x = torch.randn(B, 3, hw, hw, device="cuda")
    sd = {k: v.clone() for k, v in net.state_dict().items()}
    with torch.no_grad():
        ref = O.hourglass_net(sd, x, num_stacks=s, training=training)
        got = net(x)
    for i, (a, b) in enumerate(zip(got, ref)):
        assert _rel(a, b) < TOL, "stack %d rel %.3e" % (i, _rel(a, b))
    if training:
        after = net.state_dict()
        assert _rel(after["bn1.running_var"], sd["bn1.running_var"]) < 1e-4


def test_eval_mode_and_precision_modes():
    from oracle import hourglass_oracle as O
    torch.manual_seed(1)
    net = _net(64, 1)
    for m in net.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.running_mean.normal_(0, 0.1)
            m.running_var.uniform_(0.5, 1.5)
    net.eval()
    x = torch.randn(2, 3, 128, 128, device="cuda")
    sd = {k: v.clone() for k, v in net.state_dict().items()}
    with torch.no_grad():
        ref = O.hourglass_net(sd, x, num_stacks=1, training=False)[0]
        got = net(x)[0]
        assert _rel(got, ref) < 1e-4
        os.environ["FPD_PRECISION"] = "tf32"
        try:
            got1 = net(x)[0]
        finally:
            del os.environ["FPD_PRECISION"]
        assert _rel(got1, ref) < 2e-2   # single-pass TF32: documented as outside the parity bar


def test_flip_test_inference_pipeline_matches_oracle():
    """BASELINE configs[4] path (function.validate, function.py:212-240 + inference.get_max_preds): forward, forward on the
    W-flipped input, flip_back + 1-px shift + average, arg-max -- all on the device -- against the oracle restatement."""
    from fpd_b200 import ops
    from oracle import decode_oracle as D
    from oracle import hourglass_oracle as O
    torch.manual_seed(3)
    net = _net(128, 4)
    for m in net.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.running_mean.normal_(0, 0.1)
            m.running_var.uniform_(0.5, 1.5)
    net.eval()
    B = 4
    x = torch.randn(B, 3, 256, 256, device="cuda")
    sd = {k: v.clone() for k, v in net.state_dict().items()}
    with torch.no_grad():
        ref = O.hourglass_net(sd, x, 4, training=False)[-1].cpu().numpy()
        ref_f = O.hourglass_net(sd, x.flip(3), 4, training=False)[-1].cpu().numpy()
        hm = net.forward_nhwc(x, training=False)[-1]
        hm_f = net.forward_nhwc(x.flip(3).contiguous(), training=False)[-1]
    perm = list(range(16))
    for a, b in D.MPII_FLIP_PAIRS:
        perm[a], perm[b] = b, a
    avg, idx, maxval = ops.flip_merge_argmax(hm, hm_f, torch.tensor(perm, dtype=torch.int32, device="cuda"), shift=True)
    merged_ref = D.flip_test_merge(ref, ref_f, D.MPII_FLIP_PAIRS, True)
    preds_ref, max_ref = D.get_max_preds(merged_ref)
    got = ops.nhwc_to_nchw(avg).cpu().numpy()
    assert np.abs(got - merged_ref).max() <= TOL * np.abs(merged_ref).max()
    # arg-max of OUR merged map is bit-exact w.r.t. numpy on the same map ...
    idx_np = got.reshape(B, 16, -1).argmax(2)
    assert np.array_equal(idx.cpu().numpy(), idx_np)
    # ... and agrees with the oracle's key points wherever the top-2 margin exceeds the parity tolerance
    flat = merged_ref.reshape(B, 16, -1)
    top2 = np.sort(flat, axis=2)[:, :, -2:]
    clear = (top2[:, :, 1] - top2[:, :, 0]) > 2 * TOL * np.abs(merged_ref).max()
    ref_idx = flat.argmax(2)
    assert np.array_equal(idx.cpu().numpy()[clear], ref_idx[clear])
    assert clear.mean() > 0.5
    assert np.abs(maxval.cpu().numpy() - max_ref[..., 0]).max() <= TOL * np.abs(max_ref).max()


def test_graph_pipelined_train_step_equals_eager_steps():
    """FPDTrainStep as a CUDA graph with the teacher on a second stream, software-pipelined one batch ahead, must produce
    the same losses and weights as plain eager steps (teacher and student on one stream, no graph)."""
    import sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from bench import synthetic_batch
    from fpd_b200.train_step import FPDTrainStep
    torch.manual_seed(11)
    init_s = {k: v.clone() for k, v in _net(64, 2).state_dict().items()}
    init_t = {k: v.clone() for k, v in _net(64, 1).state_dict().items()}
    batches = [tuple(t.cuda() for t in synthetic_batch(2, 50 + i, 128, 128)) for i in range(3)]

    os.environ["FPD_PIPELINE_TEACHER"] = "1"

    def run(use_graph):
        s, t = _net(64, 2, init_s), _net(64, 1, init_t)
        st = FPDTrainStep(s, t, alpha=0.5, lr=1e-3, use_graph=use_graph)
        assert st.pipeline == use_graph
        losses = []
        for i, (x, tg, tw) in enumerate(batches):
            nxt = batches[i + 1][0] if (use_graph and i + 1 < len(batches)) else None
            losses.append(st.step(x, tg, tw, next_x=nxt).clone())
        torch.cuda.synchronize()
        return torch.stack(losses).cpu(), st.flat.flat.clone().cpu(), {k: v.clone().cpu() for k, v in s.state_dict().items()}

    try:
        l_e, w_e, sd_e = run(False)
        l_g, w_g, sd_g = run(True)
    finally:
        del os.environ["FPD_PIPELINE_TEACHER"]
    assert torch.allclose(l_e, l_g, rtol=1e-5, atol=0), (l_e, l_g)
    assert _rel(w_g, w_e) < 1e-5
    assert _rel(sd_g["bn1.running_var"], sd_e["bn1.running_var"]) < 1e-6
    assert int(sd_g["bn1.num_batches_tracked"]) == int(sd_e["bn1.num_batches_tracked"]) == 3
