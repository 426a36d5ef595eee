"""Gradient parity report on a GPU host: worst per-parameter relative error (max|d|/max|ref|) of the CUDA path's
parameter gradients vs the oracle in fp64, next to the oracle's own fp32-vs-fp64 noise floor."""
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
NS = types.SimpleNamespace


def rel(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-300)).item()


def oracle_grads(sd, x, target, tw, s, dtype, training=True):
    from oracle import hourglass_oracle as O
    sdd = {k: (v.to(dtype) if v.is_floating_point() else v.clone()) for k, v in sd.items()}
    params = {k: v.requires_grad_(True) for k, v in sdd.items() if v.is_floating_point() and "running" not in k}
    sdd.update(params)
    outs = O.hourglass_net(sdd, x.to(dtype), s, training=training)
    loss, _, _ = O.fpd_loss(outs, target.to(dtype), tw.to(dtype))
    loss.backward()
    return {k: p.grad for k, p in params.items()}, [o.detach() for o in outs]


def main():
    import fpd_b200  # noqa: F401
    from fpd_b200 import ops
    from fpd_b200.lib.models import hourglass as H
    from bench import synthetic_batch
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    for (f, s, B, hw, training) in [(64, 2, 2, 128, True), (64, 2, 2, 128, False), (128, 4, 4, 256, True),
                                    (128, 4, 4, 256, False)]:
        torch.manual_seed(0)
        cfg = NS(MODEL=NS(EXTRA=NS(NUM_FEATURES=f, NUM_STACKS=s, NUM_BLOCKS=1), NUM_JOINTS=16))
        net = H.get_pose_net(cfg, True).cuda()
        if not training:
            for m in net.modules():
                if isinstance(m, torch.nn.BatchNorm2d):
                    m.running_mean.normal_(0, 0.1)
                    m.running_var.uniform_(0.5, 1.5)
        net.train(training)
        x, target, tw = (v.cuda() for v in synthetic_batch(B, 0, hw, hw))
        sd = {k: v.clone() for k, v in net.state_dict().items()}
        g64, o64 = oracle_grads(sd, x, target, tw, s, torch.float64, training)
        g32, o32 = oracle_grads(sd, x, target, tw, s, torch.float32, training)
        eng = net.engine()
        ctx = eng.forward(x, training, record_tape=True)
        losses, grads = ops.fpd_loss([v.data for v in ctx.outs], target, None, tw.reshape(B, -1), 0.0)
        pg = eng.backward(ctx, grads)
        named = dict(net.named_parameters())
        rows = []
        gmax = max(g64[k].abs().max().item() for k in named)
        for k, p in named.items():
            if g64[k].abs().max().item() < 1e-9 * gmax:
                continue  # structurally zero gradients (conv bias in front of a train-mode BN): nothing to compare
            mine = pg[p].reshape(p.shape)
            rows.append((rel(mine, g64[k]), rel(g32[k], g64[k]), k))
        rows.sort(reverse=True)
        def flat(d):
            return torch.cat([d[k].double().flatten() for k in named])
        mine_flat = torch.cat([pg[p].double().flatten() for p in named.values()])
        r64 = flat(g64)
        print("cfg f=%d s=%d B=%d hw=%d train=%s: global rel L2 err ours %.3e, torch fp32 %.3e" % (
            f, s, B, hw, training, ((mine_flat - r64).norm() / r64.norm()).item(),
            ((flat(g32) - r64).norm() / r64.norm()).item()))
        print("   worst per-parameter max-rel err  ours-vs-fp64 | torch-fp32-vs-fp64")
        for a, b, k in rows[:8]:
            print("   %.3e | %.3e  %s" % (a, b, k))
        worst32 = max(r[1] for r in rows)
        print("   max over params: ours %.3e, torch fp32 %.3e; outputs ours-vs-fp64 %s" % (
            rows[0][0], worst32, ["%.2e" % rel(ops.nhwc_to_nchw(v.data), o) for v, o in zip(ctx.outs, o64)]), flush=True)


if __name__ == "__main__":
    main()
