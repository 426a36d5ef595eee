"""Drop-in for the reference's lib/core/loss.py: `JointsMSELoss(use_target_weight)` and
`JointsOHKMMSELoss(use_target_weight, topk=8)`, called as `(output, target, target_weight) -> 0-dim tensor` supporting
.backward(), `+=`, .item() (as lib/core/function.py:127-152 uses them). One fused CUDA pass (value + gradient)
replaces the reference's per-joint Python loop of nn.MSELoss calls (loss.py:24-39); the online hard keypoint mining
loss (loss.py:42-87) replaces its per-joint and per-sample loops (torch.topk + gather per sample) with three kernels:
per-joint sums, one warp per sample ranking the joints, and the gradient.

Differences from the reference's JointsOHKMMSELoss: joints are ranked by their fp32 loss with the lower joint index
first on exact ties (torch.topk leaves the order of ties open), and a batch of one sample works (the reference's
squeeze() breaks it). topk < 1 or topk > J raises ValueError, as torch.topk raises there; J is limited to 64."""
import torch
import torch.nn as nn


class _JointsMSEFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, output, target, target_weight):
        from fpd_b200 import ops
        out = output.contiguous().float()
        loss3, grad = ops.joints_mse(out, target.contiguous().float(),
                                     None if target_weight is None else target_weight.float(),
                                     want_grad=output.requires_grad)
        ctx.save_for_backward(grad)
        return loss3[0].clone()

    @staticmethod
    def backward(ctx, g):
        (grad,) = ctx.saved_tensors
        return (None if grad is None else grad * g), None, None


class JointsMSELoss(nn.Module):
    def __init__(self, use_target_weight):
        super().__init__()
        self.use_target_weight = use_target_weight

    def forward(self, output, target, target_weight):
        if not output.is_cuda:
            raise RuntimeError("fpd_b200 JointsMSELoss runs on CUDA tensors only (no CPU fallback)")
        tw = target_weight if self.use_target_weight else None
        return _JointsMSEFn.apply(output, target, tw)


class _JointsOHKMFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, output, target, target_weight, topk):
        from fpd_b200 import ops
        out = output.contiguous().float()
        loss3, grad = ops.joints_ohkm_mse(out, target.contiguous().float(),
                                          None if target_weight is None else target_weight.float(), topk,
                                          want_grad=output.requires_grad)
        ctx.save_for_backward(grad)
        return loss3[0].clone()

    @staticmethod
    def backward(ctx, g):
        (grad,) = ctx.saved_tensors
        return (None if grad is None else grad * g), None, None, None


class JointsOHKMMSELoss(nn.Module):
    """Online hard keypoint mining: per sample, the mean of the `topk` largest per-joint JointsMSELoss terms (without
    the division by J), averaged over the batch. Joints outside a sample's top `topk` get a zero gradient."""

    def __init__(self, use_target_weight, topk=8):
        super().__init__()
        self.use_target_weight = use_target_weight
        self.topk = topk

    def forward(self, output, target, target_weight):
        if not output.is_cuda:
            raise RuntimeError("fpd_b200 JointsOHKMMSELoss runs on CUDA tensors only (no CPU fallback)")
        tw = target_weight if self.use_target_weight else None
        return _JointsOHKMFn.apply(output, target, tw, self.topk)
