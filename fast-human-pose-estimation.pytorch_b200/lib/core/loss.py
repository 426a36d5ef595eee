"""Drop-in for the reference's lib/core/loss.py: `JointsMSELoss(use_target_weight)` and
`JointsOHKMMSELoss(use_target_weight, topk=8)`, plus `JointsKLDLoss(use_target_weight, temperature=1.0)` (a
distillation loss the reference's tools/fpd_train.py invites as a replacement criterion), called as `(output, target, target_weight) -> 0-dim tensor` supporting
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


class _JointsKLDFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, output, ref, target_weight, temperature):
        from fpd_b200 import ops
        out = output.contiguous().float()
        loss3, grad = ops.joints_kld(out, ref.contiguous().float(),
                                     None if target_weight is None else target_weight.float(), temperature,
                                     want_grad=output.requires_grad)
        ctx.save_for_backward(grad)
        return loss3[0].clone()

    @staticmethod
    def backward(ctx, g):
        (grad,) = ctx.saved_tensors
        return (None if grad is None else grad * g), None, None, None


class JointsKLDLoss(nn.Module):
    """Channel-wise distillation (Shu et al., ICCV 2021) per joint heat-map. Each [h, w] map is a distribution over
    its pixels at temperature T: p = softmax(ref / T) for the reference (the target, or the teacher's last stack under
    FPD), q = softmax(output / T) for the student, and

        L = T^2 / (B*J) * sum_{b,j} w[b,j] * KL(p || q),   dL/doutput = T * w * (q - p) / (B*J)

    w is target_weight when use_target_weight is set, else 1. It enters linearly, where JointsMSELoss squares it; for
    the usual 0/1 visibility weights the two rules give the same result. The temperature must be finite and > 0
    (ValueError otherwise); 1.0 is the usual default and has not been tuned for keypoint accuracy. J <= 64."""

    def __init__(self, use_target_weight, temperature=1.0):
        super().__init__()
        from fpd_b200.ops import _check_temperature
        self.use_target_weight = use_target_weight
        self.temperature = _check_temperature(temperature, "temperature", False)

    def forward(self, output, target, target_weight):
        if not output.is_cuda:
            raise RuntimeError("fpd_b200 JointsKLDLoss runs on CUDA tensors only (no CPU fallback)")
        tw = target_weight if self.use_target_weight else None
        return _JointsKLDFn.apply(output, target, tw, self.temperature)
