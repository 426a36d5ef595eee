"""fp64 torch model of JointsKLDLoss (channel-wise distillation per joint heat-map) and of the FPD combination with any
of the three criteria per term: the reference the KL kernels are tested against.

    p = softmax(ref[b,j,:] / T),  q = softmax(out[b,j,:] / T),  KL[b,j] = sum p (log p - log q)
    L = T^2 / (B*J) * sum_{b,j} w[b,j] KL[b,j],   dL/dout = T * w * (q - p) / (B*J)

A term is ("mse",), ("ohkm", topk) or ("kl", T); the first two come from oracle.ohkm_oracle."""
import torch


def per_map_kl(output, ref, T):
    """KL[b,j] in float64, each [h, w] map a distribution over its pixels."""
    B, J = output.shape[:2]
    logq = torch.log_softmax(output.double().reshape(B, J, -1) / T, dim=2)
    logp = torch.log_softmax(ref.double().reshape(B, J, -1) / T, dim=2)
    return (logp.exp() * (logp - logq)).sum(2)


def _weights(output, target_weight):
    B, J = output.shape[:2]
    if target_weight is None:
        return torch.ones(B, J, dtype=torch.float64, device=output.device)
    return target_weight.double().reshape(B, J)


def kld(output, ref, target_weight=None, T=1.0):
    """(value, d value / d output) in float64, the gradient in closed form."""
    B, J = output.shape[:2]
    w = _weights(output, target_weight)
    value = T * T / (B * J) * (w * per_map_kl(output, ref, T)).sum()
    q = torch.softmax(output.double().reshape(B, J, -1) / T, dim=2)
    p = torch.softmax(ref.double().reshape(B, J, -1) / T, dim=2)
    grad = T * w.unsqueeze(2) * (q - p) / (B * J)
    return value, grad.reshape(output.shape)


def kld_autograd(output, ref, target_weight=None, T=1.0):
    """The same value differentiated by autograd (checks the closed form)."""
    B, J = output.shape[:2]
    o = output.detach().double().requires_grad_(True)
    value = T * T / (B * J) * (_weights(output, target_weight) * per_map_kl(o, ref, T)).sum()
    value.backward()
    return value.detach(), o.grad


def criterion(output, ref, target_weight, term):
    if term[0] == "kl":
        return kld(output, ref, target_weight, term[1])
    from oracle import ohkm_oracle as O
    return O.criterion(output, ref, target_weight, term[1] if term[0] == "ohkm" else 0)


def fpd(outs, target, teacher, target_weight, alpha, pose, kd):
    """fpd_train's loss body with NCHW stacks: (pose, kd, total, [d total / d out_s]) in float64."""
    p_sum = k_sum = 0.0
    grads = []
    for o in outs:
        vp, gp = criterion(o, target, target_weight, pose)
        vk, gk = criterion(o, teacher, target_weight, kd)
        p_sum = p_sum + vp
        k_sum = k_sum + vk
        grads.append((1 - alpha) * gp + alpha * gk)
    return p_sum, k_sum, (1 - alpha) * p_sum + alpha * k_sum, grads


def fpd_kwargs(pose, kd):
    """The ops.fpd_loss keyword arguments of a (pose, kd) pair of terms."""
    kw = {}
    for name, term in (("pose", pose), ("kd", kd)):
        if term[0] == "kl":
            kw[name + "_temperature"] = term[1]
        elif term[0] == "ohkm":
            kw[name + "_topk"] = term[1]
    return kw
