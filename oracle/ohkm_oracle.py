"""Plain-torch fp64 restatement of the reference's JointsOHKMMSELoss (lib/core/loss.py:42-87) and of the FPD
combination (lib/core/function.py:127-134) with either criterion per term (test oracle).

Joints are ranked by their fp32-rounded per-joint loss, the lower index first on exact ties (the rule the CUDA kernels
follow; the reference's torch.topk leaves tie order open). Returns values and analytic gradients in float64."""
import torch


def per_joint(output, ref, target_weight=None):
    """l[b,j] = 0.5 * mean_p (w*o - w*g)^2 in float64; output / ref [B,J,...], target_weight [B,J,1] or None."""
    B, J = output.shape[:2]
    o = output.double().reshape(B, J, -1)
    g = ref.double().reshape(B, J, -1)
    w = torch.ones(B, J, 1, dtype=torch.float64, device=o.device) if target_weight is None else \
        target_weight.double().reshape(B, J, 1)
    return 0.5 * ((o * w - g * w) ** 2).mean(2), o, g, w


def select(l, topk):
    """[B,J] bool mask of each sample's topk joints by fp32-rounded l, lower index first on ties."""
    B, J = l.shape
    key = l.float().cpu().tolist()
    mask = torch.zeros(B, J, dtype=torch.bool)
    for b in range(B):
        order = sorted(range(J), key=lambda j: (-key[b][j], j))
        mask[b, order[:topk]] = True
    return mask.to(l.device)


def boundary_ok(l_row, topk, rel=1e-4):
    """False when a sample's topk-th and (topk+1)-th largest non-zero per-joint losses are within `rel` of each other:
    then an fp32 evaluation and an fp64 one may select different joints. Zeros are ignored (zero-weight joints get a
    zero gradient whichever of them is picked)."""
    nz = sorted((float(v) for v in l_row if float(v) != 0.0), reverse=True)
    if topk <= 0 or len(nz) <= topk:
        return True
    return nz[topk - 1] - nz[topk] > rel * nz[topk - 1]


def criterion(output, ref, target_weight=None, topk=0):
    """(value, d value / d output) of JointsOHKMMSELoss(topk) or, for topk = 0, JointsMSELoss; float64."""
    B, J = output.shape[:2]
    l, o, g, w = per_joint(output, ref, target_weight)
    hw = o.shape[2]
    if topk == 0:
        return l.sum() / (B * J), (w * w * (o - g) / (B * J * hw)).reshape(output.shape)
    if not 1 <= topk <= J:
        raise ValueError("topk=%d out of range [1, %d]" % (topk, J))
    m = select(l, topk)
    value = (l * m).sum(1).div(topk).sum() / B
    grad = m.double().unsqueeze(2) * w * w * (o - g) / (B * topk * hw)
    return value, grad.reshape(output.shape)


def fpd(outs, target, teacher, target_weight, alpha, pose_topk=0, kd_topk=0):
    """fpd_train's loss body with NCHW stacks: pose = sum_s crit(out_s, target), kd = sum_s crit(out_s, teacher),
    total = (1-alpha)*pose + alpha*kd. Returns (pose, kd, total, [d total / d out_s])."""
    pose = kd = 0.0
    grads = []
    for o in outs:
        vp, gp = criterion(o, target, target_weight, pose_topk)
        vk, gk = criterion(o, teacher, target_weight, kd_topk)
        pose = pose + vp
        kd = kd + vk
        grads.append((1 - alpha) * gp + alpha * gk)
    return pose, kd, (1 - alpha) * pose + alpha * kd, grads
