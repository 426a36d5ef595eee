"""Data-parallel plumbing: one process per GPU, replicas kept identical by ONE all-reduce of the flat gradient
buffer per step (NCCL over NVLink/NVSwitch on the GPU box; gloo in the CPU tests).

Replaces the reference's single-process nn.DataParallel (tools/fpd_train.py:143,173), which every iteration
scatters the batch, re-broadcasts all parameters (13 MB student + 102 MB teacher), gathers all outputs to GPU 0 and
reduces gradients to GPU 0. Here weights stay resident on every rank; the teacher needs no
communication; BatchNorm statistics stay per-rank (= the reference's per-replica semantics)."""
import torch
import torch.distributed as dist


def shard_range(global_batch, rank, world):
    """Contiguous per-image shard [lo, hi) of a global batch (per-image data parallelism, no data-path collective).
    NB: allreduce_mean_ averages the per-rank gradients with equal weights, which equals the global-batch mean only for
    EQUAL shards (the losses are per-rank batch means) -- keep global_batch a multiple of world for training."""
    per = global_batch // world
    rem = global_batch % world
    lo = rank * per + min(rank, rem)
    return lo, lo + per + (1 if rank < rem else 0)


def broadcast_module(module, src=0, group=None):
    """Make every rank's parameters and buffers identical once, at start-up."""
    for t in list(module.parameters()) + list(module.buffers()):
        dist.broadcast(t.data, src, group=group)


def allreduce_mean_(flat_grad, group=None):
    """Sum the flat gradient buffer over ranks in place; returns the scale (1/world) the optimizer applies, so the
    division is fused into the Adam kernel instead of costing another pass over the buffer."""
    world = dist.get_world_size(group)
    if world > 1:
        dist.all_reduce(flat_grad, op=dist.ReduceOp.SUM, group=group)
    return 1.0 / world


# ---------------------------------------------------------------------------------------------------------------------
# SyncBN (opt-in: FPD_BN_SYNC=1 or Engine.bn_sync_group). The reference's nn.DataParallel computes BatchNorm statistics
# per replica (tools/fpd_train.py:143,173), which is the default here too (N-rank results == the reference's N-GPU
# results). With the switch on, every train-mode BatchNorm uses the statistics of the GLOBAL batch: forward exchanges
# (mean, biased variance) per layer, backward exchanges (sum dz, sum dz*xhat) -- 2 x C floats per layer and direction
# (2 x 15,424 floats per hourglass-student forward over 182 layers): a latency problem, not a bandwidth one. The N-rank
# result then equals a 1-rank run on the concatenated batch (tests/test_ddp_gpu.py), and differs from the reference's
# multi-GPU numbers by design.
# ---------------------------------------------------------------------------------------------------------------------
def merge_bn_stats(mean, var, group=None):
    """Per-rank (mean, biased variance) over n elements each -> the global batch's, equal n on every rank. Chan's pairwise
    update in float64: var_g = mean_r(var_r + (mean_r - mean_g)^2) -- no E[x^2] - mean^2 cancellation."""
    world = dist.get_world_size(group)
    local = torch.stack([mean, var]).double()
    parts = [torch.empty_like(local) for _ in range(world)]
    dist.all_gather(parts, local, group=group)
    allb = torch.stack(parts)                      # [world, 2, C]
    m, v = allb[:, 0], allb[:, 1]
    mg = m.mean(0)
    vg = (v + (m - mg) ** 2).mean(0)
    return mg.float(), vg.float()


def allreduce_avg(t, group=None):
    """Mean over ranks of a small tensor, out of place (the caller keeps its local values)."""
    out = t.clone()
    world = dist.get_world_size(group)
    if world > 1:
        if dist.get_backend(group) == "nccl":
            dist.all_reduce(out, op=dist.ReduceOp.AVG, group=group)
        else:
            dist.all_reduce(out, op=dist.ReduceOp.SUM, group=group)
            out.mul_(1.0 / world)
    return out
