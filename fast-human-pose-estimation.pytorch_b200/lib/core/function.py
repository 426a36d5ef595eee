"""Drop-in for the reference's lib/core/function.py: `train`, `fpd_train`, `validate` keep the reference
signatures (function.py:28, :99, :189) so tools/train.py / tools/fpd_train.py / tools/test.py call them unchanged.

What changes underneath:
  * fpd_train / train: when the model is the fpd_b200 hourglass and the optimizer is torch.optim.Adam, the
    batch goes through the fused path -- engine forward (+ eval-mode teacher forward without tape), ONE fused
    FPD loss+gradient kernel, the explicit backward tape -- and the gradients are handed to the caller's
    optimizer through .grad, so `optimizer.step()`, LR schedulers and checkpointing keep working. Any other
    model / criterion combination takes the generic autograd route, statement for statement like the reference.
    The criteria may be JointsMSELoss or JointsOHKMMSELoss (online hard keypoint mining, any mix of the two under FPD).
  * per-iteration accuracy() and validate()'s flip test / decode run on the device; only [B,J] indices cross PCIe
    (the reference ships the full heat-maps to numpy every iteration: function.py:154-156, 218-240, 263).
  * train / fpd_train: on the fused route each batch of the epoch's batch shape is one CUDA graph replay (train_step.
    FPDTrainStep in its external-optimizer mode: student forward, teacher forward on a side stream, loss, backward tape
    with the weight gradients on their own stream, PCK counts); the caller's optimizer then steps on the gradients. Losses
    and counts go to pinned host buffers asynchronously; the host waits only to log and at the end of the epoch. Other
    batch shapes (the short last batch) and config.DEBUG.DEBUG take the eager fused route, which gives the same bits.
  * validate: for the fpd_b200 models with JointsMSELoss or JointsOHKMMSELoss, each batch is one CUDA graph replay (infer_step.
    FlipTestInference with its decode stage: both forwards, flip merge, loss, keypoints, PCK counts); the results are
    copied to pinned host buffers asynchronously and the host waits only to log and at the end of the epoch.
"""
import logging
import os
import time

import numpy as np
import torch

from .evaluate import accuracy, pck_from_counts, pck_from_preds
from .inference import get_final_preds, inverse_affines, preds_from_argmax

logger = logging.getLogger(__name__)


def _unwrap(model):
    """The fused path drives the engine of the wrapped module directly, so wrappers cannot be silently bypassed:
    nn.DataParallel over several devices would run the whole batch on one GPU -- refused (launch one process per GPU
    instead, INTEGRATION.md section 1); a 1-device DataParallel / DistributedDataParallel wrapper is transparent, and
    the gradient all-reduce DDP would have done in its autograd hooks is done explicitly in _fused_step."""
    if isinstance(model, torch.nn.DataParallel) and len(model.device_ids or []) > 1:
        raise RuntimeError("fpd_b200: nn.DataParallel over %d devices is not supported by the fused path (it would use one "
                           "GPU); run one process per GPU (torch.distributed.run), device_ids=[local_rank]"
                           % len(model.device_ids))
    return model.module if hasattr(model, "module") else model


def _loss_shape_ok(config_or_none, J, h, w):
    """The fused FPD loss kernel (csrc/loss.cu) wants h*w % 64 == 0 and J <= 64; anything else takes the generic route."""
    return (h * w) % 64 == 0 and 1 <= J <= 64


_flat_grad_cache = {}


def _allreduce_grads_(net, grads):
    """One all-reduce (mean over ranks) of all parameter gradients, through one flat buffer (what DDP's bucketing does)."""
    import torch.distributed as dist
    world = dist.get_world_size()
    n = sum(g.numel() for g in grads)
    key = (id(net), n)
    flat = _flat_grad_cache.get(key)
    if flat is None:
        _flat_grad_cache.clear()
        flat = _flat_grad_cache[key] = torch.empty(n, dtype=torch.float32, device=grads[0].device)
    views, off = [], 0
    for g in grads:
        views.append(flat[off:off + g.numel()].view(g.shape))
        off += g.numel()
    torch._foreach_copy_(views, grads)
    dist.all_reduce(flat, op=dist.ReduceOp.SUM)
    flat.mul_(1.0 / world)
    return views


def _is_fpd_net(model):
    return hasattr(_unwrap(model), "engine") and hasattr(_unwrap(model), "forward_nhwc")


def _is_fpd_criterion(c):
    from .loss import JointsMSELoss, JointsOHKMMSELoss
    return isinstance(c, (JointsMSELoss, JointsOHKMMSELoss))


def _criterion_topk(c):
    """The fused loss kernels' term selector: the criterion's topk for JointsOHKMMSELoss, 0 for JointsMSELoss."""
    from .loss import JointsOHKMMSELoss
    return c.topk if isinstance(c, JointsOHKMMSELoss) else 0


def _fused_step(model, tmodel, input, target, target_weight, alpha, use_tw, graph=None, pose_topk=0, kd_topk=0):
    """student fwd -> teacher fwd -> fused loss+grad -> backward tape; returns (losses[3] dev, last output NHWC).
    graph: a _GraphTraining whose batch shape this batch has -- the same step is then one replay of its graph, and the
    last output is None (the PCK counts come out of the graph instead)."""
    if graph is not None:
        return graph.step(input, target, target_weight), None
    from fpd_b200 import ops
    net = _unwrap(model)
    x = input.cuda(non_blocking=True).float().contiguous()
    eng = net.engine()
    ctx = eng.forward(x, True, record_tape=True)
    outs = [v.data for v in ctx.outs]
    t_last = None
    if tmodel is not None:
        t_last = _unwrap(tmodel).forward_nhwc(x, training=False)[-1]
    B, _, _, J = outs[0].shape
    tw = target_weight.reshape(B, J) if use_tw else torch.ones(B, J, device=x.device)
    losses, grads = ops.fpd_loss(outs, target.contiguous().float(), t_last, tw.contiguous().float(), alpha,
                                 pose_topk=pose_topk, kd_topk=kd_topk)
    pg = eng.backward(ctx, grads)
    params = [p for p in net.parameters() if p.requires_grad]      # frozen parameters keep whatever .grad they had
    glist = []
    for p in params:
        g = pg.get(p)
        glist.append(torch.zeros_like(p) if g is None else g.reshape(p.shape))
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        # one process per GPU: replicas stay identical only if every rank steps on the mean gradient
        glist = _allreduce_grads_(net, glist)
        glist = [g.clone() for g in glist]     # the flat buffer is reused next step; .grad must own its memory
    for p, g in zip(params, glist):
        p.grad = g
    return losses, outs[-1]


# train() / fpd_train() replay one CUDA graph per batch where they can; False forces the eager fused route (the graph
# route's reference in the tests)
_TRAIN_GRAPH = True
_train_step_cache = {}      # key -> FPDTrainStep: one captured step, reused across epochs (it keeps the networks alive)


def _train_route(config, model, tmodel, criteria, target_shape):
    """'graph', 'fused' or 'generic' for a train (tmodel None, one criterion) / fpd_train epoch whose first batch has
    targets of `target_shape`. The graph route replays exactly the eager fused route's kernels; debug images need the
    heat-maps on the host every logged step, so config.DEBUG.DEBUG keeps the eager fused route."""
    fused = (_is_fpd_net(model) and (tmodel is None or _is_fpd_net(tmodel)) and all(_is_fpd_criterion(c) for c in criteria)
             and len({c.use_target_weight for c in criteria}) == 1
             and _loss_shape_ok(config, target_shape[1], target_shape[2], target_shape[3]))
    if not fused:
        return "generic"
    dbg = getattr(config, "DEBUG", None)
    return "graph" if _TRAIN_GRAPH and not (dbg is not None and getattr(dbg, "DEBUG", False)) else "fused"


class _GraphTraining:
    """train()/fpd_train()'s per-batch work as replays of one FPDTrainStep(fused_adam=False, accuracy=True), which is
    cached across calls keyed on the networks, the batch shapes, alpha and the topks. Losses and PCK counts go to pinned
    host buffers with non-blocking copies; `flush` waits for them and applies the meter updates in batch order."""

    def __init__(self, model, tmodel, alpha, use_tw, pose_topk, kd_topk, input, target, target_weight, num_batches):
        from fpd_b200.train_step import FPDTrainStep
        net = _unwrap(model)
        tnet = _unwrap(tmodel) if tmodel is not None else None
        self.shapes = (tuple(input.shape), tuple(target.shape), tuple(target_weight.shape))
        alpha = float(alpha) if tnet is not None else 0.0
        key = (id(net), id(tnet), self.shapes, alpha, pose_topk, kd_topk)
        step = _train_step_cache.get(key)
        if step is None:
            _train_step_cache.clear()          # one graph pool at a time
            step = _train_step_cache[key] = FPDTrainStep(net, tnet, alpha=alpha, pose_topk=pose_topk, kd_topk=kd_topk,
                                                         fused_adam=False, accuracy=True)
        self.train_step = step
        self.trainable = [(p, g) for p, g in zip(step.params, step.grad_views) if p.requires_grad]
        B, J = target.shape[0], target.shape[1]
        self.ones = None if use_tw else torch.ones(B, J, device=target.device)
        self.loss = torch.empty((num_batches, 3), dtype=torch.float32, pin_memory=True)
        self.counts = torch.empty((num_batches, J, 2), dtype=torch.int32, pin_memory=True)
        self.done = torch.cuda.Event()
        self.pending = []          # (batch, num_images) not yet applied to the meters

    def accepts(self, input, target, target_weight):
        return (tuple(input.shape), tuple(target.shape), tuple(target_weight.shape)) == self.shapes

    def step(self, input, target, target_weight):
        """Replay (gradients all-reduced when there are several ranks) and hand the gradients to the parameters'
        .grad, as _fused_step does; returns the device losses[3]."""
        l3 = self.train_step.step(input, target, target_weight if self.ones is None else self.ones)
        for p, g in self.trainable:     # frozen parameters keep whatever .grad they had
            p.grad = g
        return l3

    def record(self, i, l3, num_images):
        """Queue batch i's losses and PCK counts for the host (call after the optimizer step)."""
        self.loss[i].copy_(l3, non_blocking=True)
        self.counts[i].copy_(self.train_step.counts, non_blocking=True)
        self.pending.append((i, num_images))

    def flush(self, apply):
        """apply(losses[3] as floats, avg_acc, cnt, num_images) for every pending batch, in batch order."""
        self.done.record()
        self.done.synchronize()
        for i, n in self.pending:
            _, avg_acc, cnt = pck_from_counts(self.counts[i].numpy())
            apply([float(v) for v in self.loss[i]], avg_acc, cnt, n)
        self.pending = []


def _device_accuracy(out_nhwc, target_nchw):
    """PCK bookkeeping of evaluate.accuracy from device-side arg-maxes (no heat-map D2H)."""
    from fpd_b200 import ops
    B, h, w, J = out_nhwc.shape
    _, idx, mx = ops.flip_merge_argmax(out_nhwc, want_avg=False)
    tidx, tmx = ops.argmax_nchw(target_nchw.contiguous().float())
    pred, _ = preds_from_argmax(idx.cpu().numpy(), mx.cpu().numpy(), w)
    tgt, _ = preds_from_argmax(tidx.cpu().numpy(), tmx.cpu().numpy(), w)
    _, avg, cnt = pck_from_preds(pred, tgt, h, w)
    return avg, cnt, pred


def _debug_images(config, input, meta, target, pred, output, prefix):
    """The reference's debug-image hook (function.py:93-95, 184-186, 289-292; off unless config.DEBUG.DEBUG). It lives in
    the reference's own utils/vis.py (control plane, cv2 / torchvision): called when that module is importable, i.e. under
    fpd_b200.dropin.install(); `output` may be an NHWC tensor straight from the engine."""
    dbg = getattr(config, "DEBUG", None)
    if dbg is None or not getattr(dbg, "DEBUG", False):
        return
    try:
        from utils.vis import save_debug_images
    except ImportError:
        logger.warning("config.DEBUG.DEBUG is set but utils.vis is not importable: no debug images")
        return
    if output is not None and output.dim() == 4 and output.shape[1] != target.shape[1]:
        from fpd_b200 import ops
        output = ops.nhwc_to_nchw(output.contiguous())
    save_debug_images(config, input, meta, target, pred * 4, output, prefix)


def _log_train(config, writer_dict, epoch, i, n_batches, batch_time, data_time, meters, bsz):
    parts = ['Epoch: [%d][%d/%d]' % (epoch, i, n_batches),
             'Time %.3fs (%.3fs)' % (batch_time.val, batch_time.avg),
             'Speed %.1f samples/s' % (bsz / max(batch_time.val, 1e-9)),
             'Data %.3fs (%.3fs)' % (data_time.val, data_time.avg)]
    for label, m, fmt in meters:
        parts.append(('%s ' + fmt + ' (' + fmt + ')') % (label, m.val, m.avg))
    logger.info('\t'.join(parts))
    if writer_dict:
        writer = writer_dict['writer']
        step = writer_dict['train_global_steps']
        for label, m, _ in meters:
            tag = {'Loss': 'train_loss', 'POSE_Loss': 'train_pose_loss', 'KD_POSE_Loss': 'train_kd_pose_loss',
                   'Accuracy': 'train_acc'}[label]
            writer.add_scalar(tag, m.val, step)
        writer_dict['train_global_steps'] = step + 1


def train(config, train_loader, model, criterion, optimizer, epoch, output_dir, tb_log_dir, writer_dict):
    """Plain heat-map regression epoch (reference function.py:28-96): loss = sum over stacks of the criterion."""
    batch_time, data_time, losses, acc = AverageMeter(), AverageMeter(), AverageMeter(), AverageMeter()
    model.train()
    fused = _is_fpd_net(model) and _is_fpd_criterion(criterion)
    end = time.time()
    shape_checked = False
    graph = None

    def apply(l3, avg_acc, cnt, n):
        losses.update(l3[2], n)
        acc.update(avg_acc, cnt)
    for i, (input, target, target_weight, meta) in enumerate(train_loader):
        data_time.update(time.time() - end)
        target = target.cuda(non_blocking=True)
        target_weight = target_weight.cuda(non_blocking=True)
        if fused and not shape_checked:
            route = _train_route(config, model, None, [criterion], target.shape)
            fused = route != "generic"
            shape_checked = True
            if route == "graph":
                graph = _GraphTraining(model, None, 0.0, criterion.use_target_weight, _criterion_topk(criterion), 0,
                                       input, target, target_weight, len(train_loader))
        replay = graph if graph is not None and graph.accepts(input, target, target_weight) else None
        if graph is not None and replay is None:
            graph.flush(apply)          # meter updates stay in batch order
        if fused:
            optimizer.zero_grad()
            l3, out_nhwc = _fused_step(model, None, input, target, target_weight, 0.0, criterion.use_target_weight,
                                       replay, pose_topk=_criterion_topk(criterion))
            optimizer.step()
            if replay is not None:
                replay.record(i, l3, input.size(0))
                batch_time.update(time.time() - end)
                end = time.time()
                if i % config.PRINT_FREQ == 0:
                    replay.flush(apply)
                    _log_train(config, writer_dict, epoch, i, len(train_loader), batch_time, data_time,
                               [('Loss', losses, '%.5f'), ('Accuracy', acc, '%.3f')], input.size(0))
                continue
            losses.update(float(l3[2]), input.size(0))
            avg_acc, cnt, pred = _device_accuracy(out_nhwc, target)
            output = out_nhwc
        else:
            outputs = model(input)
            if isinstance(outputs, list):
                loss = criterion(outputs[0], target, target_weight)
                for output in outputs[1:]:
                    loss += criterion(output, target, target_weight)
                output = outputs[-1]
            else:
                output = outputs
                loss = criterion(output, target, target_weight)
            optimizer.zero_grad()
            loss.backward()
            optimizer.step()
            losses.update(loss.item(), input.size(0))
            _, avg_acc, cnt, pred = accuracy(output.detach(), target.detach())
        acc.update(avg_acc, cnt)
        batch_time.update(time.time() - end)
        end = time.time()
        if i % config.PRINT_FREQ == 0:
            _log_train(config, writer_dict, epoch, i, len(train_loader), batch_time, data_time,
                       [('Loss', losses, '%.5f'), ('Accuracy', acc, '%.3f')], input.size(0))
            _debug_images(config, input, meta, target, pred, output.detach(), '{}_{}'.format(os.path.join(output_dir, 'train'), i))
    if graph is not None:
        graph.flush(apply)


def fpd_train(config, train_loader, model, tmodel, pose_criterion, kd_pose_criterion, optimizer, epoch,
              output_dir, tb_log_dir, writer_dict):
    """Fast-Pose-Distillation epoch (reference function.py:99-187):
    loss = (1-KD.ALPHA) * sum_s L(out_s, target) + KD.ALPHA * sum_s L(out_s, teacher_last)."""
    batch_time, data_time = AverageMeter(), AverageMeter()
    losses, pose_losses, kd_pose_losses, acc = AverageMeter(), AverageMeter(), AverageMeter(), AverageMeter()
    alpha = config.KD.ALPHA
    model.train()
    tmodel.eval()
    fused = (_is_fpd_net(model) and _is_fpd_net(tmodel) and _is_fpd_criterion(pose_criterion)
             and _is_fpd_criterion(kd_pose_criterion)
             and pose_criterion.use_target_weight == kd_pose_criterion.use_target_weight)
    end = time.time()
    shape_checked = False
    graph = None
    meters = [('POSE_Loss', pose_losses, '%.5f'), ('KD_POSE_Loss', kd_pose_losses, '%.5f'), ('Loss', losses, '%.5f'),
              ('Accuracy', acc, '%.3f')]

    def apply(l3, avg_acc, cnt, n):
        pose_losses.update(l3[0], n)
        kd_pose_losses.update(l3[1], n)
        losses.update(l3[2], n)
        acc.update(avg_acc, cnt)
    for i, (input, target, target_weight, meta) in enumerate(train_loader):
        data_time.update(time.time() - end)
        target = target.cuda(non_blocking=True)
        target_weight = target_weight.cuda(non_blocking=True)
        if fused and not shape_checked:
            route = _train_route(config, model, tmodel, [pose_criterion, kd_pose_criterion], target.shape)
            fused = route != "generic"
            shape_checked = True
            if route == "graph":
                graph = _GraphTraining(model, tmodel, alpha, pose_criterion.use_target_weight,
                                       _criterion_topk(pose_criterion), _criterion_topk(kd_pose_criterion),
                                       input, target, target_weight, len(train_loader))
        replay = graph if graph is not None and graph.accepts(input, target, target_weight) else None
        if graph is not None and replay is None:
            graph.flush(apply)          # meter updates stay in batch order
        if fused:
            optimizer.zero_grad()
            l3, out_nhwc = _fused_step(model, tmodel, input, target, target_weight, alpha,
                                       pose_criterion.use_target_weight, replay, pose_topk=_criterion_topk(pose_criterion),
                                       kd_topk=_criterion_topk(kd_pose_criterion))
            optimizer.step()
            if replay is not None:
                replay.record(i, l3, input.size(0))
                batch_time.update(time.time() - end)
                end = time.time()
                if i % config.PRINT_FREQ == 0:
                    replay.flush(apply)
                    _log_train(config, writer_dict, epoch, i, len(train_loader), batch_time, data_time, meters,
                               input.size(0))
                continue
            pose_v, kd_v, loss_v = [float(v) for v in l3.cpu()]
            avg_acc, cnt, pred = _device_accuracy(out_nhwc, target)
            last_out = out_nhwc
        else:
            outputs = model(input)
            with torch.no_grad():  # the teacher's gradients never reach the student update
                toutput = tmodel(input)
            if isinstance(toutput, list):
                toutput = toutput[-1]
            outs = outputs if isinstance(outputs, list) else [outputs]
            pose_loss = pose_criterion(outs[0], target, target_weight)
            kd_pose_loss = kd_pose_criterion(outs[0], toutput, target_weight)
            for output in outs[1:]:
                pose_loss += pose_criterion(output, target, target_weight)
                kd_pose_loss += kd_pose_criterion(output, toutput, target_weight)
            loss = (1 - alpha) * pose_loss + alpha * kd_pose_loss
            optimizer.zero_grad()
            loss.backward()
            optimizer.step()
            pose_v, kd_v, loss_v = pose_loss.item(), kd_pose_loss.item(), loss.item()
            _, avg_acc, cnt, pred = accuracy(outs[-1].detach(), target.detach())
            last_out = outs[-1].detach()
        pose_losses.update(pose_v, input.size(0))
        kd_pose_losses.update(kd_v, input.size(0))
        losses.update(loss_v, input.size(0))
        acc.update(avg_acc, cnt)
        batch_time.update(time.time() - end)
        end = time.time()
        if i % config.PRINT_FREQ == 0:
            _log_train(config, writer_dict, epoch, i, len(train_loader), batch_time, data_time, meters, input.size(0))
            _debug_images(config, input, meta, target, pred, last_out, '{}_{}'.format(os.path.join(output_dir, 'train'), i))
    if graph is not None:
        graph.flush(apply)


# validate() replays one CUDA graph per batch where it can; False forces the eager fused route (the graph route's
# reference in the tests)
_VALIDATE_GRAPH = True


def _validate_graph_ok(config, criterion, target):
    """The graph route computes exactly what the eager fused route does, for the batches its kernels take."""
    dbg = getattr(config, "DEBUG", None)
    _, J, h, w = target.shape
    return (_VALIDATE_GRAPH and _is_fpd_criterion(criterion) and not (dbg is not None and getattr(dbg, "DEBUG", False))
            and J <= 64 and _loss_shape_ok(config, J, h, w))


class _GraphValidation:
    """validate()'s per-batch work as FlipTestInference(decode=True) replays. The device results go to pinned host
    buffers with non-blocking copies; `flush` waits for them and applies the meter updates in batch order."""

    def __init__(self, config, net, val_dataset, criterion, num_samples, num_batches, J):
        from fpd_b200.infer_step import FlipTestInference
        self.runner = FlipTestInference(net, val_dataset.flip_pairs, shift_heatmap=bool(config.TEST.SHIFT_HEATMAP),
                                        flip_test=bool(config.TEST.FLIP_TEST), decode=True)
        self.use_tw = criterion.use_target_weight
        self.topk = _criterion_topk(criterion)
        self.post_process = bool(config.TEST.POST_PROCESS)
        self.preds = torch.empty((num_samples, J, 3), dtype=torch.float32, pin_memory=True)
        self.loss = torch.empty(num_batches, dtype=torch.float32, pin_memory=True)
        self.counts = torch.empty((num_batches, J, 2), dtype=torch.int32, pin_memory=True)
        self.done = torch.cuda.Event()
        self.pending = []          # (batch, num_images) not yet applied to the meters
        self.applied = 0           # samples whose predictions are in all_preds

    def run(self, i, input, target, target_weight, c, s, idx):
        B, _, h, w = target.shape
        r = self.runner(input, inv=inverse_affines(c, s, [w, h]), target=target, target_weight=target_weight,
                        use_target_weight=self.use_tw, post_process=self.post_process, topk=self.topk)
        self.preds[idx:idx + B].copy_(r["preds"], non_blocking=True)
        self.loss[i:i + 1].copy_(r["loss3"][:1], non_blocking=True)
        self.counts[i].copy_(r["pck"], non_blocking=True)
        self.pending.append((i, B))

    def flush(self, losses, acc, all_preds, upto):
        self.done.record()
        self.done.synchronize()
        for i, n in self.pending:
            losses.update(float(self.loss[i]), n)
            _, avg_acc, cnt = pck_from_counts(self.counts[i].numpy())
            acc.update(avg_acc, cnt)
        self.pending = []
        all_preds[self.applied:upto] = self.preds[self.applied:upto].numpy()
        self.applied = upto


def validate(config, val_loader, val_dataset, model, criterion, output_dir, tb_log_dir, writer_dict=None):
    """Evaluation epoch (reference function.py:189-333) with the flip test, shift, average, arg-max on the device."""
    from fpd_b200 import ops
    batch_time, losses, acc = AverageMeter(), AverageMeter(), AverageMeter()
    model.eval()
    num_samples = len(val_dataset)
    all_preds = np.zeros((num_samples, config.MODEL.NUM_JOINTS, 3), dtype=np.float32)
    all_boxes = np.zeros((num_samples, 6))
    image_path, filenames, imgnums = [], [], []
    idx = 0
    fpd_net = _is_fpd_net(model)
    perm_cache = {}
    graph = None
    with torch.no_grad():
        end = time.time()
        for i, (input, target, target_weight, meta) in enumerate(val_loader):
            if fpd_net and i == 0 and _validate_graph_ok(config, criterion, target):
                graph = _GraphValidation(config, _unwrap(model), val_dataset, criterion, num_samples, len(val_loader),
                                         target.shape[1])
            if graph is not None:
                num_images = input.size(0)
                c = meta['center'].numpy()
                s = meta['scale'].numpy()
                score = meta['score'].numpy()
                graph.run(i, input, target, target_weight, c, s, idx)
                batch_time.update(time.time() - end)
                end = time.time()
                all_boxes[idx:idx + num_images, 0:2] = c[:, 0:2]
                all_boxes[idx:idx + num_images, 2:4] = s[:, 0:2]
                all_boxes[idx:idx + num_images, 4] = np.prod(s * 200, 1)
                all_boxes[idx:idx + num_images, 5] = score
                image_path.extend(meta['image'])
                idx += num_images
                if i % config.PRINT_FREQ == 0:
                    graph.flush(losses, acc, all_preds, idx)
                    logger.info('Test: [%d/%d]\tTime %.3f (%.3f)\tLoss %.4f (%.4f)\tAccuracy %.3f (%.3f)' % (
                        i, len(val_loader), batch_time.val, batch_time.avg, losses.val, losses.avg, acc.val, acc.avg))
                continue
            x = input.cuda(non_blocking=True).float().contiguous()
            if fpd_net:
                net = _unwrap(model)
                hm = net.forward_nhwc(x, training=False)[-1]
                hm_f, perm = None, None
                if config.TEST.FLIP_TEST:
                    hm_f = net.forward_nhwc(x.flip(3).contiguous(), training=False)[-1]
                    J = hm.shape[-1]
                    if J not in perm_cache:
                        p = list(range(J))
                        for a, b in val_dataset.flip_pairs:
                            p[a], p[b] = b, a
                        perm_cache[J] = torch.tensor(p, dtype=torch.int32, device=x.device)
                    perm = perm_cache[J]
                avg_nhwc, _, _ = ops.flip_merge_argmax(hm, hm_f, perm, shift=bool(config.TEST.SHIFT_HEATMAP))
                output = ops.nhwc_to_nchw(avg_nhwc)
            else:
                outputs = model(x)
                output = outputs[-1] if isinstance(outputs, list) else outputs
                if config.TEST.FLIP_TEST:
                    from utils.transforms import flip_back  # resolved like the reference (lib on sys.path)
                    of = model(x.flip(3))
                    of = of[-1] if isinstance(of, list) else of
                    of = flip_back(of, val_dataset.flip_pairs).clone()
                    if config.TEST.SHIFT_HEATMAP:
                        of[:, :, :, 1:] = of.clone()[:, :, :, 0:-1]
                    output = (output + of) * 0.5
            target = target.cuda(non_blocking=True)
            target_weight = target_weight.cuda(non_blocking=True)
            loss = criterion(output, target, target_weight)
            num_images = input.size(0)
            losses.update(loss.item(), num_images)
            _, avg_acc, cnt, pred = accuracy(output, target)
            acc.update(avg_acc, cnt)
            batch_time.update(time.time() - end)
            end = time.time()
            c = meta['center'].numpy()
            s = meta['scale'].numpy()
            score = meta['score'].numpy()
            preds, maxvals = get_final_preds(config, output, c, s)
            all_preds[idx:idx + num_images, :, 0:2] = preds[:, :, 0:2]
            all_preds[idx:idx + num_images, :, 2:3] = maxvals
            all_boxes[idx:idx + num_images, 0:2] = c[:, 0:2]
            all_boxes[idx:idx + num_images, 2:4] = s[:, 0:2]
            all_boxes[idx:idx + num_images, 4] = np.prod(s * 200, 1)
            all_boxes[idx:idx + num_images, 5] = score
            image_path.extend(meta['image'])
            idx += num_images
            if i % config.PRINT_FREQ == 0:
                logger.info('Test: [%d/%d]\tTime %.3f (%.3f)\tLoss %.4f (%.4f)\tAccuracy %.3f (%.3f)' % (
                    i, len(val_loader), batch_time.val, batch_time.avg, losses.val, losses.avg, acc.val, acc.avg))
                _debug_images(config, input, meta, target, pred, output, '{}_{}'.format(os.path.join(output_dir, 'val'), i))
        if graph is not None:
            graph.flush(losses, acc, all_preds, idx)
        name_values, perf_indicator = val_dataset.evaluate(config, all_preds, output_dir, all_boxes, image_path,
                                                           filenames, imgnums)
        model_name = config.MODEL.NAME
        for nv in (name_values if isinstance(name_values, list) else [name_values]):
            _print_name_value(nv, model_name)
        if writer_dict:
            writer = writer_dict['writer']
            step = writer_dict['valid_global_steps']
            writer.add_scalar('valid_loss', losses.avg, step)
            writer.add_scalar('valid_acc', acc.avg, step)
            for nv in (name_values if isinstance(name_values, list) else [name_values]):
                writer.add_scalars('valid', dict(nv), step)
            writer_dict['valid_global_steps'] = step + 1
    return perf_indicator


def _print_name_value(name_value, full_arch_name):
    names, values = list(name_value.keys()), list(name_value.values())
    logger.info('| Arch ' + ' '.join('| %s' % n for n in names) + ' |')
    logger.info('|---' * (len(names) + 1) + '|')
    if len(full_arch_name) > 15:
        full_arch_name = full_arch_name[:8] + '...'
    logger.info('| ' + full_arch_name + ' ' + ' '.join('| %.3f' % v for v in values) + ' |')


class AverageMeter(object):
    """Running value / average (same fields the reference's meter exposes: val, avg, sum, count)."""

    def __init__(self):
        self.reset()

    def reset(self):
        self.val = self.avg = self.sum = self.count = 0

    def update(self, val, n=1):
        self.val = val
        self.sum += val * n
        self.count += n
        self.avg = self.sum / self.count if self.count != 0 else 0
