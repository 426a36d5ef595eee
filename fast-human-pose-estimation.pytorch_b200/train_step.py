"""One FPD training step as a replayable CUDA graph.

What the reference does per iteration (lib/core/function.py:119-147 fpd_train): student forward, teacher
forward, 2 x NUM_STACKS JointsMSELoss evaluations, backward (through student AND teacher), Adam -- ~20k
eager ATen launches plus a DataParallel replicate/scatter/gather. Here the same update is:

    graph replay { weight prep -> student fwd (tape) -> teacher fwd (eval, no tape) -> fused FPD loss+grad
                   -> explicit backward tape -> gradients gathered into one flat buffer }
    [NCCL all-reduce of the flat gradient buffer when world_size > 1]
    one fused Adam launch over the flat parameter buffer

With fused_adam=False the step stops after the all-reduce: the parameters keep their own storage and the caller's
optimizer (any torch.optim optimizer, its state dict, LR schedules) steps on the per-parameter views of the flat gradient
buffer -- lib/core/function.py's train / fpd_train run this way. pose_topk / kd_topk select JointsOHKMMSELoss for a term,
pose_temperature / kd_temperature JointsKLDLoss; accuracy=True adds accuracy()'s PCK counts of the last stack to the graph;
kd_unlabeled_thre distils from unlabeled samples (ops.kd_weights weights the kd term, inside the graph); feature_weight with
a FeatureAdapter adds feature distillation, a hint from the teacher's head feature (ops.feature_mse). step(..., teacher_x=)
distils from a teacher at its own input size: the teacher reads its own crop of the batch and its heat-maps are resampled
onto the student's heat-map grid (ops.resample_heatmaps).

The teacher is forward-only (its gradients never influence the student update; the reference's teacher
backward is wasted work). `plain=True` drops the teacher (function.train semantics,
function.py:44-63).
"""
import os

import torch

from . import ops
from . import _native as N

SHARE_STEM = os.environ.get("FPD_SHARE_STEM", "1") != "0"   # student + teacher share the NHWC image and stem im2col


class FlatParams:
    """Re-homes a module's parameters as views into one flat fp32 buffer (needed for the single all-reduce and the
    single Adam launch). Parameter objects are preserved (only .data changes), so optimizers / state_dict keep
    working. rehome=False keeps the parameters' own storage and builds only the flat gradient buffer (`flat` is then
    None). extra: a second module whose parameters follow the first one's (the feature distillation adapter)."""

    def __init__(self, net, rehome=True, extra=None):
        self.params = [p for p in net.parameters()]
        if extra is not None:
            self.params += [p for p in extra.parameters()]
        dev = self.params[0].device
        sizes = [p.numel() for p in self.params]
        # pad every tensor to a multiple of 4 floats so float4 kernels can run over the flat buffer
        self.offsets = []
        off = 0
        for n in sizes:
            self.offsets.append(off)
            off += (n + 3) // 4 * 4
        self.numel = off
        self.flat = torch.zeros(off, dtype=torch.float32, device=dev) if rehome else None
        self.grad = torch.zeros(off, dtype=torch.float32, device=dev)
        self.grad_views = []
        for p, o in zip(self.params, self.offsets):
            if rehome:
                v = self.flat[o:o + p.numel()].view(p.shape)
                v.copy_(p.data)
                p.data = v
            self.grad_views.append(self.grad[o:o + p.numel()].view(p.shape))

    def is_intact(self):
        if self.flat is None:
            return True
        base = self.flat.untyped_storage().data_ptr()
        return all(p.data.untyped_storage().data_ptr() == base for p in self.params)


def _check_topk(value, name):
    """0 = JointsMSELoss for that term, k >= 1 = JointsOHKMMSELoss(topk=k); the kernels take J <= 64 (the upper bound J
    itself is checked against the heat-maps by ops.fpd_loss)."""
    if isinstance(value, bool) or int(value) != value or not 0 <= value <= 64:
        raise ValueError("%s=%r must be an integer in [0, 64] (0: JointsMSELoss)" % (name, value))
    return int(value)


def head_feature_channels(net):
    """Channels of the feature the network's last heat-map head reads: NUM_FEATURES for the hourglass (the last stack's
    relu(bn(fc)), NUM_CHANNELS[0] for HRNet (the stage-4 branch-0 output). PoseResNet fuses its last BatchNorm + ReLU
    into final_layer's operand pass and has no materialised head feature: ValueError."""
    from .lib.models.hourglass import HourglassNet
    from .lib.models.pose_hrnet import PoseHighResolutionNet
    net = net.module if isinstance(net, torch.nn.DataParallel) else net
    if isinstance(net, HourglassNet):
        return net.fc[-1][0].out_channels
    if isinstance(net, PoseHighResolutionNet):
        return net.final_layer.in_channels
    raise ValueError("feature distillation needs an hourglass (HourglassNet) or HRNet (PoseHighResolutionNet) network, "
                     "got %s: PoseResNet has no materialised head feature" % type(net).__name__)


class FeatureAdapter(torch.nn.Module):
    """The 1x1 convolution (with bias) from the student's head-feature width to the teacher's that feature distillation
    trains with the student: conv(s) is matched to the teacher's head feature. Initialised like the reference's HRNet /
    pose_resnet convolutions (normal, std 0.001; zero bias). It is not a submodule of the student, so the student's
    state_dict keeps the reference's keys: train and checkpoint it next to the student."""

    def __init__(self, student, teacher):
        super().__init__()
        self.conv = torch.nn.Conv2d(head_feature_channels(student), head_feature_channels(teacher), 1, bias=True)
        torch.nn.init.normal_(self.conv.weight, std=0.001)
        torch.nn.init.constant_(self.conv.bias, 0)

    def forward(self, x):
        return self.conv(x)


def check_feature_kd(student, teacher, weight, adapter):
    """The arguments of feature distillation: -> the weight as a float (0.0: off). A weight > 0 needs a teacher and a
    FeatureAdapter whose widths match the two networks' head features, on the student's device."""
    from . import ops
    weight = ops.check_feature_weight(weight)
    if not weight:
        return 0.0
    if teacher is None:
        raise ValueError("feature_weight=%r needs a teacher" % weight)
    if adapter is None:
        raise ValueError("feature_weight=%r needs a feature_adapter (FeatureAdapter(student, teacher))" % weight)
    cs, ct = head_feature_channels(student), head_feature_channels(teacher)
    conv = getattr(adapter, "conv", None)
    if (not isinstance(conv, torch.nn.Conv2d) or conv.kernel_size != (1, 1) or conv.stride != (1, 1)
            or conv.padding != (0, 0) or conv.groups != 1 or conv.bias is None):
        raise ValueError("feature_adapter must be a FeatureAdapter: a module whose .conv is a 1x1 nn.Conv2d with a bias")
    if (conv.in_channels, conv.out_channels) != (cs, ct):
        raise ValueError("feature_adapter maps %d -> %d channels, the student's head feature has %d and the teacher's %d"
                         % (conv.in_channels, conv.out_channels, cs, ct))
    dev = next(student.parameters()).device
    if any(p.device != dev for p in adapter.parameters()):
        raise ValueError("feature_adapter must be on the student's device (%s)" % dev)
    return weight


class FPDTrainStep:
    def __init__(self, student, teacher=None, alpha=0.5, lr=2.5e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0,
                 process_group=None, use_graph=True, pose_topk=0, kd_topk=0, fused_adam=True, accuracy=False,
                 pose_temperature=0.0, kd_temperature=0.0, kd_unlabeled_thre=None, feature_weight=0.0,
                 feature_adapter=None, teacher_input_udp=False):
        """pose_topk / kd_topk: > 0 makes that loss term JointsOHKMMSELoss(topk) instead of JointsMSELoss.
        pose_temperature / kd_temperature: > 0 makes that term JointsKLDLoss(temperature) (not together with a topk).
        fused_adam=False (external-optimizer mode): step() stops once the gradients are in the flat gradient buffer
        (all-reduced, mean over ranks); the parameters keep their own storage and the caller's optimizer steps on
        `grad_views`. lr / betas / eps / weight_decay are then unused.
        accuracy=True: the step also computes accuracy()'s per-joint PCK counts of the last stack (`counts`, int32 [J,2],
        lib.core.evaluate.pck_from_counts).
        kd_unlabeled_thre: None (off), or distil from unlabeled samples, those whose target weights are all exactly 0:
        their kd term is weighted by the teacher's confident joints (last-stack map maximum > kd_unlabeled_thre,
        ops.kd_weights), while labeled samples keep their target weights. Needs a teacher and real target weights.
        feature_weight > 0: feature distillation. feature_adapter (a FeatureAdapter(student, teacher)) maps the student's
        head feature s to the teacher's width, and total += feature_weight * mean((A(s) - t)^2) over every element of
        every sample, labeled or not (ops.feature_mse; not scaled by alpha). The adapter's parameters follow the
        student's in the flat buffers (params, grad_views, fused Adam, state_dict); `feature_loss` is the device scalar
        mean((A(s) - t)^2) of the latest step. Hourglass and HRNet networks only; not with FPD_PIPELINE_TEACHER.
        teacher_input_udp: the crop convention of the teacher inputs step(..., teacher_x=) is given (False: the reference's
        crop_matrix, True: udp_crop_matrix); it picks how teacher heat-map pixels map onto the student's."""
        pose_topk, kd_topk = _check_topk(pose_topk, "pose_topk"), _check_topk(kd_topk, "kd_topk")
        if kd_topk and teacher is None:
            raise ValueError("kd_topk=%d needs a teacher" % kd_topk)
        pose_temperature = ops._check_temperature(pose_temperature, "pose_temperature", True)
        kd_temperature = ops._check_temperature(kd_temperature, "kd_temperature", True)
        if kd_temperature and teacher is None:
            raise ValueError("kd_temperature=%r needs a teacher" % kd_temperature)
        if (pose_topk and pose_temperature) or (kd_topk and kd_temperature):
            raise ValueError("a loss term is JointsOHKMMSELoss (topk) or JointsKLDLoss (temperature), not both")
        if kd_unlabeled_thre is not None:
            kd_unlabeled_thre = ops.check_kd_unlabeled_thre(kd_unlabeled_thre)
            if teacher is None:
                raise ValueError("kd_unlabeled_thre=%r needs a teacher" % kd_unlabeled_thre)
        self.kd_unlabeled_thre = kd_unlabeled_thre
        self.teacher_input_udp = bool(teacher_input_udp)
        self.feature_weight = check_feature_kd(student, teacher, feature_weight, feature_adapter)
        self.adapter = feature_adapter if self.feature_weight else None
        self.feature_loss = None
        self.student, self.teacher = student, teacher
        self.alpha = float(alpha) if teacher is not None else 0.0
        self.lr, self.betas, self.eps, self.wd = lr, betas, eps, weight_decay
        self.pose_topk, self.kd_topk = pose_topk, kd_topk
        self.pose_temperature, self.kd_temperature = pose_temperature, kd_temperature
        self.fused_adam = bool(fused_adam)
        self.want_accuracy = bool(accuracy)
        self.counts = None
        self.pg = process_group
        self.world = 1
        if process_group is not None or (torch.distributed.is_available() and torch.distributed.is_initialized()):
            self.world = torch.distributed.get_world_size(process_group)
        self.flat = FlatParams(student, rehome=self.fused_adam, extra=self.adapter)
        self.exp_avg = torch.zeros_like(self.flat.flat) if self.fused_adam else None
        self.exp_avg_sq = torch.zeros_like(self.flat.flat) if self.fused_adam else None
        self.step_count = 0
        self.use_graph = use_graph
        self.graph = None
        self.static = None
        self.losses = None
        self.launches_per_step = None
        import os
        self.overlap_teacher = os.environ.get("FPD_OVERLAP_TEACHER", "1") != "0"
        self.pipeline = (teacher is not None and use_graph and self.overlap_teacher
                         and os.environ.get("FPD_PIPELINE_TEACHER", "0") != "0")   # measured: no gain over the plain 2nd stream
        if self.pipeline and self.feature_weight:
            raise ValueError("feature distillation needs the teacher's head feature of the same batch: it does not run "
                             "with the teacher pipelined (FPD_PIPELINE_TEACHER)")
        self.x_next = self.t_cur = self.t_next = None
        self.static_tx = None       # the graph's teacher input, when the teacher reads its own crop
        self._have_next = False
        self._static_shapes = None
        self._static_ptrs = None
        self._student_prec = None
        self._teacher_gen = 0
        self._stage_x = self._copy_stream = self._stage_ev = self._stage_free = None   # next batch's images, prefetched
        self._staged_for = None
        self.last_outs = None      # student heat-maps (NHWC, per stack) and the teacher's last stack of the latest step:
        self.last_teacher = None   # kept referenced so the graph's memory pool never recycles them
        self._side = torch.cuda.Stream() if (teacher is not None and self.overlap_teacher) else None
        self._t_keep = None
        # weight gradients (leaves of the backward graph: they only feed the final gradient gather) on a third stream, so
        # they fill the SMs that the small-grid kernels of the dgrad / BatchNorm chain leave idle (hg_fpd on one H100 SXM at
        # 700 W: 84.7 ms/step without, 83.9 with)
        self._wstream = torch.cuda.Stream() if os.environ.get("FPD_WGRAD_STREAM", "1") != "0" else None
        student.train()
        if teacher is not None:
            teacher.eval()

    # ------------------------------------------------------------------ the graph body
    def _body_pipelined(self, x, target, tw, x_next):
        """Same update, with the frozen teacher software-pipelined one batch ahead: while the student does
        forward/loss/backward on batch i (using the teacher heat-map computed during step i-1), the second stream runs the
        teacher forward on batch i+1. The teacher's output does not depend on the student, so the result of every step
        is unchanged; the teacher's ~20 ms simply move off the critical path."""
        s_eng = self.student.engine()
        main = torch.cuda.current_stream()
        self._side.wait_stream(main)
        with torch.cuda.stream(self._side):
            t_ctx = self.teacher.engine().forward(x_next, False, record_tape=False)
            self._t_keep = t_ctx
            self.t_next.copy_(t_ctx.outs[-1].data)
        ctx = s_eng.forward(x, True, record_tape=True)
        outs = [v.data for v in ctx.outs]
        losses, grads = self._loss(outs, target, self.t_cur, tw)
        pg = s_eng.backward(ctx, grads, wgrad_stream=self._wstream)
        self._gather_grads(pg)
        main.wait_stream(self._side)
        return losses

    def _gather_grads(self, pg):
        srcs, dsts = [], []
        for p, gv in zip(self.flat.params, self.flat.grad_views):
            g = pg.get(p)
            if g is None:
                gv.zero_()
            else:
                srcs.append(g.reshape(p.shape))
                dsts.append(gv)
        torch._foreach_copy_(dsts, srcs)

    def _teacher_last(self, t_ctx, tx, target):
        """(the map the loss distils from, the teacher's own last-stack map). With a teacher input of its own size (tx) the
        former is the latter resampled onto the target's heat-map grid."""
        t_native = t_ctx.outs[-1].data
        if tx is None:
            return t_native, t_native
        return ops.resample_heatmaps(t_native, target.shape[2:], udp=self.teacher_input_udp), t_native

    def _body(self, x, target, tw, tx=None):
        """tx: the teacher's own input (its crop of the batch at its input size), or None: the teacher reads x."""
        s_eng = self.student.engine()
        t_last = t_native = None
        t_in = x if tx is None else tx
        if self.teacher is not None and self.overlap_teacher:
            # the frozen teacher's forward is independent of the student's: run it on a second stream so its many
            # small-grid kernels (low-resolution hourglass levels) fill SMs the student leaves idle. It uses no shared
            # workspace (eval-mode BN: no statistics passes), so the two streams touch disjoint memory.
            # Both networks start from the same image: the NHWC conversion and the 7x7-stem im2col columns (335 MB at
            # B=32) are built once, on the main stream, before the fork.
            # (a teacher input of its own size shares nothing with the student's)
            main = torch.cuda.current_stream()
            stem = {} if SHARE_STEM and tx is None else None
            if stem is not None:
                s_eng.prepare_stem(x, stem)
            self._side.wait_stream(main)
            with torch.cuda.stream(self._side):
                t_ctx = self.teacher.engine().forward(t_in, False, record_tape=False, shared_stem=stem)
                self._t_keep = t_ctx            # keep every teacher tensor alive until the streams have joined
                t_last, t_native = self._teacher_last(t_ctx, tx, target)
            ctx = s_eng.forward(x, True, record_tape=True, shared_stem=stem)
            main.wait_stream(self._side)
        else:
            ctx = s_eng.forward(x, True, record_tape=True)
            if self.teacher is not None:
                t_ctx = self.teacher.engine().forward(t_in, False, record_tape=False)
                t_last, t_native = self._teacher_last(t_ctx, tx, target)
        outs = [v.data for v in ctx.outs]
        self.last_outs, self.last_teacher = outs, t_last
        losses, grads = self._loss(outs, target, t_last, tw, t_native)
        if self.feature_weight:
            self._feature_term(s_eng, ctx, t_ctx, losses)
        pg = s_eng.backward(ctx, grads, wgrad_stream=self._wstream)
        self._gather_grads(pg)
        return losses

    def _feature_term(self, s_eng, ctx, t_ctx, losses):
        """Feature distillation: A(s) on the student's tape, the hint loss added to losses[2], and its gradient seeded at
        A(s) for the backward (the teacher's stream has joined: its head feature is complete)."""
        a = s_eng.feature_adapter(ctx, ctx.head_feature, self.adapter.conv)
        _, g = ops.feature_mse(a.data, t_ctx.head_feature.data, self.feature_weight, loss_out=self.feature_loss,
                               losses=losses)
        a.add_grad(g, owned=False)

    def _loss(self, outs, target, t_last, tw, t_native=None):
        """The fused FPD loss and its gradients (+ the PCK counts of the last stack when accuracy=True). t_native: the
        teacher's map at its own size, when t_last was resampled from it."""
        if self.kd_unlabeled_thre is not None:
            # the teacher's stream has joined by now: t_last is complete. A joint's confidence is the maximum of the
            # teacher's own map, as in the reference's rule: bilinear resampling would lower it.
            kdw = ops.kd_weights(t_last if t_native is None else t_native, tw, self.kd_unlabeled_thre)
            losses, grads = ops.fpd_loss(outs, target, t_last, tw, self.alpha, losses_out=self.losses,
                                         pose_topk=self.pose_topk, kd_topk=self.kd_topk,
                                         pose_temperature=self.pose_temperature, kd_temperature=self.kd_temperature,
                                         kd_weight=kdw)
        elif self.pose_temperature or self.kd_temperature:
            losses, grads = ops.fpd_loss(outs, target, t_last, tw, self.alpha, losses_out=self.losses,
                                         pose_topk=self.pose_topk, kd_topk=self.kd_topk,
                                         pose_temperature=self.pose_temperature, kd_temperature=self.kd_temperature)
        elif self.pose_topk or self.kd_topk:
            losses, grads = ops.fpd_loss(outs, target, t_last, tw, self.alpha, losses_out=self.losses,
                                         pose_topk=self.pose_topk, kd_topk=self.kd_topk)
        else:
            losses, grads = ops.fpd_loss(outs, target, t_last, tw, self.alpha, losses_out=self.losses)
        if self.want_accuracy:
            _, idx, maxval = ops.flip_merge_argmax(outs[-1], want_avg=False)
            ops.pck_counts(idx, maxval, target, out=self.counts)
        return losses, grads

    def _outputs(self, target):
        """The step's device outputs: losses[3] and, with accuracy=True, the PCK counts [J,2]."""
        if self.feature_weight:
            # one buffer: losses[3] and the feature loss next to it (fpd_train copies all four with one copy)
            self.losses_feature = torch.zeros(4, dtype=torch.float32, device=target.device)
            self.losses, self.feature_loss = self.losses_feature[:3], self.losses_feature[3:]
        else:
            self.losses = torch.zeros(3, dtype=torch.float32, device=target.device)
        if self.want_accuracy:
            self.counts = torch.zeros((target.shape[1], 2), dtype=torch.int32, device=target.device)

    def _run_body(self):
        if self.pipeline:
            return self._body_pipelined(self.static[0], self.static[1], self.static[2], self.x_next)
        return self._body(*self.static, tx=self.static_tx)

    def _capture(self, x, target, tw, tx=None):
        self.static = (torch.empty_like(x), torch.empty_like(target), torch.empty_like(tw))
        for s, v in zip(self.static, (x, target, tw)):
            s.copy_(v)
        self.static_tx = None if tx is None else tx.clone()
        self._outputs(target)
        if self.pipeline:
            self.x_next = x.clone()
            with torch.no_grad():
                t0 = self.teacher.engine().forward(x, False, record_tape=False).outs[-1].data
            self.t_cur = t0.clone()
            self.t_next = t0.clone()
        # eager warm-up (lazy init, workspace growth, running-stat semantics identical to a normal step)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            self._saved_bn = self._snapshot_bn()
            self._run_body()
            self._restore_bn(self._saved_bn)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        n0 = N.lib().fpd_launch_count()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self._run_body()
        self.launches_per_step = int(N.lib().fpd_launch_count() - n0) + int(self.fused_adam)  # + the Adam launch
        self._restore_bn(self._saved_bn)  # capture does not execute, but keep host-side state tidy

    def _snapshot_bn(self):
        return [b.clone() for b in self.student.buffers()]

    def _restore_bn(self, saved):
        for b, s in zip(self.student.buffers(), saved):
            b.copy_(s)

    # ------------------------------------------------------------------ public
    def step(self, x, target, target_weight, next_x=None, teacher_x=None):
        """x [B,3,H,W], target [B,J,h,w], target_weight [B,J,1] -- CUDA or pinned-host tensors.
        Returns the device tensor losses[3] = (pose, kd, total); no host synchronisation.
        `next_x` (optional): the NEXT step's images as a pinned host tensor -- their H2D copy then runs on a copy stream
        under this step, and the following call must pass that same tensor as `x`.
        With teacher pipelining (`pipeline=True`) pass `next_x`, the NEXT step's images (what a prefetching loader has at
        hand anyway): the teacher runs on them while the student trains on `x`, and the following call must pass that
        same batch as `x`. Without `next_x` the teacher for the following step is run up front (no overlap).
        With fused_adam=False the step ends with the gradients in `grad_views` (mean over ranks); the caller's optimizer
        does the update.
        `teacher_x` (optional): the teacher's own input [B,3,Ht,Wt], the same boxes cropped at the teacher's input size
        (DeviceCropLoader's meta['teacher_input']). The teacher reads it instead of `x`, and its last-stack map is resampled
        onto the target's grid (ops.resample_heatmaps, in the constructor's teacher_input_udp convention) before every loss
        term; kd_unlabeled_thre still reads the teacher's own map. Not with feature distillation or teacher pipelining."""
        tw = target_weight.reshape(target_weight.shape[0], -1)
        if teacher_x is not None:
            self._check_teacher_x(x, teacher_x)
        if self.use_graph:
            shapes = (tuple(x.shape), tuple(target.shape), tuple(tw.shape),
                      None if teacher_x is None else (tuple(teacher_x.shape), self.teacher_input_udp))
            t_gen = self.teacher.engine().generation if self.teacher is not None else 0
            s_prec = self.student.engine().training_precision
            # fused-Adam mode owns the parameters' storage (FlatParams); otherwise the caller may give them new storage
            ptrs = None if self.fused_adam else self._student_ptrs()
            if self.graph is not None and (shapes != self._static_shapes or t_gen != self._teacher_gen
                                           or ptrs != self._static_ptrs or s_prec != self._student_prec):
                # a short last batch / a different resolution, teacher weights reloaded after capture (the graph holds
                # pointers to the teacher's prepared weights), a student parameter / buffer given new storage (the
                # graph holds its old address), or another student training precision (the graph holds its kernels):
                # capture again instead of broadcasting or using stale data
                self.graph = None
            if self.graph is None:
                xd, td, wd = (t.cuda(non_blocking=True).float().contiguous() for t in (x, target, tw))
                txd = None if teacher_x is None else teacher_x.cuda(non_blocking=True).float().contiguous()
                self._capture(xd, td, wd, txd)
                self._static_shapes = shapes
                self._static_ptrs = ptrs
                self._student_prec = s_prec
                self._teacher_gen = self.teacher.engine().generation if self.teacher is not None else 0
                self._have_next = False
            if self.pipeline:
                if self._have_next:
                    # this step's images and teacher heat-map were staged by the previous call
                    self.static[0].copy_(self.x_next, non_blocking=True)
                    self.t_cur.copy_(self.t_next, non_blocking=True)
                else:
                    self.static[0].copy_(x, non_blocking=True)
                    with torch.no_grad():
                        self.t_cur.copy_(self.teacher.engine().forward(self.static[0], False,
                                                                        record_tape=False).outs[-1].data)
                self.static[1].copy_(target, non_blocking=True)
                self.static[2].copy_(tw, non_blocking=True)
                if next_x is not None:
                    self.x_next.copy_(next_x, non_blocking=True)
                self._have_next = next_x is not None
            else:
                self._stage_inputs(x, target, tw)
                if teacher_x is not None:
                    self.static_tx.copy_(teacher_x, non_blocking=True)
            self.graph.replay()
            if not self.pipeline:
                self._prefetch(next_x)
            losses = self.losses
        else:
            xd, td, wd = (t.cuda(non_blocking=True).float().contiguous() for t in (x, target, tw))
            if self.losses is None or (self.want_accuracy and self.counts.shape[0] != td.shape[1]):
                self._outputs(td)
            txd = None if teacher_x is None else teacher_x.cuda(non_blocking=True).float().contiguous()
            n0 = N.lib().fpd_launch_count()
            losses = self._body(xd, td, wd, txd)
            self.launches_per_step = int(N.lib().fpd_launch_count() - n0) + int(self.fused_adam)
        if self.fused_adam:
            gscale = 1.0
            if self.world > 1:
                from .parallel import allreduce_mean_
                gscale = allreduce_mean_(self.flat.grad, self.pg)
            self.step_count += 1
            ops.adam_flat(self.flat.flat, self.flat.grad, self.exp_avg, self.exp_avg_sq, self.lr, self.betas[0],
                          self.betas[1], self.eps, self.wd, self.step_count, grad_scale=gscale)
        else:
            if self.world > 1:
                # the same two operations as DistributedDataParallel's averaging (and lib.core.function's eager route)
                torch.distributed.all_reduce(self.flat.grad, op=torch.distributed.ReduceOp.SUM, group=self.pg)
                self.flat.grad.mul_(1.0 / self.world)
        # weights and running statistics were just rewritten through raw pointers (and, in graph mode, without running any
        # Python): drop the student's cached eval-mode operands so a following validation sees the new values
        self.student.engine().invalidate_eval_cache()
        return losses

    def _check_teacher_x(self, x, teacher_x):
        if self.teacher is None:
            raise ValueError("teacher_x needs a teacher")
        if self.feature_weight:
            raise ValueError("feature distillation does not run with a teacher input of its own size: the teacher's head "
                             "feature would have other spatial sizes than the student's")
        if self.pipeline:
            raise ValueError("teacher_x does not run with the teacher pipelined (FPD_PIPELINE_TEACHER), which runs the "
                             "teacher on next_x")
        if teacher_x.dim() != 4 or teacher_x.shape[0] != x.shape[0] or teacher_x.shape[1] != x.shape[1]:
            raise ValueError("teacher_x %s must be [B, %d, Ht, Wt] with x's batch B = %d" % (
                tuple(teacher_x.shape), x.shape[1], x.shape[0]))

    @property
    def params(self):
        """The student's parameters (then the feature adapter's), in the order of `grad_views`."""
        return self.flat.params

    @property
    def grad_views(self):
        """Per-parameter views of the flat gradient buffer (rewritten by every step; clone to keep one)."""
        return self.flat.grad_views

    def _student_ptrs(self):
        return tuple(t.data_ptr() for t in self.flat.params) + tuple(b.data_ptr() for b in self.student.buffers())

    # ------------------------------------------------------------------ host batches: H2D of batch i+1 under step i
    def _stage_inputs(self, x, target, tw):
        """Bring this step's batch into the graph's static input buffers. If `x` is the pinned host tensor the previous call
        was given as `next_x`, its images already crossed PCIe on the copy stream while that step computed: only a
        device-to-device copy (~10 us) is left on the critical path."""
        main = torch.cuda.current_stream()
        if self._staged_for is not None and self._staged_for is x:
            main.wait_event(self._stage_ev)
            self.static[0].copy_(self._stage_x, non_blocking=True)
            self._stage_free.record(main)          # the staging buffer may be overwritten once this copy has run
        else:
            self.static[0].copy_(x, non_blocking=True)
        self._staged_for = None
        self.static[1].copy_(target, non_blocking=True)
        self.static[2].copy_(tw, non_blocking=True)

    def _prefetch(self, next_x):
        """Start the H2D copy of the NEXT step's images (a pinned host tensor: what a prefetching DataLoader hands over) on
        a copy stream, overlapping this step's graph replay."""
        if next_x is None or next_x.is_cuda or not next_x.is_pinned() or tuple(next_x.shape) != tuple(self.static[0].shape):
            return
        if self._stage_x is None or self._stage_x.shape != self.static[0].shape:
            self._stage_x = torch.empty_like(self.static[0])
            self._copy_stream = torch.cuda.Stream()
            self._stage_ev, self._stage_free = torch.cuda.Event(), torch.cuda.Event()
            self._stage_free.record(torch.cuda.current_stream())
        with torch.cuda.stream(self._copy_stream):
            self._copy_stream.wait_event(self._stage_free)
            self._stage_x.copy_(next_x, non_blocking=True)
            self._stage_ev.record(self._copy_stream)
        self._staged_for = next_x

    def invalidate(self):
        """Force a re-capture on the next step (after editing teacher / student tensors in place by hand)."""
        self.graph = None

    # ------------------------------------------------------------------ checkpointing (the reference saves
    # optimizer.state_dict() next to the model, lib/utils/utils.py:75-84 / tools/fpd_train.py:277-291)
    def state_dict(self):
        self._need_fused_adam()
        return {"step": self.step_count, "exp_avg": self.exp_avg.clone(), "exp_avg_sq": self.exp_avg_sq.clone(),
                "lr": self.lr, "betas": tuple(self.betas), "eps": self.eps, "weight_decay": self.wd,
                "numel": self.flat.numel}

    def load_state_dict(self, sd):
        self._need_fused_adam()
        if int(sd["numel"]) != self.flat.numel:
            raise ValueError("optimizer state is for %d flat parameters, this step has %d" % (sd["numel"], self.flat.numel))
        self.step_count = int(sd["step"])
        self.exp_avg.copy_(sd["exp_avg"])
        self.exp_avg_sq.copy_(sd["exp_avg_sq"])
        self.lr, self.betas, self.eps, self.wd = sd["lr"], tuple(sd["betas"]), sd["eps"], sd["weight_decay"]

    def _need_fused_adam(self):
        if not self.fused_adam:
            raise RuntimeError("FPDTrainStep(fused_adam=False) has no optimizer state: checkpoint the caller's optimizer")
