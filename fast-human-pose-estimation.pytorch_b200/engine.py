"""Host-side execution engine for the stacked-hourglass hot path.

The network topology is the reference's (lib/models/hourglass.py:32-52 Bottleneck.forward, :80-95
Hourglass._hour_glass_forward, :170-192 HourglassNet.forward); the execution is not: activations live in
NHWC, every op is a libfpd_b200 kernel (wgmma implicit-GEMM convs, fused BN/ReLU/operand-split, ...),
and the backward pass is an explicit tape of kernel launches instead of a per-op autograd graph.

Python here only sequences launches and owns tensors (torch = device memory + streams); there is no
torch math on the hot path and no CPU fallback.
"""
import os

import torch

from . import ops


# conv(relu(bn(x))): the operand transform (BN-apply + ReLU + hi/lo split) always happens inside the tensor-core kernels
# (csrc/conv_wgmma.cu); the round-1 two-kernel forms (pre-split operands in HBM)
# and their A/B switches were removed in round 2.
# forward: run each hourglass level's skip branch on a side stream (see Engine.hourglass)
FORK_UP1 = os.environ.get("FPD_FORK_UP1", "1") != "0"
# opt-in SyncBN over the default process group (see parallel.py); the reference's semantics are per-replica statistics
BN_SYNC = os.environ.get("FPD_BN_SYNC", "0") != "0"


def precision_passes():
    """3 = 3xTF32 (fp32-grade, the parity mode and the default), 1 = single-pass TF32."""
    mode = os.environ.get("FPD_PRECISION", "tf32x3").lower()
    if mode in ("tf32x3", "3xtf32", "fp32"):
        return 3
    if mode in ("tf32", "tf32x1"):
        return 1
    raise ValueError("FPD_PRECISION must be tf32x3 or tf32, got %r" % mode)


class Var:
    """An activation tensor (NHWC) plus its gradient slot and cached batch statistics."""
    __slots__ = ("data", "grad", "owned", "stats", "stat_sums", "grad_sum")

    def __init__(self, data):
        self.data = data
        self.grad = None
        self.owned = False   # True if self.grad may be modified in place
        self.stats = None    # (mean, var) of data over pixels, shared by every BN that consumes it
        self.stat_sums = None  # (part[nblocks,C,2] fp64, nblocks, pivot): column sums of data from the producing conv's epilogue
        self.grad_sum = None   # (per-channel sum of grad, operand scale of grad) when grad came whole out of ONE kernel

    def add_grad(self, g, owned):
        self.grad_sum = None      # whatever was known about the previous gradient is stale now
        if self.grad is None:
            self.grad, self.owned = g, owned
        elif self.owned:
            ops.add(self.grad, g, out=self.grad)
        else:
            self.grad = ops.add(self.grad, g)
            self.owned = True

    def accum_target(self):
        """Buffer a kernel may accumulate into (or None -> kernel should write a fresh tensor)."""
        return self.grad if (self.grad is not None and self.owned) else None

    def set_or_merge(self, dx, accumulated):
        if accumulated:
            self.grad_sum = None
            return
        self.add_grad(dx, True)


# stride-2 3x3 convolutions (HRNet stem / transitions / fuse down paths) on the stride-1 tensor-core kernels:
# y = subsample2(conv_s1(x)); 4x the necessary MACs, but on the tensor cores instead of the CUDA-core fallback (hrnet_fpd on one
# H100 SXM at 700 W: 103 ms/step, 319 ms/step with the CUDA-core path)
STRIDE2_TC = os.environ.get("FPD_STRIDE2_TC", "1") != "0"


class ConvRef:
    __slots__ = ("name", "weight", "bias", "k", "stride", "pad", "cin", "cout", "as_s1", "pick_first")

    def __init__(self, name, mod):
        self.name = name
        self.weight = mod.weight
        self.bias = mod.bias
        self.k = mod.kernel_size[0]
        self.stride = mod.stride[0]
        self.pad = mod.padding[0]
        self.cin = mod.in_channels
        self.cout = mod.out_channels
        # run as a stride-1 convolution + even-position pick (decided per call: needs even H, W)
        self.as_s1 = (STRIDE2_TC and self.stride == 2 and self.k == 3 and self.pad == 1 and self.cin >= 4
                      and mod.kernel_size[1] == 3 and mod.stride[1] == 2)
        # stride-2 1x1 (pose_resnet's downsample convs, pose_resnet.py:143-148): pick the even positions FIRST, then an
        # ordinary stride-1 1x1 convolution on a quarter of the pixels
        self.pick_first = (STRIDE2_TC and self.stride == 2 and self.k == 1 and self.pad == 0 and self.cin >= 4
                           and mod.kernel_size[1] == 1 and mod.stride[1] == 2)

    @classmethod
    def derived(cls, name, weight, bias, k, pad):
        """A stride-1 convolution whose weights are derived from another module's (Engine.deconv)."""
        c = cls.__new__(cls)
        c.name, c.weight, c.bias, c.k, c.stride, c.pad = name, weight, bias, k, 1, pad
        c.cout, c.cin = weight.shape[0], weight.shape[1]
        c.as_s1 = c.pick_first = False
        return c

    @property
    def s1(self):
        return self.stride == 1 or self.as_s1 or self.pick_first

    @property
    def im2col_kpad(self):
        """Few-input-channel stem convs run as im2col + 1x1 tensor-core conv; returns the padded K or 0."""
        K = self.cin * self.k * self.k
        if self.cin < 4 and self.k > 1 and K <= 256 and self.cout % 16 == 0 and self.cout <= 256:
            return (K + 31) // 32 * 32
        return 0

    # the tensor-core kernel (csrc/conv_wgmma.cu) takes Cin <= 512, Cout <= 1024 through ops.conv2d_tc_fused and up to
    # 2048 channels each way through ops.conv2d_tc_h, at any image size
    def tc_fwd_at(self, H, W):
        return self.s1 and self.pad == self.k // 2 and (
            ops.conv2d_tc_supported(self.cin, self.cout, self.k)
            or ops.conv2d_tc_h_supported(self.cin, self.cout, self.k, H, W, True))

    def tc_dgrad_at(self, H, W):
        return self.s1 and self.pad == self.k // 2 and (
            ops.conv2d_tc_supported(self.cout, self.cin, self.k)
            or (ops.conv2d_tc_h_supported(self.cout, self.cin, self.k, H, W, True)
                and ops.conv2d_tc_h_supported(self.cout, self.cin, self.k, H, W, False)))

    @property
    def tc_fwd(self):
        return self.s1 and self.pad == self.k // 2 and ops.conv2d_tc_supported(self.cin, self.cout, self.k)

    @property
    def tc_dgrad(self):
        return self.s1 and self.pad == self.k // 2 and ops.conv2d_tc_supported(self.cout, self.cin, self.k)

    @property
    def tc_wgrad(self):
        return self.s1 and self.pad == self.k // 2 and ops.conv2d_wgrad_tc_supported(self.cin, self.cout, self.k)


class BNRef:
    __slots__ = ("name", "mod")

    def __init__(self, name, mod):
        self.name = name
        self.mod = mod


class PreparedWeights:
    """Tensor-core operand forms of the conv weights, prepared on first use within a forward (student: every step,
    inside the captured graph; frozen teacher: once, cached with the eval context):
    [tap][O][I] hi/lo (+ flipped/transposed for dgrad). Forward operands are __half pairs (3xFP16, csrc/conv_wgmma.cu)
    where ops.conv2d_tc_h takes the shape, fp32 containers holding tf32 values otherwise."""

    def __init__(self, passes, scale_without_bias=False):
        self.split = passes == 3
        self._fwd = {}
        self._dgrad = {}
        self.derived = {}      # name -> ConvRef with weights derived from another module's (Engine.deconv)
        # bias-free convolutions get the operand scale of dY from the BatchNorm-backward pass (Engine.force_apply_sum):
        # their 3xFP16 data-gradient weights can then come out of the same launch as the forward ones
        self.scale_without_bias = scale_without_bias

    def fwd(self, c, H, W, also_dgrad=False):
        """-> (w_hi, w_lo, use_h): use_h selects ops.conv2d_tc_h (Cin up to 2048, 3xFP16) over ops.conv2d_tc_fused
        (3xTF32, Cin up to 512).
        also_dgrad: a backward pass will want the data-gradient form too -- when both are 3xFP16 they come out of one
        launch (one read of the weights)."""
        e = self._fwd.get(c.name)
        if e is not None:
            return e
        w = c.weight.detach()
        k, cin = c.k, c.cin
        kpad = c.im2col_kpad
        if kpad:
            # OIHW -> [Cout][(kh,kw,ci)] zero-padded to kpad, as a 1x1 conv weight
            w2 = torch.zeros((c.cout, kpad, 1, 1), dtype=torch.float32, device=w.device)
            w2[:, :c.cin * c.k * c.k, 0, 0] = w.permute(0, 2, 3, 1).reshape(c.cout, -1)
            w, k, cin = w2, 1, kpad
        if self.split and ops.CONV_F16 and ops.conv2d_tc_h_supported(cin, c.cout, k, H, W, True):
            if (also_dgrad and not kpad and ops.CONV_F16_DGRAD and ops.FUSED_REDUCE
                    and (c.bias is not None or self.scale_without_bias) and c.tc_dgrad_at(H, W) and ops.conv2d_tc_h_supported(c.cout, c.cin, c.k, H, W, True)):
                (hi, lo), (dhi, dlo) = ops.weight_prep_f16_both(w)
                self._dgrad[c.name] = (dhi, dlo, True)
            else:
                hi, lo = ops.weight_prep_f16(w, for_dgrad=False, split=True)
            e = (hi, lo, True)
        else:
            hi, lo = ops.weight_prep(w, for_dgrad=False, split=self.split)
            e = (hi, lo, ops.conv2d_tc_h_supported(cin, c.cout, k, H, W, False))
        self._fwd[c.name] = e
        return e

    def dgrad(self, c, H, W, f16_ok=False):
        """f16_ok: the caller has the power-of-two operand scale of dY (ops.channel_sum(..., want_amax=True))."""
        e = self._dgrad.get(c.name)
        if e is not None and e[0].dtype == torch.float16 and not f16_ok:
            e = None   # prepared together with the forward form, but no operand scale for dY: use the 3xTF32 form
        if e is None:
            if (f16_ok and self.split and ops.CONV_F16_DGRAD
                    and ops.conv2d_tc_h_supported(c.cout, c.cin, c.k, H, W, True)):
                hi, lo = ops.weight_prep_f16(c.weight.detach(), for_dgrad=True, split=True)
                e = (hi, lo, True)
            else:
                hi, lo = ops.weight_prep(c.weight.detach(), for_dgrad=True, split=self.split)
                e = (hi, lo, ops.conv2d_tc_h_supported(c.cout, c.cin, c.k, H, W, False))
            self._dgrad[c.name] = e
        return e


class Engine:
    """Runs one forward (and optionally records a backward tape) of a hourglass-family module tree."""

    def __init__(self, net):
        self.net = net
        self.convs = {}
        self.bns = {}
        self.deconvs = {}
        for name, m in net.named_modules():
            if isinstance(m, torch.nn.Conv2d):
                self.convs[name] = ConvRef(name, m)
            elif isinstance(m, torch.nn.BatchNorm2d):
                self.bns[name] = BNRef(name, m)
            elif isinstance(m, torch.nn.ConvTranspose2d):
                self.deconvs[name] = m
        self._eval_cache = None
        self._eval_cache_key = None
        # True: the BatchNorm-backward apply pass always also reduces its output (sum + max |dx|): engines whose convolutions
        # have no bias (HRNet) get the 3xFP16 operand scale of dY from it -- without it their data gradients run on 3xTF32
        self.force_apply_sum = False
        self.bn_sync_group = None  # set to a process group (or True = default group) for SyncBN; FPD_BN_SYNC=1 does it globally
        self._generation = 0       # bumped by everything that writes parameters / buffers behind torch's back
        self._branch_streams = {}
        # load_state_dict() copies in place (bumps ._version, caught by _param_version) -- but a CUDA graph that baked the
        # pointers of the cached prepared weights would not notice, so owners of such graphs watch `generation`
        net.register_load_state_dict_post_hook(lambda module, incompatible: self.invalidate_eval_cache())

    # ------------------------------------------------------------------ parameter preparation
    @property
    def generation(self):
        return self._generation

    def invalidate_eval_cache(self):
        """The native kernels write parameters (fused Adam) and BatchNorm running statistics (bn_stats_fused) through raw
        pointers, which does not bump tensor._version; a replayed CUDA graph does not even run the Python that would. Every
        such writer calls this, so the next eval-mode forward re-derives the prepared weights and the BN affine."""
        self._generation += 1
        self._eval_cache = None
        self._eval_cache_key = None

    def _param_version(self):
        v = 0
        for p in self.net.parameters():
            v += p._version
        for b in self.net.buffers():
            v += b._version
        return (v, self._generation, next(self.net.parameters()).device, precision_passes())

    def _eval_prepared(self):
        key = self._param_version()
        if self._eval_cache is None or self._eval_cache_key != key:
            passes = precision_passes()
            w = PreparedWeights(passes)
            affine = {}
            for name, b in self.bns.items():
                m = b.mod
                scale, shift, invstd = ops.bn_finalize(m.running_mean, m.running_var, m.weight.detach(),
                                                       m.bias.detach(), m.eps, 1, None, None, 0.0)
                affine[name] = (scale, shift, m.running_mean, invstd)
            self._eval_cache = (w, affine)
            self._eval_cache_key = key
        return self._eval_cache

    # ------------------------------------------------------------------ building blocks
    def _bn_affine(self, ctx, x, bn_name):
        """Returns (scale, shift, mean, invstd, batch) for y = (x-mean)*scale+shift; batch=False in eval mode
        (mean/invstd then come from the running statistics)."""
        b = self.bns[bn_name]
        m = b.mod
        if ctx.training:
            count = x.data.numel() // x.data.shape[-1]
            momentum = m.momentum if m.momentum is not None else 0.1
            track = m.track_running_stats and m.running_mean is not None
            if ctx.sync is not None:
                # SyncBN: local statistics -> one small all-gather -> statistics of the global batch (parallel.py)
                from . import parallel
                if x.stats is None:
                    x.stats = parallel.merge_bn_stats(*ops.bn_stats(x.data), group=ctx.sync[0])
                mean, var = x.stats
                scale, shift, invstd = ops.bn_finalize(mean, var, m.weight.detach(), m.bias.detach(), m.eps,
                                                       count * ctx.sync[1], m.running_mean if track else None,
                                                       m.running_var if track else None, momentum)
            elif x.stats is None and x.stat_sums is not None:
                # the producing convolution's epilogue already summed this tensor per channel: finalize only (no pass over x)
                part, nblocks, pivot = x.stat_sums
                mean, var, scale, shift, invstd = ops.bn_finalize_sums(
                    part, nblocks, pivot, count, m.weight.detach(), m.bias.detach(), m.eps,
                    m.running_mean if track else None, m.running_var if track else None, momentum)
                x.stats = (mean, var)
            elif x.stats is None and ops.FUSED_REDUCE and x.data.shape[-1] % 4 == 0:
                # statistics + this BN's finalize in one launch
                mean, var, scale, shift, invstd = ops.bn_stats_finalize(
                    x.data, m.weight.detach(), m.bias.detach(), m.eps, m.running_mean if track else None,
                    m.running_var if track else None, momentum)
                x.stats = (mean, var)
            else:
                if x.stats is None:
                    x.stats = ops.bn_stats(x.data)
                mean, var = x.stats
                scale, shift, invstd = ops.bn_finalize(mean, var, m.weight.detach(), m.bias.detach(), m.eps, count,
                                                       m.running_mean if track else None,
                                                       m.running_var if track else None, momentum)
            if track and m.num_batches_tracked is not None:
                ctx.nbt.append(m.num_batches_tracked)
            return scale, shift, mean, invstd, True
        scale, shift, rmean, rinvstd = ctx.affine[bn_name]
        return scale, shift, rmean, rinvstd, False

    def _bn_backward(self, ctx, x, bn_name, relu, da, aff):
        """dL/d(act(bn(x))) = da  ->  accumulates dL/dx into x.grad and records dgamma/dbeta."""
        m = self.bns[bn_name].mod
        scale, shift, mean, invstd, batch = aff
        tgt = x.accum_target()
        if batch:
            sync_mean = None
            if ctx.sync is not None:
                from . import parallel
                sync_mean = lambda sums: parallel.allreduce_avg(sums, ctx.sync[0])     # noqa: E731
            dx, dgamma, dbeta, dsum = ops.bn_bwd(da, x.data, mean, invstd, scale, shift, m.weight.detach(), relu,
                                                 accumulate_into=tgt, sync_mean=sync_mean,
                                                 want_dx_sum="force" if self.force_apply_sum else True)
            ctx.pgrads[m.weight] = dgamma
            ctx.pgrads[m.bias] = dbeta
            x.set_or_merge(dx, tgt is not None)
            if dsum is not None and x.grad is dx:
                x.grad_sum = dsum     # x.grad is exactly this kernel's output (until someone adds to it)
            return
        else:  # eval-mode affine: statistics are constants, so no batch-statistics terms in dx
            sums = ops.bn_bwd_reduce(da, x.data, mean, invstd, scale, shift, relu)
            C = x.data.shape[-1]
            ctx.pgrads[m.weight] = sums[C:]
            ctx.pgrads[m.bias] = sums[:C]
            dx = ops.affine_act_bwd(da, x.data, scale, shift, relu, accumulate_into=tgt, mean=mean)
        x.set_or_merge(dx, tgt is not None)

    def bn_act(self, ctx, x, bn_name, relu=True):
        """Materialised y = relu(bn(x)) (stem bn1, fc bn): reference hourglass.py:117-119,161-168."""
        aff = self._bn_affine(ctx, x, bn_name)
        out = Var(ops.affine_act(x.data, aff[0], aff[1], relu, mean=aff[2]))
        if ctx.tape is not None:
            def bwd():
                if out.grad is None:
                    return
                self._bn_backward(ctx, x, bn_name, relu, out.grad, aff)
            ctx.tape.append(bwd)
        return out

    def conv(self, ctx, x, conv_name, bn_name=None, relu=False, residual=None, need_dx=True, out_bn=None):
        """y = conv(act(bn(x))) + bias (+ residual).  bn_name None -> the conv consumes x raw.
        out_bn: name of a train-mode BatchNorm that will consume y (True: some BatchNorm, name unknown) -- the conv then
        also emits y's per-channel sums from its epilogue (Var.stat_sums), pivoted on that module's running mean."""
        c = conv_name if isinstance(conv_name, ConvRef) else self.convs[conv_name]
        if c.pick_first and not getattr(ctx, "_in_s1", False):
            H_, W_ = x.data.shape[1], x.data.shape[2]
            if (H_ % 2 == 0 and W_ % 2 == 0 and bn_name is None and residual is None and x.data.shape[-1] % 4 == 0
                    and c.tc_fwd_at(H_ // 2, W_ // 2)):
                xs = self.subsample2(ctx, x)
                ctx._in_s1 = True
                try:
                    return self.conv(ctx, xs, c, None, relu, None, need_dx, out_bn=out_bn)
                finally:
                    ctx._in_s1 = False
        if c.as_s1 and not getattr(ctx, "_in_s1", False):
            H_, W_ = x.data.shape[1], x.data.shape[2]
            if (H_ % 2 == 0 and W_ % 2 == 0 and c.cout % 4 == 0 and c.tc_fwd_at(H_, W_) and residual is None
                    and not (bn_name is None and c.im2col_kpad)):
                # stride 2 = stride-1 convolution on the tensor cores + even-position pick (recorded as two tape entries:
                # the pick's backward scatters dY into a zero tensor, the stride-1 conv's backward is the ordinary one)
                ctx._in_s1 = True
                try:
                    full = self.conv(ctx, x, c, bn_name, relu, residual, need_dx, out_bn=None)
                finally:
                    ctx._in_s1 = False
                return self.subsample2(ctx, full)
        wrapped = getattr(ctx, "_in_s1", False)        # called by one of the two stride-2 wrappers above
        s1_ok = c.stride == 1 or wrapped
        Hx, Wx = x.data.shape[1], x.data.shape[2]
        tc_fwd = c.tc_fwd_at(Hx, Wx) and s1_ok
        scale = shift = mean = None
        aff = None
        if bn_name is not None:
            aff = self._bn_affine(ctx, x, bn_name)
            scale, shift, mean = aff[0], aff[1], aff[2]
        bias = c.bias.detach() if c.bias is not None else None
        res = residual.data if residual is not None else None
        kpad = c.im2col_kpad if bn_name is None else 0
        if kpad:
            key = (x.data.data_ptr(), tuple(x.data.shape), c.k, c.stride, c.pad, kpad)
            if ctx.shared_stem is not None and ctx.shared_stem.get("cols_key") == key:
                cols = ctx.shared_stem["cols"]     # the same image columns another network already built this step
            else:
                cols = ops.im2col(x.data, c.k, c.stride, c.pad, kpad)
                if ctx.shared_stem is not None and "cols_key" not in ctx.shared_stem:
                    ctx.shared_stem["cols_key"], ctx.shared_stem["cols"] = key, cols
            w_hi, w_lo, use_h = ctx.weights.fwd(c, cols.shape[1], cols.shape[2])
            conv_fn = ops.conv2d_tc_h if use_h else ops.conv2d_tc_fused
            out = Var(conv_fn(cols, w_hi, w_lo, 1, bias=bias, residual=res))
            if ctx.tape is not None:
                def bwd_stem():
                    dy = out.grad
                    if dy is None:
                        return
                    if residual is not None:
                        residual.add_grad(dy, owned=False)
                    if c.bias is not None:
                        ctx.pgrads[c.bias] = ops.channel_sum(dy)
                    dw = ops.conv2d_wgrad_tc_fused(cols, dy, 1, passes=ctx.passes)      # [Cout, kpad, 1, 1]
                    K = c.cin * c.k * c.k
                    ctx.pgrads[c.weight] = dw[:, :K, 0, 0].reshape(c.cout, c.k, c.k, c.cin).permute(0, 3, 1, 2).contiguous()
                    if need_dx:
                        x.add_grad(ops.conv2d_simt_dgrad(dy, c.weight.detach(), x.data.shape[1:3], stride=c.stride,
                                                         pad=c.pad), owned=True)
                ctx.tape.append(bwd_stem)
            return out
        if tc_fwd:
            w_hi, w_lo, use_h = ctx.weights.fwd(c, x.data.shape[1], x.data.shape[2],
                                                also_dgrad=ctx.tape is not None and need_dx)
            stat_sums = None
            if use_h and out_bn and ctx.training and ctx.sync is None:
                Bn, Hn, Wn = x.data.shape[0], x.data.shape[1], x.data.shape[2]
                nblk = ops.conv2d_tc_h_stats_blocks(Bn, Hn, Wn, c.cin, c.cout, c.k, w_hi.dtype == torch.float16)
                if nblk > 0:
                    pivot = None
                    if out_bn is not True and self.bns[out_bn].mod.running_mean is not None:
                        pivot = self.bns[out_bn].mod.running_mean
                    stat_sums = (torch.empty((nblk, c.cout, 2), dtype=torch.float64, device=x.data.device), nblk, pivot)
            if stat_sums is not None:
                y = ops.conv2d_tc_h(x.data, w_hi, w_lo, c.k, mean=mean, scale=scale, shift=shift, relu=relu, bias=bias,
                                    residual=res, stats_part=stat_sums[0], stats_pivot=stat_sums[2])
            else:
                # BN-apply + ReLU + operand split happen inside the conv kernel (no separate HBM pass)
                conv_fn = ops.conv2d_tc_h if use_h else ops.conv2d_tc_fused
                y = conv_fn(x.data, w_hi, w_lo, c.k, mean=mean, scale=scale, shift=shift, relu=relu, bias=bias,
                            residual=res)
        else:
            a = ops.affine_act(x.data, scale, shift, relu, mean=mean) if bn_name is not None else x.data
            y = ops.conv2d_simt_fwd(a, c.weight.detach(), bias=bias, residual=res, stride=c.stride, pad=c.pad)
        out = Var(y)
        if tc_fwd:
            out.stat_sums = stat_sums
        tc_wgrad = c.tc_wgrad and s1_ok
        tc_dgrad = c.tc_dgrad_at(Hx, Wx) and s1_ok
        in_s1 = c.as_s1 and wrapped          # stride-2 3x3 running as stride 1 + pick: dY arrives zero-upsampled
        stride_eff = 1 if wrapped else c.stride   # (pick-first 1x1: x is already the picked tensor, a true stride-1 conv)
        wgrad_chunks = None                  # too wide for one tensor-core wgrad launch: one launch per channel chunk
        if (ctx.tape is not None and not tc_wgrad and s1_ok and c.pad == c.k // 2
                and (bn_name is not None or not c.im2col_kpad)):
            wgrad_chunks = ops.wgrad_channel_chunks(c.cin, c.cout, c.k)
        if ctx.tape is not None:
            def bwd():
                dy = out.grad
                if dy is None:
                    return
                if residual is not None:
                    residual.add_grad(dy, owned=False)
                dy_scale = None
                if out.grad_sum is not None:
                    # dY came whole out of one BatchNorm-backward apply pass, which already summed it per channel and
                    # derived its power-of-two operand scale
                    dy_scale = out.grad_sum[1]
                    if c.bias is not None:
                        ctx.pgrads[c.bias] = out.grad_sum[0]
                elif c.bias is not None:
                    # bias gradient; the same pass over dY yields the power-of-two scale of the 3xFP16 data gradient
                    ctx.pgrads[c.bias], dy_scale = ops.channel_sum(dy, want_amax=True)
                # ---- weight gradient
                if tc_wgrad and ctx.wgrad_stream is not None:
                    # dW (and the bias gradient) are leaves of the backward graph: compute them on a side stream so they
                    # fill the SMs that the small-grid kernels of the critical dgrad/BN chain leave idle
                    main = torch.cuda.current_stream()
                    ev = torch.cuda.Event()
                    ev.record(main)
                    with torch.cuda.stream(ctx.wgrad_stream):
                        ctx.wgrad_stream.wait_event(ev)
                        ctx.pgrads[c.weight] = ops.conv2d_wgrad_tc_fused(x.data, dy, c.k, mean=mean, scale=scale,
                                                                         shift=shift, relu=relu, passes=ctx.passes)
                    ctx.keepalive.append(dy)     # dy must outlive the side-stream kernel (released after the join)
                elif tc_wgrad:
                    ctx.pgrads[c.weight] = ops.conv2d_wgrad_tc_fused(x.data, dy, c.k, mean=mean, scale=scale, shift=shift,
                                                                     relu=relu, passes=ctx.passes)
                elif wgrad_chunks is not None:
                    ctx.pgrads[c.weight] = ops.conv2d_wgrad_tc_chunked(x.data, dy, c.k, wgrad_chunks, mean=mean, scale=scale,
                                                                       shift=shift, relu=relu, passes=ctx.passes)
                else:
                    a_full = (ops.affine_act(x.data, scale, shift, relu, mean=mean) if bn_name is not None
                              else x.data)
                    # CUDA-core fallback; for a stride-2 conv in stride-1 mode go back to the compact dY (the even
                    # positions of the zero-upsampled one) and the true stride: a quarter of the work
                    dy_w = ops.subsample2(dy) if in_s1 else dy
                    ctx.pgrads[c.weight] = ops.conv2d_simt_wgrad(a_full, dy_w, c.k, stride=c.stride if (in_s1 or not wrapped) else 1,
                                                                 pad=c.pad)
                if not need_dx:
                    return
                # ---- data gradient w.r.t. the conv input a = act(bn(x))
                if tc_dgrad:
                    wd_hi, wd_lo, use_h = ctx.weights.dgrad(c, dy.shape[1], dy.shape[2], f16_ok=dy_scale is not None)
                    if use_h:
                        da = ops.conv2d_tc_h(dy, wd_hi, wd_lo, c.k,
                                             in_scale=dy_scale if wd_hi.dtype == torch.float16 else None)
                    else:
                        da = ops.conv2d_tc_fused(dy, wd_hi, wd_lo, c.k)
                else:
                    da = ops.conv2d_simt_dgrad(dy, c.weight.detach(), x.data.shape[1:3], stride=stride_eff, pad=c.pad)
                if bn_name is not None:
                    self._bn_backward(ctx, x, bn_name, relu, da, aff)
                else:
                    x.add_grad(da, owned=True)
            ctx.tape.append(bwd)
        return out

    def subsample2(self, ctx, x):
        """Even-position pick that turns a stride-1 3x3 convolution into the stride-2 one (see ConvRef.as_s1)."""
        out = Var(ops.subsample2(x.data))
        if ctx.tape is not None:
            def bwd():
                if out.grad is None:
                    return
                gs = out.grad_sum
                fresh = x.grad is None
                x.add_grad(ops.upsample_zero2(out.grad), owned=True)
                if fresh and gs is not None:
                    x.grad_sum = gs       # zeros add nothing: the per-channel sums and the maximum carry over unchanged
            ctx.tape.append(bwd)
        return out

    def deconv(self, ctx, x, name, bn_name=None, relu=False):
        """y = ConvTranspose2d_{k, stride 2}(act(bn(x))) (pose_resnet.py:176-204) = depth_to_space(conv3x3_{4 Cout}(...)):
        the four output parities of a stride-2 transposed convolution are four 2x2-tap convolutions of the input, written
        here as ONE 3x3 convolution with structurally zero taps (2.25 x the MACs, but on the tensor-core path with the
        BN + ReLU + split operand pass, the 3xFP16 data gradient and the tensor-core weight gradient that come with it)."""
        m = self.deconvs[name]
        k, pad = m.kernel_size[0], m.padding[0]
        if not (m.stride == (2, 2) and m.kernel_size[1] == k and (k, pad, m.output_padding[0]) in ((4, 1, 0), (3, 1, 1), (2, 0, 0))
                and m.groups == 1 and m.dilation == (1, 1)):
            raise NotImplementedError("deconv %s: only pose_resnet's stride-2 (kernel, padding, output_padding) = "
                                      "(4,1,0) (3,1,1) (2,0,0) are implemented" % name)
        cached = ctx.weights.derived.get(name)
        if cached is None:
            w3 = ops.deconv_weight_to_conv3(m.weight.detach(), pad)
            b3 = m.bias.detach().repeat(4) if m.bias is not None else None
            cached = ConvRef.derived(name, w3, b3, 3, 1)
            ctx.weights.derived[name] = cached
        c = cached
        if ctx.tape is not None:
            def bwd_map():      # recorded BEFORE the convolution: runs after its backward
                dw3 = ctx.pgrads.pop(c.weight, None)
                if dw3 is None:
                    return
                if ctx.wgrad_stream is not None:
                    torch.cuda.current_stream().wait_stream(ctx.wgrad_stream)
                ctx.pgrads[m.weight] = ops.conv3_grad_to_deconv(dw3, k, pad)
                if c.bias is not None:
                    ctx.pgrads[m.bias] = ctx.pgrads.pop(c.bias).view(4, -1).sum(0)
            ctx.tape.append(bwd_map)
        y = self.conv(ctx, x, c, bn_name, relu)
        out = Var(ops.depth_to_space2(y.data))
        if ctx.tape is not None:
            def bwd():
                if out.grad is None:
                    return
                gs = out.grad_sum
                y.add_grad(ops.space_to_depth2(out.grad), owned=True)
                if gs is not None and c.bias is None:
                    y.grad_sum = (None, gs[1])     # a permutation: the maximum, hence the operand scale, carries over
            ctx.tape.append(bwd)
        return out

    def maxpool3(self, ctx, x):
        """nn.MaxPool2d(3, 2, 1) of the pose_resnet stem."""
        out = Var(ops.maxpool3x3s2(x.data))
        if ctx.tape is not None:
            def bwd():
                if out.grad is None:
                    return
                tgt = x.accum_target()
                dx = ops.maxpool3x3s2_bwd(x.data, out.grad, accumulate_into=tgt)
                x.set_or_merge(dx, tgt is not None)
            ctx.tape.append(bwd)
        return out

    def maxpool(self, ctx, x):
        out = Var(ops.maxpool2x2(x.data))
        if ctx.tape is not None:
            def bwd():
                if out.grad is None:
                    return
                tgt = x.accum_target()
                dx = ops.maxpool2x2_bwd(x.data, out.grad, accumulate_into=tgt)
                x.set_or_merge(dx, tgt is not None)
            ctx.tape.append(bwd)
        return out

    def upsample_add(self, ctx, up1, low):
        out = Var(ops.upsample2x_add(up1.data, low.data))
        if ctx.tape is not None:
            def bwd():
                if out.grad is None:
                    return
                up1.add_grad(out.grad, owned=False)
                low.add_grad(ops.upsample2x_bwd(out.grad), owned=True)
            ctx.tape.append(bwd)
        return out

    # ------------------------------------------------------------------ hourglass topology
    def bottleneck(self, ctx, x, prefix, out_bn=None):
        """Pre-activation residual block, reference hourglass.py:32-52. out_bn: the block output goes straight into a
        BatchNorm (the next block's bn1): conv3's epilogue then carries its statistics too."""
        has_ds = (prefix + ".downsample.0") in self.convs
        skip = self.conv(ctx, x, prefix + ".downsample.0") if has_ds else x
        y = self.conv(ctx, x, prefix + ".conv1", prefix + ".bn1", relu=True, out_bn=prefix + ".bn2")
        y = self.conv(ctx, y, prefix + ".conv2", prefix + ".bn2", relu=True, out_bn=prefix + ".bn3")
        return self.conv(ctx, y, prefix + ".conv3", prefix + ".bn3", relu=True, residual=skip, out_bn=out_bn)

    def residual_seq(self, ctx, x, prefix, nblocks, out_bn=None):
        for i in range(nblocks):
            nxt = "%s.%d.bn1" % (prefix, i + 1) if i + 1 < nblocks else out_bn
            x = self.bottleneck(ctx, x, "%s.%d" % (prefix, i), out_bn=nxt)
        return x

    def hourglass(self, ctx, n, x, prefix, nblocks):
        """Recursive U, reference hourglass.py:80-92. The skip branch (up1) does not depend on the lower pyramid: with
        FORK_UP1 it runs on a per-level side stream, so its wide kernels fill the SMs while the low-resolution chain
        (4..64 CTAs per kernel, latency-bound) proceeds on the main stream; the branches join before the upsample-add."""
        done = None
        if FORK_UP1 and x.data.is_cuda:
            main = torch.cuda.current_stream()
            bs = self._branch_stream(main, n)
            ev = torch.cuda.Event()
            ev.record(main)
            with torch.cuda.stream(bs):
                bs.wait_event(ev)
                up1 = self.residual_seq(ctx, x, "%s.%d.0" % (prefix, n - 1), nblocks)
                done = torch.cuda.Event()
                done.record(bs)
        else:
            up1 = self.residual_seq(ctx, x, "%s.%d.0" % (prefix, n - 1), nblocks)
        low1 = self.maxpool(ctx, x)
        # low1 feeds a BatchNorm directly (the next level's skip branch / the innermost block): statistics from the epilogue
        low1 = self.residual_seq(ctx, low1, "%s.%d.1" % (prefix, n - 1), nblocks, out_bn=True)
        if n > 1:
            low2 = self.hourglass(ctx, n - 1, low1, prefix, nblocks)
        else:
            low2 = self.residual_seq(ctx, low1, "%s.%d.3" % (prefix, n - 1), nblocks,
                                     out_bn="%s.%d.2.0.bn1" % (prefix, n - 1))
        low3 = self.residual_seq(ctx, low2, "%s.%d.2" % (prefix, n - 1), nblocks)
        if done is not None:
            torch.cuda.current_stream().wait_event(done)
        return self.upsample_add(ctx, up1, low3)

    def _branch_stream(self, main, level):
        """One side stream per (calling stream, hourglass level), created once per engine."""
        key = (main.cuda_stream, level)
        st = self._branch_streams.get(key)
        if st is None:
            st = torch.cuda.Stream()
            self._branch_streams[key] = st
        return st

    def hourglass_net(self, ctx, img_nchw):
        """HourglassNet.forward, reference hourglass.py:170-192. Returns the per-stack heat-map Vars (NHWC)."""
        net = self.net
        nb = net.num_blocks
        if ctx.shared_stem is not None and ctx.shared_stem.get("img") is img_nchw:
            x = Var(ctx.shared_stem["nhwc"])      # student and teacher see the same batch: one layout conversion
        else:
            x = Var(ops.nchw_to_nhwc(img_nchw))
            if ctx.shared_stem is not None and "img" not in ctx.shared_stem:
                ctx.shared_stem["img"], ctx.shared_stem["nhwc"] = img_nchw, x.data
        x = self.conv(ctx, x, "conv1", need_dx=False)
        x = self.bn_act(ctx, x, "bn1", relu=True)
        x = self.residual_seq(ctx, x, "layer1", 1)
        x = self.maxpool(ctx, x)
        x = self.residual_seq(ctx, x, "layer2", 1, out_bn="layer3.0.bn1")
        x = self.residual_seq(ctx, x, "layer3", 1, out_bn=True)
        outs = []
        for i in range(net.num_stacks):
            y = self.hourglass(ctx, 4, x, "hg.%d.hg" % i, nb)
            y = self.residual_seq(ctx, y, "res.%d" % i, nb)
            y = self.conv(ctx, y, "fc.%d.0" % i, out_bn="fc.%d.1" % i)
            y = self.bn_act(ctx, y, "fc.%d.1" % i, relu=True)
            score = self.conv(ctx, y, "score.%d" % i)
            outs.append(score)
            if i < net.num_stacks - 1:
                t = self.conv(ctx, y, "fc_.%d" % i, residual=x)
                x = self.conv(ctx, score, "score_.%d" % i, residual=t, out_bn=True)
        return outs

    def prepare_stem(self, img_nchw, shared_stem):
        """Fills shared_stem with the NHWC image and (when the stem conv runs as im2col + tensor-core GEMM) its columns,
        on the current stream, so that several networks consuming this batch can share them."""
        if not (img_nchw.is_contiguous() and img_nchw.dtype == torch.float32):
            return
        c = self.convs.get("conv1")
        shared_stem["img"], shared_stem["nhwc"] = img_nchw, ops.nchw_to_nhwc(img_nchw)
        if c is not None and c.im2col_kpad:
            kpad = c.im2col_kpad
            x = shared_stem["nhwc"]
            shared_stem["cols_key"] = (x.data_ptr(), tuple(x.shape), c.k, c.stride, c.pad, kpad)
            shared_stem["cols"] = ops.im2col(x, c.k, c.stride, c.pad, kpad)

    def run_network(self, ctx, img_nchw):
        """Topology hook: subclasses (engine_hrnet.HRNetEngine) override this."""
        return self.hourglass_net(ctx, img_nchw)

    # ------------------------------------------------------------------ entry points
    def forward(self, img_nchw, training, record_tape, shared_stem=None):
        """shared_stem: optional dict shared between the networks that consume the SAME input batch in one step (FPD:
        student + frozen teacher). The first forward stores the NHWC image and the stem's im2col columns in it, later
        ones reuse them (the caller orders the streams: the producer's forward must have been enqueued first and the
        consumer's stream must wait on it)."""
        ctx = _Ctx()
        ctx.shared_stem = shared_stem
        ctx.training = training
        ctx.sync = self._sync_spec() if training else None
        ctx.passes = precision_passes()
        ctx.tape = [] if record_tape else None
        if training:
            ctx.weights = PreparedWeights(ctx.passes, self.force_apply_sum)
            ctx.affine = None
            self.invalidate_eval_cache()      # this forward rewrites the running statistics on the device
        else:
            w, affine = self._eval_prepared()
            if record_tape:
                w = PreparedWeights(ctx.passes, self.force_apply_sum)
            ctx.weights, ctx.affine = w, affine
        img = img_nchw if (img_nchw.is_contiguous() and img_nchw.dtype == torch.float32) else img_nchw.contiguous().float()
        outs = self.run_network(ctx, img)
        if ctx.nbt:
            torch._foreach_add_(ctx.nbt, 1)
        ctx.outs = outs
        return ctx

    def _sync_spec(self):
        """(process group or None for the default, world size) when SyncBN is on and there is more than one rank."""
        import torch.distributed as dist
        g = self.bn_sync_group
        if g is None and not BN_SYNC:
            return None
        if not (dist.is_available() and dist.is_initialized()):
            return None
        group = None if (g is None or g is True) else g
        world = dist.get_world_size(group)
        return (group, world) if world > 1 else None

    def backward(self, ctx, out_grads_nhwc, wgrad_stream=None):
        """out_grads_nhwc: list (per stack) of NHWC gradient tensors or None. Returns {param: grad}.
        wgrad_stream: optional second CUDA stream for the weight-gradient kernels (joined before returning)."""
        ctx.wgrad_stream = wgrad_stream
        ctx.keepalive = []
        for v, g in zip(ctx.outs, out_grads_nhwc):
            if g is not None:
                v.add_grad(g, owned=False)
        for fn in reversed(ctx.tape):
            fn()
        ctx.tape = None
        if wgrad_stream is not None:
            torch.cuda.current_stream().wait_stream(wgrad_stream)
        ctx.keepalive = []
        return ctx.pgrads


class _Ctx:
    def __init__(self):
        self.training = False
        self._in_s1 = False
        self.sync = None
        self.passes = 3
        self.tape = None
        self.weights = None
        self.affine = None
        self.pgrads = {}
        self.nbt = []
        self.outs = None
        self.wgrad_stream = None
        self.keepalive = []
        self.shared_stem = None
