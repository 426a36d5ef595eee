"""Execution engine for the HRNet pose network: the reference topology (lib/models/pose_hrnet.py:425-460
PoseHighResolutionNet.forward, :247-265 HighResolutionModule.forward, :41-57 BasicBlock, :78-98 Bottleneck) sequenced
over libfpd_b200 kernels, NHWC activations, explicit backward tape (see engine.py for the shared building blocks).

HRNet blocks are post-activation (conv-BN-ReLU ... conv-BN, +skip, ReLU), so besides the hourglass ops the engine needs
 * bn_add_act : y = relu(bn(x) + residual)            -- block tails
 * fuse       : y = relu(sum_j nearest_up_{2^k}(t_j)) -- the multi-resolution exchange
Inside a block the BN+ReLU between two convs is still fused into the consuming conv's operand pass.
"""
import torch

from . import ops
from .engine import Engine, Var, _f32


class HRNetEngine(Engine):
    def __init__(self, net):
        super().__init__(net)
        self.force_apply_sum = True     # bias-free convolutions: dY's 3xFP16 operand scale comes from the BN-backward pass

    def check_input_size(self, H, W):
        """Every size runs: the strided convolutions round odd sizes up, like the reference's."""

    # ------------------------------------------------------------------ extra building blocks
    def bn_add_act(self, ctx, x, bn_name, residual, relu=True):
        aff = self._bn_affine(ctx, x, bn_name)
        if x.data.dtype == residual.data.dtype == torch.float16:     # inference precision "fp16_act"
            out = Var(ops.affine_add_act_f16(x.data, residual.data, aff[0], aff[1], relu, mean=aff[2]))
        else:
            out = Var(ops.affine_add_act(_f32(x.data), _f32(residual.data), aff[0], aff[1], relu, mean=aff[2]))
        if ctx.tape is not None:
            def bwd():
                if out.grad is None:
                    return
                # ReLU of the sum: mask by the stored output, then split to the skip and the BN branch
                dz = ops.affine_act_bwd(out.grad, out.data, None, None, True) if relu else out.grad
                residual.add_grad(dz, owned=False)
                self._bn_backward(ctx, x, bn_name, False, dz, aff)
            ctx.tape.append(bwd)
        return out

    def fuse(self, ctx, terms):
        """terms: list of (Var, log2 upsampling factor). out = relu(sum), pose_hrnet.py:256-263."""
        data, shifts = [t.data for t, _ in terms], [s for _, s in terms]
        if all(d.dtype == torch.float16 for d in data):                # inference precision "fp16_act"
            out = Var(ops.fuse_sum_f16(data, shifts, relu=True))
        else:
            out = Var(ops.fuse_sum([_f32(d) for d in data], shifts, relu=True))
        if ctx.tape is not None:
            def bwd():
                if out.grad is None:
                    return
                dz = ops.affine_act_bwd(out.grad, out.data, None, None, True)
                for t, s in terms:
                    if s == 0:
                        t.add_grad(dz, owned=False)
                    else:
                        t.add_grad(ops.upsample_bwd(dz, s), owned=True)
            ctx.tape.append(bwd)
        return out

    # ------------------------------------------------------------------ blocks
    def _skip(self, ctx, x, prefix):
        if (prefix + ".downsample.0") in self.convs:
            y = self.conv(ctx, x, prefix + ".downsample.0", out_bn=prefix + ".downsample.1")
            return self.bn_act(ctx, y, prefix + ".downsample.1", relu=False)
        return x

    # every HRNet convolution feeds a BatchNorm (post-activation blocks): out_bn lets the conv epilogue carry its statistics
    def basic_block(self, ctx, x, p):
        y = self.conv(ctx, x, p + ".conv1", out_bn=p + ".bn1")
        y = self.conv(ctx, y, p + ".conv2", p + ".bn1", relu=True, out_bn=p + ".bn2")
        return self.bn_add_act(ctx, y, p + ".bn2", self._skip(ctx, x, p))

    def bottleneck_post(self, ctx, x, p):
        y = self.conv(ctx, x, p + ".conv1", out_bn=p + ".bn1")
        y = self.conv(ctx, y, p + ".conv2", p + ".bn1", relu=True, out_bn=p + ".bn2")
        y = self.conv(ctx, y, p + ".conv3", p + ".bn2", relu=True, out_bn=p + ".bn3")
        return self.bn_add_act(ctx, y, p + ".bn3", self._skip(ctx, x, p))

    def block_seq(self, ctx, x, prefix):
        i = 0
        while ("%s.%d.conv1" % (prefix, i)) in self.convs:
            p = "%s.%d" % (prefix, i)
            x = self.bottleneck_post(ctx, x, p) if (p + ".conv3") in self.convs else self.basic_block(ctx, x, p)
            i += 1
        return x

    def conv_bn_chain(self, ctx, x, prefix, relu_last):
        """Sequential of Sequential(conv, BN[, ReLU]) units: `prefix.{k}.0/.1` (transition / fuse down paths)."""
        k = 0
        n = 0
        while ("%s.%d.0" % (prefix, n)) in self.convs:
            n += 1
        for k in range(n):
            x = self.conv(ctx, x, "%s.%d.0" % (prefix, k), out_bn="%s.%d.1" % (prefix, k))
            x = self.bn_act(ctx, x, "%s.%d.1" % (prefix, k), relu=(relu_last or k < n - 1))
        return x

    def hr_module(self, ctx, xs, prefix):
        nb = len(xs)
        xs = [self.block_seq(ctx, xs[b], "%s.branches.%d" % (prefix, b)) for b in range(nb)]
        if nb == 1:
            return xs
        outs = []
        rows = len(self.net.get_submodule(prefix).fuse_layers)   # nb, or 1 for the last module of stage 4
        for i in range(rows):
            terms = []
            for j in range(nb):
                fp = "%s.fuse_layers.%d.%d" % (prefix, i, j)
                if j == i:
                    terms.append((xs[j], 0))
                elif j > i:
                    t = self.conv(ctx, xs[j], fp + ".0", out_bn=fp + ".1")
                    t = self.bn_act(ctx, t, fp + ".1", relu=False)
                    terms.append((t, j - i))
                else:
                    terms.append((self.conv_bn_chain(ctx, xs[j], fp, relu_last=False), 0))
            outs.append(self.fuse(ctx, terms))
        return outs

    def stage(self, ctx, xs, name, n_modules):
        for m in range(n_modules):
            xs = self.hr_module(ctx, xs, "%s.%d" % (name, m))
        return xs

    def transition(self, ctx, prev, name, n_branches):
        xs = []
        for i in range(n_branches):
            tp = "%s.%d" % (name, i)
            # like the reference forward (pose_hrnet.py:432-452) every non-None transition reads the LAST previous
            # branch; None keeps branch i
            if (tp + ".0") in self.convs:          # same resolution, width change: Sequential(conv, BN, ReLU)
                t = self.conv(ctx, prev[-1], tp + ".0", out_bn=tp + ".1")
                xs.append(self.bn_act(ctx, t, tp + ".1", relu=True))
            elif (tp + ".0.0") in self.convs:      # new lower-resolution branch: chain of stride-2 conv+BN+ReLU
                xs.append(self.conv_bn_chain(ctx, prev[-1], tp, relu_last=True))
            else:
                xs.append(prev[i])
        return xs

    # ------------------------------------------------------------------ network
    def run_network(self, ctx, img_nchw):
        net = self.net
        if ctx.shared_stem is not None and ctx.shared_stem.get("img") is img_nchw:
            x = Var(ctx.shared_stem["nhwc"])      # layout conversion done by the caller (shared / W-mirrored image)
        else:
            x = Var(ops.nchw_to_nhwc(img_nchw))
        x = self.conv(ctx, x, "conv1", need_dx=False)
        x = self.bn_act(ctx, x, "bn1", relu=True)
        x = self.conv(ctx, x, "conv2", out_bn="bn2")
        x = self.bn_act(ctx, x, "bn2", relu=True)
        x = self.block_seq(ctx, x, "layer1")
        ys = [x]
        for s, sc in zip((2, 3, 4), net.stage_cfgs):
            xs = self.transition(ctx, ys, "transition%d" % (s - 1), sc["num_branches"])
            ys = self.stage(ctx, xs, "stage%d" % s, sc["num_modules"])
        ctx.head_feature = ys[0]        # the stage-4 high-resolution output final_layer reads (feature distillation)
        return [self.conv(ctx, ys[0], "final_layer", head=True)]
