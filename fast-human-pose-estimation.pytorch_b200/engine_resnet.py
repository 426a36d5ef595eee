"""Execution engine for the ResNet + deconvolution-head pose network: the reference topology (lib/models/pose_resnet.py:
230-246 PoseResNet.forward, :43-59 BasicBlock, :80-101 Bottleneck, :176-204 the deconv head) sequenced over libfpd_b200
kernels, NHWC activations, explicit backward tape.

The residual blocks are the post-activation ones the HRNet engine already has (engine_hrnet.HRNetEngine.basic_block /
bottleneck_post); new here are
 * the stem pool nn.MaxPool2d(3, 2, 1)                      -> Engine.maxpool3
 * strided blocks: 3x3 stride 2 = stride-1 tensor-core conv + even pick (ConvRef.as_s1), 1x1 stride-2 downsample = even
   pick + stride-1 1x1 (ConvRef.pick_first)
 * 512..2048-channel layers: csrc/conv_wgmma.cu takes them whole, the weight gradients go chunk by chunk
   (ops.conv2d_wgrad_tc_chunked)
 * ConvTranspose2d(k, stride 2) of the head = 3x3 convolution to 4 x Cout channels + depth-to-space (Engine.deconv); the
   BatchNorm + ReLU between two head layers is fused into the consuming convolution's operand pass as everywhere else.
"""
from . import ops
from .engine import Var
from .engine_hrnet import HRNetEngine


class ResNetEngine(HRNetEngine):
    def run_network(self, ctx, img_nchw):
        net = self.net
        if ctx.shared_stem is not None and ctx.shared_stem.get("img") is img_nchw:
            x = Var(ctx.shared_stem["nhwc"])      # layout conversion done by the caller (shared / W-mirrored image)
        else:
            x = Var(ops.nchw_to_nhwc(img_nchw))
        x = self.conv(ctx, x, "conv1", need_dx=False)
        x = self.bn_act(ctx, x, "bn1", relu=True)
        x = self.maxpool3(ctx, x)
        for l in (1, 2, 3, 4):
            x = self.block_seq(ctx, x, "layer%d" % l)
        bn = None
        for i in range(net.num_deconv):
            x = self.deconv(ctx, x, "deconv_layers.%d" % (3 * i), bn, relu=bn is not None)
            bn = "deconv_layers.%d" % (3 * i + 1)
        return [self.conv(ctx, x, "final_layer", bn, relu=bn is not None)]
