"""ResNet + deconvolution-head pose network ("Simple Baselines") -- drop-in for the reference's lib/models/pose_resnet.py.

Same public surface (`get_pose_net(cfg, is_train)`, `forward(x[B,3,H,W]) -> Tensor[B,J,H/4,W/4]`, `init_weights`,
`resnet_spec`) and the same `state_dict()` keys/shapes as `PoseResNet` (pose_resnet.py:98-204), so torchvision ImageNet
ResNet checkpoints (`strict=False`, pose_resnet.py:226-228) and published pose checkpoints load unchanged. Like the other
two drop-ins the tree only stores parameters, created in the reference's construction order; the arithmetic runs in
fpd_b200.engine_resnet on libfpd_b200's sm_90a kernels (the stride-2 transposed convolutions of the head as 3x3
tensor-core convolutions + a depth-to-space shuffle, see Engine.deconv).
"""
import logging
import os

import torch
import torch.nn as nn

BN_MOMENTUM = 0.1
logger = logging.getLogger(__name__)


def _get(node, key):
    try:
        return node[key]
    except (TypeError, KeyError, IndexError):
        return getattr(node, key)


class _ParamOnly(nn.Module):
    def forward(self, *a, **k):
        raise RuntimeError("%s holds parameters only; run the enclosing PoseResNet" % type(self).__name__)


def _bn(ch):
    return nn.BatchNorm2d(ch, momentum=BN_MOMENTUM)


class BasicBlock(_ParamOnly):
    """3x3-bn-relu-3x3-bn (+skip) -relu, stride on the first conv; parameter names of pose_resnet.py:30-41."""
    expansion = 1

    def __init__(self, inplanes, planes, stride=1, downsample=None):
        super().__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, 3, stride, 1, bias=False)
        self.bn1 = _bn(planes)
        self.conv2 = nn.Conv2d(planes, planes, 3, 1, 1, bias=False)
        self.bn2 = _bn(planes)
        self.downsample = downsample
        self.stride = stride


class Bottleneck(_ParamOnly):
    """1x1-3x3-1x1 post-activation bottleneck, expansion 4, stride on the 3x3; parameter names of pose_resnet.py:62-78."""
    expansion = 4

    def __init__(self, inplanes, planes, stride=1, downsample=None):
        super().__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, 1, bias=False)
        self.bn1 = _bn(planes)
        self.conv2 = nn.Conv2d(planes, planes, 3, stride, 1, bias=False)
        self.bn2 = _bn(planes)
        self.conv3 = nn.Conv2d(planes, planes * 4, 1, bias=False)
        self.bn3 = _bn(planes * 4)
        self.downsample = downsample
        self.stride = stride


_DECONV_GEOMETRY = {4: (1, 0), 3: (1, 1), 2: (0, 0)}     # kernel -> (padding, output_padding), pose_resnet.py:162-174


class PoseResNet(nn.Module):
    def __init__(self, block, layers, cfg, **kwargs):
        super().__init__()
        model = _get(cfg, 'MODEL')
        extra = _get(model, 'EXTRA')
        self.deconv_with_bias = bool(_get(extra, 'DECONV_WITH_BIAS'))
        self.num_joints = int(_get(model, 'NUM_JOINTS'))
        self.inplanes = 64
        self.conv1 = nn.Conv2d(3, 64, 7, 2, 3, bias=False)
        self.bn1 = _bn(64)
        for i, (planes, stride) in enumerate(((64, 1), (128, 2), (256, 2), (512, 2))):
            setattr(self, 'layer%d' % (i + 1), self._stack(block, planes, layers[i], stride))
        filters = [int(v) for v in _get(extra, 'NUM_DECONV_FILTERS')]
        kernels = [int(v) for v in _get(extra, 'NUM_DECONV_KERNELS')]
        n = int(_get(extra, 'NUM_DECONV_LAYERS'))
        assert n == len(filters), 'ERROR: num_deconv_layers is different len(num_deconv_filters)'
        assert n == len(kernels), 'ERROR: num_deconv_layers is different len(num_deconv_filters)'
        head = []
        for planes, k in zip(filters, kernels):
            pad, outpad = _DECONV_GEOMETRY[k]
            head += [nn.ConvTranspose2d(self.inplanes, planes, k, stride=2, padding=pad, output_padding=outpad,
                                        bias=self.deconv_with_bias), _bn(planes), nn.ReLU(inplace=True)]
            self.inplanes = planes
        self.deconv_layers = nn.Sequential(*head)
        self.num_deconv = n
        fk = int(_get(extra, 'FINAL_CONV_KERNEL'))
        self.final_layer = nn.Conv2d(self.inplanes, self.num_joints, fk, 1, 1 if fk == 3 else 0)
        self._engine = None

    def _stack(self, block, planes, blocks, stride):
        downsample = None
        if stride != 1 or self.inplanes != planes * block.expansion:
            downsample = nn.Sequential(nn.Conv2d(self.inplanes, planes * block.expansion, 1, stride, bias=False),
                                       _bn(planes * block.expansion))
        seq = [block(self.inplanes, planes, stride, downsample)]
        self.inplanes = planes * block.expansion
        seq += [block(self.inplanes, planes) for _ in range(1, blocks)]
        return nn.Sequential(*seq)

    # ---------------------------------------------------------------- execution
    def engine(self):
        if self._engine is None:
            from fpd_b200.engine_resnet import ResNetEngine
            self._engine = ResNetEngine(self)
        return self._engine

    def forward(self, x):
        dev = self.conv1.weight.device
        if dev.type != "cuda":
            raise RuntimeError("fpd_b200 PoseResNet runs on a CUDA (sm_90a) device only; the module is on %s. There is "
                               "no CPU fallback: call .cuda() first." % dev)
        if not x.is_cuda:   # host batch from a DataLoader: stage it like nn.DataParallel's scatter would
            x = x.to(dev, non_blocking=True)
        from fpd_b200 import autograd_bridge
        return autograd_bridge.run(self, x)[0]

    def forward_nhwc(self, x, training=None):
        ctx = self.engine().forward(x, self.training if training is None else training, record_tape=False)
        return [v.data for v in ctx.outs]

    def init_weights(self, pretrained=''):
        """pose_resnet.py:206-248. With a checkpoint: N(0, 0.001) deconv / final weights, unit BN in the head, then a
        non-strict load (an ImageNet ResNet has no head). Without: N(0, 0.001) on every conv / deconv, unit BN."""
        def head_init(m):
            if isinstance(m, (nn.ConvTranspose2d, nn.Conv2d)):
                nn.init.normal_(m.weight, std=0.001)
            elif isinstance(m, nn.BatchNorm2d):
                nn.init.constant_(m.weight, 1)
                nn.init.constant_(m.bias, 0)
        if os.path.isfile(pretrained):
            logger.info('=> init deconv weights from normal distribution')
            for m in self.deconv_layers.modules():
                head_init(m)
                if isinstance(m, nn.ConvTranspose2d) and self.deconv_with_bias:
                    nn.init.constant_(m.bias, 0)
            logger.info('=> init final conv weights from normal distribution')
            head_init(self.final_layer)
            nn.init.constant_(self.final_layer.bias, 0)
            state = torch.load(pretrained, map_location='cpu')
            logger.info('=> loading pretrained model {}'.format(pretrained))
            self.load_state_dict(state, strict=False)
        else:
            logger.info('=> init weights from normal distribution')
            for m in self.modules():
                head_init(m)        # (conv biases -- only final_layer has one -- keep torch's default, as in the reference)
                if isinstance(m, nn.ConvTranspose2d) and self.deconv_with_bias:
                    nn.init.constant_(m.bias, 0)


resnet_spec = {18: (BasicBlock, [2, 2, 2, 2]),
               34: (BasicBlock, [3, 4, 6, 3]),
               50: (Bottleneck, [3, 4, 6, 3]),
               101: (Bottleneck, [3, 4, 23, 3]),
               152: (Bottleneck, [3, 8, 36, 3])}


def get_pose_net(cfg, is_train, **kwargs):
    mcfg = _get(cfg, 'MODEL')
    block, layers = resnet_spec[int(_get(_get(mcfg, 'EXTRA'), 'NUM_LAYERS'))]
    model = PoseResNet(block, layers, cfg, **kwargs)
    if is_train and _get(mcfg, 'INIT_WEIGHTS'):
        model.init_weights(_get(mcfg, 'PRETRAINED'))
    return model
