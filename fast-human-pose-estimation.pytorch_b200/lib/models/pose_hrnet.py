"""HRNet pose network -- drop-in for the reference's lib/models/pose_hrnet.py.

Same public surface (`get_pose_net(cfg, is_train)`, `forward(x[B,3,H,W]) -> Tensor[B,J,H/4,W/4]`, `init_weights`)
and the same `state_dict()` keys/shapes as `PoseHighResolutionNet` (pose_hrnet.py:274-423), so ImageNet-pretrained /
published checkpoints load unchanged. Like the hourglass drop-in the tree only stores parameters (created in the
reference's construction order); the arithmetic runs in fpd_b200.engine_hrnet on libfpd_b200's sm_90a kernels.
`cfg` may be attribute-style or dict-style (the reference mixes both: pose_hrnet.py:278,291).
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


def _bn(ch):
    return nn.BatchNorm2d(ch, momentum=BN_MOMENTUM)


def _conv(cin, cout, k, stride=1, bias=False):
    return nn.Conv2d(cin, cout, kernel_size=k, stride=stride, padding=k // 2, bias=bias)


class _ParamOnly(nn.Module):
    def forward(self, *a, **k):
        raise RuntimeError("%s holds parameters only; run the enclosing PoseHighResolutionNet" % type(self).__name__)


class BasicBlock(_ParamOnly):
    """conv3x3-bn-relu-conv3x3-bn (+skip) -relu; parameter names of pose_hrnet.py:31-39."""
    expansion = 1

    def __init__(self, inplanes, planes, stride=1, downsample=None):
        super().__init__()
        self.conv1 = _conv(inplanes, planes, 3, stride)
        self.bn1 = _bn(planes)
        self.conv2 = _conv(planes, planes, 3)
        self.bn2 = _bn(planes)
        self.downsample = downsample
        self.stride = stride


class Bottleneck(_ParamOnly):
    """1x1-3x3-1x1 post-activation bottleneck, expansion 4; parameter names of pose_hrnet.py:63-76."""
    expansion = 4

    def __init__(self, inplanes, planes, stride=1, downsample=None):
        super().__init__()
        self.conv1 = _conv(inplanes, planes, 1)
        self.bn1 = _bn(planes)
        self.conv2 = _conv(planes, planes, 3, stride)
        self.bn2 = _bn(planes)
        self.conv3 = _conv(planes, planes * self.expansion, 1)
        self.bn3 = _bn(planes * self.expansion)
        self.downsample = downsample
        self.stride = stride


_BLOCKS = {'BASIC': BasicBlock, 'BOTTLENECK': Bottleneck}


def _make_blocks(block, inplanes, planes, nblocks, stride=1):
    """First block may change width (then it carries a 1x1+BN `downsample`), the rest keep it."""
    ds = None
    if stride != 1 or inplanes != planes * block.expansion:
        ds = nn.Sequential(_conv(inplanes, planes * block.expansion, 1, stride), _bn(planes * block.expansion))
    layers = [block(inplanes, planes, stride, ds)]
    width = planes * block.expansion
    layers += [block(width, planes) for _ in range(1, nblocks)]
    return nn.Sequential(*layers), width


class HighResolutionModule(_ParamOnly):
    """Parallel branches + all-to-all fuse layers; names `branches.{b}.{blk}` / `fuse_layers.{i}.{j}...` as in
    pose_hrnet.py:101-242. fuse_layers[i][j]: j>i -> [1x1 conv, BN, (nearest up x2^(j-i))]; j<i -> chain of (i-j)
    stride-2 3x3 conv+BN (+ReLU on all but the last); j==i -> None."""

    def __init__(self, num_branches, block, num_blocks, num_inchannels, num_channels, fuse_method,
                 multi_scale_output=True):
        super().__init__()
        if not (num_branches == len(num_blocks) == len(num_channels) == len(num_inchannels)):
            raise ValueError('NUM_BRANCHES(%d) does not match NUM_BLOCKS/NUM_CHANNELS/NUM_INCHANNELS' % num_branches)
        self.num_branches = num_branches
        self.fuse_method = fuse_method
        self.multi_scale_output = multi_scale_output
        self.num_inchannels = list(num_inchannels)
        branches = []
        for b in range(num_branches):
            seq, width = _make_blocks(block, self.num_inchannels[b], num_channels[b], num_blocks[b])
            self.num_inchannels[b] = width
            branches.append(seq)
        self.branches = nn.ModuleList(branches)
        self.fuse_layers = self._fuse_layers() if num_branches > 1 else None

    def _fuse_layers(self):
        ch = self.num_inchannels
        rows = []
        for i in range(self.num_branches if self.multi_scale_output else 1):
            row = []
            for j in range(self.num_branches):
                if j > i:
                    row.append(nn.Sequential(_conv(ch[j], ch[i], 1), nn.BatchNorm2d(ch[i]),
                                             nn.Upsample(scale_factor=2 ** (j - i), mode='nearest')))
                elif j == i:
                    row.append(None)
                else:
                    chain = []
                    for k in range(i - j):
                        last = k == i - j - 1
                        cout = ch[i] if last else ch[j]
                        mods = [_conv(ch[j], cout, 3, 2), nn.BatchNorm2d(cout)]
                        if not last:
                            mods.append(nn.ReLU(True))
                        chain.append(nn.Sequential(*mods))
                    row.append(nn.Sequential(*chain))
            rows.append(nn.ModuleList(row))
        return nn.ModuleList(rows)

    def get_num_inchannels(self):
        return self.num_inchannels


class PoseHighResolutionNet(nn.Module):
    def __init__(self, cfg, **kwargs):
        super().__init__()
        model = _get(cfg, 'MODEL')
        extra = _get(model, 'EXTRA')
        self.num_joints = int(_get(model, 'NUM_JOINTS'))
        # stem: two stride-2 3x3 convs (pose_hrnet.py:281-287)
        self.conv1 = _conv(3, 64, 3, 2)
        self.bn1 = _bn(64)
        self.conv2 = _conv(64, 64, 3, 2)
        self.bn2 = _bn(64)
        self.layer1, width = _make_blocks(Bottleneck, 64, 64, 4)
        pre = [width]
        self.stage_cfgs = []
        for s in (2, 3, 4):
            scfg = _get(extra, 'STAGE%d' % s)
            block = _BLOCKS[_get(scfg, 'BLOCK')]
            chans = [c * block.expansion for c in _get(scfg, 'NUM_CHANNELS')]
            setattr(self, 'transition%d' % (s - 1), self._transition(pre, chans))
            stage, pre = self._stage(scfg, block, chans, multi_scale_output=(s != 4))
            setattr(self, 'stage%d' % s, stage)
            self.stage_cfgs.append(dict(num_modules=int(_get(scfg, 'NUM_MODULES')),
                                        num_branches=int(_get(scfg, 'NUM_BRANCHES')),
                                        num_blocks=[int(v) for v in _get(scfg, 'NUM_BLOCKS')]))
        k = int(_get(extra, 'FINAL_CONV_KERNEL'))
        self.final_layer = nn.Conv2d(pre[0], self.num_joints, kernel_size=k, stride=1, padding=1 if k == 3 else 0)
        try:
            self.pretrained_layers = _get(extra, 'PRETRAINED_LAYERS')
        except AttributeError:
            self.pretrained_layers = ['*']
        self._engine = None

    @staticmethod
    def _transition(pre, cur):
        layers = []
        for i, c in enumerate(cur):
            if i < len(pre):
                if c != pre[i]:
                    layers.append(nn.Sequential(_conv(pre[i], c, 3), nn.BatchNorm2d(c), nn.ReLU(inplace=True)))
                else:
                    layers.append(None)
            else:
                chain = []
                for j in range(i + 1 - len(pre)):
                    cout = c if j == i - len(pre) else pre[-1]
                    chain.append(nn.Sequential(_conv(pre[-1], cout, 3, 2), nn.BatchNorm2d(cout), nn.ReLU(inplace=True)))
                layers.append(nn.Sequential(*chain))
        return nn.ModuleList(layers)

    @staticmethod
    def _stage(scfg, block, num_inchannels, multi_scale_output=True):
        n_mod = int(_get(scfg, 'NUM_MODULES'))
        mods = []
        for m in range(n_mod):
            mso = multi_scale_output or m != n_mod - 1   # only the last module of stage 4 fuses to branch 0 alone
            mod = HighResolutionModule(int(_get(scfg, 'NUM_BRANCHES')), block, list(_get(scfg, 'NUM_BLOCKS')),
                                       num_inchannels, list(_get(scfg, 'NUM_CHANNELS')), _get(scfg, 'FUSE_METHOD'),
                                       mso)
            num_inchannels = mod.get_num_inchannels()
            mods.append(mod)
        return nn.Sequential(*mods), num_inchannels

    # ---------------------------------------------------------------- execution
    def engine(self):
        if self._engine is None:
            from fpd_b200.engine_hrnet import HRNetEngine
            self._engine = HRNetEngine(self)
        return self._engine

    def forward(self, x):
        dev = self.conv1.weight.device
        if dev.type != "cuda":
            raise RuntimeError("fpd_b200 PoseHighResolutionNet runs on a CUDA (sm_90a) device only; the module is on "
                               "%s. There is no CPU fallback: call .cuda() first." % dev)
        if not x.is_cuda:   # host batch from a DataLoader: stage it like nn.DataParallel's scatter would
            x = x.to(dev, non_blocking=True)
        from fpd_b200 import autograd_bridge
        return autograd_bridge.run(self, x)[0]

    def forward_nhwc(self, x, training=None):
        ctx = self.engine().forward(x, self.training if training is None else training, record_tape=False)
        return [v.data for v in ctx.outs]

    def init_weights(self, pretrained=''):
        """pose_hrnet.py:462-492: N(0, 0.001) convs, unit BN, then an optional partial load of `pretrained`."""
        logger.info('=> init weights from normal distribution')
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.normal_(m.weight, std=0.001)
                if m.bias is not None:
                    nn.init.constant_(m.bias, 0)
            elif isinstance(m, nn.BatchNorm2d):
                nn.init.constant_(m.weight, 1)
                nn.init.constant_(m.bias, 0)
        if os.path.isfile(pretrained):
            state = torch.load(pretrained, map_location='cpu')
            logger.info('=> loading pretrained model %s' % pretrained)
            keep = {k: v for k, v in state.items()
                    if k.split('.')[0] in self.pretrained_layers or self.pretrained_layers[0] == '*'}
            self.load_state_dict(keep, strict=False)
        elif pretrained:
            logger.error('=> please download pre-trained models first!')
            raise ValueError('%s is not exist!' % pretrained)


def get_pose_net(cfg, is_train, **kwargs):
    model = PoseHighResolutionNet(cfg, **kwargs)
    mcfg = _get(cfg, 'MODEL')
    if is_train and _get(mcfg, 'INIT_WEIGHTS'):
        model.init_weights(_get(mcfg, 'PRETRAINED'))
    return model
